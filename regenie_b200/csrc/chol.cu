// Batched FP64 Cholesky solve of the shifted ridge systems  (A_f + lambda_r I) beta = b_f.
//
// The reference diagonalises  GGt - G_folds[f]  once per fold with SelfAdjointEigenSolver and
// applies  V (D + lambda_r I)^-1 V^T  (src/Step1_Models.cpp:484-494; level 1: :828-835).  On
// the GPU an eigendecomposition is latency-bound; the same vectors come from K*R independent
// Cholesky factorisations (n^3/3 flops each, all batched), identical to ~1e-12 relative.
//
// Storage: row-major lower triangle, ld = nC (multiple of 64); matrix m occupies
// cm + m*stride; rows nC .. nC+Ppad-1 hold the right-hand sides as extra rows, so the
// factorisation sweep leaves  y^T = (L^-1 b)^T  there (fused forward substitution).
//
// 64-column panels, two launches per panel step:
//   chol_diag        : one CTA per system factors the (already updated) diagonal tile in registers and also produces
//                      M = L_kk^-T and M^T (the same column sweep applied to I)
//   chol_update_trsm : every row tile below the panel does, on the FP64 tensor pipe (DMMA), the left-looking update
//                      P = A[rows, k:k+64] - L[rows,0:k] L[k:k+64,0:k]^T  (the n^3/3 flops), the triangular solve as a
//                      GEMM  L[rows, k:k+64] = P M,  and the rank-64 update of its OWN diagonal tile with the block it
//                      just produced - so no serial "update the diagonal tile" launch precedes a factorisation.
// No CTA ever reads a tile that another CTA of the same launch overwrites: kernels of several
// "lanes" run concurrently, so launch-wide lockstep cannot be assumed.
// The stored inverses M also turn the backward substitution's triangular solves into GEMVs.
#include "gemm_dmma.cuh"
#include "kernels.cuh"

namespace rg {

constexpr int TB = 64;  // tile / panel width

// Row tiles strictly below the panel: update AND triangular solve in one pass,
//   P = A[r0:r0+64, k:k+64] - L[r0:, 0:k] L[k:, 0:k]^T,   L[r0:, k:k+64] = P M,   M = L_kk^-T  (both products on the DMMA pipe).
// The updated tile makes one trip through the CTA's own global tile (L1/L2 resident) instead of a separate kernel.
// grid: (row tiles below the panel, 1, batch); 256 threads.
constexpr int PS_LD = TB + 4;                                   // row stride of the staged tile (16-byte aligned rows)
constexpr size_t kFusedSmem = ((size_t)2 * TB * DM_LD + (size_t)TB * PS_LD) * sizeof(double);

__global__ void __launch_bounds__(256)
chol_update_trsm_kernel(double* __restrict__ cm, int64_t stride, int ld, int k, int tile0,
                        const double* __restrict__ inv_t, int64_t inv_stride) {
  extern __shared__ double fused_sm[];
  double* As = fused_sm;
  double* Bs = fused_sm + TB * DM_LD;
  double* Ps = fused_sm + 2 * TB * DM_LD;                       // the updated tile, then the solved tile: no global round trip
  double* A = cm + (int64_t)blockIdx.z * stride;
  const double* MT = inv_t + (int64_t)blockIdx.z * inv_stride + (int64_t)(k / TB) * TB * TB;
  const int r0 = (tile0 + 1 + blockIdx.x) * TB;
  DmmaAcc acc;
  gemm_tile_nt_dmma(A + (int64_t)r0 * ld, ld, true, A + (int64_t)k * ld, ld, true, k, acc, As, Bs);   // zero when k == 0
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const double2 v = *reinterpret_cast<const double2*>(A + (int64_t)(r0 + dm_row(i)) * ld + k + dm_col(j));
      *reinterpret_cast<double2*>(Ps + dm_row(i) * PS_LD + dm_col(j)) = make_double2(v.x - acc.c[i][j][0], v.y - acc.c[i][j][1]);
    }
  __syncthreads();
  gemm_tile_nt_dmma(Ps, PS_LD, true, MT, TB, true, TB, acc, As, Bs);                                  // L = P M
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const double2 v = make_double2(acc.c[i][j][0], acc.c[i][j][1]);
      *reinterpret_cast<double2*>(A + (int64_t)(r0 + dm_row(i)) * ld + k + dm_col(j)) = v;
      *reinterpret_cast<double2*>(Ps + dm_row(i) * PS_LD + dm_col(j)) = v;
    }
  // keep this row tile's own diagonal block up to date (right-looking for the diagonal blocks only):
  //   A[r0:, r0:] -= L[r0:, k:k+64] L[r0:, k:k+64]^T
  // so a panel step starts with the factorisation of an already updated diagonal tile - no serial update launch.
  if (r0 < ld) {
    __syncthreads();
    gemm_tile_nt_dmma(Ps, PS_LD, true, Ps, PS_LD, true, TB, acc, As, Bs);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        double2* o = reinterpret_cast<double2*>(A + (int64_t)(r0 + dm_row(i)) * ld + r0 + dm_col(j));
        double2 v = *o;
        v.x -= acc.c[i][j][0];
        v.y -= acc.c[i][j][1];
        *o = v;
      }
  }
}

// Diagonal tile: L_kk = chol(P_kk) and M = L_kk^-T, both in registers (thread (r, q) holds the
// columns q+4j of row r); one barrier per column, pivots broadcast through a double buffer.
// grid: (batch); 256 threads.
__global__ void __launch_bounds__(256)
chol_diag_kernel(double* __restrict__ cm, int64_t stride, int ld, int k,
                 double* __restrict__ inv, double* __restrict__ inv_t, int64_t inv_stride,
                 unsigned long long* __restrict__ err_slot, long long err_base) {
  __shared__ double cb[2][TB], xb[2][TB];
  double* A = cm + (int64_t)blockIdx.x * stride;
  const int r = threadIdx.x & (TB - 1), q = threadIdx.x >> 6;
  double D[16], T[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int cc = q + 4 * j;
    D[j] = (cc <= r) ? A[(int64_t)(k + r) * ld + k + cc] : 0.0;
    T[j] = (cc == r) ? 1.0 : 0.0;
  }
  bool bad = false;
#pragma unroll
  for (int jc = 0; jc < 16; ++jc) {
#pragma unroll
    for (int qc = 0; qc < 4; ++qc) {
      const int c = 4 * jc + qc;
      const int buf = c & 1;
      if (q == qc) { cb[buf][r] = D[jc]; xb[buf][r] = T[jc]; }
      __syncthreads();      // one barrier per column: the other buffer is only rewritten after the next barrier
      const double piv = cb[buf][c];
      if (!(piv > 0.0)) bad = true;
      // 1/sqrt from the FP32 unit + two Newton steps in FP64 (full double accuracy, shorter dependent chain than rsqrt())
      double inv_p = (double)rsqrtf((float)piv);
      inv_p = inv_p * (1.5 - 0.5 * piv * inv_p * inv_p);
      inv_p = inv_p * (1.5 - 0.5 * piv * inv_p * inv_p);
      const double lr = cb[buf][r] * inv_p;      // L[r][c]  (meaningful for r >= c)
      const double xr = xb[buf][r] * inv_p;      // X[r][c] = (L^-T)[r][c]
      if (q == qc) { D[jc] = (r >= c) ? lr : 0.0; T[jc] = xr; }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        if (j > jc || (j == jc && q > qc)) {      // columns cc > c
          const int cc = q + 4 * j;
          const double lcc = cb[buf][cc] * inv_p;
          if (r >= cc) D[j] = fma(-lr, lcc, D[j]);
          T[j] = fma(-xr, lcc, T[j]);
        }
      }
    }
  }
  if (bad && threadIdx.x == 0) atomicMin(err_slot, (unsigned long long)(err_base + blockIdx.x + 1));
  double* Mo = inv + (int64_t)blockIdx.x * inv_stride + (int64_t)(k / TB) * TB * TB;
  double* MTo = inv_t + (int64_t)blockIdx.x * inv_stride + (int64_t)(k / TB) * TB * TB;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int cc = q + 4 * j;
    if (cc <= r) A[(int64_t)(k + r) * ld + k + cc] = D[j];
    Mo[r * TB + cc] = (cc >= r) ? T[j] : 0.0;
    MTo[cc * TB + r] = (cc >= r) ? T[j] : 0.0;        // M^T, the "NT" operand of the fused update + solve
  }
}

// Backward substitution  L^T beta = y  for all right-hand sides, sweeping 64-column blocks from
// the last to the first.  y lives in the RHS rows (row nC+p, contiguous over columns); beta
// overwrites it.  The diagonal solves are GEMVs with the stored M = L_kk^-T; the sweep
// y[:, j] -= L[k+r][j] beta[r]  streams the 64 panel rows once.
// grid: (batch, ceil(P / BS_RHS)): one CTA per matrix and group of at most BS_RHS right-hand sides, so the shared
// memory is bounded whatever the trait count; every right-hand side goes through the same arithmetic in any group.
constexpr int BS_THREADS = 256;
constexpr int BS_JT = 2;        // columns per thread in the sweep (two batches of rows are held in registers)
constexpr int BS_PC = 10;   // right-hand sides per register pass
constexpr int BS_RHS = 64;  // right-hand sides per CTA

__global__ void __launch_bounds__(BS_THREADS)
chol_backsolve_kernel(double* __restrict__ cm, int64_t stride, int ld, int nC, int P_all,
                      const double* __restrict__ inv, int64_t inv_stride) {
  extern __shared__ double back_sm[];
  const int P = min(BS_RHS, P_all - (int)blockIdx.y * BS_RHS);   // right-hand sides of this CTA
  double* Ms = back_sm;                    // [TB][TB+1]
  double* ys = Ms + TB * (TB + 1);         // [TB][P]  y block
  double* bs = ys + TB * P;                // [TB][P]  beta block
  double* A = cm + (int64_t)blockIdx.x * stride;
  double* Y = A + (int64_t)(nC + blockIdx.y * BS_RHS) * ld;     // this CTA's right-hand-side rows
  const double* Minv = inv + (int64_t)blockIdx.x * inv_stride;
  for (int kb = nC / TB - 1; kb >= 0; --kb) {
    const int k = kb * TB;
    __syncthreads();
    for (int e = threadIdx.x; e < TB * TB; e += BS_THREADS)
      Ms[(e / TB) * (TB + 1) + (e % TB)] = Minv[(int64_t)kb * TB * TB + e];
    for (int e = threadIdx.x; e < TB * P; e += BS_THREADS) {
      const int r = e % TB, p = e / TB;
      ys[r * P + p] = Y[(int64_t)p * ld + k + r];
    }
    __syncthreads();
    // beta = L_kk^-T y = M y   (M upper triangular: M[r][c], c >= r)
    for (int e = threadIdx.x; e < TB * P; e += BS_THREADS) {
      const int r = e % TB, p = e / TB;
      double s = 0.0;
      for (int c = r; c < TB; ++c) s = fma(Ms[r * (TB + 1) + c], ys[c * P + p], s);
      bs[r * P + p] = s;
      Y[(int64_t)p * ld + k + r] = s;
    }
    __syncthreads();
    // y[p][j] -= sum_r L[k+r][j] * beta[r][p]   for all j < k   (coalesced over j; each thread owns BS_JT columns).
    // The 64 panel rows are streamed in batches of 8 with the next batch already in flight (software pipelining):
    // one CTA per system has little else to hide the HBM latency with.
    for (int j0 = threadIdx.x; j0 < k; j0 += BS_THREADS * BS_JT) {
      for (int p0 = 0; p0 < P; p0 += BS_PC) {
        const int np = min(BS_PC, P - p0);
        double acc[BS_JT][BS_PC];
#pragma unroll
        for (int m = 0; m < BS_JT; ++m)
#pragma unroll
          for (int qq = 0; qq < BS_PC; ++qq) acc[m][qq] = 0.0;
        double l[BS_JT][8], ln[BS_JT][8];
#pragma unroll
        for (int m = 0; m < BS_JT; ++m) {
          const int j = j0 + m * BS_THREADS;
#pragma unroll
          for (int u = 0; u < 8; ++u) l[m][u] = (j < k) ? A[(int64_t)(k + u) * ld + j] : 0.0;
        }
#pragma unroll 1
        for (int rb = 0; rb < TB; rb += 8) {
          if (rb + 8 < TB) {
#pragma unroll
            for (int m = 0; m < BS_JT; ++m) {
              const int j = j0 + m * BS_THREADS;
#pragma unroll
              for (int u = 0; u < 8; ++u) ln[m][u] = (j < k) ? A[(int64_t)(k + rb + 8 + u) * ld + j] : 0.0;
            }
          }
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const double* bb = bs + (rb + u) * P + p0;
#pragma unroll
            for (int qq = 0; qq < BS_PC; ++qq) {
              const double bv = (qq < np) ? bb[qq] : 0.0;
#pragma unroll
              for (int m = 0; m < BS_JT; ++m) acc[m][qq] = fma(l[m][u], bv, acc[m][qq]);
            }
          }
#pragma unroll
          for (int m = 0; m < BS_JT; ++m)
#pragma unroll
            for (int u = 0; u < 8; ++u) l[m][u] = ln[m][u];
        }
#pragma unroll
        for (int m = 0; m < BS_JT; ++m) {
          const int j = j0 + m * BS_THREADS;
          if (j < k)
#pragma unroll
            for (int qq = 0; qq < BS_PC; ++qq)
              if (qq < np) Y[(int64_t)(p0 + qq) * ld + j] -= acc[m][qq];
        }
      }
    }
  }
}

void launch_chol_factor(double* cm, int64_t stride, int nC, int n_aug, int batch, double* inv,
                        unsigned long long* err_slot, long long err_base, cudaStream_t s) {
  const int ntiles = n_aug / TB;
  const int64_t inv_stride = (int64_t)(nC / TB) * TB * TB;
  ensure_dyn_smem(reinterpret_cast<const void*>(chol_update_trsm_kernel), kFusedSmem);
  double* inv_t = inv + (int64_t)batch * inv_stride;      // M^T blocks live behind the M blocks (chol_inv_elems)
  for (int kb = 0; kb < nC / TB; ++kb) {
    const int k = kb * TB;
    chol_diag_kernel<<<batch, 256, 0, s>>>(cm, stride, nC, k, inv, inv_t, inv_stride, err_slot, err_base);
    dim3 g2(ntiles - kb - 1, 1, batch);
    if (ntiles - kb - 1 > 0) chol_update_trsm_kernel<<<g2, 256, kFusedSmem, s>>>(cm, stride, nC, k, kb, inv_t, inv_stride);
  }
}

void launch_chol_backsolve(double* cm, int64_t stride, int nC, int P, int batch, const double* inv,
                           cudaStream_t s) {
  const size_t smem = ((size_t)TB * (TB + 1) + (size_t)2 * TB * std::min(P, BS_RHS)) * sizeof(double);
  ensure_dyn_smem(reinterpret_cast<const void*>(chol_backsolve_kernel), smem);
  const int64_t inv_stride = (int64_t)(nC / TB) * TB * TB;
  chol_backsolve_kernel<<<dim3(batch, (unsigned)ceil_div(P, BS_RHS)), BS_THREADS, smem, s>>>(cm, stride, nC, nC, P, inv, inv_stride);
}

int chol_num_launches(int nC) { return 2 * (nC / TB); }
size_t chol_inv_elems(int nC, int batch) { return (size_t)2 * batch * (nC / TB) * TB * TB; }   // M and M^T

}  // namespace rg

namespace rg {

// Row-wise backward substitution for MANY right-hand sides stored as rows (LOOCV):
//   rows hold t_i^T = (L^-1 w_i)^T;  on exit they hold z_i^T = t_i^T L^-1 = (L^-T t_i)^T = (H w_i)^T.
// grid: (row tiles, 1, batch); one CTA owns 64 rows and sweeps the column blocks from last to first:
//   z_kb = t_kb * L_kk^-1 (= t_kb * M^T),   t[:, 0:k] -= z_kb * L[k:k+64, 0:k].
__global__ void __launch_bounds__(256)
chol_rows_backsolve_kernel(double* __restrict__ cm, int64_t stride, int ld, int nC, int row0,
                           const double* __restrict__ inv, int64_t inv_stride) {
  extern __shared__ double rb_sm[];
  double (*Zs)[TB + 1] = reinterpret_cast<double (*)[TB + 1]>(rb_sm);                     // z_kb / t_kb tile
  double (*Ls)[TB + 2] = reinterpret_cast<double (*)[TB + 2]>(rb_sm + TB * (TB + 1));     // M or an L tile
  double* A = cm + (int64_t)blockIdx.z * stride;
  const double* Minv = inv + (int64_t)blockIdx.z * inv_stride;
  const int r0 = row0 + blockIdx.x * TB;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  for (int kb = nC / TB - 1; kb >= 0; --kb) {
    const int k = kb * TB;
    __syncthreads();
    for (int e = threadIdx.x; e < TB * TB; e += 256) {
      const int rr = e / TB, cc = e % TB;
      Zs[rr][cc] = A[(int64_t)(r0 + rr) * ld + k + cc];
      Ls[rr][cc] = Minv[(int64_t)kb * TB * TB + e];          // M[c][p] at Ls[c][p]
    }
    __syncthreads();
    // z[row][c] = sum_p t[row][p] * M[c][p]
    double z[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) z[a][b] = 0.0;
#pragma unroll 8
    for (int p = 0; p < TB; ++p) {
      double av[4], bv[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) av[a] = Zs[ty * 4 + a][p];
#pragma unroll
      for (int b = 0; b < 4; ++b) bv[b] = Ls[tx + 16 * b][p];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) z[a][b] = fma(av[a], bv[b], z[a][b]);
    }
    __syncthreads();
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        Zs[ty * 4 + a][tx + 16 * b] = z[a][b];
        A[(int64_t)(r0 + ty * 4 + a) * ld + k + tx + 16 * b] = z[a][b];
      }
    // t[:, j0:j0+64] -= z_kb * L[k:k+64, j0:j0+64]
    for (int j0 = 0; j0 < k; j0 += TB) {
      __syncthreads();
      for (int e = threadIdx.x; e < TB * TB; e += 256) {
        const int rr = e / TB, cc = e % TB;
        Ls[rr][cc] = A[(int64_t)(k + rr) * ld + j0 + cc];    // L[k+p][j0+c] at Ls[p][c]
      }
      __syncthreads();
      double u[4][4];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) u[a][b] = 0.0;
#pragma unroll 8
      for (int p = 0; p < TB; ++p) {
        double av[4], bv[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) av[a] = Zs[ty * 4 + a][p];
#pragma unroll
        for (int b = 0; b < 4; ++b) bv[b] = Ls[p][tx + 16 * b];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int b = 0; b < 4; ++b) u[a][b] = fma(av[a], bv[b], u[a][b]);
      }
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) A[(int64_t)(r0 + ty * 4 + a) * ld + j0 + tx + 16 * b] -= u[a][b];
    }
  }
}

void launch_chol_rows_backsolve(double* cm, int64_t stride, int nC, int row0, int nrows, int batch,
                                const double* inv, cudaStream_t s) {
  const size_t smem = ((size_t)TB * (TB + 1) + (size_t)TB * (TB + 2)) * sizeof(double);
  ensure_dyn_smem(reinterpret_cast<const void*>(chol_rows_backsolve_kernel), smem);
  const int64_t inv_stride = (int64_t)(nC / TB) * TB * TB;
  dim3 grid(nrows / TB, 1, batch);
  chol_rows_backsolve_kernel<<<grid, 256, smem, s>>>(cm, stride, nC, nC, row0, inv, inv_stride);
}

}  // namespace rg
