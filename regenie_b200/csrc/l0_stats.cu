// f64 sufficient statistics of a genotype block against the covariate basis and phenotypes,
// and the assembly of the per-fold ridge systems.  Together with gram_wgmma.cu this
// replaces Data::residualize_genotypes (reference src/Data.cpp:190-228) and the k-fold branch
// of Data::calc_cv_matrices (src/Data.cpp:735-751) WITHOUT ever materialising the N x bs
// double matrix: with X orthonormal,  G~ = D^-1 (G - (GX) X^T)  so
//   G~_f G~_f^T = D^-1 [ G_f G_f^T - A_f B^T - B A_f^T + B (X_f^T X_f) B^T ] D^-1,
//   G~_f Y_f    = D^-1 [ G_f Y_f - B (X_f^T Y_f) ],     A_f = G_f X_f,  B = sum_f A_f,
// and mean imputation  G = G0 + mu o Miss  expands every product into exact integer Grams
// (tensor cores) plus these skinny f64 reductions.
#include "kernels.cuh"

namespace rg {

constexpr int kStatCols = 16;   // XY columns handled per CTA (register tile)
constexpr int kStatSub = 128;   // samples per shared-memory tile

// grid: (rows_p/128, nchunks, CPp/16); block 128 threads, thread = one SNP row.
__global__ void __launch_bounds__(128)
l0_stats_kernel(const uint32_t* __restrict__ gp, int64_t words_per_row,
                const double* __restrict__ xy, int cpp, const int4* __restrict__ chunks,
                int rows_p, int32_t* __restrict__ cnt_part, double* __restrict__ sum_part) {
  __shared__ double2 tile[kStatSub][kStatCols / 2];
  const int row = blockIdx.x * 128 + threadIdx.x;
  const int4 ch = chunks[blockIdx.y];
  const int col0 = blockIdx.z * kStatCols;
  const uint32_t* grow = gp + (int64_t)row * words_per_row;

  double acc[kStatCols], accm[kStatCols];
#pragma unroll
  for (int c = 0; c < kStatCols; ++c) acc[c] = accm[c] = 0.0;
  int n1 = 0, n2 = 0, nm = 0;

  for (int sub = 0; sub < ch.y; sub += kStatSub) {
    const int t0 = ch.x + sub;
    __syncthreads();
    // cooperative load of xy[t0 .. t0+128)[col0 .. col0+16)
    for (int e = threadIdx.x; e < kStatSub * (kStatCols / 2); e += 128) {
      const int s = e / (kStatCols / 2), c2 = e % (kStatCols / 2);
      tile[s][c2] = *reinterpret_cast<const double2*>(xy + (int64_t)(t0 + s) * cpp + col0 + 2 * c2);
    }
    __syncthreads();
#pragma unroll 1
    for (int wq = 0; wq < kStatSub / 16; ++wq) {
      const uint32_t w = __ldg(grow + (t0 >> 4) + wq);
      if (blockIdx.z == 0) {
        const uint32_t lo = w & 0x55555555u, hi = (w >> 1) & 0x55555555u;
        n1 += __popc(lo & ~hi);
        n2 += __popc(hi & ~lo);
        nm += __popc(hi & lo);
      }
      if (w == 0) continue;
#pragma unroll 4
      for (int k = 0; k < 16; ++k) {
        const uint32_t code = (w >> (2 * k)) & 3u;
        const double g = (code == 3u) ? 0.0 : (double)code;
        const double2* xr = tile[wq * 16 + k];
#pragma unroll
        for (int c2 = 0; c2 < kStatCols / 2; ++c2) {
          const double2 v = xr[c2];
          acc[2 * c2] = fma(g, v.x, acc[2 * c2]);
          acc[2 * c2 + 1] = fma(g, v.y, acc[2 * c2 + 1]);
        }
        if (code == 3u) {
#pragma unroll
          for (int c2 = 0; c2 < kStatCols / 2; ++c2) {
            const double2 v = xr[c2];
            accm[2 * c2] += v.x;
            accm[2 * c2 + 1] += v.y;
          }
        }
      }
    }
  }
  if (blockIdx.z == 0) {
    int4 c4 = make_int4(n1, n2, nm, 0);
    reinterpret_cast<int4*>(cnt_part)[(int64_t)blockIdx.y * rows_p + row] = c4;
  }
  double* o = sum_part + (((int64_t)blockIdx.y * rows_p + row) * 2) * cpp + col0;
#pragma unroll
  for (int c = 0; c < kStatCols; ++c) {
    o[c] = acc[c];
    o[cpp + c] = accm[c];
  }
}

// Fixed-order reduction of chunk partials into per-fold sums (deterministic, no atomics).
// grid: (ceil(rows_p*2*cpp/256), K)
__global__ void l0_fold_reduce_kernel(const int32_t* __restrict__ cnt_part,
                                      const double* __restrict__ sum_part, int rows_p, int cpp,
                                      const int2* __restrict__ fold_chunks,
                                      int32_t* __restrict__ cnt_fold, double* __restrict__ sum_fold) {
  const int f = blockIdx.y;
  const int2 fc = fold_chunks[f];
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t per = (int64_t)rows_p * 2 * cpp;
  if (e < per) {
    double s = 0.0;
    for (int c = fc.x; c < fc.y; ++c) s += sum_part[(int64_t)c * per + e];
    sum_fold[(int64_t)f * per + e] = s;
  }
  if (e < (int64_t)rows_p * 4) {
    int s = 0;
    for (int c = fc.x; c < fc.y; ++c) s += cnt_part[(int64_t)c * rows_p * 4 + e];
    cnt_fold[(int64_t)f * rows_p * 4 + e] = s;
  }
}

// One thread per SNP row: mean, sd, A_f, B, Q_f = (X_f^T X_f) B, per-fold RHS.
// (reference: mean src/Geno.cpp:1749-1757; sd src/Data.cpp:203; low-variance check :205-209)
__global__ void l0_snp_finalize_kernel(SnpFinalizeArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.rows_p) return;
  const int C = a.C, P = a.P, K = a.K, cpp = a.cpp;
  const int64_t per = (int64_t)a.rows_p * 2 * cpp;
  if (i >= a.bs) {
    a.mu[i] = 0.0;
    a.inv_sd[i] = 1.0;
    for (int c = 0; c < C; ++c) a.Bv[(int64_t)i * C + c] = 0.0;
    for (int f = 0; f < K; ++f) {
      for (int c = 0; c < C; ++c) {
        a.Af[((int64_t)f * a.rows_p + i) * C + c] = 0.0;
        a.Qf[((int64_t)f * a.rows_p + i) * C + c] = 0.0;
      }
      for (int p = 0; p < P; ++p) a.rhs[((int64_t)f * a.rows_p + i) * P + p] = 0.0;
    }
    return;
  }
  long long n1 = 0, n2 = 0, nm = 0;
  for (int f = 0; f < K; ++f) {
    const int32_t* c4 = a.cnt_fold + ((int64_t)f * a.rows_p + i) * 4;
    n1 += c4[0]; n2 += c4[1]; nm += c4[2];
  }
  const double mu = (double)(n1 + 2 * n2) / (double)(a.n_analyzed - nm);
  const double ss = (double)(n1 + 4 * n2) + mu * mu * (double)nm;
  // A_f and B
  double b2 = 0.0;
  for (int c = 0; c < C; ++c) {
    double b = 0.0;
    for (int f = 0; f < K; ++f) {
      const double* sf = a.sum_fold + (int64_t)f * per + ((int64_t)i * 2) * cpp;
      const double v = sf[c] + mu * sf[cpp + c];
      a.Af[((int64_t)f * a.rows_p + i) * C + c] = v;
      b += v;
    }
    a.Bv[(int64_t)i * C + c] = b;
    b2 += b * b;
  }
  const double var = (ss - b2) / (double)(a.n_analyzed - C);
  const double sd = sqrt(var);
  if (!(sd >= a.numtol)) atomicMin(a.err_slot, (unsigned long long)(a.err_base + i + 1));
  const double inv_sd = 1.0 / sd;
  a.mu[i] = mu;
  a.inv_sd[i] = inv_sd;
  // Q_f = XtX_f B
  for (int f = 0; f < K; ++f)
    for (int c = 0; c < C; ++c) {
      double q = 0.0;
      for (int c2 = 0; c2 < C; ++c2)
        q += a.XtX_f[((int64_t)f * C + c) * C + c2] * a.Bv[(int64_t)i * C + c2];
      a.Qf[((int64_t)f * a.rows_p + i) * C + c] = q;
    }
  // G~_f Y_f and the out-of-fold right-hand sides  GTY - GtY[f]   (src/Step1_Models.cpp:489)
  for (int p = 0; p < P; ++p) {
    double tot = 0.0;
    for (int f = 0; f < K; ++f) {
      const double* sf = a.sum_fold + (int64_t)f * per + ((int64_t)i * 2) * cpp;
      double v = sf[C + p] + mu * sf[cpp + C + p];
      for (int c = 0; c < C; ++c) v -= a.Bv[(int64_t)i * C + c] * a.XtY_f[((int64_t)f * C + c) * P + p];
      v *= inv_sd;
      a.gty_f[((int64_t)f * a.rows_p + i) * P + p] = v;
      tot += v;
    }
    for (int f = 0; f < K; ++f) {
      const int64_t o = ((int64_t)f * a.rows_p + i) * P + p;
      a.rhs[o] = a.loocv ? tot : tot - a.gty_f[o];
    }
  }
}

// Per-fold Gram of the residualised, scaled genotypes from the exact integer Grams, then the
// K*R shifted ridge systems  (GGt - G_folds[f] + lambda_r I)  in row-major lower storage,
// augmented with the right-hand sides as extra rows (forward substitution for free).
// grid: (nC/32, nC/32), block (32, 8); only tiles with ti >= tj do work.
__global__ void __launch_bounds__(256)
l0_assemble_kernel(AssembleArgs a) {
  const int ti = blockIdx.y, tj = blockIdx.x;
  if (ti < tj) return;
  __shared__ float mgT[32][33];
  const int K = a.K, C = a.C;
  const int j = tj * 32 + threadIdx.x;
  const int64_t ldz = a.ldz;
  double gsum[4] = {0, 0, 0, 0};
  double gf[4][kMaxFolds];
  const double mu_j = a.mu[j], isd_j = a.inv_sd[j];
  for (int f = 0; f < K; ++f) {
    const float* zz = a.zz + (int64_t)f * a.zz_fold_stride;
    __syncthreads();
    // transpose-load MG[j][i] = ZZ[rows_p + j][i] for the (tj rows, ti cols) tile
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int jj = tj * 32 + threadIdx.y * 4 + r;
      mgT[threadIdx.y * 4 + r][threadIdx.x] = zz[(int64_t)(a.rows_p + jj) * ldz + ti * 32 + threadIdx.x];
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int il = threadIdx.y * 4 + r;
      const int i = ti * 32 + il;
      double v = 0.0;
      if (i >= j && i < a.bs) {
        const double mu_i = a.mu[i];
        const double gg = zz[(int64_t)i * ldz + j];
        const double mg_ij = zz[(int64_t)(a.rows_p + i) * ldz + j];
        const double mg_ji = mgT[threadIdx.x][il];
        const double mm = zz[(int64_t)(a.rows_p + i) * ldz + a.rows_p + j];
        double t = gg + mu_i * mg_ij + mu_j * mg_ji + mu_i * mu_j * mm;
        const double* Afi = a.Af + ((int64_t)f * a.rows_p + i) * C;
        const double* Afj = a.Af + ((int64_t)f * a.rows_p + j) * C;
        const double* Qfj = a.Qf + ((int64_t)f * a.rows_p + j) * C;
        const double* Bi = a.Bv + (int64_t)i * C;
        const double* Bj = a.Bv + (int64_t)j * C;
        for (int c = 0; c < C; ++c) t += -Afi[c] * Bj[c] - Bi[c] * Afj[c] + Bi[c] * Qfj[c];
        v = t * a.inv_sd[i] * isd_j;
      }
      gf[r][f] = v;
      gsum[r] += v;
    }
  }
  // write  (GGt - G_f) + lambda_r I  for every (f, r); identity on padded rows
  // (LOOCV: R systems  GGt + lambda_r I  -- no fold is held out of the Gram)
  const int nmat = a.loocv ? a.R : K * a.R;
  for (int m = 0; m < nmat; ++m) {
    const int f = a.loocv ? 0 : m / a.R;
    const double lam = a.lambda[m % a.R];
    double* cm = a.cm + (int64_t)m * a.cm_stride;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int i = ti * 32 + threadIdx.y * 4 + r;
      if (i < j) continue;
      double v;
      if (i < a.bs) {
        v = a.loocv ? gsum[r] : gsum[r] - gf[r][f];
        if (i == j) v += lam;
      } else {
        v = (i == j) ? 1.0 : 0.0;
      }
      cm[(int64_t)i * a.ldc + j] = v;
    }
  }
}


// Mixed-precision solver input (chol_mixed.cu): the K fold systems  A_f = GGt - G_folds[f]  WITHOUT the ridge shift, as
// full symmetric FP64 matrices of dimension n = a.nC (128 * 2^k; rows >= bs carry the identity), so that the refinement
// residual is a plain row-wise matrix-vector pass and the R ridge values of a fold share one matrix.
// a.cm = base of [K][n][n], a.ldc = n.  grid: (n/32, n/32), block (32, 8); tiles with ti >= tj do the work and also
// write the mirror image through shared memory (coalesced both ways).
__global__ void __launch_bounds__(256)
l0_assemble_sym_kernel(AssembleArgs a) {
  const int ti = blockIdx.y, tj = blockIdx.x;
  if (ti < tj) return;
  __shared__ float mgT[32][33];
  __shared__ double tl[32][33];
  const int K = a.K, C = a.C;
  const int j = tj * 32 + threadIdx.x;
  const int64_t ldz = a.ldz;
  double gsum[4] = {0, 0, 0, 0};
  double gf[4][kMaxFolds];
  const bool jv = j < a.bs;
  const double mu_j = jv ? a.mu[j] : 0.0, isd_j = jv ? a.inv_sd[j] : 0.0;
  for (int f = 0; f < K; ++f) {
    const float* zz = a.zz + (int64_t)f * a.zz_fold_stride;
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int jj = tj * 32 + threadIdx.y * 4 + r, ii = ti * 32 + threadIdx.x;
      mgT[threadIdx.y * 4 + r][threadIdx.x] = (jj < a.bs && ii < a.bs) ? zz[(int64_t)(a.rows_p + jj) * ldz + ii] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int il = threadIdx.y * 4 + r;
      const int i = ti * 32 + il;
      double v = 0.0;
      if (i >= j && i < a.bs) {
        const double mu_i = a.mu[i];
        const double gg = zz[(int64_t)i * ldz + j];
        const double mg_ij = zz[(int64_t)(a.rows_p + i) * ldz + j];
        const double mg_ji = mgT[threadIdx.x][il];
        const double mm = zz[(int64_t)(a.rows_p + i) * ldz + a.rows_p + j];
        double t = gg + mu_i * mg_ij + mu_j * mg_ji + mu_i * mu_j * mm;
        const double* Afi = a.Af + ((int64_t)f * a.rows_p + i) * C;
        const double* Afj = a.Af + ((int64_t)f * a.rows_p + j) * C;
        const double* Qfj = a.Qf + ((int64_t)f * a.rows_p + j) * C;
        const double* Bi = a.Bv + (int64_t)i * C;
        const double* Bj = a.Bv + (int64_t)j * C;
        for (int c = 0; c < C; ++c) t += -Afi[c] * Bj[c] - Bi[c] * Afj[c] + Bi[c] * Qfj[c];
        v = t * a.inv_sd[i] * isd_j;
      }
      gf[r][f] = v;
      gsum[r] += v;
    }
  }
  for (int f = 0; f < K; ++f) {
    double* out = a.cm + (int64_t)f * a.cm_stride;
    float* pf = a.planes ? a.planes + (int64_t)f * a.cm_stride : nullptr;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int il = threadIdx.y * 4 + r;
      const int i = ti * 32 + il;
      double v = 0.0;
      if (i >= j) v = (i < a.bs) ? gsum[r] - gf[r][f] : (i == j ? 1.0 : 0.0);
      if (i >= j) {
        out[(int64_t)i * a.ldc + j] = v;
        if (pf) pf[(int64_t)i * a.ldc + j] = (float)v;
        if (a.lplanes && j < 128) {          // block column 0 of every ridge system of this fold: P_i0 = (A_f + lambda_r I)_i0
          for (int r2 = 0; r2 < a.R; ++r2)
            a.lplanes[(int64_t)(f * a.R + r2) * a.cm_stride + (int64_t)i * a.ldc + j] = (float)(i == j ? v + a.lambda[r2] : v);
        }
      }
      tl[il][threadIdx.x] = v;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int jl = threadIdx.y * 4 + r;
      const int i2 = ti * 32 + threadIdx.x, j2 = tj * 32 + jl;
      if (i2 > j2) {
        const double v = tl[threadIdx.x][jl];
        out[(int64_t)j2 * a.ldc + i2] = v;
        if (pf) pf[(int64_t)j2 * a.ldc + i2] = (float)v;
      }
    }
    __syncthreads();
  }
}

// bvec[f][p][i] = rhs_f[i][p]  (zero beyond bs / P).  grid: (ceil(n/256), Pp, K)
__global__ void l0_rhs_sym_kernel(const double* __restrict__ rhs, int rows_p, int bs, int P, int n, double* __restrict__ bvec) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int p = blockIdx.y, f = blockIdx.z;
  if (i >= n) return;
  double v = 0.0;
  if (p < P && i < bs) v = rhs[((int64_t)f * rows_p + i) * P + p];
  bvec[((int64_t)f * gridDim.y + p) * n + i] = v;
}

// Right-hand-side rows of the augmented systems: cm[m][nC + p][i] = rhs_f[i][p].
// grid: (ceil(nC/256), Ppad, nmat)
__global__ void l0_rhs_rows_kernel(AssembleArgs a, const double* __restrict__ rhs, int P) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int p = blockIdx.y, m = blockIdx.z;
  if (i >= a.nC) return;
  const int f = a.loocv ? 0 : m / a.R;
  double v = 0.0;
  if (p < P && i < a.bs) v = rhs[((int64_t)f * a.rows_p + i) * P + p];
  a.cm[(int64_t)m * a.cm_stride + (int64_t)(a.nC + p) * a.ldc + i] = v;
}

void launch_l0_stats(const uint32_t* gp, int64_t npad, const double* xy, int cpp, const int4* chunks,
                     int nchunks, int rows_p, int32_t* cnt_part, double* sum_part, cudaStream_t s) {
  dim3 grid(rows_p / 128, nchunks, cpp / kStatCols);
  l0_stats_kernel<<<grid, 128, 0, s>>>(gp, npad / 16, xy, cpp, chunks, rows_p, cnt_part, sum_part);
}

void launch_l0_fold_reduce(const int32_t* cnt_part, const double* sum_part, int rows_p, int cpp,
                           const int2* fold_chunks, int K, int32_t* cnt_fold, double* sum_fold,
                           cudaStream_t s) {
  const int64_t per = (int64_t)rows_p * 2 * cpp;
  dim3 grid((unsigned)ceil_div(per, 256), K);
  l0_fold_reduce_kernel<<<grid, 256, 0, s>>>(cnt_part, sum_part, rows_p, cpp, fold_chunks, cnt_fold, sum_fold);
}

void launch_l0_snp_finalize(const SnpFinalizeArgs& a, cudaStream_t s) {
  l0_snp_finalize_kernel<<<(unsigned)ceil_div(a.rows_p, 128), 128, 0, s>>>(a);
}

void launch_l0_assemble(const AssembleArgs& a, const double* rhs, int P, int Ppad, int nmat, cudaStream_t s) {
  dim3 grid(a.nC / 32, a.nC / 32);
  l0_assemble_kernel<<<grid, dim3(32, 8), 0, s>>>(a);
  dim3 g2((unsigned)ceil_div(a.nC, 256), Ppad, nmat);
  l0_rhs_rows_kernel<<<g2, 256, 0, s>>>(a, rhs, P);
}

void launch_l0_assemble_sym(const AssembleArgs& a, const double* rhs, int P, int Pp, double* bvec, cudaStream_t s) {
  // (a fold-unrolled variant with every per-fold value in registers and one barrier for all transposed tiles measured
  // slower under lane overlap: 128 registers, 2 CTAs per SM)
  dim3 grid(a.nC / 32, a.nC / 32);
  l0_assemble_sym_kernel<<<grid, dim3(32, 8), 0, s>>>(a);
  dim3 g2((unsigned)ceil_div(a.nC, 256), Pp, a.K);
  l0_rhs_sym_kernel<<<g2, 256, 0, s>>>(rhs, a.rows_p, a.bs, P, a.nC, bvec);
}

}  // namespace rg
