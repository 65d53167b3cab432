// Level-1 ridge over the stacked level-0 predictors (k-fold CV) and per-chromosome predictions.
// Replaces ridge_level_1 (reference src/Step1_Models.cpp:772-872) and the arithmetic of
// Data::make_predictions (src/Data.cpp:1238-1254).  W is real valued, so this stage is FP64
// throughout: X_folds[f] = W_f^T W_f is an FP64 GEMM over the sample axis (K = fold samples),
// the K*R1 shifted systems go through the same batched Cholesky as level 0.
#include "gemm_dmma.cuh"
#include "kernels.cuh"

namespace rg {

constexpr int LT = 64;   // output tile

// Partial Gram of one sample chunk: part[chunk][i][j] = sum_{t in chunk} W[t,i] W[t,j], i >= j tiles.
// grid: (B tiles j, B tiles i, nchunks); 256 threads, FP64 tensor pipe (DMMA) over the sample axis.
__global__ void __launch_bounds__(256)
l1_gram_kernel(const double* __restrict__ W, int64_t ldw, int B, const int4* __restrict__ chunks,
               double* __restrict__ part, int64_t part_stride, int ldp) {
  const int tj = blockIdx.x, ti = blockIdx.y;
  if (tj > ti) return;
  __shared__ double As[LT * DM_LD];
  __shared__ double Bs[LT * DM_LD];
  const int4 ch = chunks[blockIdx.z];
  const int lrow = threadIdx.x >> 2;
  const int ia = ti * LT + lrow, ib = tj * LT + lrow;
  const bool va = ia < B, vb = ib < B;
  // rows of the "NT" product are the COLUMNS of W (contiguous over samples)
  const double* abase = W + (int64_t)(ti * LT) * ldw + ch.x;
  const double* bbase = W + (int64_t)(tj * LT) * ldw + ch.x;
  DmmaAcc acc;
  gemm_tile_nt_dmma(abase, ldw, va, bbase, ldw, vb, ch.y, acc, As, Bs);
  double* o = part + (int64_t)blockIdx.z * part_stride;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int ii = ti * LT + dm_row(i), jj = tj * LT + dm_col(j) + e;
        if (ii < B && jj < B) o[(int64_t)ii * ldp + jj] = acc.c[i][j][e];
      }
}

// W_chunk^T y partials: part_y[chunk][i].  grid: (B, nchunks), block 128, fixed-order reduction.
__global__ void __launch_bounds__(128)
l1_xty_kernel(const double* __restrict__ W, int64_t ldw, const double* __restrict__ xy, int cpp, int ycol,
              const int4* __restrict__ chunks, double* __restrict__ part_y, int B) {
  __shared__ double red[128];
  const int i = blockIdx.x;
  const int4 ch = chunks[blockIdx.y];
  double s = 0.0;
  for (int t = threadIdx.x; t < ch.y; t += 128)
    s += W[(int64_t)i * ldw + ch.x + t] * xy[(int64_t)(ch.x + t) * cpp + ycol];
  s = cta_tree<128>(s, red);
  if (threadIdx.x == 0) part_y[(int64_t)blockIdx.y * B + i] = s;
}

// Sum chunk partials per fold (fixed order), form  XtX_sum - X_folds[f] + tau_j I  and the P right-hand sides
// XtY_sum - XtY[f]  in the batched Cholesky layout (row-major lower, RHS rows nC .. nC + P - 1); LOOCV (K = 1): nothing
// is held out.  part: [nchunks][nC x ldp] lower tiles; part_y: [P][nchunks][B], right-hand side p at p * part_y_stride.
// Level 1 (P = 1) and the dense level-0 route (P traits, tau = lambda, B = bs).
// grid: (ceil(nC/128), nC + P), block 128: thread = (j, row i); rows >= nC are right-hand sides.
__global__ void l1_assemble_kernel(const double* __restrict__ part, int64_t part_stride, int ldp,
                                   const double* __restrict__ part_y, int64_t part_y_stride,
                                   const int2* __restrict__ fold_chunks, int K, int R1, const double* __restrict__ tau,
                                   int B, int nC, double* __restrict__ cm, int64_t cm_stride, int loocv) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y;
  if (j >= nC) return;
  const bool is_rhs = i >= nC;
  if (!is_rhs && j > i) return;
  const int p = i - nC;
  const bool real = is_rhs ? (j < B) : (i < B);
  double fold_v[kMaxFolds];
  double tot = 0.0;
  for (int f = 0; f < K; ++f) {
    double s = 0.0;
    if (real) {
      const int2 fc = fold_chunks[f];
      for (int c = fc.x; c < fc.y; ++c)
        s += is_rhs ? part_y[(int64_t)p * part_y_stride + (int64_t)c * B + j] : part[(int64_t)c * part_stride + (int64_t)i * ldp + j];
    }
    fold_v[f] = s;
    tot += s;
  }
  for (int f = 0; f < K; ++f)
    for (int r = 0; r < R1; ++r) {
      double v;
      if (real) {
        v = loocv ? tot : tot - fold_v[f];
        if (!is_rhs && i == j) v += tau[r];
      } else {
        v = (!is_rhs && i == j) ? 1.0 : 0.0;
      }
      cm[(int64_t)(f * R1 + r) * cm_stride + (int64_t)i * nC + j] = v;
    }
}

// p1 = W_f beta_f for every tau, and the CV sums Sx, Sy, Sx2, Sy2, Sxy (src/Step1_Models.cpp:847-852).
// grid: (Npad/128); block 128: thread = sample.  part_out[tile][R1][3] + [tile][2] for y.
__global__ void __launch_bounds__(128)
l1_pred_sums_kernel(const double* __restrict__ W, int64_t ldw, int B, int R1,
                    const double* __restrict__ beta /*[K][R1][ldb]*/, int ldb,
                    const int32_t* __restrict__ tile_fold, const double* __restrict__ xy, int cpp, int ycol,
                    double* __restrict__ part_out) {
  extern __shared__ double sb[];            // beta chunk [R1][256]
  __shared__ double red[4][kMaxRidge * 3 + 2];
  const int t = blockIdx.x * 128 + threadIdx.x;
  const int f = tile_fold[blockIdx.x];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double p1[kMaxRidge];
#pragma unroll
  for (int r = 0; r < kMaxRidge; ++r) p1[r] = 0.0;
  for (int c0 = 0; c0 < B; c0 += 256) {
    const int nc = min(256, B - c0);
    __syncthreads();
    for (int e = threadIdx.x; e < R1 * nc; e += 128) {
      const int r = e / nc, c = e - r * nc;
      sb[r * 256 + c] = beta[((int64_t)f * R1 + r) * ldb + c0 + c];
    }
    __syncthreads();
    for (int c = 0; c < nc; ++c) {
      const double w = W[(int64_t)(c0 + c) * ldw + t];
#pragma unroll
      for (int r = 0; r < kMaxRidge; ++r)
        if (r < R1) p1[r] = fma(w, sb[r * 256 + c], p1[r]);
    }
  }
  const double y = xy[(int64_t)t * cpp + ycol];
  double vals[kMaxRidge * 3 + 2];
#pragma unroll
  for (int r = 0; r < kMaxRidge; ++r) {
    vals[3 * r] = p1[r]; vals[3 * r + 1] = p1[r] * p1[r]; vals[3 * r + 2] = p1[r] * y;
  }
  vals[kMaxRidge * 3] = y; vals[kMaxRidge * 3 + 1] = y * y;
#pragma unroll
  for (int v = 0; v < kMaxRidge * 3 + 2; ++v) {
    double s = vals[v];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[warp][v] = s;
  }
  __syncthreads();
  if (threadIdx.x < kMaxRidge * 3 + 2) {
    const int v = threadIdx.x;
    part_out[(int64_t)blockIdx.x * (kMaxRidge * 3 + 2) + v] = ((red[0][v] + red[1][v]) + red[2][v]) + red[3][v];
  }
}

// Per-chromosome predictions for the selected tau (src/Data.cpp:1246-1251):
//   pred[t][chr] = W_f[t, cols(chr)] . beta_f[cols(chr), best]
// grid: (Npad/128); thread = sample; chr_col_start[nchr+1] are column offsets in chromosome order.
__global__ void __launch_bounds__(128)
l1_chr_pred_kernel(const double* __restrict__ W, int64_t ldw, int nchr, const int32_t* __restrict__ chr_col_start,
                   const double* __restrict__ beta, int ldb, int R1, int best,
                   const int32_t* __restrict__ tile_fold, double* __restrict__ pred, int64_t npad) {
  const int t = blockIdx.x * 128 + threadIdx.x;
  const int f = tile_fold[blockIdx.x];
  const double* bf = beta + ((int64_t)f * R1 + best) * ldb;
  for (int ci = 0; ci < nchr; ++ci) {
    double s = 0.0;
    for (int c = chr_col_start[ci]; c < chr_col_start[ci + 1]; ++c) s = fma(W[(int64_t)c * ldw + t], __ldg(bf + c), s);
    pred[(int64_t)ci * npad + t] = s;
  }
}

void launch_l1_gram(const double* W, int64_t ldw, int B, const int4* chunks, int nchunks, double* part,
                    int64_t part_stride, int ldp, cudaStream_t s) {
  const int nt = (int)ceil_div(B, LT);
  dim3 grid(nt, nt, nchunks);
  l1_gram_kernel<<<grid, 256, 0, s>>>(W, ldw, B, chunks, part, part_stride, ldp);
}

void launch_l1_xty(const double* W, int64_t ldw, const double* xy, int cpp, int ycol, const int4* chunks,
                   int nchunks, double* part_y, int B, cudaStream_t s) {
  dim3 grid(B, nchunks);
  l1_xty_kernel<<<grid, 128, 0, s>>>(W, ldw, xy, cpp, ycol, chunks, part_y, B);
}

void launch_l1_assemble(const double* part, int64_t part_stride, int ldp, const double* part_y, int64_t part_y_stride,
                        int P, const int2* fold_chunks, int K, int R1, const double* tau, int B, int nC, double* cm,
                        int64_t cm_stride, int loocv, cudaStream_t s) {
  dim3 grid((unsigned)ceil_div(nC, 128), nC + P);
  l1_assemble_kernel<<<grid, 128, 0, s>>>(part, part_stride, ldp, part_y, part_y_stride, fold_chunks, K, R1, tau, B, nC,
                                          cm, cm_stride, loocv);
}

void launch_l1_pred_sums(const double* W, int64_t ldw, int B, int R1, const double* beta, int ldb,
                         const int32_t* tile_fold, const double* xy, int cpp, int ycol, double* part_out,
                         int ntiles, double* out, cudaStream_t s) {
  l1_pred_sums_kernel<<<ntiles, 128, (size_t)R1 * 256 * sizeof(double), s>>>(W, ldw, B, R1, beta, ldb, tile_fold, xy, cpp,
                                                                     ycol, part_out);
  launch_partial_sum(part_out, ntiles, kMaxRidge * 3 + 2, out, s);
}

void launch_l1_chr_pred(const double* W, int64_t ldw, int nchr, const int32_t* chr_col_start, const double* beta,
                        int ldb, int R1, int best, const int32_t* tile_fold, double* pred, int64_t npad,
                        cudaStream_t s) {
  l1_chr_pred_kernel<<<(unsigned)(npad / 128), 128, 0, s>>>(W, ldw, nchr, chr_col_start, beta, ldb, R1, best, tile_fold,
                                                           pred, npad);
}

}  // namespace rg
