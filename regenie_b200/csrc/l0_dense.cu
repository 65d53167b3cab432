// Level-0 block on REAL-VALUED genotypes (8-bit BGEN dosages, or any FP64 dosage matrix such as a decoded .pgen dosage
// track): the exact-integer tensor-core route of the hard-call path does not apply, so the block is handled like the
// reference handles every block - as a dense FP64 matrix - but on the device:
//   readChunkFromBGENFileToG_fast   src/Geno.cpp:1574-1699  (dosage = p1/255 + 2 p0/255, mean imputation :3183-3188)
//   Data::residualize_genotypes     src/Data.cpp:190-228
//   Data::calc_cv_matrices          src/Data.cpp:729-776    (per-fold G G^T and G Y on the FP64 tensor pipe: l1_gram_kernel)
//   ridge_level_0                   src/Step1_Models.cpp:458-613 (batched Cholesky, chol.cu)
// G~ is kept as [bs][Npad] FP64 in the padded fold layout (row = SNP, contiguous over samples), i.e. exactly the
// "N x B column-major" shape of the level-1 predictors, so level 1's Gram, X^T y, fold-system assembler and LOOCV
// sample-row fill serve unchanged (l1_kernels.cu, loocv_kernels.cu).
#include "kernels.cuh"

namespace rg {

// gd[row][t] = dosage of the sample in padded slot t (-3 = missing, 0 = outside the analysis / layout padding)
// grid: (Npad/256, bs)
__global__ void dense_from_dosage_kernel(const uint8_t* __restrict__ probs, const uint8_t* __restrict__ miss, int64_t n_file,
                                         const int32_t* __restrict__ file_idx_pad, int ref_first, double* __restrict__ gd,
                                         int64_t npad) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= npad) return;
  const int row = blockIdx.y;
  const int32_t fi = file_idx_pad[t];
  double g = 0.0;
  if (fi >= 0) {
    if (miss && (miss[(int64_t)row * n_file + fi] & 0x80)) {
      g = -3.0;
    } else {
      const uint8_t* pr = probs + ((int64_t)row * n_file + fi) * 2;
      const double prob0 = (double)pr[0] / 255.0, prob1 = (double)pr[1] / 255.0;
      const double prob2 = fmax(1.0 - prob0 - prob1, 0.0);
      g = ref_first ? prob1 + 2.0 * prob2 : prob1 + 2.0 * prob0;          // src/Geno.cpp:1675-1678
    }
  }
  gd[(int64_t)row * npad + t] = g;
}

// same from an FP64 matrix G[row][n_file] (-3 = missing); grid: (Npad/256, bs)
__global__ void dense_from_f64_kernel(const double* __restrict__ G, int64_t n_file, const int32_t* __restrict__ file_idx_pad,
                                      double* __restrict__ gd, int64_t npad) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= npad) return;
  const int row = blockIdx.y;
  const int32_t fi = file_idx_pad[t];
  gd[(int64_t)row * npad + t] = fi >= 0 ? G[(int64_t)row * n_file + fi] : 0.0;
}

// One CTA per SNP row: mean over analysed, non-missing samples; impute; project out the covariate basis; scale to unit
// sd with the N_analyzed - C divisor; flag sd < numtol like the reference's throw (src/Data.cpp:203-209).  A flagged
// row (constant, or missing everywhere) is zeroed, so the block's predictors stay finite while the error is reported.
// mu_out / inv_sd_out: the mean and 1 / sd, as the 2-bit route stores them.
// grid: (bs), block 256.  xy: [Npad][cpp] with the C orthonormal covariates first.
__global__ void __launch_bounds__(256)
dense_prepare_kernel(double* __restrict__ gd, int64_t npad, const int32_t* __restrict__ file_idx_pad,
                     const double* __restrict__ xy, int cpp, int C, long long n_analyzed, double numtol,
                     double* __restrict__ mu_out, double* __restrict__ inv_sd_out,
                     unsigned long long* __restrict__ err_slot, long long err_base) {
  __shared__ double red[256];
  __shared__ double bc[kMaxCov];
  double* g = gd + (int64_t)blockIdx.x * npad;
  double tot = 0.0, cnt = 0.0;
  for (int64_t t = threadIdx.x; t < npad; t += 256)
    if (file_idx_pad[t] >= 0 && g[t] != -3.0) { tot += g[t]; cnt += 1.0; }
  tot = cta_tree<256>(tot, red);
  cnt = cta_tree<256>(cnt, red);
  const double mean = tot / cnt;
  for (int64_t t = threadIdx.x; t < npad; t += 256)
    if (g[t] == -3.0) g[t] = mean;
  __syncthreads();
  for (int c = 0; c < C; ++c) {
    double s = 0.0;
    for (int64_t t = threadIdx.x; t < npad; t += 256) s += g[t] * xy[t * cpp + c];
    s = cta_tree<256>(s, red);
    if (threadIdx.x == 0) bc[c] = s;
  }
  __syncthreads();
  double ss = 0.0;
  for (int64_t t = threadIdx.x; t < npad; t += 256) {
    double v = g[t];
    const double* x = xy + t * cpp;
    for (int c = 0; c < C; ++c) v -= bc[c] * x[c];
    g[t] = v;
    ss += v * v;
  }
  ss = cta_tree<256>(ss, red);
  const double sd = sqrt(ss) / sqrt((double)(n_analyzed - C));
  const bool low = !(sd >= numtol);
  if (threadIdx.x == 0) {
    mu_out[blockIdx.x] = mean;
    inv_sd_out[blockIdx.x] = 1.0 / sd;
    if (low) atomicMin(err_slot, (unsigned long long)(err_base + blockIdx.x + 1));
  }
  for (int64_t t = threadIdx.x; t < npad; t += 256) g[t] = low ? 0.0 : g[t] / sd;
}

// Out-of-fold predictions  pred[t][q] = mask_p(t) * sum_i G~[i][t] beta_{f(t)}[r][p][i],  q = r * P + p, written into the
// predictor matrix W (columns col0 + r of phenotype p).  beta at cm[(f R + r) cm_stride + (nC + p) ldc + i].
// grid: (Npad/128, ceil(Q / DQ)), block 128: thread = sample, DQ outputs per pass in registers.
constexpr int DQ = 25;
__global__ void __launch_bounds__(128)
dense_predict_kernel(const double* __restrict__ gd, int64_t npad, int bs, const double* __restrict__ cm, int64_t cm_stride,
                     int ldc, int nC, int R, int P, const int32_t* __restrict__ tile_fold, const uint8_t* __restrict__ mask,
                     double* const* __restrict__ W, int col0) {
  __shared__ double sb[64][DQ];
  const int64_t t = (int64_t)blockIdx.x * 128 + threadIdx.x;
  const int f = tile_fold[blockIdx.x];
  const int q0 = blockIdx.y * DQ, Q = R * P;
  const int nq = min(DQ, Q - q0);
  double acc[DQ];
#pragma unroll
  for (int q = 0; q < DQ; ++q) acc[q] = 0.0;
  for (int i0 = 0; i0 < bs; i0 += 64) {
    __syncthreads();
    for (int e = threadIdx.x; e < 64 * DQ; e += 128) {
      const int ii = e % 64, q = e / 64;
      double v = 0.0;
      if (q < nq && i0 + ii < bs) {
        const int r = (q0 + q) / P, p = (q0 + q) % P;
        v = cm[(int64_t)(f * R + r) * cm_stride + (int64_t)(nC + p) * ldc + i0 + ii];
      }
      sb[ii][q] = v;
    }
    __syncthreads();
    const int ni = min(64, bs - i0);
    for (int ii = 0; ii < ni; ++ii) {
      const double g = gd[(int64_t)(i0 + ii) * npad + t];
#pragma unroll
      for (int q = 0; q < DQ; ++q) acc[q] = fma(g, sb[ii][q], acc[q]);
    }
  }
  for (int q = 0; q < nq; ++q) {
    const int r = (q0 + q) / P, p = (q0 + q) % P;
    W[p][(int64_t)(col0 + r) * npad + t] = mask[(int64_t)p * npad + t] ? acc[q] : 0.0;
  }
}

// ---------------------------------------------------------------------------------------------------------------
void launch_dense_from_dosage(const uint8_t* probs, const uint8_t* miss, int64_t n_file, int bs, const int32_t* file_idx_pad,
                              int ref_first, double* gd, int64_t npad, cudaStream_t s) {
  dim3 grid((unsigned)ceil_div(npad, 256), bs);
  dense_from_dosage_kernel<<<grid, 256, 0, s>>>(probs, miss, n_file, file_idx_pad, ref_first, gd, npad);
}
void launch_dense_from_f64(const double* G, int64_t n_file, int bs, const int32_t* file_idx_pad, double* gd, int64_t npad,
                           cudaStream_t s) {
  dim3 grid((unsigned)ceil_div(npad, 256), bs);
  dense_from_f64_kernel<<<grid, 256, 0, s>>>(G, n_file, file_idx_pad, gd, npad);
}
void launch_dense_prepare(double* gd, int64_t npad, int bs, const int32_t* file_idx_pad, const double* xy, int cpp, int C,
                          long long n_analyzed, double numtol, double* mu, double* inv_sd, unsigned long long* err_slot,
                          long long err_base, cudaStream_t s) {
  dense_prepare_kernel<<<bs, 256, 0, s>>>(gd, npad, file_idx_pad, xy, cpp, C, n_analyzed, numtol, mu, inv_sd, err_slot,
                                          err_base);
}
void launch_dense_predict(const double* gd, int64_t npad, int bs, const double* cm, int64_t cm_stride, int ldc, int nC, int R,
                          int P, const int32_t* tile_fold, const uint8_t* mask, double* const* W, int col0, cudaStream_t s) {
  dim3 grid((unsigned)(npad / 128), (unsigned)ceil_div(R * P, DQ));
  dense_predict_kernel<<<grid, 128, 0, s>>>(gd, npad, bs, cm, cm_stride, ldc, nC, R, P, tile_fold, mask, W, col0);
}

}  // namespace rg
