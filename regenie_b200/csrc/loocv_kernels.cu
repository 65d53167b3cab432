// Leave-one-out (LOOCV) variants of level 0 and level 1.
// Reference: ridge_level_0_loocv (src/Step1_Models.cpp:615-726), ridge_level_1_loocv (:875-963),
// Data::make_predictions_loocv (src/Data.cpp:1269-1343).  The reference uses one eigendecomposition
//   h_i = sum_k z_ik^2/(d_k+lambda),  yhat_i = sum_k z_ik w_k/(d_k+lambda),  z_i = V^T g_i
// and the closed form  pred_i = (yhat_i - h_i y_i)/(1 - h_i).  With  (A + lambda I) = L L^T  the same
// quantities are  h_i = |t_i|^2,  yhat_i = t_i . u  with  t_i = L^-1 g_i,  u = L^-1 b :  the sample
// vectors ride along as extra right-hand-side ROWS of the batched Cholesky (forward substitution
// fused into the factorisation), so no eigensolver is needed.
#include <algorithm>

#include "kernels.cuh"

namespace rg {

// rows nrow0 + t of every system r:  g~_t = (g_imp(:, t) - Bv x_t) * inv_sd   (level 0)
// grid: (Npad, ceil(nC/128)), block 128: thread = SNP i.  The sample axis is grid.x (limit 2^31 - 1): on grid.y it
// would cap LOOCV at 65 535 padded samples.
__global__ void l0_loocv_fill_kernel(const uint32_t* __restrict__ gp, int64_t words_per_row, int bs, int nC,
                                     const double* __restrict__ mu, const double* __restrict__ inv_sd,
                                     const double* __restrict__ Bv, int C, const double* __restrict__ xy, int cpp,
                                     double* __restrict__ cm, int64_t cm_stride, int nrow0, int R) {
  const int i = blockIdx.y * blockDim.x + threadIdx.x;
  const int t = blockIdx.x;
  if (i >= nC) return;
  double v = 0.0;
  if (i < bs) {
    const uint32_t w = gp[(int64_t)i * words_per_row + (t >> 4)];
    const uint32_t code = (w >> (2 * (t & 15))) & 3u;
    double g = (code == 3u) ? mu[i] : (double)code;
    const double* xr = xy + (int64_t)t * cpp;
    for (int c = 0; c < C; ++c) g -= Bv[(int64_t)i * C + c] * xr[c];
    v = g * inv_sd[i];
  }
  for (int r = 0; r < R; ++r) cm[(int64_t)r * cm_stride + (int64_t)(nrow0 + t) * nC + i] = v;
}

// One warp per sample: h = |t|^2, yhat_p = t . u_p, LOO prediction, mask, raw store + partial sums.
// grid: (Npad/128, R); block 128 threads = 4 warps, each warp loops over 32 samples of the tile.
// The phenotypes run in tiles of pt <= kMaxPhenoTile whose u rows fit in shared memory (fewer for a wide block).
__global__ void __launch_bounds__(128)
l0_loocv_pred_kernel(const double* __restrict__ cm, int64_t cm_stride, int nC, int bs, int Ppad, int P, int R,
                     const double* __restrict__ xy, int cpp, int C, const uint8_t* __restrict__ mask, int64_t npad,
                     double* const* __restrict__ W, int col0, double* __restrict__ part, int Qp, int pt) {
  extern __shared__ double us[];                 // u_p rows [pt][nC]
  __shared__ double red[2][4][kMaxPhenoTile];
  const int r = blockIdx.y;
  const double* A = cm + (int64_t)r * cm_stride;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int p0 = 0; p0 < P; p0 += pt) {
    const int np = min(pt, P - p0);
    __syncthreads();
    for (int e = threadIdx.x; e < np * nC; e += 128) us[e] = A[(int64_t)(nC + p0 + e / nC) * nC + e % nC];
    __syncthreads();
    double s1[kMaxPhenoTile], s2[kMaxPhenoTile];
#pragma unroll
    for (int p = 0; p < kMaxPhenoTile; ++p) s1[p] = s2[p] = 0.0;
    for (int sl = 0; sl < 32; ++sl) {
      const int t = blockIdx.x * 128 + warp * 32 + sl;
      const double* row = A + (int64_t)(nC + Ppad + t) * nC;
      double h = 0.0, yh[kMaxPhenoTile];
#pragma unroll
      for (int p = 0; p < kMaxPhenoTile; ++p) yh[p] = 0.0;
      for (int i = lane; i < bs; i += 32) {
        const double v = row[i];
        h = fma(v, v, h);
#pragma unroll
        for (int p = 0; p < kMaxPhenoTile; ++p)
          if (p < np) yh[p] = fma(v, us[p * nC + i], yh[p]);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        h += __shfl_xor_sync(0xffffffffu, h, o);
#pragma unroll
        for (int p = 0; p < kMaxPhenoTile; ++p) yh[p] += __shfl_xor_sync(0xffffffffu, yh[p], o);
      }
      if (lane == 0) {
#pragma unroll
        for (int p = 0; p < kMaxPhenoTile; ++p)
          if (p < np) {
            const int pp = p0 + p;
            const double y = xy[(int64_t)t * cpp + C + pp];
            double v = (yh[p] - h * y) / (1.0 - h);                       // src/Step1_Models.cpp:660-663
            v *= (double)mask[(int64_t)pp * npad + t];                    // :697
            W[pp][(int64_t)(col0 + r) * npad + t] = v;
            s1[p] += v; s2[p] += v * v;
          }
      }
    }
    if (lane == 0)
      for (int p = 0; p < np; ++p) { red[0][warp][p] = s1[p]; red[1][warp][p] = s2[p]; }
    __syncthreads();
    if (threadIdx.x < np) {
      const int p = threadIdx.x, q = r * P + p0 + p;
      part[((int64_t)blockIdx.x * Qp + q) * 2 + 0] = ((red[0][0][p] + red[0][1][p]) + red[0][2][p]) + red[0][3][p];
      part[((int64_t)blockIdx.x * Qp + q) * 2 + 1] = ((red[1][0][p] + red[1][1][p]) + red[1][2][p]) + red[1][3][p];
    }
  }
}

// LOOCV standardisation: masked entries are re-zeroed (src/Step1_Models.cpp:699-706).
// grid: (Npad/256, Q)
__global__ void l0_loocv_std_apply_kernel(double* const* __restrict__ W, int64_t npad, int col0, int P,
                                          const uint8_t* __restrict__ mask, const double* __restrict__ mean_invsd) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int q = blockIdx.y;
  if (t >= npad) return;
  const int r = q / P, p = q % P;
  double* w = W[p] + (int64_t)(col0 + r) * npad + t;
  *w = mask[(int64_t)p * npad + t] ? (*w - mean_invsd[2 * q]) * mean_invsd[2 * q + 1] : 0.0;
}

// ---------------------------------------------------------------------------------------- level 1
// sample rows of the R1 systems:  row (nrow0 + t) = W[t, 0:B]   (tile transpose, coalesced both ways); the dense level-0
// route passes its G~ as W (ldw = Npad, B = bs).
// grid: (Npad/32, ceil(nC/32)), block (32, 8); the sample axis is grid.x, like l0_loocv_fill_kernel
__global__ void l1_loocv_fill_kernel(const double* __restrict__ W, int64_t ldw, int B, int nC,
                                     double* __restrict__ cm, int64_t cm_stride, int nrow0, int R1) {
  __shared__ double tile[32][33];
  const int c0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int c = c0 + j;
    tile[j][threadIdx.x] = (c < B) ? W[(int64_t)c * ldw + t0 + threadIdx.x] : 0.0;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int t = t0 + j, c = c0 + threadIdx.x;
    if (c < nC)
      for (int r = 0; r < R1; ++r) cm[(int64_t)r * cm_stride + (int64_t)(nrow0 + t) * nC + c] = tile[threadIdx.x][j];
  }
}

// CV sums of ridge_level_1_loocv (src/Step1_Models.cpp:928-944): warp per sample.
// grid: (Npad/128, R1); out part [tile][R1][3] (Sx, Sx2, Sxy)
__global__ void __launch_bounds__(128)
l1_loocv_sums_kernel(const double* __restrict__ cm, int64_t cm_stride, int nC, int B, int nrow0,
                     const double* __restrict__ xy, int cpp, int ycol, double* __restrict__ part, int R1) {
  __shared__ double red[4][3];
  const int j = blockIdx.y;
  const double* A = cm + (int64_t)j * cm_stride;
  const double* u = A + (int64_t)nC * nC;            // L^-1 W^T y
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double sx = 0.0, sx2 = 0.0, sxy = 0.0;
  for (int sl = 0; sl < 32; ++sl) {
    const int t = blockIdx.x * 128 + warp * 32 + sl;
    const double* row = A + (int64_t)(nrow0 + t) * nC;
    double h = 0.0, yh = 0.0;
    for (int i = lane; i < B; i += 32) {
      const double v = row[i];
      h = fma(v, v, h);
      yh = fma(v, u[i], yh);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      h += __shfl_xor_sync(0xffffffffu, h, o);
      yh += __shfl_xor_sync(0xffffffffu, yh, o);
    }
    const double y = xy[(int64_t)t * cpp + ycol];
    const double pred = (yh - h * y) / (1.0 - h);                       // :936-937
    sx += pred; sx2 += pred * pred; sxy += pred * y;
  }
  if (lane == 0) { red[warp][0] = sx; red[warp][1] = sx2; red[warp][2] = sxy; }
  __syncthreads();
  if (threadIdx.x < 3) {
    const int v = threadIdx.x;
    part[((int64_t)blockIdx.x * R1 + j) * 3 + v] = ((red[0][v] + red[1][v]) + red[2][v]) + red[3][v];
  }
}

// make_predictions_loocv (src/Data.cpp:1296-1328) for the selected tau: rows `trow` hold t_i = L^-1 w_i
// (copy taken before the row backsolve), rows `zrow` hold z_i = H w_i.  Warp per sample.
//   yres_i = y_i - w_i.b;  pred[i][chr] = w_i[chr].b[chr] - (w_i[chr].z_i[chr]) * yres_i / (1 - h_i)
// grid: (Npad/128); block 128
__global__ void __launch_bounds__(128)
l1_loocv_chr_pred_kernel(const double* __restrict__ W, int64_t ldw, int B, int nC, const double* __restrict__ zrows,
                         const double* __restrict__ hvec, const double* __restrict__ bvec,
                         const double* __restrict__ xy, int cpp, int ycol, int nchr,
                         const int32_t* __restrict__ chr_col_start, double* __restrict__ pred, int64_t npad) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int sl = 0; sl < 32; ++sl) {
    const int t = blockIdx.x * 128 + warp * 32 + sl;
    double wb = 0.0;
    for (int c = lane; c < B; c += 32) wb = fma(W[(int64_t)c * ldw + t], bvec[c], wb);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wb += __shfl_xor_sync(0xffffffffu, wb, o);
    const double yres = xy[(int64_t)t * cpp + ycol] - wb;
    const double f = yres / (1.0 - hvec[t]);
    for (int ci = 0; ci < nchr; ++ci) {
      double a = 0.0, b = 0.0;
      for (int c = chr_col_start[ci] + lane; c < chr_col_start[ci + 1]; c += 32) {
        const double w = W[(int64_t)c * ldw + t];
        a = fma(w, bvec[c], a);
        b = fma(w, zrows[(int64_t)t * nC + c], b);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
      }
      if (lane == 0) pred[(int64_t)ci * npad + t] = a - b * f;
    }
  }
}

// h_i = |t_i|^2 for the rows of one system.  grid: (Npad/128), block 128 (warp per sample)
__global__ void __launch_bounds__(128)
rows_sqnorm_kernel(const double* __restrict__ rows, int nC, int B, double* __restrict__ out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int sl = 0; sl < 32; ++sl) {
    const int t = blockIdx.x * 128 + warp * 32 + sl;
    double h = 0.0;
    for (int i = lane; i < B; i += 32) { const double v = rows[(int64_t)t * nC + i]; h = fma(v, v, h); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
    if (lane == 0) out[t] = h;
  }
}

void launch_l0_loocv_fill(const uint32_t* gp, int64_t npad, int bs, int nC, const double* mu, const double* inv_sd,
                          const double* Bv, int C, const double* xy, int cpp, double* cm, int64_t cm_stride,
                          int nrow0, int R, cudaStream_t s) {
  dim3 grid((unsigned)npad, (unsigned)ceil_div(nC, 128));
  l0_loocv_fill_kernel<<<grid, 128, 0, s>>>(gp, npad / 16, bs, nC, mu, inv_sd, Bv, C, xy, cpp, cm, cm_stride, nrow0, R);
}

void launch_l0_loocv_pred(const double* cm, int64_t cm_stride, int nC, int bs, int Ppad, int P, int R,
                          const double* xy, int cpp, int C, const uint8_t* mask, int64_t npad, double* const* W,
                          int col0, double* part, int Qp, cudaStream_t s) {
  // the u rows of a phenotype tile in the dynamic shared memory the device allows next to the kernel's static arrays
  static const int64_t fit = [] {
    int dev = 0, optin = 0;
    RG_CUDA(cudaGetDevice(&dev));
    RG_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    cudaFuncAttributes fa;
    RG_CUDA(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(l0_loocv_pred_kernel)));
    return (int64_t)(optin - (int)fa.sharedSizeBytes) / (int64_t)sizeof(double);
  }();
  const int pt = (int)std::min<int64_t>({(int64_t)P, (int64_t)kMaxPhenoTile, fit / nC});
  RG_CHECK(pt >= 1, "LOOCV level 0: block too wide for the prediction kernel (nC = " + std::to_string(nC) + ")");
  const size_t smem = (size_t)pt * nC * sizeof(double);
  ensure_dyn_smem(reinterpret_cast<const void*>(l0_loocv_pred_kernel), smem);
  dim3 grid((unsigned)(npad / 128), R);
  l0_loocv_pred_kernel<<<grid, 128, smem, s>>>(cm, cm_stride, nC, bs, Ppad, P, R, xy, cpp, C, mask, npad, W,
                                              col0, part, Qp, pt);
}

void launch_l0_loocv_std_apply(double* const* W, int64_t npad, int col0, int P, int Q, const uint8_t* mask,
                               const double* mean_invsd, cudaStream_t s) {
  dim3 grid((unsigned)ceil_div(npad, 256), Q);
  l0_loocv_std_apply_kernel<<<grid, 256, 0, s>>>(W, npad, col0, P, mask, mean_invsd);
}

void launch_l1_loocv_fill(const double* W, int64_t ldw, int B, int nC, double* cm, int64_t cm_stride, int nrow0,
                          int R1, int64_t npad, cudaStream_t s) {
  dim3 grid((unsigned)(npad / 32), (unsigned)ceil_div(nC, 32));
  l1_loocv_fill_kernel<<<grid, dim3(32, 8), 0, s>>>(W, ldw, B, nC, cm, cm_stride, nrow0, R1);
}

void launch_l1_loocv_sums(const double* cm, int64_t cm_stride, int nC, int B, int nrow0, const double* xy, int cpp,
                          int ycol, double* part, int R1, int ntiles, double* out, cudaStream_t s) {
  dim3 grid(ntiles, R1);
  l1_loocv_sums_kernel<<<grid, 128, 0, s>>>(cm, cm_stride, nC, B, nrow0, xy, cpp, ycol, part, R1);
  launch_partial_sum(part, ntiles, R1 * 3, out, s);   // out[j][3]
}

void launch_rows_sqnorm(const double* rows, int nC, int B, double* out, int ntiles, cudaStream_t s) {
  rows_sqnorm_kernel<<<ntiles, 128, 0, s>>>(rows, nC, B, out);
}

void launch_l1_loocv_chr_pred(const double* W, int64_t ldw, int B, int nC, const double* zrows, const double* hvec,
                              const double* bvec, const double* xy, int cpp, int ycol, int nchr,
                              const int32_t* chr_col_start, double* pred, int64_t npad, cudaStream_t s) {
  l1_loocv_chr_pred_kernel<<<(unsigned)(npad / 128), 128, 0, s>>>(W, ldw, B, nC, zrows, hvec, bvec, xy, cpp, ycol, nchr,
                                                                 chr_col_start, pred, npad);
}

}  // namespace rg
