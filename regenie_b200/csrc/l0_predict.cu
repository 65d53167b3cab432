// Out-of-fold level-0 predictions and their standardisation.
// Replaces the prediction half of ridge_level_0 (reference src/Step1_Models.cpp:494-557):
//   pred = beta^T G~_f o mask_f;  p_sum, p_sum2;  centre by p_sum/Neff, scale by
//   sqrt((Neff-1)/(p_sum2 - Neff*mean^2)).
// G~ is never formed:  beta^T G~ = gamma^T G0 + (gamma o mu)^T Miss - (B^T gamma)^T X^T  with
// gamma = beta / sd, evaluated straight from the 2-bit codes.
#include "kernels.cuh"

namespace rg {

constexpr int QT = 10;     // (ridge, phenotype) outputs per thread
constexpr int SNPC = 64;   // SNP rows staged in shared memory per step

// gamma[f][i][q] = beta[m=(f,r)][p][i] * inv_sd[i],  q = r*P + p  (zero-padded to Qp);
// gmu = gamma * mu.  grid: (rows_p/128, K), block 128.
__global__ void l0_gamma_kernel(const double* __restrict__ cm, int64_t cm_stride, int ldc, int nC,
                                int R, int P, int Qp, int bs, int rows_p,
                                const double* __restrict__ mu, const double* __restrict__ inv_sd,
                                double* __restrict__ gam, double* __restrict__ gmu) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int f = blockIdx.y;
  if (i >= rows_p) return;
  double* g = gam + ((int64_t)f * rows_p + i) * Qp;
  double* gm = gmu + ((int64_t)f * rows_p + i) * Qp;
  const double s = inv_sd[i], m = mu[i];
  for (int q = 0; q < Qp; ++q) {
    double v = 0.0;
    if (q < R * P && i < bs) {
      const int r = q / P, p = q % P;
      v = cm[(int64_t)(f * R + r) * cm_stride + (int64_t)(nC + p) * ldc + i] * s;
    }
    g[q] = v;
    gm[q] = v * m;
  }
}

// cvec[f][q][c] = sum_i gamma[f][i][q] * Bv[i][c]   (fixed-order tree reduction per CTA)
// grid: (Qp, K), block 256.
__global__ void l0_cvec_kernel(const double* __restrict__ gam, const double* __restrict__ Bv, int C,
                               int Qp, int bs, int rows_p, double* __restrict__ cvec) {
  __shared__ double red[256];
  const int q = blockIdx.x, f = blockIdx.y;
  for (int c = 0; c < C; ++c) {
    double s = 0.0;
    for (int i = threadIdx.x; i < bs; i += 256)
      s += gam[((int64_t)f * rows_p + i) * Qp + q] * Bv[(int64_t)i * C + c];
    s = cta_tree<256>(s, red);
    if (threadIdx.x == 0) cvec[((int64_t)f * Qp + q) * C + c] = s;
  }
}

// grid: (Npad/128 sample tiles, Qp/QT); block 128 = 4 warps x 32 consecutive samples.
__global__ void __launch_bounds__(128)
l0_predict_kernel(PredictArgs a) {
  __shared__ double sg[SNPC][QT];
  __shared__ double sm[SNPC][QT];
  __shared__ double red[2][4][QT];
  const int t = blockIdx.x * 128 + threadIdx.x;
  const int f = a.tile_fold[blockIdx.x];
  const int q0 = blockIdx.y * QT;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t wpr = a.words_per_row;
  const int64_t wbase = (int64_t)(blockIdx.x * 128 + warp * 32) / 16 + (lane >> 4);
  const int sh = 2 * (lane & 15);

  double acc[QT];
#pragma unroll
  for (int q = 0; q < QT; ++q) acc[q] = 0.0;

  for (int i0 = 0; i0 < a.bs; i0 += SNPC) {
    __syncthreads();
    for (int e = threadIdx.x; e < SNPC * QT; e += 128) {
      const int r = e / QT, q = e % QT;
      const int i = i0 + r;
      const bool ok = i < a.bs;
      sg[r][q] = ok ? a.gam[((int64_t)f * a.rows_p + i) * a.Qp + q0 + q] : 0.0;
      sm[r][q] = ok ? a.gmu[((int64_t)f * a.rows_p + i) * a.Qp + q0 + q] : 0.0;
    }
    __syncthreads();
    const int nr = min(SNPC, a.bs - i0);
#pragma unroll 2
    for (int r = 0; r < nr; ++r) {
      const uint32_t w = __ldg(a.gp + (int64_t)(i0 + r) * wpr + wbase);
      const uint32_t code = (w >> sh) & 3u;
      const bool miss = code == 3u;
      const double g = miss ? 0.0 : (double)code;
      if (__any_sync(0xffffffffu, code != 0u)) {
#pragma unroll
        for (int q = 0; q < QT; ++q) acc[q] = fma(g, sg[r][q], acc[q]);
        if (miss) {
#pragma unroll
          for (int q = 0; q < QT; ++q) acc[q] += sm[r][q];
        }
      }
    }
  }
  // covariate correction, masking, raw store, partial sums
  double xr[kMaxCov];
  for (int c = 0; c < a.C; ++c) xr[c] = a.xy[(int64_t)t * a.cpp + c];
#pragma unroll
  for (int q = 0; q < QT; ++q) {
    const int qq = q0 + q;
    double v = 0.0;
    if (qq < a.R * a.P) {
      const int r = qq / a.P, p = qq % a.P;
      v = acc[q];
      const double* cv = a.cvec + ((int64_t)f * a.Qp + qq) * a.C;
      for (int c = 0; c < a.C; ++c) v -= xr[c] * cv[c];
      v *= (double)a.mask[(int64_t)p * a.npad + t];
      a.W[p][(int64_t)(a.col0 + r) * a.npad + t] = v;
    }
    // deterministic CTA reduction: warp shuffle tree then fixed-order sum of 4 warps
    double s1 = v, s2 = v * v;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if (lane == 0) { red[0][warp][q] = s1; red[1][warp][q] = s2; }
  }
  __syncthreads();
  if (threadIdx.x < QT) {
    const int q = threadIdx.x;
    const double s1 = ((red[0][0][q] + red[0][1][q]) + red[0][2][q]) + red[0][3][q];
    const double s2 = ((red[1][0][q] + red[1][1][q]) + red[1][2][q]) + red[1][3][q];
    a.part[((int64_t)blockIdx.x * a.Qp + q0 + q) * 2 + 0] = s1;
    a.part[((int64_t)blockIdx.x * a.Qp + q0 + q) * 2 + 1] = s2;
  }
}

// mean / inverse sd of each (ridge, phenotype) column: fixed-order sum over sample tiles.
// grid: (Q), block 256.
__global__ void l0_std_reduce_kernel(const double* __restrict__ part, int ntiles, int Qp, int P,
                                     const double* __restrict__ neff, double* __restrict__ mean_invsd) {
  __shared__ double red[2 * 256];
  const int q = blockIdx.x;
  double s[2] = {0.0, 0.0};
  for (int tI = threadIdx.x; tI < ntiles; tI += 256) {
    s[0] += part[((int64_t)tI * Qp + q) * 2 + 0];
    s[1] += part[((int64_t)tI * Qp + q) * 2 + 1];
  }
  cta_tree<256>(s, red);
  if (threadIdx.x == 0) {
    const double ne = neff[q % P];
    const double mean = s[0] / ne;                                    // src/Step1_Models.cpp:544
    const double invsd = sqrt((ne - 1.0) / (s[1] - ne * mean * mean));   // :545
    mean_invsd[2 * q] = mean;
    mean_invsd[2 * q + 1] = invsd;
  }
}

// grid: (Npad/256, Q).  src / dst may be the same table (in place) or the lane's local scratch -> the owners' W: with
// phenotypes owned by other GPUs the raw predictions are then produced, summed and read LOCALLY and only the finished
// values cross NVLink, as plain stores (the in-place version read-modify-wrote the peer's HBM: 75 % scaling at N = 500k).
__global__ void l0_std_apply_kernel(const double* const* __restrict__ src, int src_col0, double* const* __restrict__ W,
                                    int64_t npad, int col0, int P, const uint8_t* __restrict__ is_real,
                                    const double* __restrict__ mean_invsd) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int q = blockIdx.y;
  if (t >= npad) return;
  const int r = q / P, p = q % P;
  const double v = src[p][(int64_t)(src_col0 + r) * npad + t];
  // the reference centres every row of the fold (masked samples become -mean*invsd,
  // src/Step1_Models.cpp:556-557); layout padding rows stay exactly zero.
  W[p][(int64_t)(col0 + r) * npad + t] = is_real[t] ? (v - mean_invsd[2 * q]) * mean_invsd[2 * q + 1] : 0.0;
}

void launch_l0_gamma(const double* cm, int64_t cm_stride, int ldc, int nC, int R, int P, int Qp,
                     int bs, int rows_p, int K, const double* mu, const double* inv_sd,
                     const double* Bv, int C, double* gam, double* gmu, double* cvec, cudaStream_t s) {
  dim3 g1(rows_p / 128, K);
  l0_gamma_kernel<<<g1, 128, 0, s>>>(cm, cm_stride, ldc, nC, R, P, Qp, bs, rows_p, mu, inv_sd, gam, gmu);
  dim3 g2(Qp, K);
  l0_cvec_kernel<<<g2, 256, 0, s>>>(gam, Bv, C, Qp, bs, rows_p, cvec);
}

void launch_l0_predict(const PredictArgs& a, int ntiles, cudaStream_t s) {
  dim3 grid(ntiles, a.Qp / QT);
  l0_predict_kernel<<<grid, 128, 0, s>>>(a);
}

void launch_l0_standardize(const double* part, int ntiles, int Qp, int Q, int P, const double* neff,
                           double* mean_invsd, double* const* W, int64_t npad, int col0,
                           const uint8_t* is_real, cudaStream_t s, const double* const* src, int src_col0) {
  l0_std_reduce_kernel<<<Q, 256, 0, s>>>(part, ntiles, Qp, P, neff, mean_invsd);
  dim3 grid((unsigned)ceil_div(npad, 256), Q);
  if (src) l0_std_apply_kernel<<<grid, 256, 0, s>>>(src, src_col0, W, npad, col0, P, is_real, mean_invsd);
  else l0_std_apply_kernel<<<grid, 256, 0, s>>>(W, col0, W, npad, col0, P, is_real, mean_invsd);
}

void launch_l0_std_reduce_only(const double* part, int ntiles, int Qp, int Q, int P, const double* neff,
                               double* mean_invsd, cudaStream_t s) {
  l0_std_reduce_kernel<<<Q, 256, 0, s>>>(part, ntiles, Qp, P, neff, mean_invsd);
}

int predict_qt() { return QT; }

}  // namespace rg
