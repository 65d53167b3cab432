// Step-2 per-variant score test (quantitative traits): sufficient statistics straight from the
// 2-bit codes, then the closed-form finish.  Replaces, per variant, parseSnpfromBed /
// compute_mac / compute_aaf_info (reference src/Geno.cpp:2414-2536, 3077-3148), check_sparse_G
// (:3165), residualize_geno (:3242) and compute_score_qt (src/Step2_Models.cpp:343-467).
//
// The reference materialises the imputed N-vector g, residualises it (g - X X^T g), scales it
// and takes P dot products.  All of those are linear/quadratic forms of the three code-wise sums
//   S1 = sum_{i} g0_i   F_i,   S2 = sum_i g0_i^2 F_i,   Sm = sum_i miss_i F_i
// of one per-sample feature row  F_i = [a_i | x_i | res_i | m_i | m_ip x_ic]  (a = in analysis,
// m = per-trait mask), so a variant costs one pass over N/4 bytes and no N-length f64 temporary.
#include "kernels.cuh"

namespace rg {

constexpr int kS2Cols = 16;
constexpr int kS2Sub = 128;

// grid: (rows_p/128, nchunks, Dp/16); block 128: thread = variant row.
__global__ void __launch_bounds__(128)
s2_stats_kernel(const uint32_t* __restrict__ gp, int64_t words_per_row, const double* __restrict__ F, int dp,
                const int4* __restrict__ chunks, int rows_p, double* __restrict__ part) {
  __shared__ double2 tile[kS2Sub][kS2Cols / 2];
  const int row = blockIdx.x * 128 + threadIdx.x;
  const int4 ch = chunks[blockIdx.y];
  const int col0 = blockIdx.z * kS2Cols;
  const uint32_t* grow = gp + (int64_t)row * words_per_row;
  double a1[kS2Cols], a2[kS2Cols], am[kS2Cols];
#pragma unroll
  for (int c = 0; c < kS2Cols; ++c) a1[c] = a2[c] = am[c] = 0.0;
  for (int sub = 0; sub < ch.y; sub += kS2Sub) {
    const int t0 = ch.x + sub;
    __syncthreads();
    for (int e = threadIdx.x; e < kS2Sub * (kS2Cols / 2); e += 128) {
      const int s = e / (kS2Cols / 2), c2 = e % (kS2Cols / 2);
      tile[s][c2] = *reinterpret_cast<const double2*>(F + (int64_t)(t0 + s) * dp + col0 + 2 * c2);
    }
    __syncthreads();
#pragma unroll 1
    for (int wq = 0; wq < kS2Sub / 16; ++wq) {
      const uint32_t w = __ldg(grow + (t0 >> 4) + wq);
      if (w == 0) continue;
#pragma unroll 2
      for (int k = 0; k < 16; ++k) {
        const uint32_t code = (w >> (2 * k)) & 3u;
        if (code == 0u) continue;
        const double2* xr = tile[wq * 16 + k];
        if (code == 3u) {
#pragma unroll
          for (int c2 = 0; c2 < kS2Cols / 2; ++c2) {
            const double2 v = xr[c2];
            am[2 * c2] += v.x; am[2 * c2 + 1] += v.y;
          }
        } else {
          const double g = (double)code, g2 = g * g;
#pragma unroll
          for (int c2 = 0; c2 < kS2Cols / 2; ++c2) {
            const double2 v = xr[c2];
            a1[2 * c2] = fma(g, v.x, a1[2 * c2]);     a1[2 * c2 + 1] = fma(g, v.y, a1[2 * c2 + 1]);
            a2[2 * c2] = fma(g2, v.x, a2[2 * c2]);    a2[2 * c2 + 1] = fma(g2, v.y, a2[2 * c2 + 1]);
          }
        }
      }
    }
  }
  double* o = part + (((int64_t)blockIdx.y * rows_p + row) * 3) * dp + col0;
#pragma unroll
  for (int c = 0; c < kS2Cols; ++c) {
    o[c] = a1[c];
    o[dp + c] = a2[c];
    o[2 * dp + c] = am[c];
  }
}

// out[e] = sum_c part[c * per + e], chunks added in order.  grid: ceil(per/256)
__global__ void partial_sum_kernel(const double* __restrict__ part, int nchunks, int64_t per, double* __restrict__ out) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= per) return;
  double s = 0.0;
  for (int c = 0; c < nchunks; ++c) s += part[(int64_t)c * per + e];
  out[e] = s;
}

// one thread per variant
__global__ void s2_finalize_kernel(S2FinalizeArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.bs) return;
  const int C = a.C, P = a.P, dp = a.dp;
  const double* S1 = a.sums + ((int64_t)i * 3) * dp;
  const double* S2 = S1 + dp;
  const double* Sm = S1 + 2 * dp;
  const int cx = 1, cr = 1 + C, cm = 1 + C + P, cmx = 1 + C + 2 * P;
  const double nm = Sm[0];
  const bool xmale = a.non_par && a.non_par[i] && a.col_male >= 0;  // non-PAR chrX: see s2_count
  const S2Count all = s2_count(S1, S2, Sm, nullptr, 0, (double)a.n_analyzed, xmale ? a.col_male : -1,
                               a.male_tot, 1.0, a.ns_all + i, a.mac_all + i, a.af_all + i, nullptr);
  int flags = 0;
  const double mu = S1[0] / all.ns;
  for (int p = 0; p < P; ++p) {
    const int64_t ip = (int64_t)i * P + p;
    s2_count(S1, S2, Sm, a.info_sums + (int64_t)i * dp, cm + p, a.mask_count[p], xmale ? a.col_male + 1 + p : -1,
             a.male_tot + 1 + p, 1.0, a.ns + ip, a.mac + ip, a.af + ip, a.info ? a.info + ip : nullptr);
  }
  if (all.mac < a.min_mac) flags |= 1;                                  // src/Geno.cpp:3104-3105
  // non-zero entries among analysed samples after mean imputation (check_sparse_G)
  const double n2 = (S2[0] - S1[0]) * 0.5, n1 = S1[0] - 2.0 * n2;
  const double nnz = (a.nz_count ? a.nz_count[i] : n1 + n2) + ((mu != 0.0) ? nm : 0.0);
  const bool sparse = nnz <= (double)a.n_samples * 0.5;
  if (sparse) flags |= 4;
  double xtg2 = 0.0;
  for (int c = 0; c < C; ++c) {
    const double b = S1[cx + c] + mu * Sm[cx + c];
    xtg2 += b * b;
  }
  const double gg = S2[0] + mu * mu * nm;
  const double nk = (double)(a.n_analyzed - C);
  double sf = 1.0;
  if (!sparse) {
    sf = sqrt((gg - xtg2) / nk);                                     // src/Geno.cpp:3253-3254
    if (!(sf >= a.numtol)) flags |= 2;
  }
  a.scale_fac[i] = sf;
  a.flags[i] = flags;
  for (int p = 0; p < P; ++p) {
    double num = S1[cr + p] + mu * Sm[cr + p];
    for (int c = 0; c < C; ++c) num -= a.YtX[(int64_t)p * C + c] * (S1[cx + c] + mu * Sm[cx + c]);
    double den;
    if (a.strict) {
      den = sparse ? (gg - xtg2) : sf * sf * nk;                     // Step2_Models.cpp:386-387
    } else {
      const double mgg = S2[cm + p] + mu * mu * Sm[cm + p];
      double cross = 0.0, quad = xtg2;
      for (int c = 0; c < C; ++c) {
        const double b = S1[cx + c] + mu * Sm[cx + c];
        cross += b * (S1[cmx + p * C + c] + mu * Sm[cmx + p * C + c]);
      }
      if (!sparse) {                                                 // exact  m_p^T (g - Xb)^2   (:416)
        quad = 0.0;
        for (int c = 0; c < C; ++c) {
          const double b = S1[cx + c] + mu * Sm[cx + c];
          double r = 0.0;
          for (int c2 = 0; c2 < C; ++c2) r += a.XmX[((int64_t)p * C + c) * C + c2] * (S1[cx + c2] + mu * Sm[cx + c2]);
          quad += b * r;
        }
      }
      den = mgg - 2.0 * cross + quad;                                // sparse: approximation of :410
    }
    const double st = num / sqrt(den);
    const double beta = st * a.scf_sv[p] / sqrt(den);
    a.stat[(int64_t)i * P + p] = st;
    a.beta[(int64_t)i * P + p] = beta;
    a.se[(int64_t)i * P + p] = beta / st;
    a.chisq[(int64_t)i * P + p] = st * st;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// The same sums on the tensor cores, exactly: the planes G, G^2 and Miss of a variant row, built in registers from the
// 2-bit rows, against the radix-30 digit rows of the feature matrix F (built once per chromosome by
// l0_xy_digits_kernel), as column tiles of the INT8 Gram kernel (gram_wgmma.cu, kZStep2).  Products are integers <= 60,
// sample chunks are kept below 2^18 so every sum is an exact integer < 2^24; the chunk sums are added and reassembled
// in FP64 here.  Counts (N, A1FREQ numerators) come from the 0/1 columns of F, whose digits are exact, so they stay
// bit-exact.
// T [chunk][3 rows_p][ldt] exact digit sums -> S1, S2, Sm of row i: sums [row][3][dp], or with nnz [row][4][dp] (Se = 0,
// the layout of s2_bt_finalize_kernel) plus the counts check_sparse_G needs: non-zero calls n1 + n2 and hom-alt calls
// n2 from the column of F that flags the analysed samples (n1 = 2 S1 - S2, n2 = (S2 - S1) / 2).
// grid: (ceil(dp/128), rows_p), block 128.
__global__ void __launch_bounds__(128)
s2_tensor_finish_kernel(const float* __restrict__ T, int ldt, int64_t chunk_stride, int nchunk, int rows_p, int dp, int D,
                        const double* __restrict__ scale, double* __restrict__ sums, double* __restrict__ nnz,
                        double* __restrict__ n2o) {
  const int c = blockIdx.x * 128 + threadIdx.x;
  const int i = blockIdx.y;
  if (c >= dp) return;
  double out[3] = {0.0, 0.0, 0.0};
  if (c < D) {
    const int r0 = (c / kStatQ) * 128 + (c % kStatQ) * kLimbs;
    const double s = scale[c];
#pragma unroll
    for (int pl = 0; pl < 3; ++pl) {
      double acc = 0.0;
#pragma unroll
      for (int l = kLimbs - 1; l >= 0; --l) {
        double d = 0.0;
        for (int ch = 0; ch < nchunk; ++ch) d += (double)T[(int64_t)ch * chunk_stride + (int64_t)(pl * rows_p + i) * ldt + r0 + l];
        acc = acc * (1.0 / 30.0) + d;
      }
      out[pl] = acc * s / 15.0;      // exact for the 0/1 columns (acc = 15 k, s = 1): N and A1FREQ stay bit-exact
    }
  }
  const int nsum = nnz ? 4 : 3;
  double* o = sums + ((int64_t)i * nsum) * dp + c;
  o[0] = out[0];
  o[dp] = out[1];
  o[2 * dp] = out[2];
  if (!nnz) return;
  o[3 * dp] = 0.0;
  if (c == 0) {
    const double hom = (out[1] - out[0]) * 0.5;
    nnz[i] = (2.0 * out[0] - out[1]) + hom;
    n2o[i] = hom;
  }
}

// 2-bit rows -> the genotype words dz (kernels.cuh) that the Firth, SPA and GxE kernels read
__global__ void gp_to_dz_kernel(const uint32_t* __restrict__ gp, int64_t words_per_row, uint32_t* __restrict__ dz,
                                int64_t npad) {
  const int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int row = blockIdx.y;
  if (w >= words_per_row) return;
  const uint32_t word = __ldg(gp + (int64_t)row * words_per_row + w);
  uint32_t* o = dz + (int64_t)row * npad + w * 16;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const uint32_t code = (word >> (2 * k)) & 3u;
    o[k] = (code == 3u) ? kDzMissing : dz_word(code * 255u, 0u);
  }
}

void launch_s2_tensor_finish(const float* T, int ldt, int64_t chunk_stride, int nchunk, int rows_p, int dp, int D,
                             const double* scale, double* sums, double* nnz, double* n2, cudaStream_t s) {
  dim3 grid((unsigned)ceil_div(dp, 128), rows_p);
  s2_tensor_finish_kernel<<<grid, 128, 0, s>>>(T, ldt, chunk_stride, nchunk, rows_p, dp, D, scale, sums, nnz, n2);
}

void launch_gp_to_dz(const uint32_t* gp, int rows_p, uint32_t* dz, int64_t npad, cudaStream_t s) {
  const int64_t wpr = npad / 16;
  dim3 grid((unsigned)ceil_div(wpr, 256), rows_p);
  gp_to_dz_kernel<<<grid, 256, 0, s>>>(gp, wpr, dz, npad);
}

void launch_s2_stats(const uint32_t* gp, int64_t npad, const double* F, int dp, const int4* chunks, int nchunks,
                     int rows_p, double* part, double* sums, cudaStream_t s) {
  dim3 grid(rows_p / 128, nchunks, dp / kS2Cols);
  s2_stats_kernel<<<grid, 128, 0, s>>>(gp, npad / 16, F, dp, chunks, rows_p, part);
  launch_partial_sum(part, nchunks, (int64_t)rows_p * 3 * dp, sums, s);
}

void launch_partial_sum(const double* part, int nchunks, int64_t per, double* out, cudaStream_t s) {
  partial_sum_kernel<<<(unsigned)ceil_div(per, 256), 256, 0, s>>>(part, nchunks, per, out);
}

void launch_s2_finalize(const S2FinalizeArgs& a, cudaStream_t s) {
  s2_finalize_kernel<<<(unsigned)ceil_div(a.bs, 128), 128, 0, s>>>(a);
}

}  // namespace rg
