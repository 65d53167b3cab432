// Step-2 GxE interaction tests for quantitative traits (rg_s2_interaction): the robust (HC3 / HC4 / model-based) route of
// apply_interaction_tests_qt and the HLM route of apply_interaction_tests_HLM (src/Interaction.cpp:109-437), with E kept
// as a covariate (gwas_condtl), so the interaction model of every (variant, trait) has the two columns [G, E o G].
//
// Everything except the sandwich "meat" is a sum over samples of g or g^2 (g = mean-imputed genotype) against a feature
// column that does not depend on the variant (s2_int_sums_kernel, fixed-order chunk reduction):
//   robust  X_c, E X_c, res_p, E res_p (g) and 1, E, E^2 (g^2): X^T G, X^T (E o G), H^T res and H^T H in closed form,
//           X being the orthonormal covariate basis of rg_s2_set_chr;
//   HLM     d Px_k, d E Px_k, d yres, d E yres (g) and d^2, d^2 E, d^2 E^2 (g^2) per trait (d = Dinv_sqrt): Px^T m,
//           m^T m and m^T yres of m = d o [G, E o G], and since yres is orthogonal to Px,
//           Xres^T Xres = m^T m - (Px^T m)^T (Px^T m), Xres^T yres = m^T yres (src/HLM.cpp:236-243).
// The meat sum_i e_i^2 / (1 - h_i)^2 H_i H_i^T needs the leverages h_i and residuals e_i, which are nonlinear in the
// samples: one pass per robust variant (per 8 traits) with a fixed-order block reduction per sample chunk
// (s2_int_meat_kernel).  A first kernel fixes each variant's route, so the sums kernel forms only the columns that route
// reads and ignored variants do no work.  The binary-trait tests (s2_interaction_bt.cu) run the same sums kernel on their
// own feature rows, with the genotype in the block's minor-allele coding (launch_s2_int_sums).
#include "kernels.cuh"

namespace rg {

namespace {

constexpr int kIntVT = 16;       // variants per CTA of the sums kernel
constexpr int kIntSub = 256;     // samples staged in shared memory at a time
constexpr int kIntThreads = 128;

// the feature columns a variant's route reads: robust columns [0, nr), HLM columns [nr, nf)
__device__ __forceinline__ bool int_needs(int8_t route, int f, int nr) { return route == (f < nr ? 1 : 2); }

// part[chunk][v][f] = sum over the chunk's samples of g_v(i)^(1 or 2) F[i][f], for the (v, f) the route of v reads; a
// CTA whose variants need none of its columns returns at once
__global__ void __launch_bounds__(kIntThreads) s2_int_sums_kernel(const uint32_t* __restrict__ dz, int64_t npad,
                                                                  const double* __restrict__ af_all,
                                                                  const double* __restrict__ mu,
                                                                  const int32_t* __restrict__ flags, int bs,
                                                                  const int8_t* __restrict__ route, int nr,
                                                                  const double* __restrict__ F, int nf,
                                                                  const uint8_t* __restrict__ pow2, const int4* chunks,
                                                                  int bs_pad, double* __restrict__ part) {
  __shared__ double gs[kIntVT][kIntSub];
  const int f0 = blockIdx.x * kIntThreads, f1 = min(nf, f0 + kIntThreads) - 1;
  const int f = f0 + threadIdx.x;
  const int v0 = blockIdx.z * kIntVT;
  bool any = false;
  for (int v = v0; v < min(bs, v0 + kIntVT); ++v) any |= int_needs(route[v], f0, nr) || int_needs(route[v], f1, nr);
  if (!any) return;
  const int4 ch = chunks[blockIdx.y];
  const bool sq = f < nf && pow2[f];
  double acc[kIntVT];
#pragma unroll
  for (int v = 0; v < kIntVT; ++v) acc[v] = 0.0;
  for (int o = 0; o < ch.y; o += kIntSub) {
    const int len = min(kIntSub, ch.y - o);
    __syncthreads();
    for (int k = threadIdx.x; k < kIntVT * kIntSub; k += kIntThreads) {
      const int v = k / kIntSub, j = k % kIntSub;
      double g = 0.0;
      if (v0 + v < bs && route[v0 + v] > 0 && j < len) {
        const uint32_t w = dz[(int64_t)(v0 + v) * npad + ch.x + o + j];
        if (!mu) g = int_g(w, 2.0 * af_all[v0 + v]);
        else g = int_g(w, mu[v0 + v], flags[v0 + v] & 8);            // binary traits: minor-allele coding
      }
      gs[v][j] = g;
    }
    __syncthreads();
    if (f < nf) {
      for (int j = 0; j < len; ++j) {
        const double x = F[(int64_t)(ch.x + o + j) * nf + f];
        if (x == 0.0) continue;
#pragma unroll
        for (int v = 0; v < kIntVT; ++v) {
          const double g = gs[v][j];
          acc[v] = fma(sq ? g * g : g, x, acc[v]);
        }
      }
    }
  }
  if (f >= nf) return;
#pragma unroll
  for (int v = 0; v < kIntVT; ++v)
    if (v0 + v < bs && int_needs(route[v0 + v], f, nr)) part[((int64_t)blockIdx.y * bs_pad + v0 + v) * nf + f] = acc[v];
}

// sums[v][f] over the chunks in a fixed order, for the (v, f) that s2_int_sums_kernel wrote
__global__ void s2_int_reduce_kernel(const double* __restrict__ part, int nchunks, int64_t chunk_stride,
                                     const int8_t* __restrict__ route, int bs, int nf, int nr, double* __restrict__ sums) {
  const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (k >= (int64_t)bs * nf) return;
  if (!int_needs(route[k / nf], (int)(k % nf), nr)) return;
  double s = 0.0;
  for (int c = 0; c < nchunks; ++c) s += part[(int64_t)c * chunk_stride + k];
  sums[k] = s;
}

// route of each variant (src/Interaction.cpp:56): 0 = no rows (ignored variant), 2 = HLM when a trait has MAC below
// rare_mac and the HLM state is set (unless robust SEs are forced or no_robust), 1 = robust otherwise
__global__ void s2_int_route_kernel(S2IntArgs a) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= a.bs) return;
  int8_t r = 0;
  if (!(a.flags[v] & 3)) {
    bool rare = false;
    for (int p = 0; p < a.P; ++p) rare |= a.mac[(int64_t)v * a.P + p] < a.rare_mac;
    r = (a.K > 0 && !a.no_robust && !a.force_robust && rare) ? 2 : 1;
  }
  a.route[v] = r;
}

// per variant: for robust variants b = X^T G, a = X^T (E o G), the two scales, Z = (H^T H)^-1 and
// tau_p = Z H^T res_p.  HLM variants are finished here too (one thread per variant, traits in order: a near-singular
// trait ends the variant's rows, as the reference returns from apply_interaction_tests_HLM).
__global__ void s2_int_finish_kernel(S2IntArgs a) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= a.bs) return;
  const int C = a.C, P = a.P;
  const double* S = a.sums + (int64_t)v * a.nf;
  double* W = a.var + (int64_t)v * a.var_stride;
  int32_t* st = a.status + (int64_t)v * P;
  double* coef = a.coef + (int64_t)v * P * 2;
  double* vc = a.vcov + (int64_t)v * P * 4;
  for (int p = 0; p < P; ++p) st[p] = 0;
  W[0] = 0.0;                                                        // 1 = robust state below is valid
  const int8_t route = a.route[v];
  if (route == 0) return;                                            // ignored variant: no rows at all
  if (route == 2) {
    const int K = a.K, w = 2 * K + 5;
    bool dead = false;
    for (int p = 0; p < P; ++p) {
      if (a.mac[(int64_t)v * P + p] < a.min_mac) continue;          // ignored_trait
      if (dead) { st[p] = -1; continue; }
      const double* T = S + a.nr + p * w;
      double uu = 0.0, uw = 0.0, ww = 0.0;
      for (int k = 0; k < K; ++k) { uu += T[k] * T[k]; uw += T[k] * T[K + k]; ww += T[K + k] * T[K + k]; }
      double z[3];
      if (!int_inv2(T[2 * K + 2] - uu, T[2 * K + 3] - uw, T[2 * K + 4] - ww, a.numtol, z)) { st[p] = -1; dead = true; continue; }
      const double r1 = T[2 * K], r2 = T[2 * K + 1];
      coef[2 * p] = z[0] * r1 + z[1] * r2;
      coef[2 * p + 1] = z[1] * r1 + z[2] * r2;
      vc[4 * p] = z[0]; vc[4 * p + 1] = z[1]; vc[4 * p + 2] = z[1]; vc[4 * p + 3] = z[2];
      st[p] = 2;
    }
    return;
  }
  // robust: H = [G_res / scale_fac, resid(E o G) / scf_i] (residualize_geno, residualize_matrix)
  const double* b = S;
  const double* av = S + C;
  const double* T2 = S + 2 * C + 2 * P;
  double bb = 0.0, aa = 0.0, ab = 0.0;
  for (int c = 0; c < C; ++c) { bb += b[c] * b[c]; aa += av[c] * av[c]; ab += av[c] * b[c]; }
  const double nk = (double)(a.n_analyzed - C);
  const double a11 = T2[0] - bb, a12 = T2[1] - ab, a22 = T2[2] - aa;
  const double scf_i = sqrt(a22 / nk);
  if (!(scf_i >= a.numtol)) return;                                  // skip_int (src/Interaction.cpp:84-85)
  const double sf = sqrt(a11 / nk);
  double z[3];
  bool ok = int_inv2(a11 / (sf * sf), a12 / (sf * scf_i), a22 / (scf_i * scf_i), a.numtol, z);
  if (!ok) {                                                         // src/Interaction.cpp:120
    for (int p = 0; p < P; ++p) if (!(a.mac[(int64_t)v * P + p] < a.min_mac)) st[p] = -1;
    return;
  }
  W[0] = 1.0; W[1] = sf; W[2] = scf_i; W[3] = z[0]; W[4] = z[1]; W[5] = z[2];
  for (int c = 0; c < C; ++c) { W[8 + c] = b[c]; W[8 + C + c] = av[c]; }
  for (int p = 0; p < P; ++p) {
    const double* yx = a.YtX + (int64_t)p * C;
    double r1 = S[2 * C + p], r2 = S[2 * C + P + p];
    for (int c = 0; c < C; ++c) { r1 -= b[c] * yx[c]; r2 -= av[c] * yx[c]; }
    r1 /= sf; r2 /= scf_i;
    W[8 + 2 * C + 2 * p] = z[0] * r1 + z[1] * r2;
    W[8 + 2 * C + 2 * p + 1] = z[1] * r1 + z[2] * r2;
  }
}

// meat of one robust variant over one sample chunk, for kIntTG traits at a time (all of them when P <= kIntTG): the
// leverage h_i of a sample is formed once, then per trait sum w_i H_i H_i^T (3 entries) and sum e_i^2
__global__ void __launch_bounds__(256) s2_int_meat_kernel(S2IntArgs a) {
  const int v = blockIdx.y, p0 = blockIdx.z * kIntTG;
  const double* W = a.var + (int64_t)v * a.var_stride;
  if (!(W[0] == 1.0)) return;                                        // HLM, ignored or skipped variant: no pass
  const int C = a.C, P = a.P, dp = a.dp;
  const int np = min(kIntTG, P - p0);
  const double sf = W[1], scf_i = W[2], z0 = W[3], z1 = W[4], z2 = W[5];
  const double* b = W + 8;
  const double* av = W + 8 + C;
  double t1[kIntTG], t2[kIntTG], acc[kIntTG][4];
  bool live[kIntTG], hc4[kIntTG];
#pragma unroll
  for (int q = 0; q < kIntTG; ++q) {
    const int p = p0 + q;
    live[q] = q < np && !(a.mac[(int64_t)v * P + p] < a.min_mac);
    hc4[q] = live[q] && a.force_hc4 && a.mac[(int64_t)v * P + p] <= a.rare_mac;
    t1[q] = live[q] ? W[8 + 2 * C + 2 * p] : 0.0;
    t2[q] = live[q] ? W[8 + 2 * C + 2 * p + 1] : 0.0;
    acc[q][0] = acc[q][1] = acc[q][2] = acc[q][3] = 0.0;
  }
  const double mu = 2.0 * a.af_all[v];
  const int4 ch = a.chunks[blockIdx.x];
  for (int j = threadIdx.x; j < ch.y; j += blockDim.x) {
    const int64_t i = ch.x + j;
    const double* Fi = a.F + i * dp;
    if (Fi[0] == 0.0) continue;                                      // not analysed: H_i = 0, e_i = 0
    const double e_i = a.E[i];
    const double g = int_g(a.dz[(int64_t)v * a.npad + i], mu);
    double xb = 0.0, xa = 0.0;
    for (int c = 0; c < C; ++c) { const double x = Fi[1 + c]; xb = fma(x, b[c], xb); xa = fma(x, av[c], xa); }
    const double h1 = (g - xb) / sf, h2 = (e_i * g - xa) / scf_i;
    const double lev = h1 * (z0 * h1 + z1 * h2) + h2 * (z1 * h1 + z2 * h2);
    const double om = 1.0 - lev;
    const double hc3 = om * om;
    const double h11 = h1 * h1, h12 = h1 * h2, h22 = h2 * h2;
#pragma unroll
    for (int q = 0; q < kIntTG; ++q) {
      if (!live[q]) continue;
      const int p = p0 + q;
      const double m = Fi[1 + C + P + p];
      if (m == 0.0) continue;                                        // e_i = 0 off the trait's mask
      const double e = m * (Fi[1 + C + p] - h1 * t1[q] - h2 * t2[q]);
      const double e2 = e * e;
      acc[q][3] += e2;
      if (a.no_robust) continue;
      const double den = hc4[q] ? pow(om, fmin((double)a.n_samples * lev / 2.0, 4.0)) : hc3;
      const double wt = e2 / den;
      acc[q][0] += wt * h11; acc[q][1] += wt * h12; acc[q][2] += wt * h22;
    }
  }
  __shared__ double red[8][kIntTG * 4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int q = 0; q < kIntTG; ++q)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      double x = acc[q][k];
      for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
      if (lane == 0) red[warp][q * 4 + k] = x;
    }
  __syncthreads();
  if (threadIdx.x < np * 4) {
    const int q = threadIdx.x >> 2, k = threadIdx.x & 3;
    double s = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w][threadIdx.x];
    a.meat_part[(((int64_t)v * P + p0 + q) * a.nchunks + blockIdx.x) * 4 + k] = s;
  }
}

// robust covariance: V = Z M Z (HC3 / HC4) or s^2 Z (model-based), then the scales of the printed rows
__global__ void s2_int_robust_kernel(S2IntArgs a) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.bs * a.P) return;
  const int v = k / a.P, p = k % a.P;
  const double* W = a.var + (int64_t)v * a.var_stride;
  if (!(W[0] == 1.0) || a.mac[k] < a.min_mac) return;
  double m[4] = {0.0, 0.0, 0.0, 0.0};
  for (int c = 0; c < a.nchunks; ++c)
    for (int q = 0; q < 4; ++q) m[q] += a.meat_part[((int64_t)k * a.nchunks + c) * 4 + q];
  const int C = a.C;
  const double sf = W[1], scf_i = W[2], z0 = W[3], z1 = W[4], z2 = W[5];
  double v11, v12, v22;
  if (a.no_robust) {
    const double s2 = m[3] / (a.mask_count[p] - C - 2);
    v11 = s2 * z0; v12 = s2 * z1; v22 = s2 * z2;
  } else {                                                           // Z M Z
    const double q11 = z0 * m[0] + z1 * m[1], q12 = z0 * m[1] + z1 * m[2];
    const double q21 = z1 * m[0] + z2 * m[1], q22 = z1 * m[1] + z2 * m[2];
    v11 = q11 * z0 + q12 * z1; v12 = q11 * z1 + q12 * z2; v22 = q21 * z1 + q22 * z2;
  }
  const double s1 = a.scf_sv[p] / sf, s2 = a.scf_sv[p] / scf_i;     // gscale, iscale (src/Interaction.cpp:155-156)
  a.coef[2 * (int64_t)k] = W[8 + 2 * C + 2 * p] * s1;
  a.coef[2 * (int64_t)k + 1] = W[8 + 2 * C + 2 * p + 1] * s2;
  double* vc = a.vcov + 4 * (int64_t)k;
  vc[0] = v11 * s1 * s1; vc[1] = v12 * s1 * s2; vc[2] = vc[1]; vc[3] = v22 * s2 * s2;
  a.status[k] = 1;
}

}  // namespace

void launch_s2_int_sums(const uint32_t* dz, int64_t npad, const double* af_all, const double* mu, const int32_t* flags,
                        int bs, const int8_t* route, int nr, const double* Fint, int nf, const uint8_t* pow2,
                        const int4* chunks, int nchunks, double* part, double* sums, cudaStream_t s) {
  const int bs_pad = (int)round_up(bs, kIntVT);
  dim3 g1((unsigned)ceil_div(nf, kIntThreads), nchunks, bs_pad / kIntVT);
  s2_int_sums_kernel<<<g1, kIntThreads, 0, s>>>(dz, npad, af_all, mu, flags, bs, route, nr, Fint, nf, pow2, chunks, bs_pad,
                                                part);
  const int64_t per = (int64_t)bs * nf;
  s2_int_reduce_kernel<<<(unsigned)ceil_div(per, 256), 256, 0, s>>>(part, nchunks, (int64_t)bs_pad * nf, route, bs, nf, nr,
                                                                    sums);
}

void launch_s2_interaction(const S2IntArgs& a, const uint8_t* pow2, double* part, cudaStream_t s) {
  s2_int_route_kernel<<<(unsigned)ceil_div(a.bs, 128), 128, 0, s>>>(a);
  launch_s2_int_sums(a.dz, a.npad, a.af_all, nullptr, nullptr, a.bs, a.route, a.nr, a.Fint, a.nf, pow2, a.chunks, a.nchunks,
                     part, a.sums, s);
  s2_int_finish_kernel<<<(unsigned)ceil_div(a.bs, 64), 64, 0, s>>>(a);
  s2_int_meat_kernel<<<dim3(a.nchunks, a.bs, (unsigned)ceil_div(a.P, kIntTG)), 256, 0, s>>>(a);
  s2_int_robust_kernel<<<(unsigned)ceil_div(a.bs * a.P, 128), 128, 0, s>>>(a);
}

}  // namespace rg
