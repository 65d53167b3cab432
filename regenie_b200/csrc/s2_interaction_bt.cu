// Step-2 GxE interaction tests for binary traits (rg_s2_interaction_bt, rg_s2_interaction_firth): the logistic Wald
// tests of apply_interaction_tests_bt and the Firth likelihood-ratio tests of apply_interaction_tests_firth
// (src/Interaction.cpp:441-863), with E and E^2 kept as covariates (gwas_condtl), so the model of every (variant, trait)
// has the two columns H = [G_res / scale_fac, resid(E o G) / scf_i] and the trait's offset.
//
// Per variant, the projections X^T G, X^T (E o G) and |G|^2, |E o G|^2 are sums over samples of g or g^2 against fixed
// feature columns: the sums kernel of s2_interaction.cu on the feature rows [X_c, E X_c | 1, E^2], in the minor-allele
// coding of the block (flags bit 3, missing calls at the block's mean).  They give the two scales and the
// residualisation coefficients; a batch of variants then has its two H columns written out in FP64, and every pass of
// the fits reads them.  Each fit is Newton's method on a 2 x 2 system, so a pass is one exp (and one log) per sample and
// trait plus a handful of FMAs, reduced over the CTA in a fixed order (no atomics: results do not depend on the launch
// shape).  The scalar control flow of fit_logistic / fit_firth_nr runs uniformly in every thread of the CTA.
//   s2_int_bt_logistic_kernel  one CTA per (variant, group of kIntBtTG traits), the traits' IRLS in lockstep: a trait
//                              takes part in a pass while its fit is running, so each pass reads H once for all of them;
//                              then one pass for the HC3 meat of the traits on the robust route.
//   s2_int_bt_firth_kernel     one CTA per selected pair: the full, G-dropped and GxE-dropped fit_firth_nr fits.
#include "kernels.cuh"

namespace rg {

namespace {

constexpr int kBtThreads = 256;
constexpr int kBtWarps = kBtThreads / 32;
constexpr int kHVT = 16;                                  // variants (H slots) per CTA of the H kernel
constexpr int kHThreads = 128;
constexpr double kChi2p05 = 3.841458820694124;           // chi2_1 statistic of p = 0.05 (lpbase of :464)
constexpr double kLogTol = 1e-8;                          // fit_logistic numtol (src/Step1_Models.hpp:79)
constexpr int kLogIter = 50, kLineSearch = 25;           // niter_max, niter_max_line_search (src/Regenie.hpp:335-338)

// the variants the call tests: not ignored by the block (MAC below minMAC over all traits)
__global__ void s2_int_bt_route_kernel(S2IntBtArgs a) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < a.bs) a.route[v] = (a.flags[v] & 1) ? 0 : 1;
}

// per variant: scf_i = |resid(E o G)| / sqrt(n - C) (residualize_matrix, src/Pheno.cpp:1836-1852; below numtol: no
// rows, src/Interaction.cpp:84-85), scale_fac = |G_res| / sqrt(n - C) (residualize_geno with force, src/Geno.cpp:3212)
__global__ void s2_int_bt_scale_kernel(S2IntBtArgs a) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= a.bs) return;
  const int C = a.C;
  double* W = a.var + (int64_t)v * a.var_stride;
  W[0] = 0.0;
  if (!a.route[v]) return;
  const double* S = a.sums + (int64_t)v * a.nf;
  double bb = 0.0, aa = 0.0;
  for (int c = 0; c < C; ++c) { bb += S[c] * S[c]; aa += S[C + c] * S[C + c]; }
  const double nk = (double)(a.n_analyzed - C);
  const double scf_i = sqrt((S[2 * C + 1] - aa) / nk);
  if (!(scf_i >= a.numtol)) return;
  const double sf = sqrt((S[2 * C] - bb) / nk);
  if (!(sf >= a.numtol)) return;
  W[0] = 1.0; W[1] = sf; W[2] = scf_i;
  for (int c = 0; c < 2 * C; ++c) W[3 + c] = S[c];
}

// H slot k (variant vsel[k], or v0 + k) over all samples: H[k][0] = G_res / scale_fac, H[k][1] = resid(E o G) / scf_i,
// zero outside the analysis and for variants without rows.  grid (Npad / kHThreads, slots / kHVT)
__global__ void __launch_bounds__(kHThreads) s2_int_bt_h_kernel(S2IntBtArgs a, const int32_t* vsel) {
  __shared__ double sb[kHVT][2 * kMaxCov];
  __shared__ double ssf[kHVT], sscf[kHVT], smu[kHVT];
  __shared__ int svar[kHVT], sflip[kHVT];
  const int C = a.C, k0 = blockIdx.y * kHVT;
  if (threadIdx.x < kHVT) {
    const int slot = k0 + threadIdx.x;
    int v = -1;
    if (slot < a.nb) v = vsel ? vsel[slot] : a.v0 + slot;
    if (v >= 0 && !(a.var[(int64_t)v * a.var_stride] == 1.0)) v = -1;
    svar[threadIdx.x] = v;
    if (v >= 0) {
      const double* W = a.var + (int64_t)v * a.var_stride;
      ssf[threadIdx.x] = W[1]; sscf[threadIdx.x] = W[2];
      smu[threadIdx.x] = a.mu[v]; sflip[threadIdx.x] = a.flags[v] & 8;
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < kHVT * 2 * C; t += kHThreads) {
    const int k = t / (2 * C), c = t % (2 * C);
    const int v = svar[k];
    sb[k][c] = v >= 0 ? a.var[(int64_t)v * a.var_stride + 3 + c] : 0.0;
  }
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * kHThreads + threadIdx.x;
  if (i >= a.npad) return;
  const double* Fi = a.Fint + i * a.nf;
  const bool in = Fi[2 * C] != 0.0;
  double xb[kHVT], xa[kHVT];
#pragma unroll
  for (int k = 0; k < kHVT; ++k) xb[k] = xa[k] = 0.0;
  if (in)
    for (int c = 0; c < C; ++c) {
      const double x = Fi[c];
#pragma unroll
      for (int k = 0; k < kHVT; ++k) { xb[k] = fma(x, sb[k][c], xb[k]); xa[k] = fma(x, sb[k][C + c], xa[k]); }
    }
  const double e = a.E[i];
#pragma unroll
  for (int k = 0; k < kHVT; ++k) {
    const int slot = k0 + k;
    if (slot >= a.nb) break;
    const int v = svar[k];
    double h1 = 0.0, h2 = 0.0;
    if (in && v >= 0) {
      const double g = int_g(a.dz[(int64_t)v * a.npad + i], smu[k], sflip[k]);
      h1 = (g - xb[k]) / ssf[k];
      h2 = (e * g - xa[k]) / sscf[k];
    }
    a.H[(int64_t)(2 * slot) * a.npad + i] = h1;
    a.H[(int64_t)(2 * slot + 1) * a.npad + i] = h2;
  }
}

// one evaluation of the logistic model of a trait at (b1, b2), the sums of one pass
enum { kDev, kBad, kW0, kS1, kS2, kA11, kA12, kA22, kNS };

// fit_logistic (src/Step1_Models.cpp:156-222) of one trait as a state machine driven by the passes.  b is the point of
// the last evaluation (the reference's pivec / etavec), a is betavec (the last accepted point).  The second attempt
// (check_hs_dev = false, :464) continues from the state the first one left, as the reference does.
struct LogitFit {
  double b1, b2, a1, a2, dev_old, diff;
  int it, ls, att, state;            // state: 0 first evaluation, 1 candidate evaluated, 2 converged, 3 failed, 4 idle
  bool small;

  // the head of an iteration of the while loop (:170-185) at the last evaluation s
  __device__ void top(const double* s) {
    for (;;) {
      ++it;
      bool failed;
      if (it > kLogIter) {                                          // did not converge: the final deviance test (:216)
        if (!(diff == 0.0 || diff >= kLogTol)) { state = 2; return; }
        failed = true;
      } else {
        failed = s[kW0] > 0.0;                                      // get_wvec: a zero weight
      }
      if (!failed) break;
      if (att == 1) { state = 3; return; }
      restart(s);
    }
    // betanew = (X^T W X)^-1 X^T W z, z = eta - offset + (y - p) / w:  X^T W z = A b + score
    const double r1 = s[kA11] * b1 + s[kA12] * b2 + s[kS1], r2 = s[kA12] * b1 + s[kA22] * b2 + s[kS2];
    // solved like colPivHouseholderQr().solve(): rank 1 (nonzeroPivots) when |R_11| < eps |R_00| / sqrt(2), i.e.
    // |det| < eps / sqrt(2) max(|col_1|^2, |col_2|^2), and then the coefficient of the column not pivoted on stays 0
    // (E o G collinear with G, e.g. E constant)
    const double det = s[kA11] * s[kA22] - s[kA12] * s[kA12];
    const double n1 = s[kA11] * s[kA11] + s[kA12] * s[kA12], n2 = s[kA12] * s[kA12] + s[kA22] * s[kA22];
    if (fabs(det) < 2.220446049250313e-16 * 0.7071067811865476 * fmax(n1, n2)) {
      if (n1 >= n2) { b1 = (s[kA11] * r1 + s[kA12] * r2) / n1; b2 = 0.0; }
      else { b2 = (s[kA12] * r1 + s[kA22] * r2) / n2; b1 = 0.0; }
    } else {
      b1 = (s[kA22] * r1 - s[kA12] * r2) / det;
      b2 = (s[kA11] * r2 - s[kA12] * r1) / det;
    }
    ls = 1;
    state = 1;
  }
  // the second attempt, from the evaluation the first one ended on
  __device__ void restart(const double* s) {
    att = 1; dev_old = s[kDev]; it = 0; small = false; diff = 0.0;
  }
  __device__ void fail(const double* s) {
    if (att == 1) { state = 3; return; }
    restart(s);
    top(s);
  }
  __device__ void step(const double* s) {
    if (state == 0) {
      dev_old = s[kDev]; it = 0; att = 0; small = false; diff = 0.0;
      top(s);
      return;
    }
    if (s[kBad] == 0.0 && (att == 1 || s[kDev] < dev_old)) {       // candidate accepted
      const double smax = fmax(fabs(s[kS1]), fabs(s[kS2]));
      if (smax < kLogTol) { state = 2; return; }
      if (!small && it < 20 && smax < 1.0) small = true;
      if (small && it > 20 && smax > 5.0) { fail(s); return; }
      diff = fabs(s[kDev] - dev_old) / (0.1 + fabs(s[kDev]));
      a1 = b1; a2 = b2; dev_old = s[kDev];
      top(s);
      return;
    }
    if (ls == kLineSearch) { fail(s); return; }
    ++ls;
    b1 = 0.5 * (a1 + b1); b2 = 0.5 * (a2 + b2);
  }
};

// Wald tests of one variant (blockIdx.x of the batch) for traits p0 .. p0 + kIntBtTG (blockIdx.y)
__global__ void __launch_bounds__(kBtThreads) s2_int_bt_logistic_kernel(S2IntBtArgs a) {
  __shared__ double sh[kBtWarps * kIntBtTG * kNS];
  const int slot = blockIdx.x, v = a.v0 + slot, P = a.P, p0 = blockIdx.y * kIntBtTG;
  const int np = min(kIntBtTG, P - p0);
  const bool ok = a.var[(int64_t)v * a.var_stride] == 1.0;
  if (threadIdx.x < np) a.status[(int64_t)v * P + p0 + threadIdx.x] = 0;
  if (!ok) return;
  const double* W = a.var + (int64_t)v * a.var_stride;
  const double sf = W[1], scf_i = W[2];
  const double* H1 = a.H + (int64_t)(2 * slot) * a.npad;
  const double* H2 = H1 + a.npad;
  LogitFit f[kIntBtTG];
  bool any = false;
#pragma unroll
  for (int q = 0; q < kIntBtTG; ++q) {
    const bool live = q < np && !(a.mac[(int64_t)v * P + p0 + q] < a.min_mac);   // ignored_trait
    f[q].b1 = f[q].b2 = f[q].a1 = f[q].a2 = 0.0;
    f[q].state = live ? 0 : 4;
    any |= live;
  }
  if (!any) return;
  double s[kIntBtTG * kNS];
  double A[kIntBtTG][3];                                             // H^T W H at each trait's last evaluation
  for (;;) {
    bool act[kIntBtTG];
    bool run = false;
#pragma unroll
    for (int q = 0; q < kIntBtTG; ++q) { act[q] = f[q].state <= 1; run |= act[q]; }
    if (!run) break;
#pragma unroll
    for (int k = 0; k < kIntBtTG * kNS; ++k) s[k] = 0.0;
    for (int64_t i = threadIdx.x; i < a.npad; i += kBtThreads) {
      const double h1 = H1[i], h2 = H2[i];
#pragma unroll
      for (int q = 0; q < kIntBtTG; ++q) {
        if (!act[q]) continue;
        const int64_t pi = (int64_t)(p0 + q) * a.npad + i;
        const int8_t code = a.ym[pi];
        if (!code) continue;
        const double p = get_pvec(a.off[pi] + (h1 * f[q].b1 + h2 * f[q].b2));
        double* t = s + q * kNS;
        t[kDev] += -2.0 * ((code == 2) ? log(p) : log(1.0 - p));
        if (!(p > 0.0 && p < 1.0)) t[kBad] += 1.0;
        const double w = p * (1.0 - p), r = (code == 2 ? 1.0 : 0.0) - p;
        if (w == 0.0) t[kW0] += 1.0;
        t[kS1] = fma(h1, r, t[kS1]); t[kS2] = fma(h2, r, t[kS2]);
        const double wh1 = w * h1;
        t[kA11] = fma(wh1, h1, t[kA11]); t[kA12] = fma(wh1, h2, t[kA12]); t[kA22] = fma(w * h2, h2, t[kA22]);
      }
    }
    cta_sum<kBtWarps>(s, sh);
#pragma unroll
    for (int q = 0; q < kIntBtTG; ++q)
      if (act[q]) {
        A[q][0] = s[q * kNS + kA11]; A[q][1] = s[q * kNS + kA12]; A[q][2] = s[q * kNS + kA22];
        f[q].step(s + q * kNS);
      }
  }
  // a converged fit ends on an evaluation at its final point: V = (H^T W H)^-1, the route, and the HC3 meat pass
  double V[kIntBtTG][3];
  bool rob[kIntBtTG], any_rob = false;
  int8_t st[kIntBtTG];
#pragma unroll
  for (int q = 0; q < kIntBtTG; ++q) {
    rob[q] = false;
    st[q] = f[q].state == 2 ? 3 : (f[q].state == 3 ? -2 : 0);
    if (st[q] != 3) continue;
    if (!int_inv2(A[q][0], A[q][1], A[q][2], a.numtol, V[q])) { st[q] = -1; continue; }
    const double mac = a.mac[(int64_t)v * P + p0 + q];
    rob[q] = a.force_robust || (!a.no_robust && mac > a.rare_mac &&
                                (f[q].b1 * f[q].b1 / V[q][0] > kChi2p05 || f[q].b2 * f[q].b2 / V[q][2] > kChi2p05));
    any_rob |= rob[q];
  }
  if (any_rob) {
    double m[kIntBtTG * 3];
#pragma unroll
    for (int k = 0; k < kIntBtTG * 3; ++k) m[k] = 0.0;
    for (int64_t i = threadIdx.x; i < a.npad; i += kBtThreads) {
      const double h1 = H1[i], h2 = H2[i];
#pragma unroll
      for (int q = 0; q < kIntBtTG; ++q) {
        if (!rob[q]) continue;
        const int64_t pi = (int64_t)(p0 + q) * a.npad + i;
        const int8_t code = a.ym[pi];
        if (!code) continue;
        const double p = get_pvec(a.off[pi] + (h1 * f[q].b1 + h2 * f[q].b2));
        const double w = p * (1.0 - p);
        const double hv = w * (h1 * (V[q][0] * h1 + V[q][1] * h2) + h2 * (V[q][1] * h1 + V[q][2] * h2));
        const double r = ((code == 2 ? 1.0 : 0.0) - p) / (1.0 - hv), r2 = r * r;
        m[3 * q] = fma(r2 * h1, h1, m[3 * q]); m[3 * q + 1] = fma(r2 * h1, h2, m[3 * q + 1]);
        m[3 * q + 2] = fma(r2 * h2, h2, m[3 * q + 2]);
      }
    }
    cta_sum<kBtWarps>(m, sh);
#pragma unroll
    for (int q = 0; q < kIntBtTG; ++q) {
      if (!rob[q]) continue;
      const double z0 = V[q][0], z1 = V[q][1], z2 = V[q][2];
      const double* M = m + 3 * q;
      const double q11 = z0 * M[0] + z1 * M[1], q12 = z0 * M[1] + z1 * M[2];
      const double q21 = z1 * M[0] + z2 * M[1], q22 = z1 * M[1] + z2 * M[2];
      V[q][0] = q11 * z0 + q12 * z1; V[q][1] = q11 * z1 + q12 * z2; V[q][2] = q21 * z1 + q22 * z2;
      st[q] = 1;
    }
  }
  if (threadIdx.x != 0) return;
  const double sg = (a.flags[v] & 8) ? -1.0 : 1.0;
#pragma unroll
  for (int q = 0; q < kIntBtTG; ++q) {
    if (q >= np) break;
    const int64_t k = (int64_t)v * P + p0 + q;
    if ((st[q] == 1 || st[q] == 3) && (V[q][0] < 0.0 || V[q][2] < 0.0)) st[q] = -1;   // robust SE failed (:477)
    a.status[k] = st[q];
    if (st[q] != 1 && st[q] != 3) continue;
    a.coef[2 * k] = sg * f[q].b1 / sf;
    a.coef[2 * k + 1] = sg * f[q].b2 / scf_i;
    double* vc = a.vcov + 4 * k;
    vc[0] = V[q][0] / (sf * sf); vc[1] = V[q][1] / (sf * scf_i); vc[2] = vc[1]; vc[3] = V[q][2] / (scf_i * scf_i);
  }
}

// Firth sums at (b1, b2): the deviance over the mask and H^T W H with w = p (1 - p) on the mask, 1 off it (get_wvec for
// Firth, src/Step1_Models.cpp:1784)
__device__ void firth_pass1(const double* H1, const double* H2, const int8_t* ym, const double* off, int64_t npad,
                            double b1, double b2, double* sh, double (&s)[4]) {
  s[0] = s[1] = s[2] = s[3] = 0.0;
  for (int64_t i = threadIdx.x; i < npad; i += kBtThreads) {
    const double h1 = H1[i], h2 = H2[i];
    const int8_t code = ym[i];
    double w = 1.0;
    if (code) {
      const double p = get_pvec(off[i] + (h1 * b1 + h2 * b2));
      s[0] += -2.0 * ((code == 2) ? log(p) : log(1.0 - p));
      w = p * (1.0 - p);
    }
    const double wh1 = w * h1;
    s[1] = fma(wh1, h1, s[1]); s[2] = fma(wh1, h2, s[2]); s[3] = fma(w * h2, h2, s[3]);
  }
  cta_sum<kBtWarps>(s, sh);
}

// the modified score X^T (y - p + h (1/2 - p)) over the mask, h the diagonal of the hat matrix of W^1/2 H (Ai = A^-1)
__device__ void firth_pass2(const double* H1, const double* H2, const int8_t* ym, const double* off, int64_t npad,
                            double b1, double b2, const double* Ai, double* sh, double (&u)[2]) {
  u[0] = u[1] = 0.0;
  for (int64_t i = threadIdx.x; i < npad; i += kBtThreads) {
    const int8_t code = ym[i];
    if (!code) continue;
    const double h1 = H1[i], h2 = H2[i];
    const double p = get_pvec(off[i] + (h1 * b1 + h2 * b2));
    const double w = p * (1.0 - p);
    const double hv = w * (h1 * (Ai[0] * h1 + Ai[1] * h2) + h2 * (Ai[1] * h1 + Ai[2] * h2));
    const double r = (code == 2 ? 1.0 : 0.0) - p + hv * (0.5 - p);
    u[0] = fma(h1, r, u[0]); u[1] = fma(h2, r, u[1]);
  }
  cta_sum<kBtWarps>(u, sh);
}

// fit_firth_nr (src/Step2_Models.cpp:1267-1383) on the two columns of H.  free: 0 = both coefficients, 1 = only the
// first (G), 2 = only the second (E o G); the other one stays 0 (cols_incl = 1 with the free column first, :747-751 and
// :836-840), while the penalty and the hat values use the full 2 x 2 H^T W H.  comp_lrt: dev0 (at the starting point
// beta = 0) and the standard errors.  Returns false when the fit fails.
__device__ bool firth_fit(const double* H1, const double* H2, const int8_t* ym, const double* off, int64_t npad,
                          const S2IntBtArgs& a, int free, bool comp_lrt, double& b1, double& b2, double& dev,
                          double& dev0, double* se, double* sh) {
  int it = 0, n_inc = 0;
  double dev_new = 0.0, score_old = 1e16;
  double A[4], Ai[3];
  // the sums at the current point: the reference recomputes them at the head of each iteration; after an accepted
  // halving search they are those of the accepted candidate (b + step, the same bits), so that pass is skipped
  bool have = false;
  while (it++ < a.niter) {
    if (!have) firth_pass1(H1, H2, ym, off, npad, b1, b2, sh, A);
    const double det = A[1] * A[3] - A[2] * A[2];
    const double dev_old = A[0] - log(fabs(det));
    if (comp_lrt && it == 1) dev0 = dev_old;
    Ai[0] = A[3] / det; Ai[1] = -A[2] / det; Ai[2] = A[1] / det;
    double u[2];
    firth_pass2(H1, H2, ym, off, npad, b1, b2, Ai, sh, u);
    double st1 = 0.0, st2 = 0.0, smax;
    if (free == 0) {
      st1 = Ai[0] * u[0] + Ai[1] * u[1]; st2 = Ai[1] * u[0] + Ai[2] * u[1];
      smax = fmax(fabs(u[0]), fabs(u[1]));
    } else if (free == 1) {
      st1 = u[0] / A[1]; smax = fabs(u[0]);
    } else {
      st2 = u[1] / A[3]; smax = fabs(u[1]);
    }
    if (smax < a.tol && it >= 2) break;
    if (!comp_lrt) {
      n_inc = smax > score_old ? n_inc + 1 : 0;
      if (n_inc > 25) return false;
    }
    const double mx = fmax(fabs(st1), fabs(st2)) / a.maxstep;
    if (mx > 1.0) { st1 /= mx; st2 /= mx; }
    int ls = 1;
    for (; ls <= kLineSearch; ++ls) {
      if (ls > 1) { st1 /= 2.0; st2 /= 2.0; }
      double s[4];
      firth_pass1(H1, H2, ym, off, npad, b1 + st1, b2 + st2, sh, s);
      dev_new = s[0] - log(fabs(s[1] * s[3] - s[2] * s[2]));
      if (dev_new < dev_old) {
        for (int k = 0; k < 4; ++k) A[k] = s[k];
        break;
      }
    }
    have = ls <= kLineSearch;
    if (ls > kLineSearch) {
      if (!comp_lrt) return false;
      if (free == 2) st2 += 1e-6; else st1 += 1e-6;               // step_size(0): the first free coefficient
    }
    b1 += st1; b2 += st2;
    score_old = smax;
  }
  if (it > a.niter) return false;
  dev = dev_new;
  if (comp_lrt) {
    if (dev0 - dev_new < 0.0) return false;
    se[0] = sqrt(Ai[0]); se[1] = sqrt(Ai[2]);
  }
  return true;
}

// the three Firth fits of pair blockIdx.x (apply_interaction_tests_firth, src/Interaction.cpp:680-863, beg = 0)
__global__ void __launch_bounds__(kBtThreads, 1) s2_int_bt_firth_kernel(S2IntBtArgs a) {
  __shared__ double sh[kBtWarps * 4];
  const int k = blockIdx.x, v = a.sel_var[k], p = a.sel_trait[k];
  const double* H1 = a.H + (int64_t)(2 * k) * a.npad;
  const double* H2 = H1 + a.npad;
  const int8_t* ym = a.ym + (int64_t)p * a.npad;
  const double* off = a.off + (int64_t)p * a.npad;
  const double* W = a.var + (int64_t)v * a.var_stride;
  int status = 0;
  double b1 = 0.0, b2 = 0.0, dev = 0.0, dev0 = 0.0, se[2] = {0.0, 0.0}, lrt[3] = {0.0, 0.0, 0.0};
  if (!(W[0] == 1.0)) {
    status = 5;                                                     // the variant has no interaction rows
  } else if (!firth_fit(H1, H2, ym, off, a.npad, a, 0, true, b1, b2, dev, dev0, se, sh)) {
    status = 1;
  } else {
    lrt[0] = dev0 - dev;
    double c1 = 0.0, c2 = b2, dev_s = 0.0, unused = 0.0;           // G dropped: start (0, beta_GxE)
    if (!firth_fit(H1, H2, ym, off, a.npad, a, 2, false, c1, c2, dev_s, unused, nullptr, sh)) {
      status = 2;
    } else if ((lrt[1] = dev_s - dev) < 0.0) {
      status = 4;
    } else {
      c1 = b1; c2 = 0.0;                                            // GxE dropped: start (beta_G, 0)
      if (!firth_fit(H1, H2, ym, off, a.npad, a, 1, false, c1, c2, dev_s, unused, nullptr, sh)) status = 3;
      else if ((lrt[2] = dev_s - dev) < 0.0) status = 4;
    }
  }
  if (threadIdx.x != 0) return;
  const double sg = (a.flags[v] & 8) ? -1.0 : 1.0;
  const double sf = W[1], scf_i = W[2];
  a.f_status[k] = status;
  a.f_coef[2 * k] = status ? 0.0 : sg * b1 / sf;
  a.f_coef[2 * k + 1] = status ? 0.0 : sg * b2 / scf_i;
  a.f_se[2 * k] = status ? 0.0 : se[0] / sf;
  a.f_se[2 * k + 1] = status ? 0.0 : se[1] / scf_i;
  for (int j = 0; j < 3; ++j) a.f_lrt[3 * k + j] = status ? 0.0 : lrt[j];
}

}  // namespace

void launch_s2_int_bt_prep(const S2IntBtArgs& a, const uint8_t* pow2, double* part, cudaStream_t s) {
  s2_int_bt_route_kernel<<<(unsigned)ceil_div(a.bs, 128), 128, 0, s>>>(a);
  launch_s2_int_sums(a.dz, a.npad, a.af_all, a.mu, a.flags, a.bs, a.route, a.nf, a.Fint, a.nf, pow2, a.chunks, a.nchunks,
                     part, a.sums, s);
  s2_int_bt_scale_kernel<<<(unsigned)ceil_div(a.bs, 64), 64, 0, s>>>(a);
}

void launch_s2_int_bt_wald(const S2IntBtArgs& a, cudaStream_t s) {
  s2_int_bt_h_kernel<<<dim3((unsigned)ceil_div(a.npad, kHThreads), (unsigned)ceil_div(a.nb, kHVT)), kHThreads, 0, s>>>(
      a, nullptr);
  s2_int_bt_logistic_kernel<<<dim3(a.nb, (unsigned)ceil_div(a.P, kIntBtTG)), kBtThreads, 0, s>>>(a);
}

void launch_s2_int_bt_firth(const S2IntBtArgs& a, cudaStream_t s) {
  s2_int_bt_h_kernel<<<dim3((unsigned)ceil_div(a.npad, kHThreads), (unsigned)ceil_div(a.nb, kHVT)), kHThreads, 0, s>>>(
      a, a.sel_var);
  s2_int_bt_firth_kernel<<<a.nb, kBtThreads, 0, s>>>(a);
}

}  // namespace rg
