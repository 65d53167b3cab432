// Saddlepoint approximation (SPA) for binary traits: one CTA per flagged (variant, trait).
// Replaces run_SPA_test_snp + solve_K1_snp + get_SPA_pvalue_snp and the K / K' / K'' evaluators (reference
// src/Step2_Models.cpp:2072-2294), including the "fast" variant for sparse genotypes (exact terms over the
// non-zero genotypes, normal approximation for the rest).  Every evaluation of the cumulant generating function
// is one pass over the active sample set with a fixed-order block reduction; the Newton / bisection root search
// of the reference then runs uniformly in all threads.
#include "kernels.cuh"

namespace rg {

constexpr int kSpaThreads = 512;

__global__ void __launch_bounds__(kSpaThreads)
s2_spa_kernel(SpaArgs a) {
  __shared__ double sh[(kSpaThreads / 32) * 6];
  double v[kMaxCov];
  const S2Sel sp(a, v);
  const int64_t npad = a.npad;
  const double* gsq = sp.gs;
  const double* phat = a.phat + (int64_t)sp.ph * npad;
  const int8_t* ym = sp.ym;
  double* gv = sp.gv;
  int8_t* inS = sp.cf;
  const bool fast = sp.sparse;
  const int64_t ip = (int64_t)sp.i * a.P + sp.ph;
  const double stat = a.stat[ip], denum = a.den[ip];
  const double c = sqrt(denum);

  // ---- Gmod = Gres / Gamma^{1/2} on the masked samples, the active set, and the constants a, b, d, K' limits
  double s5[5] = {0, 0, 0, 0, 0};      // a, neg, pos, sum_S gres^2, sum_S gmu
  for (int64_t t = threadIdx.x; t < npad; t += kSpaThreads) {
    double g;
    const double r = sp.gres(a, t, g);
    const bool m = ym[t] != 0;
    const double gm = m ? r / gsq[t] : 0.0;
    gv[t] = gm;
    const bool s_in = m && (!fast || g != 0.0);
    inS[t] = s_in ? 1 : 0;
    const double gmu = gm * phat[t];
    s5[0] += gmu;
    s5[1] += fmin(gm, 0.0);
    s5[2] += fmax(gm, 0.0);
    if (s_in && fast) { s5[3] += r * r; s5[4] += gmu; }
  }
  cta_sum<kSpaThreads / 32>(s5, sh);
  const double va = s5[0], vb = denum - s5[3], vd = s5[4];
  int status = 0;
  double ptot = 0.0;
  const double score_num = stat * c;
  if (score_num < s5[1] - va || score_num > s5[2] - va) status = 1;

  // K, K', K'' at t over the active set (+ the closed-form remainder of the fast variant)
  auto eval = [&](double t, bool want_k, double& k0, double& k1, double& k2) {
    double s[4] = {0, 0, 0, 0};        // K, K1, K2, overflow flag
    const double tc = t / c;
    for (int64_t tt = threadIdx.x; tt < npad; tt += kSpaThreads) {
      if (!inS[tt]) continue;
      const double gm = gv[tt], p = phat[tt], gsv = gsq[tt];
      const double vexp = -tc * gm;
      if (vexp > 708.0) s[3] += 1.0;
      const double e = exp(vexp);
      const double den = p + (1.0 - p) * e;
      s[1] += (gm * p / c) / den;
      s[2] += (gm * gm * gsv * gsv / (c * c) * e) / (den * den);
      if (want_k) s[0] += log(1.0 - p + p * exp(tc * gm));
    }
    cta_sum<kSpaThreads / 32>(s, sh);
    if (fast) {
      k0 = s[0] - t * vd / c + t * t / 2.0 / denum * vb;
      k1 = s[1] - vd / c + t / denum * vb;
      k2 = (s[3] > 0.0) ? 0.0 : s[2] + vb / denum;
    } else {
      k0 = s[0] - t * va / c;
      k1 = s[1] - va / c;
      k2 = (s[3] > 0.0) ? 0.0 : s[2];
    }
  };

  const double tval = stat >= 0.0 ? -stat : stat;
  for (int tail = 0; tail < 2 && status == 0; ++tail) {
    const double lam = tail == 0 ? 1.0 : -1.0;
    double min_x = (tval >= 0.0) ? 0.0 : -1.7976931348623157e308, max_x = (tval >= 0.0) ? 1.7976931348623157e308 : 0.0;
    double t_old = 0.0, k0, k1, hess, t_new = -1.0, f_new = 0.0;
    eval(lam * t_old, false, k0, k1, hess);
    double f_old = lam * k1 - tval;
    int it = 0;
    bool done = false;
    while (!done) {
      if (++it > a.niter) { status = 2; break; }
      if (hess == 0.0) { status = 3; break; }
      t_new = t_old - f_old / hess;
      double h_new;
      eval(lam * t_new, false, k0, k1, h_new);
      f_new = lam * k1 - tval;
      if (fabs(f_new) < a.tol) { done = true; break; }
      if (t_new != 0.0 && t_new > min_x && t_new < max_x) {
        if (f_new > 0.0) max_x = t_new; else min_x = t_new;
      } else {
        t_new = (min_x + max_x) / 2.0;
        eval(lam * t_new, false, k0, k1, h_new);
        f_new = lam * k1 - tval;
        if (f_new <= 0.0) min_x = t_new; else max_x = t_new;
      }
      t_old = t_new; f_old = f_new; hess = h_new;
    }
    if (status) break;
    const double root = t_new;
    double kval, k2val;
    eval(lam * root, true, kval, k1, k2val);
    if (k2val == 0.0) { status = 4; break; }
    const double vval = root * sqrt(k2val);
    double pv;
    if (vval == 0.0) {
      pv = 0.5;
    } else {
      const double wval = copysign(1.0, root) * sqrt(2.0 * (root * tval - kval));
      const double rval = wval + log(vval / wval) / wval;
      pv = 0.5 * erfc(-rval * 0.70710678118654752440);
    }
    ptot += pv;
  }
  if (status == 0 && !(ptot <= 1.0)) status = 5;
  if (threadIdx.x == 0) {
    a.pval[blockIdx.x] = ptot;
    a.status[blockIdx.x] = status | (fast ? 256 : 0);
  }
}

void launch_s2_spa(const SpaArgs& a, cudaStream_t s) { s2_spa_kernel<<<a.n_sel, kSpaThreads, 0, s>>>(a); }

}  // namespace rg
