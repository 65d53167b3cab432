// Approximate Firth fallback for binary traits: one CTA per flagged (variant, trait).
// Replaces fit_firth_logistic_snp_fast -> fit_firth_pseudo / fit_firth for a single tested SNP with the
// covariate effects held in an offset (reference src/Step2_Models.cpp:1158-1252, 1527-1737), including the
// "carriers only" shortcut for sparse variants with MAC < 50.
//
// Every iteration of both solvers needs the same five sums over the active sample set S (masked samples, or
// the carriers): the deviance, X'WX = sum g^2 w, sum g p, sum g^3 w (1/2 - p) and a w == 0 flag; a pass
// evaluates them with one exp (+ one log) per sample and a fixed-order block reduction, so the scalar control
// flow of the reference runs uniformly in every thread of the CTA.
#include "kernels.cuh"

namespace rg {

constexpr int kFirthThreads = 512;

struct FirthSums { double dev, xtwx, gp, b3, w0; };

__global__ void __launch_bounds__(kFirthThreads)
s2_firth_kernel(FirthArgs a) {
  __shared__ double sh[(kFirthThreads / 32) * 6];
  double v[kMaxCov];
  const S2Sel sp(a, v);
  const int64_t npad = a.npad;
  const double* off = a.off + (int64_t)sp.ph * npad;
  const int8_t* ym = sp.ym;
  double* gv = sp.gv;
  int8_t* cf = sp.cf;
  const bool try_fast = sp.sparse && a.mac[(int64_t)sp.i * a.P + sp.ph] < 50.0;

  // ---- pass A: the residualised genotype G_res / Gamma^{1/2} and the carrier flags
  double cnt[1] = {0.0};
  for (int64_t t = threadIdx.x; t < npad; t += kFirthThreads) {
    double g;
    const double r = sp.gres(a, t, g);
    const double gsv = sp.gs[t];
    gv[t] = (gsv != 0.0) ? r / gsv : 0.0;
    const bool car = try_fast && ym[t] != 0 && g > 1e-4;
    cf[t] = car ? 1 : 0;
    cnt[0] += car ? 1.0 : 0.0;
  }
  cta_sum<kFirthThreads / 32>(cnt, sh);
  const bool fast = try_fast && cnt[0] > 0.0;

  // sums over S at coefficient b; with_dev adds the deviance over S (and over all masked samples in dev_all)
  double sum_gy = 0.0;
  auto pass = [&](double b, bool with_dev, bool all_mask_dev, double* dev_all) {
    double s[6] = {0, 0, 0, 0, 0, 0};
    for (int64_t t = threadIdx.x; t < npad; t += kFirthThreads) {
      const int8_t code = ym[t];
      if (code == 0) continue;
      const bool inS = fast ? (cf[t] != 0) : true;
      if (!inS && !all_mask_dev) continue;
      const double g = gv[t];
      const double p = get_pvec(off[t] + g * b);
      if (with_dev) {
        const double ll = -2.0 * ((code == 1) ? log(1.0 - p) : log(p));
        s[5] += ll;
        if (inS) s[0] += ll;
      }
      if (inS) {
        const double wv = p * (1.0 - p), g2 = g * g;
        s[1] = fma(g2, wv, s[1]);
        s[2] = fma(g, p, s[2]);
        s[3] = fma(g2 * g, wv * (0.5 - p), s[3]);
        if (wv == 0.0) s[4] += 1.0;
      }
    }
    cta_sum<kFirthThreads / 32>(s, sh);
    if (dev_all) *dev_all = s[5];
    FirthSums r{s[0], s[1], s[2], s[3], s[4]};
    return r;
  };
  {  // sum g y over S (constant)
    double s[1] = {0.0};
    for (int64_t t = threadIdx.x; t < npad; t += kFirthThreads) {
      const int8_t code = ym[t];
      if (code == 2 && (!fast || cf[t])) s[0] += gv[t];
    }
    cta_sum<kFirthThreads / 32>(s, sh);
    sum_gy = s[0];
  }
  double dev_mask0;
  const FirthSums z = pass(0.0, true, true, &dev_mask0);
  const double dev0 = dev_mask0 - log(z.xtwx);
  const double dev_nc = fast ? dev_mask0 - z.dev : 0.0;
  const double tol = a.tol;
  const int niter_pseudo = fast ? a.niter / 2 : min(a.niter / 2, 50);

  // ---- fit_firth_pseudo (:1527-1641)
  int state = 1;
  double beta = 0.0, betanew = 0.0, b14 = 0.0, xtwx = 1.0, dev_new = 0.0;
  {
    int it = 0;
    bool converged = false;
    while (it < niter_pseudo) {
      ++it;
      const FirthSums r = (it == 1) ? z : pass(beta, true, false, nullptr);
      xtwx = r.xtwx;
      dev_new = dev_nc + r.dev - log(xtwx);
      const double ystar_g = sum_gy + r.b3 / xtwx;
      double score = ystar_g - r.gp;
      if (fabs(score) < tol && it >= 2) { converged = true; break; }
      if (it == 14) b14 = beta;
      if (it == 15 && fabs(beta - b14) > 0.1) { state = 1; goto pseudo_done; }
      int nl = 0;
      double bdiff = 1e16;
      while (nl < 25) {
        ++nl;
        const double step = score / xtwx, bnew = fabs(step);
        if (bnew > bdiff) { state = 2; goto pseudo_done; }
        const double mx = bnew / 5.0;
        betanew = beta + (mx > 1.0 ? step / mx : step);
        const FirthSums q = pass(betanew, false, false, nullptr);
        score = ystar_g - q.gp;
        if (fabs(score) < tol) break;
        if (q.w0 > 0.0) { state = 3; goto pseudo_done; }
        xtwx = q.xtwx;
        beta = betanew;
        bdiff = bnew;
      }
      beta = betanew;
    }
    if (converged) state = 0;
  }
pseudo_done:
  double se = 0.0, lrt = 0.0;
  int status = 0;
  if (state == 0) {
    lrt = dev0 - dev_new;
    if (lrt < 0.0) state = 4; else se = sqrt(1.0 / xtwx);
  }
  if (state != 0) {
    // ---- fit_firth, Newton-Raphson with step halving (:1644-1737)
    beta = 0.0;
    FirthSums r = z;
    xtwx = r.xtwx;
    double dev_old = dev_mask0 - log(xtwx);
    dev_new = dev_old;
    int it = 0;
    bool converged = false;
    const int niter = a.niter / 2;
    while (it < niter) {
      ++it;
      const double score = sum_gy - r.gp + r.b3 / xtwx;
      if (fabs(score) < tol && it >= 2) { converged = true; break; }
      double step = score / xtwx;
      const double mx = fabs(step) / a.maxstep;
      if (mx > 1.0) step /= mx;
      bool ok = false;
      for (int ls = 1; ls <= 25; ++ls) {
        if (ls > 1) step /= 2.0;
        r = pass(beta + step, true, false, nullptr);
        xtwx = r.xtwx;
        dev_new = dev_nc + r.dev - log(xtwx);
        if (dev_new < dev_old) { ok = true; break; }
      }
      if (!ok) step += 1e-6;
      beta += step;
      dev_old = dev_new;
    }
    if (converged) {
      lrt = dev0 - dev_new;
      if (lrt < 0.0) status = 1; else se = sqrt(1.0 / xtwx);
    } else {
      status = 1;
    }
    if (status == 0) status = 0;
  }
  if (threadIdx.x == 0) {
    a.beta[blockIdx.x] = sp.flip ? -beta : beta;
    a.se[blockIdx.x] = se;
    a.lrt[blockIdx.x] = lrt;
    a.status[blockIdx.x] = status | (state << 4) | (fast ? 256 : 0);
  }
}

void launch_s2_firth(const FirthArgs& a, cudaStream_t s) {
  s2_firth_kernel<<<a.n_sel, kFirthThreads, 0, s>>>(a);
}

}  // namespace rg
