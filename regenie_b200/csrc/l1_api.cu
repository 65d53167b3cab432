// Level-1 ridge, LOCO assembly and Step-2 entry points of the C ABI (include/rg_b200.h).
#include <string.h>

#include <algorithm>
#include <cmath>
#include <string>

#include "context.cuh"

using namespace rg;

// chunk table for the sample-axis reductions: bounded partial storage (<= ~1 GiB).  A fold of n samples takes
// ceil(n / len) chunks <= n / len + 1, so the K folds take at most max_chunks chunks of nC x nC partials.
static void l1_setup_chunks(rg_ctx* h, Step1State& s1, int nC) {
  cudaStream_t s = h->stream;
  const int K = s1.K;
  const int64_t per = (int64_t)nC * nC * 8;
  const int64_t max_chunks = std::max<int64_t>(K, (1ll << 30) / per);
  int64_t len = round_up(std::max<int64_t>(kStatChunk, ceil_div(h->Npad, max_chunks - K + 1)), 128);
  s1.l1_chunk_len = len;
  std::vector<int4> chunks;
  std::vector<int2> fold_chunks;
  fold_chunk_table(s1, len, chunks, fold_chunks);
  s1.l1_nchunks = (int)chunks.size();
  upload(s1.l1_chunks, chunks, s);
  upload(s1.l1_fold_chunks, fold_chunks, s);
  RG_CUDA(cudaStreamSynchronize(s));
}

// The systems of a level-1 fit: nmat systems of n_aug rows of nC doubles each (matrix rows, the RHS row nC and, for
// LOOCV, the Npad sample rows from row nC + 64 on).
struct L1Dims {
  int nC, nmat, n_aug, ntiles;
  int64_t cm_stride;
};

// What both level-1 fits do first.  The checks come before anything is launched, and l1_done is cleared before the
// first of them can throw, so a refused fit leaves no earlier fit behind.  Then level 0 is waited for, the chunk table
// is built and the buffers both fits use are sized: the quantitative k-fold fit solves K * R1 systems per phenotype,
// quantitative LOOCV R1, the binary fit one system refactored at every Newton step.
static L1Dims l1_begin(rg_ctx* h, Step1State& s1, bool bt) {
  s1.l1_done = false;                                     // until this fit completes, rg_loco and the hooks refuse
  RG_CHECK(s1.R1 >= 1 && s1.R1 <= kMaxRidge, "n_ridge_l1 out of range");
  if (bt) RG_CHECK(s1.B <= 6000, "logistic level 1 supports up to 6000 level-0 predictors (blocks x ridge values) in this build");
  RG_CUDA(cudaSetDevice(h->device));
  rg::sync_lanes(h);   // all level-0 blocks are in W
  ensure_W(h, s1);
  const int K = s1.K, R1 = s1.R1, P = h->P, B = (int)s1.B;
  const int64_t Npad = h->Npad;
  L1Dims d;
  d.nC = (int)round_up(B, 64);
  d.nmat = bt ? 1 : (s1.loocv ? 1 : K) * R1;
  d.n_aug = d.nC + 64 + (s1.loocv ? (int)Npad : 0);
  d.cm_stride = (int64_t)d.n_aug * d.nC;
  d.ntiles = (int)(Npad / 128);
  s1.l1_nC = d.nC;
  s1.l1_nmat = d.nmat;
  s1.l1_n_aug = d.n_aug;
  s1.l1_bt = bt;                                          // which prediction route rg_loco takes after this fit
  l1_setup_chunks(h, s1, d.nC);
  s1.l1_part.alloc((size_t)s1.l1_nchunks * d.nC * d.nC);
  s1.l1_part_y.alloc((size_t)s1.l1_nchunks * B);
  s1.l1_cm.alloc((size_t)d.nmat * d.cm_stride);
  s1.l1_inv.alloc(chol_inv_elems(d.nC, d.nmat));
  s1.l1_tau.alloc((size_t)P * R1);
  if (s1.loocv) {
    s1.l1_zrows.alloc((size_t)P * Npad * d.nC);
    s1.l1_hvec.alloc((size_t)P * Npad);
    s1.l1_bvec.alloc((size_t)P * d.nC);
  } else {
    s1.l1_beta.alloc((size_t)P * K * R1 * d.nC);
  }
  RG_CUDA(cudaMemsetAsync(s1.l1_cm.p, 0, (size_t)d.nmat * d.cm_stride * 8, h->stream));
  s1.best_idx.assign(P, 0);
  return d;
}

// Tau selection (src/Data.cpp:1021-1037) for phenotype p and tau j: the nrows cumsum rows of the pair, and
// s1.best_idx[p] (copied to best_idx) moves to j when perf is below `best`, the lowest criterion of the phenotype so
// far (1e10 before its first tau).  The phenotypes a handle does not fit (rg_l1_select) never get here: their cumsum
// rows and best_idx entries stay as the caller passed them.
static void l1_record_tau(rg_ctx* h, Step1State& s1, int p, int j, const double* rows, int nrows, double perf, double& best,
                          double* cumsum, int32_t* best_idx) {
  if (cumsum) for (int k = 0; k < nrows; ++k) cumsum[((size_t)k * h->P + p) * s1.R1 + j] = rows[k];
  if (perf < best) { best = perf; s1.best_idx[p] = j; }
  if (best_idx) best_idx[p] = s1.best_idx[p];
}

// The LOOCV state rg_loco reads at tau*: the nC coefficients b (a device or a host array, per `kind`) into l1_bvec[p],
// and the sample rows of system `sys` backsolved against its factor (inverse blocks at inv) into z_i = H^-1 w_i,
// copied to l1_zrows[p].
static void l1_keep_loocv_state(rg_ctx* h, Step1State& s1, int p, double* sys, const double* inv, const double* b, cudaMemcpyKind kind) {
  cudaStream_t s = h->stream;
  const int nC = s1.l1_nC;
  const int64_t Npad = h->Npad;
  RG_CUDA(cudaMemcpyAsync(s1.l1_bvec.p + (size_t)p * nC, b, (size_t)nC * 8, kind, s));
  launch_chol_rows_backsolve(sys, (int64_t)s1.l1_n_aug * nC, nC, nC + 64, (int)Npad, 1, inv, s);
  RG_CUDA(cudaMemcpyAsync(s1.l1_zrows.p + (size_t)p * Npad * nC, sys + (size_t)(nC + 64) * nC, (size_t)Npad * nC * 8,
                          cudaMemcpyDeviceToDevice, s));
  h->launches += 1;
}

static void l1_fit(rg_ctx* h, const double* tau_host, double* cumsum, int32_t* best_idx) {
  Step1State& s1 = step1(h);
  const L1Dims d = l1_begin(h, s1, false);
  cudaStream_t s = h->stream;
  const int K = s1.K, R1 = s1.R1, P = h->P, B = (int)s1.B, nC = d.nC, nmat = d.nmat, nch = s1.l1_nchunks;
  const int64_t Npad = h->Npad, part_stride = (int64_t)nC * nC, cm_stride = d.cm_stride;
  const int NV = kMaxRidge * 3 + 2;
  s1.l1_sums.alloc((size_t)P * NV);
  s1.l1_part_out.alloc((size_t)d.ntiles * NV);
  RG_CUDA(cudaMemcpyAsync(s1.l1_tau.p, tau_host, (size_t)P * R1 * 8, cudaMemcpyHostToDevice, s));
  for (int p = 0; p < P; ++p) {
    if (!s1.l1_select[p]) continue;                       // fitted by the rank that owns this phenotype
    const double* Wp = s1.W_host_tab[p];
    const int ycol = h->C + p;
    launch_l1_gram(Wp, Npad, B, s1.l1_chunks.p, nch, s1.l1_part.p, part_stride, nC, s);
    launch_l1_xty(Wp, Npad, s1.xy.p, s1.cpp, ycol, s1.l1_chunks.p, nch, s1.l1_part_y.p, B, s);
    launch_l1_assemble(s1.l1_part.p, part_stride, nC, s1.l1_part_y.p, 0, 1, s1.l1_fold_chunks.p, K, R1,
                       s1.l1_tau.p + (size_t)p * R1, B, nC, s1.l1_cm.p, cm_stride, s1.loocv, s);
    if (s1.loocv) launch_l1_loocv_fill(Wp, Npad, B, nC, s1.l1_cm.p, cm_stride, nC + 64, R1, Npad, s);
    launch_chol_factor(s1.l1_cm.p, cm_stride, nC, d.n_aug, nmat, s1.l1_inv.p, s1.err_slot.p, (long long)(1ll << 41) + p * 1024, s);
    if (s1.loocv) {
      // CV sums of the closed-form LOO predictions for every tau, then the state rg_loco needs at tau*
      launch_l1_loocv_sums(s1.l1_cm.p, cm_stride, nC, B, nC + 64, s1.xy.p, s1.cpp, ycol, s1.l1_part_out.p, R1, d.ntiles,
                           s1.l1_sums.p + (size_t)p * NV, s);
      std::vector<double> sv((size_t)R1 * 3);
      RG_CUDA(cudaMemcpyAsync(sv.data(), s1.l1_sums.p + (size_t)p * NV, sv.size() * 8, cudaMemcpyDeviceToHost, s));
      double ne = 0.0;
      RG_CUDA(cudaMemcpyAsync(&ne, s1.neff.p + p, 8, cudaMemcpyDeviceToHost, s));
      RG_CUDA(cudaStreamSynchronize(s));
      const double sy2 = ne - (double)h->C;                              // src/Step1_Models.cpp:891
      double best = 1e10;
      for (int j = 0; j < R1; ++j) {
        const double r[5] = {sv[3 * j], 0.0, sv[3 * j + 1], sy2, sv[3 * j + 2]};   // Sx, Sy, Sx2, Sy2, Sxy
        l1_record_tau(h, s1, p, j, r, 5, (r[2] + r[3] - 2 * r[4]) / ne, best, cumsum, best_idx);
      }
      const int bj = s1.best_idx[p];
      double* sys = s1.l1_cm.p + (size_t)bj * cm_stride;
      const double* inv = s1.l1_inv.p + (size_t)bj * (nC / 64) * 64 * 64;
      launch_rows_sqnorm(sys + (size_t)(nC + 64) * nC, nC, B, s1.l1_hvec.p + (size_t)p * Npad, d.ntiles, s);
      launch_chol_backsolve(sys, cm_stride, nC, 1, 1, inv, s);   // b = H W^T y
      l1_keep_loocv_state(h, s1, p, sys, inv, sys + (size_t)nC * nC, cudaMemcpyDeviceToDevice);
      h->launches += 5;
      continue;
    }
    launch_chol_backsolve(s1.l1_cm.p, cm_stride, nC, 1, nmat, s1.l1_inv.p, s);
    // keep beta[f][r][0:nC] (RHS row nC of every system)
    RG_CUDA(cudaMemcpy2DAsync(s1.l1_beta.p + (size_t)p * nmat * nC, (size_t)nC * 8,
                              s1.l1_cm.p + (size_t)nC * nC, (size_t)cm_stride * 8, (size_t)nC * 8, nmat,
                              cudaMemcpyDeviceToDevice, s));
    launch_l1_pred_sums(Wp, Npad, B, R1, s1.l1_beta.p + (size_t)p * nmat * nC, nC, s1.tile_fold.p, s1.xy.p, s1.cpp,
                        ycol, s1.l1_part_out.p, d.ntiles, s1.l1_sums.p + (size_t)p * NV, s);
    h->launches += 5 + chol_num_launches(nC) + 1 + 2;
  }
  if (!s1.loocv) {
    std::vector<double> sums((size_t)P * NV), neff(P);
    RG_CUDA(cudaMemcpyAsync(sums.data(), s1.l1_sums.p, sums.size() * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaMemcpyAsync(neff.data(), s1.neff.p, P * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaStreamSynchronize(s));
    for (int p = 0; p < P; ++p) {
      if (!s1.l1_select[p]) continue;
      const double* v = &sums[(size_t)p * NV];
      double best = 1e10;
      for (int j = 0; j < R1; ++j) {
        const double r[5] = {v[3 * j], v[3 * kMaxRidge], v[3 * j + 1], v[3 * kMaxRidge + 1], v[3 * j + 2]};
        l1_record_tau(h, s1, p, j, r, 5, (r[2] + r[3] - 2 * r[4]) / neff[p], best, cumsum, best_idx);
      }
    }
  }
  s1.l1_done = true;
}


// ------------------------------------------------------------------ binary traits: logistic level 1
namespace {
constexpr int kNiterRidge = 100, kNiterLsL1 = 25;            // src/Regenie.hpp:287, :338
constexpr double kL1RidgeTol = 1e-4, kL1RidgeEps = 1e-5, kTolL1 = 1e-8, kNumtolL1 = 1e-6;   // :289, :290, :226

struct LgState {
  rg_ctx* h;
  Step1State& s1;
  const double* Wp;
  int B, nC, nch;
  int64_t Npad, cm_stride, part_stride;
  const double* off;
  const int8_t* ym;
  std::vector<double> beta;     // host copy of the coefficients
};

double max_abs(const std::vector<double>& v) {
  double m = 0.0;
  for (double x : v) m = std::max(m, std::fabs(x));
  return m;
}

// eta, w, residual and deviance at `b` (device vectors are overwritten)
double lg_eval(LgState& st, const std::vector<double>& b) {
  rg_ctx* h = st.h;
  cudaStream_t s = h->stream;
  RG_CUDA(cudaMemcpyAsync(st.s1.lg_beta.p, b.data(), (size_t)st.B * 8, cudaMemcpyHostToDevice, s));
  launch_l1_bt_eta(st.Wp, st.Npad, st.B, st.s1.lg_beta.p, st.off, st.ym, st.s1.lg_eta.p, st.s1.lg_wm.p, st.s1.lg_res.p,
                   st.s1.lg_devp.p, st.s1.lg_scal.p, s);
  double d = 0.0;
  RG_CUDA(cudaMemcpyAsync(&d, st.s1.lg_scal.p, 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaStreamSynchronize(s));
  h->launches += 2;
  return d;
}

// score = W^T (y - p) m - tau b at the state of the last lg_eval
std::vector<double> lg_score(LgState& st, double tau, const std::vector<double>& b) {
  rg_ctx* h = st.h;
  cudaStream_t s = h->stream;
  RG_CUDA(cudaMemcpyAsync(st.s1.lg_beta.p, b.data(), (size_t)st.B * 8, cudaMemcpyHostToDevice, s));
  launch_l1_xty(st.Wp, st.Npad, st.s1.lg_res.p, 1, 0, st.s1.l1_chunks.p, st.nch, st.s1.l1_part_y.p, st.B, s);
  launch_l1_bt_score(st.s1.l1_part_y.p, st.nch, st.B, st.nC, tau, st.s1.lg_beta.p, st.s1.lg_score.p, nullptr, s);
  std::vector<double> sc(st.B);
  RG_CUDA(cudaMemcpyAsync(sc.data(), st.s1.lg_score.p, (size_t)st.B * 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaStreamSynchronize(s));
  h->launches += 2;
  return sc;
}

// H = tau I + W^T diag(w m) W at the current weights, assembled into system 0 (the caller factors it)
void lg_factor(LgState& st, double tau) {
  rg_ctx* h = st.h;
  cudaStream_t s = h->stream;
  const int nC = st.nC;
  launch_l1_scale_rows(st.Wp, st.Npad, st.B, st.s1.lg_wm.p, st.s1.lg_Ws.p, s);
  launch_l1_gram(st.s1.lg_Ws.p, st.Npad, st.B, st.s1.l1_chunks.p, st.nch, st.s1.l1_part.p, st.part_stride, nC, s);
  RG_CUDA(cudaMemcpyAsync(st.s1.l1_tau.p, &tau, 8, cudaMemcpyHostToDevice, s));
  // the RHS row is (re)written by the caller after this; part_y content is irrelevant here
  launch_l1_assemble(st.s1.l1_part.p, st.part_stride, nC, st.s1.l1_part_y.p, 0, 1, st.s1.lg_all_chunks.p, 1, 1, st.s1.l1_tau.p,
                     st.B, nC, st.s1.l1_cm.p, st.cm_stride, 1, s);
  h->launches += 3;
}

// the Newton step H^-1 score at the current weights; `tag` marks a failed factorisation in err_slot
std::vector<double> lg_step(LgState& st, double tau, const std::vector<double>& score, long long tag) {
  rg_ctx* h = st.h;
  cudaStream_t s = h->stream;
  const int nC = st.nC;
  lg_factor(st, tau);
  std::vector<double> rhs(nC, 0.0), step(st.B);
  std::copy(score.begin(), score.end(), rhs.begin());
  RG_CUDA(cudaMemcpyAsync(st.s1.l1_cm.p + (size_t)nC * nC, rhs.data(), (size_t)nC * 8, cudaMemcpyHostToDevice, s));
  launch_chol_factor(st.s1.l1_cm.p, st.cm_stride, nC, nC + 64, 1, st.s1.l1_inv.p, st.s1.err_slot.p, tag, s);
  launch_chol_backsolve(st.s1.l1_cm.p, st.cm_stride, nC, 1, 1, st.s1.l1_inv.p, s);
  RG_CUDA(cudaMemcpyAsync(step.data(), st.s1.l1_cm.p + (size_t)nC * nC, (size_t)st.B * 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaStreamSynchronize(s));
  h->launches += chol_num_launches(nC) + 1;
  return step;
}

// run_log_ridge_loocv (src/Step1_Models.cpp:1288-1375): Newton steps halved until the penalised deviance drops;
// beta in/out (warm start)
bool lg_newton(LgState& st, double tau) {
  const int B = st.B;
  std::vector<double>& beta = st.beta;
  auto pen = [&](const std::vector<double>& b) { double q = 0.0; for (double v : b) q += v * v; return tau * q; };
  double fn_start = lg_eval(st, beta) + pen(beta), fn_end = fn_start;
  std::vector<double> score = lg_score(st, tau, beta), betanew = beta;
  bool dev_conv = false;
  for (int it = 0; it < kNiterRidge; ++it) {
    std::vector<double> step = lg_step(st, tau, score, (long long)(1ll << 42));
    for (int ls = 0; ls < kNiterLsL1; ++ls) {
      for (int c = 0; c < B; ++c) betanew[c] = beta[c] + step[c];
      fn_end = lg_eval(st, betanew) + pen(betanew);
      if (fn_end < fn_start + kNumtolL1) break;
      for (auto& v : step) v /= 2.0;
    }
    score = lg_score(st, tau, betanew);
    dev_conv = std::fabs(fn_end - fn_start) / (0.01 + std::fabs(fn_end)) < kTolL1;
    beta = betanew;
    if (max_abs(score) < kL1RidgeTol) return true;
    fn_start = fn_end;
  }
  return dev_conv;
}

// IRLS of ridge_logistic_level_1 (src/Step1_Models.cpp:966-1157): full Newton steps (the IRLS solve) until the score
// is below kL1RidgeTol; beta in/out (warm start)
bool lg_irls(LgState& st, double tau) {
  lg_eval(st, st.beta);
  std::vector<double> score = lg_score(st, tau, st.beta);
  for (int it = 0; it < kNiterRidge; ++it) {
    const std::vector<double> step = lg_step(st, tau, score, (long long)(1ll << 42) + 2);
    for (int c = 0; c < st.B; ++c) st.beta[c] += step[c];
    lg_eval(st, st.beta);
    score = lg_score(st, tau, st.beta);
    if (max_abs(score) < kL1RidgeTol) return true;
  }
  return false;
}

// leverages q_i = w_i^T H^-1 w_i at the converged state (sample rows as RHS rows of the factorisation)
void lg_leverages(LgState& st, double tau, int ntiles) {
  rg_ctx* h = st.h;
  cudaStream_t s = h->stream;
  const int nC = st.nC;
  lg_factor(st, tau);
  RG_CUDA(cudaMemsetAsync(st.s1.l1_cm.p + (size_t)nC * nC, 0, (size_t)64 * nC * 8, s));
  launch_l1_loocv_fill(st.Wp, st.Npad, st.B, nC, st.s1.l1_cm.p, st.cm_stride, nC + 64, 1, st.Npad, s);
  launch_chol_factor(st.s1.l1_cm.p, st.cm_stride, nC, nC + 64 + (int)st.Npad, 1, st.s1.l1_inv.p, st.s1.err_slot.p,
                     (long long)(1ll << 42) + 1, s);
  launch_rows_sqnorm(st.s1.l1_cm.p + (size_t)(nC + 64) * nC, nC, st.B, st.s1.lg_q.p, ntiles, s);
  h->launches += chol_num_launches(nC) + 2;
}
}  // namespace

// ridge_logistic_level_1, k-fold branch (src/Step1_Models.cpp:966-1157): IRLS on the samples outside fold i, warm
// starts over tau, CV sums over fold i.
static void l1_fit_bt_kfold_pheno(rg_ctx* h, Step1State& s1, LgState& st, int p, const std::vector<int8_t>& ym, const double* tau_p,
                                  double* cs_out /* [R1][6] */) {
  cudaStream_t s = h->stream;
  const int K = s1.K, R1 = s1.R1, nC = st.nC;
  const int64_t Npad = h->Npad;
  std::vector<int8_t> ymv(Npad);
  std::vector<double> bpad(nC, 0.0);
  for (int j = 0; j < 6 * R1; ++j) cs_out[j] = 0.0;
  RG_CUDA(cudaMemsetAsync(s1.lg_q.p, 0, Npad * 8, s));
  for (int f = 0; f < K; ++f) {
    const int64_t f0 = s1.fold_pad_start[f], f1 = f0 + s1.fold_pad_len[f];
    auto upload = [&](bool train) {
      for (int64_t t = 0; t < Npad; ++t) {
        const bool in_fold = t >= f0 && t < f1;
        ymv[t] = (in_fold != train) ? ym[t] : 0;
      }
      RG_CUDA(cudaMemcpyAsync(s1.lg_ym.p, ymv.data(), Npad, cudaMemcpyHostToDevice, s));
      RG_CUDA(cudaStreamSynchronize(s));
    };
    std::fill(st.beta.begin(), st.beta.end(), 0.0);
    for (int j = 0; j < R1; ++j) {
      upload(true);
      if (!lg_irls(st, tau_p[j]))
        throw Error{"Penalized logistic regression did not converge (level 1, phenotype " + std::to_string(p + 1) + ")"};
      std::copy(st.beta.begin(), st.beta.end(), bpad.begin());
      RG_CUDA(cudaMemcpyAsync(s1.l1_beta.p + ((size_t)p * K * R1 + (size_t)f * R1 + j) * nC, bpad.data(), (size_t)nC * 8,
                              cudaMemcpyHostToDevice, s));
      // CV sums over the held-out fold: eta is already at the converged coefficients for every sample
      upload(false);
      double cs[6];
      launch_l1_bt_loo_sums(s1.lg_eta.p, s1.lg_q.p, s1.lg_wm.p, s1.lg_res.p, s1.lg_ym.p, kL1RidgeEps, nullptr,
                            s1.lg_devp.p, s1.lg_scal.p, Npad, s);
      RG_CUDA(cudaMemcpyAsync(cs, s1.lg_scal.p, 48, cudaMemcpyDeviceToHost, s));
      RG_CUDA(cudaStreamSynchronize(s));
      h->launches += 2;
      for (int k = 0; k < 6; ++k) cs_out[6 * j + k] += cs[k];
    }
  }
}

static void l1_fit_bt(rg_ctx* h, const double* y_raw, const double* offset, const double* tau_host, double* cumsum,
                      int32_t* best_idx) {
  Step1State& s1 = step1(h);
  const L1Dims d = l1_begin(h, s1, true);
  cudaStream_t s = h->stream;
  const int R1 = s1.R1, P = h->P, B = (int)s1.B, nC = d.nC, nch = s1.l1_nchunks;
  const int64_t Npad = h->Npad, N = h->N;
  {
    const int2 all = make_int2(0, nch);
    s1.lg_all_chunks.alloc(1);
    RG_CUDA(cudaMemcpyAsync(s1.lg_all_chunks.p, &all, sizeof(int2), cudaMemcpyHostToDevice, s));
  }
  s1.lg_Ws.alloc((size_t)Npad * B); s1.lg_eta.alloc(Npad); s1.lg_wm.alloc(Npad);
  s1.lg_res.alloc(Npad); s1.lg_off.alloc(Npad); s1.lg_beta.alloc(nC); s1.lg_score.alloc(nC); s1.lg_q.alloc(Npad);
  s1.lg_devp.alloc((size_t)d.ntiles * 6); s1.lg_scal.alloc(8); s1.lg_ym.alloc(Npad);
  for (int p = 0; p < P; ++p) {
    if (!s1.l1_select[p]) continue;
    // pad-order copies of the trait's 0/1 values, mask and null-model offset
    std::vector<double> off(Npad, 0.0);
    std::vector<int8_t> ym(Npad, 0);
    for (int64_t i = 0; i < N; ++i) {
      const int64_t t = s1.pad_of[i];
      off[t] = offset[(size_t)p * N + i];
      ym[t] = h->maskh[(size_t)p * N + i] ? (y_raw[(size_t)p * N + i] != 0.0 ? 2 : 1) : 0;
    }
    RG_CUDA(cudaMemcpyAsync(s1.lg_off.p, off.data(), Npad * 8, cudaMemcpyHostToDevice, s));
    RG_CUDA(cudaMemcpyAsync(s1.lg_ym.p, ym.data(), Npad, cudaMemcpyHostToDevice, s));
    RG_CUDA(cudaStreamSynchronize(s));
    LgState st{h, s1, s1.W_host_tab[p], B, nC, nch, Npad, d.cm_stride, (int64_t)nC * nC, s1.lg_off.p, s1.lg_ym.p,
               std::vector<double>(B, 0.0)};
    double best = 1e10;
    double ne = 0.0;
    for (int64_t i = 0; i < N; ++i) ne += h->maskh[(size_t)p * N + i] ? 1.0 : 0.0;
    if (!s1.loocv) {
      std::vector<double> cs((size_t)6 * R1);
      l1_fit_bt_kfold_pheno(h, s1, st, p, ym, tau_host + (size_t)p * R1, cs.data());
      for (int j = 0; j < R1; ++j) l1_record_tau(h, s1, p, j, &cs[6 * j], 6, cs[6 * j + 5] / ne, best, cumsum, best_idx);
      continue;
    }
    for (int j = 0; j < R1; ++j) {
      const double tau = tau_host[(size_t)p * R1 + j];
      if (!lg_newton(st, tau)) throw Error{"ridge logistic regression did not converge (level 1, phenotype " + std::to_string(p + 1) + ")"};
      lg_eval(st, st.beta);                       // weights / residuals at the converged coefficients
      lg_leverages(st, tau, d.ntiles);
      double cs[6];
      launch_l1_bt_loo_sums(s1.lg_eta.p, s1.lg_q.p, s1.lg_wm.p, s1.lg_res.p, s1.lg_ym.p, kL1RidgeEps, nullptr,
                            s1.lg_devp.p, s1.lg_scal.p, Npad, s);
      RG_CUDA(cudaMemcpyAsync(cs, s1.lg_scal.p, 48, cudaMemcpyDeviceToHost, s));
      RG_CUDA(cudaStreamSynchronize(s));
      h->launches += 2;
      l1_record_tau(h, s1, p, j, cs, 6, cs[5] / ne, best, cumsum, best_idx);   // -logLik / N, src/Data.cpp:1025-1037
    }
    // state for rg_loco at tau*: refit from zero like make_predictions_binary_loocv (src/Data.cpp:1505-1520)
    const double tau = tau_host[(size_t)p * R1 + s1.best_idx[p]];
    std::fill(st.beta.begin(), st.beta.end(), 0.0);
    if (!lg_newton(st, tau)) throw Error{"ridge logistic regression did not converge (predictions, phenotype " + std::to_string(p + 1) + ")"};
    lg_eval(st, st.beta);
    lg_leverages(st, tau, d.ntiles);
    launch_l1_bt_loo_sums(s1.lg_eta.p, s1.lg_q.p, s1.lg_wm.p, s1.lg_res.p, s1.lg_ym.p, kL1RidgeEps,
                          s1.l1_hvec.p + (size_t)p * Npad, s1.lg_devp.p, s1.lg_scal.p, Npad, s);
    std::vector<double> bpad(nC, 0.0);
    std::copy(st.beta.begin(), st.beta.end(), bpad.begin());
    l1_keep_loocv_state(h, s1, p, s1.l1_cm.p, s1.l1_inv.p, bpad.data(), cudaMemcpyHostToDevice);
    RG_CUDA(cudaStreamSynchronize(s));
    h->launches += 2;
  }
  s1.l1_done = true;
}

static void loco(rg_ctx* h, const int32_t* chr_of_block, double* pred_out) {
  Step1State& s1 = step1(h);
  RG_CHECK(s1.l1_done, "rg_l1_fit must run before rg_loco");
  RG_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  const int K = s1.K, R1 = s1.R1, P = h->P, R = s1.R;
  const int nC = s1.l1_nC, nmat = K * R1;
  const int64_t Npad = h->Npad, N = h->N;
  // chromosomes in block order (blocks never straddle chromosomes, src/Data.cpp:311-334)
  std::vector<int32_t> chrs, col_start;
  for (int b = 0; b < s1.total_blocks; ++b) {
    const int c = chr_of_block[b];
    RG_CHECK(c >= 1 && c <= 23, "chromosome out of range");
    if (chrs.empty() || chrs.back() != c) {
      RG_CHECK(chrs.empty() || c > chrs.back(), "blocks must be ordered by chromosome");
      chrs.push_back(c);
      col_start.push_back(b * R);
    }
  }
  col_start.push_back(s1.total_blocks * R);
  const int nchr = (int)chrs.size();
  s1.l1_chr_cols.alloc(col_start.size());
  RG_CUDA(cudaMemcpyAsync(s1.l1_chr_cols.p, col_start.data(), col_start.size() * 4, cudaMemcpyHostToDevice, s));
  s1.l1_pred.alloc((size_t)nchr * Npad);
  std::vector<double> pred((size_t)nchr * Npad);
  s1.prs_host.assign((size_t)P * N, 0.0);
  for (int p = 0; p < P; ++p) {
    if (!s1.l1_select[p]) continue;
    if (s1.l1_bt && s1.loocv)
      launch_l1_bt_chr_pred(s1.W_host_tab[p], Npad, nC, s1.l1_zrows.p + (size_t)p * Npad * nC,
                            s1.l1_hvec.p + (size_t)p * Npad, s1.l1_bvec.p + (size_t)p * nC, nchr, s1.l1_chr_cols.p,
                            s1.l1_pred.p, Npad, s);
    else if (s1.loocv)
      launch_l1_loocv_chr_pred(s1.W_host_tab[p], Npad, (int)s1.B, nC, s1.l1_zrows.p + (size_t)p * Npad * nC,
                               s1.l1_hvec.p + (size_t)p * Npad, s1.l1_bvec.p + (size_t)p * nC, s1.xy.p, s1.cpp,
                               h->C + p, nchr, s1.l1_chr_cols.p, s1.l1_pred.p, Npad, s);
    else
      launch_l1_chr_pred(s1.W_host_tab[p], Npad, nchr, s1.l1_chr_cols.p,
                         s1.l1_beta.p + (size_t)p * nmat * nC, nC, R1, s1.best_idx[p], s1.tile_fold.p, s1.l1_pred.p, Npad, s);
    h->launches += 1;
    RG_CUDA(cudaMemcpyAsync(pred.data(), s1.l1_pred.p, pred.size() * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaStreamSynchronize(s));
    // LOCO assembly (src/Data.cpp:1846-1858): all-chromosome sum minus the chromosome's own part
    double* out = pred_out + (size_t)p * 23 * N;
    for (int64_t i = 0; i < N; ++i) {
      const int64_t t = s1.pad_of[i];
      double tot = 0.0;
      for (int ci = 0; ci < nchr; ++ci) tot += pred[(size_t)ci * Npad + t];
      s1.prs_host[(size_t)p * N + i] = tot;
      for (int c = 0; c < 23; ++c) out[(size_t)c * N + i] = tot;
      for (int ci = 0; ci < nchr; ++ci) out[(size_t)(chrs[ci] - 1) * N + i] = tot - pred[(size_t)ci * Npad + t];
    }
  }
}

extern "C" {

int rg_l1_fit(rg_handle h, const double* tau, double* cumsum, int32_t* best_idx) {
  RG_API_BEGIN
  RG_CHECK(h && tau, "null argument");
  l1_fit(h, tau, cumsum, best_idx);
  RG_CUDA(cudaGetLastError());
  RG_API_END
}

int rg_l1_fit_bt(rg_handle h, const double* y_raw, const double* offset, const double* tau, double* cumsum,
                 int32_t* best_idx) {
  RG_API_BEGIN
  RG_CHECK(h && y_raw && offset && tau, "null argument");
  l1_fit_bt(h, y_raw, offset, tau, cumsum, best_idx);
  RG_CUDA(cudaGetLastError());
  RG_API_END
}

int rg_loco(rg_handle h, const int32_t* chr_of_block, double* pred_out) {
  RG_API_BEGIN
  RG_CHECK(h && chr_of_block && pred_out, "null argument");
  loco(h, chr_of_block, pred_out);
  RG_CUDA(cudaGetLastError());
  RG_API_END
}

int rg_prs(rg_handle h, double* prs_out) {
  RG_API_BEGIN
  RG_CHECK(h && prs_out, "null argument");
  const Step1State& s1 = step1(h);
  RG_CHECK(s1.prs_host.size() == (size_t)h->P * h->N, "rg_loco must run before rg_prs");
  memcpy(prs_out, s1.prs_host.data(), s1.prs_host.size() * sizeof(double));
  RG_API_END
}

int rg_W_info(rg_handle h, int32_t ph, void** dev_ptr, int64_t* ld, int64_t* ncols) {
  RG_API_BEGIN
  RG_CHECK(h && ph >= 0 && ph < h->P, "bad argument");
  Step1State& s1 = step1(h);
  RG_CUDA(cudaSetDevice(h->device));
  ensure_W(h, s1);
  if (dev_ptr) *dev_ptr = s1.W_host_tab[ph];
  if (ld) *ld = h->Npad;
  if (ncols) *ncols = s1.B;
  RG_API_END
}

}  // extern "C"
