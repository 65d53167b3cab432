// Level-1 ridge, LOCO assembly and Step-2 entry points of the C ABI (include/rg_b200.h).
#include <string.h>

#include <algorithm>
#include <cmath>
#include <string>

#include "context.cuh"

using namespace rg;

static void l1_setup_chunks(rg_ctx* h, int nC, int ldp) {
  cudaStream_t s = h->stream;
  const int K = h->K;
  const int64_t Npad = h->Npad;
  // chunk table for the sample-axis reductions: bounded partial storage (<= ~1 GiB).  A fold of n samples takes
  // ceil(n / len) chunks <= n / len + 1, so the K folds take at most max_chunks chunks of nC x ldp partials.
  {
    const int64_t per = (int64_t)nC * ldp * 8;
    const int64_t max_chunks = std::max<int64_t>(K, (1ll << 30) / per);
    int64_t len = round_up(std::max<int64_t>(kStatChunk, ceil_div(Npad, max_chunks - K + 1)), 128);
    h->l1_chunk_len = len;
    std::vector<int4> chunks;
    std::vector<int2> fold_chunks(K);
    for (int f = 0; f < K; ++f) {
      fold_chunks[f].x = (int)chunks.size();
      for (int64_t o = 0; o < h->fold_pad_len[f]; o += len)
        chunks.push_back(make_int4((int)(h->fold_pad_start[f] + o),
                                   (int)std::min<int64_t>(len, h->fold_pad_len[f] - o), f, 0));
      fold_chunks[f].y = (int)chunks.size();
    }
    h->l1_nchunks = (int)chunks.size();
    h->l1_chunks.alloc(chunks.size());
    h->l1_fold_chunks.alloc(K);
    RG_CUDA(cudaMemcpyAsync(h->l1_chunks.p, chunks.data(), chunks.size() * sizeof(int4), cudaMemcpyHostToDevice, s));
    RG_CUDA(cudaMemcpyAsync(h->l1_fold_chunks.p, fold_chunks.data(), K * sizeof(int2), cudaMemcpyHostToDevice, s));
    RG_CUDA(cudaStreamSynchronize(s));
  }
}

static void l1_fit(rg_ctx* h, const double* tau_host, double* cumsum, int32_t* best_idx) {
  RG_CHECK(h->kind == 1, "handle is not a Step-1 handle");
  h->l1_done = false;                                     // until this fit completes, rg_loco and the hooks refuse
  RG_CHECK(h->R1 >= 1 && h->R1 <= kMaxRidge, "n_ridge_l1 out of range");
  RG_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  rg::sync_lanes(h);   // all level-0 blocks are in W
  ensure_W(h);
  const int K = h->K, R1 = h->R1, P = h->P;
  const int B = (int)h->B;
  const int loocv = h->loocv;
  const int nC = (int)round_up(B, 64), n_aug = nC + 64 + (loocv ? (int)h->Npad : 0), nmat = (loocv ? 1 : K) * R1;
  const int ldp = nC;
  const int64_t Npad = h->Npad;
  h->l1_nC = nC;
  h->l1_nmat = nmat;
  h->l1_n_aug = n_aug;
  h->l1_bt = false;                                       // rg_loco takes the QT route after this fit
  l1_setup_chunks(h, nC, ldp);
  const int nch = h->l1_nchunks;
  const int64_t part_stride = (int64_t)nC * ldp;
  const int64_t cm_stride = (int64_t)n_aug * nC;
  const int ntiles = (int)(Npad / 128);
  const int NV = kMaxRidge * 3 + 2;
  h->l1_part.alloc((size_t)nch * part_stride);
  h->l1_part_y.alloc((size_t)nch * B);
  h->l1_cm.alloc((size_t)nmat * cm_stride);
  h->l1_inv.alloc(chol_inv_elems(nC, nmat));
  h->l1_beta.alloc((size_t)P * nmat * nC);
  h->l1_sums.alloc((size_t)P * NV);
  h->l1_part_out.alloc((size_t)ntiles * NV);
  h->l1_tau.alloc((size_t)P * R1);
  RG_CUDA(cudaMemcpyAsync(h->l1_tau.p, tau_host, (size_t)P * R1 * 8, cudaMemcpyHostToDevice, s));
  RG_CUDA(cudaMemsetAsync(h->l1_cm.p, 0, (size_t)nmat * cm_stride * 8, s));
  std::vector<int> loocv_best(P, 0);
  std::vector<double> loocv_cs((size_t)5 * P * R1, 0.0);
  if (loocv) {
    h->l1_zrows.alloc((size_t)P * Npad * nC);
    h->l1_hvec.alloc((size_t)P * Npad);
    h->l1_bvec.alloc((size_t)P * nC);
  }
  for (int p = 0; p < P; ++p) {
    if (!h->l1_select[p]) continue;                       // fitted by the rank that owns this phenotype
    const double* Wp = h->W_host_tab[p];
    const int ycol = h->C + p;
    launch_l1_gram(Wp, Npad, B, h->l1_chunks.p, nch, h->l1_part.p, part_stride, ldp, s);
    launch_l1_xty(Wp, Npad, h->xy.p, h->cpp, ycol, h->l1_chunks.p, nch, h->l1_part_y.p, B, s);
    launch_l1_assemble(h->l1_part.p, part_stride, ldp, h->l1_part_y.p, h->l1_fold_chunks.p, K, R1,
                       h->l1_tau.p + (size_t)p * R1, B, nC, h->l1_cm.p, cm_stride, loocv, s);
    if (loocv) launch_l1_loocv_fill(Wp, Npad, B, nC, h->l1_cm.p, cm_stride, nC + 64, R1, Npad, s);
    launch_chol_factor(h->l1_cm.p, cm_stride, nC, n_aug, nmat, h->l1_inv.p, h->err_slot.p, (long long)(1ll << 41) + p * 1024, s);
    if (loocv) {
      // CV sums of the closed-form LOO predictions for every tau, then the state rg_loco needs at tau*
      const int64_t inv_stride = (int64_t)(nC / 64) * 64 * 64;
      launch_l1_loocv_sums(h->l1_cm.p, cm_stride, nC, B, nC + 64, h->xy.p, h->cpp, ycol, h->l1_part_out.p, R1, ntiles,
                           h->l1_sums.p + (size_t)p * NV, s);
      std::vector<double> sv((size_t)R1 * 3);
      RG_CUDA(cudaMemcpyAsync(sv.data(), h->l1_sums.p + (size_t)p * NV, sv.size() * 8, cudaMemcpyDeviceToHost, s));
      double ne = 0.0;
      RG_CUDA(cudaMemcpyAsync(&ne, h->neff.p + p, 8, cudaMemcpyDeviceToHost, s));
      RG_CUDA(cudaStreamSynchronize(s));
      const double sy2 = ne - (double)h->C;                              // src/Step1_Models.cpp:891
      int bj = 0; double bv = 1e10;
      for (int j = 0; j < R1; ++j) {
        const double perf = (sv[3 * j + 1] + sy2 - 2 * sv[3 * j + 2]) / ne;
        if (perf < bv) { bv = perf; bj = j; }
      }
      loocv_best[p] = bj;
      for (int j = 0; j < R1; ++j) {
        loocv_cs[((size_t)0 * P + p) * R1 + j] = sv[3 * j];
        loocv_cs[((size_t)1 * P + p) * R1 + j] = 0.0;
        loocv_cs[((size_t)2 * P + p) * R1 + j] = sv[3 * j + 1];
        loocv_cs[((size_t)3 * P + p) * R1 + j] = sy2;
        loocv_cs[((size_t)4 * P + p) * R1 + j] = sv[3 * j + 2];
      }
      double* sys = h->l1_cm.p + (size_t)bj * cm_stride;
      double* rows = sys + (size_t)(nC + 64) * nC;
      launch_rows_sqnorm(rows, nC, B, h->l1_hvec.p + (size_t)p * Npad, ntiles, s);
      launch_chol_backsolve(sys, cm_stride, nC, 1, 1, h->l1_inv.p + (size_t)bj * inv_stride, s);   // b = H W^T y
      RG_CUDA(cudaMemcpyAsync(h->l1_bvec.p + (size_t)p * nC, sys + (size_t)nC * nC, (size_t)nC * 8,
                              cudaMemcpyDeviceToDevice, s));
      launch_chol_rows_backsolve(sys, cm_stride, nC, nC + 64, (int)Npad, 1, h->l1_inv.p + (size_t)bj * inv_stride, s);
      RG_CUDA(cudaMemcpyAsync(h->l1_zrows.p + (size_t)p * Npad * nC, rows, (size_t)Npad * nC * 8,
                              cudaMemcpyDeviceToDevice, s));
      h->launches += 6;
      continue;
    }
    launch_chol_backsolve(h->l1_cm.p, cm_stride, nC, 1, nmat, h->l1_inv.p, s);
    // keep beta[f][r][0:nC] (RHS row nC of every system)
    RG_CUDA(cudaMemcpy2DAsync(h->l1_beta.p + (size_t)p * nmat * nC, (size_t)nC * 8,
                              h->l1_cm.p + (size_t)nC * nC, (size_t)cm_stride * 8, (size_t)nC * 8, nmat,
                              cudaMemcpyDeviceToDevice, s));
    launch_l1_pred_sums(Wp, Npad, B, R1, h->l1_beta.p + (size_t)p * nmat * nC, nC, h->tile_fold.p, h->xy.p, h->cpp,
                        ycol, h->l1_part_out.p, ntiles, h->l1_sums.p + (size_t)p * NV, s);
    h->launches += 5 + chol_num_launches(nC) + 1 + 2;
  }
  if (loocv) {
    h->best_idx.assign(loocv_best.begin(), loocv_best.end());
    if (cumsum) memcpy(cumsum, loocv_cs.data(), loocv_cs.size() * 8);
    if (best_idx) for (int p = 0; p < P; ++p) best_idx[p] = loocv_best[p];
    h->l1_done = true;
    return;
  }
  std::vector<double> sums((size_t)P * NV), neff(P);
  RG_CUDA(cudaMemcpyAsync(sums.data(), h->l1_sums.p, sums.size() * 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaMemcpyAsync(neff.data(), h->neff.p, P * 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaStreamSynchronize(s));
  h->best_idx.assign(P, 0);
  for (int p = 0; p < P; ++p) {
    if (!h->l1_select[p]) continue;
    const double* v = &sums[(size_t)p * NV];
    double best = 1e10;                                   // src/Data.cpp:1021-1037
    for (int j = 0; j < R1; ++j) {
      const double sx = v[3 * j], sx2 = v[3 * j + 1], sxy = v[3 * j + 2], sy = v[3 * kMaxRidge], sy2 = v[3 * kMaxRidge + 1];
      if (cumsum) {
        cumsum[((size_t)0 * P + p) * R1 + j] = sx;
        cumsum[((size_t)1 * P + p) * R1 + j] = sy;
        cumsum[((size_t)2 * P + p) * R1 + j] = sx2;
        cumsum[((size_t)3 * P + p) * R1 + j] = sy2;
        cumsum[((size_t)4 * P + p) * R1 + j] = sxy;
      }
      const double perf = (sx2 + sy2 - 2 * sxy) / neff[p];
      if (perf < best) { best = perf; h->best_idx[p] = j; }
    }
    if (best_idx) best_idx[p] = h->best_idx[p];
  }
  h->l1_done = true;
}


// ------------------------------------------------------------------ binary traits: logistic level 1 (LOOCV)
namespace {
constexpr int kNiterRidge = 100, kNiterLsL1 = 25;            // src/Regenie.hpp:287, :338
constexpr double kL1RidgeTol = 1e-4, kL1RidgeEps = 1e-5, kTolL1 = 1e-8, kNumtolL1 = 1e-6;   // :289, :290, :226

struct LgState {
  rg_ctx* h;
  const double* Wp;
  int B, nC, nch;
  int64_t Npad, cm_stride, part_stride;
  const double* off;
  const int8_t* ym;
  std::vector<double> beta;     // host copy of the coefficients
  double dev = 0.0;             // deviance at the last evaluated beta
};

// eta, p, w, residual and deviance at `b` (device vectors are overwritten)
double lg_eval(LgState& st, const std::vector<double>& b) {
  rg_ctx* h = st.h;
  cudaStream_t s = h->stream;
  RG_CUDA(cudaMemcpyAsync(h->lg_beta.p, b.data(), (size_t)st.B * 8, cudaMemcpyHostToDevice, s));
  launch_l1_bt_eta(st.Wp, st.Npad, st.B, h->lg_beta.p, st.off, st.ym, h->lg_eta.p, h->lg_p.p, h->lg_wm.p, h->lg_res.p,
                   h->lg_devp.p, h->lg_scal.p, s);
  double d = 0.0;
  RG_CUDA(cudaMemcpyAsync(&d, h->lg_scal.p, 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaStreamSynchronize(s));
  h->launches += 2;
  return d;
}

// score = W^T (y - p) m - tau b at the state of the last lg_eval; optionally also into the RHS row of system 0
std::vector<double> lg_score(LgState& st, double tau, const std::vector<double>& b, bool to_rhs) {
  rg_ctx* h = st.h;
  cudaStream_t s = h->stream;
  RG_CUDA(cudaMemcpyAsync(h->lg_beta.p, b.data(), (size_t)st.B * 8, cudaMemcpyHostToDevice, s));
  launch_l1_xty(st.Wp, st.Npad, h->lg_res.p, 1, 0, h->l1_chunks.p, st.nch, h->l1_part_y.p, st.B, s);
  launch_l1_bt_score(h->l1_part_y.p, st.nch, st.B, st.nC, tau, h->lg_beta.p, h->lg_score.p,
                     to_rhs ? h->l1_cm.p + (size_t)st.nC * st.nC : nullptr, s);
  std::vector<double> sc(st.B);
  RG_CUDA(cudaMemcpyAsync(sc.data(), h->lg_score.p, (size_t)st.B * 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaStreamSynchronize(s));
  h->launches += 2;
  return sc;
}

// H = tau I + W^T diag(w m) W at the current weights, factored; n_rows extra RHS rows (sample rows) ride along
void lg_factor(LgState& st, double tau, bool with_rows) {
  rg_ctx* h = st.h;
  cudaStream_t s = h->stream;
  const int nC = st.nC;
  launch_l1_scale_rows(st.Wp, st.Npad, st.B, h->lg_wm.p, h->lg_Ws.p, s);
  launch_l1_gram(h->lg_Ws.p, st.Npad, st.B, h->l1_chunks.p, st.nch, h->l1_part.p, st.part_stride, nC, s);
  RG_CUDA(cudaMemcpyAsync(h->l1_tau.p, &tau, 8, cudaMemcpyHostToDevice, s));
  // the RHS row is (re)written by the caller after this; part_y content is irrelevant here
  launch_l1_assemble(h->l1_part.p, st.part_stride, nC, h->l1_part_y.p, h->lg_all_chunks.p, 1, 1, h->l1_tau.p, st.B, nC,
                     h->l1_cm.p, st.cm_stride, 1, s);
  h->launches += 3;
  (void)with_rows;
}

// run_log_ridge_loocv (src/Step1_Models.cpp:1288-1375); beta in/out (warm start)
bool lg_newton(LgState& st, double tau) {
  rg_ctx* h = st.h;
  cudaStream_t s = h->stream;
  const int B = st.B, nC = st.nC;
  std::vector<double>& beta = st.beta;
  auto pen = [&](const std::vector<double>& b) { double q = 0.0; for (double v : b) q += v * v; return tau * q; };
  double fn_start = lg_eval(st, beta) + pen(beta), fn_end = fn_start;
  std::vector<double> score = lg_score(st, tau, beta, false), betanew = beta, step(B);
  bool dev_conv = false, by_score = false;
  int it = 0;
  while (it < kNiterRidge) {
    ++it;
    lg_factor(st, tau, false);
    // RHS row = score
    std::vector<double> rhs(nC, 0.0);
    std::copy(score.begin(), score.end(), rhs.begin());
    RG_CUDA(cudaMemcpyAsync(h->l1_cm.p + (size_t)nC * nC, rhs.data(), (size_t)nC * 8, cudaMemcpyHostToDevice, s));
    launch_chol_factor(h->l1_cm.p, st.cm_stride, nC, nC + 64, 1, h->l1_inv.p, h->err_slot.p, (long long)(1ll << 42), s);
    launch_chol_backsolve(h->l1_cm.p, st.cm_stride, nC, 1, 1, h->l1_inv.p, s);
    RG_CUDA(cudaMemcpyAsync(step.data(), h->l1_cm.p + (size_t)nC * nC, (size_t)B * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaStreamSynchronize(s));
    h->launches += chol_num_launches(nC) + 1;
    for (int ls = 0; ls < kNiterLsL1; ++ls) {
      for (int c = 0; c < B; ++c) betanew[c] = beta[c] + step[c];
      fn_end = lg_eval(st, betanew) + pen(betanew);
      if (fn_end < fn_start + kNumtolL1) break;
      for (auto& v : step) v /= 2.0;
    }
    score = lg_score(st, tau, betanew, false);
    dev_conv = std::fabs(fn_end - fn_start) / (0.01 + std::fabs(fn_end)) < kTolL1;
    double smax = 0.0;
    for (double v : score) smax = std::max(smax, std::fabs(v));
    if (smax < kL1RidgeTol) { by_score = true; break; }
    beta = betanew;
    fn_start = fn_end;
  }
  beta = betanew;
  return by_score || dev_conv;
}

// leverages q_i = w_i^T H^-1 w_i at the converged state (sample rows as RHS rows of the factorisation)
void lg_leverages(LgState& st, double tau, int ntiles) {
  rg_ctx* h = st.h;
  cudaStream_t s = h->stream;
  const int nC = st.nC;
  lg_factor(st, tau, true);
  RG_CUDA(cudaMemsetAsync(h->l1_cm.p + (size_t)nC * nC, 0, (size_t)64 * nC * 8, s));
  launch_l1_loocv_fill(st.Wp, st.Npad, st.B, nC, h->l1_cm.p, st.cm_stride, nC + 64, 1, st.Npad, s);
  launch_chol_factor(h->l1_cm.p, st.cm_stride, nC, nC + 64 + (int)st.Npad, 1, h->l1_inv.p, h->err_slot.p, (long long)(1ll << 42) + 1, s);
  launch_rows_sqnorm(h->l1_cm.p + (size_t)(nC + 64) * nC, nC, st.B, h->lg_q.p, ntiles, s);
  h->launches += chol_num_launches(nC) + 2;
}
}  // namespace

// ridge_logistic_level_1, k-fold branch (src/Step1_Models.cpp:966-1157): IRLS on the samples outside fold i
// (the Newton step beta + H^-1 score is the IRLS solve), warm starts over tau, CV sums over fold i.
static void l1_fit_bt_kfold_pheno(rg_ctx* h, LgState& st, int p, const std::vector<int8_t>& ym, const double* tau_p,
                                  double* cs_out /* [6][R1] */) {
  cudaStream_t s = h->stream;
  const int K = h->K, R1 = h->R1, B = st.B, nC = st.nC;
  const int64_t Npad = h->Npad;
  std::vector<int8_t> ymv(Npad);
  std::vector<double> bpad(nC, 0.0);
  for (int j = 0; j < 6 * R1; ++j) cs_out[j] = 0.0;
  RG_CUDA(cudaMemsetAsync(h->lg_q.p, 0, Npad * 8, s));
  for (int f = 0; f < K; ++f) {
    const int64_t f0 = h->fold_pad_start[f], f1 = f0 + h->fold_pad_len[f];
    auto upload = [&](bool train) {
      for (int64_t t = 0; t < Npad; ++t) {
        const bool in_fold = t >= f0 && t < f1;
        ymv[t] = (in_fold != train) ? ym[t] : 0;
      }
      RG_CUDA(cudaMemcpyAsync(h->lg_ym.p, ymv.data(), Npad, cudaMemcpyHostToDevice, s));
      RG_CUDA(cudaStreamSynchronize(s));
    };
    std::fill(st.beta.begin(), st.beta.end(), 0.0);
    for (int j = 0; j < R1; ++j) {
      const double tau = tau_p[j];
      upload(true);
      lg_eval(st, st.beta);
      bool converged = false;
      std::vector<double> score = lg_score(st, tau, st.beta, false), step(B), rhs(nC, 0.0);
      for (int it = 0; it < kNiterRidge && !converged; ++it) {
        lg_factor(st, tau, false);
        std::copy(score.begin(), score.end(), rhs.begin());
        RG_CUDA(cudaMemcpyAsync(h->l1_cm.p + (size_t)nC * nC, rhs.data(), (size_t)nC * 8, cudaMemcpyHostToDevice, s));
        launch_chol_factor(h->l1_cm.p, st.cm_stride, nC, nC + 64, 1, h->l1_inv.p, h->err_slot.p, (long long)(1ll << 42) + 2, s);
        launch_chol_backsolve(h->l1_cm.p, st.cm_stride, nC, 1, 1, h->l1_inv.p, s);
        RG_CUDA(cudaMemcpyAsync(step.data(), h->l1_cm.p + (size_t)nC * nC, (size_t)B * 8, cudaMemcpyDeviceToHost, s));
        RG_CUDA(cudaStreamSynchronize(s));
        h->launches += chol_num_launches(nC) + 1;
        for (int c = 0; c < B; ++c) st.beta[c] += step[c];
        lg_eval(st, st.beta);
        score = lg_score(st, tau, st.beta, false);
        double smax = 0.0;
        for (double v : score) smax = std::max(smax, std::fabs(v));
        converged = smax < kL1RidgeTol;
      }
      if (!converged) throw Error{"Penalized logistic regression did not converge (level 1, phenotype " + std::to_string(p + 1) + ")"};
      std::copy(st.beta.begin(), st.beta.end(), bpad.begin());
      RG_CUDA(cudaMemcpyAsync(h->l1_beta.p + ((size_t)p * K * R1 + (size_t)f * R1 + j) * nC, bpad.data(), (size_t)nC * 8,
                              cudaMemcpyHostToDevice, s));
      // CV sums over the held-out fold: eta is already at the converged coefficients for every sample
      upload(false);
      double cs[6];
      launch_l1_bt_loo_sums(h->lg_eta.p, h->lg_q.p, h->lg_wm.p, h->lg_res.p, h->lg_ym.p, kL1RidgeEps, nullptr,
                            h->lg_devp.p, h->lg_scal.p, Npad, s);
      RG_CUDA(cudaMemcpyAsync(cs, h->lg_scal.p, 48, cudaMemcpyDeviceToHost, s));
      RG_CUDA(cudaStreamSynchronize(s));
      h->launches += 2;
      for (int k = 0; k < 6; ++k) cs_out[k * R1 + j] += cs[k];
    }
  }
}

static void l1_fit_bt(rg_ctx* h, const double* y_raw, const double* offset, const double* tau_host, double* cumsum,
                      int32_t* best_idx) {
  RG_CHECK(h->kind == 1, "handle is not a Step-1 handle");
  h->l1_done = false;                                     // as in l1_fit: a fit that fails leaves no fit behind
  RG_CHECK(h->R1 >= 1 && h->R1 <= kMaxRidge, "n_ridge_l1 out of range");
  RG_CHECK(h->B <= 6000, "logistic level 1 supports up to 6000 level-0 predictors (blocks x ridge values) in this build");
  RG_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  rg::sync_lanes(h);
  const int R1 = h->R1, P = h->P, B = (int)h->B;
  const int nC = (int)round_up(B, 64);
  const int64_t Npad = h->Npad, N = h->N;
  const int ntiles = (int)(Npad / 128);
  h->l1_nC = nC;
  l1_setup_chunks(h, nC, nC);
  const int nch = h->l1_nchunks;
  const int loocv = h->loocv;
  const int64_t cm_stride = (int64_t)(nC + 64 + (loocv ? Npad : 0)) * nC;
  h->l1_nmat = 1;                                         // one system, refactored at every Newton step
  h->l1_n_aug = (int)(cm_stride / nC);
  {
    const int2 all = make_int2(0, nch);
    h->lg_all_chunks.alloc(1);
    RG_CUDA(cudaMemcpyAsync(h->lg_all_chunks.p, &all, sizeof(int2), cudaMemcpyHostToDevice, s));
  }
  if (!loocv) h->l1_beta.alloc((size_t)P * h->K * R1 * nC);
  h->l1_part.alloc((size_t)nch * nC * nC);
  h->l1_part_y.alloc((size_t)nch * B);
  h->l1_cm.alloc((size_t)cm_stride);
  h->l1_inv.alloc(chol_inv_elems(nC, 1));
  h->l1_tau.alloc(1);
  if (loocv) {
    h->l1_zrows.alloc((size_t)P * Npad * nC);
    h->l1_hvec.alloc((size_t)P * Npad);
    h->l1_bvec.alloc((size_t)P * nC);
  }
  h->lg_Ws.alloc((size_t)Npad * B); h->lg_eta.alloc(Npad); h->lg_p.alloc(Npad); h->lg_wm.alloc(Npad);
  h->lg_res.alloc(Npad); h->lg_off.alloc(Npad); h->lg_beta.alloc(nC); h->lg_score.alloc(nC); h->lg_q.alloc(Npad);
  h->lg_devp.alloc((size_t)ntiles * 6); h->lg_scal.alloc(8); h->lg_ym.alloc(Npad);
  RG_CUDA(cudaMemsetAsync(h->l1_cm.p, 0, (size_t)cm_stride * 8, s));
  h->best_idx.assign(P, 0);
  for (int p = 0; p < P; ++p) {
    if (!h->l1_select[p]) continue;
    // pad-order copies of the trait's 0/1 values, mask and null-model offset
    std::vector<double> off(Npad, 0.0);
    std::vector<int8_t> ym(Npad, 0);
    for (int64_t i = 0; i < N; ++i) {
      const int64_t t = h->pad_of[i];
      off[t] = offset[(size_t)p * N + i];
      ym[t] = h->maskh[(size_t)p * N + i] ? (y_raw[(size_t)p * N + i] != 0.0 ? 2 : 1) : 0;
    }
    RG_CUDA(cudaMemcpyAsync(h->lg_off.p, off.data(), Npad * 8, cudaMemcpyHostToDevice, s));
    RG_CUDA(cudaMemcpyAsync(h->lg_ym.p, ym.data(), Npad, cudaMemcpyHostToDevice, s));
    RG_CUDA(cudaStreamSynchronize(s));
    LgState st{h, h->W_host_tab[p], B, nC, nch, Npad, cm_stride, (int64_t)nC * nC, h->lg_off.p, h->lg_ym.p,
               std::vector<double>(B, 0.0)};
    double best = 1e10;
    double ne = 0.0;
    for (int64_t i = 0; i < N; ++i) ne += h->maskh[(size_t)p * N + i] ? 1.0 : 0.0;
    if (!loocv) {
      std::vector<double> cs((size_t)6 * R1);
      l1_fit_bt_kfold_pheno(h, st, p, ym, tau_host + (size_t)p * R1, cs.data());
      for (int j = 0; j < R1; ++j) {
        if (cumsum) for (int k = 0; k < 6; ++k) cumsum[((size_t)k * P + p) * R1 + j] = cs[(size_t)k * R1 + j];
        const double perf = cs[(size_t)5 * R1 + j] / ne;
        if (perf < best) { best = perf; h->best_idx[p] = j; }
      }
      if (best_idx) best_idx[p] = h->best_idx[p];
      continue;
    }
    for (int j = 0; j < R1; ++j) {
      const double tau = tau_host[(size_t)p * R1 + j];
      if (!lg_newton(st, tau)) throw Error{"ridge logistic regression did not converge (level 1, phenotype " + std::to_string(p + 1) + ")"};
      lg_eval(st, st.beta);                       // weights / residuals at the converged coefficients
      lg_leverages(st, tau, ntiles);
      double cs[6];
      launch_l1_bt_loo_sums(h->lg_eta.p, h->lg_q.p, h->lg_wm.p, h->lg_res.p, h->lg_ym.p, kL1RidgeEps, nullptr,
                            h->lg_devp.p, h->lg_scal.p, Npad, s);
      RG_CUDA(cudaMemcpyAsync(cs, h->lg_scal.p, 48, cudaMemcpyDeviceToHost, s));
      RG_CUDA(cudaStreamSynchronize(s));
      h->launches += 2;
      if (cumsum) for (int k = 0; k < 6; ++k) cumsum[((size_t)k * P + p) * R1 + j] = cs[k];
      const double perf = cs[5] / ne;             // -logLik / N, src/Data.cpp:1025-1037
      if (perf < best) { best = perf; h->best_idx[p] = j; }
    }
    if (best_idx) best_idx[p] = h->best_idx[p];
    // state for rg_loco at tau*: refit from zero like make_predictions_binary_loocv (src/Data.cpp:1505-1520)
    const double tau = tau_host[(size_t)p * R1 + h->best_idx[p]];
    std::fill(st.beta.begin(), st.beta.end(), 0.0);
    if (!lg_newton(st, tau)) throw Error{"ridge logistic regression did not converge (predictions, phenotype " + std::to_string(p + 1) + ")"};
    lg_eval(st, st.beta);
    lg_leverages(st, tau, ntiles);
    launch_l1_bt_loo_sums(h->lg_eta.p, h->lg_q.p, h->lg_wm.p, h->lg_res.p, h->lg_ym.p, kL1RidgeEps,
                          h->l1_hvec.p + (size_t)p * Npad, h->lg_devp.p, h->lg_scal.p, Npad, s);
    std::vector<double> bpad(nC, 0.0);
    std::copy(st.beta.begin(), st.beta.end(), bpad.begin());
    RG_CUDA(cudaMemcpyAsync(h->l1_bvec.p + (size_t)p * nC, bpad.data(), (size_t)nC * 8, cudaMemcpyHostToDevice, s));
    launch_chol_rows_backsolve(h->l1_cm.p, cm_stride, nC, nC + 64, (int)Npad, 1, h->l1_inv.p, s);
    RG_CUDA(cudaMemcpyAsync(h->l1_zrows.p + (size_t)p * Npad * nC, h->l1_cm.p + (size_t)(nC + 64) * nC,
                            (size_t)Npad * nC * 8, cudaMemcpyDeviceToDevice, s));
    RG_CUDA(cudaStreamSynchronize(s));
    h->launches += 3;
  }
  h->l1_bt = true;
  h->l1_done = true;
}

static void loco(rg_ctx* h, const int32_t* chr_of_block, double* pred_out) {
  RG_CHECK(h->kind == 1 && h->l1_done, "rg_l1_fit must run before rg_loco");
  RG_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  const int K = h->K, R1 = h->R1, P = h->P, R = h->R;
  const int nC = h->l1_nC, nmat = K * R1;
  const int64_t Npad = h->Npad, N = h->N;
  // chromosomes in block order (blocks never straddle chromosomes, src/Data.cpp:311-334)
  std::vector<int32_t> chrs, col_start;
  for (int b = 0; b < h->total_blocks; ++b) {
    const int c = chr_of_block[b];
    RG_CHECK(c >= 1 && c <= 23, "chromosome out of range");
    if (chrs.empty() || chrs.back() != c) {
      RG_CHECK(chrs.empty() || c > chrs.back(), "blocks must be ordered by chromosome");
      chrs.push_back(c);
      col_start.push_back(b * R);
    }
  }
  col_start.push_back(h->total_blocks * R);
  const int nchr = (int)chrs.size();
  h->l1_chr_cols.alloc(col_start.size());
  RG_CUDA(cudaMemcpyAsync(h->l1_chr_cols.p, col_start.data(), col_start.size() * 4, cudaMemcpyHostToDevice, s));
  h->l1_pred.alloc((size_t)nchr * Npad);
  std::vector<double> pred((size_t)nchr * Npad);
  h->prs_host.assign((size_t)P * N, 0.0);
  for (int p = 0; p < P; ++p) {
    if (!h->l1_select[p]) continue;
    if (h->l1_bt && h->loocv)
      launch_l1_bt_chr_pred(h->W_host_tab[p], Npad, nC, h->l1_zrows.p + (size_t)p * Npad * nC,
                            h->l1_hvec.p + (size_t)p * Npad, h->l1_bvec.p + (size_t)p * nC, nchr, h->l1_chr_cols.p,
                            h->l1_pred.p, Npad, s);
    else if (h->loocv)
      launch_l1_loocv_chr_pred(h->W_host_tab[p], Npad, (int)h->B, nC, h->l1_zrows.p + (size_t)p * Npad * nC,
                               h->l1_hvec.p + (size_t)p * Npad, h->l1_bvec.p + (size_t)p * nC, h->xy.p, h->cpp,
                               h->C + p, nchr, h->l1_chr_cols.p, h->l1_pred.p, Npad, s);
    else
      launch_l1_chr_pred(h->W_host_tab[p], Npad, nchr, h->l1_chr_cols.p,
                         h->l1_beta.p + (size_t)p * nmat * nC, nC, R1, h->best_idx[p], h->tile_fold.p, h->l1_pred.p, Npad, s);
    h->launches += 1;
    RG_CUDA(cudaMemcpyAsync(pred.data(), h->l1_pred.p, pred.size() * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaStreamSynchronize(s));
    // LOCO assembly (src/Data.cpp:1846-1858): all-chromosome sum minus the chromosome's own part
    double* out = pred_out + (size_t)p * 23 * N;
    for (int64_t i = 0; i < N; ++i) {
      const int64_t t = h->pad_of[i];
      double tot = 0.0;
      for (int ci = 0; ci < nchr; ++ci) tot += pred[(size_t)ci * Npad + t];
      h->prs_host[(size_t)p * N + i] = tot;
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
  RG_CHECK(h->kind == 1 && h->prs_host.size() == (size_t)h->P * h->N, "rg_loco must run before rg_prs");
  memcpy(prs_out, h->prs_host.data(), h->prs_host.size() * sizeof(double));
  RG_API_END
}

int rg_W_info(rg_handle h, int32_t ph, void** dev_ptr, int64_t* ld, int64_t* ncols) {
  RG_API_BEGIN
  RG_CHECK(h && h->kind == 1 && ph >= 0 && ph < h->P, "bad argument");
  RG_CUDA(cudaSetDevice(h->device));
  ensure_W(h);
  if (dev_ptr) *dev_ptr = h->W_host_tab[ph];
  if (ld) *ld = h->Npad;
  if (ncols) *ncols = h->B;
  RG_API_END
}

}  // extern "C"
