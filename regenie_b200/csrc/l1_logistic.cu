// Level-1 penalised logistic regression with closed-form leave-one-out predictions (binary traits, Step 1).
// Replaces ridge_logistic_level_1_loocv + run_log_ridge_loocv (reference src/Step1_Models.cpp:1159-1375) and the
// arithmetic of make_predictions_binary_loocv (src/Data.cpp:1484-1573).  The heavy pieces reuse the level-1 ridge
// machinery: the weighted Gram  W^T diag(w m) W  is the DMMA Gram of the row-scaled copy  sqrt(w m) o W, the Newton
// systems and the leverages  w_i^T H^-1 w_i  go through the batched Cholesky with the sample rows riding along as
// right-hand sides.  The scalar Newton control flow (step halving, two convergence tests, warm starts over tau) is
// driven from the host exactly as the reference writes it.
#include "kernels.cuh"

namespace rg {

// Ws[t, c] = W[t, c] * sqrt(wm[t]).  grid: (Npad/256, B)
__global__ void l1_scale_rows_kernel(const double* __restrict__ W, int64_t ldw, const double* __restrict__ wm,
                                     double* __restrict__ Ws) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t c = blockIdx.y;
  if (t < ldw) Ws[c * ldw + t] = W[c * ldw + t] * sqrt(wm[t]);
}

// eta = offset + W beta, w m, (y - p) m and the deviance partial of each 128-sample tile.
// grid: Npad/128, block 128 (thread = sample), dynamic smem: B doubles.
__global__ void __launch_bounds__(128)
l1_bt_eta_kernel(const double* __restrict__ W, int64_t ldw, int B, const double* __restrict__ beta,
                 const double* __restrict__ offset, const int8_t* __restrict__ ym, double* __restrict__ eta,
                 double* __restrict__ wm, double* __restrict__ resid, double* __restrict__ dev_part) {
  extern __shared__ double sb[];
  __shared__ double red[128];
  for (int c = threadIdx.x; c < B; c += 128) sb[c] = beta[c];
  __syncthreads();
  const int64_t t = blockIdx.x * 128 + threadIdx.x;
  double e = offset[t];
  for (int c = 0; c < B; ++c) e = fma(W[(int64_t)c * ldw + t], sb[c], e);
  const int8_t code = ym[t];
  const double p = get_pvec(e);
  eta[t] = e;
  wm[t] = code ? p * (1.0 - p) : 0.0;
  resid[t] = code ? ((code == 2 ? 1.0 : 0.0) - p) : 0.0;
  const double dev = cta_tree<128>(code ? -2.0 * ((code == 1) ? log(1.0 - p) : log(p)) : 0.0, red);
  if (threadIdx.x == 0) dev_part[blockIdx.x] = dev;
}

// score = W^T resid - tau beta from the chunk partials of l1_xty; also written into the RHS row of the system.
__global__ void l1_bt_score_kernel(const double* __restrict__ part_y, int nchunks, int B, int nC, double tau,
                                   const double* __restrict__ beta, double* __restrict__ score,
                                   double* __restrict__ rhs_row) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nC) return;
  double s = 0.0;
  if (c < B) {
    for (int k = 0; k < nchunks; ++k) s += part_y[(int64_t)k * B + c];
    s -= tau * beta[c];
  }
  score[c] = s;
  if (rhs_row) rhs_row[c] = s;
}

// LOO prediction sums of ridge_logistic_level_1_loocv (src/Step1_Models.cpp:1250-1275):
//   pred_i = eta_i - q_i (y_i - p_i) / (1 - q_i w_i),  p1 = clip(logistic(pred)),  Sx Sy Sx2 Sy2 Sxy -LL over mask.
// also stores f_i = (y_i - p_i) / (1 - q_i w_i) for the per-chromosome predictions.  grid: Npad/128.
__global__ void __launch_bounds__(128)
l1_bt_loo_sums_kernel(const double* __restrict__ eta, const double* __restrict__ q, const double* __restrict__ wm,
                      const double* __restrict__ resid, const int8_t* __restrict__ ym, double eps,
                      double* __restrict__ fvec, double* __restrict__ part) {
  __shared__ double red[6 * 128];
  const int64_t t = blockIdx.x * 128 + threadIdx.x;
  const int8_t code = ym[t];
  double v[6] = {0, 0, 0, 0, 0, 0};
  double f = 0.0;
  if (code) {
    f = resid[t] / (1.0 - q[t] * wm[t]);
    const double pred = eta[t] - q[t] * f;
    double p1 = 1.0 - 1.0 / (exp(pred) + 1.0);
    p1 = fmin(fmax(p1, eps), 1.0 - eps);
    const double y = (code == 2) ? 1.0 : 0.0;
    v[0] = p1; v[1] = y; v[2] = p1 * p1; v[3] = y * y; v[4] = p1 * y;
    v[5] = -((code == 1) ? log(1.0 - p1) : log(p1));
  }
  if (fvec) fvec[t] = f;
  cta_tree<128>(v, red);
  if (threadIdx.x == 0)
    for (int k = 0; k < 6; ++k) part[(int64_t)blockIdx.x * 6 + k] = v[k];
}

// per-chromosome LOO predictions: pred[t, chr] = W_chr[t] . beta_chr - (W_chr[t] . z_chr[t]) f_t   (src/Data.cpp:1560-1566)
// grid: Npad/128, block 128 (thread = sample); zrows row-major [t][nC].
__global__ void __launch_bounds__(128)
l1_bt_chr_pred_kernel(const double* __restrict__ W, int64_t ldw, int nC, const double* __restrict__ zrows,
                      const double* __restrict__ fvec, const double* __restrict__ bvec, int nchr,
                      const int32_t* __restrict__ chr_col_start, double* __restrict__ pred, int64_t npad) {
  const int64_t t = blockIdx.x * 128 + threadIdx.x;
  const double f = fvec[t];
  for (int ci = 0; ci < nchr; ++ci) {
    double a = 0.0, b = 0.0;
    for (int c = chr_col_start[ci]; c < chr_col_start[ci + 1]; ++c) {
      const double w = W[(int64_t)c * ldw + t];
      a = fma(w, bvec[c], a);
      b = fma(w, zrows[t * nC + c], b);
    }
    pred[(int64_t)ci * npad + t] = a - b * f;
  }
}

void launch_l1_scale_rows(const double* W, int64_t ldw, int B, const double* wm, double* Ws, cudaStream_t s) {
  dim3 grid((unsigned)ceil_div(ldw, 256), B);
  l1_scale_rows_kernel<<<grid, 256, 0, s>>>(W, ldw, wm, Ws);
}
void launch_l1_bt_eta(const double* W, int64_t ldw, int B, const double* beta, const double* offset, const int8_t* ym,
                      double* eta, double* wm, double* resid, double* dev_part, double* dev_out, cudaStream_t s) {
  const int ntiles = (int)(ldw / 128);
  l1_bt_eta_kernel<<<ntiles, 128, B * sizeof(double), s>>>(W, ldw, B, beta, offset, ym, eta, wm, resid, dev_part);
  launch_partial_sum(dev_part, ntiles, 1, dev_out, s);
}
void launch_l1_bt_score(const double* part_y, int nchunks, int B, int nC, double tau, const double* beta, double* score,
                        double* rhs_row, cudaStream_t s) {
  l1_bt_score_kernel<<<(unsigned)ceil_div(nC, 128), 128, 0, s>>>(part_y, nchunks, B, nC, tau, beta, score, rhs_row);
}
void launch_l1_bt_loo_sums(const double* eta, const double* q, const double* wm, const double* resid, const int8_t* ym,
                           double eps, double* fvec, double* part, double* out6, int64_t npad, cudaStream_t s) {
  const int ntiles = (int)(npad / 128);
  l1_bt_loo_sums_kernel<<<ntiles, 128, 0, s>>>(eta, q, wm, resid, ym, eps, fvec, part);
  launch_partial_sum(part, ntiles, 6, out6, s);
}
void launch_l1_bt_chr_pred(const double* W, int64_t ldw, int nC, const double* zrows, const double* fvec,
                           const double* bvec, int nchr, const int32_t* chr_col_start, double* pred, int64_t npad,
                           cudaStream_t s) {
  l1_bt_chr_pred_kernel<<<(unsigned)(npad / 128), 128, 0, s>>>(W, ldw, nC, zrows, fvec, bvec, nchr, chr_col_start, pred, npad);
}

}  // namespace rg
