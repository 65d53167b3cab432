// C ABI of librg_b200.so (see include/rg_b200.h): handle lifetime, Step-1 level-0 block path.
#include <string.h>

#include <algorithm>
#include <mutex>

#include "context.cuh"

namespace rg {

static thread_local std::string g_last_error;
void set_last_error(const std::string& m) { g_last_error = m; }

bool is_device_pointer(const void* p) {
  cudaPointerAttributes at;
  cudaError_t e = cudaPointerGetAttributes(&at, p);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

void copy_to_device(void* dst, const void* src, size_t bytes, cudaStream_t stream) {
  if (bytes == 0) return;
  RG_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, stream));
}

struct ScopedTimer {
  rg_ctx* h;
  std::string name;
  Event a, b;
  cudaStream_t st;
  ScopedTimer(rg_ctx* h_, const char* n, cudaStream_t s_) : h(h_), name(n), st(s_) {
    if (!h->timing) return;
    cudaEventRecord(a.ensure(cudaEventDefault), st);
    b.ensure(cudaEventDefault);
  }
  ~ScopedTimer() {
    if (!h->timing) return;
    cudaEventRecord(b, st);
    h->pending.emplace_back(name, std::move(a), std::move(b));
  }
};

void flush_timers(rg_ctx* h) {
  for (auto& t : h->pending) {
    float ms = 0.f;
    cudaEventSynchronize(std::get<2>(t));
    cudaEventElapsedTime(&ms, std::get<1>(t), std::get<2>(t));
    auto& acc = h->timers[std::get<0>(t)];
    acc.first += ms;
    acc.second += 1;
  }
  h->pending.clear();
}

void require_gpu(int device) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    cudaGetLastError();
    throw Error{"no CUDA device available: librg_b200 has no CPU fallback"};
  }
  RG_CHECK(device >= 0 && device < n, "invalid CUDA device ordinal");
  cudaDeviceProp prop;
  RG_CUDA(cudaGetDeviceProperties(&prop, device));
  RG_CHECK(prop.major == 9 && prop.minor == 0, std::string("librg_b200 is built for sm_90a only; device is sm_") +
                                 std::to_string(prop.major) + std::to_string(prop.minor));
}

void fold_chunk_table(const Step1State& s1, int64_t len, std::vector<int4>& chunks, std::vector<int2>& fold_chunks) {
  const int K = s1.K;
  chunks.clear();
  fold_chunks.assign(K, make_int2(0, 0));
  for (int f = 0; f < K; ++f) {
    fold_chunks[f].x = (int)chunks.size();
    for (int64_t o = 0; o < s1.fold_pad_len[f]; o += len)
      chunks.push_back(make_int4((int)(s1.fold_pad_start[f] + o), (int)std::min<int64_t>(len, s1.fold_pad_len[f] - o), f, 0));
    fold_chunks[f].y = (int)chunks.size();
  }
}

// Build the padded fold layout + all device state shared by the blocks.
static void build_layout(rg_ctx* h, Step1State& s1, const double* X, const double* Y, const uint8_t* mask,
                         const uint8_t* in_analysis, const int64_t* fold_sizes) {
  const int64_t N = h->N;
  const int K = s1.K, C = h->C, P = h->P;
  s1.fold_sizes.assign(K, 0);
  if (s1.loocv) {
    s1.fold_sizes[0] = N;
  } else {
    int64_t tot = 0;
    for (int f = 0; f < K; ++f) {
      RG_CHECK(fold_sizes[f] > 0, "fold sizes must be positive");
      s1.fold_sizes[f] = fold_sizes[f];
      tot += fold_sizes[f];
    }
    RG_CHECK(tot == N, "fold sizes must sum to n_samples");
  }
  s1.fold_pad_start.assign(K, 0);
  s1.fold_pad_len.assign(K, 0);
  int64_t off = 0;
  for (int f = 0; f < K; ++f) {
    s1.fold_pad_start[f] = off;
    s1.fold_pad_len[f] = round_up(s1.fold_sizes[f], kFoldPad);
    off += s1.fold_pad_len[f];
  }
  h->Npad = off;
  RG_CHECK(h->Npad < (1ll << 31), "padded sample count must fit in int32");
  s1.pad_of.assign(N, 0);
  h->src_of.assign(h->Npad, -1);
  std::vector<int32_t> tile_fold(h->Npad / 128);
  {
    int64_t s = 0;
    for (int f = 0; f < K; ++f) {
      for (int64_t o = 0; o < s1.fold_sizes[f]; ++o, ++s) {
        s1.pad_of[s] = (int32_t)(s1.fold_pad_start[f] + o);
        h->src_of[s1.fold_pad_start[f] + o] = (int32_t)s;
      }
      for (int64_t t = s1.fold_pad_start[f]; t < s1.fold_pad_start[f] + s1.fold_pad_len[f]; t += 128)
        tile_fold[t / 128] = f;
    }
  }
  h->in_analysis.assign(in_analysis, in_analysis + N);

  // (X | Y) sample-major, zero padded to cpp columns
  s1.cpp = (int)round_up(C + P, 16);
  std::vector<double> xy((size_t)h->Npad * s1.cpp, 0.0);
  std::vector<uint8_t> maskp((size_t)P * h->Npad, 0), is_real(h->Npad, 0);
  h->maskh.assign(mask, mask + (size_t)N * P);
  for (int64_t s = 0; s < N; ++s) {
    const int64_t t = s1.pad_of[s];
    is_real[t] = 1;
    double* r = &xy[(size_t)t * s1.cpp];
    for (int c = 0; c < C; ++c) r[c] = X[(size_t)c * N + s];
    for (int p = 0; p < P; ++p) {
      r[C + p] = Y[(size_t)p * N + s];
      maskp[(size_t)p * h->Npad + t] = mask[(size_t)p * N + s] ? 1 : 0;
    }
  }
  // per-fold X_f^T X_f and X_f^T Y_f (Appendix B item 6 of SURVEY.md), summed with Neumaier compensation: the level-0
  // Gram subtracts B (X_f^T X_f) B^T from G_f G_f^T, and for a variant whose mean is large against its spread (the
  // counted allele nearly fixed) the two agree to 1 part in 10^3 or more, so the ~n u error of a plain running sum over
  // a fold of 10^5 .. 10^6 samples would show in the predictors
  std::vector<double> XtX((size_t)K * C * C, 0.0), XtY((size_t)K * C * P, 0.0);
  {
    std::vector<double> cXtX(XtX.size(), 0.0), cXtY(XtY.size(), 0.0);
    auto add = [](double& sum, double& comp, double v) {
      const double t = sum + v;
      comp += (std::fabs(sum) >= std::fabs(v)) ? (sum - t) + v : (v - t) + sum;
      sum = t;
    };
    int64_t s = 0;
    for (int f = 0; f < K; ++f)
      for (int64_t o = 0; o < s1.fold_sizes[f]; ++o, ++s)
        for (int c = 0; c < C; ++c) {
          const double xc = X[(size_t)c * N + s];
          if (xc == 0.0) continue;
          for (int c2 = 0; c2 < C; ++c2) {
            const size_t e = ((size_t)f * C + c) * C + c2;
            add(XtX[e], cXtX[e], xc * X[(size_t)c2 * N + s]);
          }
          for (int p = 0; p < P; ++p) {
            const size_t e = ((size_t)f * C + c) * P + p;
            add(XtY[e], cXtY[e], xc * Y[(size_t)p * N + s]);
          }
        }
    for (size_t e = 0; e < XtX.size(); ++e) XtX[e] += cXtX[e];
    for (size_t e = 0; e < XtY.size(); ++e) XtY[e] += cXtY[e];
  }
  // chunk table for the f64 reductions
  std::vector<int4> chunks;
  std::vector<int2> fold_chunks, fold_k(K);
  fold_chunk_table(s1, kStatChunk, chunks, fold_chunks);
  for (int f = 0; f < K; ++f)
    fold_k[f] = make_int2((int)(s1.fold_pad_start[f] / 128), (int)(s1.fold_pad_len[f] / 128));
  s1.nchunks = (int)chunks.size();

  cudaStream_t s = h->stream;
  upload(s1.xy, xy, s);
  upload(s1.mask, maskp, s);
  upload(s1.is_real, is_real, s);
  upload(s1.tile_fold, tile_fold, s);
  upload(s1.chunks, chunks, s);
  upload(s1.fold_chunks, fold_chunks, s);
  upload(s1.fold_k, fold_k, s);
  upload(s1.XtX_f, XtX, s);
  upload(s1.XtY_f, XtY, s);
  // statistics as extra Gram tiles: digit rows of (X | Y), once per run.  Exact while 30 * fold length < 2^24.
  {
    int64_t max_fold = 0;
    for (int f = 0; f < K; ++f) max_fold = std::max(max_fold, s1.fold_pad_len[f]);
    const char* e = getenv("RG_B200_STATS");
    s1.stats_tc = !(e && std::string(e) == "f64") && max_fold * 30 < (1ll << 24);
    if (s1.stats_tc) {
      const int ngroups = (int)ceil_div(C + P, kStatQ);
      s1.stat_drows = ngroups * 128;          // an odd group count runs as 128 x 128 tiles (stat_bn)
      s1.xyD.alloc((size_t)s1.stat_drows * h->Npad);
      s1.xy_scale.alloc(s1.cpp);
      RG_CUDA(cudaMemsetAsync(s1.xyD.p, 0, (size_t)s1.stat_drows * h->Npad, s));
      launch_l0_xy_digits(s1.xy.p, s1.cpp, C + P, h->Npad, s1.is_real.p, s1.xy_scale.p, s1.xyD.p, s);
      make_gram_tensor_map(&s1.tmD, s1.xyD.p, h->Npad, s1.stat_drows);
    }
  }
  // Miss rows of the Gram as sparse sums while a block has at most kMissSparseRate missing calls (miss_gram.cu)
  {
    // RG_B200_GRAM=dense: always the dense tiles; =sparse: a list for every call (tools/miss_rate_sweep.py)
    const char* e = getenv("RG_B200_GRAM");
    const std::string mode = e ? e : "";
    s1.gram_dense = mode == "dense";
    const double rate = mode == "sparse" ? 1.0 : kMissSparseRate;
    s1.miss_cap = std::min<int64_t>((int64_t)(rate * h->bs_max * h->n_analyzed), INT32_MAX);
    // the relayout's column tiles: 512 samples (32 words) each, cut at the fold ends so that a tile's calls belong to
    // one fold
    std::vector<int2> fold_ct(K);
    s1.miss_ctile_host.clear();
    for (int f = 0; f < K; ++f) {
      fold_ct[f].x = (int)s1.miss_ctile_host.size();
      const int64_t w1 = (s1.fold_pad_start[f] + s1.fold_pad_len[f]) / 16;
      for (int64_t w = s1.fold_pad_start[f] / 16; w < w1; w += 32)
        s1.miss_ctile_host.push_back(make_int4((int)w, (int)std::min<int64_t>(32, w1 - w), f, 0));
      fold_ct[f].y = (int)s1.miss_ctile_host.size();
    }
    s1.miss_nct = (int)s1.miss_ctile_host.size();
    upload(s1.miss_ctile, s1.miss_ctile_host, s);
    upload(s1.miss_fold_ct, fold_ct, s);
  }
  RG_CUDA(cudaStreamSynchronize(s));   // host vectors go out of scope
}

// file_idx_pad[t] = index of the sample in the .bed row, or -1 for layout padding and for
// samples outside the analysis (whose genotypes the reference zeroes, src/Data.cpp:196).
static void build_file_idx(rg_ctx* h, const int32_t* sample_idx_host) {
  std::vector<int32_t> fi(h->Npad, -1);
  for (int64_t t = 0; t < h->Npad; ++t) {
    const int32_t s = h->src_of[t];
    if (s < 0 || !h->in_analysis[s]) continue;
    fi[t] = sample_idx_host ? sample_idx_host[s] : s;
  }
  const int64_t nw = h->Npad / 16;
  std::vector<int32_t> wb(nw, -1);
  std::vector<uint32_t> wk(nw, 0);
  for (int64_t w = 0; w < nw; ++w) {
    int32_t base = -1;
    bool contiguous = true;
    for (int j = 0; j < 16; ++j) {
      const int32_t f = fi[w * 16 + j];
      if (f < 0) continue;
      wk[w] |= 3u << (2 * j);
      if (base == -1) base = f - j;
      else if (f - j != base) contiguous = false;
    }
    wb[w] = (wk[w] == 0) ? -1 : ((contiguous && base >= 0) ? base : -2);
  }
  upload(h->word_base, wb, h->stream);
  upload(h->word_keep, wk, h->stream);
  upload(h->file_idx_pad, fi, h->stream);
  RG_CUDA(cudaStreamSynchronize(h->stream));
  h->file_idx_valid = true;
}

// sample index map of the genotype file (cached): rebuilt only when the caller's sample_idx changes
void ensure_file_idx(rg_ctx* h, const int32_t* sample_idx) {
  if (!sample_idx) {
    if (!h->file_idx_valid || !h->cached_sample_idx.empty()) {
      build_file_idx(h, nullptr);
      h->cached_sample_idx.clear();
    }
    return;
  }
  std::vector<int32_t> host_idx(h->N);
  if (is_device_pointer(sample_idx)) RG_CUDA(cudaMemcpy(host_idx.data(), sample_idx, h->N * 4, cudaMemcpyDefault));
  else host_idx.assign(sample_idx, sample_idx + h->N);
  if (!h->file_idx_valid || h->cached_sample_idx != host_idx) {
    build_file_idx(h, host_idx.data());
    h->cached_sample_idx = std::move(host_idx);
  }
}

// Storage of the level-0 predictors, allocated on first use: one compact slab per phenotype this rank owns
// (all of them unless rg_W_set_owned said otherwise); entries of phenotypes owned elsewhere stay null until
// rg_W_attach_peer maps the owner's memory.
void ensure_W(rg_ctx* h, Step1State& s1) {
  if (s1.W.p) return;
  size_t n_owned = 0;
  for (int p = 0; p < h->P; ++p) n_owned += s1.W_owned[p] ? 1 : 0;
  const size_t per = (size_t)h->Npad * s1.B;
  s1.W.alloc(std::max<size_t>(1, n_owned) * per);
  RG_CUDA(cudaMemset(s1.W.p, 0, std::max<size_t>(1, n_owned) * per * 8));
  size_t slot = 0;
  for (int p = 0; p < h->P; ++p)
    if (s1.W_owned[p]) s1.W_host_tab[p] = s1.W.p + (slot++) * per;
  RG_CUDA(cudaMemcpy(s1.W_tab.p, s1.W_host_tab.data(), h->P * sizeof(double*), cudaMemcpyHostToDevice));
}

// Points the phenotypes owned_by_peer at the owner's W, which is compact over the phenotypes the owner holds
// (rg_W_set_owned with the same mask there), and leaves their level-1 fits to the owner.
static void attach_W(rg_ctx* h, Step1State& s1, double* owner_W, const uint8_t* owned_by_peer) {
  size_t slot = 0;
  for (int p = 0; p < h->P; ++p)
    if (owned_by_peer[p]) {
      s1.W_host_tab[p] = owner_W + (slot++) * (size_t)h->Npad * s1.B;
      s1.l1_select[p] = 0;
    }
  RG_CUDA(cudaMemcpy(s1.W_tab.p, s1.W_host_tab.data(), h->P * sizeof(double*), cudaMemcpyHostToDevice));
}

struct BlockDims {
  int bs, rows_p, nC, Ppad, n_aug, nmat, Q, Qp, col0, block_id, ntiles_s;
};

static int mx_pp(int P) { return (int)round_up(P, 2); }
constexpr int kMxSteps = 3;               // refinement steps of the mixed solver

// Assembler arguments the FP64 and the mixed path share; each path adds the layout of its systems (nC, cm, cm_stride, ldc).
static AssembleArgs assemble_args(const rg_ctx* h, const Step1State& s1, const Step1State::Lane& L, const BlockDims& d) {
  AssembleArgs aa;
  aa.bs = d.bs; aa.rows_p = d.rows_p; aa.C = h->C; aa.K = s1.K; aa.R = s1.R; aa.loocv = s1.loocv;
  aa.zz = L.zz.p; aa.ldz = 2 * d.rows_p; aa.zz_fold_stride = (int64_t)4 * d.rows_p * d.rows_p;
  aa.mu = L.mu.p; aa.inv_sd = L.inv_sd.p; aa.Bv = L.Bv.p; aa.Af = L.Af.p; aa.Qf = L.Qf.p;
  aa.lambda = s1.lambda.p;
  return aa;
}

// The lane's FP64 systems [nmat][n_aug][nC] (LOOCV: the sample vectors ride along as right-hand-side rows) and the
// inverses of their diagonal blocks, sized for the largest block of the run; the systems are zeroed when allocated.
static void ensure_f64_systems(rg_ctx* h, Step1State& s1, Step1State::Lane& L, const BlockDims& d, cudaStream_t s) {
  const int nC_max = (int)round_up(h->bs_max, 64);
  const size_t need = (size_t)d.nmat * (nC_max + d.Ppad + (s1.loocv ? h->Npad : 0)) * nC_max;
  if (L.cm.n < need) {
    L.cm.alloc(need);
    RG_CUDA(cudaMemsetAsync(L.cm.p, 0, need * 8, s));
  }
  L.inv.alloc(chol_inv_elems(nC_max, d.nmat));
}

// LOOCV: closed-form leave-one-out predictions from the factorised systems (src/Step1_Models.cpp:654-663), standardised
// into W (:694-706)
static void enqueue_loocv_predict(rg_ctx* h, Step1State& s1, Step1State::Lane& L, const BlockDims& d, cudaStream_t s) {
  const int P = h->P;
  launch_l0_loocv_pred(L.cm.p, (int64_t)d.n_aug * d.nC, d.nC, d.bs, d.Ppad, P, s1.R, s1.xy.p, s1.cpp, h->C, s1.mask.p, h->Npad,
                       s1.W_tab.p, d.col0, L.part.p, d.Qp, s);
  launch_l0_std_reduce_only(L.part.p, d.ntiles_s, d.Qp, d.Q, P, s1.neff.p, L.mean_invsd.p, s);
  launch_l0_loocv_std_apply(s1.W_tab.p, h->Npad, d.col0, P, d.Q, s1.mask.p, L.mean_invsd.p, s);
  h->launches += 3;
}

// What both level-0 routes run once their FP64 systems are in L.cm: the batched Cholesky (DMMA), then either the LOOCV
// predictions (they read the factorisation directly) or the backward substitution, which leaves the solutions in the
// right-hand-side rows of L.cm.
static void enqueue_factor_solve_f64(rg_ctx* h, Step1State& s1, Step1State::Lane& L, const BlockDims& d, cudaStream_t s) {
  const int64_t cm_stride = (int64_t)d.n_aug * d.nC;
  L.part.alloc((size_t)d.ntiles_s * d.Qp * 2);
  L.mean_invsd.alloc((size_t)2 * d.Qp);
  {
    ScopedTimer t(h, "chol_factor", s);
    launch_chol_factor(L.cm.p, cm_stride, d.nC, d.n_aug, d.nmat, L.inv.p, s1.err_slot.p,
                       (long long)(1ll << 40) + (long long)d.block_id * 1024, s);
    h->launches += chol_num_launches(d.nC);
  }
  if (s1.loocv) {
    ScopedTimer t(h, "l0_predict", s);
    enqueue_loocv_predict(h, s1, L, d, s);
    return;
  }
  ScopedTimer t(h, "chol_backsolve", s);
  launch_chol_backsolve(L.cm.p, cm_stride, d.nC, h->P, d.nmat, L.inv.p, s);
  h->launches += 1;
}

// FP64 path of the 2-bit route: assemble the K*R shifted systems (LOOCV: with the sample rows), then factor and solve.
static void enqueue_solve_f64(rg_ctx* h, Step1State& s1, Step1State::Lane& L, const BlockDims& d, cudaStream_t s) {
  ensure_f64_systems(h, s1, L, d, s);
  AssembleArgs aa = assemble_args(h, s1, L, d);
  aa.nC = d.nC; aa.cm = L.cm.p; aa.cm_stride = (int64_t)d.n_aug * d.nC; aa.ldc = d.nC;
  {
    ScopedTimer t(h, "l0_assemble", s);
    launch_l0_assemble(aa, L.rhs.p, h->P, d.Ppad, d.nmat, s);
    h->launches += 2;
  }
  if (s1.loocv) {
    ScopedTimer t(h, "loocv_fill", s);
    launch_l0_loocv_fill(L.gp.p, h->Npad, d.bs, d.nC, L.mu.p, L.inv_sd.p, L.Bv.p, h->C, s1.xy.p, s1.cpp, L.cm.p,
                         aa.cm_stride, d.nC + d.Ppad, s1.R, s);
    h->launches += 1;
  }
  enqueue_factor_solve_f64(h, s1, L, d, s);
}

// Mixed path: K symmetric FP64 fold systems -> tensor-core factorisation / inverse -> FP64 refinement.  Solutions in L.mx_x.
static void enqueue_solve_mixed(rg_ctx* h, Step1State& s1, Step1State::Lane& L, const BlockDims& d, int n, cudaStream_t s) {
  const int P = h->P, K = s1.K, R = s1.R;
  const int Pp = mx_pp(P);
  if (!L.mx) {
    L.mx = std::make_unique<MixedSolver>();
    L.mx_fail.alloc(1);
    L.mx_fail_host.alloc(1);
    L.mx_ev.ensure();
  }
  // sized from the block being solved: with bsize > 2048 the largest blocks take the FP64 path, but a chromosome's short
  // last block still comes here (alloc is a no-op once the buffers are large enough)
  const size_t need_A = (size_t)K * n * n, need_b = (size_t)K * Pp * n, need_x = (size_t)K * R * Pp * n;
  L.mx_Af.alloc(need_A);
  L.mx_b.alloc(need_b);
  L.mx_x.alloc(need_x);
  L.mx_r.alloc(need_x);
  RG_CHECK(L.mx_Af.n >= need_A && L.mx_b.n >= need_b && L.mx_x.n >= need_x && L.mx_r.n >= need_x,
           "mixed solver: scratch smaller than the block's systems");
  L.mx->prepare(n, K, R, Pp);
  RG_CUDA(cudaMemsetAsync(L.mx_fail.p, 0, sizeof(unsigned int), s));
  AssembleArgs aa = assemble_args(h, s1, L, d);
  aa.nC = n; aa.cm = L.mx_Af.p; aa.cm_stride = (int64_t)n * n; aa.ldc = n;
  aa.planes = L.mx->a_planes();
  aa.lplanes = L.mx->l_planes();           // block column 0 of the factor: the solver skips its first update
  {
    ScopedTimer t(h, "l0_assemble", s);
    launch_l0_assemble_sym(aa, L.rhs.p, P, Pp, L.mx_b.p, s);
    h->launches += 2;
  }
  {
    ScopedTimer t(h, "mx_solve", s);
    L.mx->solve(L.mx_Af.p, s1.lambda.p, L.mx_b.p, L.mx_x.p, L.mx_r.p, P, kMxSteps, s1.mx_tol, L.mx_fail.p, s, true);
    h->launches += MixedSolver::launches_per_solve(n, kMxSteps, P) - 1;
  }
}

// Tensor map of the lane's 2-bit rows.
static const CUtensorMap& gp_map(const rg_ctx* h, Step1State::Lane& L, int rows_p) {
  return gp_tensor_map(L.gmaps, L.gp.p, h->Npad, rows_p);
}

// Out-of-fold predictions from the coefficients x[m][p][i] at xsrc + m * xstride + (xrow0 + p) * xld + i.
static void enqueue_predict(rg_ctx* h, Step1State& s1, Step1State::Lane& L, const BlockDims& d, const double* xsrc,
                            int64_t xstride, int xld, int xrow0, cudaStream_t s) {
  const int C = h->C, P = h->P, K = s1.K, R = s1.R;
  const int64_t Npad = h->Npad;
  ScopedTimer t(h, "l0_predict", s);
  // raw predictions go to the lane's LOCAL scratch; the standardisation pass reads them there and writes the finished
  // columns into W - the owner's HBM, which may be another GPU's (then only plain stores cross NVLink)
  if (L.wraw.n < (size_t)P * R * Npad) {
    L.wraw.alloc((size_t)P * R * Npad);
    std::vector<double*> tab(P);
    for (int p = 0; p < P; ++p) tab[p] = L.wraw.p + (size_t)p * R * Npad;
    upload(L.wraw_tab, tab, s);
    RG_CUDA(cudaStreamSynchronize(s));           // tab goes out of scope (once per lane)
  }
  PredictArgs pa;
  pa.bs = d.bs; pa.rows_p = d.rows_p; pa.C = C; pa.P = P; pa.R = R; pa.Qp = d.Qp; pa.cpp = s1.cpp;
  pa.col0 = 0; pa.npad = Npad; pa.words_per_row = Npad / 16;
  pa.gp = L.gp.p; pa.tile_fold = s1.tile_fold.p; pa.gam = L.gam.p; pa.gmu = L.gmu.p;
  pa.cvec = L.cvec.p; pa.xy = s1.xy.p; pa.mask = s1.mask.p; pa.W = L.wraw_tab.p; pa.part = L.part.p;
  // INT8 tensor cores (s8 wgmma, 5 radix-254 limbs) up to 2 rows_p = 4096; the FP64 CUDA-core kernel beyond (bsize > 2048).
  // Both leave per-tile column sums in L.part.
  const bool use_i8 = 2 * d.rows_p <= 4096;
  L.last_pred_i8 = use_i8 ? 1 : 0;
  if (!use_i8) {
    launch_l0_gamma(xsrc, xstride, xld, xrow0, R, P, d.Qp, d.bs, d.rows_p, K, L.mu.p, L.inv_sd.p, L.Bv.p, C,
                    L.gam.p, L.gmu.p, L.cvec.p, s);
    launch_l0_predict(pa, d.ntiles_s, s);
    h->launches += 3;
  } else {
    // exact tensor-core path: digit rows of gamma against the genotype planes, decoded from the 2-bit rows
    const int ngroups = (int)ceil_div(d.Q, kLimbQI8);
    const int drows_per_group = 256;
    const size_t need = predict_i8_dig_bytes(K, ngroups, h->rows_p_max);
    if (L.dig.n < need) {
      L.dig.alloc(need);
      RG_CUDA(cudaMemsetAsync(L.dig.p, 0, need, s));
      L.dmaps.clear();
    }
    L.dscale.alloc((size_t)K * d.Qp);
    if (!L.dmaps.count(d.rows_p)) {
      CUtensorMap tm;
      make_byte_tensor_map(&tm, L.dig.p, 2 * d.rows_p, (int64_t)K * ngroups * drows_per_group);
      L.dmaps[d.rows_p] = tm;
    }
    launch_l0_coef_i8(xsrc, xstride, xld, xrow0, R, P, d.Q, d.Qp, d.bs, d.rows_p, K, L.mu.p, L.inv_sd.p, L.Bv.p, C,
                      L.gam.p, L.gmu.p, L.cvec.p, L.dscale.p, L.dig.p, ngroups, s);
    PredictTcArgs ta;
    ta.rows_p = d.rows_p; ta.C = C; ta.P = P; ta.Q = d.Q; ta.Qp = d.Qp; ta.cpp = s1.cpp; ta.col0 = 0; ta.ngroups = ngroups;
    ta.npad = Npad; ta.tile_fold = s1.tile_fold.p; ta.scale = L.dscale.p; ta.cvec = L.cvec.p;
    ta.xy = s1.xy.p; ta.mask = s1.mask.p; ta.W = L.wraw_tab.p; ta.part = L.part.p;
    launch_l0_predict_i8(gp_map(h, L, d.rows_p), L.dmaps[d.rows_p], ta, d.ntiles_s, s);
    h->launches += 2;
  }
  launch_l0_standardize(L.part.p, d.ntiles_s, d.Qp, d.Q, P, s1.neff.p, L.mean_invsd.p, s1.W_tab.p, Npad, d.col0,
                        s1.is_real.p, s, L.wraw_tab.p, 0);
  h->launches += 2;
}

static BlockDims block_dims(const rg_ctx* h, const Step1State& s1, int bs, int block_id) {
  BlockDims d;
  d.bs = bs; d.rows_p = (int)round_up(bs, kRowPad); d.nC = (int)round_up(bs, 64); d.Ppad = (int)round_up(h->P, 64);
  d.n_aug = d.nC + d.Ppad + (s1.loocv ? (int)h->Npad : 0);
  d.nmat = (s1.loocv ? 1 : s1.K) * s1.R;
  d.Q = s1.R * h->P; d.Qp = (int)round_up(d.Q, predict_qt());
  d.col0 = block_id * s1.R; d.block_id = block_id; d.ntiles_s = (int)(h->Npad / 128);
  return d;
}

// Read the mixed-solver flag of the block this lane ran last; if the refinement did not converge (ill-conditioned
// system) or a pivot was not positive, re-solve that block in FP64 from the lane's scratch (statistics, Grams and 2-bit
// rows of the block are still there) and redo its predictions.
void resolve_lane(rg_ctx* h, Step1State& s1, Step1State::Lane& L) {
  if (!L.mx_pending) return;
  RG_CUDA(cudaEventSynchronize(L.mx_ev));
  L.mx_pending = false;
  if (*L.mx_fail_host.p == 0) return;
  s1.mx_fallbacks += 1;
  L.last_mx_n = 0;
  const BlockDims d = block_dims(h, s1, L.mx_bs, L.mx_block_id);
  enqueue_solve_f64(h, s1, L, d, L.stream);
  enqueue_predict(h, s1, L, d, L.cm.p, (int64_t)d.n_aug * d.nC, d.nC, d.nC, L.stream);
}

void sync_lanes(rg_ctx* h) {
  RG_CUDA(cudaSetDevice(h->device));
  if (!h->s1) return;
  for (auto& l : h->s1->lanes) resolve_lane(h, *h->s1, *l);
  for (auto& l : h->s1->lanes) RG_CUDA(cudaStreamSynchronize(l->stream));
}

// What both level-0 block routes do first: check the call, map the samples of the genotype file, take the next lane and
// record the block's dimensions (rg_debug_fetch "dims").  Each route reads the flag of the lane's previous block itself
// (resolve_lane), because the .bed route enqueues its input copy before the host waits on that flag.
static Step1State::Lane& l0_begin_block(rg_ctx* h, Step1State& s1, int bs, int block_id, const int32_t* sample_idx, BlockDims& d) {
  RG_CHECK(bs > 0 && bs <= h->bs_max, "block size out of range");
  RG_CHECK(block_id >= 0 && block_id < s1.total_blocks, "block_id out of range");
  ensure_W(h, s1);
  for (int p = 0; p < h->P; ++p)
    RG_CHECK(s1.W_host_tab[p] != nullptr, "a phenotype has neither local storage nor an attached owner (rg_W_set_owned / rg_W_attach_peer)");
  RG_CUDA(cudaSetDevice(h->device));
  ensure_file_idx(h, sample_idx);
  Step1State::Lane& L = *s1.lanes[s1.next_lane];
  s1.last_lane = s1.next_lane;
  s1.next_lane = (s1.next_lane + 1) % (int)s1.lanes.size();
  d = block_dims(h, s1, bs, block_id);
  s1.last_bs = bs; s1.last_rows_p = d.rows_p; s1.last_nC = d.nC; s1.last_n_aug = d.n_aug; s1.last_nmat = d.nmat;
  return L;
}

static void l0_block_bed(rg_ctx* h, const uint8_t* packed, int64_t row_stride, int bs,
                         const int32_t* sample_idx, int ref_first, int block_id) {
  Step1State& s1 = step1(h);
  BlockDims d;
  Step1State::Lane& L = l0_begin_block(h, s1, bs, block_id, sample_idx, d);
  const int C = h->C, P = h->P, K = s1.K;
  const int rows_p = d.rows_p, Qp = d.Qp;
  const int64_t Npad = h->Npad;
  cudaStream_t s = L.stream;

  // --- input rows to the device: enqueued BEFORE the host waits for the solver flag of the lane's previous block
  // (resolve_lane below), so the PCIe transfer runs while that block is still in its kernels
  const uint8_t* packed_d = packed;
  int staged = -1;                         // index of the staging buffer the rows went to (host input)
  if (!is_device_pointer(packed)) {
    staged = (L.packed_flip ^= 1);
    rg::DevBuf<uint8_t>& buf = L.packed_buf[staged];
    buf.alloc((size_t)h->bs_max * row_stride);
    cudaStream_t cs = L.copy_stream.ensure();
    // the buffer was last read by the relayout kernel of the block this lane ran two blocks ago
    if (L.relayout_done[staged]) RG_CUDA(cudaStreamWaitEvent(cs, L.relayout_done[staged], 0));
    {
      ScopedTimer t(h, "h2d", cs);
      copy_to_device(buf.p, packed, (size_t)bs * row_stride, cs);
    }
    RG_CUDA(cudaEventRecord(L.h2d_done.ensure(), cs));
    RG_CUDA(cudaStreamWaitEvent(s, L.h2d_done, 0));
    packed_d = buf.p;
  }
  resolve_lane(h, s1, L);                      // flag of the block this lane ran before (FP64 re-solve if it was raised)

  // --- scratch
  L.gp.alloc((size_t)h->rows_p_max * (Npad / 16));
  L.zz.alloc((size_t)K * 4 * h->rows_p_max * h->rows_p_max);
  L.cnt_part.alloc((size_t)s1.nchunks * h->rows_p_max * 4);
  L.sum_part.alloc((size_t)s1.nchunks * h->rows_p_max * 2 * s1.cpp);
  L.cnt_fold.alloc((size_t)K * h->rows_p_max * 4);
  L.sum_fold.alloc((size_t)K * h->rows_p_max * 2 * s1.cpp);
  L.mu.alloc(h->rows_p_max);
  L.inv_sd.alloc(h->rows_p_max);
  L.Bv.alloc((size_t)h->rows_p_max * C);
  L.Af.alloc((size_t)K * h->rows_p_max * C);
  L.Qf.alloc((size_t)K * h->rows_p_max * C);
  L.gty_f.alloc((size_t)K * h->rows_p_max * P);
  L.rhs.alloc((size_t)K * h->rows_p_max * P);
  const int Kg = s1.loocv ? 1 : K;
  L.gam.alloc((size_t)Kg * h->rows_p_max * Qp);
  L.gmu.alloc((size_t)Kg * h->rows_p_max * Qp);
  L.cvec.alloc((size_t)Kg * Qp * C);
  L.part.alloc((size_t)d.ntiles_s * Qp * 2);
  L.mean_invsd.alloc((size_t)2 * Qp);

  // --- 1. decode: PLINK rows -> padded 2-bit rows (the tensor-core tiles build their int8 operands from them); on the
  //        sparse Miss path the same pass writes the missing lists and the sample-major rows Gt (miss_gram.cu)
  {
    ScopedTimer t(h, "bed_relayout", s);
    if (s1.gram_dense) {
      launch_bed_relayout(packed_d, row_stride, bs, rows_p, h->file_idx_pad.p, h->word_base.p, h->word_keep.p,
                          ref_first, L.gp.p, Npad, s);
    } else {
      L.miss_total.alloc(1);
      L.miss_seg.alloc((size_t)h->rows_p_max * s1.miss_nct);
      L.miss_list.alloc((size_t)std::max<int64_t>(s1.miss_cap, 1));
      L.gt.alloc((size_t)Npad * (h->rows_p_max / 16));
      BedMissOut mo;
      mo.ctile = s1.miss_ctile.p; mo.nct = s1.miss_nct; mo.rows_p = rows_p;
      mo.total = L.miss_total.p; mo.cap = (unsigned long long)s1.miss_cap;
      mo.seg = L.miss_seg.p; mo.list = L.miss_list.p; mo.gt = L.gt.p;
      launch_bed_relayout_miss(packed_d, row_stride, bs, rows_p, h->file_idx_pad.p, h->word_base.p, h->word_keep.p,
                               ref_first, L.gp.p, Npad, mo, s);
      h->launches += 1;                    // the memset of the total
    }
    if (staged >= 0) RG_CUDA(cudaEventRecord(L.relayout_done[staged].ensure(), s));
  }
  h->launches += 1;

  // --- 2. sufficient statistics: FP64 CUDA-core path (fallback) or, after the Gram, as extra tensor-core tiles
  auto snp_finalize = [&]() {
    SnpFinalizeArgs a;
    a.bs = bs; a.rows_p = rows_p; a.C = C; a.P = P; a.K = K; a.cpp = s1.cpp; a.loocv = s1.loocv;
    a.n_analyzed = h->n_analyzed; a.numtol = 1e-6;
    a.cnt_fold = L.cnt_fold.p; a.sum_fold = L.sum_fold.p; a.XtX_f = s1.XtX_f.p; a.XtY_f = s1.XtY_f.p;
    a.mu = L.mu.p; a.inv_sd = L.inv_sd.p; a.Bv = L.Bv.p; a.Af = L.Af.p; a.Qf = L.Qf.p;
    a.gty_f = L.gty_f.p; a.rhs = L.rhs.p; a.err_slot = s1.err_slot.p;
    a.err_base = (long long)block_id * h->bs_max;
    launch_l0_snp_finalize(a, s);
    h->launches += 1;
  };
  if (!s1.stats_tc) {
    ScopedTimer t(h, "l0_stats", s);
    launch_l0_stats(L.gp.p, Npad, s1.xy.p, s1.cpp, s1.chunks.p, s1.nchunks, rows_p, L.cnt_part.p,
                    L.sum_part.p, s);
    launch_l0_fold_reduce(L.cnt_part.p, L.sum_part.p, rows_p, s1.cpp, s1.fold_chunks.p, K,
                          L.cnt_fold.p, L.sum_fold.p, s);
    snp_finalize();
    h->launches += 2;
  }

  // --- 3. exact integer Grams on the tensor cores
  {
    const TileList& tl =
        cached_tiles(s1.tile_lists, rows_p, [&](std::vector<int2>& tiles) { gram_tile_list(2 * rows_p, tiles); });
    const int64_t zz_stride = (int64_t)4 * rows_p * rows_p;
    ScopedTimer t(h, "gram_wgmma", s);
    if (s1.gram_dense) {
      launch_gram_gp(gp_map(h, L, rows_p), nullptr, rows_p, kZLevel0, tl.buf.p, tl.count, s1.fold_k.p, K,
                     L.zz.p, 2 * rows_p, zz_stride, kZScaleGram, s);
      h->launches += 1;
    } else {
      // the Miss rows: the device picks the sparse sums or the dense tiles from the block's missing-call count
      launch_gram_gp(gp_map(h, L, rows_p), nullptr, rows_p, kZLevel0, tl.buf.p, tl.count, s1.fold_k.p, K,
                     L.zz.p, 2 * rows_p, zz_stride, kZScaleGram, s, 256, L.miss_total.p, s1.miss_cap, rows_p / 128);
      launch_miss_sparse(L.gt.p, rows_p, L.miss_seg.p, s1.miss_nct, s1.miss_fold_ct.p, L.miss_list.p, K,
                         L.miss_total.p, s1.miss_cap, L.zz.p, zz_stride, s);
      h->launches += 2;
    }
    L.last_gram_dense = s1.gram_dense;
  }
  if (s1.stats_tc) {
    // Z [X | Y]-digits: one more column tile per row tile of the same kernel, then the FP64 Horner
    ScopedTimer t(h, "l0_stats", s);
    const int stat_bn = (s1.stat_drows % 256 == 0) ? 256 : 128;
    const TileList& tl = cached_tiles(s1.stat_tile_lists, rows_p, [&](std::vector<int2>& tiles) {
      stat_tile_list(2 * rows_p, s1.stat_drows, stat_bn, tiles);
    });
    L.tstat.alloc((size_t)K * 2 * h->rows_p_max * s1.stat_drows);
    const int64_t tfs = (int64_t)2 * rows_p * s1.stat_drows;
    launch_gram_gp(gp_map(h, L, rows_p), &s1.tmD, rows_p, kZLevel0, tl.buf.p, tl.count, s1.fold_k.p,
                   K, L.tstat.p, s1.stat_drows, tfs, kZScaleStat, s, stat_bn);
    launch_l0_stats_finish(L.tstat.p, s1.stat_drows, tfs, L.zz.p, 2 * rows_p, (int64_t)4 * rows_p * rows_p, rows_p,
                           s1.cpp, C + P, K, s1.xy_scale.p, L.cnt_fold.p, L.sum_fold.p, s);
    snp_finalize();
    h->launches += 2;
  }

  // --- 4./5. ridge systems -> coefficients -> out-of-fold predictions, standardised into W
  const int mx_n = (!s1.loocv && s1.solver_mixed) ? MixedSolver::dim_for(bs) : 0;
  L.last_mx_n = mx_n;
  if (mx_n > 0) {
    enqueue_solve_mixed(h, s1, L, d, mx_n, s);
    enqueue_predict(h, s1, L, d, L.mx_x.p, (int64_t)mx_pp(P) * mx_n, mx_n, 0, s);
    // the flag travels to pinned host memory behind the block; it is read when this lane is next used or at a sync
    RG_CUDA(cudaMemcpyAsync(L.mx_fail_host.p, L.mx_fail.p, sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaEventRecord(L.mx_ev, s));
    L.mx_pending = true; L.mx_bs = bs; L.mx_block_id = block_id;
    s1.mx_blocks += 1;
    return;
  }
  enqueue_solve_f64(h, s1, L, d, s);
  if (!s1.loocv) enqueue_predict(h, s1, L, d, L.cm.p, (int64_t)d.n_aug * d.nC, d.nC, d.nC, s);
}


// One level-0 block from real-valued genotypes: 8-bit BGEN probability pairs (probs / miss) or an FP64 matrix (G64).
// Dense FP64 throughout, like the reference: decode + impute + residualise + scale, per-fold Gram / G Y on the FP64
// tensor pipe, batched Cholesky, out-of-fold (or closed-form leave-one-out) predictions, standardisation into W.
static void l0_block_dense(rg_ctx* h, const uint8_t* probs, const uint8_t* miss, const double* G64, int64_t n_file, int bs,
                           const int32_t* sample_idx, int ref_first, int block_id) {
  Step1State& s1 = step1(h);
  RG_CHECK(n_file > 0, "bad sample count of the genotype file");
  BlockDims d;
  Step1State::Lane& L = l0_begin_block(h, s1, bs, block_id, sample_idx, d);
  resolve_lane(h, s1, L);
  const int C = h->C, P = h->P, K = s1.K, R = s1.R;
  const int64_t Npad = h->Npad;
  cudaStream_t s = L.stream;
  L.last_pred_i8 = 0; L.last_mx_n = 0;     // dense FP64 prediction and Cholesky

  L.gd.alloc((size_t)h->bs_max * Npad);
  L.mu.alloc(h->rows_p_max);
  L.inv_sd.alloc(h->rows_p_max);
  // --- input to the device, then G (FP64, padded fold layout)
  if (G64) {
    const double* src = G64;
    if (!is_device_pointer(G64)) {
      L.dense_in.alloc((size_t)h->bs_max * n_file * 8);
      copy_to_device(L.dense_in.p, G64, (size_t)bs * n_file * 8, s);
      src = reinterpret_cast<const double*>(L.dense_in.p);
    }
    launch_dense_from_f64(src, n_file, bs, h->file_idx_pad.p, L.gd.p, Npad, s);
  } else {
    const uint8_t *pd = probs, *md = miss;
    if (!is_device_pointer(probs)) {
      L.dense_in.alloc((size_t)h->bs_max * n_file * 3);
      copy_to_device(L.dense_in.p, probs, (size_t)bs * n_file * 2, s);
      pd = L.dense_in.p;
      if (miss) {
        copy_to_device(L.dense_in.p + (size_t)h->bs_max * n_file * 2, miss, (size_t)bs * n_file, s);
        md = L.dense_in.p + (size_t)h->bs_max * n_file * 2;
      }
    }
    launch_dense_from_dosage(pd, md, n_file, bs, h->file_idx_pad.p, ref_first, L.gd.p, Npad, s);
  }
  launch_dense_prepare(L.gd.p, Npad, bs, h->file_idx_pad.p, s1.xy.p, s1.cpp, C, h->n_analyzed, 1e-6, L.mu.p, L.inv_sd.p,
                       s1.err_slot.p, (long long)block_id * h->bs_max, s);
  // --- per-chunk G G^T (DMMA) and G Y, summed per fold in a fixed order by the assembler
  const int nC = d.nC, nch = s1.nchunks;
  const int64_t part_stride = (int64_t)nC * nC;
  L.dpart.alloc((size_t)nch * round_up(h->bs_max, 64) * round_up(h->bs_max, 64));
  L.dpart_y.alloc((size_t)P * nch * h->bs_max);
  launch_l1_gram(L.gd.p, Npad, bs, s1.chunks.p, nch, L.dpart.p, part_stride, nC, s);
  for (int p = 0; p < P; ++p)
    launch_l1_xty(L.gd.p, Npad, s1.xy.p, s1.cpp, C + p, s1.chunks.p, nch, L.dpart_y.p + (size_t)p * nch * bs, bs, s);
  ensure_f64_systems(h, s1, L, d, s);
  const int64_t cm_stride = (int64_t)d.n_aug * nC;
  launch_l1_assemble(L.dpart.p, part_stride, nC, L.dpart_y.p, (int64_t)nch * bs, P, s1.fold_chunks.p, K, R, s1.lambda.p, bs,
                     nC, L.cm.p, cm_stride, s1.loocv, s);
  if (s1.loocv) launch_l1_loocv_fill(L.gd.p, Npad, bs, nC, L.cm.p, cm_stride, nC + d.Ppad, R, Npad, s);
  h->launches += 5 + P;
  enqueue_factor_solve_f64(h, s1, L, d, s);
  if (s1.loocv) return;
  launch_dense_predict(L.gd.p, Npad, bs, L.cm.p, cm_stride, nC, nC, R, P, s1.tile_fold.p, s1.mask.p, s1.W_tab.p, d.col0, s);
  const int nparts = launch_l0_colsum(s1.W_tab.p, Npad, d.col0, P, d.Q, d.Qp, L.part.p, s);
  launch_l0_standardize(L.part.p, nparts, d.Qp, d.Q, P, s1.neff.p, L.mean_invsd.p, s1.W_tab.p, Npad, d.col0, s1.is_real.p, s);
  h->launches += 5;
}

// ---- rg_debug_fetch (test hook): a name resolves to device bytes or to a small vector built on the host
struct DebugView {
  const void* dev = nullptr;
  std::vector<uint8_t> host;
  size_t bytes = 0;
};

static DebugView dev_view(const void* p, size_t bytes) {
  DebugView v;
  v.dev = p;
  v.bytes = bytes;
  return v;
}

template <class T>
static DebugView host_view(const T* p, size_t count) {
  DebugView v;
  v.host.assign(reinterpret_cast<const uint8_t*>(p), reinterpret_cast<const uint8_t*>(p + count));
  v.bytes = v.host.size();
  return v;
}

// how Step 2 computed its resident block (digit rows of its trait kind, else the quantitative one's) and its sums
static DebugView s2_debug_view(const rg_ctx* h, const Step2State& s2, const std::string& n) {
  const S2Block& b = s2.block;
  const S2Chr& c = b.kind == S2Block::bt ? static_cast<const S2Chr&>(s2.bt) : s2.qt;
  if (n == "s2_paths") {
    const int64_t v[8] = {c.tc ? 1 : 0, c.nchunk, c.chunk_len, c.drows, s2.nchunks, h->Npad, s2.qt.dp, s2.bt.dp};
    return host_view(v, 8);
  }
  // [rows_p][3][dp] of a quantitative-trait block, [rows_p][4][dp] and counts of a dosage or binary-trait block
  if (n == "s2_sums") return dev_view(b.kind == S2Block::qt ? s2.sums.s3.p : nullptr, (size_t)b.rows_p * 3 * b.dp * 8);
  if (n == "bt_sums") return dev_view(b.dose ? s2.sums.s4.p : nullptr, (size_t)b.rows_p * 4 * b.dp * 8);
  if (n == "bt_nnz") return dev_view(b.dose ? s2.sums.nnz.p : nullptr, (size_t)b.rows_p * 8);
  if (n == "bt_n510") return dev_view(b.dose ? s2.sums.n510.p : nullptr, (size_t)b.rows_p * 8);
  // the tensor sums, when the block is a 2-bit one: its rows [rows_p][Npad/16], the digit sums
  // [nchunk][3 rows_p][drows] of the planes [G; G^2; Miss], and the digit rows of F [drows][Npad] they were taken against
  if (n == "s2_gp") return dev_view(s2.in.gp.p, (size_t)b.rows_p * (h->Npad / 16) * 4);
  if (n == "s2_T" && c.tc) return dev_view(s2.sums.T.p, (size_t)c.nchunk * 3 * b.rows_p * c.drows * 4);
  if (n == "s2_FD" && c.tc) return dev_view(c.FD.p, (size_t)c.drows * h->Npad);
  // GxE interaction state of the chromosome: its feature rows [Npad][nf] once rg_s2_set_interaction has run; the shape,
  // the routes [bs] and the chunk-reduced sums [bs][nf] (defined where the variant's route reads them) of the last
  // rg_s2_interaction call since then
  if (n.compare(0, 4, "int_") == 0) {
    const Step2State::Gxe& g = s2.gxe;
    RG_CHECK(g.set, "no interaction state on this handle: " + n);
    if (n == "int_F") return dev_view(g.F.p, (size_t)h->Npad * g.nf * 8);
    RG_CHECK(g.last_bs > 0, "no rg_s2_interaction call since rg_s2_set_interaction: " + n);
    if (n == "int_paths") {
      const int64_t v[8] = {s2.nchunks, h->Npad, g.nf, g.nr, g.K, ceil_div(h->P, kIntTG), ceil_div(h->Npad, kIntSlab),
                            g.last_bs};
      return host_view(v, 8);
    }
    if (n == "int_route") return dev_view(g.route.p, (size_t)g.last_bs);
    if (n == "int_sums") return dev_view(g.sums.p, (size_t)g.last_bs * g.nf * 8);
  }
  throw Error{"unknown Step-2 debug buffer: " + n};
}

// shape and state of the last level-1 fit
static DebugView l1_debug_view(const rg_ctx* h, const Step1State& s1, const std::string& n) {
  RG_CHECK(s1.l1_done, "no level-1 fit on this handle: " + n);
  const int64_t nC = s1.l1_nC, P = h->P;
  if (n == "l1_dims") {
    const int64_t v[8] = {s1.B, nC, s1.R1, s1.K, s1.l1_nmat, s1.l1_n_aug, s1.l1_nchunks, s1.l1_chunk_len};
    return host_view(v, 8);
  }
  if (n == "l1_chunks") return dev_view(s1.l1_chunks.p, (size_t)s1.l1_nchunks * sizeof(int4));          // (t0, len, fold, 0)
  if (n == "l1_beta" && !s1.loocv) return dev_view(s1.l1_beta.p, (size_t)P * s1.K * s1.R1 * nC * 8);    // [P][K R1][nC]
  if (n == "l1_sums" && !s1.l1_bt) return dev_view(s1.l1_sums.p, (size_t)P * (kMaxRidge * 3 + 2) * 8);
  if (n == "l1_bvec" && s1.loocv) return dev_view(s1.l1_bvec.p, (size_t)P * nC * 8);
  if (n == "l1_hvec" && s1.loocv) return dev_view(s1.l1_hvec.p, (size_t)P * h->Npad * 8);
  throw Error{"no level-1 debug buffer " + n + " for this fit"};
}

// intermediates of the last level-0 block
static DebugView l0_debug_view(rg_ctx* h, Step1State& s1, const std::string& n) {
  RG_CHECK(!s1.lanes.empty(), "no level-0 lane: " + n);
  Step1State::Lane& L = *s1.lanes[s1.last_lane];
  const int rp = s1.last_rows_p;
  if (n == "gp") return dev_view(L.gp.p, (size_t)rp * (h->Npad / 16) * 4);
  if (n == "zz") return dev_view(L.zz.p, (size_t)s1.K * 4 * rp * rp * 4);
  if (n == "tstat" && s1.stats_tc) return dev_view(L.tstat.p, (size_t)s1.K * 2 * rp * s1.stat_drows * 4);  // [K][2 rp][drows]
  if (n == "xyD" && s1.stats_tc) return dev_view(s1.xyD.p, (size_t)s1.stat_drows * h->Npad);                // [drows][Npad]
  if (n == "mu") return dev_view(L.mu.p, (size_t)rp * 8);
  if (n == "inv_sd") return dev_view(L.inv_sd.p, (size_t)rp * 8);
  if (n == "Bv") return dev_view(L.Bv.p, (size_t)rp * h->C * 8);
  if (n == "gty_f") return dev_view(L.gty_f.p, (size_t)s1.K * rp * h->P * 8);
  if (n == "rhs") return dev_view(L.rhs.p, (size_t)s1.K * rp * h->P * 8);
  if (n == "cm") return dev_view(L.cm.p, (size_t)s1.last_nmat * s1.last_n_aug * s1.last_nC * 8);
  if (n == "mean_invsd") return dev_view(L.mean_invsd.p, (size_t)2 * s1.R * h->P * 8);
  if (n == "wraw") return dev_view(L.wraw.p, (size_t)h->P * s1.R * h->Npad * 8);
  if (n == "gam" || n == "gmu" || n == "cvec") {
    const size_t Kg = s1.loocv ? 1 : s1.K, Qp = (size_t)round_up(s1.R * h->P, predict_qt());
    const DevBuf<double>& b = n == "gam" ? L.gam : n == "gmu" ? L.gmu : L.cvec;
    return dev_view(b.p, (n == "cvec" ? Kg * Qp * h->C : Kg * rp * Qp) * 8);
  }
  if (n == "cnt_fold") return dev_view(L.cnt_fold.p, (size_t)s1.K * rp * 4 * 4);
  if (n == "sum_fold") return dev_view(L.sum_fold.p, (size_t)s1.K * rp * 2 * s1.cpp * 8);
  if (n == "paths") {
    // which kernels produced the last block: statistics on the tensor cores, INT8 prediction, mixed-solver dimension
    const int64_t v[3] = {s1.stats_tc ? 1 : 0, L.last_pred_i8, L.last_mx_n};
    return host_view(v, 3);
  }
  if (n == "dims") {
    const int64_t v[8] = {h->Npad, rp, s1.last_nC, s1.last_n_aug, s1.last_nmat, s1.K, s1.cpp, s1.nchunks};
    return host_view(v, 8);
  }
  if (n == "gram_path") {
    // how the Miss rows of the last block's Gram were computed: 1 = sparse sums, 0 = dense tiles; the block's
    // missing calls (-1 when RG_B200_GRAM=dense skipped the count) and the sparse path's capacity
    int64_t v[3] = {0, -1, s1.miss_cap};
    if (!L.last_gram_dense) {
      RG_CHECK(L.miss_total.p, "debug buffer not filled yet: gram_path");
      unsigned long long tot = 0;
      RG_CUDA(cudaStreamSynchronize(L.stream));
      RG_CUDA(cudaMemcpy(&tot, L.miss_total.p, sizeof(tot), cudaMemcpyDeviceToHost));
      v[0] = (int64_t)tot <= s1.miss_cap ? 1 : 0;
      v[1] = (int64_t)tot;
    }
    return host_view(v, 3);
  }
  if (n == "miss_ctile") return host_view(s1.miss_ctile_host.data(), s1.miss_ctile_host.size());  // (word, words, fold, 0)
  if (n == "miss_seg" || n == "miss_list") {
    // the relayout's missing lists of the last block (sparse path only): seg [rows_p][miss_nct] (offset, count) into
    // list; a view holds them once the block's total is within the capacity
    RG_CHECK(!L.last_gram_dense && L.miss_seg.p, "no missing lists for the last block: " + n);
    if (n == "miss_seg") return dev_view(L.miss_seg.p, (size_t)rp * s1.miss_nct * sizeof(int2));
    return dev_view(L.miss_list.p, (size_t)std::max<int64_t>(s1.miss_cap, 1) * 4);
  }
  if (n == "pad_of") return host_view(s1.pad_of.data(), h->N);
  if (n == "zz_ref") {
    // the integer Grams recomputed on the CUDA cores from the 2-bit rows
    RG_CHECK(L.gp.p, "debug buffer not filled yet: gp");
    const size_t per = (size_t)4 * rp * rp;
    DevBuf<float> ref;
    ref.alloc(per * s1.K);
    RG_CUDA(cudaMemsetAsync(ref.p, 0, per * s1.K * 4, h->stream));
    for (int f = 0; f < s1.K; ++f)
      launch_gram_reference(L.gp.p, h->Npad, rp, (int)s1.fold_pad_start[f], (int)(s1.fold_pad_start[f] + s1.fold_pad_len[f]),
                            ref.p + per * f, 2 * rp, h->stream);
    std::vector<float> v(per * s1.K);
    RG_CUDA(cudaMemcpyAsync(v.data(), ref.p, v.size() * 4, cudaMemcpyDeviceToHost, h->stream));
    RG_CUDA(cudaStreamSynchronize(h->stream));
    return host_view(v.data(), v.size());
  }
  throw Error{"unknown debug buffer: " + n};
}

static DebugView debug_view(rg_ctx* h, const std::string& n, int64_t max_bytes) {
  if (n == "pgen_rows") {
    // the rows the last rg_pgen_decode produced (Step 1: the next lane's input), cut to the caller's buffer
    const DevBuf<uint8_t>& r = h->s1 ? h->s1->lanes[h->s1->next_lane]->packed_dev : h->s2->in.pgen_rows;
    RG_CHECK(r.p, "pgen_rows: no rg_pgen_decode has filled it");
    return dev_view(r.p, std::min<size_t>(r.n, (size_t)std::max<int64_t>(max_bytes, 0)));
  }
  if (h->s2) return s2_debug_view(h, *h->s2, n);
  if (n.compare(0, 3, "l1_") == 0) return l1_debug_view(h, *h->s1, n);
  return l0_debug_view(h, *h->s1, n);
}

// rg_l0_status of an error-slot word; the failure it names goes to rg_last_error
static int64_t l0_status_of(unsigned long long v) {
  if (v == ~0ull) return 0;
  if (v >= (1ull << 40)) set_last_error("Cholesky pivot not positive (system id " + std::to_string(v - (1ull << 40)) + ")");
  else set_last_error("SNP has low variance (index " + std::to_string(v - 1) + ")");
  return (int64_t)v;
}

static int64_t copy_debug_view(const DebugView& v, const std::string& n, void* out, int64_t max_bytes) {
  RG_CHECK(v.dev || !v.host.empty(), "debug buffer not filled yet: " + n);
  RG_CHECK((int64_t)v.bytes <= max_bytes, "buffer too small for " + n + ": it needs " + std::to_string(v.bytes) + " bytes");
  if (v.dev) RG_CUDA(cudaMemcpy(out, v.dev, v.bytes, cudaMemcpyDeviceToHost));
  else memcpy(out, v.host.data(), v.bytes);
  return (int64_t)v.bytes;
}

}  // namespace rg

using namespace rg;

extern "C" {

const char* rg_last_error(void) { return rg::g_last_error.c_str(); }
const char* rg_version(void) { return "regenie_b200 0.1 (sm_90a)"; }

int rg_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

int rg_warmup(int32_t device) {
  RG_API_BEGIN
  require_gpu(device);
  RG_CUDA(cudaSetDevice(device));
  RG_CUDA(cudaFree(nullptr));
  RG_API_END
}

int rg_step1_create(const rg_step1_config* cfg, const double* X, const double* Y, const uint8_t* mask,
                    const uint8_t* in_analysis, const int64_t* fold_sizes, const double* lambda,
                    const double* neff, rg_handle* out) {
  RG_API_BEGIN
  RG_CHECK(cfg && X && Y && mask && in_analysis && lambda && neff && out, "null argument");
  require_gpu(cfg->device);
  RG_CHECK(cfg->n_samples > 0 && cfg->n_cov > 0 && cfg->n_pheno > 0, "bad sizes");
  RG_CHECK(cfg->n_cov <= kMaxCov, "too many covariates for this build");
  RG_CHECK(cfg->loocv || (cfg->n_folds >= 2 && cfg->n_folds <= kMaxFolds), "n_folds out of range");
  RG_CHECK(cfg->n_ridge_l0 >= 1 && cfg->max_block_size >= 1 && cfg->total_blocks >= 1, "bad sizes");
  RG_CUDA(cudaSetDevice(cfg->device));
  std::unique_ptr<rg_ctx> h(new rg_ctx());
  h->s1 = std::make_unique<Step1State>();
  Step1State& s1 = *h->s1;
  h->device = cfg->device;
  h->stream.ensure();
  {
    // The CUDA driver multiplexes streams onto CUDA_DEVICE_MAX_CONNECTIONS hardware queues (default 8, read when the context
    // is created); streams that share a queue serialise behind each other, which is why more than 8 lanes do not pay at the
    // default.  With 32 queues 12 lanes do - but a context with 32 queues takes about a second longer
    // to create (RG_B200_PHASES of rgb200), so the library leaves the choice to the process: a long job exports
    // CUDA_DEVICE_MAX_CONNECTIONS=32 before its first CUDA call (bench.py does), a short one does not.
    int nl = 8;
    if (const char* q = getenv("CUDA_DEVICE_MAX_CONNECTIONS")) if (atoi(q) >= 16) nl = 12;
    if (const char* e = getenv("RG_B200_LANES")) nl = std::max(1, std::min(32, atoi(e)));
    for (int i = 0; i < nl; ++i) {
      s1.lanes.push_back(std::make_unique<Step1State::Lane>());
      s1.lanes.back()->stream.ensure();
    }
  }
  h->N = cfg->n_samples; h->C = cfg->n_cov; h->P = cfg->n_pheno;
  s1.loocv = cfg->loocv ? 1 : 0;
  s1.K = s1.loocv ? 1 : cfg->n_folds;
  s1.R = cfg->n_ridge_l0; s1.R1 = cfg->n_ridge_l1;
  h->bs_max = cfg->max_block_size;
  h->rows_p_max = (int)round_up(h->bs_max, kRowPad);
  s1.total_blocks = cfg->total_blocks;
  s1.B = (int64_t)s1.total_blocks * s1.R;
  h->n_analyzed = cfg->n_analyzed;
  if (const char* e = getenv("RG_B200_SOLVER")) s1.solver_mixed = std::string(e) == "f64" ? 0 : 1;
  if (const char* e = getenv("RG_B200_MX_TOL")) s1.mx_tol = (float)atof(e);
  build_layout(h.get(), s1, X, Y, mask, in_analysis, fold_sizes);
  s1.lambda.alloc(s1.R);
  s1.neff.alloc(h->P);
  RG_CUDA(cudaMemcpy(s1.lambda.p, lambda, s1.R * 8, cudaMemcpyHostToDevice));
  RG_CUDA(cudaMemcpy(s1.neff.p, neff, h->P * 8, cudaMemcpyHostToDevice));
  s1.err_slot.alloc(1);
  RG_CUDA(cudaMemset(s1.err_slot.p, 0xFF, 8));
  s1.W_owned.assign(h->P, 1);                 // storage itself is allocated on first use (rg::ensure_W)
  // every level-0 kernel addresses W through this table; rg_W_attach_peer redirects a phenotype to the HBM of
  // the GPU that owns its level-1 fit (stores travel over NVLink as the tiles are produced)
  s1.W_host_tab.assign(h->P, nullptr);
  s1.W_tab.alloc(h->P);
  s1.l1_select.assign(h->P, 1);
  *out = h.release();
  RG_API_END
}

void rg_destroy(rg_handle h) {
  if (!h) return;
  cudaSetDevice(h->device);
  std::vector<cudaStream_t> streams{h->stream};
  if (h->s1) {
    streams.push_back(h->s1->poll_stream);
    for (auto& l : h->s1->lanes) streams.insert(streams.end(), {l->stream, l->copy_stream});
  }
  if (h->s2) streams.push_back(h->s2->stage.copy_stream);
  for (cudaStream_t s : streams) if (s) cudaStreamSynchronize(s);
  rg::flush_timers(h);
  delete h;                                 // the members release their streams, events, pinned buffers and mappings
}

int rg_W_export(rg_handle h, void* ipc_handle_64) {
  RG_API_BEGIN
  RG_CHECK(h && ipc_handle_64, "bad argument");
  Step1State& s1 = step1(h);
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  RG_CUDA(cudaSetDevice(h->device));
  ensure_W(h, s1);
  cudaIpcMemHandle_t mh;
  RG_CUDA(cudaIpcGetMemHandle(&mh, s1.W.p));
  memcpy(ipc_handle_64, &mh, 64);
  RG_API_END
}

int rg_W_set_owned(rg_handle h, const uint8_t* owned) {
  RG_API_BEGIN
  RG_CHECK(h && owned, "bad argument");
  Step1State& s1 = step1(h);
  rg::sync_lanes(h);
  RG_CHECK(!s1.W.p, "rg_W_set_owned must be called before the first block / export");
  s1.W_owned.assign(owned, owned + h->P);
  for (int p = 0; p < h->P; ++p) s1.l1_select[p] = owned[p] ? 1 : 0;
  ensure_W(h, s1);
  RG_API_END
}

int rg_W_attach_peer(rg_handle h, const void* ipc_handle_64, const uint8_t* owned_by_peer) {
  RG_API_BEGIN
  RG_CHECK(h && ipc_handle_64 && owned_by_peer, "bad argument");
  Step1State& s1 = step1(h);
  rg::sync_lanes(h);
  ensure_W(h, s1);
  cudaIpcMemHandle_t mh;
  memcpy(&mh, ipc_handle_64, 64);
  s1.W_peer_mapped.emplace_back(mh);
  attach_W(h, s1, static_cast<double*>(s1.W_peer_mapped.back().p), owned_by_peer);
  RG_API_END
}

int rg_W_attach_local(rg_handle h, rg_handle peer, const uint8_t* owned_by_peer) {
  RG_API_BEGIN
  RG_CHECK(h && peer && h != peer && owned_by_peer, "bad argument");
  Step1State &s1 = step1(h), &peer1 = step1(peer);
  RG_CHECK(h->P == peer->P && h->Npad == peer->Npad && s1.B == peer1.B, "handles describe different problems");
  RG_CUDA(cudaSetDevice(peer->device));
  ensure_W(peer, peer1);
  rg::sync_lanes(h);
  ensure_W(h, s1);
  if (h->device != peer->device) {
    int can = 0;
    RG_CUDA(cudaDeviceCanAccessPeer(&can, h->device, peer->device));
    RG_CHECK(can, "no peer access between the two devices");
    const cudaError_t e = cudaDeviceEnablePeerAccess(peer->device, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
    else RG_CUDA(e);
  }
  for (int p = 0; p < h->P; ++p)
    RG_CHECK(!owned_by_peer[p] || peer1.W_owned[p], "the peer does not own storage for a phenotype it is said to own");
  attach_W(h, s1, peer1.W.p, owned_by_peer);
  RG_API_END
}

int rg_l1_select(rg_handle h, const uint8_t* sel) {
  RG_API_BEGIN
  RG_CHECK(h && sel, "bad argument");
  step1(h).l1_select.assign(sel, sel + h->P);
  RG_API_END
}

int rg_sync(rg_handle h) {
  RG_API_BEGIN
  RG_CHECK(h, "null handle");
  rg::sync_lanes(h);
  RG_CUDA(cudaStreamSynchronize(h->stream));
  rg::flush_timers(h);
  rg::pgen_check_errors(h);
  RG_API_END
}

int rg_fence(rg_handle h) {
  RG_API_BEGIN
  RG_CHECK(h, "null handle");
  RG_CUDA(cudaSetDevice(h->device));
  // blocks whose mixed-precision solve raised its flag are re-solved in FP64 first (host waits on those lanes' events)
  if (!h->s1) return 0;
  for (auto& l : h->s1->lanes) rg::resolve_lane(h, *h->s1, *l);
  for (auto& l : h->s1->lanes) {
    RG_CUDA(cudaEventRecord(l->done.ensure(), l->stream));
    RG_CUDA(cudaStreamWaitEvent(h->stream, l->done, 0));
  }
  RG_API_END
}

int rg_l0_block_bed(rg_handle h, const uint8_t* packed, int64_t row_stride, int32_t bs,
                    const int32_t* sample_idx, int32_t ref_first, int32_t block_id) {
  RG_API_BEGIN
  RG_CHECK(h && packed, "null argument");
  l0_block_bed(h, packed, row_stride, bs, sample_idx, ref_first, block_id);
  RG_CUDA(cudaGetLastError());
  RG_API_END
}

int rg_l0_block_dosage_u8(rg_handle h, const uint8_t* probs, const uint8_t* ploidy_missing, int64_t n_file, int32_t bs,
                          const int32_t* sample_idx, int32_t ref_first, int32_t block_id) {
  RG_API_BEGIN
  RG_CHECK(h && probs, "null argument");
  l0_block_dense(h, probs, ploidy_missing, nullptr, n_file, bs, sample_idx, ref_first, block_id);
  RG_CUDA(cudaGetLastError());
  RG_API_END
}

int rg_l0_block_f64(rg_handle h, const double* G, int64_t n_file, int32_t bs, const int32_t* sample_idx, int32_t block_id) {
  RG_API_BEGIN
  RG_CHECK(h && G, "null argument");
  l0_block_dense(h, nullptr, nullptr, G, n_file, bs, sample_idx, 0, block_id);
  RG_CUDA(cudaGetLastError());
  RG_API_END
}

int rg_l0_wait_input(rg_handle h) {
  RG_API_BEGIN
  RG_CHECK(h, "not a Step-1 handle");     // a null handle is no Step-1 handle either
  Step1State& s1 = step1(h);
  RG_CUDA(cudaSetDevice(h->device));
  Step1State::Lane& L = *s1.lanes[s1.last_lane];
  if (L.h2d_done) RG_CUDA(cudaEventSynchronize(L.h2d_done));
  RG_API_END
}

int rg_l0_load_W(rg_handle h, int32_t block_id, int32_t ph, const double* in) {
  RG_API_BEGIN
  RG_CHECK(h && in, "null argument");
  Step1State& s1 = step1(h);
  RG_CHECK(block_id >= 0 && block_id < s1.total_blocks && ph >= 0 && ph < h->P, "bad index");
  RG_CUDA(cudaSetDevice(h->device));
  std::vector<double> tmp((size_t)h->Npad * s1.R, 0.0);
  for (int r = 0; r < s1.R; ++r)
    for (int64_t s = 0; s < h->N; ++s) tmp[(size_t)r * h->Npad + s1.pad_of[s]] = in[(size_t)r * h->N + s];
  ensure_W(h, s1);
  RG_CHECK(s1.W_host_tab[ph] != nullptr, "this rank holds no storage for that phenotype (rg_W_set_owned)");
  double* dst = s1.W_host_tab[ph] + (size_t)block_id * s1.R * h->Npad;
  RG_CUDA(cudaMemcpyAsync(dst, tmp.data(), tmp.size() * 8, cudaMemcpyHostToDevice, h->stream));
  RG_CUDA(cudaStreamSynchronize(h->stream));
  RG_API_END
}

int64_t rg_l0_status(rg_handle h) {
  if (!h) return -1;
  cudaSetDevice(h->device);
  try { rg::sync_lanes(h); } catch (const rg::Error& e) { rg::set_last_error(e.msg); return -1; }
  if (cudaStreamSynchronize(h->stream) != cudaSuccess) {
    rg::set_last_error(std::string("CUDA error: ") + cudaGetErrorString(cudaGetLastError()));
    return -1;
  }
  rg::flush_timers(h);
  try { rg::pgen_check_errors(h); } catch (const rg::Error& e) { rg::set_last_error(e.msg); return (int64_t)1 << 41; }
  if (!h->s1) return 0;
  unsigned long long v = 0;
  cudaMemcpy(&v, h->s1->err_slot.p, 8, cudaMemcpyDeviceToHost);
  return rg::l0_status_of(v);
}

int64_t rg_l0_poll_status(rg_handle h) {
  if (!h) return -1;
  unsigned long long v = 0;
  try {
    Step1State& s1 = step1(h);
    cudaSetDevice(h->device);
    s1.poll_host.alloc(1);
    const cudaStream_t ps = s1.poll_stream.ensure();
    if (cudaMemcpyAsync(s1.poll_host.p, s1.err_slot.p, 8, cudaMemcpyDeviceToHost, ps) != cudaSuccess ||
        cudaStreamSynchronize(ps) != cudaSuccess)
      throw rg::Error{std::string("CUDA error: ") + cudaGetErrorString(cudaGetLastError())};
    v = *s1.poll_host.p;
  } catch (const rg::Error& e) {
    rg::set_last_error(e.msg);
    return -1;
  }
  return rg::l0_status_of(v);
}

int rg_l0_fetch_W(rg_handle h, int32_t block_id, int32_t ph, double* out) {
  RG_API_BEGIN
  RG_CHECK(h && out, "null argument");
  Step1State& s1 = step1(h);
  RG_CHECK(block_id >= 0 && block_id < s1.total_blocks && ph >= 0 && ph < h->P, "bad index");
  rg::sync_lanes(h);
  std::vector<double> tmp((size_t)h->Npad * s1.R);
  ensure_W(h, s1);
  RG_CHECK(s1.W_host_tab[ph] != nullptr, "this rank holds no storage for that phenotype (rg_W_set_owned)");
  const double* src = s1.W_host_tab[ph] + (size_t)block_id * s1.R * h->Npad;   // local or peer-mapped
  RG_CUDA(cudaMemcpyAsync(tmp.data(), src, tmp.size() * 8, cudaMemcpyDeviceToHost, h->stream));
  RG_CUDA(cudaStreamSynchronize(h->stream));
  for (int r = 0; r < s1.R; ++r)
    for (int64_t s = 0; s < h->N; ++s) out[(size_t)r * h->N + s] = tmp[(size_t)r * h->Npad + s1.pad_of[s]];
  RG_API_END
}

int64_t rg_debug_fetch(rg_handle h, const char* name, void* out, int64_t max_bytes) {
  if (!h || !name || !out) { rg::set_last_error("rg_debug_fetch: null argument"); return -1; }
  cudaSetDevice(h->device);
  try {
    rg::sync_lanes(h);
    cudaStreamSynchronize(h->stream);
    const std::string n(name);
    return rg::copy_debug_view(rg::debug_view(h, n, max_bytes), n, out, max_bytes);
  } catch (const rg::Error& e) {
    rg::set_last_error(e.msg);
    return -1;
  }
}

int rg_l0_solver_stats(rg_handle h, int64_t* mixed_blocks, int64_t* f64_fallbacks) {
  RG_API_BEGIN
  RG_CHECK(h, "not a Step-1 handle");     // a null handle is no Step-1 handle either
  Step1State& s1 = step1(h);
  rg::sync_lanes(h);
  if (mixed_blocks) *mixed_blocks = s1.mx_blocks;
  if (f64_fallbacks) *f64_fallbacks = s1.mx_fallbacks;
  RG_API_END
}

int rg_dbg_mixed_solve(int32_t device, int32_t n, int32_t K, int32_t R, int32_t P, const double* Af,
                       const double* lambda, const double* b, int32_t steps, double tol, double* x_out,
                       float* X_out, uint32_t* fail_out) {
  RG_API_BEGIN
  RG_CHECK(Af && lambda && b && x_out && fail_out, "null argument");
  rg::require_gpu(device);
  RG_CUDA(cudaSetDevice(device));
  const int Pp = (int)rg::round_up(P, 2), nmat = K * R;
  rg::MixedSolver mx;
  mx.prepare(n, K, R, Pp);
  rg::DevBuf<double> dA, dl, db, dx, dr;
  rg::DevBuf<unsigned int> dfail;
  dA.alloc((size_t)K * n * n); dl.alloc(R); db.alloc((size_t)K * Pp * n); dx.alloc((size_t)nmat * Pp * n); dr.alloc((size_t)nmat * Pp * n);
  dfail.alloc(1);
  RG_CUDA(cudaMemset(db.p, 0, db.n * 8));
  RG_CUDA(cudaMemset(dx.p, 0, dx.n * 8));
  RG_CUDA(cudaMemset(dfail.p, 0, 4));
  RG_CUDA(cudaMemcpy(dA.p, Af, dA.n * 8, cudaMemcpyHostToDevice));
  {
    // the systems in FP32 (the product path gets them from l0_assemble_sym_kernel)
    std::vector<float> pl((size_t)K * n * n);
    for (size_t e = 0; e < pl.size(); ++e) pl[e] = (float)Af[e];
    RG_CUDA(cudaMemcpy(mx.a_planes(), pl.data(), pl.size() * 4, cudaMemcpyHostToDevice));
  }
  RG_CUDA(cudaMemcpy(dl.p, lambda, R * 8, cudaMemcpyHostToDevice));
  for (int f = 0; f < K; ++f)
    RG_CUDA(cudaMemcpy(db.p + (size_t)f * Pp * n, b + (size_t)f * P * n, (size_t)P * n * 8, cudaMemcpyHostToDevice));
  rg::Stream st;
  mx.solve(dA.p, dl.p, db.p, dx.p, dr.p, P, steps, (float)tol, dfail.p, st.ensure());
  cudaError_t e = cudaGetLastError();                        // a launch the device refused (shared memory, grid)
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  RG_CHECK(e == cudaSuccess, std::string("mixed solver kernels failed: ") + cudaGetErrorString(e));
  for (int m = 0; m < nmat; ++m)
    RG_CUDA(cudaMemcpy(x_out + (size_t)m * P * n, dx.p + (size_t)m * Pp * n, (size_t)P * n * 8, cudaMemcpyDeviceToHost));
  if (X_out) RG_CUDA(cudaMemcpy(X_out, mx.debug_planes(2), (size_t)nmat * n * n * 4, cudaMemcpyDeviceToHost));
  RG_CUDA(cudaMemcpy(fail_out, dfail.p, 4, cudaMemcpyDeviceToHost));
  RG_API_END
}

int64_t rg_launch_count(rg_handle h) { return h ? h->launches : 0; }
void* rg_stream(rg_handle h) { return h ? (void*)h->stream : nullptr; }

int rg_set_timing(rg_handle h, int32_t enable) {
  RG_API_BEGIN
  RG_CHECK(h, "null handle");
  h->timing = enable != 0;
  RG_API_END
}

int rg_get_timing(rg_handle h, const char* kernel, double* total_ms, int64_t* launches) {
  RG_API_BEGIN
  RG_CHECK(h && kernel, "null argument");
  rg::sync_lanes(h);
  RG_CUDA(cudaStreamSynchronize(h->stream));
  rg::flush_timers(h);
  auto it = h->timers.find(kernel);
  if (total_ms) *total_ms = it == h->timers.end() ? 0.0 : it->second.first;
  if (launches) *launches = it == h->timers.end() ? 0 : it->second.second;
  RG_API_END
}

int rg_timing_reset(rg_handle h) {
  RG_API_BEGIN
  RG_CHECK(h, "null handle");
  RG_CUDA(cudaStreamSynchronize(h->stream));
  rg::flush_timers(h);
  h->timers.clear();
  RG_API_END
}

}  // extern "C"
