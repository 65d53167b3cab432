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
  cudaEvent_t a = nullptr, b = nullptr;
  cudaStream_t st;
  ScopedTimer(rg_ctx* h_, const char* n, cudaStream_t s_) : h(h_), name(n), st(s_) {
    if (!h->timing) return;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    cudaEventRecord(a, st);
  }
  ~ScopedTimer() {
    if (!h->timing) return;
    cudaEventRecord(b, st);
    h->pending.emplace_back(name, a, b);
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
    cudaEventDestroy(std::get<1>(t));
    cudaEventDestroy(std::get<2>(t));
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

// Build the padded fold layout + all device state shared by the blocks.
static void build_layout(rg_ctx* h, const double* X, const double* Y, const uint8_t* mask,
                         const uint8_t* in_analysis, const int64_t* fold_sizes) {
  const int64_t N = h->N;
  const int K = h->K, C = h->C, P = h->P;
  h->fold_sizes.assign(K, 0);
  if (h->loocv) {
    h->fold_sizes[0] = N;
  } else {
    int64_t tot = 0;
    for (int f = 0; f < K; ++f) {
      RG_CHECK(fold_sizes[f] > 0, "fold sizes must be positive");
      h->fold_sizes[f] = fold_sizes[f];
      tot += fold_sizes[f];
    }
    RG_CHECK(tot == N, "fold sizes must sum to n_samples");
  }
  h->fold_pad_start.assign(K, 0);
  h->fold_pad_len.assign(K, 0);
  int64_t off = 0;
  for (int f = 0; f < K; ++f) {
    h->fold_pad_start[f] = off;
    h->fold_pad_len[f] = round_up(h->fold_sizes[f], kFoldPad);
    off += h->fold_pad_len[f];
  }
  h->Npad = off;
  RG_CHECK(h->Npad < (1ll << 31), "padded sample count must fit in int32");
  h->pad_of.assign(N, 0);
  h->src_of.assign(h->Npad, -1);
  std::vector<int32_t> tile_fold(h->Npad / 128);
  {
    int64_t s = 0;
    for (int f = 0; f < K; ++f) {
      for (int64_t o = 0; o < h->fold_sizes[f]; ++o, ++s) {
        h->pad_of[s] = (int32_t)(h->fold_pad_start[f] + o);
        h->src_of[h->fold_pad_start[f] + o] = (int32_t)s;
      }
      for (int64_t t = h->fold_pad_start[f]; t < h->fold_pad_start[f] + h->fold_pad_len[f]; t += 128)
        tile_fold[t / 128] = f;
    }
  }
  h->in_analysis.assign(in_analysis, in_analysis + N);

  // (X | Y) sample-major, zero padded to cpp columns
  h->cpp = (int)round_up(C + P, 16);
  std::vector<double> xy((size_t)h->Npad * h->cpp, 0.0);
  std::vector<uint8_t> maskp((size_t)P * h->Npad, 0), is_real(h->Npad, 0);
  h->maskh.assign(mask, mask + (size_t)N * P);
  for (int64_t s = 0; s < N; ++s) {
    const int64_t t = h->pad_of[s];
    is_real[t] = 1;
    double* r = &xy[(size_t)t * h->cpp];
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
      for (int64_t o = 0; o < h->fold_sizes[f]; ++o, ++s)
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
  std::vector<int2> fold_chunks(K), fold_k(K);
  for (int f = 0; f < K; ++f) {
    fold_chunks[f].x = (int)chunks.size();
    for (int64_t o = 0; o < h->fold_pad_len[f]; o += kStatChunk) {
      const int len = (int)std::min<int64_t>(kStatChunk, h->fold_pad_len[f] - o);
      chunks.push_back(make_int4((int)(h->fold_pad_start[f] + o), len, f, 0));
    }
    fold_chunks[f].y = (int)chunks.size();
    fold_k[f] = make_int2((int)(h->fold_pad_start[f] / 128), (int)(h->fold_pad_len[f] / 128));
  }
  h->nchunks = (int)chunks.size();

  cudaStream_t s = h->stream;
  h->xy.alloc(xy.size());
  h->mask.alloc(maskp.size());
  h->is_real.alloc(is_real.size());
  h->tile_fold.alloc(tile_fold.size());
  h->chunks.alloc(chunks.size());
  h->fold_chunks.alloc(K);
  h->fold_k.alloc(K);
  h->XtX_f.alloc(XtX.size());
  h->XtY_f.alloc(XtY.size());
  RG_CUDA(cudaMemcpyAsync(h->xy.p, xy.data(), xy.size() * 8, cudaMemcpyHostToDevice, s));
  RG_CUDA(cudaMemcpyAsync(h->mask.p, maskp.data(), maskp.size(), cudaMemcpyHostToDevice, s));
  RG_CUDA(cudaMemcpyAsync(h->is_real.p, is_real.data(), is_real.size(), cudaMemcpyHostToDevice, s));
  RG_CUDA(cudaMemcpyAsync(h->tile_fold.p, tile_fold.data(), tile_fold.size() * 4, cudaMemcpyHostToDevice, s));
  RG_CUDA(cudaMemcpyAsync(h->chunks.p, chunks.data(), chunks.size() * sizeof(int4), cudaMemcpyHostToDevice, s));
  RG_CUDA(cudaMemcpyAsync(h->fold_chunks.p, fold_chunks.data(), K * sizeof(int2), cudaMemcpyHostToDevice, s));
  RG_CUDA(cudaMemcpyAsync(h->fold_k.p, fold_k.data(), K * sizeof(int2), cudaMemcpyHostToDevice, s));
  RG_CUDA(cudaMemcpyAsync(h->XtX_f.p, XtX.data(), XtX.size() * 8, cudaMemcpyHostToDevice, s));
  RG_CUDA(cudaMemcpyAsync(h->XtY_f.p, XtY.data(), XtY.size() * 8, cudaMemcpyHostToDevice, s));
  // statistics as extra Gram tiles: digit rows of (X | Y), once per run.  Exact while 30 * fold length < 2^24.
  {
    int64_t max_fold = 0;
    for (int f = 0; f < K; ++f) max_fold = std::max(max_fold, h->fold_pad_len[f]);
    const char* e = getenv("RG_B200_STATS");
    h->stats_tc = !(e && std::string(e) == "f64") && max_fold * 30 < (1ll << 24);
    if (h->stats_tc) {
      const int ngroups = (int)ceil_div(C + P, kStatQ);
      h->stat_drows = ngroups * 128;          // an odd group count runs as 128 x 128 tiles (stat_bn)
      h->xyD.alloc((size_t)h->stat_drows * h->Npad);
      h->xy_scale.alloc(h->cpp);
      RG_CUDA(cudaMemsetAsync(h->xyD.p, 0, (size_t)h->stat_drows * h->Npad, s));
      launch_l0_xy_digits(h->xy.p, h->cpp, C + P, h->Npad, h->is_real.p, h->xy_scale.p, h->xyD.p, s);
      make_gram_tensor_map(&h->tmD, h->xyD.p, h->Npad, h->stat_drows);
    }
  }
  // Miss rows of the Gram as sparse sums while a block has at most kMissSparseRate missing calls (miss_gram.cu)
  {
    // RG_B200_GRAM=dense: always the dense tiles; =sparse: a list for every call (tools/miss_rate_sweep.py)
    const char* e = getenv("RG_B200_GRAM");
    const std::string mode = e ? e : "";
    h->gram_dense = mode == "dense";
    const double rate = mode == "sparse" ? 1.0 : kMissSparseRate;
    h->miss_cap = std::min<int64_t>((int64_t)(rate * h->bs_max * h->n_analyzed), INT32_MAX);
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
  h->file_idx_pad.alloc(h->Npad);
  h->word_base.alloc(nw);
  h->word_keep.alloc(nw);
  RG_CUDA(cudaMemcpyAsync(h->word_base.p, wb.data(), nw * 4, cudaMemcpyHostToDevice, h->stream));
  RG_CUDA(cudaMemcpyAsync(h->word_keep.p, wk.data(), nw * 4, cudaMemcpyHostToDevice, h->stream));
  RG_CUDA(cudaMemcpyAsync(h->file_idx_pad.p, fi.data(), fi.size() * 4, cudaMemcpyHostToDevice, h->stream));
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
void ensure_W(::rg_ctx* h) {
  if (h->W.p) return;
  size_t n_owned = 0;
  for (int p = 0; p < h->P; ++p) n_owned += h->W_owned[p] ? 1 : 0;
  const size_t per = (size_t)h->Npad * h->B;
  h->W.alloc(std::max<size_t>(1, n_owned) * per);
  RG_CUDA(cudaMemset(h->W.p, 0, std::max<size_t>(1, n_owned) * per * 8));
  size_t slot = 0;
  for (int p = 0; p < h->P; ++p)
    if (h->W_owned[p]) h->W_host_tab[p] = h->W.p + (slot++) * per;
  RG_CUDA(cudaMemcpy(h->W_tab.p, h->W_host_tab.data(), h->P * sizeof(double*), cudaMemcpyHostToDevice));
}

struct BlockDims {
  int bs, rows_p, nC, Ppad, n_aug, nmat, Q, Qp, col0, block_id, ntiles_s;
};

static int mx_pp(int P) { return (int)round_up(P, 2); }
constexpr int kMxSteps = 3;               // refinement steps of the mixed solver

// Assembler arguments the FP64 and the mixed path share; each path adds the layout of its systems (nC, cm, cm_stride, ldc).
static AssembleArgs assemble_args(const rg_ctx* h, const rg_ctx::Lane& L, const BlockDims& d) {
  AssembleArgs aa;
  aa.bs = d.bs; aa.rows_p = d.rows_p; aa.C = h->C; aa.K = h->K; aa.R = h->R; aa.loocv = h->loocv;
  aa.zz = L.zz.p; aa.ldz = 2 * d.rows_p; aa.zz_fold_stride = (int64_t)4 * d.rows_p * d.rows_p;
  aa.mu = L.mu.p; aa.inv_sd = L.inv_sd.p; aa.Bv = L.Bv.p; aa.Af = L.Af.p; aa.Qf = L.Qf.p;
  aa.lambda = h->lambda.p;
  return aa;
}

// The lane's FP64 systems [nmat][n_aug][nC] (LOOCV: the sample vectors ride along as right-hand-side rows) and the
// inverses of their diagonal blocks, sized for the largest block of the run; the systems are zeroed when allocated.
static void ensure_f64_systems(rg_ctx* h, rg_ctx::Lane& L, const BlockDims& d, cudaStream_t s) {
  const int nC_max = (int)round_up(h->bs_max, 64);
  const size_t need = (size_t)d.nmat * (nC_max + d.Ppad + (h->loocv ? h->Npad : 0)) * nC_max;
  if (L.cm.n < need) {
    L.cm.alloc(need);
    RG_CUDA(cudaMemsetAsync(L.cm.p, 0, need * 8, s));
  }
  L.inv.alloc(chol_inv_elems(nC_max, d.nmat));
}

// LOOCV: closed-form leave-one-out predictions from the factorised systems (src/Step1_Models.cpp:654-663), standardised
// into W (:694-706)
static void enqueue_loocv_predict(rg_ctx* h, rg_ctx::Lane& L, const BlockDims& d, cudaStream_t s) {
  const int P = h->P;
  launch_l0_loocv_pred(L.cm.p, (int64_t)d.n_aug * d.nC, d.nC, d.bs, d.Ppad, P, h->R, h->xy.p, h->cpp, h->C, h->mask.p, h->Npad,
                       h->W_tab.p, d.col0, L.part.p, d.Qp, s);
  launch_l0_std_reduce_only(L.part.p, d.ntiles_s, d.Qp, d.Q, P, h->neff.p, L.mean_invsd.p, s);
  launch_l0_loocv_std_apply(h->W_tab.p, h->Npad, d.col0, P, d.Q, h->mask.p, L.mean_invsd.p, s);
  h->launches += 3;
}

// FP64 path: assemble the K*R shifted systems, batched Cholesky (DMMA), backward substitution; LOOCV predictions
// included (they read the factorisation directly).  Solutions end up in the right-hand-side rows of L.cm.
static void enqueue_solve_f64(rg_ctx* h, rg_ctx::Lane& L, const BlockDims& d, cudaStream_t s) {
  const int C = h->C, P = h->P, R = h->R;
  ensure_f64_systems(h, L, d, s);
  AssembleArgs aa = assemble_args(h, L, d);
  aa.nC = d.nC; aa.cm = L.cm.p; aa.cm_stride = (int64_t)d.n_aug * d.nC; aa.ldc = d.nC;
  {
    ScopedTimer t(h, "l0_assemble", s);
    launch_l0_assemble(aa, L.rhs.p, P, d.Ppad, d.nmat, s);
    h->launches += 2;
  }
  if (h->loocv) {
    ScopedTimer t(h, "loocv_fill", s);
    launch_l0_loocv_fill(L.gp.p, h->Npad, d.bs, d.nC, L.mu.p, L.inv_sd.p, L.Bv.p, C, h->xy.p, h->cpp, L.cm.p, aa.cm_stride,
                         d.nC + d.Ppad, R, s);
    h->launches += 1;
  }
  {
    ScopedTimer t(h, "chol_factor", s);
    launch_chol_factor(L.cm.p, aa.cm_stride, d.nC, d.n_aug, d.nmat, L.inv.p, h->err_slot.p,
                       (long long)(1ll << 40) + (long long)d.block_id * 1024, s);
    h->launches += chol_num_launches(d.nC);
  }
  if (h->loocv) {
    ScopedTimer t(h, "l0_predict", s);
    enqueue_loocv_predict(h, L, d, s);
    return;
  }
  {
    ScopedTimer t(h, "chol_backsolve", s);
    launch_chol_backsolve(L.cm.p, aa.cm_stride, d.nC, P, d.nmat, L.inv.p, s);
    h->launches += 1;
  }
}

// Mixed path: K symmetric FP64 fold systems -> tensor-core factorisation / inverse -> FP64 refinement.  Solutions in L.mx_x.
static void enqueue_solve_mixed(rg_ctx* h, rg_ctx::Lane& L, const BlockDims& d, int n, cudaStream_t s) {
  const int P = h->P, K = h->K, R = h->R;
  const int Pp = mx_pp(P);
  if (!L.mx) {
    L.mx = std::make_unique<MixedSolver>();
    L.mx_fail.alloc(1);
    RG_CUDA(cudaMallocHost(&L.mx_fail_host, sizeof(unsigned int)));
    RG_CUDA(cudaEventCreateWithFlags(&L.mx_ev, cudaEventDisableTiming));
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
  AssembleArgs aa = assemble_args(h, L, d);
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
    L.mx->solve(L.mx_Af.p, h->lambda.p, L.mx_b.p, L.mx_x.p, L.mx_r.p, P, kMxSteps, h->mx_tol, L.mx_fail.p, s, true);
    h->launches += MixedSolver::launches_per_solve(n, kMxSteps, P) - 1;
  }
}

// Out-of-fold predictions from the coefficients x[m][p][i] at xsrc + m * xstride + (xrow0 + p) * xld + i.
static void enqueue_predict(rg_ctx* h, rg_ctx::Lane& L, const BlockDims& d, const double* xsrc, int64_t xstride, int xld,
                            int xrow0, cudaStream_t s) {
  const int C = h->C, P = h->P, K = h->K, R = h->R;
  const int64_t Npad = h->Npad;
  ScopedTimer t(h, "l0_predict", s);
  // raw predictions go to the lane's LOCAL scratch; the standardisation pass reads them there and writes the finished
  // columns into W - the owner's HBM, which may be another GPU's (then only plain stores cross NVLink)
  if (L.wraw.n < (size_t)P * R * Npad) {
    L.wraw.alloc((size_t)P * R * Npad);
    L.wraw_tab.alloc(P);
    std::vector<double*> tab(P);
    for (int p = 0; p < P; ++p) tab[p] = L.wraw.p + (size_t)p * R * Npad;
    RG_CUDA(cudaMemcpyAsync(L.wraw_tab.p, tab.data(), P * sizeof(double*), cudaMemcpyHostToDevice, s));
    RG_CUDA(cudaStreamSynchronize(s));           // tab goes out of scope (once per lane)
  }
  PredictArgs pa;
  pa.bs = d.bs; pa.rows_p = d.rows_p; pa.C = C; pa.P = P; pa.R = R; pa.Qp = d.Qp; pa.cpp = h->cpp;
  pa.col0 = 0; pa.npad = Npad; pa.words_per_row = Npad / 16;
  pa.gp = L.gp.p; pa.tile_fold = h->tile_fold.p; pa.gam = L.gam.p; pa.gmu = L.gmu.p;
  pa.cvec = L.cvec.p; pa.xy = h->xy.p; pa.mask = h->mask.p; pa.W = L.wraw_tab.p; pa.part = L.part.p;
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
    if (!L.gmaps.count(d.rows_p)) {
      CUtensorMap tm;
      make_gp_tensor_map(&tm, L.gp.p, Npad / 16, d.rows_p);
      L.gmaps[d.rows_p] = tm;
    }
    launch_l0_coef_i8(xsrc, xstride, xld, xrow0, R, P, d.Q, d.Qp, d.bs, d.rows_p, K, L.mu.p, L.inv_sd.p, L.Bv.p, C,
                      L.gam.p, L.gmu.p, L.cvec.p, L.dscale.p, L.dig.p, ngroups, s);
    PredictTcArgs ta;
    ta.rows_p = d.rows_p; ta.C = C; ta.P = P; ta.Q = d.Q; ta.Qp = d.Qp; ta.cpp = h->cpp; ta.col0 = 0; ta.ngroups = ngroups;
    ta.npad = Npad; ta.tile_fold = h->tile_fold.p; ta.scale = L.dscale.p; ta.cvec = L.cvec.p;
    ta.xy = h->xy.p; ta.mask = h->mask.p; ta.W = L.wraw_tab.p; ta.part = L.part.p;
    launch_l0_predict_i8(L.gmaps[d.rows_p], L.dmaps[d.rows_p], ta, d.ntiles_s, s);
    h->launches += 2;
  }
  launch_l0_standardize(L.part.p, d.ntiles_s, d.Qp, d.Q, P, h->neff.p, L.mean_invsd.p, h->W_tab.p, Npad, d.col0,
                        h->is_real.p, s, L.wraw_tab.p, 0);
  h->launches += 2;
}

static BlockDims block_dims(const rg_ctx* h, int bs, int block_id) {
  BlockDims d;
  d.bs = bs; d.rows_p = (int)round_up(bs, kRowPad); d.nC = (int)round_up(bs, 64); d.Ppad = (int)round_up(h->P, 64);
  d.n_aug = d.nC + d.Ppad + (h->loocv ? (int)h->Npad : 0);
  d.nmat = (h->loocv ? 1 : h->K) * h->R;
  d.Q = h->R * h->P; d.Qp = (int)round_up(d.Q, predict_qt());
  d.col0 = block_id * h->R; d.block_id = block_id; d.ntiles_s = (int)(h->Npad / 128);
  return d;
}

// Read the mixed-solver flag of the block this lane ran last; if the refinement did not converge (ill-conditioned
// system) or a pivot was not positive, re-solve that block in FP64 from the lane's scratch (statistics, Grams and 2-bit
// rows of the block are still there) and redo its predictions.
void resolve_lane(rg_ctx* h, rg_ctx::Lane& L) {
  if (!L.mx_pending) return;
  RG_CUDA(cudaEventSynchronize(L.mx_ev));
  L.mx_pending = false;
  if (*L.mx_fail_host == 0) return;
  h->mx_fallbacks += 1;
  L.last_mx_n = 0;
  const BlockDims d = block_dims(h, L.mx_bs, L.mx_block_id);
  enqueue_solve_f64(h, L, d, L.stream);
  enqueue_predict(h, L, d, L.cm.p, (int64_t)d.n_aug * d.nC, d.nC, d.nC, L.stream);
}

void sync_lanes(rg_ctx* h) {
  RG_CUDA(cudaSetDevice(h->device));
  for (auto& l : h->lanes) resolve_lane(h, *l);
  for (auto& l : h->lanes) RG_CUDA(cudaStreamSynchronize(l->stream));
}

// What both level-0 block routes do first: check the call, map the samples of the genotype file, take the next lane and
// record the block's dimensions (rg_debug_fetch "dims").  Each route reads the flag of the lane's previous block itself
// (resolve_lane), because the .bed route enqueues its input copy before the host waits on that flag.
static rg_ctx::Lane& l0_begin_block(rg_ctx* h, int bs, int block_id, const int32_t* sample_idx, BlockDims& d) {
  RG_CHECK(h->kind == 1, "handle is not a Step-1 handle");
  RG_CHECK(bs > 0 && bs <= h->bs_max, "block size out of range");
  RG_CHECK(block_id >= 0 && block_id < h->total_blocks, "block_id out of range");
  ensure_W(h);
  for (int p = 0; p < h->P; ++p)
    RG_CHECK(h->W_host_tab[p] != nullptr, "a phenotype has neither local storage nor an attached owner (rg_W_set_owned / rg_W_attach_peer)");
  RG_CUDA(cudaSetDevice(h->device));
  ensure_file_idx(h, sample_idx);
  rg_ctx::Lane& L = *h->lanes[h->next_lane];
  h->last_lane = h->next_lane;
  h->next_lane = (h->next_lane + 1) % (int)h->lanes.size();
  d = block_dims(h, bs, block_id);
  h->last_bs = bs; h->last_rows_p = d.rows_p; h->last_nC = d.nC; h->last_n_aug = d.n_aug; h->last_nmat = d.nmat;
  return L;
}

// Device copy of a tile list, built and uploaded on first use for each rows_p.
template <class Fill>
static const rg_ctx::TileList& cached_tiles(std::map<int, rg_ctx::TileList>& cache, int rows_p, Fill fill) {
  rg_ctx::TileList& e = cache[rows_p];
  if (e.count == 0) {
    std::vector<int2> tiles;
    fill(tiles);
    e.buf.alloc(tiles.size());
    RG_CUDA(cudaMemcpy(e.buf.p, tiles.data(), tiles.size() * sizeof(int2), cudaMemcpyHostToDevice));
    e.count = (int)tiles.size();
  }
  return e;
}

static void l0_block_bed(rg_ctx* h, const uint8_t* packed, int64_t row_stride, int bs,
                         const int32_t* sample_idx, int ref_first, int block_id) {
  BlockDims d;
  rg_ctx::Lane& L = l0_begin_block(h, bs, block_id, sample_idx, d);
  const int C = h->C, P = h->P, K = h->K;
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
    if (!L.copy_stream) RG_CUDA(cudaStreamCreateWithFlags(&L.copy_stream, cudaStreamNonBlocking));
    if (!L.h2d_done) RG_CUDA(cudaEventCreateWithFlags(&L.h2d_done, cudaEventDisableTiming));
    cudaStream_t cs = L.copy_stream;
    // the buffer was last read by the relayout kernel of the block this lane ran two blocks ago
    if (L.relayout_recorded[staged]) RG_CUDA(cudaStreamWaitEvent(cs, L.relayout_done[staged], 0));
    {
      ScopedTimer t(h, "h2d", cs);
      copy_to_device(buf.p, packed, (size_t)bs * row_stride, cs);
    }
    RG_CUDA(cudaEventRecord(L.h2d_done, cs));
    L.h2d_recorded = true;
    RG_CUDA(cudaStreamWaitEvent(s, L.h2d_done, 0));
    packed_d = buf.p;
  }
  resolve_lane(h, L);                      // flag of the block this lane ran before (FP64 re-solve if it was raised)

  // --- scratch
  L.gp.alloc((size_t)h->rows_p_max * (Npad / 16));
  L.z.alloc((size_t)2 * h->rows_p_max * Npad);
  L.zz.alloc((size_t)K * 4 * h->rows_p_max * h->rows_p_max);
  L.cnt_part.alloc((size_t)h->nchunks * h->rows_p_max * 4);
  L.sum_part.alloc((size_t)h->nchunks * h->rows_p_max * 2 * h->cpp);
  L.cnt_fold.alloc((size_t)K * h->rows_p_max * 4);
  L.sum_fold.alloc((size_t)K * h->rows_p_max * 2 * h->cpp);
  L.mu.alloc(h->rows_p_max);
  L.inv_sd.alloc(h->rows_p_max);
  L.Bv.alloc((size_t)h->rows_p_max * C);
  L.Af.alloc((size_t)K * h->rows_p_max * C);
  L.Qf.alloc((size_t)K * h->rows_p_max * C);
  L.gty_f.alloc((size_t)K * h->rows_p_max * P);
  L.rhs.alloc((size_t)K * h->rows_p_max * P);
  const int Kg = h->loocv ? 1 : K;
  L.gam.alloc((size_t)Kg * h->rows_p_max * Qp);
  L.gmu.alloc((size_t)Kg * h->rows_p_max * Qp);
  L.cvec.alloc((size_t)Kg * Qp * C);
  L.part.alloc((size_t)d.ntiles_s * Qp * 2);
  L.mean_invsd.alloc((size_t)2 * Qp);

  // --- 1. decode: PLINK rows -> padded 2-bit rows -> int8 planes
  {
    ScopedTimer t(h, "bed_relayout", s);
    launch_bed_relayout(packed_d, row_stride, bs, rows_p, h->file_idx_pad.p, h->word_base.p, h->word_keep.p, ref_first, L.gp.p, Npad, s);
    if (staged >= 0) {
      if (!L.relayout_done[staged]) RG_CUDA(cudaEventCreateWithFlags(&L.relayout_done[staged], cudaEventDisableTiming));
      RG_CUDA(cudaEventRecord(L.relayout_done[staged], s));
      L.relayout_recorded[staged] = true;
    }
  }
  {
    ScopedTimer t(h, "bed_expand", s);
    launch_bed_expand_fp8(L.gp.p, rows_p, L.z.p, Npad, s);
  }
  h->launches += 2;

  // --- 2. sufficient statistics: FP64 CUDA-core path (fallback) or, after the Gram, as extra tensor-core tiles
  auto snp_finalize = [&]() {
    SnpFinalizeArgs a;
    a.bs = bs; a.rows_p = rows_p; a.C = C; a.P = P; a.K = K; a.cpp = h->cpp; a.loocv = h->loocv;
    a.n_analyzed = h->n_analyzed; a.numtol = 1e-6;
    a.cnt_fold = L.cnt_fold.p; a.sum_fold = L.sum_fold.p; a.XtX_f = h->XtX_f.p; a.XtY_f = h->XtY_f.p;
    a.mu = L.mu.p; a.inv_sd = L.inv_sd.p; a.Bv = L.Bv.p; a.Af = L.Af.p; a.Qf = L.Qf.p;
    a.gty_f = L.gty_f.p; a.rhs = L.rhs.p; a.err_slot = h->err_slot.p;
    a.err_base = (long long)block_id * h->bs_max;
    launch_l0_snp_finalize(a, s);
    h->launches += 1;
  };
  if (!h->stats_tc) {
    ScopedTimer t(h, "l0_stats", s);
    launch_l0_stats(L.gp.p, Npad, h->xy.p, h->cpp, h->chunks.p, h->nchunks, rows_p, L.cnt_part.p,
                    L.sum_part.p, s);
    launch_l0_fold_reduce(L.cnt_part.p, L.sum_part.p, rows_p, h->cpp, h->fold_chunks.p, K,
                          L.cnt_fold.p, L.sum_fold.p, s);
    snp_finalize();
    h->launches += 2;
  }

  // --- 3. exact integer Grams on the tensor cores
  {
    if (!L.tmaps.count(rows_p)) {
      CUtensorMap tm;
      make_gram_tensor_map(&tm, L.z.p, Npad, 2 * rows_p);
      L.tmaps[rows_p] = tm;
    }
    const rg_ctx::TileList& tl =
        cached_tiles(h->tile_lists, rows_p, [&](std::vector<int2>& tiles) { gram_tile_list(2 * rows_p, tiles); });
    const int64_t zz_stride = (int64_t)4 * rows_p * rows_p;
    ScopedTimer t(h, "gram_wgmma", s);
    if (h->gram_dense) {
      launch_gram_wgmma(L.tmaps[rows_p], L.tmaps[rows_p], tl.buf.p, tl.count, h->fold_k.p, K,
                        L.zz.p, 2 * rows_p, zz_stride, kZScaleGram, s);
      h->launches += 1;
    } else {
      // the Miss rows: the device picks the sparse sums or the dense tiles from the block's missing-call count
      L.miss_total.alloc(1);
      L.miss_seg.alloc((size_t)K * h->rows_p_max);
      L.miss_list.alloc((size_t)std::max<int64_t>(h->miss_cap, 1));
      L.gt.alloc((size_t)Npad * (h->rows_p_max / 16));
      launch_miss_list(L.gp.p, Npad, rows_p, h->fold_k.p, K, L.miss_total.p, h->miss_cap, L.miss_seg.p, L.miss_list.p, s);
      launch_miss_transpose(L.gp.p, Npad, rows_p, L.miss_total.p, h->miss_cap, L.gt.p, s);
      launch_gram_wgmma(L.tmaps[rows_p], L.tmaps[rows_p], tl.buf.p, tl.count, h->fold_k.p, K,
                        L.zz.p, 2 * rows_p, zz_stride, kZScaleGram, s, 256, L.miss_total.p, h->miss_cap, rows_p / 128);
      launch_miss_sparse(L.gt.p, rows_p, L.miss_seg.p, L.miss_list.p, K, L.miss_total.p, h->miss_cap, L.zz.p, zz_stride, s);
      h->launches += 5;
    }
    L.last_gram_dense = h->gram_dense;
  }
  if (h->stats_tc) {
    // Z [X | Y]-digits: one more column tile per row tile of the same kernel, then the FP64 Horner
    ScopedTimer t(h, "l0_stats", s);
    const int stat_bn = (h->stat_drows % 256 == 0) ? 256 : 128;
    const rg_ctx::TileList& tl = cached_tiles(h->stat_tile_lists, rows_p, [&](std::vector<int2>& tiles) {
      for (int nj = 0; nj < h->stat_drows / stat_bn; ++nj)
        for (int mi = 0; mi < 2 * rows_p / 128; ++mi) tiles.push_back(make_int2(mi, nj));
    });
    L.tstat.alloc((size_t)K * 2 * h->rows_p_max * h->stat_drows);
    const int64_t tfs = (int64_t)2 * rows_p * h->stat_drows;
    launch_gram_wgmma(L.tmaps[rows_p], h->tmD, tl.buf.p, tl.count, h->fold_k.p,
                      K, L.tstat.p, h->stat_drows, tfs, kZScaleStat, s, stat_bn);
    launch_l0_stats_finish(L.tstat.p, h->stat_drows, tfs, L.zz.p, 2 * rows_p, (int64_t)4 * rows_p * rows_p, rows_p,
                           h->cpp, C + P, K, h->xy_scale.p, L.cnt_fold.p, L.sum_fold.p, s);
    snp_finalize();
    h->launches += 2;
  }

  // --- 4./5. ridge systems -> coefficients -> out-of-fold predictions, standardised into W
  const int mx_n = (!h->loocv && h->solver_mixed) ? MixedSolver::dim_for(bs) : 0;
  L.last_mx_n = mx_n;
  if (mx_n > 0) {
    enqueue_solve_mixed(h, L, d, mx_n, s);
    enqueue_predict(h, L, d, L.mx_x.p, (int64_t)mx_pp(P) * mx_n, mx_n, 0, s);
    // the flag travels to pinned host memory behind the block; it is read when this lane is next used or at a sync
    RG_CUDA(cudaMemcpyAsync(L.mx_fail_host, L.mx_fail.p, sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaEventRecord(L.mx_ev, s));
    L.mx_pending = true; L.mx_bs = bs; L.mx_block_id = block_id;
    h->mx_blocks += 1;
    return;
  }
  enqueue_solve_f64(h, L, d, s);
  if (!h->loocv) enqueue_predict(h, L, d, L.cm.p, (int64_t)d.n_aug * d.nC, d.nC, d.nC, s);
}


// One level-0 block from real-valued genotypes: 8-bit BGEN probability pairs (probs / miss) or an FP64 matrix (G64).
// Dense FP64 throughout, like the reference: decode + impute + residualise + scale, per-fold Gram / G Y on the FP64
// tensor pipe, batched Cholesky, out-of-fold (or closed-form leave-one-out) predictions, standardisation into W.
static void l0_block_dense(rg_ctx* h, const uint8_t* probs, const uint8_t* miss, const double* G64, int64_t n_file, int bs,
                           const int32_t* sample_idx, int ref_first, int block_id) {
  RG_CHECK(n_file > 0, "bad sample count of the genotype file");
  BlockDims d;
  rg_ctx::Lane& L = l0_begin_block(h, bs, block_id, sample_idx, d);
  resolve_lane(h, L);
  const int C = h->C, P = h->P, K = h->K, R = h->R;
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
  launch_dense_prepare(L.gd.p, Npad, bs, h->file_idx_pad.p, h->xy.p, h->cpp, C, h->n_analyzed, 1e-6, L.mu.p, L.inv_sd.p,
                       h->err_slot.p, (long long)block_id * h->bs_max, s);
  // --- per-chunk G G^T (DMMA) and G Y, summed per fold in a fixed order by the assembler
  const int nC = d.nC, nch = h->nchunks;
  const int64_t part_stride = (int64_t)nC * nC;
  L.dpart.alloc((size_t)nch * round_up(h->bs_max, 64) * round_up(h->bs_max, 64));
  L.dpart_y.alloc((size_t)P * nch * h->bs_max);
  launch_l1_gram(L.gd.p, Npad, bs, h->chunks.p, nch, L.dpart.p, part_stride, nC, s);
  for (int p = 0; p < P; ++p)
    launch_l1_xty(L.gd.p, Npad, h->xy.p, h->cpp, C + p, h->chunks.p, nch, L.dpart_y.p + (size_t)p * nch * bs, bs, s);
  ensure_f64_systems(h, L, d, s);
  const int64_t cm_stride = (int64_t)d.n_aug * nC;
  launch_dense_assemble(L.dpart.p, part_stride, nC, L.dpart_y.p, (int64_t)nch * bs, h->fold_chunks.p, K, R, h->lambda.p, bs, nC,
                        P, L.cm.p, cm_stride, h->loocv, s);
  if (h->loocv) launch_dense_loocv_fill(L.gd.p, Npad, bs, nC, L.cm.p, cm_stride, nC + d.Ppad, R, s);
  launch_chol_factor(L.cm.p, cm_stride, nC, d.n_aug, d.nmat, L.inv.p, h->err_slot.p,
                     (long long)(1ll << 40) + (long long)block_id * 1024, s);
  h->launches += 5 + P + chol_num_launches(nC);
  L.part.alloc((size_t)d.ntiles_s * d.Qp * 2);
  L.mean_invsd.alloc((size_t)2 * d.Qp);
  if (h->loocv) {
    enqueue_loocv_predict(h, L, d, s);
    return;
  }
  launch_chol_backsolve(L.cm.p, cm_stride, nC, P, d.nmat, L.inv.p, s);
  launch_dense_predict(L.gd.p, Npad, bs, L.cm.p, cm_stride, nC, nC, R, P, h->tile_fold.p, h->mask.p, h->W_tab.p, d.col0, s);
  const int nparts = launch_l0_colsum(h->W_tab.p, Npad, d.col0, P, d.Q, d.Qp, L.part.p, s);
  launch_l0_standardize(L.part.p, nparts, d.Qp, d.Q, P, h->neff.p, L.mean_invsd.p, h->W_tab.p, Npad, d.col0, h->is_real.p, s);
  h->launches += 6;
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

// how Step 2 computed its last block, and the sums it came from
static DebugView s2_debug_view(const rg_ctx* h, const std::string& n) {
  if (n == "s2_paths") {
    const int64_t v[8] = {h->s2_tc ? 1 : 0, h->s2_nchunk, h->s2_chunk_len, h->s2_drows, h->nchunks, h->Npad, h->dp, h->bt_dp};
    return host_view(v, 8);
  }
  if (n == "s2_sums") return dev_view(h->s2_sums.p, (size_t)h->s2_sums_rows * 3 * h->dp * 8);                 // [rows_p][3][dp]
  if (n == "bt_sums") return dev_view(h->bt_sums.p, (size_t)h->bt_sums_rows * 4 * h->bt_sums_dp * 8);   // [rows_p][4][dp]
  if (n == "bt_nnz") return dev_view(h->bt_nnz.p, (size_t)h->bt_sums_rows * 8);
  if (n == "bt_n510") return dev_view(h->bt_n510.p, (size_t)h->bt_sums_rows * 8);
  throw Error{"unknown Step-2 debug buffer: " + n};
}

// shape and state of the last level-1 fit
static DebugView l1_debug_view(const rg_ctx* h, const std::string& n) {
  RG_CHECK(h->l1_done, "no level-1 fit on this handle: " + n);
  const int64_t nC = h->l1_nC, P = h->P;
  if (n == "l1_dims") {
    const int64_t v[8] = {h->B, nC, h->R1, h->K, h->l1_nmat, h->l1_n_aug, h->l1_nchunks, h->l1_chunk_len};
    return host_view(v, 8);
  }
  if (n == "l1_chunks") return dev_view(h->l1_chunks.p, (size_t)h->l1_nchunks * sizeof(int4));          // (t0, len, fold, 0)
  if (n == "l1_beta" && !h->loocv) return dev_view(h->l1_beta.p, (size_t)P * h->K * h->R1 * nC * 8);    // [P][K R1][nC]
  if (n == "l1_sums" && !h->l1_bt) return dev_view(h->l1_sums.p, (size_t)P * (kMaxRidge * 3 + 2) * 8);
  if (n == "l1_bvec" && h->loocv) return dev_view(h->l1_bvec.p, (size_t)P * nC * 8);
  if (n == "l1_hvec" && h->loocv) return dev_view(h->l1_hvec.p, (size_t)P * h->Npad * 8);
  throw Error{"no level-1 debug buffer " + n + " for this fit"};
}

// intermediates of the last level-0 block
static DebugView l0_debug_view(rg_ctx* h, const std::string& n) {
  RG_CHECK(!h->lanes.empty(), "no level-0 lane: " + n);
  rg_ctx::Lane& L = *h->lanes[h->last_lane];
  const int rp = h->last_rows_p;
  if (n == "gp") return dev_view(L.gp.p, (size_t)rp * (h->Npad / 16) * 4);
  if (n == "z") return dev_view(L.z.p, (size_t)2 * rp * h->Npad);
  if (n == "zz") return dev_view(L.zz.p, (size_t)h->K * 4 * rp * rp * 4);
  if (n == "mu") return dev_view(L.mu.p, (size_t)rp * 8);
  if (n == "inv_sd") return dev_view(L.inv_sd.p, (size_t)rp * 8);
  if (n == "Bv") return dev_view(L.Bv.p, (size_t)rp * h->C * 8);
  if (n == "gty_f") return dev_view(L.gty_f.p, (size_t)h->K * rp * h->P * 8);
  if (n == "rhs") return dev_view(L.rhs.p, (size_t)h->K * rp * h->P * 8);
  if (n == "cm") return dev_view(L.cm.p, (size_t)h->last_nmat * h->last_n_aug * h->last_nC * 8);
  if (n == "mean_invsd") return dev_view(L.mean_invsd.p, (size_t)2 * h->R * h->P * 8);
  if (n == "wraw") return dev_view(L.wraw.p, (size_t)h->P * h->R * h->Npad * 8);
  if (n == "gam" || n == "gmu" || n == "cvec") {
    const size_t Kg = h->loocv ? 1 : h->K, Qp = (size_t)round_up(h->R * h->P, predict_qt());
    const DevBuf<double>& b = n == "gam" ? L.gam : n == "gmu" ? L.gmu : L.cvec;
    return dev_view(b.p, (n == "cvec" ? Kg * Qp * h->C : Kg * rp * Qp) * 8);
  }
  if (n == "cnt_fold") return dev_view(L.cnt_fold.p, (size_t)h->K * rp * 4 * 4);
  if (n == "sum_fold") return dev_view(L.sum_fold.p, (size_t)h->K * rp * 2 * h->cpp * 8);
  if (n == "paths") {
    // which kernels produced the last block: statistics on the tensor cores, INT8 prediction, mixed-solver dimension
    const int64_t v[3] = {h->stats_tc ? 1 : 0, L.last_pred_i8, L.last_mx_n};
    return host_view(v, 3);
  }
  if (n == "dims") {
    const int64_t v[8] = {h->Npad, rp, h->last_nC, h->last_n_aug, h->last_nmat, h->K, h->cpp, h->nchunks};
    return host_view(v, 8);
  }
  if (n == "gram_path") {
    // how the Miss rows of the last block's Gram were computed: 1 = sparse sums, 0 = dense tiles; the block's
    // missing calls (-1 when RG_B200_GRAM=dense skipped the count) and the sparse path's capacity
    int64_t v[3] = {0, -1, h->miss_cap};
    if (!L.last_gram_dense) {
      RG_CHECK(L.miss_total.p, "debug buffer not filled yet: gram_path");
      unsigned long long tot = 0;
      RG_CUDA(cudaStreamSynchronize(L.stream));
      RG_CUDA(cudaMemcpy(&tot, L.miss_total.p, sizeof(tot), cudaMemcpyDeviceToHost));
      v[0] = (int64_t)tot <= h->miss_cap ? 1 : 0;
      v[1] = (int64_t)tot;
    }
    return host_view(v, 3);
  }
  if (n == "pad_of") return host_view(h->pad_of.data(), h->N);
  if (n == "zz_ref") {
    // the integer Grams recomputed on the CUDA cores from the int8 planes
    RG_CHECK(L.z.p, "debug buffer not filled yet: z");
    const size_t per = (size_t)4 * rp * rp;
    DevBuf<float> ref;
    ref.alloc(per * h->K);
    RG_CUDA(cudaMemsetAsync(ref.p, 0, per * h->K * 4, h->stream));
    for (int f = 0; f < h->K; ++f)
      launch_gram_reference(L.z.p, h->Npad, 2 * rp, (int)h->fold_pad_start[f], (int)(h->fold_pad_start[f] + h->fold_pad_len[f]),
                            ref.p + per * f, 2 * rp, h->stream);
    std::vector<float> v(per * h->K);
    RG_CUDA(cudaMemcpyAsync(v.data(), ref.p, v.size() * 4, cudaMemcpyDeviceToHost, h->stream));
    RG_CUDA(cudaStreamSynchronize(h->stream));
    return host_view(v.data(), v.size());
  }
  throw Error{"unknown debug buffer: " + n};
}

static DebugView debug_view(rg_ctx* h, const std::string& n, int64_t max_bytes) {
  if (n == "pgen_rows") {
    // the rows the last rg_pgen_decode produced (Step 1: the next lane's input), cut to the caller's buffer
    const DevBuf<uint8_t>& r = h->kind == 1 && !h->lanes.empty() ? h->lanes[h->next_lane]->packed_dev : h->pgen_rows;
    RG_CHECK(r.p, "pgen_rows: no rg_pgen_decode has filled it");
    return dev_view(r.p, std::min<size_t>(r.n, (size_t)std::max<int64_t>(max_bytes, 0)));
  }
  if (h->kind == 2) return s2_debug_view(h, n);
  if (n.compare(0, 3, "l1_") == 0) return l1_debug_view(h, n);
  return l0_debug_view(h, n);
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
  h->kind = 1;
  h->device = cfg->device;
  RG_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
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
      auto l = std::make_unique<rg_ctx::Lane>();
      RG_CUDA(cudaStreamCreateWithFlags(&l->stream, cudaStreamNonBlocking));
      RG_CUDA(cudaEventCreateWithFlags(&l->done, cudaEventDisableTiming));
      h->lanes.push_back(std::move(l));
    }
  }
  h->N = cfg->n_samples; h->C = cfg->n_cov; h->P = cfg->n_pheno;
  h->loocv = cfg->loocv ? 1 : 0;
  h->K = h->loocv ? 1 : cfg->n_folds;
  h->R = cfg->n_ridge_l0; h->R1 = cfg->n_ridge_l1;
  h->bs_max = cfg->max_block_size;
  h->rows_p_max = (int)round_up(h->bs_max, kRowPad);
  h->total_blocks = cfg->total_blocks;
  h->B = (int64_t)h->total_blocks * h->R;
  h->n_analyzed = cfg->n_analyzed;
  if (const char* e = getenv("RG_B200_SOLVER")) h->solver_mixed = std::string(e) == "f64" ? 0 : 1;
  if (const char* e = getenv("RG_B200_MX_TOL")) h->mx_tol = (float)atof(e);
  build_layout(h.get(), X, Y, mask, in_analysis, fold_sizes);
  h->lambda.alloc(h->R);
  h->neff.alloc(h->P);
  RG_CUDA(cudaMemcpy(h->lambda.p, lambda, h->R * 8, cudaMemcpyHostToDevice));
  RG_CUDA(cudaMemcpy(h->neff.p, neff, h->P * 8, cudaMemcpyHostToDevice));
  h->err_slot.alloc(1);
  RG_CUDA(cudaMemset(h->err_slot.p, 0xFF, 8));
  h->W_owned.assign(h->P, 1);                 // storage itself is allocated on first use (rg::ensure_W)
  // every level-0 kernel addresses W through this table; rg_W_attach_peer redirects a phenotype to the HBM of
  // the GPU that owns its level-1 fit (stores travel over NVLink as the tiles are produced)
  h->W_host_tab.resize(h->P);
  h->W_host_tab.assign(h->P, nullptr);
  h->W_tab.alloc(h->P);
  h->l1_select.assign(h->P, 1);
  *out = h.release();
  RG_API_END
}

void rg_destroy(rg_handle h) {
  if (!h) return;
  cudaSetDevice(h->device);
  for (void* m : h->W_peer_mapped) cudaIpcCloseMemHandle(m);
  if (h->poll_stream) { cudaStreamSynchronize(h->poll_stream); cudaStreamDestroy(h->poll_stream); }
  if (h->poll_host) cudaFreeHost(h->poll_host);
  for (auto& l : h->lanes) cudaStreamSynchronize(l->stream);
  cudaStreamSynchronize(h->stream);
  rg::flush_timers(h);
  for (auto& l : h->lanes) {
    if (l->mx_ev) cudaEventDestroy(l->mx_ev);
    if (l->h2d_done) cudaEventDestroy(l->h2d_done);
    for (int k = 0; k < 2; ++k) if (l->relayout_done[k]) cudaEventDestroy(l->relayout_done[k]);
    if (l->copy_stream) { cudaStreamSynchronize(l->copy_stream); cudaStreamDestroy(l->copy_stream); }
    if (l->mx_fail_host) cudaFreeHost(l->mx_fail_host);
    cudaEventDestroy(l->done);
    cudaStreamDestroy(l->stream);
  }
  cudaStreamDestroy(h->stream);
  if (h->s2_hd) cudaFreeHost(h->s2_hd);
  if (h->s2_hi) cudaFreeHost(h->s2_hi);
  if (h->s2_copy_stream) { cudaStreamSynchronize(h->s2_copy_stream); cudaStreamDestroy(h->s2_copy_stream); }
  for (int k = 0; k < rg_ctx::kStageSlots; ++k) if (h->s2_stage_ev[k]) cudaEventDestroy(h->s2_stage_ev[k]);
  delete h;
}

int rg_W_export(rg_handle h, void* ipc_handle_64) {
  RG_API_BEGIN
  RG_CHECK(h && h->kind == 1 && ipc_handle_64, "bad argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  RG_CUDA(cudaSetDevice(h->device));
  ensure_W(h);
  cudaIpcMemHandle_t mh;
  RG_CUDA(cudaIpcGetMemHandle(&mh, h->W.p));
  memcpy(ipc_handle_64, &mh, 64);
  RG_API_END
}

int rg_W_set_owned(rg_handle h, const uint8_t* owned) {
  RG_API_BEGIN
  RG_CHECK(h && h->kind == 1 && owned, "bad argument");
  rg::sync_lanes(h);
  RG_CHECK(!h->W.p, "rg_W_set_owned must be called before the first block / export");
  h->W_owned.assign(owned, owned + h->P);
  for (int p = 0; p < h->P; ++p) h->l1_select[p] = owned[p] ? 1 : 0;
  ensure_W(h);
  RG_API_END
}

int rg_W_attach_peer(rg_handle h, const void* ipc_handle_64, const uint8_t* owned_by_peer) {
  RG_API_BEGIN
  RG_CHECK(h && h->kind == 1 && ipc_handle_64 && owned_by_peer, "bad argument");
  rg::sync_lanes(h);
  ensure_W(h);
  cudaIpcMemHandle_t mh;
  memcpy(&mh, ipc_handle_64, 64);
  void* base = nullptr;
  RG_CUDA(cudaIpcOpenMemHandle(&base, mh, cudaIpcMemLazyEnablePeerAccess));
  h->W_peer_mapped.push_back(base);
  // the peer's allocation is compact over ITS owned phenotypes (rg_W_set_owned with the same mask on that rank)
  size_t slot = 0;
  for (int p = 0; p < h->P; ++p)
    if (owned_by_peer[p]) {
      h->W_host_tab[p] = static_cast<double*>(base) + (slot++) * (size_t)h->Npad * h->B;
      h->l1_select[p] = 0;
    }
  RG_CUDA(cudaMemcpy(h->W_tab.p, h->W_host_tab.data(), h->P * sizeof(double*), cudaMemcpyHostToDevice));
  RG_API_END
}

int rg_W_attach_local(rg_handle h, rg_handle peer, const uint8_t* owned_by_peer) {
  RG_API_BEGIN
  RG_CHECK(h && peer && h != peer && h->kind == 1 && peer->kind == 1 && owned_by_peer, "bad argument");
  RG_CHECK(h->P == peer->P && h->Npad == peer->Npad && h->B == peer->B, "handles describe different problems");
  RG_CUDA(cudaSetDevice(peer->device));
  ensure_W(peer);
  rg::sync_lanes(h);
  ensure_W(h);
  if (h->device != peer->device) {
    int can = 0;
    RG_CUDA(cudaDeviceCanAccessPeer(&can, h->device, peer->device));
    RG_CHECK(can, "no peer access between the two devices");
    const cudaError_t e = cudaDeviceEnablePeerAccess(peer->device, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
    else RG_CUDA(e);
  }
  size_t slot = 0;
  for (int p = 0; p < h->P; ++p)
    if (owned_by_peer[p]) {
      RG_CHECK(peer->W_owned[p], "the peer does not own storage for a phenotype it is said to own");
      h->W_host_tab[p] = peer->W.p + (slot++) * (size_t)h->Npad * h->B;
      h->l1_select[p] = 0;
    }
  RG_CUDA(cudaMemcpy(h->W_tab.p, h->W_host_tab.data(), h->P * sizeof(double*), cudaMemcpyHostToDevice));
  RG_API_END
}

int rg_l1_select(rg_handle h, const uint8_t* sel) {
  RG_API_BEGIN
  RG_CHECK(h && h->kind == 1 && sel, "bad argument");
  h->l1_select.assign(sel, sel + h->P);
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
  if (h->kind == 1) for (auto& l : h->lanes) rg::resolve_lane(h, *l);
  for (auto& l : h->lanes) {
    RG_CUDA(cudaEventRecord(l->done, l->stream));
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
  RG_CHECK(h && h->kind == 1, "not a Step-1 handle");
  RG_CUDA(cudaSetDevice(h->device));
  rg_ctx::Lane& L = *h->lanes[h->last_lane];
  if (L.h2d_recorded) RG_CUDA(cudaEventSynchronize(L.h2d_done));
  RG_API_END
}

int rg_l0_load_W(rg_handle h, int32_t block_id, int32_t ph, const double* in) {
  RG_API_BEGIN
  RG_CHECK(h && in, "null argument");
  RG_CHECK(h->kind == 1 && block_id >= 0 && block_id < h->total_blocks && ph >= 0 && ph < h->P, "bad index");
  RG_CUDA(cudaSetDevice(h->device));
  std::vector<double> tmp((size_t)h->Npad * h->R, 0.0);
  for (int r = 0; r < h->R; ++r)
    for (int64_t s = 0; s < h->N; ++s) tmp[(size_t)r * h->Npad + h->pad_of[s]] = in[(size_t)r * h->N + s];
  ensure_W(h);
  RG_CHECK(h->W_host_tab[ph] != nullptr, "this rank holds no storage for that phenotype (rg_W_set_owned)");
  double* dst = h->W_host_tab[ph] + (size_t)block_id * h->R * h->Npad;
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
  unsigned long long v = 0;
  cudaMemcpy(&v, h->err_slot.p, 8, cudaMemcpyDeviceToHost);
  if (v == ~0ull) return 0;
  if (v >= (1ull << 40)) {
    rg::set_last_error("Cholesky pivot not positive (system id " + std::to_string(v - (1ull << 40)) + ")");
    return (int64_t)v;
  }
  rg::set_last_error("SNP has low variance (index " + std::to_string(v - 1) + ")");
  return (int64_t)v;
}

int64_t rg_l0_poll_status(rg_handle h) {
  if (!h || h->kind != 1 || !h->err_slot.p) return -1;
  cudaSetDevice(h->device);
  if (!h->poll_stream && cudaStreamCreateWithFlags(&h->poll_stream, cudaStreamNonBlocking) != cudaSuccess) return -1;
  if (!h->poll_host && cudaHostAlloc((void**)&h->poll_host, 8, cudaHostAllocDefault) != cudaSuccess) return -1;
  if (cudaMemcpyAsync(h->poll_host, h->err_slot.p, 8, cudaMemcpyDeviceToHost, h->poll_stream) != cudaSuccess ||
      cudaStreamSynchronize(h->poll_stream) != cudaSuccess) {
    rg::set_last_error(std::string("CUDA error: ") + cudaGetErrorString(cudaGetLastError()));
    return -1;
  }
  const unsigned long long v = *h->poll_host;
  if (v == ~0ull) return 0;
  if (v >= (1ull << 40)) rg::set_last_error("Cholesky pivot not positive (system id " + std::to_string(v - (1ull << 40)) + ")");
  else rg::set_last_error("SNP has low variance (index " + std::to_string(v - 1) + ")");
  return (int64_t)v;
}

int rg_l0_fetch_W(rg_handle h, int32_t block_id, int32_t ph, double* out) {
  RG_API_BEGIN
  RG_CHECK(h && out, "null argument");
  RG_CHECK(h->kind == 1 && block_id >= 0 && block_id < h->total_blocks && ph >= 0 && ph < h->P, "bad index");
  rg::sync_lanes(h);
  std::vector<double> tmp((size_t)h->Npad * h->R);
  ensure_W(h);
  RG_CHECK(h->W_host_tab[ph] != nullptr, "this rank holds no storage for that phenotype (rg_W_set_owned)");
  const double* src = h->W_host_tab[ph] + (size_t)block_id * h->R * h->Npad;   // local or peer-mapped
  RG_CUDA(cudaMemcpyAsync(tmp.data(), src, tmp.size() * 8, cudaMemcpyDeviceToHost, h->stream));
  RG_CUDA(cudaStreamSynchronize(h->stream));
  for (int r = 0; r < h->R; ++r)
    for (int64_t s = 0; s < h->N; ++s) out[(size_t)r * h->N + s] = tmp[(size_t)r * h->Npad + h->pad_of[s]];
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
  RG_CHECK(h && h->kind == 1, "not a Step-1 handle");
  rg::sync_lanes(h);
  if (mixed_blocks) *mixed_blocks = h->mx_blocks;
  if (f64_fallbacks) *f64_fallbacks = h->mx_fallbacks;
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
  cudaStream_t st;
  RG_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  mx.solve(dA.p, dl.p, db.p, dx.p, dr.p, P, steps, (float)tol, dfail.p, st);
  cudaError_t e = cudaGetLastError();                        // a launch the device refused (shared memory, grid)
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  cudaStreamDestroy(st);
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
