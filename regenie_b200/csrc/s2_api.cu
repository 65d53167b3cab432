// Step-2 entry points of the C ABI (include/rg_b200.h).
#include <stdlib.h>

#include <algorithm>
#include <string>

#include "context.cuh"

using namespace rg;

static void s2_create(rg_ctx* h, const rg_step2_config* cfg, const double* X, const uint8_t* mask,
                      const uint8_t* in_analysis) {
  h->kind = 2;
  h->device = cfg->device;
  RG_CUDA(cudaSetDevice(h->device));
  RG_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  h->N = cfg->n_samples; h->C = cfg->n_cov; h->P = cfg->n_pheno; h->K = 1;
  h->bs_max = cfg->max_block_size;
  h->rows_p_max = (int)round_up(h->bs_max, kRowPad);
  h->n_analyzed = cfg->n_analyzed;
  h->strict = (cfg->strict_mode || h->P == 1) ? 1 : 0;
  const int64_t N = h->N;
  const int C = h->C, P = h->P;
  h->Npad = round_up(N, kSamplePad);
  h->pad_of.resize(N);
  h->src_of.assign(h->Npad, -1);
  for (int64_t s = 0; s < N; ++s) { h->pad_of[s] = (int32_t)s; h->src_of[s] = (int32_t)s; }
  h->in_analysis.assign(in_analysis, in_analysis + N);
  h->Xh.assign(X, X + (size_t)N * C);
  h->maskh.assign(mask, mask + (size_t)N * P);
  h->dp = (int)round_up(1 + C + 2 * P + P * C, 16);
  std::vector<int4> chunks;
  for (int64_t o = 0; o < h->Npad; o += kStatChunk)
    chunks.push_back(make_int4((int)o, (int)std::min<int64_t>(kStatChunk, h->Npad - o), 0, 0));
  h->nchunks = (int)chunks.size();
  h->chunks.alloc(chunks.size());
  RG_CUDA(cudaMemcpy(h->chunks.p, chunks.data(), chunks.size() * sizeof(int4), cudaMemcpyHostToDevice));
  // per-trait constants: mask counts and X_p^T X_p = sum_i m_ip x_i x_i^T
  std::vector<double> mc(P, 0.0), XmX((size_t)P * C * C, 0.0);
  for (int p = 0; p < P; ++p)
    for (int64_t s = 0; s < N; ++s) {
      if (!mask[(size_t)p * N + s]) continue;
      mc[p] += 1.0;
      for (int c = 0; c < C; ++c) {
        const double xc = X[(size_t)c * N + s];
        if (xc == 0.0) continue;
        for (int c2 = 0; c2 < C; ++c2) XmX[((size_t)p * C + c) * C + c2] += xc * X[(size_t)c2 * N + s];
      }
    }
  h->s2_maskcount.alloc(P); h->s2_XmX.alloc(XmX.size()); h->s2_YtX.alloc((size_t)P * C); h->s2_scf.alloc(P);
  RG_CUDA(cudaMemcpy(h->s2_maskcount.p, mc.data(), P * 8, cudaMemcpyHostToDevice));
  RG_CUDA(cudaMemcpy(h->s2_XmX.p, XmX.data(), XmX.size() * 8, cudaMemcpyHostToDevice));
  h->F.alloc((size_t)h->Npad * h->dp);
  h->err_slot.alloc(1);
  RG_CUDA(cudaMemset(h->err_slot.p, 0xFF, 8));
}

// tensor-core statistics for 2-bit input: digit rows of the chromosome's feature matrix (exact, see s2_kernels.cu)
static void s2_build_digits(rg_ctx* h, const double* Fdev, int dp, int D) {
  // read on every call (once per chromosome), like RG_B200_STATS at level 0, so each handle follows the current setting
  const char* e = getenv("RG_B200_S2_STATS");
  h->s2_tc = !(e && std::string(e) == "f64");
  if (!h->s2_tc) {
    h->s2_nchunk = 0; h->s2_chunk_len = 0; h->s2_drows = 0;
    return;
  }
  cudaStream_t s = h->stream;
  h->s2_ncol = D;
  h->s2_drows = (int)round_up((int64_t)ceil_div(D, kStatQ) * 128, 256);
  h->s2_FD.alloc((size_t)h->s2_drows * h->Npad);
  h->s2_Fscale.alloc(dp);
  if (!h->s2_ones.p) {
    h->s2_ones.alloc(h->Npad);
    RG_CUDA(cudaMemsetAsync(h->s2_ones.p, 1, h->Npad, s));
  }
  RG_CUDA(cudaMemsetAsync(h->s2_FD.p, 0, (size_t)h->s2_drows * h->Npad, s));
  launch_l0_xy_digits(Fdev, dp, D, h->Npad, h->s2_ones.p, h->s2_Fscale.p, h->s2_FD.p, s);
  make_gram_tensor_map(&h->s2_tmD, h->s2_FD.p, h->Npad, h->s2_drows);
  // sample chunks: exact integer sums need 60 * chunk < 2^24; more chunks also fill the SMs
  const int ntile = (3 * h->rows_p_max / 128) * (h->s2_drows / 256);
  int64_t nchunk = std::max<int64_t>(ceil_div(h->Npad, (int64_t)262144), ceil_div((int64_t)296, (int64_t)ntile));
  nchunk = std::max<int64_t>(1, std::min<int64_t>(nchunk, h->Npad / 1024));
  const int64_t len = round_up(ceil_div(h->Npad, nchunk), 128);
  std::vector<int2> fk;
  for (int64_t o = 0; o < h->Npad; o += len)
    fk.push_back(make_int2((int)(o / 128), (int)(std::min<int64_t>(len, h->Npad - o) / 128)));
  h->s2_nchunk = (int)fk.size();
  h->s2_chunk_len = len;
  h->s2_fold_k.alloc(fk.size());
  RG_CUDA(cudaMemcpyAsync(h->s2_fold_k.p, fk.data(), fk.size() * sizeof(int2), cudaMemcpyHostToDevice, s));
}

// 2-bit rows in h->gp -> S1 / S2 / Sm digit sums in h->s2_T: the planes [G; G^2; Miss] against the digit rows, INT8 Gram
// kernel
static void s2_tensor_sums(rg_ctx* h, int rows_p, cudaStream_t s) {
  const int drows = h->s2_drows;
  h->s2_T.alloc((size_t)h->s2_nchunk * 3 * h->rows_p_max * drows);
  const rg_ctx::TileList& tl = cached_tiles(h->stat_tile_lists, rows_p * 4096 + drows / 256, [&](std::vector<int2>& tiles) {
    stat_tile_list(3 * rows_p, drows, 256, tiles);
  });
  launch_gram_gp(gp_tensor_map(h->gmaps, h->gp.p, h->Npad, rows_p), &h->s2_tmD, rows_p, kZStep2, tl.buf.p, tl.count,
                 h->s2_fold_k.p, h->s2_nchunk, h->s2_T.p, drows, (int64_t)3 * rows_p * drows, kZScaleStat, s);
}

static void s2_set_chr(rg_ctx* h, const double* res, const double* scf_sv) {
  RG_CHECK(h->kind == 2, "handle is not a Step-2 handle");
  RG_CUDA(cudaSetDevice(h->device));
  const int64_t N = h->N;
  const int C = h->C, P = h->P;
  const bool with_sex = !h->s2_male.empty();
  const int base = 1 + C + 2 * P + P * C;
  h->s2_col_male = with_sex ? base : -1;
  h->dp = (int)round_up(base + (with_sex ? 1 + P : 0), 16);
  h->s2_fcols = base + (with_sex ? 1 + P : 0);
  const int dp = h->dp;
  h->F.alloc((size_t)h->Npad * dp);
  std::vector<double> F((size_t)h->Npad * dp, 0.0), YtX((size_t)P * C, 0.0), male_tot(1 + P, 0.0);
  for (int64_t s = 0; s < N; ++s) {
    double* r = &F[(size_t)s * dp];
    r[0] = h->in_analysis[s] ? 1.0 : 0.0;
    if (with_sex && h->s2_male[s] && h->in_analysis[s]) {
      r[base] = 1.0; male_tot[0] += 1.0;
      for (int p = 0; p < P; ++p)
        if (h->maskh[(size_t)p * N + s]) { r[base + 1 + p] = 1.0; male_tot[1 + p] += 1.0; }
    }
    for (int c = 0; c < C; ++c) r[1 + c] = h->Xh[(size_t)c * N + s];
    for (int p = 0; p < P; ++p) {
      const double m = h->maskh[(size_t)p * N + s] ? 1.0 : 0.0;
      const double rv = res[(size_t)p * N + s];
      r[1 + C + p] = rv;
      r[1 + C + P + p] = m;
      for (int c = 0; c < C; ++c) {
        r[1 + C + 2 * P + p * C + c] = m * r[1 + c];
        YtX[(size_t)p * C + c] += rv * r[1 + c];
      }
    }
  }
  RG_CUDA(cudaMemcpyAsync(h->F.p, F.data(), F.size() * 8, cudaMemcpyHostToDevice, h->stream));
  RG_CUDA(cudaMemcpyAsync(h->s2_YtX.p, YtX.data(), YtX.size() * 8, cudaMemcpyHostToDevice, h->stream));
  RG_CUDA(cudaMemcpyAsync(h->s2_scf.p, scf_sv, P * 8, cudaMemcpyHostToDevice, h->stream));
  h->s2_male_tot.alloc(1 + P);
  RG_CUDA(cudaMemcpyAsync(h->s2_male_tot.p, male_tot.data(), (1 + P) * 8, cudaMemcpyHostToDevice, h->stream));
  s2_build_digits(h, h->F.p, dp, base + (with_sex ? 1 + P : 0));
  RG_CUDA(cudaStreamSynchronize(h->stream));
  h->s2_chr_set = true;
  h->int_set = false;                                                // rg_s2_set_interaction follows, per chromosome
  h->int_last_bs = 0;
  h->s2_dz_qt = false;
}

// per-variant non-PAR flags set by rg_s2_set_non_par apply to exactly one block call
static const uint8_t* take_non_par(rg_ctx* h, int bs) {
  if (!h->s2_nonpar_set) return nullptr;
  h->s2_nonpar_set = false;
  RG_CHECK((int)h->s2_nonpar.n >= bs, "rg_s2_set_non_par was given fewer flags than the block has variants");
  return h->s2_nonpar.p;
}

namespace rg {
// A block whose input pointer lies in a staging buffer (rg_s2_stage) waits for that slot's copy, and only for it: the
// copy of the block AFTER it may already be in flight on the copy stream.
static void s2_wait_stage(rg_ctx* h, const void* in, cudaStream_t s) {
  if (!in) return;
  for (int k = 0; k < rg_ctx::kStageSlots; ++k) {
    if (!h->s2_stage_pending[k] || !h->s2_stage[k].p) continue;
    const uint8_t* b = h->s2_stage[k].p;
    if ((const uint8_t*)in >= b && (const uint8_t*)in < b + h->s2_stage[k].n) {
      RG_CUDA(cudaStreamWaitEvent(s, h->s2_stage_ev[k], 0));
      h->s2_stage_pending[k] = false;
    }
  }
}
}

// Packed per-variant outputs of a block, laid out alike in s2_out_d / s2_out_i and in their pinned host mirrors: f64 slabs
// af, mac, stat, beta, se, chisq [bs_max x P], then af_all, mac_all, scale_fac [bs_max]; i32 slabs ns [bs_max x P], then
// ns_all, flags [bs_max].
static size_t s2_out_f64(const rg_ctx* h) { return (size_t)h->bs_max * (6 * (size_t)h->P + 3); }
static size_t s2_out_i32(const rg_ctx* h) { return (size_t)h->bs_max * ((size_t)h->P + 2); }
static rg_s2_out s2_out_at(const rg_ctx* h, double* d, int32_t* i) {
  const size_t bp = (size_t)h->bs_max * h->P, b1 = h->bs_max;
  rg_s2_out o;
  o.af = d; o.mac = d + bp; o.stat = d + 2 * bp; o.beta = d + 3 * bp; o.se = d + 4 * bp; o.chisq = d + 5 * bp;
  o.af_all = d + 6 * bp; o.mac_all = d + 6 * bp + b1; o.scale_fac = d + 6 * bp + 2 * b1;
  o.ns = i; o.ns_all = i + bp; o.flags = i + bp + b1;
  return o;
}

// Results of a block back to the caller: the packed f64 / i32 output buffers cross PCIe as TWO copies into pinned mirrors
// (instead of twelve copies into whatever memory the caller's arrays live in) and are handed out with memcpy after the
// stream has drained - the block calls are synchronous, so every microsecond of this tail is exposed.
static void s2_copy_out(rg_ctx* h, int bs, const rg_s2_out* out, double* info_out, const double* info_dev, cudaStream_t s) {
  const size_t bp = (size_t)h->bs_max * h->P, nd = s2_out_f64(h), ni = s2_out_i32(h);
  if (h->s2_host_cap < nd + bp) {
    if (h->s2_hd) RG_CUDA(cudaFreeHost(h->s2_hd));
    if (h->s2_hi) RG_CUDA(cudaFreeHost(h->s2_hi));
    RG_CUDA(cudaMallocHost(&h->s2_hd, (nd + bp) * sizeof(double)));
    RG_CUDA(cudaMallocHost(&h->s2_hi, ni * sizeof(int32_t)));
    h->s2_host_cap = nd + bp;
  }
  RG_CUDA(cudaMemcpyAsync(h->s2_hd, h->s2_out_d.p, nd * sizeof(double), cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaMemcpyAsync(h->s2_hi, h->s2_out_i.p, ni * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  if (info_out) RG_CUDA(cudaMemcpyAsync(h->s2_hd + nd, info_dev, (size_t)bs * h->P * 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaStreamSynchronize(s));
  const rg_s2_out m = s2_out_at(h, h->s2_hd, h->s2_hi);
  const size_t vp = (size_t)bs * h->P, v1 = bs;
  auto cp = [](auto* dst, const auto* src, size_t n) { if (dst) memcpy(dst, src, n * sizeof(*src)); };
  cp(out->af, m.af, vp); cp(out->mac, m.mac, vp); cp(out->stat, m.stat, vp); cp(out->beta, m.beta, vp); cp(out->se, m.se, vp);
  cp(out->chisq, m.chisq, vp); cp(out->af_all, m.af_all, v1); cp(out->mac_all, m.mac_all, v1); cp(out->scale_fac, m.scale_fac, v1);
  cp(out->ns, m.ns, vp); cp(out->ns_all, m.ns_all, v1); cp(out->flags, m.flags, v1);
  cp(info_out, h->s2_hd + nd, vp);
}

// What every block route does first: the handle, block-size and chromosome-state checks (quantitative-trait routes need
// rg_s2_set_chr, binary-trait routes rg_s2_set_chr_bt), then the device, the staged copies of the block's inputs, the
// sample index map and the packed output buffers.
static void s2_block_begin(rg_ctx* h, bool bt, int bs, const int32_t* sample_idx, const void* in, const void* in2 = nullptr) {
  RG_CHECK(h->kind == 2, "handle is not a Step-2 handle");
  RG_CHECK(bs > 0 && bs <= h->bs_max, "block size out of range");
  if (bt) RG_CHECK(h->bt_chr_set, "rg_s2_set_chr_bt has not been called");
  else RG_CHECK(h->s2_chr_set, "rg_s2_set_chr has not been called");
  h->s2_dz_qt = false;                                               // set again by a QT route that writes dz
  RG_CUDA(cudaSetDevice(h->device));
  s2_wait_stage(h, in, h->stream);
  s2_wait_stage(h, in2, h->stream);
  ensure_file_idx(h, sample_idx);
  h->s2_out_d.alloc(s2_out_f64(h));
  h->s2_out_i.alloc(s2_out_i32(h));
}

// 2-bit rows of the block on the device: a device pointer as it is, host rows through packed_dev
static const uint8_t* s2_rows_in(rg_ctx* h, const uint8_t* packed, int64_t row_stride, int bs) {
  if (is_device_pointer(packed)) return packed;
  h->packed_dev.alloc((size_t)h->bs_max * row_stride);
  copy_to_device(h->packed_dev.p, packed, (size_t)bs * row_stride, h->stream);
  return h->packed_dev.p;
}

// 8-bit probability pairs and ploidy / missing bytes of the block on the device, likewise through probs_dev / miss_dev
static void s2_probs_in(rg_ctx* h, const uint8_t** probs, const uint8_t** miss, int64_t n_file, int bs) {
  if (is_device_pointer(*probs)) return;
  h->probs_dev.alloc((size_t)h->bs_max * n_file * 2);
  copy_to_device(h->probs_dev.p, *probs, (size_t)bs * n_file * 2, h->stream);
  *probs = h->probs_dev.p;
  if (*miss) {
    h->miss_dev.alloc((size_t)h->bs_max * n_file);
    copy_to_device(h->miss_dev.p, *miss, (size_t)bs * n_file, h->stream);
    *miss = h->miss_dev.p;
  }
}

// the fields S2FinalizeArgs and S2BtFinalizeArgs share, the packed outputs included; consumes the block's non-PAR flags
template <typename Args>
static void s2_finalize_args(rg_ctx* h, Args& a, int bs, int dp, double min_mac, const double* sums, int col_male) {
  a.bs = bs; a.C = h->C; a.P = h->P; a.dp = dp;
  a.n_analyzed = h->n_analyzed; a.n_samples = h->N; a.min_mac = min_mac; a.numtol = 1e-6;
  a.sums = sums; a.non_par = take_non_par(h, bs); a.col_male = col_male;
  const rg_s2_out o = s2_out_at(h, h->s2_out_d.p, h->s2_out_i.p);
  a.af = o.af; a.mac = o.mac; a.stat = o.stat; a.beta = o.beta; a.se = o.se; a.chisq = o.chisq;
  a.af_all = o.af_all; a.mac_all = o.mac_all; a.scale_fac = o.scale_fac;
  a.ns = o.ns; a.ns_all = o.ns_all; a.flags = o.flags;
}

static void s2_block_bed(rg_ctx* h, const uint8_t* packed, int64_t row_stride, int bs, const int32_t* sample_idx,
                         int ref_first, double min_mac, const rg_s2_out* out) {
  s2_block_begin(h, false, bs, sample_idx, packed);
  cudaStream_t s = h->stream;
  const int rows_p = (int)round_up(bs, kRowPad);
  const int64_t Npad = h->Npad;
  const uint8_t* packed_d = s2_rows_in(h, packed, row_stride, bs);
  h->gp.alloc((size_t)h->rows_p_max * (Npad / 16));
  if (!h->s2_tc) h->s2_part.alloc((size_t)h->nchunks * h->rows_p_max * 3 * h->dp);
  h->s2_sums.alloc((size_t)h->rows_p_max * 3 * h->dp);
  launch_bed_relayout(packed_d, row_stride, bs, rows_p, h->file_idx_pad.p, h->word_base.p, h->word_keep.p, ref_first, h->gp.p, Npad, s);
  if (h->s2_tc) {
    s2_tensor_sums(h, rows_p, s);
    launch_s2_tensor_finish(h->s2_T.p, h->s2_drows, (int64_t)3 * rows_p * h->s2_drows, h->s2_nchunk, rows_p, h->dp,
                            h->s2_ncol, h->s2_Fscale.p, h->s2_sums.p, nullptr, nullptr, s);
  } else {
    launch_s2_stats(h->gp.p, Npad, h->F.p, h->dp, h->chunks.p, h->nchunks, rows_p, h->s2_part.p, h->s2_sums.p, s);
  }
  S2FinalizeArgs a;
  s2_finalize_args(h, a, bs, h->dp, min_mac, h->s2_sums.p, h->s2_col_male);
  a.strict = h->strict; a.mask_count = h->s2_maskcount.p; a.YtX = h->s2_YtX.p; a.XmX = h->s2_XmX.p; a.scf_sv = h->s2_scf.p;
  a.male_tot = h->s2_male_tot.p;
  launch_s2_finalize(a, s);
  h->launches += 4;
  if (h->int_set) {                                                  // what rg_s2_interaction reads
    h->dz.alloc((size_t)h->rows_p_max * Npad);
    launch_gp_to_dz(h->gp.p, rows_p, h->dz.p, Npad, s);
    h->launches += 1;
    h->s2_dz_qt = true;
  }
  h->s2_last_bs = bs;
  h->s2_sums_rows = rows_p;
  s2_copy_out(h, bs, out, nullptr, nullptr, s);
}

// ---------------------------------------------------------------- binary traits + 8-bit dosages
static void s2_set_chr_bt(rg_ctx* h, const rg_s2_bt_chr* st) {
  RG_CHECK(h->kind == 2, "handle is not a Step-2 handle");
  RG_CUDA(cudaSetDevice(h->device));
  const int64_t N = h->N, Npad = h->Npad;
  const int C = h->C, P = h->P;
  const bool with_sex = !h->s2_male.empty();
  const int base = 1 + P * (3 + C);
  h->bt_col_male = with_sex ? base : -1;
  const int dp = (int)round_up((int64_t)base + (with_sex ? 1 + P : 0), 16);
  h->bt_dp = dp;
  h->bt_ncol = base + (with_sex ? 1 + P : 0);
  std::vector<double> F((size_t)Npad * dp, 0.0), coltot(dp, 0.0), xwy((size_t)P * C, 0.0);
  std::vector<double> w((size_t)P * Npad, 0.0), gs((size_t)P * Npad, 0.0), off((size_t)P * Npad, 0.0),
      xw((size_t)P * C * Npad, 0.0), phat((size_t)P * Npad, 0.0);
  std::vector<int8_t> ym((size_t)P * Npad, 0);
  for (int64_t s = 0; s < N; ++s) {
    double* r = &F[(size_t)s * dp];
    const bool ina = h->in_analysis[s] != 0;
    r[0] = ina ? 1.0 : 0.0;
    if (with_sex && h->s2_male[s] && ina) {
      r[base] = 1.0;
      for (int p = 0; p < P; ++p) if (h->maskh[(size_t)p * N + s]) r[base + 1 + p] = 1.0;
    }
    for (int p = 0; p < P; ++p) {
      const size_t ps = (size_t)p * N + s, pp = (size_t)p * Npad + s;
      const bool m = h->maskh[ps] != 0;
      const double wv = ina ? st->gamma_sqrt_mask[ps] : 0.0;
      const double yr = st->yres[ps];
      w[pp] = wv; gs[pp] = st->gamma_sqrt[ps]; off[pp] = st->firth_offset ? st->firth_offset[ps] : 0.0;
      phat[pp] = st->y_hat_p ? st->y_hat_p[ps] : 0.0;
      ym[pp] = m ? (st->y_raw[ps] != 0.0 ? 2 : 1) : 0;
      double* f = r + 1 + p * (3 + C);
      f[0] = (m && ina) ? 1.0 : 0.0;
      f[1] = wv * wv;
      f[2] = wv * yr;
      for (int c = 0; c < C; ++c) {
        const double x = st->x_gamma[((size_t)p * C + c) * N + s];
        xw[((size_t)p * C + c) * Npad + s] = x;
        f[3 + c] = wv * x;
        xwy[(size_t)p * C + c] += x * yr;
      }
    }
    if (ina) for (int k = 0; k < dp; ++k) coltot[k] += r[k];
  }
  auto up = [&](auto& buf, const auto& v) {
    buf.alloc(v.size());
    RG_CUDA(cudaMemcpyAsync(buf.p, v.data(), v.size() * sizeof(v[0]), cudaMemcpyHostToDevice, h->stream));
  };
  up(h->bt_F, F); up(h->bt_coltot, coltot); up(h->bt_xwy, xwy); up(h->bt_w, w); up(h->bt_gs, gs);
  up(h->bt_off, off); up(h->bt_xw, xw); up(h->bt_ym, ym); up(h->bt_phat, phat);
  s2_build_digits(h, h->bt_F.p, dp, base + (with_sex ? 1 + P : 0));        // for rg_s2_block_bed_bt
  RG_CUDA(cudaStreamSynchronize(h->stream));
  h->bt_chr_set = true;
}

// the per-variant buffers of the binary-trait finish (S2BtFinalizeArgs), which rg_s2_firth / rg_s2_spa read back
static void s2_bt_outputs(rg_ctx* h, S2BtFinalizeArgs& a) {
  const size_t bp = (size_t)h->bs_max * h->P;
  h->bt_xtwg.alloc(bp * h->C); h->bt_mu.alloc(h->bs_max); h->bt_info.alloc(bp); h->bt_den.alloc(bp);
  a.with_flip = 1; a.col_tot = h->bt_coltot.p; a.xwy = h->bt_xwy.p; a.nz_count = h->bt_nnz.p; a.n510 = h->bt_n510.p;
  a.info = h->bt_info.p; a.xtwg = h->bt_xtwg.p; a.mu = h->bt_mu.p; a.den = h->bt_den.p;
}

static void s2_block_bgen8_bt(rg_ctx* h, const uint8_t* probs, const uint8_t* miss, int64_t n_file, int bs,
                              const int32_t* sample_idx, int ref_first, double min_mac, const rg_s2_out* out,
                              double* info_out) {
  s2_block_begin(h, true, bs, sample_idx, probs, miss);
  cudaStream_t s = h->stream;
  const int dp = h->bt_dp;
  const int rows_p = (int)round_up(bs, kRowPad);
  const int64_t Npad = h->Npad;
  s2_probs_in(h, &probs, &miss, n_file, bs);
  h->dz.alloc((size_t)h->rows_p_max * Npad);
  h->bt_part.alloc((size_t)h->nchunks * h->rows_p_max * 4 * dp);
  h->bt_sums.alloc((size_t)h->rows_p_max * 4 * dp);
  h->bt_nnz.alloc(h->rows_p_max); h->bt_n510.alloc(h->rows_p_max);
  h->bt_cnt_part.alloc((size_t)h->nchunks * h->rows_p_max);
  launch_dosage_relayout(probs, miss, n_file, bs, rows_p, h->file_idx_pad.p, ref_first, h->dz.p, Npad, s);
  launch_dosage_stats(h->dz.p, Npad, h->bt_F.p, dp, h->chunks.p, h->nchunks, rows_p, h->bt_part.p, h->bt_cnt_part.p, h->bt_sums.p,
                      h->bt_nnz.p, h->bt_n510.p, s, h->bt_ncol);
  S2BtFinalizeArgs a;
  s2_bt_outputs(h, a);
  s2_finalize_args(h, a, bs, dp, min_mac, h->bt_sums.p, h->bt_col_male);
  launch_s2_bt_finalize(a, s);
  h->launches += 5;
  h->s2_last_bs = bs;
  h->bt_sums_rows = rows_p; h->bt_sums_dp = dp;
  s2_copy_out(h, bs, out, info_out, a.info, s);
}

// quantitative traits on 8-bit dosages: same statistics kernel, closed-form finish of s2_kernels.cu
static void s2_block_bgen8_qt(rg_ctx* h, const uint8_t* probs, const uint8_t* miss, int64_t n_file, int bs,
                              const int32_t* sample_idx, int ref_first, double min_mac, const rg_s2_out* out,
                              double* info_out) {
  s2_block_begin(h, false, bs, sample_idx, probs, miss);
  cudaStream_t s = h->stream;
  const int dp = h->dp;
  const int rows_p = (int)round_up(bs, kRowPad);
  const int64_t Npad = h->Npad;
  s2_probs_in(h, &probs, &miss, n_file, bs);
  h->dz.alloc((size_t)h->rows_p_max * Npad);
  h->bt_part.alloc((size_t)h->nchunks * h->rows_p_max * 4 * dp);
  h->bt_sums.alloc((size_t)h->rows_p_max * 4 * dp);
  h->bt_nnz.alloc(h->rows_p_max); h->bt_n510.alloc(h->rows_p_max);
  h->s2_sums.alloc((size_t)h->rows_p_max * 3 * dp);
  h->bt_xtwg.alloc((size_t)h->rows_p_max * dp);            // Se in dosage units
  h->bt_info.alloc((size_t)h->bs_max * h->P);
  h->bt_cnt_part.alloc((size_t)h->nchunks * h->rows_p_max);
  launch_dosage_relayout(probs, miss, n_file, bs, rows_p, h->file_idx_pad.p, ref_first, h->dz.p, Npad, s);
  launch_dosage_stats(h->dz.p, Npad, h->F.p, dp, h->chunks.p, h->nchunks, rows_p, h->bt_part.p, h->bt_cnt_part.p, h->bt_sums.p,
                      h->bt_nnz.p, h->bt_n510.p, s, h->s2_fcols);
  launch_dosage_scale(h->bt_sums.p, rows_p, dp, h->s2_sums.p, h->bt_xtwg.p, s);
  S2FinalizeArgs a;
  s2_finalize_args(h, a, bs, dp, min_mac, h->s2_sums.p, h->s2_col_male);
  a.strict = h->strict; a.mask_count = h->s2_maskcount.p; a.YtX = h->s2_YtX.p; a.XmX = h->s2_XmX.p; a.scf_sv = h->s2_scf.p;
  a.male_tot = h->s2_male_tot.p; a.nz_count = h->bt_nnz.p; a.info_sums = h->bt_xtwg.p; a.info = h->bt_info.p;
  launch_s2_finalize(a, s);
  h->launches += 6;
  h->s2_last_bs = bs;
  h->s2_dz_qt = true;
  h->s2_sums_rows = rows_p;
  h->bt_sums_rows = rows_p; h->bt_sums_dp = dp;
  s2_copy_out(h, bs, out, info_out, a.info, s);
}

// binary traits on 2-bit hard calls (.bed / .pgen): tensor-core sums, then the same finish as the dosage path
static void s2_block_bed_bt(rg_ctx* h, const uint8_t* packed, int64_t row_stride, int bs, const int32_t* sample_idx,
                            int ref_first, double min_mac, const rg_s2_out* out) {
  s2_block_begin(h, true, bs, sample_idx, packed);
  RG_CHECK(h->s2_tc, "rg_s2_block_bed_bt needs the tensor-core statistics (RG_B200_S2_STATS=f64 disables them)");
  cudaStream_t s = h->stream;
  const int dp = h->bt_dp;
  const int rows_p = (int)round_up(bs, kRowPad);
  const int64_t Npad = h->Npad;
  const uint8_t* packed_d = s2_rows_in(h, packed, row_stride, bs);
  h->gp.alloc((size_t)h->rows_p_max * (Npad / 16));
  h->dz.alloc((size_t)h->rows_p_max * Npad);
  h->bt_sums.alloc((size_t)h->rows_p_max * 4 * dp);
  h->bt_nnz.alloc(h->rows_p_max); h->bt_n510.alloc(h->rows_p_max);
  launch_bed_relayout(packed_d, row_stride, bs, rows_p, h->file_idx_pad.p, h->word_base.p, h->word_keep.p, ref_first, h->gp.p, Npad, s);
  s2_tensor_sums(h, rows_p, s);
  launch_s2_tensor_finish(h->s2_T.p, h->s2_drows, (int64_t)3 * rows_p * h->s2_drows, h->s2_nchunk, rows_p, dp, h->s2_ncol,
                          h->s2_Fscale.p, h->bt_sums.p, h->bt_nnz.p, h->bt_n510.p, s);
  launch_gp_to_dz(h->gp.p, rows_p, h->dz.p, Npad, s);               // what rg_s2_firth / rg_s2_spa read
  S2BtFinalizeArgs a;
  s2_bt_outputs(h, a);
  s2_finalize_args(h, a, bs, dp, min_mac, h->bt_sums.p, h->bt_col_male);
  a.unit = 1.0;
  launch_s2_bt_finalize(a, s);
  h->launches += 5;
  h->s2_last_bs = bs;
  h->bt_sums_rows = rows_p; h->bt_sums_dp = dp;
  s2_copy_out(h, bs, out, nullptr, nullptr, s);
}

// Firth and SPA on (variant, trait) selections of the block left resident by a binary-trait route, kSelBatch at a time.
// `batch(o, nb)` fills its kernel's arguments for selections o .. o + nb (uploaded to firth_sel), launches the kernel and
// queues the copies of its results; the batch is complete when this returns to the loop.
constexpr int kSelBatch = 256;
template <typename Batch>
static void s2_selections(rg_ctx* h, const char* call, int n_sel, const int32_t* var_idx, const int32_t* trait_idx,
                          Batch&& batch) {
  RG_CHECK(h->kind == 2 && h->bt_chr_set && h->s2_last_bs > 0, std::string(call) + " needs a resident dosage block");
  RG_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  for (int k = 0; k < n_sel; ++k)
    RG_CHECK(var_idx[k] >= 0 && var_idx[k] < h->s2_last_bs && trait_idx[k] >= 0 && trait_idx[k] < h->P, "selection out of range");
  h->firth_gvec.alloc((size_t)kSelBatch * h->Npad); h->firth_cflag.alloc((size_t)kSelBatch * h->Npad);
  h->firth_sel.alloc(2 * kSelBatch); h->firth_status.alloc(kSelBatch); h->firth_out.alloc(3 * kSelBatch);
  for (int o = 0; o < n_sel; o += kSelBatch) {
    const int nb = std::min(kSelBatch, n_sel - o);
    RG_CUDA(cudaMemcpyAsync(h->firth_sel.p, var_idx + o, nb * 4, cudaMemcpyHostToDevice, s));
    RG_CUDA(cudaMemcpyAsync(h->firth_sel.p + kSelBatch, trait_idx + o, nb * 4, cudaMemcpyHostToDevice, s));
    batch(o, nb);
    h->launches += 1;
    RG_CUDA(cudaStreamSynchronize(s));
  }
}

static void s2_firth(rg_ctx* h, int n_sel, const int32_t* var_idx, const int32_t* trait_idx, double* beta, double* se,
                     double* lrt, int32_t* status) {
  s2_selections(h, "rg_s2_firth", n_sel, var_idx, trait_idx, [&](int o, int nb) {
    cudaStream_t s = h->stream;
    const rg_s2_out d = s2_out_at(h, h->s2_out_d.p, h->s2_out_i.p);
    FirthArgs a;
    a.n_sel = nb; a.C = h->C; a.P = h->P; a.dp = h->bt_dp; a.niter = 250; a.tol = 2.5e-4; a.maxstep = 5.0;
    a.npad = h->Npad; a.sel_var = h->firth_sel.p; a.sel_trait = h->firth_sel.p + kSelBatch;
    a.dz = h->dz.p; a.F = h->bt_F.p; a.w = h->bt_w.p; a.gs = h->bt_gs.p; a.xw = h->bt_xw.p; a.off = h->bt_off.p;
    a.ym = h->bt_ym.p; a.xtwg = h->bt_xtwg.p; a.mu = h->bt_mu.p; a.mac = d.mac; a.flags = d.flags;
    a.gvec = h->firth_gvec.p; a.cflag = h->firth_cflag.p;
    a.beta = h->firth_out.p; a.se = h->firth_out.p + kSelBatch; a.lrt = h->firth_out.p + 2 * kSelBatch;
    a.status = h->firth_status.p;
    launch_s2_firth(a, s);
    RG_CUDA(cudaMemcpyAsync(beta + o, a.beta, nb * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaMemcpyAsync(se + o, a.se, nb * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaMemcpyAsync(lrt + o, a.lrt, nb * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaMemcpyAsync(status + o, a.status, nb * 4, cudaMemcpyDeviceToHost, s));
  });
}

static void s2_spa(rg_ctx* h, int n_sel, const int32_t* var_idx, const int32_t* trait_idx, double* pval, int32_t* status) {
  s2_selections(h, "rg_s2_spa", n_sel, var_idx, trait_idx, [&](int o, int nb) {
    cudaStream_t s = h->stream;
    const rg_s2_out d = s2_out_at(h, h->s2_out_d.p, h->s2_out_i.p);
    SpaArgs a;
    a.n_sel = nb; a.C = h->C; a.P = h->P; a.dp = h->bt_dp; a.niter = 1000; a.tol = 1.220703125e-4;   // eps^(1/4), src/Regenie.hpp:330
    a.npad = h->Npad; a.sel_var = h->firth_sel.p; a.sel_trait = h->firth_sel.p + kSelBatch;
    a.dz = h->dz.p; a.F = h->bt_F.p; a.w = h->bt_w.p; a.gs = h->bt_gs.p; a.xw = h->bt_xw.p; a.phat = h->bt_phat.p;
    a.ym = h->bt_ym.p; a.xtwg = h->bt_xtwg.p; a.mu = h->bt_mu.p; a.stat = d.stat; a.den = h->bt_den.p; a.flags = d.flags;
    a.gvec = h->firth_gvec.p; a.cflag = h->firth_cflag.p; a.pval = h->firth_out.p; a.status = h->firth_status.p;
    launch_s2_spa(a, s);
    RG_CUDA(cudaMemcpyAsync(pval + o, a.pval, nb * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaMemcpyAsync(status + o, a.status, nb * 4, cudaMemcpyDeviceToHost, s));
  });
}

// ---------------------------------------------------------------- GxE interaction tests (quantitative traits)
// Feature rows [Npad][nf] of s2_int_sums_kernel: robust columns X_c, E X_c, res_p, E res_p (times g), 1, E, E^2 (times
// g^2); then per trait d Px_k, d E Px_k, d yres, d E yres (times g), d^2, d^2 E, d^2 E^2 (times g^2).  Built on the host
// from the state of rg_s2_set_chr (X, res, in_analysis) and the HLM state, like the feature rows of s2_set_chr.
static void s2_set_interaction(rg_ctx* h, const rg_s2_int_chr* st) {
  RG_CHECK(h->kind == 2 && h->s2_chr_set, "rg_s2_set_interaction needs a Step-2 handle after rg_s2_set_chr");
  RG_CHECK(st->n_px >= 0 && (st->n_px == 0 || (st->dinv_sqrt && st->px && st->yres)), "HLM state incomplete");
  RG_CUDA(cudaSetDevice(h->device));
  const int64_t N = h->N, Npad = h->Npad;
  const int C = h->C, P = h->P, K = st->n_px, dp = h->dp;
  const int nr = 2 * C + 2 * P + 3, nh = K > 0 ? P * (2 * K + 5) : 0, nf = nr + nh;
  std::vector<double> E(Npad, 0.0);
  std::vector<uint8_t> pow2(nf, 0);
  for (int k = 0; k < 3; ++k) pow2[2 * C + 2 * P + k] = 1;
  for (int p = 0; p < P && K > 0; ++p)
    for (int k = 0; k < 3; ++k) pow2[nr + p * (2 * K + 5) + 2 * K + 2 + k] = 1;
  for (int64_t s = 0; s < N; ++s) E[s] = h->in_analysis[s] ? st->E[s] : 0.0;
  h->int_F.alloc((size_t)Npad * nf); h->int_E.alloc(Npad); h->int_pow2.alloc(nf);
  RG_CUDA(cudaMemcpyAsync(h->int_E.p, E.data(), Npad * 8, cudaMemcpyHostToDevice, h->stream));
  RG_CUDA(cudaMemcpyAsync(h->int_pow2.p, pow2.data(), nf, cudaMemcpyHostToDevice, h->stream));
  // the rows go up in slabs of kSlab samples, so the host holds one slab of them (and of F) at a time
  constexpr int64_t kSlab = kIntSlab;
  std::vector<double> Fh((size_t)kSlab * dp), F((size_t)kSlab * nf);
  for (int64_t s0 = 0; s0 < Npad; s0 += kSlab) {
    const int64_t ns = std::min(kSlab, Npad - s0);
    RG_CUDA(cudaMemcpyAsync(Fh.data(), h->F.p + (size_t)s0 * dp, (size_t)ns * dp * 8, cudaMemcpyDeviceToHost, h->stream));
    RG_CUDA(cudaStreamSynchronize(h->stream));                       // also: the previous slab's upload has finished
    std::fill(F.begin(), F.end(), 0.0);
    for (int64_t s = s0; s < std::min(s0 + ns, N); ++s) {
      if (!h->in_analysis[s]) continue;
      const double e = E[s];
      const double* fr = &Fh[(size_t)(s - s0) * dp];
      double* r = &F[(size_t)(s - s0) * nf];
      for (int c = 0; c < C; ++c) { r[c] = fr[1 + c]; r[C + c] = e * fr[1 + c]; }
      for (int p = 0; p < P; ++p) { r[2 * C + p] = fr[1 + C + p]; r[2 * C + P + p] = e * fr[1 + C + p]; }
      r[2 * C + 2 * P] = 1.0; r[2 * C + 2 * P + 1] = e; r[2 * C + 2 * P + 2] = e * e;
      for (int p = 0; p < P && K > 0; ++p) {
        double* t = r + nr + p * (2 * K + 5);
        const double d = st->dinv_sqrt[(size_t)p * N + s], y = st->yres[(size_t)p * N + s];
        for (int k = 0; k < K; ++k) {
          const double x = d * st->px[((size_t)p * K + k) * N + s];
          t[k] = x; t[K + k] = e * x;
        }
        t[2 * K] = d * y; t[2 * K + 1] = d * e * y;
        t[2 * K + 2] = d * d; t[2 * K + 3] = d * d * e; t[2 * K + 4] = d * d * e * e;
      }
    }
    RG_CUDA(cudaMemcpyAsync(h->int_F.p + (size_t)s0 * nf, F.data(), (size_t)ns * nf * 8, cudaMemcpyHostToDevice, h->stream));
  }
  RG_CUDA(cudaStreamSynchronize(h->stream));
  h->int_K = K; h->int_nr = nr; h->int_nf = nf;
  h->int_last_bs = 0;
  h->int_set = true;
}

static void s2_interaction(rg_ctx* h, const rg_s2_int_opts* o, int32_t* status, double* coef, double* vcov) {
  RG_CHECK(h->kind == 2 && h->int_set, "rg_s2_interaction needs rg_s2_set_interaction");
  // the genotype words of the last block: written by rg_s2_block_bgen8, and by rg_s2_block_bed only when the interaction
  // state was set before the block ran; any other block call or rg_s2_set_chr since then leaves none for this chromosome
  RG_CHECK(h->s2_dz_qt && h->s2_last_bs > 0,
           "rg_s2_interaction needs the block of the last rg_s2_block_bed / rg_s2_block_bgen8 call, run after "
           "rg_s2_set_interaction on the current chromosome");
  RG_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  const int bs = h->s2_last_bs, P = h->P, C = h->C, nf = h->int_nf;
  const int bs_pad = (int)round_up(bs, 16);
  const rg_s2_out d = s2_out_at(h, h->s2_out_d.p, h->s2_out_i.p);
  S2IntArgs a;
  a.bs = bs; a.C = C; a.P = P; a.dp = h->dp; a.K = h->int_K; a.nf = nf; a.nr = h->int_nr; a.nchunks = h->nchunks;
  a.var_stride = 8 + 2 * C + 2 * P;
  a.force_robust = o->force_robust; a.force_hc4 = o->force_hc4; a.no_robust = o->no_robust;
  a.n_analyzed = h->n_analyzed; a.n_samples = h->N;
  a.rare_mac = o->rare_mac; a.min_mac = o->min_mac; a.numtol = 1e-6;
  a.npad = h->Npad; a.dz = h->dz.p; a.Fint = h->int_F.p; a.F = h->F.p; a.E = h->int_E.p; a.chunks = h->chunks.p;
  a.af_all = d.af_all; a.mac = d.mac; a.YtX = h->s2_YtX.p; a.scf_sv = h->s2_scf.p; a.mask_count = h->s2_maskcount.p;
  a.flags = d.flags;
  h->int_part.alloc((size_t)h->nchunks * bs_pad * nf);
  h->int_sums.alloc((size_t)bs * nf);
  h->int_var.alloc((size_t)bs * a.var_stride);
  h->int_meat.alloc((size_t)bs * P * h->nchunks * 4);
  h->int_out.alloc((size_t)bs * P * 6);
  h->int_status.alloc((size_t)bs * P);
  h->int_route.alloc(bs);
  a.route = h->int_route.p;
  a.sums = h->int_sums.p; a.var = h->int_var.p; a.meat_part = h->int_meat.p; a.status = h->int_status.p;
  a.coef = h->int_out.p; a.vcov = h->int_out.p + (size_t)bs * P * 2;
  launch_s2_interaction(a, h->int_pow2.p, h->int_part.p, s);
  h->launches += 5;
  h->int_last_bs = bs;
  RG_CUDA(cudaMemcpyAsync(status, a.status, (size_t)bs * P * 4, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaMemcpyAsync(coef, a.coef, (size_t)bs * P * 2 * 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaMemcpyAsync(vcov, a.vcov, (size_t)bs * P * 4 * 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaStreamSynchronize(s));
}

extern "C" {

int rg_s2_set_interaction(rg_handle h, const rg_s2_int_chr* st) {
  RG_API_BEGIN
  RG_CHECK(h && st && st->E, "null argument");
  s2_set_interaction(h, st);
  RG_API_END
}

int rg_s2_interaction(rg_handle h, const rg_s2_int_opts* opts, int32_t* status, double* coef, double* vcov) {
  RG_API_BEGIN
  RG_CHECK(h && opts && status && coef && vcov, "null argument");
  s2_interaction(h, opts, status, coef, vcov);
  RG_CUDA(cudaGetLastError());
  RG_API_END
}

int rg_s2_spa(rg_handle h, int32_t n_sel, const int32_t* variant_idx, const int32_t* trait_idx, double* pval,
              int32_t* status) {
  RG_API_BEGIN
  RG_CHECK(h && (n_sel == 0 || (variant_idx && trait_idx && pval && status)), "null argument");
  if (n_sel > 0) s2_spa(h, n_sel, variant_idx, trait_idx, pval, status);
  RG_CUDA(cudaGetLastError());
  RG_API_END
}

int rg_s2_set_sex(rg_handle h, const uint8_t* male) {
  RG_API_BEGIN
  RG_CHECK(h && h->kind == 2, "bad argument");
  if (male) h->s2_male.assign(male, male + h->N); else h->s2_male.clear();
  RG_API_END
}

int rg_s2_set_non_par(rg_handle h, const uint8_t* flags, int32_t n) {
  RG_API_BEGIN
  RG_CHECK(h && h->kind == 2 && flags && n > 0, "bad argument");
  RG_CUDA(cudaSetDevice(h->device));
  h->s2_nonpar.alloc(std::max<size_t>((size_t)n, (size_t)h->bs_max));
  RG_CUDA(cudaMemcpyAsync(h->s2_nonpar.p, flags, n, cudaMemcpyHostToDevice, h->stream));
  RG_CUDA(cudaStreamSynchronize(h->stream));
  h->s2_nonpar_set = true;
  RG_API_END
}

int rg_s2_set_chr_bt(rg_handle h, const rg_s2_bt_chr* st) {
  RG_API_BEGIN
  RG_CHECK(h && st && st->gamma_sqrt_mask && st->gamma_sqrt && st->yres && st->x_gamma && st->y_raw, "null argument");
  s2_set_chr_bt(h, st);
  RG_API_END
}

int rg_s2_block_bgen8_bt(rg_handle h, const uint8_t* probs, const uint8_t* ploidy_missing, int64_t n_file, int32_t bs,
                         const int32_t* sample_idx, int32_t ref_first, double min_mac, const rg_s2_out* out,
                         double* info_out) {
  RG_API_BEGIN
  RG_CHECK(h && probs && out, "null argument");
  s2_block_bgen8_bt(h, probs, ploidy_missing, n_file, bs, sample_idx, ref_first, min_mac, out, info_out);
  RG_CUDA(cudaGetLastError());
  RG_API_END
}

int rg_s2_block_bgen8(rg_handle h, const uint8_t* probs, const uint8_t* ploidy_missing, int64_t n_file, int32_t bs,
                      const int32_t* sample_idx, int32_t ref_first, double min_mac, const rg_s2_out* out,
                      double* info_out) {
  RG_API_BEGIN
  RG_CHECK(h && probs && out, "null argument");
  s2_block_bgen8_qt(h, probs, ploidy_missing, n_file, bs, sample_idx, ref_first, min_mac, out, info_out);
  RG_CUDA(cudaGetLastError());
  RG_API_END
}

int rg_s2_block_bed_bt(rg_handle h, const uint8_t* packed, int64_t row_stride, int32_t bs, const int32_t* sample_idx,
                       int32_t ref_first, double min_mac, const rg_s2_out* out) {
  RG_API_BEGIN
  RG_CHECK(h && packed && out, "null argument");
  s2_block_bed_bt(h, packed, row_stride, bs, sample_idx, ref_first, min_mac, out);
  RG_CUDA(cudaGetLastError());
  RG_API_END
}

int rg_s2_firth(rg_handle h, int32_t n_sel, const int32_t* variant_idx, const int32_t* trait_idx, double* beta,
                double* se, double* lrt, int32_t* status) {
  RG_API_BEGIN
  RG_CHECK(h && (n_sel == 0 || (variant_idx && trait_idx && beta && se && lrt && status)), "null argument");
  if (n_sel > 0) s2_firth(h, n_sel, variant_idx, trait_idx, beta, se, lrt, status);
  RG_CUDA(cudaGetLastError());
  RG_API_END
}

int rg_s2_stage(rg_handle h, int32_t slot, const void* host, int64_t bytes, const uint8_t** dev) {
  RG_API_BEGIN
  RG_CHECK(h && host && dev && bytes > 0, "null argument");
  RG_CHECK(h->kind == 2, "handle is not a Step-2 handle");
  RG_CHECK(slot >= 0 && slot < rg_ctx::kStageSlots, "staging slot out of range");
  RG_CUDA(cudaSetDevice(h->device));
  if (!h->s2_copy_stream) RG_CUDA(cudaStreamCreateWithFlags(&h->s2_copy_stream, cudaStreamNonBlocking));
  if (!h->s2_stage_ev[slot]) RG_CUDA(cudaEventCreateWithFlags(&h->s2_stage_ev[slot], cudaEventDisableTiming));
  if (h->s2_stage[slot].n < (size_t)bytes) {            // grows only between blocks: nothing reads the old buffer any more
    RG_CUDA(cudaStreamSynchronize(h->s2_copy_stream));
    RG_CUDA(cudaStreamSynchronize(h->stream));
    h->s2_stage[slot].alloc((size_t)bytes);
  }
  RG_CUDA(cudaMemcpyAsync(h->s2_stage[slot].p, host, (size_t)bytes, cudaMemcpyHostToDevice, h->s2_copy_stream));
  RG_CUDA(cudaEventRecord(h->s2_stage_ev[slot], h->s2_copy_stream));
  h->s2_stage_pending[slot] = true;
  *dev = h->s2_stage[slot].p;
  RG_API_END
}

int rg_host_alloc(void** p, int64_t bytes) {
  RG_API_BEGIN
  RG_CHECK(p && bytes > 0, "bad argument");
  RG_CUDA(cudaMallocHost(p, (size_t)bytes));
  RG_API_END
}

int rg_host_free(void* p) {
  RG_API_BEGIN
  if (p) RG_CUDA(cudaFreeHost(p));
  RG_API_END
}

int rg_step2_create(const rg_step2_config* cfg, const double* X, const uint8_t* mask,
                    const uint8_t* in_analysis, rg_handle* out) {
  RG_API_BEGIN
  RG_CHECK(cfg && X && mask && in_analysis && out, "null argument");
  require_gpu(cfg->device);
  RG_CHECK(cfg->n_samples > 0 && cfg->n_cov > 0 && cfg->n_pheno > 0 && cfg->max_block_size > 0, "bad sizes");
  RG_CHECK(cfg->n_cov <= kMaxCov, "too many covariates for this build");
  std::unique_ptr<rg_ctx> h(new rg_ctx());
  s2_create(h.get(), cfg, X, mask, in_analysis);
  *out = h.release();
  RG_API_END
}

int rg_s2_set_chr(rg_handle h, const double* res, const double* scf_sv) {
  RG_API_BEGIN
  RG_CHECK(h && res && scf_sv, "null argument");
  s2_set_chr(h, res, scf_sv);
  RG_API_END
}

int rg_s2_block_bed(rg_handle h, const uint8_t* packed, int64_t row_stride, int32_t bs,
                    const int32_t* sample_idx, int32_t ref_first, double min_mac, const rg_s2_out* out) {
  RG_API_BEGIN
  RG_CHECK(h && packed && out, "null argument");
  s2_block_bed(h, packed, row_stride, bs, sample_idx, ref_first, min_mac, out);
  RG_CUDA(cudaGetLastError());
  RG_API_END
}

}  // extern "C"
