// Step-2 entry points of the C ABI (include/rg_b200.h).
#include <stdlib.h>

#include <algorithm>
#include <string>

#include "context.cuh"

using namespace rg;

static void s2_create(rg_ctx* h, const rg_step2_config* cfg, const double* X, const uint8_t* mask,
                      const uint8_t* in_analysis) {
  h->s2 = std::make_unique<Step2State>();
  Step2State& s2 = *h->s2;
  h->device = cfg->device;
  RG_CUDA(cudaSetDevice(h->device));
  h->stream.ensure();
  h->N = cfg->n_samples; h->C = cfg->n_cov; h->P = cfg->n_pheno;
  h->bs_max = cfg->max_block_size;
  h->rows_p_max = (int)round_up(h->bs_max, kRowPad);
  h->n_analyzed = cfg->n_analyzed;
  s2.strict = (cfg->strict_mode || h->P == 1) ? 1 : 0;
  const int64_t N = h->N;
  const int C = h->C, P = h->P;
  h->Npad = round_up(N, kSamplePad);
  h->src_of.assign(h->Npad, -1);
  for (int64_t s = 0; s < N; ++s) h->src_of[s] = (int32_t)s;
  h->in_analysis.assign(in_analysis, in_analysis + N);
  s2.Xh.assign(X, X + (size_t)N * C);
  h->maskh.assign(mask, mask + (size_t)N * P);
  s2.dp = (int)round_up(1 + C + 2 * P + P * C, 16);
  std::vector<int4> chunks;
  for (int64_t o = 0; o < h->Npad; o += kStatChunk)
    chunks.push_back(make_int4((int)o, (int)std::min<int64_t>(kStatChunk, h->Npad - o), 0, 0));
  s2.nchunks = (int)chunks.size();
  upload(s2.chunks, chunks, h->stream);
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
  s2.maskcount.alloc(P); s2.XmX.alloc(XmX.size()); s2.YtX.alloc((size_t)P * C); s2.scf.alloc(P);
  RG_CUDA(cudaMemcpy(s2.maskcount.p, mc.data(), P * 8, cudaMemcpyHostToDevice));
  RG_CUDA(cudaMemcpy(s2.XmX.p, XmX.data(), XmX.size() * 8, cudaMemcpyHostToDevice));
  s2.F.alloc((size_t)h->Npad * s2.dp);
}

// tensor-core statistics for 2-bit input: digit rows of the chromosome's feature matrix (exact, see s2_kernels.cu)
static void s2_build_digits(rg_ctx* h, Step2State& s2, const double* Fdev, int dp, int D) {
  // read on every call (once per chromosome), like RG_B200_STATS at level 0, so each handle follows the current setting
  const char* e = getenv("RG_B200_S2_STATS");
  s2.tc = !(e && std::string(e) == "f64");
  if (!s2.tc) {
    s2.nchunk = 0; s2.chunk_len = 0; s2.drows = 0;
    return;
  }
  cudaStream_t s = h->stream;
  s2.ncol = D;
  s2.drows = (int)round_up((int64_t)ceil_div(D, kStatQ) * 128, 256);
  s2.FD.alloc((size_t)s2.drows * h->Npad);
  s2.Fscale.alloc(dp);
  if (!s2.ones.p) {
    s2.ones.alloc(h->Npad);
    RG_CUDA(cudaMemsetAsync(s2.ones.p, 1, h->Npad, s));
  }
  RG_CUDA(cudaMemsetAsync(s2.FD.p, 0, (size_t)s2.drows * h->Npad, s));
  launch_l0_xy_digits(Fdev, dp, D, h->Npad, s2.ones.p, s2.Fscale.p, s2.FD.p, s);
  make_gram_tensor_map(&s2.tmD, s2.FD.p, h->Npad, s2.drows);
  // sample chunks: exact integer sums need 60 * chunk < 2^24; more chunks also fill the SMs
  const int ntile = (3 * h->rows_p_max / 128) * (s2.drows / 256);
  int64_t nchunk = std::max<int64_t>(ceil_div(h->Npad, (int64_t)262144), ceil_div((int64_t)296, (int64_t)ntile));
  nchunk = std::max<int64_t>(1, std::min<int64_t>(nchunk, h->Npad / 1024));
  const int64_t len = round_up(ceil_div(h->Npad, nchunk), 128);
  std::vector<int2> fk;
  for (int64_t o = 0; o < h->Npad; o += len)
    fk.push_back(make_int2((int)(o / 128), (int)(std::min<int64_t>(len, h->Npad - o) / 128)));
  s2.nchunk = (int)fk.size();
  s2.chunk_len = len;
  upload(s2.fold_k, fk, s);
}

// 2-bit rows in s2.gp -> S1 / S2 / Sm digit sums in s2.T: the planes [G; G^2; Miss] against the digit rows, INT8 Gram
// kernel
static void s2_tensor_sums(rg_ctx* h, Step2State& s2, int rows_p, cudaStream_t s) {
  const int drows = s2.drows;
  s2.T.alloc((size_t)s2.nchunk * 3 * h->rows_p_max * drows);
  const TileList& tl = cached_tiles(s2.stat_tile_lists, rows_p * 4096 + drows / 256, [&](std::vector<int2>& tiles) {
    stat_tile_list(3 * rows_p, drows, 256, tiles);
  });
  launch_gram_gp(gp_tensor_map(s2.gmaps, s2.gp.p, h->Npad, rows_p), &s2.tmD, rows_p, kZStep2, tl.buf.p, tl.count,
                 s2.fold_k.p, s2.nchunk, s2.T.p, drows, (int64_t)3 * rows_p * drows, kZScaleStat, s);
}

static void s2_set_chr(rg_ctx* h, const double* res, const double* scf_sv) {
  Step2State& s2 = step2(h);
  RG_CUDA(cudaSetDevice(h->device));
  const int64_t N = h->N;
  const int C = h->C, P = h->P;
  const bool with_sex = !s2.male.empty();
  const int base = 1 + C + 2 * P + P * C;
  s2.col_male = with_sex ? base : -1;
  s2.dp = (int)round_up(base + (with_sex ? 1 + P : 0), 16);
  s2.fcols = base + (with_sex ? 1 + P : 0);
  const int dp = s2.dp;
  std::vector<double> F((size_t)h->Npad * dp, 0.0), YtX((size_t)P * C, 0.0), male_tot(1 + P, 0.0);
  for (int64_t s = 0; s < N; ++s) {
    double* r = &F[(size_t)s * dp];
    r[0] = h->in_analysis[s] ? 1.0 : 0.0;
    if (with_sex && s2.male[s] && h->in_analysis[s]) {
      r[base] = 1.0; male_tot[0] += 1.0;
      for (int p = 0; p < P; ++p)
        if (h->maskh[(size_t)p * N + s]) { r[base + 1 + p] = 1.0; male_tot[1 + p] += 1.0; }
    }
    for (int c = 0; c < C; ++c) r[1 + c] = s2.Xh[(size_t)c * N + s];
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
  upload(s2.F, F, h->stream);
  upload(s2.YtX, YtX, h->stream);
  RG_CUDA(cudaMemcpyAsync(s2.scf.p, scf_sv, P * 8, cudaMemcpyHostToDevice, h->stream));
  upload(s2.male_tot, male_tot, h->stream);
  s2_build_digits(h, s2, s2.F.p, dp, base + (with_sex ? 1 + P : 0));
  RG_CUDA(cudaStreamSynchronize(h->stream));
  s2.chr_set = true;
  s2.int_set = false;                                                // rg_s2_set_interaction follows, per chromosome
  s2.int_last_bs = 0;
  s2.dz_qt = false;
}

// per-variant non-PAR flags set by rg_s2_set_non_par apply to exactly one block call
static const uint8_t* take_non_par(rg_ctx* h, Step2State& s2, int bs) {
  if (!s2.nonpar_set) return nullptr;
  s2.nonpar_set = false;
  RG_CHECK((int)s2.nonpar.n >= bs, "rg_s2_set_non_par was given fewer flags than the block has variants");
  return s2.nonpar.p;
}

namespace rg {
// A block whose input pointer lies in a staging buffer (rg_s2_stage) waits for that slot's copy, and only for it: the
// copy of the block AFTER it may already be in flight on the copy stream.
static void s2_wait_stage(rg_ctx* h, Step2State& s2, const void* in, cudaStream_t s) {
  if (!in) return;
  for (int k = 0; k < Step2State::kStageSlots; ++k) {
    if (!s2.stage_pending[k] || !s2.stage[k].p) continue;
    const uint8_t* b = s2.stage[k].p;
    if ((const uint8_t*)in >= b && (const uint8_t*)in < b + s2.stage[k].n) {
      RG_CUDA(cudaStreamWaitEvent(s, s2.stage_ev[k], 0));
      s2.stage_pending[k] = false;
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
static void s2_copy_out(rg_ctx* h, Step2State& s2, int bs, const rg_s2_out* out, double* info_out, const double* info_dev, cudaStream_t s) {
  const size_t bp = (size_t)h->bs_max * h->P, nd = s2_out_f64(h), ni = s2_out_i32(h);
  s2.out_hd.alloc(nd + bp);
  s2.out_hi.alloc(ni);
  RG_CUDA(cudaMemcpyAsync(s2.out_hd.p, s2.out_d.p, nd * sizeof(double), cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaMemcpyAsync(s2.out_hi.p, s2.out_i.p, ni * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  if (info_out) RG_CUDA(cudaMemcpyAsync(s2.out_hd.p + nd, info_dev, (size_t)bs * h->P * 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaStreamSynchronize(s));
  const rg_s2_out m = s2_out_at(h, s2.out_hd.p, s2.out_hi.p);
  const size_t vp = (size_t)bs * h->P, v1 = bs;
  auto cp = [](auto* dst, const auto* src, size_t n) { if (dst) memcpy(dst, src, n * sizeof(*src)); };
  cp(out->af, m.af, vp); cp(out->mac, m.mac, vp); cp(out->stat, m.stat, vp); cp(out->beta, m.beta, vp); cp(out->se, m.se, vp);
  cp(out->chisq, m.chisq, vp); cp(out->af_all, m.af_all, v1); cp(out->mac_all, m.mac_all, v1); cp(out->scale_fac, m.scale_fac, v1);
  cp(out->ns, m.ns, vp); cp(out->ns_all, m.ns_all, v1); cp(out->flags, m.flags, v1);
  cp(info_out, s2.out_hd.p + nd, vp);
}

// What every block route does first: the handle, block-size and chromosome-state checks (quantitative-trait routes need
// rg_s2_set_chr, binary-trait routes rg_s2_set_chr_bt), then the device, the staged copies of the block's inputs, the
// sample index map and the packed output buffers.  Returns the handle's Step-2 state.
static Step2State& s2_block_begin(rg_ctx* h, bool bt, int bs, const int32_t* sample_idx, const void* in,
                                  const void* in2 = nullptr) {
  Step2State& s2 = step2(h);
  RG_CHECK(bs > 0 && bs <= h->bs_max, "block size out of range");
  if (bt) RG_CHECK(s2.bt_chr_set, "rg_s2_set_chr_bt has not been called");
  else RG_CHECK(s2.chr_set, "rg_s2_set_chr has not been called");
  s2.dz_qt = false;                                               // set again by a QT route that writes dz
  RG_CUDA(cudaSetDevice(h->device));
  s2_wait_stage(h, s2, in, h->stream);
  s2_wait_stage(h, s2, in2, h->stream);
  ensure_file_idx(h, sample_idx);
  s2.out_d.alloc(s2_out_f64(h));
  s2.out_i.alloc(s2_out_i32(h));
  return s2;
}

// 2-bit rows of the block on the device: a device pointer as it is, host rows through packed_dev
static const uint8_t* s2_rows_in(rg_ctx* h, Step2State& s2, const uint8_t* packed, int64_t row_stride, int bs) {
  if (is_device_pointer(packed)) return packed;
  s2.packed_dev.alloc((size_t)h->bs_max * row_stride);
  copy_to_device(s2.packed_dev.p, packed, (size_t)bs * row_stride, h->stream);
  return s2.packed_dev.p;
}

// 8-bit probability pairs and ploidy / missing bytes of the block on the device, likewise through probs_dev / miss_dev
static void s2_probs_in(rg_ctx* h, Step2State& s2, const uint8_t** probs, const uint8_t** miss, int64_t n_file, int bs) {
  if (is_device_pointer(*probs)) return;
  s2.probs_dev.alloc((size_t)h->bs_max * n_file * 2);
  copy_to_device(s2.probs_dev.p, *probs, (size_t)bs * n_file * 2, h->stream);
  *probs = s2.probs_dev.p;
  if (*miss) {
    s2.miss_dev.alloc((size_t)h->bs_max * n_file);
    copy_to_device(s2.miss_dev.p, *miss, (size_t)bs * n_file, h->stream);
    *miss = s2.miss_dev.p;
  }
}

// the fields S2FinalizeArgs and S2BtFinalizeArgs share, the packed outputs included; consumes the block's non-PAR flags
template <typename Args>
static void s2_finalize_args(rg_ctx* h, Step2State& s2, Args& a, int bs, int dp, double min_mac, const double* sums, int col_male) {
  a.bs = bs; a.C = h->C; a.P = h->P; a.dp = dp;
  a.n_analyzed = h->n_analyzed; a.n_samples = h->N; a.min_mac = min_mac; a.numtol = 1e-6;
  a.sums = sums; a.non_par = take_non_par(h, s2, bs); a.col_male = col_male;
  const rg_s2_out o = s2_out_at(h, s2.out_d.p, s2.out_i.p);
  a.af = o.af; a.mac = o.mac; a.stat = o.stat; a.beta = o.beta; a.se = o.se; a.chisq = o.chisq;
  a.af_all = o.af_all; a.mac_all = o.mac_all; a.scale_fac = o.scale_fac;
  a.ns = o.ns; a.ns_all = o.ns_all; a.flags = o.flags;
}

static void s2_block_bed(rg_ctx* h, const uint8_t* packed, int64_t row_stride, int bs, const int32_t* sample_idx,
                         int ref_first, double min_mac, const rg_s2_out* out) {
  Step2State& s2 = s2_block_begin(h, false, bs, sample_idx, packed);
  cudaStream_t s = h->stream;
  const int rows_p = (int)round_up(bs, kRowPad);
  const int64_t Npad = h->Npad;
  const uint8_t* packed_d = s2_rows_in(h, s2, packed, row_stride, bs);
  s2.gp.alloc((size_t)h->rows_p_max * (Npad / 16));
  if (!s2.tc) s2.part.alloc((size_t)s2.nchunks * h->rows_p_max * 3 * s2.dp);
  s2.sums.alloc((size_t)h->rows_p_max * 3 * s2.dp);
  launch_bed_relayout(packed_d, row_stride, bs, rows_p, h->file_idx_pad.p, h->word_base.p, h->word_keep.p, ref_first, s2.gp.p, Npad, s);
  if (s2.tc) {
    s2_tensor_sums(h, s2, rows_p, s);
    launch_s2_tensor_finish(s2.T.p, s2.drows, (int64_t)3 * rows_p * s2.drows, s2.nchunk, rows_p, s2.dp,
                            s2.ncol, s2.Fscale.p, s2.sums.p, nullptr, nullptr, s);
  } else {
    launch_s2_stats(s2.gp.p, Npad, s2.F.p, s2.dp, s2.chunks.p, s2.nchunks, rows_p, s2.part.p, s2.sums.p, s);
  }
  S2FinalizeArgs a;
  s2_finalize_args(h, s2, a, bs, s2.dp, min_mac, s2.sums.p, s2.col_male);
  a.strict = s2.strict; a.mask_count = s2.maskcount.p; a.YtX = s2.YtX.p; a.XmX = s2.XmX.p; a.scf_sv = s2.scf.p;
  a.male_tot = s2.male_tot.p;
  launch_s2_finalize(a, s);
  h->launches += 4;
  if (s2.int_set) {                                                  // what rg_s2_interaction reads
    s2.dz.alloc((size_t)h->rows_p_max * Npad);
    launch_gp_to_dz(s2.gp.p, rows_p, s2.dz.p, Npad, s);
    h->launches += 1;
    s2.dz_qt = true;
  }
  s2.last_bs = bs;
  s2.sums_rows = rows_p;
  s2_copy_out(h, s2, bs, out, nullptr, nullptr, s);
}

// ---------------------------------------------------------------- binary traits + 8-bit dosages
static void s2_set_chr_bt(rg_ctx* h, const rg_s2_bt_chr* st) {
  Step2State& s2 = step2(h);
  RG_CUDA(cudaSetDevice(h->device));
  const int64_t N = h->N, Npad = h->Npad;
  const int C = h->C, P = h->P;
  const bool with_sex = !s2.male.empty();
  const int base = 1 + P * (3 + C);
  s2.bt_col_male = with_sex ? base : -1;
  const int dp = (int)round_up((int64_t)base + (with_sex ? 1 + P : 0), 16);
  s2.bt_dp = dp;
  s2.bt_ncol = base + (with_sex ? 1 + P : 0);
  std::vector<double> F((size_t)Npad * dp, 0.0), coltot(dp, 0.0), xwy((size_t)P * C, 0.0);
  std::vector<double> w((size_t)P * Npad, 0.0), gs((size_t)P * Npad, 0.0), off((size_t)P * Npad, 0.0),
      xw((size_t)P * C * Npad, 0.0), phat((size_t)P * Npad, 0.0);
  std::vector<int8_t> ym((size_t)P * Npad, 0);
  for (int64_t s = 0; s < N; ++s) {
    double* r = &F[(size_t)s * dp];
    const bool ina = h->in_analysis[s] != 0;
    r[0] = ina ? 1.0 : 0.0;
    if (with_sex && s2.male[s] && ina) {
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
  upload(s2.bt_F, F, h->stream); upload(s2.bt_coltot, coltot, h->stream); upload(s2.bt_xwy, xwy, h->stream);
  upload(s2.bt_w, w, h->stream); upload(s2.bt_gs, gs, h->stream); upload(s2.bt_off, off, h->stream);
  upload(s2.bt_xw, xw, h->stream); upload(s2.bt_ym, ym, h->stream); upload(s2.bt_phat, phat, h->stream);
  s2_build_digits(h, s2, s2.bt_F.p, dp, base + (with_sex ? 1 + P : 0));        // for rg_s2_block_bed_bt
  RG_CUDA(cudaStreamSynchronize(h->stream));
  s2.bt_chr_set = true;
}

// the per-variant buffers of the binary-trait finish (S2BtFinalizeArgs), which rg_s2_firth / rg_s2_spa read back
static void s2_bt_outputs(rg_ctx* h, Step2State& s2, S2BtFinalizeArgs& a) {
  const size_t bp = (size_t)h->bs_max * h->P;
  s2.bt_xtwg.alloc(bp * h->C); s2.bt_mu.alloc(h->bs_max); s2.dose_info.alloc(bp); s2.bt_den.alloc(bp);
  a.with_flip = 1; a.col_tot = s2.bt_coltot.p; a.xwy = s2.bt_xwy.p; a.nz_count = s2.dose_nnz.p; a.n510 = s2.dose_n510.p;
  a.info = s2.dose_info.p; a.xtwg = s2.bt_xtwg.p; a.mu = s2.bt_mu.p; a.den = s2.bt_den.p;
}

static void s2_block_bgen8_bt(rg_ctx* h, const uint8_t* probs, const uint8_t* miss, int64_t n_file, int bs,
                              const int32_t* sample_idx, int ref_first, double min_mac, const rg_s2_out* out,
                              double* info_out) {
  Step2State& s2 = s2_block_begin(h, true, bs, sample_idx, probs, miss);
  cudaStream_t s = h->stream;
  const int dp = s2.bt_dp;
  const int rows_p = (int)round_up(bs, kRowPad);
  const int64_t Npad = h->Npad;
  s2_probs_in(h, s2, &probs, &miss, n_file, bs);
  s2.dz.alloc((size_t)h->rows_p_max * Npad);
  s2.dose_part.alloc((size_t)s2.nchunks * h->rows_p_max * 4 * dp);
  s2.dose_sums.alloc((size_t)h->rows_p_max * 4 * dp);
  s2.dose_nnz.alloc(h->rows_p_max); s2.dose_n510.alloc(h->rows_p_max);
  s2.dose_cnt_part.alloc((size_t)s2.nchunks * h->rows_p_max);
  launch_dosage_relayout(probs, miss, n_file, bs, rows_p, h->file_idx_pad.p, ref_first, s2.dz.p, Npad, s);
  launch_dosage_stats(s2.dz.p, Npad, s2.bt_F.p, dp, s2.chunks.p, s2.nchunks, rows_p, s2.dose_part.p, s2.dose_cnt_part.p, s2.dose_sums.p,
                      s2.dose_nnz.p, s2.dose_n510.p, s, s2.bt_ncol);
  S2BtFinalizeArgs a;
  s2_bt_outputs(h, s2, a);
  s2_finalize_args(h, s2, a, bs, dp, min_mac, s2.dose_sums.p, s2.bt_col_male);
  launch_s2_bt_finalize(a, s);
  h->launches += 5;
  s2.last_bs = bs;
  s2.dose_sums_rows = rows_p; s2.dose_sums_dp = dp;
  s2_copy_out(h, s2, bs, out, info_out, a.info, s);
}

// quantitative traits on 8-bit dosages: same statistics kernel, closed-form finish of s2_kernels.cu
static void s2_block_bgen8_qt(rg_ctx* h, const uint8_t* probs, const uint8_t* miss, int64_t n_file, int bs,
                              const int32_t* sample_idx, int ref_first, double min_mac, const rg_s2_out* out,
                              double* info_out) {
  Step2State& s2 = s2_block_begin(h, false, bs, sample_idx, probs, miss);
  cudaStream_t s = h->stream;
  const int dp = s2.dp;
  const int rows_p = (int)round_up(bs, kRowPad);
  const int64_t Npad = h->Npad;
  s2_probs_in(h, s2, &probs, &miss, n_file, bs);
  s2.dz.alloc((size_t)h->rows_p_max * Npad);
  s2.dose_part.alloc((size_t)s2.nchunks * h->rows_p_max * 4 * dp);
  s2.dose_sums.alloc((size_t)h->rows_p_max * 4 * dp);
  s2.dose_nnz.alloc(h->rows_p_max); s2.dose_n510.alloc(h->rows_p_max);
  s2.sums.alloc((size_t)h->rows_p_max * 3 * dp);
  s2.qt_info_sums.alloc((size_t)h->rows_p_max * dp);
  s2.dose_info.alloc((size_t)h->bs_max * h->P);
  s2.dose_cnt_part.alloc((size_t)s2.nchunks * h->rows_p_max);
  launch_dosage_relayout(probs, miss, n_file, bs, rows_p, h->file_idx_pad.p, ref_first, s2.dz.p, Npad, s);
  launch_dosage_stats(s2.dz.p, Npad, s2.F.p, dp, s2.chunks.p, s2.nchunks, rows_p, s2.dose_part.p, s2.dose_cnt_part.p, s2.dose_sums.p,
                      s2.dose_nnz.p, s2.dose_n510.p, s, s2.fcols);
  launch_dosage_scale(s2.dose_sums.p, rows_p, dp, s2.sums.p, s2.qt_info_sums.p, s);
  S2FinalizeArgs a;
  s2_finalize_args(h, s2, a, bs, dp, min_mac, s2.sums.p, s2.col_male);
  a.strict = s2.strict; a.mask_count = s2.maskcount.p; a.YtX = s2.YtX.p; a.XmX = s2.XmX.p; a.scf_sv = s2.scf.p;
  a.male_tot = s2.male_tot.p; a.nz_count = s2.dose_nnz.p; a.info_sums = s2.qt_info_sums.p; a.info = s2.dose_info.p;
  launch_s2_finalize(a, s);
  h->launches += 6;
  s2.last_bs = bs;
  s2.dz_qt = true;
  s2.sums_rows = rows_p;
  s2.dose_sums_rows = rows_p; s2.dose_sums_dp = dp;
  s2_copy_out(h, s2, bs, out, info_out, a.info, s);
}

// binary traits on 2-bit hard calls (.bed / .pgen): tensor-core sums, then the same finish as the dosage path
static void s2_block_bed_bt(rg_ctx* h, const uint8_t* packed, int64_t row_stride, int bs, const int32_t* sample_idx,
                            int ref_first, double min_mac, const rg_s2_out* out) {
  Step2State& s2 = s2_block_begin(h, true, bs, sample_idx, packed);
  RG_CHECK(s2.tc, "rg_s2_block_bed_bt needs the tensor-core statistics (RG_B200_S2_STATS=f64 disables them)");
  cudaStream_t s = h->stream;
  const int dp = s2.bt_dp;
  const int rows_p = (int)round_up(bs, kRowPad);
  const int64_t Npad = h->Npad;
  const uint8_t* packed_d = s2_rows_in(h, s2, packed, row_stride, bs);
  s2.gp.alloc((size_t)h->rows_p_max * (Npad / 16));
  s2.dz.alloc((size_t)h->rows_p_max * Npad);
  s2.dose_sums.alloc((size_t)h->rows_p_max * 4 * dp);
  s2.dose_nnz.alloc(h->rows_p_max); s2.dose_n510.alloc(h->rows_p_max);
  launch_bed_relayout(packed_d, row_stride, bs, rows_p, h->file_idx_pad.p, h->word_base.p, h->word_keep.p, ref_first, s2.gp.p, Npad, s);
  s2_tensor_sums(h, s2, rows_p, s);
  launch_s2_tensor_finish(s2.T.p, s2.drows, (int64_t)3 * rows_p * s2.drows, s2.nchunk, rows_p, dp, s2.ncol,
                          s2.Fscale.p, s2.dose_sums.p, s2.dose_nnz.p, s2.dose_n510.p, s);
  launch_gp_to_dz(s2.gp.p, rows_p, s2.dz.p, Npad, s);               // what rg_s2_firth / rg_s2_spa read
  S2BtFinalizeArgs a;
  s2_bt_outputs(h, s2, a);
  s2_finalize_args(h, s2, a, bs, dp, min_mac, s2.dose_sums.p, s2.bt_col_male);
  a.unit = 1.0;
  launch_s2_bt_finalize(a, s);
  h->launches += 5;
  s2.last_bs = bs;
  s2.dose_sums_rows = rows_p; s2.dose_sums_dp = dp;
  s2_copy_out(h, s2, bs, out, nullptr, nullptr, s);
}

// Firth and SPA on (variant, trait) selections of the block left resident by a binary-trait route, kSelBatch at a time.
// `batch(s2, o, nb)` fills its kernel's arguments for selections o .. o + nb (uploaded to firth_sel), launches the kernel and
// queues the copies of its results; the batch is complete when this returns to the loop.
constexpr int kSelBatch = 256;
template <typename Batch>
static void s2_selections(rg_ctx* h, const char* call, int n_sel, const int32_t* var_idx, const int32_t* trait_idx,
                          Batch&& batch) {
  Step2State& s2 = step2(h);
  RG_CHECK(s2.bt_chr_set && s2.last_bs > 0, std::string(call) + " needs a resident dosage block");
  RG_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  for (int k = 0; k < n_sel; ++k)
    RG_CHECK(var_idx[k] >= 0 && var_idx[k] < s2.last_bs && trait_idx[k] >= 0 && trait_idx[k] < h->P, "selection out of range");
  s2.firth_gvec.alloc((size_t)kSelBatch * h->Npad); s2.firth_cflag.alloc((size_t)kSelBatch * h->Npad);
  s2.firth_sel.alloc(2 * kSelBatch); s2.firth_status.alloc(kSelBatch); s2.firth_out.alloc(3 * kSelBatch);
  for (int o = 0; o < n_sel; o += kSelBatch) {
    const int nb = std::min(kSelBatch, n_sel - o);
    RG_CUDA(cudaMemcpyAsync(s2.firth_sel.p, var_idx + o, nb * 4, cudaMemcpyHostToDevice, s));
    RG_CUDA(cudaMemcpyAsync(s2.firth_sel.p + kSelBatch, trait_idx + o, nb * 4, cudaMemcpyHostToDevice, s));
    batch(s2, o, nb);
    h->launches += 1;
    RG_CUDA(cudaStreamSynchronize(s));
  }
}

static void s2_firth(rg_ctx* h, int n_sel, const int32_t* var_idx, const int32_t* trait_idx, double* beta, double* se,
                     double* lrt, int32_t* status) {
  s2_selections(h, "rg_s2_firth", n_sel, var_idx, trait_idx, [&](Step2State& s2, int o, int nb) {
    cudaStream_t s = h->stream;
    const rg_s2_out d = s2_out_at(h, s2.out_d.p, s2.out_i.p);
    FirthArgs a;
    a.n_sel = nb; a.C = h->C; a.P = h->P; a.dp = s2.bt_dp; a.niter = 250; a.tol = 2.5e-4; a.maxstep = 5.0;
    a.npad = h->Npad; a.sel_var = s2.firth_sel.p; a.sel_trait = s2.firth_sel.p + kSelBatch;
    a.dz = s2.dz.p; a.F = s2.bt_F.p; a.w = s2.bt_w.p; a.gs = s2.bt_gs.p; a.xw = s2.bt_xw.p; a.off = s2.bt_off.p;
    a.ym = s2.bt_ym.p; a.xtwg = s2.bt_xtwg.p; a.mu = s2.bt_mu.p; a.mac = d.mac; a.flags = d.flags;
    a.gvec = s2.firth_gvec.p; a.cflag = s2.firth_cflag.p;
    a.beta = s2.firth_out.p; a.se = s2.firth_out.p + kSelBatch; a.lrt = s2.firth_out.p + 2 * kSelBatch;
    a.status = s2.firth_status.p;
    launch_s2_firth(a, s);
    RG_CUDA(cudaMemcpyAsync(beta + o, a.beta, nb * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaMemcpyAsync(se + o, a.se, nb * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaMemcpyAsync(lrt + o, a.lrt, nb * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaMemcpyAsync(status + o, a.status, nb * 4, cudaMemcpyDeviceToHost, s));
  });
}

static void s2_spa(rg_ctx* h, int n_sel, const int32_t* var_idx, const int32_t* trait_idx, double* pval, int32_t* status) {
  s2_selections(h, "rg_s2_spa", n_sel, var_idx, trait_idx, [&](Step2State& s2, int o, int nb) {
    cudaStream_t s = h->stream;
    const rg_s2_out d = s2_out_at(h, s2.out_d.p, s2.out_i.p);
    SpaArgs a;
    a.n_sel = nb; a.C = h->C; a.P = h->P; a.dp = s2.bt_dp; a.niter = 1000; a.tol = 1.220703125e-4;   // eps^(1/4), src/Regenie.hpp:330
    a.npad = h->Npad; a.sel_var = s2.firth_sel.p; a.sel_trait = s2.firth_sel.p + kSelBatch;
    a.dz = s2.dz.p; a.F = s2.bt_F.p; a.w = s2.bt_w.p; a.gs = s2.bt_gs.p; a.xw = s2.bt_xw.p; a.phat = s2.bt_phat.p;
    a.ym = s2.bt_ym.p; a.xtwg = s2.bt_xtwg.p; a.mu = s2.bt_mu.p; a.stat = d.stat; a.den = s2.bt_den.p; a.flags = d.flags;
    a.gvec = s2.firth_gvec.p; a.cflag = s2.firth_cflag.p; a.pval = s2.firth_out.p; a.status = s2.firth_status.p;
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
  Step2State& s2 = step2(h);
  RG_CHECK(s2.chr_set, "rg_s2_set_interaction needs a Step-2 handle after rg_s2_set_chr");
  RG_CHECK(st->n_px >= 0 && (st->n_px == 0 || (st->dinv_sqrt && st->px && st->yres)), "HLM state incomplete");
  RG_CUDA(cudaSetDevice(h->device));
  const int64_t N = h->N, Npad = h->Npad;
  const int C = h->C, P = h->P, K = st->n_px, dp = s2.dp;
  const int nr = 2 * C + 2 * P + 3, nh = K > 0 ? P * (2 * K + 5) : 0, nf = nr + nh;
  std::vector<double> E(Npad, 0.0);
  std::vector<uint8_t> pow2(nf, 0);
  for (int k = 0; k < 3; ++k) pow2[2 * C + 2 * P + k] = 1;
  for (int p = 0; p < P && K > 0; ++p)
    for (int k = 0; k < 3; ++k) pow2[nr + p * (2 * K + 5) + 2 * K + 2 + k] = 1;
  for (int64_t s = 0; s < N; ++s) E[s] = h->in_analysis[s] ? st->E[s] : 0.0;
  s2.int_F.alloc((size_t)Npad * nf); s2.int_E.alloc(Npad); s2.int_pow2.alloc(nf);
  RG_CUDA(cudaMemcpyAsync(s2.int_E.p, E.data(), Npad * 8, cudaMemcpyHostToDevice, h->stream));
  RG_CUDA(cudaMemcpyAsync(s2.int_pow2.p, pow2.data(), nf, cudaMemcpyHostToDevice, h->stream));
  // the rows go up in slabs of kSlab samples, so the host holds one slab of them (and of F) at a time
  constexpr int64_t kSlab = kIntSlab;
  std::vector<double> Fh((size_t)kSlab * dp), F((size_t)kSlab * nf);
  for (int64_t s0 = 0; s0 < Npad; s0 += kSlab) {
    const int64_t ns = std::min(kSlab, Npad - s0);
    RG_CUDA(cudaMemcpyAsync(Fh.data(), s2.F.p + (size_t)s0 * dp, (size_t)ns * dp * 8, cudaMemcpyDeviceToHost, h->stream));
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
    RG_CUDA(cudaMemcpyAsync(s2.int_F.p + (size_t)s0 * nf, F.data(), (size_t)ns * nf * 8, cudaMemcpyHostToDevice, h->stream));
  }
  RG_CUDA(cudaStreamSynchronize(h->stream));
  s2.int_K = K; s2.int_nr = nr; s2.int_nf = nf;
  s2.int_last_bs = 0;
  s2.int_set = true;
}

static void s2_interaction(rg_ctx* h, const rg_s2_int_opts* o, int32_t* status, double* coef, double* vcov) {
  Step2State& s2 = step2(h);
  RG_CHECK(s2.int_set, "rg_s2_interaction needs rg_s2_set_interaction");
  // the genotype words of the last block: written by rg_s2_block_bgen8, and by rg_s2_block_bed only when the interaction
  // state was set before the block ran; any other block call or rg_s2_set_chr since then leaves none for this chromosome
  RG_CHECK(s2.dz_qt && s2.last_bs > 0,
           "rg_s2_interaction needs the block of the last rg_s2_block_bed / rg_s2_block_bgen8 call, run after "
           "rg_s2_set_interaction on the current chromosome");
  RG_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  const int bs = s2.last_bs, P = h->P, C = h->C, nf = s2.int_nf;
  const int bs_pad = (int)round_up(bs, 16);
  const rg_s2_out d = s2_out_at(h, s2.out_d.p, s2.out_i.p);
  S2IntArgs a;
  a.bs = bs; a.C = C; a.P = P; a.dp = s2.dp; a.K = s2.int_K; a.nf = nf; a.nr = s2.int_nr; a.nchunks = s2.nchunks;
  a.var_stride = 8 + 2 * C + 2 * P;
  a.force_robust = o->force_robust; a.force_hc4 = o->force_hc4; a.no_robust = o->no_robust;
  a.n_analyzed = h->n_analyzed; a.n_samples = h->N;
  a.rare_mac = o->rare_mac; a.min_mac = o->min_mac; a.numtol = 1e-6;
  a.npad = h->Npad; a.dz = s2.dz.p; a.Fint = s2.int_F.p; a.F = s2.F.p; a.E = s2.int_E.p; a.chunks = s2.chunks.p;
  a.af_all = d.af_all; a.mac = d.mac; a.YtX = s2.YtX.p; a.scf_sv = s2.scf.p; a.mask_count = s2.maskcount.p;
  a.flags = d.flags;
  s2.int_part.alloc((size_t)s2.nchunks * bs_pad * nf);
  s2.int_sums.alloc((size_t)bs * nf);
  s2.int_var.alloc((size_t)bs * a.var_stride);
  s2.int_meat.alloc((size_t)bs * P * s2.nchunks * 4);
  s2.int_out.alloc((size_t)bs * P * 6);
  s2.int_status.alloc((size_t)bs * P);
  s2.int_route.alloc(bs);
  a.route = s2.int_route.p;
  a.sums = s2.int_sums.p; a.var = s2.int_var.p; a.meat_part = s2.int_meat.p; a.status = s2.int_status.p;
  a.coef = s2.int_out.p; a.vcov = s2.int_out.p + (size_t)bs * P * 2;
  launch_s2_interaction(a, s2.int_pow2.p, s2.int_part.p, s);
  h->launches += 5;
  s2.int_last_bs = bs;
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
  RG_CHECK(h, "bad argument");
  Step2State& s2 = step2(h);
  if (male) s2.male.assign(male, male + h->N); else s2.male.clear();
  RG_API_END
}

int rg_s2_set_non_par(rg_handle h, const uint8_t* flags, int32_t n) {
  RG_API_BEGIN
  RG_CHECK(h && flags && n > 0, "bad argument");
  Step2State& s2 = step2(h);
  RG_CUDA(cudaSetDevice(h->device));
  s2.nonpar.alloc(std::max<size_t>((size_t)n, (size_t)h->bs_max));
  RG_CUDA(cudaMemcpyAsync(s2.nonpar.p, flags, n, cudaMemcpyHostToDevice, h->stream));
  RG_CUDA(cudaStreamSynchronize(h->stream));
  s2.nonpar_set = true;
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
  Step2State& s2 = step2(h);
  RG_CHECK(slot >= 0 && slot < Step2State::kStageSlots, "staging slot out of range");
  RG_CUDA(cudaSetDevice(h->device));
  const cudaStream_t cs = s2.copy_stream.ensure();
  if (s2.stage[slot].n < (size_t)bytes) {            // grows only between blocks: nothing reads the old buffer any more
    RG_CUDA(cudaStreamSynchronize(cs));
    RG_CUDA(cudaStreamSynchronize(h->stream));
    s2.stage[slot].alloc((size_t)bytes);
  }
  RG_CUDA(cudaMemcpyAsync(s2.stage[slot].p, host, (size_t)bytes, cudaMemcpyHostToDevice, cs));
  RG_CUDA(cudaEventRecord(s2.stage_ev[slot].ensure(), cs));
  s2.stage_pending[slot] = true;
  *dev = s2.stage[slot].p;
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
