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
  s2.maskcount.alloc(P); s2.XmX.alloc(XmX.size()); s2.qt.scf.alloc(P);
  RG_CUDA(cudaMemcpy(s2.maskcount.p, mc.data(), P * 8, cudaMemcpyHostToDevice));
  RG_CUDA(cudaMemcpy(s2.XmX.p, XmX.data(), XmX.size() * 8, cudaMemcpyHostToDevice));
}

// both chromosome calls first end the kind's state and resident block, then shape F: base columns (+ chrX: 1 + P)
template <class Chr>
static Chr& s2_chr_begin(rg_ctx* h, Step2State& s2, Chr& c, S2Block::Kind kind, int base) {
  if (s2.block.kind == kind) s2.block = S2Block();
  c.set = false;
  const bool with_sex = !s2.male.empty();
  c.col_male = with_sex ? base : -1;
  c.ncol = base + (with_sex ? 1 + h->P : 0);
  c.dp = (int)round_up(c.ncol, 16);
  return c;
}

// tensor-core statistics for 2-bit input: digit rows of the chromosome's feature matrix (exact, see s2_kernels.cu)
static void s2_build_digits(rg_ctx* h, Step2State& s2, S2Chr& c) {
  // read on every call (once per chromosome), like RG_B200_STATS at level 0, so each handle follows the current setting
  const char* e = getenv("RG_B200_S2_STATS");
  c.tc = !(e && std::string(e) == "f64");
  if (!c.tc) {
    c.nchunk = 0; c.chunk_len = 0; c.drows = 0;
    return;
  }
  cudaStream_t s = h->stream;
  c.drows = (int)round_up((int64_t)ceil_div(c.ncol, kStatQ) * 128, 256);
  c.FD.alloc((size_t)c.drows * h->Npad);
  c.Fscale.alloc(c.dp);
  if (!s2.ones.p) {
    s2.ones.alloc(h->Npad);
    RG_CUDA(cudaMemsetAsync(s2.ones.p, 1, h->Npad, s));
  }
  RG_CUDA(cudaMemsetAsync(c.FD.p, 0, (size_t)c.drows * h->Npad, s));
  launch_l0_xy_digits(c.F.p, c.dp, c.ncol, h->Npad, s2.ones.p, c.Fscale.p, c.FD.p, s);
  make_gram_tensor_map(&c.tmD, c.FD.p, h->Npad, c.drows);
  // sample chunks: exact integer sums need 60 * chunk < 2^24; more chunks also fill the SMs
  const int ntile = (3 * h->rows_p_max / 128) * (c.drows / 256);
  int64_t nchunk = std::max<int64_t>(ceil_div(h->Npad, (int64_t)262144), ceil_div((int64_t)296, (int64_t)ntile));
  nchunk = std::max<int64_t>(1, std::min<int64_t>(nchunk, h->Npad / 1024));
  const int64_t len = round_up(ceil_div(h->Npad, nchunk), 128);
  std::vector<int2> fk;
  for (int64_t o = 0; o < h->Npad; o += len)
    fk.push_back(make_int2((int)(o / 128), (int)(std::min<int64_t>(len, h->Npad - o) / 128)));
  c.nchunk = (int)fk.size();
  c.chunk_len = len;
  upload(c.fold_k, fk, s);
}

// 2-bit rows in gp -> S1 / S2 / Sm digit sums in T: the planes [G; G^2; Miss] against the kind's digit rows, INT8 Gram
// kernel -> FP64 sums [rows_p][3 or 4][dp] (4 with the non-zero / hom-alt counts nnz / n510)
static void s2_tensor_sums(rg_ctx* h, Step2State& s2, const S2Chr& c, int rows_p, double* sums, double* nnz, double* n510,
                           cudaStream_t s) {
  const int drows = c.drows;
  s2.sums.T.alloc((size_t)c.nchunk * 3 * h->rows_p_max * drows);
  const TileList& tl = cached_tiles(s2.sums.tiles, rows_p * 4096 + drows / 256, [&](std::vector<int2>& tiles) {
    stat_tile_list(3 * rows_p, drows, 256, tiles);
  });
  launch_gram_gp(gp_tensor_map(s2.in.gmaps, s2.in.gp.p, h->Npad, rows_p), &c.tmD, rows_p, kZStep2, tl.buf.p, tl.count,
                 c.fold_k.p, c.nchunk, s2.sums.T.p, drows, (int64_t)3 * rows_p * drows, kZScaleStat, s);
  launch_s2_tensor_finish(s2.sums.T.p, drows, (int64_t)3 * rows_p * drows, c.nchunk, rows_p, c.dp, c.ncol, c.Fscale.p, sums,
                          nnz, n510, s);
}

static void s2_set_chr(rg_ctx* h, const double* res, const double* scf_sv) {
  Step2State& s2 = step2(h);
  RG_CUDA(cudaSetDevice(h->device));
  const int64_t N = h->N;
  const int C = h->C, P = h->P;
  const bool with_sex = !s2.male.empty();
  const int base = 1 + C + 2 * P + P * C;
  S2QtChr& q = s2_chr_begin(h, s2, s2.qt, S2Block::qt, base);
  const int dp = q.dp;
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
  upload(q.F, F, h->stream);
  upload(q.YtX, YtX, h->stream);
  RG_CUDA(cudaMemcpyAsync(q.scf.p, scf_sv, P * 8, cudaMemcpyHostToDevice, h->stream));
  upload(q.male_tot, male_tot, h->stream);
  s2_build_digits(h, s2, q);
  RG_CUDA(cudaStreamSynchronize(h->stream));
  q.set = true;
  s2.gxe.set = false;                                                // rg_s2_set_interaction follows, per chromosome
  s2.gxe.last_bs = 0;
}

// per-variant non-PAR flags set by rg_s2_set_non_par apply to exactly one block call
static const uint8_t* take_non_par(rg_ctx* h, Step2State& s2, int bs) {
  if (!s2.nonpar_set) return nullptr;
  s2.nonpar_set = false;
  RG_CHECK(s2.nonpar_n >= bs, "rg_s2_set_non_par was given fewer flags than the block has variants");
  return s2.nonpar.p;
}

namespace rg {
// A block whose input pointer lies in a staging buffer (rg_s2_stage) waits for that slot's copy, and only for it: the
// copy of the block AFTER it may already be in flight on the copy stream.
static void s2_wait_stage(rg_ctx* h, Step2State& s2, const void* in, cudaStream_t s) {
  if (!in) return;
  for (int k = 0; k < Step2State::kStageSlots; ++k) {
    if (!s2.stage.pending[k] || !s2.stage.buf[k].p) continue;
    const uint8_t* b = s2.stage.buf[k].p;
    if ((const uint8_t*)in >= b && (const uint8_t*)in < b + s2.stage.buf[k].n) {
      RG_CUDA(cudaStreamWaitEvent(s, s2.stage.ev[k], 0));
      s2.stage.pending[k] = false;
    }
  }
}
}

// Packed per-variant outputs of a block, laid out alike in out.d / out.i and in their pinned host mirrors: f64 slabs
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
  s2.out.hd.alloc(nd + bp);
  s2.out.hi.alloc(ni);
  RG_CUDA(cudaMemcpyAsync(s2.out.hd.p, s2.out.d.p, nd * sizeof(double), cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaMemcpyAsync(s2.out.hi.p, s2.out.i.p, ni * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  if (info_out) RG_CUDA(cudaMemcpyAsync(s2.out.hd.p + nd, info_dev, (size_t)bs * h->P * 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaStreamSynchronize(s));
  const rg_s2_out m = s2_out_at(h, s2.out.hd.p, s2.out.hi.p);
  const size_t vp = (size_t)bs * h->P, v1 = bs;
  auto cp = [](auto* dst, const auto* src, size_t n) { if (dst) memcpy(dst, src, n * sizeof(*src)); };
  cp(out->af, m.af, vp); cp(out->mac, m.mac, vp); cp(out->stat, m.stat, vp); cp(out->beta, m.beta, vp); cp(out->se, m.se, vp);
  cp(out->chisq, m.chisq, vp); cp(out->af_all, m.af_all, v1); cp(out->mac_all, m.mac_all, v1); cp(out->scale_fac, m.scale_fac, v1);
  cp(out->ns, m.ns, vp); cp(out->ns_all, m.ns_all, v1); cp(out->flags, m.flags, v1);
  cp(info_out, s2.out.hd.p + nd, vp);
}

// What every block route does first: the handle, block-size and chromosome-state checks of the route's trait kind, then
// the end of the resident block, the device, the staged copies of the block's inputs, the sample index map and the packed
// output buffers.  Returns the handle's Step-2 state and the kind's chromosome state.
template <class Chr>
static std::pair<Step2State&, Chr&> s2_block_begin(rg_ctx* h, Chr Step2State::*kind, int bs, const int32_t* sample_idx,
                                                   const void* in, const void* in2 = nullptr) {
  Step2State& s2 = step2(h);
  Chr& c = s2.*kind;
  RG_CHECK(bs > 0 && bs <= h->bs_max, "block size out of range");
  RG_CHECK(c.set, std::string(std::is_same<Chr, S2BtChr>::value ? "rg_s2_set_chr_bt" : "rg_s2_set_chr") + " has not been called");
  s2.block = S2Block();
  ++s2.block_serial;
  RG_CUDA(cudaSetDevice(h->device));
  s2_wait_stage(h, s2, in, h->stream);
  s2_wait_stage(h, s2, in2, h->stream);
  ensure_file_idx(h, sample_idx);
  s2.out.d.alloc(s2_out_f64(h));
  s2.out.i.alloc(s2_out_i32(h));
  return {s2, c};
}

// 2-bit rows of the block on the device: a device pointer as it is, host rows through packed_dev
static const uint8_t* s2_rows_in(rg_ctx* h, Step2State& s2, const uint8_t* packed, int64_t row_stride, int bs) {
  if (is_device_pointer(packed)) return packed;
  s2.in.packed_dev.alloc((size_t)h->bs_max * row_stride);
  copy_to_device(s2.in.packed_dev.p, packed, (size_t)bs * row_stride, h->stream);
  return s2.in.packed_dev.p;
}

// the fields S2FinalizeArgs and S2BtFinalizeArgs share, the packed outputs included; consumes the block's non-PAR flags
template <typename Args>
static void s2_finalize_args(rg_ctx* h, Step2State& s2, const S2Chr& c, Args& a, int bs, double min_mac, const double* sums) {
  a.bs = bs; a.C = h->C; a.P = h->P; a.dp = c.dp;
  a.n_analyzed = h->n_analyzed; a.n_samples = h->N; a.min_mac = min_mac; a.numtol = 1e-6;
  a.sums = sums; a.non_par = take_non_par(h, s2, bs); a.col_male = c.col_male;
  const rg_s2_out o = s2_out_at(h, s2.out.d.p, s2.out.i.p);
  a.af = o.af; a.mac = o.mac; a.stat = o.stat; a.beta = o.beta; a.se = o.se; a.chisq = o.chisq;
  a.af_all = o.af_all; a.mac_all = o.mac_all; a.scale_fac = o.scale_fac;
  a.ns = o.ns; a.ns_all = o.ns_all; a.flags = o.flags;
}

static void s2_block_bed(rg_ctx* h, const uint8_t* packed, int64_t row_stride, int bs, const int32_t* sample_idx,
                         int ref_first, double min_mac, const rg_s2_out* out) {
  auto [s2, q] = s2_block_begin(h, &Step2State::qt, bs, sample_idx, packed);
  cudaStream_t s = h->stream;
  const int rows_p = (int)round_up(bs, kRowPad);
  const int64_t Npad = h->Npad;
  const uint8_t* packed_d = s2_rows_in(h, s2, packed, row_stride, bs);
  s2.in.gp.alloc((size_t)h->rows_p_max * (Npad / 16));
  if (!q.tc) s2.sums.part.alloc((size_t)s2.nchunks * h->rows_p_max * 3 * q.dp);
  s2.sums.s3.alloc((size_t)h->rows_p_max * 3 * q.dp);
  launch_bed_relayout(packed_d, row_stride, bs, rows_p, h->file_idx_pad.p, h->word_base.p, h->word_keep.p, ref_first, s2.in.gp.p, Npad, s);
  if (q.tc) {
    s2_tensor_sums(h, s2, q, rows_p, s2.sums.s3.p, nullptr, nullptr, s);
  } else {
    launch_s2_stats(s2.in.gp.p, Npad, q.F.p, q.dp, s2.chunks.p, s2.nchunks, rows_p, s2.sums.part.p, s2.sums.s3.p, s);
  }
  S2FinalizeArgs a;
  s2_finalize_args(h, s2, q, a, bs, min_mac, s2.sums.s3.p);
  a.strict = s2.strict; a.mask_count = s2.maskcount.p; a.YtX = q.YtX.p; a.XmX = s2.XmX.p; a.scf_sv = q.scf.p;
  a.male_tot = q.male_tot.p;
  launch_s2_finalize(a, s);
  h->launches += 4;
  if (s2.gxe.set) {                                                  // what rg_s2_interaction reads
    s2.in.dz.alloc((size_t)h->rows_p_max * Npad);
    launch_gp_to_dz(s2.in.gp.p, rows_p, s2.in.dz.p, Npad, s);
    h->launches += 1;
  }
  s2.block = S2Block{S2Block::qt, bs, rows_p, q.dp, s2.gxe.set, false};
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
  S2BtChr& b = s2_chr_begin(h, s2, s2.bt, S2Block::bt, base);
  const int dp = b.dp;
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
  upload(b.F, F, h->stream); upload(b.coltot, coltot, h->stream); upload(b.xwy, xwy, h->stream);
  upload(b.w, w, h->stream); upload(b.gs, gs, h->stream); upload(b.off, off, h->stream);
  upload(b.xw, xw, h->stream); upload(b.ym, ym, h->stream); upload(b.phat, phat, h->stream);
  s2_build_digits(h, s2, b);                                         // for rg_s2_block_bed_bt
  RG_CUDA(cudaStreamSynchronize(h->stream));
  b.firth = st->firth_offset != nullptr;
  b.set = true;
  s2.gxe_bt.set = false;                                             // rg_s2_set_interaction_bt follows, per chromosome
  s2.gxe_bt.wald_serial = -1;
}

// the per-variant buffers of the binary-trait finish (S2BtFinalizeArgs), which rg_s2_firth / rg_s2_spa read back
static void s2_bt_outputs(rg_ctx* h, Step2State& s2, S2BtFinalizeArgs& a) {
  const size_t bp = (size_t)h->bs_max * h->P;
  s2.out.xtwg.alloc(bp * h->C); s2.out.mu.alloc(h->bs_max); s2.out.info.alloc(bp); s2.out.den.alloc(bp);
  a.with_flip = 1; a.col_tot = s2.bt.coltot.p; a.xwy = s2.bt.xwy.p; a.nz_count = s2.sums.nnz.p; a.n510 = s2.sums.n510.p;
  a.info = s2.out.info.p; a.xtwg = s2.out.xtwg.p; a.mu = s2.out.mu.p; a.den = s2.out.den.p;
}

// 8-bit dosages of the block (host ones through probs_dev / miss_dev) -> its words in dz -> 4-plane sums and non-zero /
// hom-alt counts against the kind's F
static void s2_dosage_sums(rg_ctx* h, Step2State& s2, const S2Chr& c, const uint8_t* probs, const uint8_t* miss,
                           int64_t n_file, int bs, int rows_p, int ref_first, cudaStream_t s) {
  if (!is_device_pointer(probs)) {
    s2.in.probs_dev.alloc((size_t)h->bs_max * n_file * 2);
    copy_to_device(s2.in.probs_dev.p, probs, (size_t)bs * n_file * 2, s);
    probs = s2.in.probs_dev.p;
    if (miss) {
      s2.in.miss_dev.alloc((size_t)h->bs_max * n_file);
      copy_to_device(s2.in.miss_dev.p, miss, (size_t)bs * n_file, s);
      miss = s2.in.miss_dev.p;
    }
  }
  s2.in.dz.alloc((size_t)h->rows_p_max * h->Npad);
  s2.sums.part4.alloc((size_t)s2.nchunks * h->rows_p_max * 4 * c.dp);
  s2.sums.s4.alloc((size_t)h->rows_p_max * 4 * c.dp);
  s2.sums.nnz.alloc(h->rows_p_max); s2.sums.n510.alloc(h->rows_p_max);
  s2.sums.cnt_part.alloc((size_t)s2.nchunks * h->rows_p_max);
  launch_dosage_relayout(probs, miss, n_file, bs, rows_p, h->file_idx_pad.p, ref_first, s2.in.dz.p, h->Npad, s);
  launch_dosage_stats(s2.in.dz.p, h->Npad, c.F.p, c.dp, s2.chunks.p, s2.nchunks, rows_p, s2.sums.part4.p, s2.sums.cnt_part.p, s2.sums.s4.p,
                      s2.sums.nnz.p, s2.sums.n510.p, s, c.ncol);
}

static void s2_block_bgen8_bt(rg_ctx* h, const uint8_t* probs, const uint8_t* miss, int64_t n_file, int bs,
                              const int32_t* sample_idx, int ref_first, double min_mac, const rg_s2_out* out,
                              double* info_out) {
  auto [s2, b] = s2_block_begin(h, &Step2State::bt, bs, sample_idx, probs, miss);
  cudaStream_t s = h->stream;
  const int rows_p = (int)round_up(bs, kRowPad);
  s2_dosage_sums(h, s2, b, probs, miss, n_file, bs, rows_p, ref_first, s);
  S2BtFinalizeArgs a;
  s2_bt_outputs(h, s2, a);
  s2_finalize_args(h, s2, b, a, bs, min_mac, s2.sums.s4.p);
  launch_s2_bt_finalize(a, s);
  h->launches += 5;
  s2.block = S2Block{S2Block::bt, bs, rows_p, b.dp, true, true};
  s2_copy_out(h, s2, bs, out, info_out, a.info, s);
}

// quantitative traits on 8-bit dosages: same statistics kernel, closed-form finish of s2_kernels.cu
static void s2_block_bgen8_qt(rg_ctx* h, const uint8_t* probs, const uint8_t* miss, int64_t n_file, int bs,
                              const int32_t* sample_idx, int ref_first, double min_mac, const rg_s2_out* out,
                              double* info_out) {
  auto [s2, q] = s2_block_begin(h, &Step2State::qt, bs, sample_idx, probs, miss);
  cudaStream_t s = h->stream;
  const int rows_p = (int)round_up(bs, kRowPad);
  s2.sums.s3.alloc((size_t)h->rows_p_max * 3 * q.dp);
  s2.sums.qt_info.alloc((size_t)h->rows_p_max * q.dp);
  s2.out.info.alloc((size_t)h->bs_max * h->P);
  s2_dosage_sums(h, s2, q, probs, miss, n_file, bs, rows_p, ref_first, s);
  launch_dosage_scale(s2.sums.s4.p, rows_p, q.dp, s2.sums.s3.p, s2.sums.qt_info.p, s);
  S2FinalizeArgs a;
  s2_finalize_args(h, s2, q, a, bs, min_mac, s2.sums.s3.p);
  a.strict = s2.strict; a.mask_count = s2.maskcount.p; a.YtX = q.YtX.p; a.XmX = s2.XmX.p; a.scf_sv = q.scf.p;
  a.male_tot = q.male_tot.p; a.nz_count = s2.sums.nnz.p; a.info_sums = s2.sums.qt_info.p; a.info = s2.out.info.p;
  launch_s2_finalize(a, s);
  h->launches += 6;
  s2.block = S2Block{S2Block::qt, bs, rows_p, q.dp, true, true};
  s2_copy_out(h, s2, bs, out, info_out, a.info, s);
}

// binary traits on 2-bit hard calls (.bed / .pgen): tensor-core sums, then the same finish as the dosage path
static void s2_block_bed_bt(rg_ctx* h, const uint8_t* packed, int64_t row_stride, int bs, const int32_t* sample_idx,
                            int ref_first, double min_mac, const rg_s2_out* out) {
  auto [s2, b] = s2_block_begin(h, &Step2State::bt, bs, sample_idx, packed);
  RG_CHECK(b.tc, "rg_s2_block_bed_bt needs the tensor-core statistics (RG_B200_S2_STATS=f64 disables them)");
  cudaStream_t s = h->stream;
  const int rows_p = (int)round_up(bs, kRowPad);
  const int64_t Npad = h->Npad;
  const uint8_t* packed_d = s2_rows_in(h, s2, packed, row_stride, bs);
  s2.in.gp.alloc((size_t)h->rows_p_max * (Npad / 16));
  s2.in.dz.alloc((size_t)h->rows_p_max * Npad);
  s2.sums.s4.alloc((size_t)h->rows_p_max * 4 * b.dp);
  s2.sums.nnz.alloc(h->rows_p_max); s2.sums.n510.alloc(h->rows_p_max);
  launch_bed_relayout(packed_d, row_stride, bs, rows_p, h->file_idx_pad.p, h->word_base.p, h->word_keep.p, ref_first, s2.in.gp.p, Npad, s);
  s2_tensor_sums(h, s2, b, rows_p, s2.sums.s4.p, s2.sums.nnz.p, s2.sums.n510.p, s);
  launch_gp_to_dz(s2.in.gp.p, rows_p, s2.in.dz.p, Npad, s);         // what rg_s2_firth / rg_s2_spa read
  S2BtFinalizeArgs a;
  s2_bt_outputs(h, s2, a);
  s2_finalize_args(h, s2, b, a, bs, min_mac, s2.sums.s4.p);
  a.unit = 1.0;
  launch_s2_bt_finalize(a, s);
  h->launches += 5;
  s2.block = S2Block{S2Block::bt, bs, rows_p, b.dp, true, true};
  s2_copy_out(h, s2, bs, out, nullptr, nullptr, s);
}

// The selection loop of rg_s2_firth, rg_s2_spa and rg_s2_interaction_firth on the resident binary-trait block: batches of
// len (variant, trait) selections, whose indices go up to idx[0, len) and idx[len, 2 len).  `batch(s2, o, nb)` launches
// its kernels for selections o .. o + nb and queues the copies of their results; the batch is complete when this returns
// to the loop.
template <typename Batch>
static void s2_selections(rg_ctx* h, const char* call, int n_sel, const int32_t* var_idx, const int32_t* trait_idx, int len,
                          DevBuf<int32_t>& idx, Batch&& batch) {
  Step2State& s2 = step2(h);
  RG_CHECK(s2.block.kind == S2Block::bt, std::string(call) + " needs a resident binary-trait block");
  RG_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  for (int k = 0; k < n_sel; ++k)
    RG_CHECK(var_idx[k] >= 0 && var_idx[k] < s2.block.bs && trait_idx[k] >= 0 && trait_idx[k] < h->P, "selection out of range");
  idx.alloc(2 * len);
  for (int o = 0; o < n_sel; o += len) {
    const int nb = std::min(len, n_sel - o);
    RG_CUDA(cudaMemcpyAsync(idx.p, var_idx + o, nb * 4, cudaMemcpyHostToDevice, s));
    RG_CUDA(cudaMemcpyAsync(idx.p + len, trait_idx + o, nb * 4, cudaMemcpyHostToDevice, s));
    batch(s2, o, nb);
    RG_CUDA(cudaStreamSynchronize(s));
  }
}

// Firth and SPA: kSelBatch selections at a time.  The arguments both kernels read for a batch of nb, with its scratch and
// result buffers.
constexpr int kSelBatch = 256;
static void s2_sel_args(rg_ctx* h, Step2State& s2, int nb, int niter, double tol, S2SelArgs& a) {
  s2.sel.gvec.alloc((size_t)kSelBatch * h->Npad); s2.sel.cflag.alloc((size_t)kSelBatch * h->Npad);
  s2.sel.status.alloc(kSelBatch); s2.sel.out.alloc(3 * kSelBatch);
  a.n_sel = nb; a.C = h->C; a.P = h->P; a.dp = s2.bt.dp; a.niter = niter; a.tol = tol;
  a.npad = h->Npad; a.sel_var = s2.sel.idx.p; a.sel_trait = s2.sel.idx.p + kSelBatch;
  a.dz = s2.in.dz.p; a.F = s2.bt.F.p; a.w = s2.bt.w.p; a.gs = s2.bt.gs.p; a.xw = s2.bt.xw.p; a.ym = s2.bt.ym.p;
  a.xtwg = s2.out.xtwg.p; a.mu = s2.out.mu.p; a.flags = s2_out_at(h, s2.out.d.p, s2.out.i.p).flags;
  a.gvec = s2.sel.gvec.p; a.cflag = s2.sel.cflag.p; a.status = s2.sel.status.p;
}

static void s2_firth(rg_ctx* h, int n_sel, const int32_t* var_idx, const int32_t* trait_idx, double* beta, double* se,
                     double* lrt, int32_t* status) {
  s2_selections(h, "rg_s2_firth", n_sel, var_idx, trait_idx, kSelBatch, step2(h).sel.idx, [&](Step2State& s2, int o, int nb) {
    cudaStream_t s = h->stream;
    FirthArgs a;
    s2_sel_args(h, s2, nb, 250, 2.5e-4, a);
    a.maxstep = 5.0; a.off = s2.bt.off.p; a.mac = s2_out_at(h, s2.out.d.p, s2.out.i.p).mac;
    a.beta = s2.sel.out.p; a.se = s2.sel.out.p + kSelBatch; a.lrt = s2.sel.out.p + 2 * kSelBatch;
    launch_s2_firth(a, s);
    h->launches += 1;
    RG_CUDA(cudaMemcpyAsync(beta + o, a.beta, nb * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaMemcpyAsync(se + o, a.se, nb * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaMemcpyAsync(lrt + o, a.lrt, nb * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaMemcpyAsync(status + o, a.status, nb * 4, cudaMemcpyDeviceToHost, s));
  });
}

static void s2_spa(rg_ctx* h, int n_sel, const int32_t* var_idx, const int32_t* trait_idx, double* pval, int32_t* status) {
  s2_selections(h, "rg_s2_spa", n_sel, var_idx, trait_idx, kSelBatch, step2(h).sel.idx, [&](Step2State& s2, int o, int nb) {
    cudaStream_t s = h->stream;
    SpaArgs a;
    s2_sel_args(h, s2, nb, 1000, 1.220703125e-4, a);                  // eps^(1/4), src/Regenie.hpp:330
    a.phat = s2.bt.phat.p; a.stat = s2_out_at(h, s2.out.d.p, s2.out.i.p).stat; a.den = s2.out.den.p;
    a.pval = s2.sel.out.p;
    launch_s2_spa(a, s);
    h->launches += 1;
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
  RG_CHECK(s2.qt.set, "rg_s2_set_interaction needs a Step-2 handle after rg_s2_set_chr");
  RG_CHECK(st->n_px >= 0 && (st->n_px == 0 || (st->dinv_sqrt && st->px && st->yres)), "HLM state incomplete");
  RG_CUDA(cudaSetDevice(h->device));
  const int64_t N = h->N, Npad = h->Npad;
  const int C = h->C, P = h->P, K = st->n_px, dp = s2.qt.dp;
  const int nr = 2 * C + 2 * P + 3, nh = K > 0 ? P * (2 * K + 5) : 0, nf = nr + nh;
  std::vector<double> E(Npad, 0.0);
  std::vector<uint8_t> pow2(nf, 0);
  for (int k = 0; k < 3; ++k) pow2[2 * C + 2 * P + k] = 1;
  for (int p = 0; p < P && K > 0; ++p)
    for (int k = 0; k < 3; ++k) pow2[nr + p * (2 * K + 5) + 2 * K + 2 + k] = 1;
  for (int64_t s = 0; s < N; ++s) E[s] = h->in_analysis[s] ? st->E[s] : 0.0;
  s2.gxe.F.alloc((size_t)Npad * nf); s2.gxe.E.alloc(Npad); s2.gxe.pow2.alloc(nf);
  RG_CUDA(cudaMemcpyAsync(s2.gxe.E.p, E.data(), Npad * 8, cudaMemcpyHostToDevice, h->stream));
  RG_CUDA(cudaMemcpyAsync(s2.gxe.pow2.p, pow2.data(), nf, cudaMemcpyHostToDevice, h->stream));
  // the rows go up in slabs of kSlab samples, so the host holds one slab of them (and of F) at a time
  constexpr int64_t kSlab = kIntSlab;
  std::vector<double> Fh((size_t)kSlab * dp), F((size_t)kSlab * nf);
  for (int64_t s0 = 0; s0 < Npad; s0 += kSlab) {
    const int64_t ns = std::min(kSlab, Npad - s0);
    RG_CUDA(cudaMemcpyAsync(Fh.data(), s2.qt.F.p + (size_t)s0 * dp, (size_t)ns * dp * 8, cudaMemcpyDeviceToHost, h->stream));
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
    RG_CUDA(cudaMemcpyAsync(s2.gxe.F.p + (size_t)s0 * nf, F.data(), (size_t)ns * nf * 8, cudaMemcpyHostToDevice, h->stream));
  }
  RG_CUDA(cudaStreamSynchronize(h->stream));
  s2.gxe.K = K; s2.gxe.nr = nr; s2.gxe.nf = nf;
  s2.gxe.last_bs = 0;
  s2.gxe.set = true;
}

static void s2_interaction(rg_ctx* h, const rg_s2_int_opts* o, int32_t* status, double* coef, double* vcov) {
  Step2State& s2 = step2(h);
  RG_CHECK(s2.gxe.set, "rg_s2_interaction needs rg_s2_set_interaction");
  // the genotype words of the last block: written by rg_s2_block_bgen8, and by rg_s2_block_bed only when the interaction
  // state was set before the block ran; any other block call or rg_s2_set_chr since then leaves none for this chromosome
  RG_CHECK(s2.block.kind == S2Block::qt && s2.block.dz,
           "rg_s2_interaction needs the block of the last rg_s2_block_bed / rg_s2_block_bgen8 call, run after "
           "rg_s2_set_interaction on the current chromosome");
  RG_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  const int bs = s2.block.bs, P = h->P, C = h->C, nf = s2.gxe.nf;
  const int bs_pad = (int)round_up(bs, 16);
  const rg_s2_out d = s2_out_at(h, s2.out.d.p, s2.out.i.p);
  S2IntArgs a;
  a.bs = bs; a.C = C; a.P = P; a.dp = s2.qt.dp; a.K = s2.gxe.K; a.nf = nf; a.nr = s2.gxe.nr; a.nchunks = s2.nchunks;
  a.var_stride = 8 + 2 * C + 2 * P;
  a.force_robust = o->force_robust; a.force_hc4 = o->force_hc4; a.no_robust = o->no_robust;
  a.n_analyzed = h->n_analyzed; a.n_samples = h->N;
  a.rare_mac = o->rare_mac; a.min_mac = o->min_mac; a.numtol = 1e-6;
  a.npad = h->Npad; a.dz = s2.in.dz.p; a.Fint = s2.gxe.F.p; a.F = s2.qt.F.p; a.E = s2.gxe.E.p; a.chunks = s2.chunks.p;
  a.af_all = d.af_all; a.mac = d.mac; a.YtX = s2.qt.YtX.p; a.scf_sv = s2.qt.scf.p; a.mask_count = s2.maskcount.p;
  a.flags = d.flags;
  s2.gxe.part.alloc((size_t)s2.nchunks * bs_pad * nf);
  s2.gxe.sums.alloc((size_t)bs * nf);
  s2.gxe.var.alloc((size_t)bs * a.var_stride);
  s2.gxe.meat.alloc((size_t)bs * P * s2.nchunks * 4);
  s2.gxe.out.alloc((size_t)bs * P * 6);
  s2.gxe.status.alloc((size_t)bs * P);
  s2.gxe.route.alloc(bs);
  a.route = s2.gxe.route.p;
  a.sums = s2.gxe.sums.p; a.var = s2.gxe.var.p; a.meat_part = s2.gxe.meat.p; a.status = s2.gxe.status.p;
  a.coef = s2.gxe.out.p; a.vcov = s2.gxe.out.p + (size_t)bs * P * 2;
  launch_s2_interaction(a, s2.gxe.pow2.p, s2.gxe.part.p, s);
  h->launches += 5;
  s2.gxe.last_bs = bs;
  RG_CUDA(cudaMemcpyAsync(status, a.status, (size_t)bs * P * 4, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaMemcpyAsync(coef, a.coef, (size_t)bs * P * 2 * 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaMemcpyAsync(vcov, a.vcov, (size_t)bs * P * 4 * 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaStreamSynchronize(s));
}

// ---------------------------------------------------------------- GxE interaction tests (binary traits)
// Feature rows [Npad][2 C + 2] of the per-variant sums: X_c, E X_c (times g), 1, E^2 (times g^2), zero outside the
// analysis; X is the covariate basis of rg_step2_create, which spans E and E^2 as well.
static void s2_set_interaction_bt(rg_ctx* h, const rg_s2_int_bt_chr* st) {
  Step2State& s2 = step2(h);
  RG_CHECK(s2.bt.set, "rg_s2_set_interaction_bt needs a Step-2 handle after rg_s2_set_chr_bt");
  RG_CUDA(cudaSetDevice(h->device));
  const int64_t N = h->N, Npad = h->Npad;
  const int C = h->C, P = h->P, nf = 2 * C + 2;
  auto& g = s2.gxe_bt;
  std::vector<double> E(Npad, 0.0), off((size_t)P * Npad, 0.0);
  std::vector<uint8_t> pow2(nf, 0);
  pow2[2 * C] = pow2[2 * C + 1] = 1;
  for (int64_t s = 0; s < N; ++s) E[s] = h->in_analysis[s] ? st->E[s] : 0.0;
  for (int p = 0; p < P; ++p)
    for (int64_t s = 0; s < N; ++s) off[(size_t)p * Npad + s] = st->offset[(size_t)p * N + s];
  upload(g.E, E, h->stream); upload(g.off, off, h->stream); upload(g.pow2, pow2, h->stream);
  g.F.alloc((size_t)Npad * nf);
  std::vector<double> F((size_t)kIntSlab * nf);
  for (int64_t s0 = 0; s0 < Npad; s0 += kIntSlab) {
    const int64_t ns = std::min(kIntSlab, Npad - s0);
    RG_CUDA(cudaStreamSynchronize(h->stream));                       // the previous slab's upload has finished
    std::fill(F.begin(), F.end(), 0.0);
    for (int64_t s = s0; s < std::min(s0 + ns, N); ++s) {
      if (!h->in_analysis[s]) continue;
      const double e = E[s];
      double* r = &F[(size_t)(s - s0) * nf];
      for (int c = 0; c < C; ++c) { r[c] = s2.Xh[(size_t)c * N + s]; r[C + c] = e * r[c]; }
      r[2 * C] = 1.0; r[2 * C + 1] = e * e;
    }
    RG_CUDA(cudaMemcpyAsync(g.F.p + (size_t)s0 * nf, F.data(), (size_t)ns * nf * 8, cudaMemcpyHostToDevice, h->stream));
  }
  RG_CUDA(cudaStreamSynchronize(h->stream));
  g.nf = nf;
  g.wald_serial = -1;
  g.set = true;
}

// the arguments both binary-trait interaction calls share
static S2IntBtArgs s2_int_bt_args(rg_ctx* h, Step2State& s2) {
  const rg_s2_out d = s2_out_at(h, s2.out.d.p, s2.out.i.p);
  auto& g = s2.gxe_bt;
  S2IntBtArgs a{};
  a.bs = s2.block.bs; a.C = h->C; a.P = h->P; a.nf = g.nf; a.nchunks = s2.nchunks; a.var_stride = 3 + 2 * h->C;
  a.n_analyzed = h->n_analyzed; a.numtol = 1e-6; a.npad = h->Npad;
  a.dz = s2.in.dz.p; a.Fint = g.F.p; a.E = g.E.p; a.ym = s2.bt.ym.p; a.chunks = s2.chunks.p;
  a.af_all = d.af_all; a.mu = s2.out.mu.p; a.mac = d.mac; a.flags = d.flags;
  g.var.alloc((size_t)h->bs_max * a.var_stride);
  g.H.alloc((size_t)kIntBtBatch * 2 * h->Npad);
  a.route = g.route.p; a.sums = g.sums.p; a.var = g.var.p; a.H = g.H.p;
  return a;
}

static void s2_interaction_bt(rg_ctx* h, const rg_s2_int_opts* o, int32_t* status, double* coef, double* vcov) {
  Step2State& s2 = step2(h);
  auto& g = s2.gxe_bt;
  RG_CHECK(g.set, "rg_s2_interaction_bt needs rg_s2_set_interaction_bt");
  RG_CHECK(s2.block.kind == S2Block::bt && s2.block.dz,
           "rg_s2_interaction_bt needs the block of the last rg_s2_block_bed_bt / rg_s2_block_bgen8_bt call on the "
           "current chromosome");
  RG_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  const int bs = s2.block.bs, P = h->P;
  g.route.alloc(h->bs_max); g.sums.alloc((size_t)h->bs_max * g.nf);
  g.part.alloc((size_t)s2.nchunks * round_up(h->bs_max, 16) * g.nf);
  g.out.alloc((size_t)h->bs_max * P * 6); g.status.alloc((size_t)h->bs_max * P);
  S2IntBtArgs a = s2_int_bt_args(h, s2);
  a.off = g.off.p;
  a.rare_mac = o->rare_mac; a.min_mac = o->min_mac; a.force_robust = o->force_robust; a.no_robust = o->no_robust;
  a.status = g.status.p; a.coef = g.out.p; a.vcov = g.out.p + (size_t)bs * P * 2;
  launch_s2_int_bt_prep(a, g.pow2.p, g.part.p, s);
  h->launches += 4;
  for (int v0 = 0; v0 < bs; v0 += kIntBtBatch) {
    a.v0 = v0; a.nb = std::min(kIntBtBatch, bs - v0);
    launch_s2_int_bt_wald(a, s);
    h->launches += 2;
  }
  RG_CUDA(cudaMemcpyAsync(status, a.status, (size_t)bs * P * 4, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaMemcpyAsync(coef, a.coef, (size_t)bs * P * 2 * 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaMemcpyAsync(vcov, a.vcov, (size_t)bs * P * 4 * 8, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaStreamSynchronize(s));
  g.wald_serial = s2.block_serial;
}

static void s2_interaction_firth(rg_ctx* h, int n_sel, const int32_t* var_idx, const int32_t* trait_idx, double* coef,
                                 double* se, double* lrt, int32_t* status) {
  Step2State& s2 = step2(h);
  auto& g = s2.gxe_bt;
  RG_CHECK(s2.block.kind == S2Block::bt && g.set && g.wald_serial == s2.block_serial,
           "rg_s2_interaction_firth needs rg_s2_interaction_bt on the resident binary-trait block");
  RG_CHECK(s2.bt.firth, "rg_s2_interaction_firth needs the null-Firth offsets (rg_s2_bt_chr.firth_offset)");
  s2_selections(h, "rg_s2_interaction_firth", n_sel, var_idx, trait_idx, kIntBtBatch, g.sel, [&](Step2State&, int o, int nb) {
    cudaStream_t s = h->stream;
    S2IntBtArgs a = s2_int_bt_args(h, s2);
    a.off = s2.bt.off.p; a.niter = 250; a.tol = 2.5e-4; a.maxstep = 5.0;    // niter_max_firth, numtol_firth, maxstep
    g.out.alloc(7 * kIntBtBatch); g.status.alloc(kIntBtBatch);
    a.sel_var = g.sel.p; a.sel_trait = g.sel.p + kIntBtBatch; a.nb = nb;
    a.f_coef = g.out.p; a.f_se = g.out.p + 2 * kIntBtBatch; a.f_lrt = g.out.p + 4 * kIntBtBatch; a.f_status = g.status.p;
    launch_s2_int_bt_firth(a, s);
    h->launches += 2;
    RG_CUDA(cudaMemcpyAsync(coef + 2 * o, a.f_coef, nb * 2 * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaMemcpyAsync(se + 2 * o, a.f_se, nb * 2 * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaMemcpyAsync(lrt + 3 * o, a.f_lrt, nb * 3 * 8, cudaMemcpyDeviceToHost, s));
    RG_CUDA(cudaMemcpyAsync(status + o, a.f_status, nb * 4, cudaMemcpyDeviceToHost, s));
  });
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

int rg_s2_set_interaction_bt(rg_handle h, const rg_s2_int_bt_chr* st) {
  RG_API_BEGIN
  RG_CHECK(h && st && st->E && st->offset, "null argument");
  s2_set_interaction_bt(h, st);
  RG_API_END
}

int rg_s2_interaction_bt(rg_handle h, const rg_s2_int_opts* opts, int32_t* status, double* coef, double* vcov) {
  RG_API_BEGIN
  RG_CHECK(h && opts && status && coef && vcov, "null argument");
  s2_interaction_bt(h, opts, status, coef, vcov);
  RG_CUDA(cudaGetLastError());
  RG_API_END
}

int rg_s2_interaction_firth(rg_handle h, int32_t n_sel, const int32_t* variant_idx, const int32_t* trait_idx, double* coef,
                            double* se, double* lrt, int32_t* status) {
  RG_API_BEGIN
  RG_CHECK(h && (n_sel == 0 || (variant_idx && trait_idx && coef && se && lrt && status)), "null argument");
  RG_CHECK(n_sel >= 0, "n_sel < 0");
  if (n_sel > 0) s2_interaction_firth(h, n_sel, variant_idx, trait_idx, coef, se, lrt, status);
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
  s2.nonpar_n = n;
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
  const cudaStream_t cs = s2.stage.copy_stream.ensure();
  if (s2.stage.buf[slot].n < (size_t)bytes) {            // grows only between blocks: nothing reads the old buffer any more
    RG_CUDA(cudaStreamSynchronize(cs));
    RG_CUDA(cudaStreamSynchronize(h->stream));
    s2.stage.buf[slot].alloc((size_t)bytes);
  }
  RG_CUDA(cudaMemcpyAsync(s2.stage.buf[slot].p, host, (size_t)bytes, cudaMemcpyHostToDevice, cs));
  RG_CUDA(cudaEventRecord(s2.stage.ev[slot].ensure(), cs));
  s2.stage.pending[slot] = true;
  *dev = s2.stage.buf[slot].p;
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
