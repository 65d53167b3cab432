// Per-GPU state behind an rg_handle.
#pragma once
#include <map>
#include <memory>

#include "../../include/rg_b200.h"
#include "kernels.cuh"

namespace rg {
// Device copy of a tile list (cached_tiles).
struct TileList {
  DevBuf<int2> buf;
  int count = 0;
};

// Level 0, level 1 and LOCO / PRS: the state only a Step-1 handle has.  Members are declared before the streams that use
// them (the lanes come last), so the destructor drains each stream before freeing what its work reads.
struct Step1State {
  // ---- problem sizes
  int K = 1, R = 0, R1 = 0, loocv = 0;
  int total_blocks = 0, cpp = 0;
  int64_t B = 0;  // total_blocks * R

  // ---- padded fold layout (host copies)
  std::vector<int64_t> fold_sizes, fold_pad_start, fold_pad_len;
  std::vector<int32_t> pad_of;   // [N]   sample -> padded slot

  // ---- device state shared by all blocks
  DevBuf<double> xy;            // [Npad][cpp]  (X | Y), zero padded
  DevBuf<uint8_t> mask;         // [P][Npad]
  DevBuf<uint8_t> is_real;      // [Npad]
  DevBuf<int32_t> tile_fold;    // [Npad/128]
  DevBuf<int4> chunks;          // [nchunks] chunks of the f64 reductions, cut at the fold ends: (t0, len, fold, 0)
  int nchunks = 0;
  DevBuf<int2> fold_chunks;     // [K]
  DevBuf<int2> fold_k;          // [K] (first 128-sample K block, #blocks)
  DevBuf<double> XtX_f, XtY_f, lambda, neff;
  DevBuf<unsigned long long> err_slot;   // first failure of a level-0 / level-1 kernel (rg_l0_status), ~0 = none
  PinnedBuf<unsigned long long> poll_host;
  Stream poll_stream;                    // rg_l0_poll_status: the error word is read here, beside the lanes

  // Gram tile lists: the Z Z^T tiles and the statistics tiles Z [X | Y]-digits, both keyed by rows_p
  std::map<int, TileList> tile_lists, stat_tile_lists;
  // statistics on the tensor cores: digit rows of (X | Y), built once
  bool stats_tc = false;
  int stat_drows = 0;
  DevBuf<uint8_t> xyD;
  DevBuf<double> xy_scale;
  CUtensorMap tmD;

  // ---- Miss rows of the level-0 Gram: sparse sums up to miss_cap missing calls per block, or always the dense tiles
  //      (RG_B200_GRAM=dense)
  bool gram_dense = false;
  int64_t miss_cap = 0;
  // column tiles of the relayout's missing lists (BedMissOut): (first word, words, fold) and each fold's tile range
  int miss_nct = 0;
  std::vector<int4> miss_ctile_host;
  DevBuf<int4> miss_ctile;
  DevBuf<int2> miss_fold_ct;

  // ---- level-0 solver selection (RG_B200_SOLVER = mixed | f64) and its counters
  int solver_mixed = 1;
  float mx_tol = 1e-9f;
  int64_t mx_blocks = 0, mx_fallbacks = 0;

  // ---- level-0 output and where each phenotype's part of it lives
  DevBuf<double> W;                            // [P][Npad x B] column-major
  int last_bs = 0, last_rows_p = 0, last_nC = 0, last_n_aug = 0, last_nmat = 0;
  DevBuf<double*> W_tab;                       // [P] where each phenotype's W lives (local or peer HBM)
  std::vector<double*> W_host_tab;
  std::vector<uint8_t> W_owned;                // phenotypes with local storage (rg_W_set_owned)
  std::vector<IpcMapping> W_peer_mapped;       // other processes' W (rg_W_attach_peer)

  // ---- level 1
  DevBuf<int4> l1_chunks;
  DevBuf<int2> l1_fold_chunks;
  int l1_nchunks = 0;
  DevBuf<double> l1_part, l1_part_y, l1_cm, l1_inv, l1_beta, l1_sums, l1_part_out, l1_tau, l1_pred;
  DevBuf<int32_t> l1_chr_cols;
  DevBuf<double> l1_zrows, l1_hvec, l1_bvec;   // LOOCV: H w_i rows, leverages, coefficients per phenotype
  std::vector<int32_t> best_idx;
  std::vector<double> prs_host;                // [P][N] whole-genome predictions kept by rg_loco for rg_prs
  int l1_nC = 0;
  int l1_nmat = 0, l1_n_aug = 0;               // systems and rows per system of the last fit (rg_debug_fetch "l1_dims")
  int64_t l1_chunk_len = 0;                    // sample chunk length of the last fit's chunk table
  bool l1_done = false;
  std::vector<uint8_t> l1_select;              // phenotypes this handle fits at level 1
  bool l1_bt = false;                          // logistic level 1: l1_hvec holds f_i = (y - p) / (1 - q w)
  DevBuf<double> lg_Ws, lg_eta, lg_wm, lg_res, lg_off, lg_beta, lg_score, lg_q, lg_devp, lg_scal;
  DevBuf<int8_t> lg_ym;
  DevBuf<int2> lg_all_chunks;                  // one entry covering every sample chunk

  // ---- per-lane scratch: consecutive blocks go to different lanes (own stream + buffers) so the
  //      latency-bound solver phases of one block overlap the tensor/HBM phases of the next
  struct Lane {
    DevBuf<uint8_t> packed_dev;   // rows decoded on the device (rg_pgen_decode)
    // host rows: two staging buffers in rotation, filled on the lane's COPY stream, so the PCIe transfer of this lane's
    // next block runs under the kernels of its current one (on the lane's own stream the copy waited for them)
    DevBuf<uint8_t> packed_buf[2];
    Event h2d_done;                   // recorded behind the host-to-device copy of the block's input rows
    Event relayout_done[2];           // behind the kernel that last read packed_buf[k]
    int packed_flip = 0;
    DevBuf<uint8_t> pgen_in;      // rg_pgen_decode: metadata blob + record bytes of the block this lane runs next
    DevBuf<uint32_t> gp;          // [rows_p][Npad/16]
    DevBuf<float> zz;             // [K][2 rows_p][2 rows_p]
    // sparse Miss rows of zz (miss_gram.cu), written by the relayout: missing-call total of the block (> miss_cap =
    // dense tiles), list segments [rows_p][miss_nct] (offset, count), sample lists, the block as sample-major 2-bit rows
    // [Npad][rows_p / 16]
    DevBuf<unsigned long long> miss_total;
    DevBuf<int2> miss_seg;
    DevBuf<int32_t> miss_list;
    DevBuf<uint32_t> gt;
    DevBuf<float> tstat;          // [K][2 rows_p][stat_drows] exact digit sums of the statistics tiles
    DevBuf<int32_t> cnt_part, cnt_fold;
    DevBuf<double> sum_part, sum_fold;
    DevBuf<double> mu, inv_sd, Bv, Af, Qf, gty_f, rhs;
    DevBuf<double> cm;            // [nmat][n_aug][nC]
    DevBuf<double> inv;           // [nmat][nC/64][64x64]  L_kk^-T blocks
    DevBuf<double> gam, gmu, cvec, part, mean_invsd;
    DevBuf<uint8_t> dig;          // radix-254 digit rows of gamma for the tensor-core prediction
    DevBuf<double> wraw;          // [P][R][Npad] raw (unstandardised) predictions of the block, local to this GPU
    DevBuf<double*> wraw_tab;     // [P] per-phenotype base pointers into wraw (same addressing as W_tab with col0 = 0)
    DevBuf<double> dscale;        // [K][Qp] column scales
    std::map<int, CUtensorMap> dmaps; // digit-matrix tensor maps keyed by rows_p
    std::map<int, CUtensorMap> gmaps; // 2-bit row (gp) tensor maps of the Gram, statistics and INT8 prediction tiles,
                                      // keyed by rows_p
    // dense FP64 route for real-valued genotypes (l0_dense.cu)
    DevBuf<uint8_t> dense_in;                 // staged host input (probability / ploidy bytes or FP64 rows)
    DevBuf<double> gd, dpart, dpart_y;        // [bs][Npad] G~; chunk partials of G G^T and G Y
    // mixed-precision ridge solver (chol_mixed.cu): tensor-core factorisation + FP64 refinement, FP64 Cholesky fallback
    std::unique_ptr<MixedSolver> mx;
    DevBuf<double> mx_Af, mx_b, mx_x, mx_r;   // [K][n][n] fold systems; [K][Pp][n] rhs; [K R][Pp][n] solutions / residuals
    DevBuf<unsigned int> mx_fail;            // device flag: refinement did not converge / pivot not positive
    PinnedBuf<unsigned int> mx_fail_host;    // pinned copy, valid once mx_ev has fired
    Event mx_ev;
    bool mx_pending = false;                  // a block went through the mixed path and its flag has not been read yet
    int mx_bs = 0, mx_block_id = 0;           // the block to re-solve in FP64 if the flag is set
    // kernels that produced this lane's last block (rg_debug_fetch "paths"): INT8 (1) or FP64 (0) prediction; the
    // mixed solver's dimension, or 0 when the FP64 Cholesky solved it
    int last_pred_i8 = 0, last_mx_n = 0;
    bool last_gram_dense = false;             // RG_B200_GRAM=dense: the Miss rows ran as dense tiles unconditionally
    Event done;                               // rg_fence
    Stream copy_stream, stream;
  };
  std::vector<std::unique_ptr<Lane>> lanes;
  int next_lane = 0, last_lane = 0;
};

// What rg_s2_set_chr / rg_s2_set_chr_bt build for one trait kind: the chromosome's feature rows F and, unless
// RG_B200_S2_STATS=f64 was set at that call (tc), their digit rows for the tensor-core statistics of 2-bit blocks.
struct S2Chr {
  bool set = false, tc = false;      // set: the kind's chromosome call has run
  int dp = 0, ncol = 0, col_male = -1;   // F [Npad][dp], ncol columns used; chrX: the male indicator's column (-1: none)
  int drows = 0, nchunk = 0;
  int64_t chunk_len = 0;             // samples per tensor-core chunk (the last one may be shorter)
  DevBuf<double> F, Fscale;
  DevBuf<uint8_t> FD;                // [drows][Npad] digit rows of F
  DevBuf<int2> fold_k;               // the tensor-core sample chunks
  CUtensorMap tmD;
};
struct S2QtChr : S2Chr { DevBuf<double> YtX, scf, male_tot; };
struct S2BtChr : S2Chr {
  DevBuf<double> w, gs, xw, off, coltot, xwy, phat;
  DevBuf<int8_t> ym;
  bool firth = false;                // off holds the null-Firth offsets (rg_s2_bt_chr.firth_offset was given)
};
// The block the last block call left in the input, sum and output buffers, for rg_s2_firth / rg_s2_spa /
// rg_s2_interaction and the sums hooks of rg_debug_fetch.  A block call replaces it; a chromosome call of its kind ends it.
struct S2Block {
  enum Kind { none, qt, bt } kind = none;
  int bs = 0, rows_p = 0, dp = 0;
  bool dz = false, dose = false;     // dz / the 4-plane sums hold the block's genotype words / sums
};
// The state only a Step-2 handle has.
struct Step2State {
  int strict = 0;
  std::vector<double> Xh;            // [N x C] host copy
  DevBuf<int4> chunks;               // [nchunks] sample chunks of the f64 reductions: (t0, len, 0, 0)
  int nchunks = 0;
  DevBuf<double> maskcount, XmX;
  DevBuf<uint8_t> ones;
  std::vector<uint8_t> male;         // chrX: male indicator of every sample (empty = none), per-block non-PAR flags
  DevBuf<uint8_t> nonpar;             // allocated for bs_max flags at least; nonpar_n of them were given
  int32_t nonpar_n = 0;
  bool nonpar_set = false;
  S2QtChr qt;
  S2BtChr bt;
  S2Block block;
  int64_t block_serial = 0;          // block calls so far: tells whether a result belongs to the resident block
  struct Input {
    DevBuf<uint8_t> packed_dev, probs_dev, miss_dev;   // host rows / probabilities / ploidy bytes copied to the device
    DevBuf<uint32_t> gp;                            // the padded 2-bit rows and their tensor maps keyed by rows_p
    std::map<int, CUtensorMap> gmaps;
    DevBuf<uint8_t> inflate_comp, inflate_raw;      // rg_bgen_inflate: compressed streams, inflated payloads
    DevBuf<uint64_t> inflate_offs;
    DevBuf<int32_t> inflate_status;
    DevBuf<uint8_t> pgen_in, pgen_rows;             // rg_pgen_decode: records in, 2-bit rows out
    DevBuf<uint32_t> dz;                            // [rows_p][Npad] d | e << 10 | missing << 31
  } in;
  struct Sums {
    // 3-plane sums [rows_p][3][dp] of the quantitative-trait finish, from FP64 chunk partials or the tensor digit sums
    DevBuf<double> part, s3;
    DevBuf<float> T;                 // [chunk][3 rows_p][drows]
    std::map<int, TileList> tiles;   // the tiles Z F-digits, keyed by rows_p * 4096 + drows / 256
    // 4-plane sums [rows_p][4][dp] of dosages or 2-bit binary-trait calls, with their chunk partials and non-zero /
    // hom-alt counts; [rows_p][dp] INFO sums of the quantitative-trait dosage route
    DevBuf<double> part4, s4, nnz, n510, qt_info;
    DevBuf<int2> cnt_part;
  } sums;
  struct Outputs {
    DevBuf<double> d; DevBuf<int32_t> i;          // packed f64 / i32 outputs
    PinnedBuf<double> hd; PinnedBuf<int32_t> hi;  // their pinned mirrors (+ the INFO block)
    DevBuf<double> xtwg, mu, den, info;   // of the binary-trait finish, read back by Firth and SPA; INFO scores
  } out;
  struct Selections {                // rg_s2_firth / rg_s2_spa: (variant, trait) indices of a batch, scratch, results
    DevBuf<int32_t> idx, status;
    DevBuf<double> gvec, out;
    DevBuf<int8_t> cflag;
  } sel;
  struct Gxe {                       // rg_s2_set_interaction / rg_s2_interaction, csrc/s2_interaction.cu
    bool set = false;
    int K = 0, nr = 0, nf = 0, last_bs = 0;   // last_bs: variants of the last rg_s2_interaction since the set call
    DevBuf<double> F, E, part, sums, var, meat, out;
    DevBuf<uint8_t> pow2;
    DevBuf<int8_t> route;
    DevBuf<int32_t> status;
  } gxe;
  struct GxeBt {                     // rg_s2_set_interaction_bt / rg_s2_interaction_bt / _firth, csrc/s2_interaction_bt.cu
    bool set = false;
    int nf = 0;
    int64_t wald_serial = -1;        // block_serial of the block the last rg_s2_interaction_bt ran on
    DevBuf<double> F, E, off, part, sums, var, H, out;
    DevBuf<uint8_t> pow2;
    DevBuf<int8_t> route;
    DevBuf<int32_t> status, sel;
  } gxe_bt;
  // rg_s2_stage: input bytes of the NEXT block travel on a copy stream while the current block computes
  static constexpr int kStageSlots = 4;
  struct Staging {
    DevBuf<uint8_t> buf[kStageSlots];
    Event ev[kStageSlots];
    bool pending[kStageSlots] = {false, false, false, false};
    Stream copy_stream;
  } stage;
};

}  // namespace rg

// Per-GPU state behind an rg_handle: what both kinds of handle use, and the state of its kind.
struct rg_ctx {
  int device = 0;
  int64_t launches = 0;

  // ---- problem sizes and the padded sample layout
  int64_t N = 0, Npad = 0, n_analyzed = 0;
  int C = 0, P = 0, bs_max = 0, rows_p_max = 0;
  std::vector<int32_t> src_of;       // [Npad] padded slot -> sample or -1
  std::vector<uint8_t> in_analysis;  // [N]
  std::vector<uint8_t> maskh;        // [N x P]

  // ---- sample index map of the genotype file (ensure_file_idx)
  std::vector<int32_t> cached_sample_idx;
  bool file_idx_valid = false;
  rg::DevBuf<int32_t> file_idx_pad; // [Npad]
  rg::DevBuf<int32_t> word_base;    // [Npad/16] first file index of a 16-sample word (-1 empty, -2 not contiguous)
  rg::DevBuf<uint32_t> word_keep;   // [Npad/16] 2-bit lane mask of the samples that are read
  rg::DevBuf<unsigned long long> pgen_err;   // first malformed .pgen record: (block + 1) << 32 | variant << 4 | code

  // ---- timing
  bool timing = false;
  std::map<std::string, std::pair<double, int64_t>> timers;
  std::vector<std::tuple<std::string, rg::Event, rg::Event>> pending;   // timing ranges flush_timers has not read

  // ---- exactly one is set: a Step-1 or a Step-2 handle
  std::unique_ptr<rg::Step1State> s1;
  std::unique_ptr<rg::Step2State> s2;
  rg::Stream stream;                 // last: drained and destroyed before anything its work reads is freed
};

namespace rg {
// the state of a Step-1 / Step-2 handle; throws if the handle is of the other kind
inline Step1State& step1(rg_ctx* h) {
  RG_CHECK(h->s1, "handle is not a Step-1 handle");
  return *h->s1;
}
inline Step2State& step2(rg_ctx* h) {
  RG_CHECK(h->s2, "handle is not a Step-2 handle");
  return *h->s2;
}
void ensure_W(rg_ctx* h, Step1State& s1);
// chunk table of the sample-axis reductions: every fold of the padded layout cut into chunks of at most len samples,
// (start, length, fold, 0) in fold order, and fold_chunks[f] = [first, last) chunk of fold f
void fold_chunk_table(const Step1State& s1, int64_t len, std::vector<int4>& chunks, std::vector<int2>& fold_chunks);
// buf = v, allocated to fit and copied on stream s (v stays alive until s has read it)
template <class T>
void upload(DevBuf<T>& buf, const std::vector<T>& v, cudaStream_t s) {
  buf.alloc(v.size());
  RG_CUDA(cudaMemcpyAsync(buf.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, s));
}
// throws unless `device` is an sm_90 GPU
void require_gpu(int device);
// the genotype file's sample index map (file_idx_pad, word_base, word_keep), rebuilt only when sample_idx changes;
// sample_idx is a host or a device array of n_samples entries, or null for the identity
void ensure_file_idx(rg_ctx* h, const int32_t* sample_idx);
void flush_timers(rg_ctx* h);
// read the mixed-solver flags of every lane (re-solving flagged blocks in FP64) and wait for all level-0 work
void sync_lanes(rg_ctx* h);
// throws when a kernel of rg_pgen_decode flagged a malformed record (pgen_decode.cu)
void pgen_check_errors(rg_ctx* h);

// Tensor map of the 2-bit rows gp [rows_p][npad / 16] (the operand of the Gram, statistics and INT8 prediction tiles),
// made once per rows_p: gp is allocated once, for rows_p_max rows, so its address does not change.
inline const CUtensorMap& gp_tensor_map(std::map<int, CUtensorMap>& cache, const uint32_t* gp, int64_t npad, int rows_p) {
  auto it = cache.find(rows_p);
  if (it == cache.end()) {
    CUtensorMap tm;
    make_gp_tensor_map(&tm, gp, npad / 16, rows_p);
    it = cache.emplace(rows_p, tm).first;
  }
  return it->second;
}

// Device copy of a tile list, built by fill and uploaded on first use of each key.
template <class Fill>
const TileList& cached_tiles(std::map<int, TileList>& cache, int key, Fill fill) {
  TileList& e = cache[key];
  if (e.count == 0) {
    std::vector<int2> tiles;
    fill(tiles);
    e.buf.alloc(tiles.size());
    RG_CUDA(cudaMemcpy(e.buf.p, tiles.data(), tiles.size() * sizeof(int2), cudaMemcpyHostToDevice));
    e.count = (int)tiles.size();
  }
  return e;
}
}

// body of every C ABI entry point: an exception becomes return code 1 and the message of rg_last_error
#define RG_API_BEGIN try {
#define RG_API_END                         \
  }                                        \
  catch (const rg::Error& e) {             \
    rg::set_last_error(e.msg);             \
    return 1;                              \
  }                                        \
  catch (const std::exception& e) {        \
    rg::set_last_error(e.what());          \
    return 1;                              \
  }                                        \
  return 0;
