// Per-GPU state behind an rg_handle.
#pragma once
#include <map>
#include <memory>

#include "../../include/rg_b200.h"
#include "kernels.cuh"

struct rg_ctx;
namespace rg { void ensure_W(::rg_ctx* h); }

struct rg_ctx {
  int kind = 0;  // 1 = step 1, 2 = step 2
  int device = 0;
  cudaStream_t stream = nullptr;
  int64_t launches = 0;

  // ---- problem sizes
  int64_t N = 0, Npad = 0, n_analyzed = 0;
  int C = 0, P = 0, K = 1, R = 0, R1 = 0, loocv = 0;
  int bs_max = 0, rows_p_max = 0, total_blocks = 0, cpp = 0;
  int64_t B = 0;  // total_blocks * R

  // ---- padded fold layout (host copies)
  std::vector<int64_t> fold_sizes, fold_pad_start, fold_pad_len;
  std::vector<int32_t> pad_of;   // [N]   sample -> padded slot
  std::vector<int32_t> src_of;   // [Npad] padded slot -> sample or -1
  std::vector<uint8_t> in_analysis;
  std::vector<int32_t> cached_sample_idx;
  bool file_idx_valid = false;
  int nchunks = 0;

  // ---- device state shared by all blocks
  rg::DevBuf<double> xy;            // [Npad][cpp]  (X | Y), zero padded
  rg::DevBuf<uint8_t> mask;         // [P][Npad]
  rg::DevBuf<uint8_t> is_real;      // [Npad]
  rg::DevBuf<int32_t> tile_fold;    // [Npad/128]
  rg::DevBuf<int4> chunks;          // [nchunks] (t0, len, fold, 0)
  rg::DevBuf<int2> fold_chunks;     // [K]
  rg::DevBuf<int2> fold_k;          // [K] (first 128-sample K block, #blocks)
  rg::DevBuf<double> XtX_f, XtY_f, lambda, neff;
  rg::DevBuf<int32_t> file_idx_pad; // [Npad]
  rg::DevBuf<int32_t> word_base;    // [Npad/16] first file index of a 16-sample word (-1 empty, -2 not contiguous)
  rg::DevBuf<uint32_t> word_keep;   // [Npad/16] 2-bit lane mask of the samples that are read
  rg::DevBuf<unsigned long long> err_slot;
  cudaStream_t poll_stream = nullptr;              // rg_l0_poll_status: the error word is read here, beside the lanes
  unsigned long long* poll_host = nullptr;         // pinned

  // ---- per-lane scratch: consecutive blocks go to different lanes (own stream + buffers) so the
  //      latency-bound solver phases of one block overlap the tensor/HBM phases of the next
  struct Lane {
    cudaStream_t stream = nullptr;
    cudaEvent_t done = nullptr;
    cudaEvent_t h2d_done = nullptr;   // recorded behind the host-to-device copy of the block's input rows
    bool h2d_recorded = false;
    rg::DevBuf<uint8_t> packed_dev;   // rows decoded on the device (rg_pgen_decode)
    // host rows: two staging buffers in rotation, filled on the lane's COPY stream, so the PCIe transfer of this lane's
    // next block runs under the kernels of its current one (on the lane's own stream the copy waited for them)
    rg::DevBuf<uint8_t> packed_buf[2];
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t relayout_done[2] = {nullptr, nullptr};   // behind the kernel that last read packed_buf[k]
    bool relayout_recorded[2] = {false, false};
    int packed_flip = 0;
    rg::DevBuf<uint8_t> pgen_in;      // rg_pgen_decode: metadata blob + record bytes of the block this lane runs next
    rg::DevBuf<uint32_t> gp;          // [rows_p][Npad/16]
    rg::DevBuf<uint8_t> z;            // [2 rows_p][Npad] int8
    rg::DevBuf<float> zz;             // [K][2 rows_p][2 rows_p]
    // sparse Miss rows of zz (miss_gram.cu): missing-call total of the block (> miss_cap = dense tiles), list segments
    // [K][rows_p] (offset, count), sample lists, the block as sample-major 2-bit rows [Npad][rows_p / 16]
    rg::DevBuf<unsigned long long> miss_total;
    rg::DevBuf<int2> miss_seg;
    rg::DevBuf<int32_t> miss_list;
    rg::DevBuf<uint32_t> gt;
    rg::DevBuf<float> tstat;          // [K][2 rows_p][stat_drows] exact digit sums of the statistics tiles
    rg::DevBuf<int32_t> cnt_part, cnt_fold;
    rg::DevBuf<double> sum_part, sum_fold;
    rg::DevBuf<double> mu, inv_sd, Bv, Af, Qf, gty_f, rhs;
    rg::DevBuf<double> cm;            // [nmat][n_aug][nC]
    rg::DevBuf<double> inv;           // [nmat][nC/64][64x64]  L_kk^-T blocks
    rg::DevBuf<double> gam, gmu, cvec, part, mean_invsd;
    std::map<int, CUtensorMap> tmaps; // keyed by rows_p (z base differs per lane)
    rg::DevBuf<uint8_t> dig;          // radix-254 digit rows of gamma for the tensor-core prediction
    rg::DevBuf<double> wraw;          // [P][R][Npad] raw (unstandardised) predictions of the block, local to this GPU
    rg::DevBuf<double*> wraw_tab;     // [P] per-phenotype base pointers into wraw (same addressing as W_tab with col0 = 0)
    rg::DevBuf<double> dscale;        // [K][Qp] column scales
    std::map<int, CUtensorMap> dmaps; // digit-matrix tensor maps keyed by rows_p
    std::map<int, CUtensorMap> gmaps; // 2-bit row (gp) tensor maps of the INT8 prediction, keyed by rows_p
    // dense FP64 route for real-valued genotypes (l0_dense.cu)
    rg::DevBuf<uint8_t> dense_in;                 // staged host input (probability / ploidy bytes or FP64 rows)
    rg::DevBuf<double> gd, dpart, dpart_y;        // [bs][Npad] G~; chunk partials of G G^T and G Y
    // mixed-precision ridge solver (chol_mixed.cu): tensor-core factorisation + FP64 refinement, FP64 Cholesky fallback
    std::unique_ptr<rg::MixedSolver> mx;
    rg::DevBuf<double> mx_Af, mx_b, mx_x, mx_r;   // [K][n][n] fold systems; [K][Pp][n] rhs; [K R][Pp][n] solutions / residuals
    rg::DevBuf<unsigned int> mx_fail;            // device flag: refinement did not converge / pivot not positive
    unsigned int* mx_fail_host = nullptr;         // pinned copy, valid once mx_ev has fired
    cudaEvent_t mx_ev = nullptr;
    bool mx_pending = false;                      // a block went through the mixed path and its flag has not been read yet
    int mx_bs = 0, mx_block_id = 0;               // the block to re-solve in FP64 if the flag is set
    // kernels that produced this lane's last block (rg_debug_fetch "paths"): INT8 (1) or FP64 (0) prediction; the
    // mixed solver's dimension, or 0 when the FP64 Cholesky solved it
    int last_pred_i8 = 0, last_mx_n = 0;
    bool last_gram_dense = false;                 // RG_B200_GRAM=dense: the Miss rows ran as dense tiles unconditionally
  };
  std::vector<std::unique_ptr<Lane>> lanes;
  int next_lane = 0, last_lane = 0;
  rg::DevBuf<uint8_t> packed_dev;    // step 2 (single lane)
  rg::DevBuf<uint32_t> gp;           // step 2
  // Gram tile lists on the device, keyed by rows_p: the Z Z^T tiles, and the statistics tiles Z [X | Y]-digits
  struct TileList {
    rg::DevBuf<int2> buf;
    int count = 0;
  };
  std::map<int, TileList> tile_lists, stat_tile_lists;
  // statistics on the tensor cores: digit rows of (X | Y), built once
  bool stats_tc = false;
  int stat_drows = 0;
  rg::DevBuf<uint8_t> xyD;
  rg::DevBuf<double> xy_scale;
  CUtensorMap tmD;

  // ---- level-0 output
  rg::DevBuf<double> W;             // [P][Npad x B] column-major
  int last_bs = 0, last_rows_p = 0, last_nC = 0, last_n_aug = 0, last_nmat = 0;

  // ---- level 1
  rg::DevBuf<int4> l1_chunks;
  rg::DevBuf<int2> l1_fold_chunks;
  int l1_nchunks = 0;
  rg::DevBuf<double> l1_part, l1_part_y, l1_cm, l1_inv, l1_beta, l1_sums, l1_part_out, l1_tau, l1_pred;
  rg::DevBuf<int32_t> l1_chr_cols;
  rg::DevBuf<double> l1_zrows, l1_hvec, l1_bvec;   // LOOCV: H w_i rows, leverages, coefficients per phenotype
  std::vector<int32_t> best_idx;
  std::vector<double> prs_host;                      // [P][N] whole-genome predictions kept by rg_loco for rg_prs
  int l1_nC = 0;
  int l1_nmat = 0, l1_n_aug = 0;                     // systems and rows per system of the last fit (rg_debug_fetch "l1_dims")
  int64_t l1_chunk_len = 0;                          // sample chunk length of the last fit's chunk table
  bool l1_done = false;
  rg::DevBuf<double*> W_tab;                         // [P] where each phenotype's W lives (local or peer HBM)
  std::vector<double*> W_host_tab;
  std::vector<uint8_t> W_owned;                      // phenotypes with local storage (rg_W_set_owned)
  std::vector<void*> W_peer_mapped;                  // cudaIpcOpenMemHandle results to close
  std::vector<uint8_t> l1_select;                    // phenotypes this handle fits at level 1
  bool l1_bt = false;                                // logistic level 1: l1_hvec holds f_i = (y - p) / (1 - q w)
  rg::DevBuf<double> lg_Ws, lg_eta, lg_p, lg_wm, lg_res, lg_off, lg_beta, lg_score, lg_q, lg_devp, lg_scal;
  rg::DevBuf<int8_t> lg_ym;
  rg::DevBuf<int2> lg_all_chunks;                    // one entry covering every sample chunk

  // ---- step 2
  int strict = 0, dp = 0;
  std::vector<double> Xh;            // [N x C] host copy
  std::vector<uint8_t> maskh;        // [N x P]
  rg::DevBuf<double> F, s2_part, s2_sums, s2_maskcount, s2_YtX, s2_XmX, s2_scf;
  rg::DevBuf<double> s2_out_d;       // packed f64 outputs
  rg::DevBuf<int32_t> s2_out_i;      // packed i32 outputs
  double* s2_hd = nullptr;           // pinned mirrors of the two output buffers (+ the INFO block)
  int32_t* s2_hi = nullptr;
  size_t s2_host_cap = 0;
  // quantitative-trait statistics on the tensor cores (bed / pgen input)
  bool s2_tc = false;
  int s2_drows = 0, s2_nchunk = 0, s2_ncol = 0;
  int64_t s2_chunk_len = 0;                   // samples per tensor-core chunk (the last one may be shorter)
  rg::DevBuf<uint8_t> s2_z3, s2_FD;           // [3 rows_p][Npad] planes; digit rows of F
  rg::DevBuf<double> s2_Fscale;
  rg::DevBuf<float> s2_T;                     // [chunk][3 rows_p][drows]
  rg::DevBuf<int2> s2_fold_k;
  std::map<int, std::unique_ptr<rg::DevBuf<int2>>> s2_tile_lists;
  rg::DevBuf<uint8_t> s2_ones;
  CUtensorMap s2_tmD;
  std::map<int, CUtensorMap> s2_tmZ;          // keyed by rows_p
  std::map<int, int> s2_ntiles;
  // chrX: male indicator of every sample (empty = none), F column of it, per-block non-PAR flags
  std::vector<uint8_t> s2_male;
  int s2_col_male = -1, bt_col_male = -1;
  rg::DevBuf<uint8_t> s2_nonpar;
  bool s2_nonpar_set = false;
  rg::DevBuf<double> s2_male_tot;
  // binary traits / dosages
  int bt_mode = 0, bt_dp = 0, bt_ncol = 0;   // bt_ncol: used feature columns of the bt_dp padded ones
  int s2_fcols = 0;                           // the same for the quantitative-trait feature rows (dp)
  bool s2_chr_set = false, bt_chr_set = false;   // rg_s2_set_chr / rg_s2_set_chr_bt has run
  int s2_last_bs = 0;                // variants resident in dz (for rg_s2_firth)
  // shape of the sums the last block left (rg_debug_fetch "s2_sums" / "bt_sums"): padded rows, and the row width of bt_sums
  int s2_sums_rows = 0, bt_sums_rows = 0, bt_sums_dp = 0;
  // rg_s2_stage: input bytes of the NEXT block travel on a copy stream while the current block computes
  static constexpr int kStageSlots = 4;
  rg::DevBuf<uint8_t> s2_stage[kStageSlots];
  cudaStream_t s2_copy_stream = nullptr;
  cudaEvent_t s2_stage_ev[kStageSlots] = {nullptr, nullptr, nullptr, nullptr};
  bool s2_stage_pending[kStageSlots] = {false, false, false, false};
  rg::DevBuf<uint8_t> probs_dev, miss_dev;
  rg::DevBuf<uint8_t> inflate_comp, inflate_raw;      // rg_bgen_inflate: compressed streams, inflated payloads
  rg::DevBuf<uint64_t> inflate_offs;
  rg::DevBuf<int32_t> inflate_status;
  rg::DevBuf<uint8_t> pgen_in, pgen_rows;             // rg_pgen_decode on a Step-2 handle: records in, 2-bit rows out
  rg::DevBuf<unsigned long long> pgen_err;            // first malformed record: (block + 1) << 32 | variant << 4 | code
  rg::DevBuf<uint32_t> dz;           // [rows_p][Npad] d | e << 10 | missing << 31
  rg::DevBuf<double> bt_F, bt_w, bt_gs, bt_xw, bt_off, bt_coltot, bt_xwy, bt_part, bt_sums, bt_nnz, bt_n510;
  rg::DevBuf<double> bt_xtwg, bt_mu, bt_info, firth_gvec, firth_out, bt_den, bt_phat;
  rg::DevBuf<int8_t> bt_ym, firth_cflag;
  rg::DevBuf<int2> bt_cnt_part;      // [chunk][rows_p] non-zero / hom-alt counts of the dosage statistics kernel
  rg::DevBuf<int32_t> firth_sel, firth_status;

  // ---- Miss rows of the level-0 Gram: sparse sums up to miss_cap missing calls per block, or always the dense tiles
  //      (RG_B200_GRAM=dense)
  bool gram_dense = false;
  int64_t miss_cap = 0;

  // ---- level-0 solver selection (RG_B200_SOLVER = mixed | f64) and its counters
  int solver_mixed = 1;
  float mx_tol = 1e-9f;
  int64_t mx_blocks = 0, mx_fallbacks = 0;

  // ---- timing
  bool timing = false;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  std::map<std::string, std::pair<double, int64_t>> timers;
  std::vector<std::tuple<std::string, cudaEvent_t, cudaEvent_t>> pending;
};

namespace rg {
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
