// Kernel launchers and argument bundles shared between the .cu translation units.
#pragma once
#include "common.cuh"

namespace rg {

constexpr int kMaxFolds = 16;
constexpr int kMaxCov = 64;
constexpr int kMaxRidge = 8;
constexpr int kMaxPhenoTile = 8;
constexpr int kLimbs = 9;          // radix-30 digits per coefficient (44 bits)
constexpr int kLimbsI8 = 5;        // radix-254 int8 digits per coefficient of the INT8 prediction kernel (40 bits)
constexpr int kLimbQI8 = 50;       // outputs per INT8 prediction pass (5 x 50 = 250 <= 256 digit rows)   // phenotypes per register pass of the LOOCV prediction kernel

// ---- s2_kernels.cu: out[e] = sum_c part[c * per + e] over the nchunks partial vectors, added in chunk order, so the
// result does not depend on the launch shape (Step-2 statistics, level-1 CV sums and deviances)
void launch_partial_sum(const double* part, int nchunks, int64_t per, double* out, cudaStream_t s);

// ---- bed_kernels.cu
// bit 2k set where the 2-bit code k of w is 3 (missing)
__device__ __forceinline__ uint32_t miss_bits(uint32_t w) { return w & (w >> 1) & 0x55555555u; }
// What the Step-1 relayout writes for the sparse Miss rows of the Gram (miss_gram.cu).  Column tile ct covers words
// ctile[ct].x .. + ctile[ct].y - 1 (at most 32) of fold ctile[ct].z; fold f owns tiles fold_ct[f].x .. fold_ct[f].y - 1.
struct BedMissOut {
  const int4* ctile = nullptr;
  int nct = 0;
  int rows_p = 0;
  unsigned long long* total = nullptr;   // missing calls of the block; > cap: the dense Miss tiles run
  unsigned long long cap = 0;
  int2* seg = nullptr;                   // [rows_p][nct] (offset, count) into list
  int32_t* list = nullptr;               // missing samples, cap entries
  uint32_t* gt = nullptr;                // [Npad][rows_p / 16] sample-major 2-bit rows
};
// PLINK rows -> padded 2-bit rows gp [rows_p][npad / 16] (rows_p a multiple of 128)
void launch_bed_relayout(const uint8_t* packed, int64_t row_stride, int bs, int rows_p,
                         const int32_t* file_idx_pad, const int32_t* word_base, const uint32_t* word_keep, int ref_first,
                         uint32_t* gp, int64_t npad,
                         cudaStream_t s);
// the same, and the missing lists and Gt of the sparse Miss rows from the same pass (zeroes *mo.total first)
void launch_bed_relayout_miss(const uint8_t* packed, int64_t row_stride, int bs, int rows_p,
                              const int32_t* file_idx_pad, const int32_t* word_base, const uint32_t* word_keep,
                              int ref_first, uint32_t* gp, int64_t npad, const BedMissOut& mo, cudaStream_t s);

// ---- l0_stats.cu
struct SnpFinalizeArgs {
  int bs, rows_p, C, P, K, cpp, loocv;
  long long n_analyzed;
  double numtol;
  const int32_t* cnt_fold;   // [K][rows_p][4]
  const double* sum_fold;    // [K][rows_p][2][cpp]
  const double* XtX_f;       // [K][C][C]
  const double* XtY_f;       // [K][C][P]
  double *mu, *inv_sd;       // [rows_p]
  double* Bv;                // [rows_p][C]
  double *Af, *Qf;           // [K][rows_p][C]
  double *gty_f, *rhs;       // [K][rows_p][P]
  unsigned long long* err_slot;
  long long err_base;
};

struct AssembleArgs {
  int bs, rows_p, nC, C, K, R, loocv;
  const float* zz;           // [K][2*rows_p][ldz] exact integer Grams
  int64_t ldz, zz_fold_stride;
  const double *mu, *inv_sd, *Bv, *Af, *Qf;
  const double* lambda;      // [R]
  double* cm;                // batched row-major lower systems
  int64_t cm_stride;
  int ldc;
  float* planes = nullptr;   // l0_assemble_sym only: the same matrices in FP32 [K][n][n] (tensor-core operand)
  float* lplanes = nullptr;  // l0_assemble_sym only: factor matrices [K*R][n][n] of the mixed solver; their first 128 columns
                             // receive A_f + lambda_r I (panel step 0 of the left-looking factorisation has nothing to subtract)
};

void launch_l0_stats(const uint32_t* gp, int64_t npad, const double* xy, int cpp, const int4* chunks,
                     int nchunks, int rows_p, int32_t* cnt_part, double* sum_part, cudaStream_t s);
void launch_l0_fold_reduce(const int32_t* cnt_part, const double* sum_part, int rows_p, int cpp,
                           const int2* fold_chunks, int K, int32_t* cnt_fold, double* sum_fold,
                           cudaStream_t s);
void launch_l0_snp_finalize(const SnpFinalizeArgs& a, cudaStream_t s);
void launch_l0_assemble(const AssembleArgs& a, const double* rhs, int P, int Ppad, int nmat, cudaStream_t s);

// ---- gram_wgmma.cu
void make_gram_tensor_map(CUtensorMap* tm, const uint8_t* z, int64_t npad, int rows2);
// ---- l0_stats_tc.cu: the statistics as extra Gram column tiles
constexpr int kStatQ = 14;          // xy columns per 128-row digit group (14 x 9 limbs = 126 rows)
constexpr int kStatOnesRow = 126;   // row of the all-ones column (group 0)
void launch_l0_xy_digits(const double* xy, int cpp, int ncol, int64_t npad, const uint8_t* is_real, double* scale,
                         uint8_t* D, cudaStream_t s);
void launch_l0_stats_finish(const float* T, int ldt, int64_t t_fold_stride, const float* zz, int ldz,
                            int64_t zz_fold_stride, int rows_p, int cpp, int ncol, int K, const double* scale,
                            int32_t* cnt_fold, double* sum_fold, cudaStream_t s);
void gram_tile_list(int rows2, std::vector<int2>& tiles);
void stat_tile_list(int zrows, int drows, int bn, std::vector<int2>& tiles);
// The int8 planes of Z, built from the 2-bit rows inside the Gram kernel: Z row r is plane r / rows_p of 2-bit row
// r % rows_p, and lut[plane] is a PRMT table whose byte c is the plane's value for code c (3 = missing).  Every table
// carries a factor 8, which out_scale takes back out.
struct ZPlanes {
  uint32_t lut[3];
};
constexpr uint32_t kPlaneG = 0x00100800u;      // 8 g, 0 for a missing call
constexpr uint32_t kPlaneG2 = 0x00200800u;     // 8 g^2
constexpr uint32_t kPlaneMiss = 0x08000000u;   // 8 for a missing call
constexpr ZPlanes kZLevel0 = {{kPlaneG, kPlaneMiss, 0u}};         // Z = [G0; Miss] of a level-0 block
constexpr ZPlanes kZStep2 = {{kPlaneG, kPlaneG2, kPlaneMiss}};    // Z = [G; G^2; Miss]: Step 2's S1, S2, Sm
// Z of the 2-bit rows (tmG: make_gp_tensor_map over rows_p rows) against itself (tmD == nullptr: the Z Z^T tiles of
// gram_tile_list, bn 256) or against int8 digit rows (tmD: the statistics tiles of stat_tile_list, bn 256 or 128).
// miss_total != null: tiles of m tile >= miss_tile0 return at once when *miss_total <= miss_cap (miss_gram.cu)
void launch_gram_gp(const CUtensorMap& tmG, const CUtensorMap* tmD, int rows_p, const ZPlanes& planes,
                    const int2* tiles, int ntiles, const int2* fold_k, int K, float* out, int ldo, int64_t fold_stride,
                    float out_scale, cudaStream_t s, int bn = 256, const unsigned long long* miss_total = nullptr,
                    int64_t miss_cap = 0, int miss_tile0 = 0);
constexpr float kZScaleGram = 1.f / 64;   // Z Z^T tiles: both operands carry 8
// Z digit-row tiles: the digit rows are plain int8 integers.  Each accumulator is 8 x an integer sum, and a multiple of
// 8 below 2^27 converts to FP32 exactly, so the power-of-two scale leaves that sum exact.  Step 2's sample chunks (at
// most 2^18 samples, s2_build_digits) keep |acc| <= 8 * 60 * 2^18 < 2^27 (digits |d| <= 15, planes <= 4).
constexpr float kZScaleStat = 1.f / 8;
// ---- miss_gram.cu: the Miss rows of the Z Z^T Gram from per-(SNP, fold) lists of the missing calls
// missing calls per block (as a fraction of bs_max x analysed samples) up to which the sparse sums run: the crossover
// of tools/miss_rate_sweep.py (DESIGN.md section 3)
constexpr double kMissSparseRate = 0.015;
// one warp per (SNP row, fold): the fold's column tiles of seg (launch_bed_relayout_miss) -> Miss rows of zz
void launch_miss_sparse(const uint32_t* gt, int rows_p, const int2* seg, int nct, const int2* fold_ct,
                        const int32_t* list, int K, const unsigned long long* total, int64_t cap, float* zz,
                        int64_t fold_stride, cudaStream_t s);
// CUDA-core reference of the Z Z^T Gram of samples k0 .. k1 - 1, from the 2-bit rows (integer sums, not x 64)
void launch_gram_reference(const uint32_t* gp, int64_t npad, int rows_p, int k0, int k1, float* out, int ldo,
                           cudaStream_t s);

// ---- chol.cu
void launch_chol_factor(double* cm, int64_t stride, int nC, int n_aug, int batch, double* inv,
                        unsigned long long* err_slot, long long err_base, cudaStream_t s);
void launch_chol_backsolve(double* cm, int64_t stride, int nC, int P, int batch, const double* inv,
                           cudaStream_t s);
int chol_num_launches(int nC);
size_t chol_inv_elems(int nC, int batch);
void launch_chol_rows_backsolve(double* cm, int64_t stride, int nC, int row0, int nrows, int batch,
                                const double* inv, cudaStream_t s);

// ---- tf32_gemm.cu: batched 128x128 "NT" tiles in 3xTF32 on wgmma (operands = FP32 matrices, split into hi/lo in the kernel)
struct Tf32GemmEpilogue {
  int n;                      // matrix dimension = row stride of the output
  int64_t out_mat_stride;     // elements per matrix (n * n)
  float* out;                 // D as FP32 [batch][n][n]
  int mirror;                 // also store D^T into the mirror tile (what the backward substitution streams)
  int b_cols_local;           // B is [batch][n][128]: its columns count from the tile's first chunk, not from tile.z
  int negate;                 // D = -acc
  int lower_only;             // zero the strict upper part of diagonal tiles
  const double* cin;          // D = (float)(cin - acc) with FP64 matrices cin[mat / cin_mat_div][row][col], or null
  int64_t cin_mat_stride;
  int cin_ld, cin_mat_div;
  const double* diag_add;     // added to the diagonal of diagonal tiles: diag_add[mat % diag_mod] (the ridge shift), or null
  int diag_mod;
  int c_chunks;               // 0, or 4: leading K chunks  acc = C_tile * I  followed by the main chunks with A negated
  int c_mat_div;              // C matrix index = mat / c_mat_div
};
void make_tf32_operand_tensor_map(CUtensorMap* tm, const float* base, int cols, int rows, int batch);
void make_f32_rows_tensor_map(CUtensorMap* tm, const float* base, int cols, int64_t rows, int box_cols, int box_rows);
void launch_tf32x3_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const int4* tiles, int ntiles, int batch,
                        const Tf32GemmEpilogue& ep, cudaStream_t s, const CUtensorMap* tmC = nullptr);

// ---- chol_mixed.cu: tensor-core factorisation + FP64 iterative refinement of the level-0 ridge systems
constexpr int kMxMaxSteps = 6;
class MixedSolver {
 public:
  MixedSolver();
  ~MixedSolver();
  MixedSolver(const MixedSolver&) = delete;
  MixedSolver& operator=(const MixedSolver&) = delete;
  static int dim_for(int bs);                 // 128 * 2^k >= bs, or 0 when the block is too large for this path
  void prepare(int n, int K, int R, int Pp);
  // Af [K][n][n] FP64 full symmetric (no ridge shift) and the same in FP32, Ap [K][n][n], lambda [R],
  // bvec [K][Pp][n]; xvec / rvec [K*R][Pp][n]
  float* a_planes();                          // where the assembler writes Ap (owned by the solver, valid after prepare)
  float* l_planes();                          // the factor [K*R][n][n]: the assembler may fill block column 0 (first_col_ready)
  void solve(const double* Af, const double* lambda, const double* bvec, double* xvec, double* rvec, int P, int steps,
             float tol, unsigned int* fail_flag, cudaStream_t s, bool first_col_ready = false);
  static int launches_per_solve(int n, int steps, int P);
  const float* debug_planes(int which) const;  // 2 the factor (L below, L^T above the diagonal tiles), 3 the M_k; else null
 private:
  struct Impl;
  Impl* impl;
};
// K full symmetric fold systems (no ridge shift) + right-hand sides as rows, for the mixed solver
void launch_l0_assemble_sym(const AssembleArgs& a, const double* rhs, int P, int Pp, double* bvec, cudaStream_t s);

// ---- l0_dense.cu: level-0 block on real-valued genotypes (8-bit dosages / FP64), dense FP64 like the reference
void launch_dense_from_dosage(const uint8_t* probs, const uint8_t* miss, int64_t n_file, int bs, const int32_t* file_idx_pad,
                              int ref_first, double* gd, int64_t npad, cudaStream_t s);
void launch_dense_from_f64(const double* G, int64_t n_file, int bs, const int32_t* file_idx_pad, double* gd, int64_t npad,
                           cudaStream_t s);
void launch_dense_prepare(double* gd, int64_t npad, int bs, const int32_t* file_idx_pad, const double* xy, int cpp, int C,
                          long long n_analyzed, double numtol, double* mu, double* inv_sd, unsigned long long* err_slot,
                          long long err_base, cudaStream_t s);
void launch_dense_predict(const double* gd, int64_t npad, int bs, const double* cm, int64_t cm_stride, int ldc, int nC, int R,
                          int P, const int32_t* tile_fold, const uint8_t* mask, double* const* W, int col0, cudaStream_t s);

// ---- l0_predict.cu
struct PredictArgs {
  int bs, rows_p, C, P, R, Qp, cpp, col0;
  int64_t npad, words_per_row;
  const uint32_t* gp;
  const int32_t* tile_fold;  // [npad/128]
  const double *gam, *gmu;   // [K][rows_p][Qp]
  const double* cvec;        // [K][Qp][C]
  const double* xy;          // [npad][cpp]
  const uint8_t* mask;       // [P][npad]
  double* const* W;          // [P] base of each phenotype's npad x B column-major predictor matrix (may be peer memory)
  double* part;              // [ntiles][Qp][2]
};
void launch_l0_gamma(const double* cm, int64_t cm_stride, int ldc, int nC, int R, int P, int Qp,
                     int bs, int rows_p, int K, const double* mu, const double* inv_sd,
                     const double* Bv, int C, double* gam, double* gmu, double* cvec, cudaStream_t s);
void launch_l0_predict(const PredictArgs& a, int ntiles, cudaStream_t s);
void launch_l0_standardize(const double* part, int ntiles, int Qp, int Q, int P, const double* neff,
                           double* mean_invsd, double* const* W, int64_t npad, int col0,
                           const uint8_t* is_real, cudaStream_t s, const double* const* src = nullptr, int src_col0 = 0);
int predict_qt();

// ---- predict_wgmma.cu
struct PredictTcArgs {
  int rows_p, C, P, Q, Qp, cpp, col0, ngroups;
  int64_t npad;
  const int32_t* tile_fold;
  const double* scale;       // [K][Qp]
  const double* cvec;        // [K][Qp][C]
  const double* xy;
  const uint8_t* mask;
  double* const* W;
  double* part;
};
void make_byte_tensor_map(CUtensorMap* tm, const uint8_t* basep, int64_t inner, int64_t rows);
void make_gp_tensor_map(CUtensorMap* tm, const uint32_t* gp, int64_t words_per_row, int64_t rows);
int launch_l0_colsum(double* const* W, int64_t npad, int col0, int P, int Q, int Qp, double* part,
                     cudaStream_t s);
// INT8 digits: 5 radix-254 digit rows per output, s8 x s8 -> s32 wgmma
size_t predict_i8_dig_bytes(int K, int ngroups, int rows_p);
// gam, gmu, cvec, scales and digit rows of every (output, fold) from the solutions, one CTA each
void launch_l0_coef_i8(const double* cm, int64_t cm_stride, int ldc, int nC, int R, int P, int Q, int Qp, int bs,
                       int rows_p, int K, const double* mu, const double* inv_sd, const double* Bv, int C, double* gam,
                       double* gmu, double* cvec, double* scale, uint8_t* dig, int ngroups, cudaStream_t s);
// A operand from the 2-bit rows (tmG over gp), digit rows (tmD); raw predictions to a.W, per-tile column sums to a.part
void launch_l0_predict_i8(const CUtensorMap& tmG, const CUtensorMap& tmD, const PredictTcArgs& a, int ntiles,
                          cudaStream_t s);

// ---- l1_kernels.cu
void launch_l1_gram(const double* W, int64_t ldw, int B, const int4* chunks, int nchunks, double* part,
                    int64_t part_stride, int ldp, cudaStream_t s);
void launch_l1_xty(const double* W, int64_t ldw, const double* xy, int cpp, int ycol, const int4* chunks,
                   int nchunks, double* part_y, int B, cudaStream_t s);
// the fold systems of level 1 (P = 1) and of the dense level-0 route; every caller with loocv = 1 passes K = 1
void launch_l1_assemble(const double* part, int64_t part_stride, int ldp, const double* part_y, int64_t part_y_stride,
                        int P, const int2* fold_chunks, int K, int R1, const double* tau, int B, int nC, double* cm,
                        int64_t cm_stride, int loocv, cudaStream_t s);
void launch_l1_pred_sums(const double* W, int64_t ldw, int B, int R1, const double* beta, int ldb,
                         const int32_t* tile_fold, const double* xy, int cpp, int ycol, double* part_out,
                         int ntiles, double* out, cudaStream_t s);
void launch_l1_chr_pred(const double* W, int64_t ldw, int nchr, const int32_t* chr_col_start, const double* beta,
                        int ldb, int R1, int best, const int32_t* tile_fold, double* pred, int64_t npad,
                        cudaStream_t s);

// ---- loocv_kernels.cu
void launch_l0_loocv_fill(const uint32_t* gp, int64_t npad, int bs, int nC, const double* mu, const double* inv_sd,
                          const double* Bv, int C, const double* xy, int cpp, double* cm, int64_t cm_stride,
                          int nrow0, int R, cudaStream_t s);
void launch_l0_loocv_pred(const double* cm, int64_t cm_stride, int nC, int bs, int Ppad, int P, int R,
                          const double* xy, int cpp, int C, const uint8_t* mask, int64_t npad, double* const* W,
                          int col0, double* part, int Qp, cudaStream_t s);
void launch_l0_loocv_std_apply(double* const* W, int64_t npad, int col0, int P, int Q, const uint8_t* mask,
                               const double* mean_invsd, cudaStream_t s);
void launch_l1_loocv_fill(const double* W, int64_t ldw, int B, int nC, double* cm, int64_t cm_stride, int nrow0,
                          int R1, int64_t npad, cudaStream_t s);
void launch_l1_loocv_sums(const double* cm, int64_t cm_stride, int nC, int B, int nrow0, const double* xy, int cpp,
                          int ycol, double* part, int R1, int ntiles, double* out, cudaStream_t s);
void launch_rows_sqnorm(const double* rows, int nC, int B, double* out, int ntiles, cudaStream_t s);

// ---- l1_logistic.cu
void launch_l1_scale_rows(const double* W, int64_t ldw, int B, const double* wm, double* Ws, cudaStream_t s);
void launch_l1_bt_eta(const double* W, int64_t ldw, int B, const double* beta, const double* offset, const int8_t* ym,
                      double* eta, double* wm, double* resid, double* dev_part, double* dev_out, cudaStream_t s);
void launch_l1_bt_score(const double* part_y, int nchunks, int B, int nC, double tau, const double* beta, double* score,
                        double* rhs_row, cudaStream_t s);
void launch_l1_bt_loo_sums(const double* eta, const double* q, const double* wm, const double* resid, const int8_t* ym,
                           double eps, double* fvec, double* part, double* out6, int64_t npad, cudaStream_t s);
void launch_l1_bt_chr_pred(const double* W, int64_t ldw, int nC, const double* zrows, const double* fvec,
                           const double* bvec, int nchr, const int32_t* chr_col_start, double* pred, int64_t npad,
                           cudaStream_t s);
void launch_l1_loocv_chr_pred(const double* W, int64_t ldw, int B, int nC, const double* zrows, const double* hvec,
                              const double* bvec, const double* xy, int cpp, int ycol, int nchr,
                              const int32_t* chr_col_start, double* pred, int64_t npad, cudaStream_t s);
void launch_l0_std_reduce_only(const double* part, int ntiles, int Qp, int Q, int P, const double* neff,
                               double* mean_invsd, cudaStream_t s);

// ---- Step 2: device helpers of the per-variant kernels
// The genotype word dz of one (variant, sample), DESIGN.md "Step-2 genotype words": d = dosage x 255 (0..510) in bits
// 0-9, e = 4 p0 + p1 in bits 10-20 (8-bit dosages; 0 for hard calls), or the missing bit 31 alone.
constexpr uint32_t kDzMissing = 0x80000000u;
__device__ __forceinline__ uint32_t dz_word(uint32_t d, uint32_t e) { return d | (e << 10); }
__device__ __forceinline__ bool dz_missing(uint32_t w) { return (w & kDzMissing) != 0u; }
__device__ __forceinline__ uint32_t dz_d(uint32_t w) { return w & 0x3FFu; }
__device__ __forceinline__ uint32_t dz_e(uint32_t w) { return (w >> 10) & 0x7FFu; }

// The genotype value of a word has two arithmetic forms: Firth and SPA divide d by 255 (s2_sel_g), the GxE kernels
// multiply it by 1 / 255 (int_g).  They differ by one ulp on 48 of the 511 codes (never on the hard calls 0, 255, 510),
// so one form for both would change the results of the other on fractional dosages.
// Both: the value in the minor-allele coding (flip: 2 - g), and mu for a missing call.
__device__ __forceinline__ double s2_sel_g(uint32_t w, double mu, bool flip) {
  return dz_missing(w) ? mu : (flip ? 2.0 - (double)dz_d(w) / 255.0 : (double)dz_d(w) / 255.0);
}
__device__ __forceinline__ double int_g(uint32_t w, double mu, bool flip = false) {
  if (dz_missing(w)) return mu;
  const double g = (double)dz_d(w) * (1.0 / 255.0);
  return flip ? 2.0 - g : g;
}

constexpr double kNumtolEps = 10.0 * 2.220446049250313e-16;   // numtol_eps, src/Regenie.hpp:225
__device__ __forceinline__ double get_pvec(double eta) {      // src/Step1_Models.cpp:1797-1804
  if (eta > 30.0) return 1.0 / (1.0 + kNumtolEps);
  if (eta < -30.0) return kNumtolEps / (1.0 + kNumtolEps);
  return 1.0 - 1.0 / (exp(eta) + 1.0);
}

// Fixed-order sum of v over a CTA of kWarps warps (lanes by shuffles, then the warps in ascending order), so the totals do
// not depend on timing; every thread receives them.  sh holds kWarps * K doubles.
template <int kWarps, int K>
__device__ __forceinline__ void cta_sum(double (&v)[K], double* sh) {
#pragma unroll
  for (int k = 0; k < K; ++k)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < K; ++k) sh[warp * K + k] = v[k];
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += sh[w * K + k];
    v[k] = s;
  }
}

// A CTA's fixed-order reduction has two forms: cta_sum (Step 2) adds the lanes of each warp by shuffles and then the
// warps in order, cta_tree (the Step-1 FP64 kernels) halves a shared-memory tree, sh[t] op sh[t + o] for o = kThreads / 2
// .. 1.  They pair the values differently, so one form for both would change the last bits of the other step's results.
// cta_tree: v[k] of every thread combined by kOp (sum or fmax) over a CTA of kThreads threads (128 or 256); every thread
// receives the totals.  sh holds K * kThreads doubles.  It starts with a barrier, so a caller may loop over it.
enum class CtaOp { kSum, kMax };
template <int kThreads, CtaOp kOp = CtaOp::kSum, int K>
__device__ __forceinline__ void cta_tree(double (&v)[K], double* sh) {
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) sh[k * kThreads + threadIdx.x] = v[k];
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
#pragma unroll
      for (int k = 0; k < K; ++k) {
        double* r = sh + k * kThreads + threadIdx.x;
        *r = kOp == CtaOp::kMax ? fmax(r[0], r[o]) : r[0] + r[o];
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = sh[k * kThreads];
}
template <int kThreads, CtaOp kOp = CtaOp::kSum>
__device__ __forceinline__ double cta_tree(double v, double* sh) {
  double a[1] = {v};
  cta_tree<kThreads, kOp>(a, sh);
  return a[0];
}

// N, MAC and AF of column c of a variant's sums (compute_mac / compute_aaf_info, src/Geno.cpp:3077-3148), and INFO when
// info is not null.  S1, S2, Se are in units of 1 / k (k = 1: dosage units), Sm counts the missing calls and n is the
// column's total over the analysed samples.  Non-PAR chrX (cm >= 0, the column of the same samples' males, *n_male
// their total): males are coded 0/2 but count half towards the allele count (src/Geno.cpp:2447-2462).
struct S2Count { double ns, mac; };
__device__ __forceinline__ S2Count s2_count(const double* S1, const double* S2, const double* Sm, const double* Se, int c,
                                            double n, int cm, const double* n_male, double k, int32_t* ns_out, double* mac_out,
                                            double* af_out, double* info) {
  const double ns = n - Sm[c];
  const double tp = S1[c] * k;
  double mac;
  if (cm >= 0) {
    const double macr = tp - 0.5 * S1[cm] * k;
    mac = fmin(macr, 2.0 * ns - (*n_male - Sm[cm]) - macr);
  } else {
    mac = fmin(tp, 2.0 * ns - tp);
  }
  *ns_out = (int)ns;
  *mac_out = mac;
  const double af = tp / (2.0 * ns);
  *af_out = af;
  if (info) {                                                        // 1 - sum(4 p0 + p1 - g^2) / (2 n af (1 - af))
    const double num = Se[c] * k - S2[c] * (k * k);
    *info = (af == 0.0 || af == 1.0) ? 1.0 : 1.0 - num / (2.0 * ns * af * (1.0 - af));
  }
  return {ns, mac};
}

// ---- s2_kernels.cu
struct S2FinalizeArgs {
  int bs, C, P, dp, strict;
  long long n_analyzed, n_samples;
  double min_mac, numtol;
  const double* sums;        // [rows_p][3][dp]
  const double* mask_count;  // [P]
  const double* YtX;         // [P][C]
  const double* XmX;         // [P][C][C]
  const double* scf_sv;      // [P]
  const uint8_t* non_par = nullptr;   // [bs] variant lies in the non-PAR part of chrX (males count half towards MAC)
  int col_male = -1;                  // F column of the male indicator (followed by male x mask_p), -1 = no sex information
  const double* male_tot = nullptr;   // [1 + P] analysed males, masked-in males per trait
  const double* nz_count = nullptr;   // [rows_p] non-zero dosages among analysed samples (dosage input only)
  const double* info_sums = nullptr;  // [rows_p][dp] sum (4 p0 + p1) F (dosage input only)
  double* info = nullptr;             // [bs x P] INFO (dosage input only)
  double *af, *mac, *af_all, *mac_all, *scale_fac, *stat, *beta, *se, *chisq;
  int32_t *ns, *ns_all, *flags;
};
void launch_s2_stats(const uint32_t* gp, int64_t npad, const double* F, int dp, const int4* chunks, int nchunks,
                     int rows_p, double* part, double* sums, cudaStream_t s);
void launch_s2_finalize(const S2FinalizeArgs& a, cudaStream_t s);
// tensor sums T [chunk][3 rows_p][ldt] -> S1, S2, Sm: sums [rows][3][dp] for s2_finalize_kernel (nnz == nullptr), or
// for the binary-trait finish on hard calls [rows][4][dp] (S1, S2, Sm, 0) + non-zero / hom-alt counts nnz / n2
void launch_s2_tensor_finish(const float* T, int ldt, int64_t chunk_stride, int nchunk, int rows_p, int dp, int D,
                             const double* scale, double* sums, double* nnz, double* n2, cudaStream_t s);
void launch_gp_to_dz(const uint32_t* gp, int rows_p, uint32_t* dz, int64_t npad, cudaStream_t s);

// ---- s2_dosage_kernels.cu
struct S2BtFinalizeArgs {
  int bs, C, P, dp, with_flip;
  long long n_analyzed, n_samples;
  double min_mac, numtol;
  const double* sums;        // [rows_p][4][dp]  S1, S2, Sm, Se in integer dosage units
  const double* col_tot;     // [dp] sum of every feature column over all samples
  const double* xwy;         // [P][C]  XW^T yres
  const uint8_t* non_par = nullptr;   // see S2FinalizeArgs
  int col_male = -1;
  double unit = 255.0;                // S1 / S2 / Se are in units of 1/unit (255 for 8-bit dosages, 1 for hard calls)
  const double* nz_count;    // [rows_p] analysed samples with non-zero dosage
  const double* n510;        // [rows_p] analysed samples with dosage exactly 2
  double *af, *mac, *info, *af_all, *mac_all, *scale_fac, *stat, *beta, *se, *chisq, *xtwg, *mu, *den;
  int32_t *ns, *ns_all, *flags;
};
void launch_dosage_relayout(const uint8_t* probs, const uint8_t* miss, int64_t n_file, int bs, int rows_p,
                            const int32_t* file_idx_pad, int ref_first, uint32_t* dz, int64_t npad, cudaStream_t s);
void launch_dosage_stats(const uint32_t* dz, int64_t npad, const double* F, int dp, const int4* chunks, int nchunks,
                         int rows_p, double* part, int2* part_cnt, double* sums, double* nnz, double* n510, cudaStream_t s,
                         int ncol = 0 /* used feature columns (<= dp), 0 = all */);
void launch_s2_bt_finalize(const S2BtFinalizeArgs& a, cudaStream_t s);
// integer-unit sums [rows][4][dp] -> dosage-unit [rows][3][dp] (S1, S2, Sm) + [rows][dp] (Se)
void launch_dosage_scale(const double* sums4, int rows_p, int dp, double* sums3, double* se, cudaStream_t s);

// ---- s2_firth.cu / s2_spa.cu: one CTA per selected (variant, trait) of the resident binary-trait block
struct S2SelArgs {
  int n_sel, C, P, dp, niter;
  double tol;
  int64_t npad;
  const int32_t *sel_var, *sel_trait;
  const uint32_t* dz;
  const double* F;                   // [Npad][dp] binary-trait feature rows (column 0: in the analysis)
  const double *w, *gs, *xw;         // [P][Npad], xw [P][C][Npad]
  const int8_t* ym;                  // [P][Npad] 0 masked, 1 control, 2 case
  const double* xtwg;                // [bs][P][C]
  const double* mu;                  // [bs] imputed mean (after flip)
  const int32_t* flags;              // [bs]
  double* gvec;                      // [n_sel][Npad] scratch
  int8_t* cflag;                     // [n_sel][Npad] scratch (carrier / active-set flags)
  int32_t* status;                   // [n_sel]
};
// What both kernels read first for selection blockIdx.x: the pair's rows, the variant's coding and X^T W g, which goes
// to the kernel's own array v (a member array would put the whole struct in local memory)
struct S2Sel {
  int C;
  int64_t npad;
  int i, ph;                         // variant, trait
  bool flip, sparse;                 // flags bits 3 and 2
  double mu;
  const uint32_t* drow;
  const double *w, *gs, *xw;
  const int8_t* ym;
  double* gv;
  int8_t* cf;
  double* v;                         // [C]
  __device__ __forceinline__ S2Sel(const S2SelArgs& a, double (&vr)[kMaxCov]) : C(a.C), npad(a.npad), v(vr) {
    const int sel = blockIdx.x;
    i = a.sel_var[sel]; ph = a.sel_trait[sel];
    const int flags = a.flags[i];
    flip = flags & 8; sparse = flags & 4;
    mu = a.mu[i];
    drow = a.dz + (int64_t)i * a.npad;
    w = a.w + (int64_t)ph * a.npad; gs = a.gs + (int64_t)ph * a.npad; xw = a.xw + (int64_t)ph * a.C * a.npad;
    ym = a.ym + (int64_t)ph * a.npad;
    gv = a.gvec + (int64_t)sel * a.npad; cf = a.cflag + (int64_t)sel * a.npad;
    for (int c = 0; c < a.C; ++c) v[c] = a.xtwg[((int64_t)i * a.P + ph) * a.C + c];
  }
  // the genotype g of sample t (0 outside the analysis) and its residual r = g w - sum_c xw_c v_c
  __device__ __forceinline__ double gres(const S2SelArgs& a, int64_t t, double& g) const {
    g = s2_sel_g(drow[t], mu, flip);
    if (a.F[t * a.dp] == 0.0) g = 0.0;
    double r = g * w[t];
    for (int c = 0; c < C; ++c) r -= xw[(int64_t)c * npad + t] * v[c];
    return r;
  }
};

struct FirthArgs : S2SelArgs {
  double maxstep;
  const double* off;                 // [P][Npad]
  const double* mac;                 // [bs][P]
  double *beta, *se, *lrt;
};
void launch_s2_firth(const FirthArgs& a, cudaStream_t s);

struct SpaArgs : S2SelArgs {
  const double* phat;                // [P][Npad]
  const double *stat, *den;          // [bs][P] score statistic and its denominator G'WG
  double* pval;                      // [n_sel] sum of the two tail probabilities
};
void launch_s2_spa(const SpaArgs& a, cudaStream_t s);

// ---- s2_interaction.cu
// near-singular check and inverse of a symmetric 2 x 2 (SelfAdjointEigenSolver + eigenvalues().minCoeff() < numtol)
__device__ inline bool int_inv2(double a11, double a12, double a22, double numtol, double* z) {
  const double hm = 0.5 * (a11 + a22), hd = 0.5 * (a11 - a22);
  const double lmin = hm - sqrt(hd * hd + a12 * a12);
  if (!(lmin >= numtol)) return false;
  const double det = a11 * a22 - a12 * a12;
  z[0] = a22 / det; z[1] = -a12 / det; z[2] = a11 / det;
  return true;
}
constexpr int kIntTG = 8;            // traits per CTA of the meat kernel (blockIdx.z = trait group)
constexpr int64_t kIntSlab = 16384;  // samples per host slab of the feature rows (rg_s2_set_interaction)
struct S2IntArgs {
  int bs, C, P, dp, K, nf, nr, nchunks, var_stride;
  int force_robust, force_hc4, no_robust;
  long long n_analyzed, n_samples;
  double rare_mac, min_mac, numtol;
  int64_t npad;
  const uint32_t* dz;                // [rows_p][Npad] genotype words of the resident block
  const double* Fint;                // [Npad][nf] interaction features (robust nr columns, then HLM P x (2K + 5))
  const double* F;                   // [Npad][dp] the QT feature rows of rg_s2_set_chr (X, res, mask)
  const double* E;                   // [Npad]
  const int4* chunks;
  const double *af_all, *mac, *YtX, *scf_sv, *mask_count;
  const int32_t* flags;
  double* sums;                      // [bs][nf]
  double* var;                       // [bs][var_stride] per-variant robust state
  double* meat_part;                 // [bs][P][nchunks][4]
  int32_t* status;                   // [bs][P]
  double *coef, *vcov;               // [bs][P][2], [bs][P][4]
  int8_t* route;                     // [bs] 0 none, 1 robust, 2 HLM (written by the first kernel)
};
void launch_s2_interaction(const S2IntArgs& a, const uint8_t* pow2, double* part, cudaStream_t s);
// sums[v][f] = sum over the samples of g_v^(1 or 2) Fint[i][f] (pow2[f]) for the variants with route[v] == 1 (the robust
// columns [0, nr) of s2_int_sums_kernel; nr = nf for the binary-trait feature rows).  g is the mean-imputed genotype:
// missing calls take 2 af_all[v] when mu is null, else mu[v], with non-missing calls flipped to 2 - g when flags[v] & 8.
void launch_s2_int_sums(const uint32_t* dz, int64_t npad, const double* af_all, const double* mu, const int32_t* flags,
                        int bs, const int8_t* route, int nr, const double* Fint, int nf, const uint8_t* pow2,
                        const int4* chunks, int nchunks, double* part, double* sums, cudaStream_t s);

// ---- s2_interaction_bt.cu
constexpr int kIntBtTG = 4;          // traits per CTA of the logistic kernel (blockIdx.y = trait group)
constexpr int kIntBtBatch = 128;     // variants (Wald) or pairs (Firth) whose H columns are materialised at a time
struct S2IntBtArgs {
  int bs, C, P, nf, nchunks, var_stride;
  int force_robust, no_robust;
  long long n_analyzed;
  double rare_mac, min_mac, numtol;
  int64_t npad;
  const uint32_t* dz;                // [rows_p][Npad] genotype words of the resident block
  const double* Fint;                // [Npad][nf] X_c, E X_c (times g), 1, E, E^2 (times g^2); zero outside the analysis
  const double* E;                   // [Npad]
  const int8_t* ym;                  // [P][Npad] 0 masked, 1 control, 2 case
  const double* off;                 // [P][Npad] offset of the fits (offset_nullreg, or the null-Firth offset)
  const int4* chunks;
  const double *af_all, *mu, *mac;
  const int32_t* flags;
  int8_t* route;                     // [bs] 1 = the variant is tested
  double* sums;                      // [bs][nf]
  double* var;                       // [bs][var_stride]: ok, scale_fac, scf_i, X^T G [C], X^T (E o G) [C]
  double* H;                         // [kIntBtBatch][2][Npad] the H columns of a batch
  int v0, nb;                        // the batch: variants v0 .. v0 + nb (Wald)
  // Wald outputs [bs][P]
  int32_t* status;
  double *coef, *vcov;               // [bs][P][2], [bs][P][4]
  // Firth: pair k of the batch is (sel_var[k], sel_trait[k]); H slot k holds its variant's columns
  const int32_t *sel_var, *sel_trait;
  int niter;
  double tol, maxstep;
  double *f_coef, *f_se, *f_lrt;     // [nb][2], [nb][2], [nb][3]
  int32_t* f_status;                 // [nb]
};
// route, per-variant sums, scales and residualisation coefficients of every variant of the block
void launch_s2_int_bt_prep(const S2IntBtArgs& a, const uint8_t* pow2, double* part, cudaStream_t s);
// H columns of the batch, then the logistic fits of its variants (every trait)
void launch_s2_int_bt_wald(const S2IntBtArgs& a, cudaStream_t s);
// H columns of the batch's pairs, then the three Firth fits of each pair
void launch_s2_int_bt_firth(const S2IntBtArgs& a, cudaStream_t s);

}  // namespace rg
