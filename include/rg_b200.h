/*
 * rg_b200.h -- C ABI of the H100-native regenie hot path (librg_b200.so).
 *
 * The reference (rgcgithub/regenie v4.1.2) has no FFI: its hot path is a sequence of
 * C++ member/free functions called from Data::run_step1 / Data::test_snps_fast.  Each
 * entry point below replaces the call(s) cited next to it; INTEGRATION.md shows the
 * binding a maintainer would add to src/Data.cpp.
 *
 * Conventions
 *   - plain pointers + sizes, no C++/torch types; all matrices are column-major f64
 *     exactly like Eigen::MatrixXd unless stated.
 *   - every function returns 0 on success, non-zero on error; rg_last_error() gives the
 *     message (the reference throws std::string, src/Regenie.cpp:67-92).
 *   - the host owns host buffers, the library owns device buffers.  Pointers flagged
 *     [host|device] may be either: the library inspects them with
 *     cudaPointerGetAttributes and copies host memory itself (pinned memory is copied
 *     asynchronously).
 *   - one rg_handle per GPU / per host thread; calls on a handle are serialised on the
 *     handle's CUDA stream and are asynchronous until rg_sync or a call that returns
 *     host data.
 *   - there is NO CPU fallback: every call fails with an error when no CUDA device
 *     (sm_90) is usable.
 */
#ifndef RG_B200_H
#define RG_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct rg_ctx* rg_handle;

/* ------------------------------------------------------------------ library */
const char* rg_last_error(void);
const char* rg_version(void);
/* number of usable CUDA devices (0 => nothing below can run) */
int rg_device_count(void);
/* Optional: create the CUDA context of `device` now (driver initialisation + context creation take of the order of a
 * second on a multi-GPU node).  A caller may run it on a side thread while it parses its text inputs, as rgb200 does;
 * the create calls below do the same work when it has not been done. */
int rg_warmup(int32_t device);

/* ------------------------------------------------------------------ Step 1 */
typedef struct rg_step1_config {
  int32_t device;          /* CUDA ordinal                                               */
  int64_t n_samples;       /* N  = params.n_samples (after --keep/--remove)              */
  int32_t n_cov;           /* C  = params.ncov, columns of the orthonormal basis X       */
  int32_t n_pheno;         /* P                                                          */
  int32_t n_folds;         /* K  = params.cv_folds (ignored when loocv != 0)             */
  int32_t n_ridge_l0;      /* R  = params.n_ridge_l0                                     */
  int32_t n_ridge_l1;      /* R1 = params.n_ridge_l1                                     */
  int32_t loocv;           /* params.use_loocv                                           */
  int32_t max_block_size;  /* params.block_size                                          */
  int32_t total_blocks;    /* params.total_n_block  (columns of W = total_blocks * R)    */
  int64_t n_analyzed;      /* params.n_analyzed                                          */
} rg_step1_config;

/*
 * rg_step1_create -- replaces Data::setmem / set_folds (src/Data.cpp:401-431,478-577):
 * uploads the state every block shares.
 *   X           [N x C]  pheno_data.new_cov   (orthonormal, zero rows outside analysis)
 *   Y           [N x P]  pheno_data.phenotypes (residualised, scaled, masked)
 *   mask        [N x P]  pheno_data.masked_indivs as bytes (column-major)
 *   in_analysis [N]      filters.ind_in_analysis as bytes
 *   fold_sizes  [K]      params.cv_sizes (contiguous folds in sample order)
 *   lambda      [R]      params.lambda AFTER the M(1-h)/h map (src/Data.cpp:607)
 *   neff        [P]      pheno_data.Neff
 */
int rg_step1_create(const rg_step1_config* cfg, const double* X, const double* Y,
                    const uint8_t* mask, const uint8_t* in_analysis,
                    const int64_t* fold_sizes, const double* lambda, const double* neff,
                    rg_handle* out);
void rg_destroy(rg_handle h);
/* Block the host until every call issued on the handle has finished. */
int rg_sync(rg_handle h);
/* Device-side join: consecutive level-0 blocks run on several internal streams ("lanes"); rg_fence
 * makes the handle's stream (rg_stream) wait for all of them without blocking the host, so an event
 * recorded on rg_stream afterwards covers all outstanding work. */
int rg_fence(rg_handle h);

/*
 * rg_l0_block_bed -- one level-0 block from 2-bit PLINK rows.  Replaces, for one block,
 *   readChunkFromBedFileToG (decode + mean-impute)   src/Geno.cpp:1702-1768
 *   Data::residualize_genotypes                      src/Data.cpp:190-228
 *   Data::calc_cv_matrices                           src/Data.cpp:729-776
 *   ridge_level_0 / ridge_level_0_loocv              src/Step1_Models.cpp:458-613 / 615-726
 * and leaves the block's N x R level-0 predictors of every phenotype in the device
 * resident W (columns block_id*R .. block_id*R+R-1).
 *   packed      [host|device] bs rows of row_stride bytes, the .bed rows of the block.
 *               LIFETIME: the call only enqueues work.  A pageable host buffer is staged before the call returns and
 *               may be reused at once; a PINNED host buffer is read by DMA later - do not overwrite it before
 *               rg_l0_wait_input(h) (or rg_sync) returns.  Device buffers: until the block has run (rg_sync / rg_fence).
 *   sample_idx  [host|device] N entries: index in the .bed row of sample i (handles
 *               --keep/--remove, i.e. filters.ind_ignore); NULL = identity
 *   ref_first   params.ref_first
 * Error (non-zero) when a SNP has sd < 1e-6 is deferred to the next rg_sync /
 * rg_l0_status (reference throws at src/Data.cpp:207).
 */
int rg_l0_block_bed(rg_handle h, const uint8_t* packed, int64_t row_stride, int32_t bs,
                    const int32_t* sample_idx, int32_t ref_first, int32_t block_id);

/*
 * rg_l0_block_dosage_u8 -- the same level-0 block from 8-bit BGEN probability pairs (after inflate).  Replaces
 *   readChunkFromBGENFileToG_fast   src/Geno.cpp:1574-1699  (dosage = p1/255 + 2 p0/255, or p1/255 + 2 p2/255 with
 *                                   --ref-first; missing = bit 7 of the ploidy byte; mean imputation)
 * followed by the functions rg_l0_block_bed lists.  Real-valued genotypes take the dense FP64 route (csrc/l0_dense.cu:
 * per-fold Gram on the FP64 tensor pipe, batched Cholesky) instead of the exact-integer tensor-core route of hard calls.
 *   probs           [host|device] [bs][n_file][2] bytes (P(hom first allele), P(het)) - the layout rg_bgen_inflate and
 *                   the host BGEN reader produce
 *   ploidy_missing  [host|device] [bs][n_file] bytes, bit 7 = missing; NULL = nothing missing
 *   n_file          samples per variant in the file; sample_idx as in rg_l0_block_bed
 */
int rg_l0_block_dosage_u8(rg_handle h, const uint8_t* probs, const uint8_t* ploidy_missing, int64_t n_file, int32_t bs,
                          const int32_t* sample_idx, int32_t ref_first, int32_t block_id);

/* rg_l0_block_f64 -- the same from an FP64 genotype matrix G [bs][n_file] (row-major, -3 = missing): the shape the
 * reference's PGEN dosage reader fills (readChunkFromPGENFileToG, src/Geno.cpp:1773-1821). */
int rg_l0_block_f64(rg_handle h, const double* G, int64_t n_file, int32_t bs, const int32_t* sample_idx, int32_t block_id);

/* Wait until the input rows of the most recent rg_l0_block_bed call have been copied to the device (see LIFETIME). */
int rg_l0_wait_input(rg_handle h);

/* 0 = all blocks so far fine; otherwise 1 + index (block_id * max_block_size + snp) of the
 * first low-variance SNP (src/Data.cpp:205-209).  Synchronises the stream. */
int64_t rg_l0_status(rg_handle h);

/* The same word WITHOUT waiting for the blocks in flight: what the blocks that have finished so far reported (the word is
 * sticky - the first low-variance SNP stays until the handle is destroyed - so a caller that polls once per pass and
 * calls rg_l0_status / rg_sync at the end misses nothing).  One 8-byte device-to-host read on a stream of its own; the
 * lanes keep running.  Does not re-solve blocks whose mixed-precision solve was flagged (rg_l0_status / rg_sync do). */
int64_t rg_l0_poll_status(rg_handle h);

/*
 * rg_l0_fetch_W -- copy a block's level-0 predictors of phenotype ph to the host as the
 * N x R column-major slab the reference appends to <prefix>_l0_Y<ph+1> under --lowmem
 * (write_l0_file, src/Step1_Models.cpp:728-733).
 */
int rg_l0_fetch_W(rg_handle h, int32_t block_id, int32_t ph, double* out_NxR);
/* inverse of rg_l0_fetch_W: place a block's N x R slab read from a level-0 file (read_l0_chunk,
 * src/Step1_Models.cpp:1956-1987; --run-l1 after --run-l0 jobs, possibly produced by the reference itself) */
int rg_l0_load_W(rg_handle h, int32_t block_id, int32_t ph, const double* in_NxR);

/*
 * rg_l1_fit -- level-1 ridge for all phenotypes.  Replaces ridge_level_1 /
 * ridge_level_1_loocv (src/Step1_Models.cpp:772-872 / 875-963) and the tau* choice of
 * Data::output (src/Data.cpp:1025-1037).
 *   tau      [P x R1] row-major: params.tau[ph] AFTER the B(1-h)/h map
 *   cumsum   [5 x P x R1] out: l1_ests.cumsum_values[0..4] (Sx, Sy, Sx2, Sy2, Sxy)
 *   best_idx [P] out: argmin_j (Sx2 + Sy2 - 2 Sxy)/Neff
 * Only the phenotypes this handle fits (rg_l1_select) are written: the cumsum rows and best_idx entries of the others
 * keep what the caller passed (pass zeroed buffers to get zeros there).
 */
int rg_l1_fit(rg_handle h, const double* tau, double* cumsum, int32_t* best_idx);

/*
 * rg_loco -- per-chromosome predictions + LOCO assembly.  Replaces make_predictions /
 * make_predictions_loocv (src/Data.cpp:1196-1343) and the arithmetic of
 * write_predictions (src/Data.cpp:1846-1858).
 *   chr_of_block [total_blocks]  chromosome (1..23) of each level-0 block
 *   pred_out     [P][N x 23] column-major per phenotype: the values of `pred` written row
 *                by row into <out>_<ph+1>.loco
 */
int rg_loco(rg_handle h, const int32_t* chr_of_block, double* pred_out);

/*
 * rg_prs -- whole-genome predictions of the last rg_loco call: the row sums `predictions[0].rowwise().sum()` that
 * write_predictions prints with --print-prs (src/Data.cpp:1906-1922).  Host-side copy, no kernel.
 *   prs_out [P][N]; phenotypes this handle does not fit (rg_l1_select) are zero
 */
int rg_prs(rg_handle h, double* prs_out);

/*
 * rg_l1_fit_bt -- binary traits: penalised logistic level 1 with closed-form leave-one-out predictions.
 * LOOCV handles (cfg.loocv = 1): replaces ridge_logistic_level_1_loocv + run_log_ridge_loocv
 * (src/Step1_Models.cpp:1159-1375); rg_loco then performs make_predictions_binary_loocv (src/Data.cpp:1484-1573).
 * k-fold handles: replaces ridge_logistic_level_1 (src/Step1_Models.cpp:966-1157, IRLS per fold and tau with warm
 * starts); rg_loco then performs make_predictions_binary (src/Data.cpp:1346-1428).  Level 0 is the QT path
 * (rg_l0_block_bed with the residualised 0/1 phenotypes as Y).
 *   y_raw  [N x P] phenotypes_raw (0/1), offset [N x P] m_ests.offset_nullreg (covariate-only logistic fit)
 *   tau    [P x R1] ridge values (B (1-h)/h * 3/pi^2, src/Step1_Models.cpp:2115-2117)
 *   cumsum [6][P][R1]  Sx, Sy, Sx2, Sy2, Sxy, -logLik (cumsum_values[0..5]);  best_idx = argmin -logLik/Neff
 * As in rg_l1_fit, phenotypes this handle does not fit keep the cumsum rows and best_idx entries the caller passed.
 */
int rg_l1_fit_bt(rg_handle h, const double* y_raw, const double* offset, const double* tau, double* cumsum,
                 int32_t* best_idx);

/* ------------------------------------------------------------------ Step 2 (QT) */
typedef struct rg_step2_config {
  int32_t device;
  int64_t n_samples;       /* N                                                          */
  int32_t n_cov;           /* C  = params.ncov (orthonormal basis columns)               */
  int32_t n_pheno;         /* P                                                          */
  int32_t max_block_size;  /* params.block_size                                          */
  int64_t n_analyzed;      /* params.n_analyzed                                          */
  int32_t strict_mode;     /* params.strict_mode (forced when P == 1, src/Pheno.cpp:198) */
} rg_step2_config;

/*
 * rg_step2_create -- state shared by every variant of a Step-2 run:
 *   X [N x C] pheno_data.new_cov, mask [N x P] pheno_data.masked_indivs (after blup_read),
 *   in_analysis [N] filters.ind_in_analysis.
 * rg_s2_set_chr -- per chromosome, what Data::compute_res (src/Data.cpp:2386-2404) produces:
 *   res [N x P] = (Y - blup) o mask / p_sd_yres,  scf_sv [P] = scale_Y * p_sd_yres.
 *   (YtX = res^T X is formed on the device.)
 */
int rg_step2_create(const rg_step2_config* cfg, const double* X, const uint8_t* mask,
                    const uint8_t* in_analysis, rg_handle* out);
int rg_s2_set_chr(rg_handle h, const double* res, const double* scf_sv);

/*
 * chrX: rg_s2_set_sex gives the male indicator of every sample (params.sex == 1; NULL = forget it) and takes
 * effect at the next rg_s2_set_chr / rg_s2_set_chr_bt; rg_s2_set_non_par flags the variants of the NEXT block
 * call that lie in the non-PAR part of chrX (in_non_par, src/Geno.cpp:2802-2814).  For those variants males
 * count half towards the allele count and MAC = min(mac, 2 N - N_males - mac) (src/Geno.cpp:2447-2462,
 * compute_mac :3077-3108), which decides the --minMAC filter; A1FREQ, N and the test itself are unchanged.
 */
int rg_s2_set_sex(rg_handle h, const uint8_t* male);
int rg_s2_set_non_par(rg_handle h, const uint8_t* flags, int32_t n);

/* per-variant outputs of one Step-2 block; host arrays, variant-major ([i*P + p]) */
typedef struct rg_s2_out {
  double* af;        /* [bs x P] block_info->af   (A1FREQ per trait)                      */
  int32_t* ns;       /* [bs x P] block_info->ns   (N per trait)                           */
  double* mac;       /* [bs x P] block_info->mac                                          */
  double* af_all;    /* [bs]     af1                                                      */
  int32_t* ns_all;   /* [bs]     ns1                                                      */
  double* mac_all;   /* [bs]     mac1                                                     */
  int32_t* flags;    /* [bs]     bit0 ignored (MAC < minMAC), bit1 ignored (scale_fac <
                                 numtol), bit2 sparse-genotype formulas were used         */
  double* scale_fac; /* [bs]     residualize_geno scale (1 on the sparse path)            */
  double* stat;      /* [bs x P] dt_thr->stats = num / sqrt(denum)                        */
  double* beta;      /* [bs x P] dt_thr->bhat                                             */
  double* se;        /* [bs x P] dt_thr->se_b                                             */
  double* chisq;     /* [bs x P] dt_thr->chisq_val                                        */
} rg_s2_out;

/*
 * rg_s2_stage -- start the host -> device copy of a LATER block's input bytes (PLINK rows, BGEN probability or
 * ploidy bytes) on the handle's copy stream and return the device address to pass as `packed` / `probs` /
 * `ploidy_missing` to the rg_s2_block_* call of that block, which waits for exactly this copy.  The reference
 * overlaps reading block b+1 with testing block b on its OpenMP threads (src/Data.cpp:2284-2312, Gblock read ahead
 * of compute_tests_mt); here the PCIe transfer of block b+1 rides under the kernels of block b.  slot in 0..3: a slot's
 * buffer is reused, so stage block b+2 into the slot of block b only after block b's call has returned.  `host` must
 * stay untouched until the consuming block call returns; the copy is asynchronous only from pinned memory
 * (rg_host_alloc).
 */
int rg_s2_stage(rg_handle h, int32_t slot, const void* host, int64_t bytes, const uint8_t** dev);

/* pinned host memory for staged inputs (cudaMallocHost / cudaFreeHost behind the C ABI) */
int rg_host_alloc(void** p, int64_t bytes);
int rg_host_free(void* p);

/*
 * rg_s2_block_bed -- Step-2 score test for bs variants from 2-bit PLINK rows.  Replaces, per
 * variant: parseSnpfromBed + compute_mac + compute_aaf_info (src/Geno.cpp:2414-2536,
 * 3077-3148), check_sparse_G (:3165), residualize_geno (:3242) and compute_score_qt
 * (src/Step2_Models.cpp:343-467) up to chisq; LOG10P (get_logp) and text are host work.
 * sample_idx [host|device] as in rg_l0_block_bed.
 */
int rg_s2_block_bed(rg_handle h, const uint8_t* packed, int64_t row_stride, int32_t bs,
                    const int32_t* sample_idx, int32_t ref_first, double min_mac,
                    const rg_s2_out* out);

/* ------------------------------------------------------------------ Step 2 (BT, BGEN dosages) */
/*
 * Per-chromosome null-model state of the binary traits, as left by fit_null_logistic in test mode
 * (src/Step1_Models.cpp:54-140), Data::compute_res_bin (src/Data.cpp:2439-2455) and, for --firth --approx,
 * fit_null_firth (src/Step2_Models.cpp:985-1060).  All arrays are trait-major [P][N] host arrays.
 */
typedef struct rg_s2_bt_chr {
  const double* gamma_sqrt_mask; /* [P][N]     m_est.Gamma_sqrt_mask                          */
  const double* gamma_sqrt;      /* [P][N]     m_est.Gamma_sqrt                               */
  const double* yres;            /* [P][N]     res = (Y - p) / Gamma_sqrt o mask              */
  const double* x_gamma;         /* [P][C][N]  m_est.X_Gamma (orthonormal basis of Gamma^1/2 X) */
  const double* y_raw;           /* [P][N]     phenotypes_raw (0/1)                           */
  const double* firth_offset;    /* [P][N]     firth_est.cov_blup_offset (NULL without --firth) */
  const double* y_hat_p;         /* [P][N]     m_ests.Y_hat_p, fitted null probabilities (NULL without --spa) */
} rg_s2_bt_chr;
int rg_s2_set_chr_bt(rg_handle h, const rg_s2_bt_chr* st);

/*
 * rg_s2_block_bgen8_bt -- binary-trait score test for bs variants given as BGEN v1.2 layout-2 8-bit
 * probability rows (the inflated payload the reference parses in parseSnpfromBGEN, src/Geno.cpp:2186-2345):
 *   probs          [bs][n_file][2]  P(AA), P(AB) bytes per sample, in file order
 *   ploidy_missing [bs][n_file]     the ploidy/missingness bytes (bit 7 = missing), or NULL
 * Computes dosage, A1FREQ / INFO / N / MAC, flip_geno, mean imputation, check_sparse_G and compute_score_bt
 * (src/Step2_Models.cpp:470-556).  flags bit3 = allele flipped (beta already sign-corrected), bit4 = ignored
 * (sqrt(denum) < numtol).  info_out [bs x P].  The block stays resident for rg_s2_firth.
 * sample_idx [host|device] as in rg_l0_block_bed.
 */
int rg_s2_block_bgen8_bt(rg_handle h, const uint8_t* probs, const uint8_t* ploidy_missing, int64_t n_file,
                         int32_t bs, const int32_t* sample_idx, int32_t ref_first, double min_mac,
                         const rg_s2_out* out, double* info_out);

/*
 * rg_s2_spa -- saddlepoint approximation for selected (variant, trait) pairs of the resident block; replaces
 * run_SPA_test_snp / solve_K1_snp / get_SPA_pvalue_snp (src/Step2_Models.cpp:2072-2294, fast variant for sparse
 * genotypes included).  pval = sum of the two tail probabilities; the caller finishes like check_pval_snp
 * (:2021-2029): chisq = chi2_1 quantile of max(pval, 10 DBL_MIN), SE = 1/sqrt(G'WG), beta = sign(z) sqrt(chisq) SE.
 * status & 15 != 0: the test failed (TEST_FAIL).
 */
int rg_s2_spa(rg_handle h, int32_t n_sel, const int32_t* variant_idx, const int32_t* trait_idx, double* pval,
              int32_t* status);

/*
 * rg_s2_block_bgen8 -- the quantitative-trait score test of rg_s2_block_bed (after rg_s2_set_chr) on BGEN
 * 8-bit probability rows: parseSnpfromBGEN dosages + INFO (src/Geno.cpp:2186-2345) then check_sparse_G,
 * residualize_geno and compute_score_qt (src/Step2_Models.cpp:343-467).  No allele flip for QTs (with_flip is
 * false for trait_mode 0, src/Data.cpp:2108).  sample_idx [host|device] as in rg_l0_block_bed.
 */
int rg_s2_block_bgen8(rg_handle h, const uint8_t* probs, const uint8_t* ploidy_missing, int64_t n_file,
                      int32_t bs, const int32_t* sample_idx, int32_t ref_first, double min_mac,
                      const rg_s2_out* out, double* info_out);

/*
 * rg_bgen_inflate -- inflate the zlib payloads of `bs` BGEN v1.2 variants on the device.  Replaces the host-side
 * `uncompress` of the reference's BGEN parsers (src/Geno.cpp:1608, :2207): one warp per variant stream, then the payload
 * header check (N, K = 2, ploidy 2..2, unphased, 8 bits - the subset src/Geno.cpp:2122-2170 handles) and the split into the
 * two arrays the dosage entry points take.
 *   comp       the compressed bytes (host or device); stream v is comp[comp_offs[v] .. comp_offs[v+1]): the C-4 bytes
 *              that follow the 4-byte uncompressed-length field D of the variant's genotype block, D == 10 + 3 n_file
 *   comp_offs  [bs + 1] byte offsets into comp (host)
 *   probs_dev / miss_dev   out: DEVICE pointers owned by the handle, valid until the next rg_bgen_inflate /
 *              rg_s2_block_bgen8[_bt] call with host buffers: [bs][n_file][2] probability bytes and [bs][n_file] ploidy
 *              bytes (bit 7 = missing); pass them to rg_s2_block_bgen8 / rg_s2_block_bgen8_bt as they are
 * Fails (with the variant's index in rg_last_error) on a corrupt stream, an Adler-32 mismatch or an unsupported layout.
 */
int rg_bgen_inflate(rg_handle h, const uint8_t* comp, const uint64_t* comp_offs, int64_t n_file, int32_t bs,
                    const uint8_t** probs_dev, const uint8_t** miss_dev);

/*
 * rg_s2_block_bed_bt -- the same binary-trait score test on 2-bit PLINK rows (.bed / decoded .pgen hard calls):
 * parseSnpfromBed (src/Geno.cpp:2414-2536) + compute_score_bt.  The block stays resident for rg_s2_firth / rg_s2_spa.
 * sample_idx [host|device] as in rg_l0_block_bed.
 */
int rg_s2_block_bed_bt(rg_handle h, const uint8_t* packed, int64_t row_stride, int32_t bs, const int32_t* sample_idx,
                       int32_t ref_first, double min_mac, const rg_s2_out* out);

/*
 * rg_s2_firth -- approximate Firth test for selected (variant, trait) pairs of the resident block; replaces
 * fit_firth_logistic_snp_fast + fit_firth_pseudo / fit_firth (src/Step2_Models.cpp:1158-1252, 1527-1737).
 * beta is reported on the original allele coding; status != 0 in the low 4 bits = did not converge.
 * The resident block (here and for rg_s2_spa) is that of the last block call if it was a binary-trait route and no
 * rg_s2_set_chr_bt came after it; without one the call fails.
 */
int rg_s2_firth(rg_handle h, int32_t n_sel, const int32_t* variant_idx, const int32_t* trait_idx, double* beta,
                double* se, double* lrt, int32_t* status);

/* ------------------------------------------------------------------ Step 2 (QT): GxE interaction tests */
/*
 * Per-chromosome state of the interaction tests with a quantitative variable E (--interaction VAR, E kept as a
 * covariate: regenie's default gwas_condtl).  Takes effect for the blocks run after it on a handle that has had
 * rg_s2_set_chr; the robust route reads the residuals and the covariate basis of rg_s2_set_chr.
 *   E          [N]        pheno_data.interaction_cov (raw values, 0 outside the analysis)
 *   n_px       K          columns of the HLM projection Px (0 = no HLM state: every variant takes the robust route)
 *   dinv_sqrt  [P][N]     HLM Dinv_sqrt = exp(-V beta / 2) o mask                         (src/HLM.cpp:224)
 *   px         [P][K][N]  orthonormal basis of Dinv_sqrt o X_hlm                         (src/HLM.cpp:225-229)
 *   yres       [P][N]     Dinv_sqrt o y - Px Px^T (Dinv_sqrt o y)                        (src/HLM.cpp:232, :236-243)
 */
typedef struct rg_s2_int_chr {
  const double* E;
  int32_t n_px;
  const double* dinv_sqrt;
  const double* px;
  const double* yres;
} rg_s2_int_chr;
int rg_s2_set_interaction(rg_handle h, const rg_s2_int_chr* st);

/* options of rg_s2_interaction (src/Regenie.cpp: --rare-mac, --force-robust, --force-hc4, --no-robust, --minMAC) */
typedef struct rg_s2_int_opts {
  double rare_mac;       /* params.rareMAC_inter (default 1000)                                   */
  double min_mac;        /* params.min_MAC: a trait with MAC below it is ignored (no rows)         */
  int32_t force_robust;  /* params.force_robust                                                   */
  int32_t force_hc4;     /* params.force_hc4 (HC4 for traits with MAC <= rare_mac)                */
  int32_t no_robust;     /* params.no_robust (model-based SE)                                     */
} rg_s2_int_opts;

/*
 * rg_s2_interaction -- the interaction model of every (variant, trait) pair of the block left resident by the last
 * rg_s2_block_bed / rg_s2_block_bgen8 call (get_interaction_terms + apply_interaction_tests_qt / _HLM,
 * src/Interaction.cpp:44-92, :109-437).  That call must be the last block call on the handle and must have run after
 * rg_s2_set_interaction on the current chromosome (rg_s2_block_bed writes the per-sample genotype words this call reads
 * only then); otherwise the call fails.  Per variant the route is HLM when any trait has MAC < rare_mac and the HLM
 * state is set (unless force_robust or no_robust), the robust sandwich otherwise.  Outputs are host arrays, variant-major:
 *   status [bs][P]     0 = no interaction rows (variant or trait ignored, or resid(E o G) has sd < numtol),
 *                      1 = robust route, 2 = HLM route, -1 = H^T H (robust) or Xres^T Xres (HLM) is near-singular
 *   coef   [bs][P][2]  (beta_G, beta_GxE), on the phenotype scale of the printed rows
 *   vcov   [bs][P][4]  their 2 x 2 covariance (row-major), on the same scale
 */
int rg_s2_interaction(rg_handle h, const rg_s2_int_opts* opts, int32_t* status, double* coef, double* vcov);

/* ------------------------------------------------------------------ Step 2 (BT): GxE interaction tests */
/*
 * Per-chromosome state of the interaction tests of binary traits with a quantitative variable E (--interaction VAR, E
 * kept as a covariate).  Call it after rg_s2_set_chr_bt; the next rg_s2_set_chr_bt clears it.  As in the reference, E and
 * E^2 join the covariates of a binary-trait run (src/Pheno.cpp:91-95, :1073-1076), so the X of rg_step2_create must be
 * the basis of [covariates, E, E^2].
 *   E       [N]     pheno_data.interaction_cov (raw values; only the analysed samples are read)
 *   offset  [P][N]  m_ests.offset_nullreg: linear predictor of each trait's null logistic fit with its LOCO offset
 *                   (src/Step1_Models.cpp:63, :135)
 */
typedef struct rg_s2_int_bt_chr {
  const double* E;
  const double* offset;
} rg_s2_int_bt_chr;
int rg_s2_set_interaction_bt(rg_handle h, const rg_s2_int_bt_chr* st);

/*
 * rg_s2_interaction_bt -- the logistic interaction model of every (variant, trait) pair of the block left resident by
 * the last rg_s2_block_bed_bt / rg_s2_block_bgen8_bt call (get_interaction_terms + apply_interaction_tests_bt,
 * src/Interaction.cpp:44-92, :441-678): H = [G_res / scale_fac, resid(E o G) / scf_i] in the minor-allele coding,
 * fit_logistic from beta = 0 with offset_nullreg (check_hs_dev on, then off), V = (H^T W H)^-1, and the HC3 sandwich when
 * robust SEs are forced, or unless no_robust, for traits with MAC > rare_mac where either Wald p-value is below 0.05.
 * opts.force_hc4 is not used for binary traits.  Outputs are host arrays, variant-major:
 *   status [bs][P]     0 = no interaction rows (variant or trait ignored, or resid(E o G) or G_res has sd < numtol),
 *                      1 = robust (HC3) SEs, 3 = model-based SEs, -1 = H^T W H near-singular or a negative robust
 *                      variance, -2 = the logistic regression failed
 *   coef   [bs][P][2]  (beta_G, beta_GxE) on the scale of the printed rows (divided by scale_fac, scf_i), sign-corrected
 *                      for flipped alleles
 *   vcov   [bs][P][4]  their 2 x 2 covariance (row-major), on the same scale
 * ADD-INT_SNP and ADD-INT_SNPxVAR are beta / sqrt(vcov diagonal) Wald tests, ADD-INT_2DF is coef^T vcov^-1 coef (2 df).
 */
int rg_s2_interaction_bt(rg_handle h, const rg_s2_int_opts* opts, int32_t* status, double* coef, double* vcov);

/*
 * rg_s2_interaction_firth -- the Firth fallback of the interaction tests (--firth, for pairs whose GxE Wald p-value is
 * at most pThresh; apply_interaction_tests_firth, src/Interaction.cpp:680-863) for selected (variant, trait) pairs.
 * Needs rg_s2_interaction_bt on the resident block and the null-Firth offsets (rg_s2_bt_chr.firth_offset).  Three
 * penalised fits (fit_firth_nr, src/Step2_Models.cpp:1267-1383, with the offsets): both columns from 0, G dropped from
 * (0, beta_GxE), GxE dropped from (beta_G, 0).  Outputs per pair, host arrays:
 *   coef [n][2], se [n][2]  of the full fit, on the printed scale, sign-corrected for flipped alleles
 *   lrt  [n][3]             ADD-INT_2DF = dev0 - dev (2 df), ADD-INT_SNP and ADD-INT_SNPxVAR = dev_dropped - dev (1 df)
 *   status [n]              0 = rows, 1 / 2 / 3 = the full / G-dropped / GxE-dropped fit failed, 4 = a negative LRT,
 *                           5 = the variant has no interaction rows; any non-zero status means no rows for the pair
 */
int rg_s2_interaction_firth(rg_handle h, int32_t n_sel, const int32_t* variant_idx, const int32_t* trait_idx,
                            double* coef, double* se, double* lrt, int32_t* status);

/* ------------------------------------------------------------------ PGEN records (SURVEY 8 (f)3) */
/*
 * rg_pgen_decode -- the variant records of one block of a PLINK 2 .pgen (hard calls), decoded ON THE DEVICE into
 * PLINK 1 2-bit rows (ALT count 0 / 1 / 2 / missing -> codes 11 / 10 / 00 / 01, ref-last).  Replaces the per-variant
 * pgenlib reads of the reference: PgenReader::Read in readChunkFromPGENFileToG (src/Geno.cpp:1773-1821, Step 1) and in
 * readChunkFromPGENFileToG / parseSnpfromPGEN of Step 2 (src/Geno.cpp:2538-2594, :2596-2712).  The caller only slices
 * the file: it passes the bytes of the records as they are (record types 0-7: plain 2-bit, 1 bit + difflist, difflist
 * over a constant, LD-compressed against an earlier record), the device expands them (csrc/pgen_decode.cu).
 *   bytes      [host] the records the block needs (own records and the bases of LD-compressed ones), each starting at a
 *              multiple of 4 bytes: record r is bytes[rec_off[r] .. rec_off[r] + rec_len[r])
 *   rec_type   [n_rec] low 3 bits of the variant record type
 *   own        [bs] record index of variant j of the block;  base [bs] record index of the most recent record that is
 *              not LD-compressed when own[j] is of type 2 / 3, -1 otherwise
 *   n_file     samples in the file (rows are in file order: pass sample_idx to the block call as for a .bed)
 *   block_id   only used in error messages
 *   rows_dev / row_stride   out: DEVICE pointer to bs rows and their stride in bytes (>= ceil(n_file / 4)); pass both
 *              to rg_l0_block_bed / rg_s2_block_bed / rg_s2_block_bed_bt as `packed` / `row_stride`.
 * Step-1 handle: asynchronous, on the stream of the lane that the NEXT rg_l0_block_bed call uses - that call must be
 * the consumer; a malformed record is reported by rg_l0_status / rg_sync like a low-variance SNP.  Step-2 handle: returns
 * after the decode, errors at once; the rows stay valid until the next rg_pgen_decode on the handle.
 */
typedef struct rg_pgen_block {
  const uint8_t* bytes;
  int64_t n_bytes;
  const uint64_t* rec_off;
  const uint32_t* rec_len;
  const uint8_t* rec_type;
  int32_t n_rec;
  const int32_t* own;
  const int32_t* base;
  int32_t bs;
  int64_t n_file;
  int32_t block_id;
} rg_pgen_block;
int rg_pgen_decode(rg_handle h, const rg_pgen_block* blk, const uint8_t** rows_dev, int64_t* row_stride);

/* ------------------------------------------------------------------ multi-GPU */
/*
 * One process per GPU. Level-0 blocks are sharded across ranks (the reference's --split-l0 partition,
 * src/Data.cpp:268-301); level 1 is sharded by phenotype.  Instead of a separate exchange step, every rank
 * maps the predictor matrix W of the phenotype owners into its address space (CUDA IPC over NVLink/NVSwitch):
 *   all:    rg_W_set_owned(h, owned)           -> local W storage only for the phenotypes this rank fits (N x B x P/nranks)
 *   owner:  rg_W_export(h, handle)             -> 64-byte cudaIpcMemHandle_t of its W allocation
 *   peers:  rg_W_attach_peer(h, handle, owned) -> level-0 kernels of this rank store the W tiles of every
 *                                                 phenotype with owned[p] != 0 (the mask the peer passed to
 *                                                 rg_W_set_owned) directly into the owner's HBM
 * After all ranks have finished level 0 (rg_sync + a barrier in the caller), each owner holds the complete
 * N x B matrix of its phenotypes and runs rg_l1_fit / rg_l1_fit_bt / rg_loco, which skip phenotypes that
 * were handed to a peer (rg_l1_select overrides the selection).  No collective is on the data path.
 */
int rg_W_set_owned(rg_handle h, const uint8_t* owned);
int rg_W_export(rg_handle h, void* ipc_handle_64);
int rg_W_attach_peer(rg_handle h, const void* ipc_handle_64, const uint8_t* owned_by_peer);
int rg_l1_select(rg_handle h, const uint8_t* selected);

/* Number of level-0 predictor columns held locally; W of other ranks is attached with
 * rg_l1_attach_W before rg_l1_fit (the exchange itself is done by the caller with NCCL). */
int rg_W_info(rg_handle h, int32_t ph, void** dev_ptr, int64_t* ld, int64_t* ncols);

/* Same redirection as rg_W_attach_peer for a peer handle that lives in THIS process on another GPU (one host thread per
 * GPU, rgb200 --gpus N): peer access is enabled from h's device to peer's device and the entries of the phenotypes
 * `owned_by_peer` marks point straight at the peer's W allocation (no CUDA IPC: an IPC handle cannot be opened by the
 * process that exported it).  Both handles must have had rg_W_set_owned called with their own masks. */
int rg_W_attach_local(rg_handle h, rg_handle peer, const uint8_t* owned_by_peer);

/* ------------------------------------------------------------------ test / profiling hooks */
/* Copy a named intermediate of the last level-0 block or level-1 fit ("l1_*"), or of the last Step-2 block on a Step-2
 * handle, to the host (tests only).  Returns the number of bytes written, or <0 on error.  See DESIGN.md for names. */
int64_t rg_debug_fetch(rg_handle h, const char* name, void* out, int64_t max_bytes);
/* Level-0 ridge solver bookkeeping: blocks whose K*R systems were solved by the tensor-core factorisation + FP64
 * iterative refinement (csrc/chol_mixed.cu), and how many of those raised the convergence flag and were re-solved
 * by the FP64 Cholesky.  RG_B200_SOLVER=f64 selects the FP64 path for every block. */
int rg_l0_solver_stats(rg_handle h, int64_t* mixed_blocks, int64_t* f64_fallbacks);
/* Test hook for the mixed-precision solver alone: solves (Af[f] + lambda[r] I) x = b[f] for all K*R pairs
 * (system index f*R + r) on `device`.  All pointers are host memory: Af [K][n][n] full symmetric FP64, lambda [R],
 * b [K][P][n]; x_out [K*R][P][n]; X_out (optional) [K*R][n][n] FP32: the off-diagonal tiles of the Cholesky factors
 * (diagnostic only); fail_out: 0 = every system
 * met `tol` within `steps` corrections.  n must be 128 * 2^k <= 2048. */
int rg_dbg_mixed_solve(int32_t device, int32_t n, int32_t K, int32_t R, int32_t P, const double* Af,
                       const double* lambda, const double* b, int32_t steps, double tol, double* x_out,
                       float* X_out, uint32_t* fail_out);
/* Number of kernels launched by this handle since creation (for bench.py gpu_launches). */
int64_t rg_launch_count(rg_handle h);
/* CUDA stream of the handle as a void* (cudaStream_t), so callers can record events. */
void* rg_stream(rg_handle h);
/* Accumulated device time (ms) of the tensor-core Gram kernel, measured with CUDA events on
 * the handle's stream when timing is enabled. */
int rg_set_timing(rg_handle h, int32_t enable);
int rg_get_timing(rg_handle h, const char* kernel, double* total_ms, int64_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* RG_B200_H */
