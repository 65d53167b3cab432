// Out-of-fold level-0 predictions on the tensor cores, exactly.
//
//   pred[t, q] = sum_i gamma[i,q] g0(i,t) + sum_i (gamma mu)[i,q] miss(i,t) - x_t . cvec_q
// (reference: `beta.transpose() * Gmat.block(...)`, src/Step1_Models.cpp:503 - 2 P R bs N flops/block).
// The genotype operand is the plane pair [G0; Miss] of the Gram kernel (8 x dosage and 8 x missing as int8), built in
// registers from the block's padded 2-bit rows: one 32-bit word holds both planes of 16 samples, an eighth of the bytes
// of the int8 planes.  The real-valued coefficients
// are split into FIVE balanced radix-254 digits
//   gamma[i,q] = (s_q / 127) * sum_l d_l[i,q] 254^-l,   d_l in {-127..127}  (int8),
// so the s8 x s8 -> s32 MMAs accumulate exact integer sums (|sum| <= K2 * 16 * 127 < 2^24 for K2 <= 4096) and the FP64
// epilogue reassembles the prediction to s_q 254^-5 = 9.4e-13 s_q per coefficient (the last limb is rounded to within 1/2,
// and one unit of it is worth (s_q / 127) 254^-4), far inside the 1e-5 parity budget.
//
// Orientation: samples are the MMA M dimension, the 5 x 50 digit rows are N (256, zero padded), the SNP/plane index
// is K: all G0 k-blocks, then all Miss k-blocks (the same 2-bit tiles again, mostly from L2).  The digit rows are K-major
// in shared memory (wgmma B operand); the A operand comes from registers.  Each consumer warpgroup owns one 64-sample
// half of the tile and all 256 digit rows (m64n256k32).  A warp's 16 samples are one 2-bit word of each SNP row: a thread
// loads the words of the 8 k rows of its fragment, keeps the nibble of its two samples from each and turns the codes into
// plane bytes with a few bit operations.  The fragments of MMA u + 1 are built while MMA u runs.
// The epilogue also leaves per-tile column sums (sum, sum of squares) of the raw predictions for the standardisation.
#include <stdlib.h>

#include <algorithm>
#include <atomic>

#include "kernels.cuh"
#include "wgmma_sm90.cuh"

namespace rg {

namespace {

using namespace sm90;

constexpr int PT_BM = 128;            // samples per CTA
constexpr int PT_BK = 128;            // SNP rows of one plane per stage
constexpr int PI_BN = 256;            // digit rows (5 limbs x 50 outputs, zero padded)
constexpr int PI_STAGES = 4;
constexpr int PI_A_WORDS = PT_BM / 16;             // 2-bit words per SNP row of a sample tile
constexpr int PI_A_BYTES = PT_BK * PI_A_WORDS * 4; // 4 KiB: 128 SNP rows x 128 samples of 2-bit codes
constexpr int PI_B_BYTES = PI_BN * PT_BK;          // 32 KiB: 256 digit rows x 128 k bytes
constexpr int PI_STAGE_BYTES = PI_A_BYTES + PI_B_BYTES;
constexpr int PI_THREADS = 384;                    // 2 MMA warpgroups (samples 0-63 / 64-127), 1 epilogue warpgroup
constexpr int PI_LDV = PT_BM + 1;                  // row stride (double) of the handoff tile V[output][sample]
constexpr int PI_EG = 10;                          // outputs per group of independent chains in the epilogue
constexpr int PI_MAX_ROWS = 2048;                  // rows_p bound of the INT8 route (2 rows_p <= 4096)
// the handoff's limb walk: limb l of output q is column q + 50 l, and 50 = 6 x 8 + 2 moves it one quad lane per limb
static_assert(kLimbsI8 == 5 && kLimbQI8 == 50 && kLimbsI8 * kLimbQI8 <= PI_BN, "INT8 prediction layout");
static_assert(kLimbQI8 % PI_EG == 0, "epilogue output groups");

}  // namespace

// Everything the INT8 prediction needs from the solution column of one output q = r P + p and fold f, in one CTA:
//   gam[f][i][q] = beta[m=(f,r)][p][i] * inv_sd[i],  gmu = gam * mu   (rows bs..rows_p zero),
//   cvec[f][q][c] = sum_i gam[f][i][q] Bv[i][c]                       (256-thread stride loop, fixed-order tree),
//   scale[f][q] = s = the largest |gam|, |gmu| of the column (1 if it is all zero),
//   dig[f][g][l*50 + qq][k] = the balanced radix-254 digits l of 127 v / s, v = gam (k < rows_p) or gmu (k >= rows_p).
// The values, the order of every sum and the digits are those of l0_gamma_kernel + l0_cvec_kernel, which the FP64 route
// still runs.  grid: (Q, K folds), block 256.
__global__ void __launch_bounds__(256)
l0_coef_i8_kernel(const double* __restrict__ cm, int64_t cm_stride, int ldc, int nC, int R, int P, int Qp, int bs,
                  int rows_p, const double* __restrict__ mu, const double* __restrict__ inv_sd,
                  const double* __restrict__ Bv, int C, double* __restrict__ gam, double* __restrict__ gmu,
                  double* __restrict__ cvec, double* __restrict__ scale, uint8_t* __restrict__ dig, int ngroups) {
  __shared__ double sg[PI_MAX_ROWS], sm[PI_MAX_ROWS];
  __shared__ double red[256];
  const int q = blockIdx.x, f = blockIdx.y;
  const int r = q / P, p = q % P;
  const double* x = cm + (int64_t)(f * R + r) * cm_stride + (int64_t)(nC + p) * ldc;
  double* gcol = gam + (int64_t)f * rows_p * Qp + q;
  double* mcol = gmu + (int64_t)f * rows_p * Qp + q;
  double mx = 0.0;
  for (int i = threadIdx.x; i < rows_p; i += 256) {
    const double v = i < bs ? x[i] * inv_sd[i] : 0.0;
    const double vm = v * mu[i];
    gcol[(int64_t)i * Qp] = v;
    mcol[(int64_t)i * Qp] = vm;
    sg[i] = v;
    sm[i] = vm;
    if (i < bs) mx = fmax(mx, fmax(fabs(v), fabs(vm)));
  }
  for (int c = 0; c < C; ++c) {
    double s = 0.0;
    for (int i = threadIdx.x; i < bs; i += 256) s += sg[i] * Bv[(int64_t)i * C + c];
    s = cta_tree<256>(s, red);
    if (threadIdx.x == 0) cvec[((int64_t)f * Qp + q) * C + c] = s;
  }
  mx = cta_tree<256, CtaOp::kMax>(mx, red);
  const double s = mx > 0.0 ? mx : 1.0;
  if (threadIdx.x == 0) scale[(int64_t)f * Qp + q] = s;
  const int g = q / kLimbQI8, qq = q % kLimbQI8;
  const int K2 = 2 * rows_p;
  uint8_t* base = dig + ((int64_t)f * ngroups + g) * (int64_t)PI_BN * K2;
  for (int k = threadIdx.x; k < K2; k += 256) {
    const int plane = k >= rows_p, i = plane ? k - rows_p : k;
    double v = 0.0;
    if (i < bs) v = (plane ? sm[i] : sg[i]) / s * 127.0;
#pragma unroll
    for (int l = 0; l < kLimbsI8; ++l) {
      const double d = rint(v);                    // |v| <= 127: the remainder (<= 1/2) x 254 stays in range
      base[(int64_t)(l * kLimbQI8 + qq) * K2 + k] = (uint8_t)(int8_t)(int)d;
      v = (v - d) * 254.0;
    }
  }
}

// Persistent: grid = min(items, SMs), items = (sample tile, q group) pairs, item = tile * ngroups + g, and CTA b runs
// items b, b + grid, b + 2 grid, ...  384 threads: warpgroups 0 and 1 run the MMAs of an item (one 64-sample half each)
// and keep the stage ring full themselves, warpgroup 2 runs the epilogue of the previous item meanwhile.
//   - ring: the k-blocks of all of a CTA's items form one sequence it = k nkb + kb over PI_STAGES stages.  Each MMA
//     warpgroup counts its release of a stage in rel[s]; the second of the two loads k-block it + PI_STAGES into it, so
//     the next item's first stages are in flight while this item's last MMAs run, and nothing ever waits for a stage
//     to empty.
//   - handoff: after its last MMA of an item, an MMA warpgroup reduces the five limbs of each output to the FP64 Horner
//     sum (the limbs of output q sit in columns q + 50 l, spread over the four threads of a quad) and writes it to
//     V[q][sample], which does not alias the stages; arrivals on hfull publish V, the epilogue's arrivals on hfree
//     give it back.
//   - epilogue: thread = sample, all 50 outputs: scale, covariate correction, mask, store to W, then the tile's column
//     sums (sum, sum of squares) from V in sample order, the two 64-sample halves added.  It loads the item's scales,
//     cvec, W columns, mask bytes and covariates before it waits for V.
__global__ void __launch_bounds__(PI_THREADS, 1)
l0_predict_i8_kernel(const __grid_constant__ CUtensorMap tmG, const __grid_constant__ CUtensorMap tmD, PredictTcArgs a,
                     int ntiles) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gen_base = smem_raw + (base - raw);
  const uint32_t sB = base;                                         // [NST][32 KiB], 1 KiB aligned (128B swizzle)
  const uint32_t sA = base + PI_STAGES * PI_B_BYTES;                // [NST][4 KiB]
  uint64_t* bars = reinterpret_cast<uint64_t*>(gen_base + PI_STAGES * PI_STAGE_BYTES);
  const uint32_t full_bar = smem_u32(bars);                         // [NST]
  const uint32_t hfull = smem_u32(bars + PI_STAGES);
  const uint32_t hfree = smem_u32(bars + PI_STAGES + 1);
  uint32_t* rel = reinterpret_cast<uint32_t*>(bars + PI_STAGES + 2);   // [NST] stage releases
  double* V = reinterpret_cast<double*>(gen_base + PI_STAGES * PI_STAGE_BYTES + 128);   // [kLimbQI8][PI_LDV]
  double* Vs = V + kLimbQI8 * PI_LDV;                                  // [2 sample halves][kLimbQI8][2]
  double* s_scale = Vs + 4 * kLimbQI8;                                 // [kLimbQI8]
  double* s_cvec = s_scale + kLimbQI8;                                 // [kLimbQI8][C]
  double** s_dst = reinterpret_cast<double**>(s_cvec + kLimbQI8 * a.C);                     // [kLimbQI8] W columns
  const uint8_t** s_msk = reinterpret_cast<const uint8_t**>(s_cvec + kLimbQI8 * (a.C + 1));  // [kLimbQI8] mask rows

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role
  const int nk = (ntiles * a.ngroups - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // items of this CTA
  const int nkh = a.rows_p / PT_BK;                 // k-blocks per plane
  const int nkb = 2 * nkh;
  auto item_of = [&](int k) { return (int)blockIdx.x + k * (int)gridDim.x; };

  if (threadIdx.x == 0) {
    for (int s = 0; s < PI_STAGES; ++s) { mbar_init(full_bar + 8 * s, 1); rel[s] = 0; }
    mbar_init(hfull, 256);
    mbar_init(hfree, 128);
    fence_barrier_init();
    prefetch_tmap(&tmG);
    prefetch_tmap(&tmD);
  }
  __syncthreads();

  if (warp >= 8) {
    // ===== epilogue warpgroup: gives 16 of its 168 registers per thread to the MMA warpgroups =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 152;\n" ::: "memory");
    const int ct = threadIdx.x - 256;               // sample of the tile
    for (int k = 0; k < nk; ++k) {
      const int tile = item_of(k) / a.ngroups, g = item_of(k) % a.ngroups;
      const int f = a.tile_fold[tile];
      const int q0 = g * kLimbQI8;
      const int nq = min(kLimbQI8, a.Q - q0);
      // the previous item's readers of these are past its last named barrier
      for (int e = ct; e < kLimbQI8; e += 128) {
        const int q = q0 + e, r = q / a.P, p = q % a.P;
        s_scale[e] = (e < nq) ? a.scale[(int64_t)f * a.Qp + q] / 127.0 : 0.0;
        s_dst[e] = (e < nq) ? a.W[p] + (int64_t)(a.col0 + r) * a.npad : nullptr;
        s_msk[e] = (e < nq) ? a.mask + (int64_t)p * a.npad : nullptr;
      }
      for (int e = ct; e < kLimbQI8 * a.C; e += 128) {
        const int qq = e / a.C, c = e % a.C;
        s_cvec[e] = (qq < nq) ? a.cvec[((int64_t)f * a.Qp + q0 + qq) * a.C + c] : 0.0;
      }
      named_sync(1, 128);
      const int t = tile * PT_BM + ct;
      // every global load of the epilogue is issued here, ahead of the stores below, so that the 50 mask rows cost one
      // memory latency rather than one each (the compiler may not move a load across a store through another pointer)
      uint32_t mk[kLimbQI8];
#pragma unroll
      for (int j = 0; j < kLimbQI8; ++j) mk[j] = (j < nq) ? s_msk[j][t] : 0u;
      double xr[kMaxCov];
      for (int c = 0; c < a.C; ++c) xr[c] = a.xy[(int64_t)t * a.cpp + c];
      mbar_wait(hfull, k & 1);
      // outputs in groups of PI_EG, the covariates outermost inside a group: the same operations per output, in the
      // same order, as independent chains
#pragma unroll
      for (int j0 = 0; j0 < kLimbQI8; j0 += PI_EG) {
        double val[PI_EG];
#pragma unroll
        for (int j = 0; j < PI_EG; ++j) val[j] = V[(j0 + j) * PI_LDV + ct] * s_scale[j0 + j];
        for (int c = 0; c < a.C; ++c) {
#pragma unroll
          for (int j = 0; j < PI_EG; ++j) val[j] -= xr[c] * s_cvec[(j0 + j) * a.C + c];
        }
#pragma unroll
        for (int j = 0; j < PI_EG; ++j) {
          const int qq = j0 + j;
          double v = 0.0;
          if (qq < nq) {
            v = val[j] * (double)mk[qq];
            s_dst[qq][t] = v;
          }
          V[qq * PI_LDV + ct] = v;
        }
      }
      named_sync(1, 128);
      if (ct < 2 * kLimbQI8) {
        const int qq = ct % kLimbQI8, sh = ct / kLimbQI8;
        const double* v = V + qq * PI_LDV + sh * (PT_BM / 2);
        double s1 = 0.0, s2 = 0.0;
#pragma unroll 8
        for (int i = 0; i < PT_BM / 2; ++i) {
          s1 += v[i];
          s2 = fma(v[i], v[i], s2);
        }
        Vs[(sh * kLimbQI8 + qq) * 2 + 0] = s1;
        Vs[(sh * kLimbQI8 + qq) * 2 + 1] = s2;
      }
      named_sync(1, 128);
      mbar_arrive(hfree);                           // V is read: the MMA warpgroups may write the next item's
      if (ct < nq) {
        a.part[((int64_t)tile * a.Qp + q0 + ct) * 2 + 0] = Vs[ct * 2 + 0] + Vs[(kLimbQI8 + ct) * 2 + 0];
        a.part[((int64_t)tile * a.Qp + q0 + ct) * 2 + 1] = Vs[ct * 2 + 1] + Vs[(kLimbQI8 + ct) * 2 + 1];
      }
    }
    return;
  }

  // ===== MMA warpgroups: warpgroup wg = samples 64 wg .. 64 wg + 63 x all 256 digit rows =====
  // Thread (warp w of the warpgroup, lane l, r = l / 4, t4 = l % 4) holds fragment rows r and r + 8 of its warp's 16,
  // which are the samples 2 r and 2 r + 1 of the warp's 16 (from 64 wg + 16 w): the nibble at bit 4 r of word 4 wg + w
  // of each SNP row.  Its k are the quads 4 t4 .. +3 and 16 + 4 t4 .. +3 of each MMA's 32.  At load j, lane t4 reads row
  // 4 t4 + (j + t4) % 4 of its quad, so the four t4 of an instruction meet four distinct banks and the eight lanes of
  // each t4 read one word (broadcast); qsel undoes the rotation.
  asm volatile("setmaxnreg.inc.sync.aligned.u32 176;\n" ::: "memory");
  const int wg = warp >> 2, w = warp & 3, r = lane >> 2, t4 = lane & 3;
  const bool leader = w == 0 && lane == 0;
  // Ring cursor of the leaders (both track it; the second releaser of a stage issues): item ck, k-block ckb, the fold
  // of item ck and, loaded one item ahead, of item ck + 1.
  int ck = 0, ckb = 0, cf = 0, cfn = 0;
  if (leader) {
    cf = a.tile_fold[item_of(0) / a.ngroups];
    if (nk > 1) cfn = a.tile_fold[item_of(1) / a.ngroups];
  }
  // A = 128 SNP rows x 8 words (128 samples) of 2-bit codes, the G0 rows and then the same rows for the Miss plane;
  // B = 256 digit rows x 128 k bytes
  auto refill = [&](bool issue) {
    if (ck >= nk) return;
    if (issue) {
      const int s = (ck * nkb + ckb) % PI_STAGES;
      const uint32_t fb = full_bar + 8 * s;
      const int drow0 = (cf * a.ngroups + item_of(ck) % a.ngroups) * PI_BN;
      mbar_expect_tx(fb, PI_STAGE_BYTES);
      tma_load_2d(sA + s * PI_A_BYTES, &tmG, fb, (item_of(ck) / a.ngroups) * PI_A_WORDS, (ckb % nkh) * PT_BK);
      tma_load_2d(sB + s * PI_B_BYTES, &tmD, fb, ckb * PT_BK, drow0);
      tma_load_2d(sB + s * PI_B_BYTES + 16384, &tmD, fb, ckb * PT_BK, drow0 + 128);
    }
    if (++ckb == nkb) {
      ckb = 0;
      ++ck;
      cf = cfn;
      if (ck + 1 < nk) cfn = a.tile_fold[item_of(ck + 1) / a.ngroups];
    }
  };
  // this warpgroup's MMAs have read stage it % PI_STAGES for the last time in round it
  auto release = [&](int it) {
    if (leader) refill(atomicAdd(&rel[it % PI_STAGES], 1u) & 1u);
  };
  if (leader) {
    for (int s = 0; s < PI_STAGES; ++s) refill(wg == 0);
  }

  int aoff[4];                                      // byte offset of load j inside a 16-row quad slice of the A stage
  uint32_t qsel = 0;                                // byte k of a quad comes from load (k - t4) % 4
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    aoff[j] = (4 * t4 + ((j + t4) & 3)) * (PI_A_WORDS * 4) + (4 * wg + w) * 4;
    const int src = (j - t4) & 3;                   // for byte k = j
    qsel |= (uint32_t)((src & 1) | ((src >> 1) << 2)) << (4 * j);
  }
  const uint32_t bsel = (uint32_t)(r >> 1) | ((uint32_t)(4 + (r >> 1)) << 4);   // byte r / 2 of two words
  const int nsh = 4 * (r & 1);                                                   // nibble of that byte
  const uint8_t* gA = gen_base + PI_STAGES * PI_B_BYTES;   // generic view of the A stages

  // A fragment of MMA kk of stage s: {sample 2 r, 2 r + 1} x {k 4 t4 .. +3, k 16 + 4 t4 .. +3} of the stage's 32-k slice
  // kk, as the Gram kernel's plane bytes: G0 = 8 x code (0 for code 3), Miss = 8 x (code == 3).
  auto build = [&](int s, int kk, bool miss, uint32_t (&af)[4]) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint8_t* src = gA + s * PI_A_BYTES + (kk * 32 + 16 * h) * (PI_A_WORDS * 4);
      uint32_t t[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) t[j] = *reinterpret_cast<const uint32_t*>(src + aoff[j]);
      // byte k: the codes of samples 2 r (bits 0-1) and 2 r + 1 (bits 2-3) at k, other samples' codes above
      const uint32_t y = __byte_perm(__byte_perm(t[0], t[1], bsel), __byte_perm(t[2], t[3], bsel), qsel) >> nsh;
      const uint32_t c0 = y & 0x03030303u, c1 = (y >> 2) & 0x03030303u;
      const uint32_t m0 = c0 & (c0 >> 1), m1 = c1 & (c1 >> 1);     // 1 in the bytes of missing calls (code 3)
      af[2 * h] = miss ? m0 << 3 : (c0 ^ (m0 * 3u)) << 3;
      af[2 * h + 1] = miss ? m1 << 3 : (c1 ^ (m1 * 3u)) << 3;
    }
  };
  // One commit group per MMA, two fragment register sets: while MMA u runs, MMA u - 1 is retired (freeing its fragment
  // registers, and at the first MMA of a stage the previous stage's buffers) and the fragment of MMA u + 1 is built.
  // Double-buffering whole stages would need 32 fragment registers beside the 128 accumulators, more than the 176 an
  // MMA thread gets.
  int32_t acc[128];
  uint32_t afr[2][4];
  const double inv254 = 1.0 / 254.0;
  int it = 0;                                       // ring round of the current k-block
  for (int k = 0; k < nk; ++k) {
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0;
    fence_regs(acc);
    mbar_wait(full_bar + 8 * (it % PI_STAGES), (it / PI_STAGES) & 1);
    build(it % PI_STAGES, 0, false, afr[0]);
    for (int kb = 0; kb < nkb; ++kb, ++it) {
      const int s = it % PI_STAGES;
      const bool miss = kb >= nkh;
      const uint64_t db = desc_k128(sB + s * PI_B_BYTES);
#pragma unroll
      for (int kk = 0; kk < PT_BK / 32; ++kk) {
        wgmma_fence();
        // +32 bytes (K of one MMA) inside the 128-byte swizzle atom: +2 in 16-byte units
        wgmma_s8_rs_n256(acc, afr[kk & 1], db + (uint64_t)(2 * kk));
        wgmma_commit();
        wgmma_wait<1>();
        if (kk == 0 && kb > 0) release(it - 1);
        if (kk + 1 < PT_BK / 32) {
          build(s, kk + 1, miss, afr[(kk + 1) & 1]);
        } else if (kb + 1 < nkb) {
          mbar_wait(full_bar + 8 * ((it + 1) % PI_STAGES), ((it + 1) / PI_STAGES) & 1);
          build((it + 1) % PI_STAGES, 0, kb + 1 >= nkh, afr[0]);
        }
      }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    release(it - 1);

    // ===== handoff: V[q][sample] = FP64 Horner of the five limb sums (exact int32 multiples of 8) from the lowest limb
    // up.  Accumulator i of this thread is column 8 (i / 4) + 2 t4 + (i & 1) of sample 2 r + (i / 2) % 2.  The thread
    // forms the outputs q = 8 m + 2 t4 + b; limb l of q is column q + 50 l = 8 (m + 6 l + c) + 2 ((t4 + l) % 4) + b with
    // c = (t4 + l >= 4), held by quad lane (t4 + l) % 4, which (seen from that lane, t4' = (t4 + l) % 4) has c = (t4' < l).
    mbar_wait(hfree, (k & 1) ^ 1);
    const int smp0 = 64 * wg + 16 * w + 2 * r;
#pragma unroll
    for (int hb = 0; hb < 2; ++hb) {
#pragma unroll
      for (int m = 0; m < (kLimbQI8 + 7) / 8; ++m) {
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          int32_t e[kLimbsI8];
#pragma unroll
          for (int l = 0; l < kLimbsI8; ++l) {
            const int i0 = 4 * (m + 6 * l) + 2 * hb + b;
            if (l == 0) {
              e[l] = acc[i0];
            } else if (l == 4) {
              e[l] = acc[i0 + 4];
            } else {
              const int32_t sv = t4 < l ? acc[i0 + 4] : acc[i0];
              e[l] = __shfl_sync(0xffffffffu, sv, (lane & ~3) | ((t4 + l) & 3));
            }
          }
          double d = 0.0;
#pragma unroll
          for (int l = kLimbsI8 - 1; l >= 0; --l) d = fma(d, inv254, (double)(e[l] >> 3));
          const int q = 8 * m + 2 * t4 + b;
          if (q < kLimbQI8) V[q * PI_LDV + smp0 + hb] = d;
        }
      }
    }
    mbar_arrive(hfull);
  }
}

// Column sums of predictions that no prediction kernel summed (the dense route of l0_dense.cu): part[chunk][q] =
// (sum, sum of squares) over a chunk of 8192 samples, fixed-order tree reduction.  grid: (Q, nchunks), block 256.
__global__ void __launch_bounds__(256)
l0_colsum_kernel(double* const* __restrict__ W, int64_t npad, int col0, int P, int Qp,
                 double* __restrict__ part) {
  __shared__ double red[2 * 256];
  const int q = blockIdx.x, r = q / P, p = q % P;
  const int64_t t0 = (int64_t)blockIdx.y * 8192;
  const double* w = W[p] + (int64_t)(col0 + r) * npad;
  double s[2] = {0.0, 0.0};
  for (int64_t t = t0 + threadIdx.x; t < min(t0 + 8192, npad); t += 256) {
    const double v = w[t];
    s[0] += v;
    s[1] = fma(v, v, s[1]);
  }
  cta_tree<256>(s, red);
  if (threadIdx.x == 0) {
    part[((int64_t)blockIdx.y * Qp + q) * 2 + 0] = s[0];
    part[((int64_t)blockIdx.y * Qp + q) * 2 + 1] = s[1];
  }
}

int launch_l0_colsum(double* const* W, int64_t npad, int col0, int P, int Q, int Qp, double* part,
                     cudaStream_t s) {
  const int nchunks = (int)ceil_div(npad, 8192);
  dim3 grid(Q, nchunks);
  l0_colsum_kernel<<<grid, 256, 0, s>>>(W, npad, col0, P, Qp, part);
  return nchunks;
}

// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn pt_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    RG_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres));
    RG_CHECK(p != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2D byte tensor [rows][inner] with a 128 x 128 box and 128B swizzle
void make_byte_tensor_map(CUtensorMap* tm, const uint8_t* basep, int64_t inner, int64_t rows) {
  const cuuint64_t gdim[2] = {(cuuint64_t)inner, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)inner};
  const cuuint32_t box[2] = {128, 128};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = pt_encode_fn()(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t*>(basep), gdim, gstride, box,
                              estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  RG_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
}

size_t predict_i8_dig_bytes(int K, int ngroups, int rows_p) { return (size_t)K * ngroups * PI_BN * 2 * rows_p; }

// 2-bit rows [rows][words_per_row] (uint32) with an 8-word x 128-row box (128 samples x 128 SNPs), no swizzle
void make_gp_tensor_map(CUtensorMap* tm, const uint32_t* gp, int64_t words_per_row, int64_t rows) {
  const cuuint64_t gdim[2] = {(cuuint64_t)words_per_row, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)words_per_row * 4};
  const cuuint32_t box[2] = {(cuuint32_t)PI_A_WORDS, (cuuint32_t)PT_BK};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = pt_encode_fn()(tm, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, const_cast<uint32_t*>(gp), gdim, gstride, box,
                              estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  RG_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
}

void launch_l0_coef_i8(const double* cm, int64_t cm_stride, int ldc, int nC, int R, int P, int Q, int Qp, int bs,
                       int rows_p, int K, const double* mu, const double* inv_sd, const double* Bv, int C, double* gam,
                       double* gmu, double* cvec, double* scale, uint8_t* dig, int ngroups, cudaStream_t s) {
  RG_CHECK(rows_p <= PI_MAX_ROWS, "INT8 prediction: rows_p <= 2048");
  dim3 grid(Q, K);
  l0_coef_i8_kernel<<<grid, 256, 0, s>>>(cm, cm_stride, ldc, nC, R, P, Qp, bs, rows_p, mu, inv_sd, Bv, C, gam, gmu, cvec,
                                         scale, dig, ngroups);
}

// SMs of the current device, read once per device
static int sm_count() {
  static std::atomic<int> n_sm[64];
  int dev = 0;
  RG_CUDA(cudaGetDevice(&dev));
  RG_CHECK(dev < 64, "INT8 prediction: device ordinal above 63");
  int n = n_sm[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    RG_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
    n_sm[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

void launch_l0_predict_i8(const CUtensorMap& tmG, const CUtensorMap& tmD, const PredictTcArgs& a, int ntiles,
                          cudaStream_t s) {
  RG_CHECK(2 * a.rows_p <= 4096, "INT8 prediction: 2 * rows_p <= 4096 (int32 Horner bound)");
  // stages, barriers, V, its column sums, then scales, cvec and 2 pointers per output
  const size_t smem = 1024 + (size_t)PI_STAGES * PI_STAGE_BYTES + 128 +
                      ((size_t)kLimbQI8 * PI_LDV + 4 * kLimbQI8 + (size_t)kLimbQI8 * (3 + a.C)) * sizeof(double);
  ensure_dyn_smem(reinterpret_cast<const void*>(l0_predict_i8_kernel), smem);
  const int grid = (int)std::min<int64_t>((int64_t)ntiles * a.ngroups, sm_count());
  l0_predict_i8_kernel<<<grid, PI_THREADS, smem, s>>>(tmG, tmD, a, ntiles);
}

}  // namespace rg
