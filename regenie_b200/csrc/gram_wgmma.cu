// Integer Grams of 2-bit genotype rows on the Hopper tensor cores (wgmma + TMA + mbarrier).
//
// Z is a stack of int8 planes of the block's padded 2-bit rows: Z row r is plane r / rows_p of 2-bit row r % rows_p, and
// each plane maps the four codes to bytes through its own PRMT table (ZPlanes, kernels.cuh).  Level 0 uses
// Z = [G0; Miss]: 8 x G0 (G0 in {0,1,2} with missing calls as 0) and 8 x Miss (Miss in {0,1}).  The s8 x s8 -> s32 MMAs
// accumulate exactly (every product is <= 256, every fold sum < 2^31), so the accumulators hold 64 x the EXACT integer
// Grams
//   G0 G0^T, Miss G0^T, Miss Miss^T   restricted to the fold's sample range,
// which is all of Data::calc_cv_matrices' bs x bs x N work (reference src/Data.cpp:748:
// `G_folds[i] = Gmat * Gmat.transpose()`, 2*bs^2*N flops) - the rank-C covariate/scale/mean
// corrections are applied afterwards in FP64 (l0_stats.cu).  The same kernel computes the statistics tiles, Z against
// int8 digit rows of the covariates / phenotypes (l0_stats_tc.cu) or of Step 2's feature rows, with Z = [G; G^2; Miss]
// (s2_api.cu).  The FP8 MMAs are not used: Hopper keeps only part of the FP32 mantissa while it accumulates them, so
// their sums stop being exact long before 2^24.
//
// Kernel shape: one CTA per (128 x BN) output tile (the lower triangle for Z Z^T) per fold.
//   warps 0..7 : two consumer warpgroups; warpgroup w owns tile rows 64 w .. 64 w + 63 (wgmma m64nBNk32, accumulators
//                in registers, int32) and stores them, times out_scale, as FP32 straight from the fragments
//   warp 8     : TMA producer (cp.async.bulk.tensor 2D, mbarrier ring)
// K loop = the fold's samples in steps of 128, 4 MMAs per step.
// The A rows are built in registers from the 2-bit rows (one 32-bit word = 16 samples, an eighth of the plane bytes):
// the producer loads 128 rows x 8 words per step, and each thread turns byte t4 of two consecutive words of each of its
// two fragment rows into the plane bytes of its k quads.  rows_p is a multiple of 128, so every 128-row box lies in one
// plane.  Where the B rows come from (template parameter B2):
//   B2 (level 0's Z Z^T tiles): the B rows too come as 2-bit rows; the consumers expand them, one word into one 16-byte
//       chunk, into a 128B-swizzled int8 buffer (three buffers: step kb + 1 is written while the MMAs of step kb run,
//       over the buffer whose MMAs of step kb - 2 every warpgroup has retired before the last named barrier);
//   !B2 (statistics tiles): int8 digit rows in HBM through 128B-swizzled TMA boxes.
// Tiles of rows >= 128 miss_tile0 (the Miss rows of the Z Z^T Gram) return at once when the block's missing calls fit
// the sparse path's list (*miss_total <= miss_cap): miss_gram.cu writes those rows then.
#include "kernels.cuh"
#include "wgmma_sm90.cuh"

namespace rg {

namespace {

using namespace sm90;

constexpr int BM = 128;
constexpr int BK = 128;             // samples per K step (one 128B swizzle atom of the int8 operands)
constexpr int STAGES = 4;
constexpr int A_BYTES = BM * BK;    // 16 KiB: one 128-row int8 box
constexpr int GROW = BK / 16 * 4;   // bytes of one 2-bit row per K step (8 words)
constexpr int G_BYTES = 128 * GROW; // 4 KiB: one 128-row box of 2-bit rows
constexpr int XBUF = 3;             // expanded B buffers (B2)
// BN (template parameter): 256 for the Gram and wide statistics tiles, 128 for a single 128-row digit group
constexpr int NTHREADS = 288;

template <int BN, bool B2>
struct GramLayout {
  static constexpr int NST = B2 ? 6 : STAGES;          // the 2-bit stages are small: a deeper ring
  static constexpr int A_ST = G_BYTES;
  static constexpr int B_ST = B2 ? 2 * G_BYTES : BN * BK;
  static constexpr int X_BYTES = B2 ? XBUF * BN * BK : 0;
  static constexpr int RING = NST * (A_ST + B_ST);
  static constexpr size_t SMEM = (size_t)X_BYTES + RING + 1024 + 128;
};

// the two-bit codes at bits 0-7 and 16-23 of n, one per nibble (a PRMT selector for four bytes in each half)
__device__ __forceinline__ uint32_t code_nibbles(uint32_t n) {
  n = (n | (n << 4)) & 0x0F0F0F0Fu;
  return (n | (n << 2)) & 0x33333333u;
}
// byte t4 (psel = t4 | (4 + t4) << 8) of words x and y -> the four plane bytes of each
__device__ __forceinline__ void plane_pair(uint32_t x, uint32_t y, uint32_t psel, uint32_t lut, uint32_t& px,
                                           uint32_t& py) {
  const uint32_t n = code_nibbles(__byte_perm(x, y, psel) & 0x00FF00FFu);
  px = __byte_perm(lut, 0, n);
  py = __byte_perm(lut, 0, n >> 16);
}
// one 2-bit word (16 samples) -> its 16 plane bytes
__device__ __forceinline__ uint4 plane_chunk(uint32_t w, uint32_t lut) {
  const uint32_t a = code_nibbles(__byte_perm(w, 0, 0x4140)), b = code_nibbles(__byte_perm(w, 0, 0x4342));
  return make_uint4(__byte_perm(lut, 0, a), __byte_perm(lut, 0, a >> 16), __byte_perm(lut, 0, b),
                    __byte_perm(lut, 0, b >> 16));
}
// Z row zrow: its 2-bit row and the PRMT table of its plane
__device__ __forceinline__ int gp_row(int zrow, int rows_p) { return zrow % rows_p; }
__device__ __forceinline__ uint32_t plane_lut(const ZPlanes& z, int zrow, int rows_p) {
  const int p = zrow / rows_p;
  return p == 0 ? z.lut[0] : p == 1 ? z.lut[1] : z.lut[2];
}

}  // namespace

// grid: (ntiles, K folds).  tmA: the 2-bit rows (make_gp_tensor_map); tmB: the 2-bit rows again (B2) or int8 digit rows
// (make_gram_tensor_map).
template <int BN, bool B2>
__global__ void __launch_bounds__(NTHREADS, 1)
gram_s8_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                      const int2* __restrict__ tiles,
                      const int2* __restrict__ fold_k, float* __restrict__ out, int ldo,
                      int64_t fold_stride, float out_scale, const unsigned long long* __restrict__ miss_total,
                      unsigned long long miss_cap, int miss_tile0, int rows_p, const ZPlanes planes) {
  static_assert(!B2 || BN == 256, "2-bit B rows only in 128 x 256 tiles");
  using Lo = GramLayout<BN, B2>;
  constexpr int NST = Lo::NST;
  constexpr int NACC = BN / 2;
  extern __shared__ uint8_t smem_raw[];
  // 128B swizzle needs 1024-byte aligned int8 buffers: the expanded B buffers, then the B ring, then the A ring
  // (2-bit boxes need 16 bytes)
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gen_base = smem_raw + (base - raw);
  const uint32_t sX = base;
  const uint32_t sB = base + Lo::X_BYTES;
  const uint32_t sA = sB + NST * Lo::B_ST;
  uint64_t* bars = reinterpret_cast<uint64_t*>(gen_base + Lo::X_BYTES + Lo::RING);
  const uint32_t full_bar = smem_u32(bars);                  // [NST]
  const uint32_t empty_bar = smem_u32(bars + NST);           // [NST]

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role
  const int2 tile = tiles[blockIdx.x];          // (m tile of 128 rows, n tile of BN rows)
  if (miss_total && tile.x >= miss_tile0 && *miss_total <= miss_cap) return;
  const int2 fk = fold_k[blockIdx.y];           // (first K block, number of K blocks)
  const int nkb = fk.y;

  if (warp == 8 && lane == 0) {
    for (int s = 0; s < NST; ++s) {
      mbar_init(full_bar + 8 * s, 1);
      mbar_init(empty_bar + 8 * s, 2);         // one arrival per consumer warpgroup
    }
    fence_barrier_init();
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      // ===== TMA producer =====
      for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % NST;
        const uint32_t ph = (kb / NST) & 1;
        const uint32_t fb = full_bar + 8 * s;
        mbar_wait(empty_bar + 8 * s, ph ^ 1);
        mbar_expect_tx(fb, Lo::A_ST + Lo::B_ST);
        const int kc = (fk.x + kb) * BK;
        tma_load_2d(sA + s * Lo::A_ST, &tmA, fb, kc / 16, gp_row(tile.x * BM, rows_p));
        if constexpr (B2) {
          tma_load_2d(sB + s * Lo::B_ST, &tmB, fb, kc / 16, gp_row(tile.y * BN, rows_p));
          tma_load_2d(sB + s * Lo::B_ST + G_BYTES, &tmB, fb, kc / 16, gp_row(tile.y * BN + 128, rows_p));
        } else {
          tma_load_2d(sB + s * Lo::B_ST, &tmB, fb, kc, tile.y * BN);
          if (BN == 256) tma_load_2d(sB + s * Lo::B_ST + A_BYTES, &tmB, fb, kc, tile.y * BN + 128);
        }
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg = rows 64 wg .. 64 wg + 63 of the tile =====
  const int wg = warp >> 2;
  int32_t acc[NACC];
#pragma unroll
  for (int i = 0; i < NACC; ++i) acc[i] = 0;
  fence_regs(acc);
  // A fragment of thread (warp w of the warpgroup, lane l, r = l / 4, t4 = l % 4): rows r and r + 8 of the warp's 16,
  // k quads 4 t4 .. +3 and 16 + 4 t4 .. +3 of an MMA's 32 samples = byte t4 of words 2 kk and 2 kk + 1 of the row.
  // The 8-byte loads of a half-warp hit four rows 32 bytes apart: distinct banks.
  const int w = warp & 3, t4 = lane & 3;
  const uint32_t psel = (uint32_t)t4 | ((uint32_t)(4 + t4) << 8);
  const uint32_t lut_a = plane_lut(planes, tile.x * BM, rows_p);
  const uint8_t* gA = gen_base + (sA - base) + (64 * wg + 16 * w + (lane >> 2)) * GROW;
  auto build = [&](int s, int kk, uint32_t (&af)[4]) {
    const uint8_t* p = gA + s * Lo::A_ST + 8 * kk;
    const uint2 v0 = *reinterpret_cast<const uint2*>(p);
    const uint2 v1 = *reinterpret_cast<const uint2*>(p + 8 * GROW);
    plane_pair(v0.x, v0.y, psel, lut_a, af[0], af[2]);
    plane_pair(v1.x, v1.y, psel, lut_a, af[1], af[3]);
  };
  // B2: consumer thread ct expands word ct % 8 of rows ct / 8 + 32 i (i = 0..7; i < 4 from the first 128-row box) into
  // chunk (ct % 8) ^ (row % 8) of the row: a quarter-warp writes one whole 128-byte row
  const int ct = threadIdx.x;
  const uint32_t lut_b0 = plane_lut(planes, tile.y * BN, rows_p);
  const uint32_t lut_b1 = plane_lut(planes, tile.y * BN + 128, rows_p);
  const uint8_t* gB = gen_base + (sB - base) + 4 * ct;
  uint8_t* gX = gen_base + (ct >> 3) * 128 + ((((ct & 7) ^ (ct >> 3)) & 7) << 4);
  auto expand = [&](int s, int xb, int i) {
    const uint32_t v = *reinterpret_cast<const uint32_t*>(gB + s * Lo::B_ST + 1024 * i);
    *reinterpret_cast<uint4*>(gX + xb * (BN * BK) + 4096 * i) = plane_chunk(v, i < 4 ? lut_b0 : lut_b1);
  };
  auto publish = [&]() {                           // expanded rows -> visible to the MMAs of both warpgroups
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    named_sync(1, 256);
  };
  // One commit group per MMA, two fragment register sets: while MMA u runs, MMA u - 1 is retired (at the first MMA of
  // a step: the previous step's MMAs, whose 2-bit stage goes back to the producer) and the fragment of MMA u + 1 is
  // built; with B2, two of the thread's eight words of step kb + 1 are expanded beside each MMA.
  uint32_t afr[2][4];
  mbar_wait(full_bar, 0);
  if constexpr (B2) {
#pragma unroll
    for (int i = 0; i < 8; ++i) expand(0, 0, i);
    publish();
  }
  build(0, 0, afr[0]);
  for (int kb = 0; kb < nkb; ++kb) {
    const int s = kb % NST, s1 = (kb + 1) % NST;
    const bool more = kb + 1 < nkb;
    const uint64_t db = desc_k128(B2 ? sX + (kb % XBUF) * (BN * BK) : sB + s * Lo::B_ST);
#pragma unroll
    for (int kk = 0; kk < BK / 32; ++kk) {
      wgmma_fence();
      // +32 bytes (K of one MMA) inside the 128-byte swizzle atom: +2 in 16-byte units
      if constexpr (BN == 256) wgmma_s8_rs_n256(acc, afr[kk & 1], db + (uint64_t)(2 * kk));
      else wgmma_s8_rs_n128(acc, afr[kk & 1], db + (uint64_t)(2 * kk));
      wgmma_commit();
      wgmma_wait<1>();
      if (kk == 0 && kb > 0 && w == 0 && lane == 0) mbar_arrive(empty_bar + 8 * ((kb - 1) % NST));
      if constexpr (B2) {
        if (more) {
          if (kk == 0) mbar_wait(full_bar + 8 * s1, ((kb + 1) / NST) & 1);
          expand(s1, (kb + 1) % XBUF, 2 * kk);
          expand(s1, (kb + 1) % XBUF, 2 * kk + 1);
        }
      }
      if (kk + 1 < BK / 32) {
        build(s, kk + 1, afr[(kk + 1) & 1]);
      } else if (more) {
        if constexpr (!B2) mbar_wait(full_bar + 8 * s1, ((kb + 1) / NST) & 1);
        build(s1, 0, afr[0]);
      }
    }
    if constexpr (B2) {
      if (more) publish();
    }
  }
  wgmma_wait<0>();
  fence_regs(acc);

  // ===== epilogue: fragments -> global (each quad of lanes writes 32 contiguous bytes of a row) =====
  const int r0 = tile.x * BM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  float* obase = out + (int64_t)blockIdx.y * fold_stride + tile.y * BN + 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    *reinterpret_cast<float2*>(obase + (int64_t)r0 * ldo + 8 * j) =
        make_float2((float)acc[4 * j] * out_scale, (float)acc[4 * j + 1] * out_scale);
    *reinterpret_cast<float2*>(obase + (int64_t)(r0 + 8) * ldo + 8 * j) =
        make_float2((float)acc[4 * j + 2] * out_scale, (float)acc[4 * j + 3] * out_scale);
  }
}

// ---------------------------------------------------------------------------------------
// Test-only reference: same quantity on CUDA cores straight from the 2-bit codes (used by
// tests through rg_debug_fetch to localise a tensor-core protocol bug; never on the product path).
__global__ void gram_reference_kernel(const uint32_t* __restrict__ gp, int64_t words_per_row, int rows_p, int k0,
                                      int k1, float* __restrict__ out, int ldo) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y;
  if (j >= 2 * rows_p || j > i) return;
  const uint32_t* gi = gp + (int64_t)(i % rows_p) * words_per_row;
  const uint32_t* gj = gp + (int64_t)(j % rows_p) * words_per_row;
  const bool mi = i >= rows_p, mj = j >= rows_p;
  int acc = 0;
  for (int t = k0; t < k1; ++t) {
    const int ci = (gi[t >> 4] >> (2 * (t & 15))) & 3;   // dosage 0 / 1 / 2, 3 = missing
    const int cj = (gj[t >> 4] >> (2 * (t & 15))) & 3;
    const int a = mi ? ci == 3 : (ci == 3 ? 0 : ci);
    const int b = mj ? cj == 3 : (cj == 3 ? 0 : cj);
    acc += a * b;
  }
  out[(int64_t)i * ldo + j] = (float)acc;
}

// ---------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
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

void make_gram_tensor_map(CUtensorMap* tm, const uint8_t* z, int64_t npad, int rows2) {
  const cuuint64_t gdim[2] = {(cuuint64_t)npad, (cuuint64_t)rows2};
  const cuuint64_t gstride[1] = {(cuuint64_t)npad};
  const cuuint32_t box[2] = {BK, 128};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode_fn()(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t*>(z), gdim, gstride, box,
                               estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  RG_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
}

void gram_tile_list(int rows2, std::vector<int2>& tiles) {
  tiles.clear();
  for (int nj = 0; nj < rows2 / 256; ++nj)
    for (int mi = 2 * nj; mi < rows2 / BM; ++mi) tiles.push_back(make_int2(mi, nj));
}

// statistics tiles: every 128-row tile of the zrows Z rows against every bn-row tile of the drows digit rows
void stat_tile_list(int zrows, int drows, int bn, std::vector<int2>& tiles) {
  tiles.clear();
  for (int nj = 0; nj < drows / bn; ++nj)
    for (int mi = 0; mi < zrows / BM; ++mi) tiles.push_back(make_int2(mi, nj));
}

template <int BN, bool B2>
static void launch_gram(const CUtensorMap& tmA, const CUtensorMap& tmB, const int2* tiles, int ntiles,
                        const int2* fold_k, int K, float* out, int ldo, int64_t fold_stride, float out_scale,
                        cudaStream_t s, const unsigned long long* miss_total, int64_t miss_cap, int miss_tile0,
                        int rows_p, const ZPlanes& planes) {
  const void* fn = reinterpret_cast<const void*>(gram_s8_wgmma_kernel<BN, B2>);
  const size_t smem = GramLayout<BN, B2>::SMEM;
  ensure_dyn_smem(fn, smem);
  gram_s8_wgmma_kernel<BN, B2><<<dim3(ntiles, K), NTHREADS, smem, s>>>(
      tmA, tmB, tiles, fold_k, out, ldo, fold_stride, out_scale, miss_total, miss_cap, miss_tile0, rows_p, planes);
}

void launch_gram_gp(const CUtensorMap& tmG, const CUtensorMap* tmD, int rows_p, const ZPlanes& planes,
                    const int2* tiles, int ntiles, const int2* fold_k, int K, float* out, int ldo, int64_t fold_stride,
                    float out_scale, cudaStream_t s, int bn, const unsigned long long* miss_total, int64_t miss_cap,
                    int miss_tile0) {
  RG_CHECK(rows_p % 128 == 0, "gram tiles: rows_p is a multiple of 128");
  if (!tmD) {
    RG_CHECK(bn == 256, "Z Z^T tiles are 128 x 256");
    launch_gram<256, true>(tmG, tmG, tiles, ntiles, fold_k, K, out, ldo, fold_stride, out_scale, s, miss_total,
                           miss_cap, miss_tile0, rows_p, planes);
  } else {
    RG_CHECK(bn == 256 || bn == 128, "gram tiles are 128 x 256 or 128 x 128");
    if (bn == 256)
      launch_gram<256, false>(tmG, *tmD, tiles, ntiles, fold_k, K, out, ldo, fold_stride, out_scale, s, miss_total,
                              miss_cap, miss_tile0, rows_p, planes);
    else
      launch_gram<128, false>(tmG, *tmD, tiles, ntiles, fold_k, K, out, ldo, fold_stride, out_scale, s, miss_total,
                              miss_cap, miss_tile0, rows_p, planes);
  }
}

void launch_gram_reference(const uint32_t* gp, int64_t npad, int rows_p, int k0, int k1, float* out, int ldo,
                           cudaStream_t s) {
  dim3 grid((unsigned)ceil_div(2 * rows_p, 128), 2 * rows_p);
  gram_reference_kernel<<<grid, 128, 0, s>>>(gp, npad / 16, rows_p, k0, k1, out, ldo);
}

}  // namespace rg
