// Per-fold integer Gram  Z_f Z_f^T  on the Hopper tensor cores (wgmma + TMA + mbarrier).
//
// Z = [G0; Miss] is the (2*rows_p) x Npad operand written by bed_expand_fp8_kernel: 8 x G0 (G0 in {0,1,2} with
// missing calls as 0) and 8 x Miss (Miss in {0,1}) as int8.  The s8 x s8 -> s32 MMAs accumulate exactly (every product
// is <= 256, every fold sum < 2^31), so the accumulators hold 64 x the EXACT integer Grams
//   G0 G0^T, Miss G0^T, Miss Miss^T   restricted to the fold's sample range,
// which is all of Data::calc_cv_matrices' bs x bs x N work (reference src/Data.cpp:748:
// `G_folds[i] = Gmat * Gmat.transpose()`, 2*bs^2*N flops) - the rank-C covariate/scale/mean
// corrections are applied afterwards in FP64 (l0_stats.cu).  The same kernel computes the statistics tiles, Z against
// int8 digit rows of the covariates / phenotypes (l0_stats_tc.cu, s2_kernels.cu).  The FP8 MMAs are not used: Hopper
// keeps only part of the FP32 mantissa while it accumulates them, so their sums stop being exact long before 2^24.
//
// Kernel shape: one CTA per (128 x BN) output tile of the lower triangle per fold.
//   warps 0..7 : two consumer warpgroups; warpgroup w owns tile rows 64 w .. 64 w + 63 (wgmma m64nBNk32, accumulators
//                in registers, int32) and stores them, times out_scale, as FP32 straight from the fragments
//   warp 8     : TMA producer (cp.async.bulk.tensor 2D, 128B swizzle, 4-stage mbarrier ring)
// K loop = the fold's samples in 128-byte (= 128-sample) swizzle atoms, 4 MMAs per atom.
// Tiles of rows >= 128 miss_tile0 (the Miss rows of the Z Z^T Gram) return at once when the block's missing calls fit
// the sparse path's list (*miss_total <= miss_cap): miss_gram.cu writes those rows then.
#include "kernels.cuh"
#include "wgmma_sm90.cuh"

namespace rg {

namespace {

using namespace sm90;

constexpr int BM = 128;
constexpr int BK = 128;             // bytes == samples per K step (one 128B swizzle atom)
constexpr int STAGES = 4;
constexpr int A_BYTES = BM * BK;    // 16 KiB
// BN (template parameter): 256 for the Gram and wide statistics tiles (B stage 32 KiB), 128 for a single 128-row digit group
constexpr int NTHREADS = 288;

}  // namespace

// grid: (ntiles, K folds)
template <int BN>
__global__ void __launch_bounds__(NTHREADS, 1)
gram_s8_wgmma_kernel(const __grid_constant__ CUtensorMap tmZ, const __grid_constant__ CUtensorMap tmB,
                      const int2* __restrict__ tiles,
                      const int2* __restrict__ fold_k, float* __restrict__ out, int ldo,
                      int64_t fold_stride, float out_scale, const unsigned long long* __restrict__ miss_total,
                      unsigned long long miss_cap, int miss_tile0) {
  constexpr int B_BYTES = BN * BK;
  constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int NACC = BN / 2;
  extern __shared__ uint8_t smem_raw[];
  // 128B swizzle needs 1024-byte aligned stage buffers
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gen_base = smem_raw + (base - raw);
  const uint32_t sA = base;
  const uint32_t sB = base + STAGES * A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(gen_base + STAGES * STAGE_BYTES);
  const uint32_t full_bar = smem_u32(bars);                  // [STAGES]
  const uint32_t empty_bar = smem_u32(bars + STAGES);        // [STAGES]

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role
  const int2 tile = tiles[blockIdx.x];          // (m tile of 128 rows, n tile of BN rows)
  if (miss_total && tile.x >= miss_tile0 && *miss_total <= miss_cap) return;
  const int2 fk = fold_k[blockIdx.y];           // (first K block, number of K blocks)
  const int nkb = fk.y;

  if (warp == 8 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar + 8 * s, 1);
      mbar_init(empty_bar + 8 * s, 2);         // one arrival per consumer warpgroup
    }
    fence_barrier_init();
    prefetch_tmap(&tmZ);
    prefetch_tmap(&tmB);
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      // ===== TMA producer =====
      for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % STAGES;
        const uint32_t ph = (kb / STAGES) & 1;
        mbar_wait(empty_bar + 8 * s, ph ^ 1);
        mbar_expect_tx(full_bar + 8 * s, STAGE_BYTES);
        const int kc = (fk.x + kb) * BK;
        tma_load_2d(sA + s * A_BYTES, &tmZ, full_bar + 8 * s, kc, tile.x * BM);
        tma_load_2d(sB + s * B_BYTES, &tmB, full_bar + 8 * s, kc, tile.y * BN);
        if (BN == 256) tma_load_2d(sB + s * B_BYTES + A_BYTES, &tmB, full_bar + 8 * s, kc, tile.y * BN + 128);
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
  for (int kb = 0; kb < nkb; ++kb) {
    const int s = kb % STAGES;
    const uint32_t ph = (kb / STAGES) & 1;
    mbar_wait(full_bar + 8 * s, ph);
    const uint64_t da = desc_k128(sA + s * A_BYTES + wg * (64 * BK));
    const uint64_t db = desc_k128(sB + s * B_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 32; ++k) {
      // advance 32 bytes (= K of one s8 MMA) inside the swizzle atom: +2 in 16-byte units
      if constexpr (BN == 256) wgmma_s8_n256(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k));
      else wgmma_s8_n128(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k));
    }
    wgmma_commit();
    wgmma_wait<1>();                             // the MMAs of stage kb-1 have retired: hand that stage back
    if (kb > 0 && (warp & 3) == 0 && lane == 0) mbar_arrive(empty_bar + 8 * ((kb - 1) % STAGES));
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
__global__ void gram_reference_kernel(const uint8_t* __restrict__ z, int64_t npad, int rows2, int k0, int k1,
                                      float* __restrict__ out, int ldo) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y;
  if (j >= rows2 || j > i) return;
  const uint8_t* zi = z + (int64_t)i * npad;
  const uint8_t* zj = z + (int64_t)j * npad;
  int acc = 0;
  for (int t = k0; t < k1; ++t) {
    const int a = zi[t] >> 3;        // plane bytes 0x00 / 0x08 / 0x10 = 8 x dosage (bed_expand_fp8_kernel)
    const int b = zj[t] >> 3;
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

size_t gram_smem_bytes(int bn) {
  return (size_t)STAGES * (A_BYTES + bn * BK) + 1024 + 128;
}

void gram_tile_list(int rows2, std::vector<int2>& tiles) {
  tiles.clear();
  for (int nj = 0; nj < rows2 / 256; ++nj)
    for (int mi = 2 * nj; mi < rows2 / BM; ++mi) tiles.push_back(make_int2(mi, nj));
}

void launch_gram_wgmma(const CUtensorMap& tm, const CUtensorMap& tmB, const int2* tiles, int ntiles, const int2* fold_k, int K,
                         float* out, int ldo, int64_t fold_stride, float out_scale, cudaStream_t s, int bn,
                         const unsigned long long* miss_total, int64_t miss_cap, int miss_tile0) {
  RG_CHECK(bn == 256 || bn == 128, "gram tiles are 128 x 256 or 128 x 128");
  dim3 grid(ntiles, K);
  if (bn == 256) {
    ensure_dyn_smem(reinterpret_cast<const void*>(gram_s8_wgmma_kernel<256>), gram_smem_bytes(256));
    gram_s8_wgmma_kernel<256><<<grid, NTHREADS, gram_smem_bytes(256), s>>>(tm, tmB, tiles, fold_k, out, ldo, fold_stride, out_scale,
                                                                                     miss_total, miss_cap, miss_tile0);
  } else {
    ensure_dyn_smem(reinterpret_cast<const void*>(gram_s8_wgmma_kernel<128>), gram_smem_bytes(128));
    gram_s8_wgmma_kernel<128><<<grid, NTHREADS, gram_smem_bytes(128), s>>>(tm, tmB, tiles, fold_k, out, ldo, fold_stride, out_scale,
                                                                                     miss_total, miss_cap, miss_tile0);
  }
}

void launch_gram_reference(const uint8_t* z, int64_t npad, int rows2, int k0, int k1, float* out, int ldo,
                           cudaStream_t s) {
  dim3 grid((unsigned)ceil_div(rows2, 128), rows2);
  gram_reference_kernel<<<grid, 128, 0, s>>>(z, npad, rows2, k0, k1, out, ldo);
}

}  // namespace rg
