// Batched "NT" GEMM tiles  D = A B^T  in 3xTF32 on the Hopper tensor cores (wgmma + TMA + mbarrier):
// the arithmetic engine of the mixed-precision ridge solver (chol_mixed.cu).
//
// Every FP32 operand x is used as two TF32 values, hi = rn_tf32(x) and lo = x - hi (exact in FP32, itself truncated
// to TF32 by the tensor core), so that
//     a b  ~  a_hi b_hi + a_hi b_lo + a_lo b_hi          (relative error ~2^-21, FP32 accumulation)
// which is what an FP32 factorisation needs; the FP64 iterative refinement on top (chol_mixed.cu) removes the rest.
// hi and lo exist in shared memory only: global memory holds x once, and the consumer warps split every loaded tile
// position for position (so the TMA swizzle is never decoded) before the MMAs read it.  Storing the pair instead
// doubled the operand bytes of a kernel that is bound by them (BENCH.md).
//
// Operand buffers are [batch][rows][cols] FP32, row-major: a tile of A is 128 rows of one matrix, a tile of B 128
// rows of another (or the same) matrix, the contraction runs along the contiguous column index ("K-major" on both
// sides), exactly the shape of a left-looking Cholesky update  L_i,0:k L_k,0:k^T  and of a triangular solve against a
// stored inverse  P_ik M_k^T.
//
// One CTA per (tile, matrix of the batch):
//   warps 0..3 : one consumer warpgroup: splits the stage (hi over the loaded tile, lo into a buffer of its own), two
//                wgmma m64n128k8 accumulators (tile rows 0-63, 64-127, 12 MMAs each per stage), then the epilogue:
//                accumulators -> shared memory -> optional  C_in - acc  in FP64 -> one FP32 plane (and its mirror
//                image), one thread per tile row
//   warp 4     : TMA producer - 3-D boxes {32 floats, 128 rows, 1 matrix} with 128B swizzle, mbarrier ring
#include "kernels.cuh"
#include "wgmma_sm90.cuh"

namespace rg {

namespace {

using namespace sm90;

constexpr int TG_M = 128, TG_N = 128;
constexpr int TG_KC = 32;                          // floats per K chunk = one 128-byte swizzle atom
// two 32 KiB stages of loaded tiles plus one 32 KiB buffer for the lo tiles of the chunk being multiplied: 96 KiB, two
// CTAs per SM (the 128 accumulator registers allow no more).  The tiles of this solver are short (K <= 1024) and the
// launches small, so what the second stage does not hide is hidden across CTAs.
constexpr int TG_STAGES = 2;
constexpr int TG_TILE_BYTES = TG_M * 128;          // one operand tile of one chunk: 16 KiB
constexpr int TG_STAGE_BYTES = 2 * TG_TILE_BYTES;  // A + B as loaded; the hi tiles overwrite them in place
constexpr int TG_LO_OFF = TG_STAGES * TG_STAGE_BYTES;
constexpr int TG_SMEM_BYTES = TG_LO_OFF + TG_STAGE_BYTES;   // >= 64 KiB: also holds the 128 x 128 FP32 result tile
constexpr int TG_THREADS = 160;

__device__ __forceinline__ float4 tf32_rn4(const float4 v) {
  uint4 t;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t.x) : "f"(v.x));
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t.y) : "f"(v.y));
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t.z) : "f"(v.z));
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t.w) : "f"(v.w));
  return make_float4(__uint_as_float(t.x), __uint_as_float(t.y), __uint_as_float(t.z), __uint_as_float(t.w));
}

// one loaded 16 KiB tile -> hi in place, lo at the same offsets of `lo`; thread t of 128 owns 16-byte pieces t, t + 128, ..
__device__ __forceinline__ void split_tile(uint8_t* raw, uint8_t* lo, int t) {
  float4 v[TG_TILE_BYTES / 16 / 128];
#pragma unroll
  for (int i = 0; i < TG_TILE_BYTES / 16 / 128; ++i) v[i] = *reinterpret_cast<const float4*>(raw + 16 * (t + 128 * i));
#pragma unroll
  for (int i = 0; i < TG_TILE_BYTES / 16 / 128; ++i) {
    const float4 h = tf32_rn4(v[i]);
    *reinterpret_cast<float4*>(raw + 16 * (t + 128 * i)) = h;
    *reinterpret_cast<float4*>(lo + 16 * (t + 128 * i)) = make_float4(v[i].x - h.x, v[i].y - h.y, v[i].z - h.z, v[i].w - h.w);
  }
}

// columns 32 kc .. 32 kc + 31 of the 128 x 128 identity as a B tile (row c = identity row c), written where TMA with
// 128B swizzle would have put them: 16-byte piece q of row c holds columns 4 (q ^ (c % 8)) .. + 3 of the chunk
__device__ __forceinline__ void identity_tile(uint8_t* dst, int kc, int t) {
#pragma unroll
  for (int i = 0; i < TG_TILE_BYTES / 16 / 128; ++i) {
    const int e = t + 128 * i;
    const int c = e >> 3, q = e & 7;
    const int d = c - kc * TG_KC - 4 * (q ^ (c & 7));      // position of the one inside this piece, if 0..3
    *reinterpret_cast<float4*>(dst + 16 * e) = make_float4(d == 0 ? 1.f : 0.f, d == 1 ? 1.f : 0.f, d == 2 ? 1.f : 0.f, d == 3 ? 1.f : 0.f);
  }
}

}  // namespace

// grid: (ntiles, batch); tile entry = (A row tile, B row tile, first K chunk, number of K chunks)
__global__ void __launch_bounds__(TG_THREADS, 2)
tf32x3_gemm_nt_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                      const __grid_constant__ CUtensorMap tmC, const int4* __restrict__ tiles, Tf32GemmEpilogue ep) {
  extern __shared__ uint8_t tg_smem_raw[];
  const uint32_t raw = smem_u32(tg_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;            // 128B swizzle needs 1024-byte aligned stage buffers
  uint8_t* gen_base = tg_smem_raw + (base - raw);
  uint64_t* bars = reinterpret_cast<uint64_t*>(gen_base + TG_SMEM_BYTES);
  const uint32_t full_bar = smem_u32(bars);
  const uint32_t empty_bar = smem_u32(bars + TG_STAGES);

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role
  const int4 tile = tiles[blockIdx.x];
  const int mat = blockIdx.y;
  // optional leading chunks:  acc = C_tile * I  (C = the FP32 matrix the product is subtracted from, I = identity
  // columns built in shared memory), then the main chunks with A negated:  acc = C - A B^T  without an epilogue load
  const int ncc = ep.c_chunks;
  const int nkc = tile.w + ncc;

  if (warp == 4 && lane == 0) {
    for (int s = 0; s < TG_STAGES; ++s) {
      mbar_init(full_bar + 8 * s, 1);
      mbar_init(empty_bar + 8 * s, 1);
    }
    fence_barrier_init();
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    if (ncc > 0) prefetch_tmap(&tmC);
  }
  __syncthreads();

  if (warp == 4) {
    if (lane == 0) {
      const int cmat = ep.c_mat_div > 0 ? mat / ep.c_mat_div : mat;
      // chunk kc: (kc < ncc) the C tile alone, else A / B row tiles at column (tile.z + kc - ncc) * TG_KC (B counts its
      // columns from the tile's first chunk when it is a stack of 128-column matrices)
      for (int kc = 0; kc < nkc; ++kc) {
        const int s = kc % TG_STAGES;
        const uint32_t ph = (kc / TG_STAGES) & 1;
        mbar_wait(empty_bar + 8 * s, ph ^ 1);
        if (kc < ncc) {
          mbar_expect_tx(full_bar + 8 * s, TG_TILE_BYTES);
          tma_load_3d(base + s * TG_STAGE_BYTES, &tmC, full_bar + 8 * s, tile.y * TG_N + kc * TG_KC, tile.x * TG_M, cmat);
        } else {
          mbar_expect_tx(full_bar + 8 * s, TG_STAGE_BYTES);
          const int col = (tile.z + kc - ncc) * TG_KC;
          tma_load_3d(base + s * TG_STAGE_BYTES, &tmA, full_bar + 8 * s, col, tile.x * TG_M, mat);
          tma_load_3d(base + s * TG_STAGE_BYTES + TG_TILE_BYTES, &tmB, full_bar + 8 * s, ep.b_cols_local ? (kc - ncc) * TG_KC : col,
                      tile.y * TG_N, mat);
        }
      }
    }
    return;
  }

  // ===== consumer warpgroup: acc0 = tile rows 0..63, acc1 = rows 64..127 =====
  float acc0[64], acc1[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc0[i] = acc1[i] = 0.f;
  fence_regs(acc0);
  fence_regs(acc1);
  constexpr uint64_t kHalf = (64 * 128) >> 4;              // 64 rows further down the tile, in 16-byte units
  for (int kc = 0; kc < nkc; ++kc) {
    const int s = kc % TG_STAGES;
    const uint32_t ph = (kc / TG_STAGES) & 1;
    mbar_wait(full_bar + 8 * s, ph);
    // hi / lo of this chunk, bit for bit what cvt.rna + an exact subtraction give anywhere else.  The MMAs read shared
    // memory through the async proxy, hence the proxy fence before the barrier; the same fence orders these stores
    // before the TMA write that reuses the stage.
    uint8_t* stage = gen_base + s * TG_STAGE_BYTES;
    split_tile(stage, gen_base + TG_LO_OFF, threadIdx.x);
    if (kc < ncc) identity_tile(stage + TG_TILE_BYTES, kc, threadIdx.x);
    else split_tile(stage + TG_TILE_BYTES, gen_base + TG_LO_OFF + TG_TILE_BYTES, threadIdx.x);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    named_sync(1, 128);
    const uint64_t a_hi = desc_k128(base + s * TG_STAGE_BYTES);
    const uint64_t a_lo = desc_k128(base + TG_LO_OFF);
    const uint64_t b_hi = desc_k128(base + s * TG_STAGE_BYTES + TG_TILE_BYTES);
    const uint64_t b_lo = desc_k128(base + TG_LO_OFF + TG_TILE_BYTES);
    wgmma_fence();
    if (kc < ncc) {
#pragma unroll
      for (int k = 0; k < TG_KC / 8; ++k) {             // (C_lo + C_hi) * 1: the lo tile of the identity is zero
        const uint64_t dk = (uint64_t)(2 * k);          // +32 bytes per K = 8 step inside the swizzle atom
        wgmma_tf32_n128(acc0, a_lo + dk, b_hi + dk);
        wgmma_tf32_n128(acc1, a_lo + kHalf + dk, b_hi + dk);
        wgmma_tf32_n128(acc0, a_hi + dk, b_hi + dk);
        wgmma_tf32_n128(acc1, a_hi + kHalf + dk, b_hi + dk);
      }
    } else if (ncc > 0) {                               // acc = C - A B^T: A negated; small terms first
#pragma unroll
      for (int k = 0; k < TG_KC / 8; ++k) {
        const uint64_t dk = (uint64_t)(2 * k);
        wgmma_tf32_n128_nega(acc0, a_lo + dk, b_hi + dk);
        wgmma_tf32_n128_nega(acc1, a_lo + kHalf + dk, b_hi + dk);
        wgmma_tf32_n128_nega(acc0, a_hi + dk, b_lo + dk);
        wgmma_tf32_n128_nega(acc1, a_hi + kHalf + dk, b_lo + dk);
        wgmma_tf32_n128_nega(acc0, a_hi + dk, b_hi + dk);
        wgmma_tf32_n128_nega(acc1, a_hi + kHalf + dk, b_hi + dk);
      }
    } else {
#pragma unroll
      for (int k = 0; k < TG_KC / 8; ++k) {
        const uint64_t dk = (uint64_t)(2 * k);
        wgmma_tf32_n128(acc0, a_lo + dk, b_hi + dk);
        wgmma_tf32_n128(acc1, a_lo + kHalf + dk, b_hi + dk);
        wgmma_tf32_n128(acc0, a_hi + dk, b_lo + dk);
        wgmma_tf32_n128(acc1, a_hi + kHalf + dk, b_lo + dk);
        wgmma_tf32_n128(acc0, a_hi + dk, b_hi + dk);
        wgmma_tf32_n128(acc1, a_hi + kHalf + dk, b_hi + dk);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    named_sync(1, 128);                                  // every warp's MMAs are done: the lo buffer and the stage are free
    if (threadIdx.x == 0) mbar_arrive(empty_bar + 8 * s);
  }
  fence_regs(acc0);
  fence_regs(acc1);

  // ===== epilogue =====
  // the result tile goes to shared memory (the first 64 KiB, free now) as 128 rows of 128 floats, 16-byte chunk c of
  // row r at chunk c ^ (r % 32); every thread then owns one tile row, as the row-major staging below expects
  {
    float* tilef = reinterpret_cast<float*>(gen_base);
    const int fr = (warp & 3) * 16 + (lane >> 2);       // fragment row (+8, +64)
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int col = 8 * j + 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 4; ++h) {                      // (acc, +8 rows)
        const int r = fr + 8 * (h & 1) + 64 * (h >> 1);
        const float* a = (h >> 1) ? acc1 : acc0;
        *reinterpret_cast<float2*>(tilef + (size_t)r * TG_N + 4 * ((col >> 2) ^ (r & 31)) + (col & 3)) =
            make_float2(a[4 * j + 2 * (h & 1)], a[4 * j + 2 * (h & 1) + 1]);
      }
    }
  }
  named_sync(1, 128);
  {
    const int q = warp & 3;
    const int r_loc = q * 32 + lane;
    const int row = tile.x * TG_M + r_loc;               // output row (A row index)
    const int col0 = tile.y * TG_N;                      // first output column (B row index)
    const int64_t n = ep.n;
    const int64_t mat_off = (int64_t)mat * ep.out_mat_stride;
    const double* cin = ep.cin ? ep.cin + (int64_t)(ep.cin_mat_div > 0 ? mat / ep.cin_mat_div : mat) * ep.cin_mat_stride + (int64_t)row * ep.cin_ld + col0
                               : nullptr;
    const double diag_add = (ep.diag_add != nullptr && tile.x == tile.y) ? ep.diag_add[ep.diag_mod > 0 ? mat % ep.diag_mod : mat] : 0.0;
    const bool diag_tile = tile.x == tile.y;
    float* st = reinterpret_cast<float*>(gen_base) + (size_t)q * (32 * TG_N) + (size_t)lane * TG_N;   // this thread's row
    constexpr int EC = 16;                               // columns per epilogue pass
#pragma unroll 1
    for (int c = 0; c < TG_N / EC; ++c) {
      float v[EC];
#pragma unroll
      for (int j = 0; j < EC; j += 4) {
        const float4 t4 = *reinterpret_cast<const float4*>(st + 4 * (((c * EC + j) >> 2) ^ lane));
        v[j] = t4.x; v[j + 1] = t4.y; v[j + 2] = t4.z; v[j + 3] = t4.w;
      }
      float o[EC];
      if (cin) {
#pragma unroll
        for (int j = 0; j < EC; j += 2) {
          const double2 cc = *reinterpret_cast<const double2*>(cin + c * EC + j);
          o[j] = (float)(cc.x - (double)v[j]);
          o[j + 1] = (float)(cc.y - (double)v[j + 1]);
        }
      } else {
#pragma unroll
        for (int j = 0; j < EC; ++j) o[j] = ep.negate ? -v[j] : v[j];
      }
      if (diag_tile && diag_add != 0.0) {
#pragma unroll
        for (int j = 0; j < EC; ++j) if (c * EC + j == r_loc) o[j] = (float)((double)o[j] + diag_add);
      }
      if (ep.lower_only && diag_tile) {
#pragma unroll
        for (int j = 0; j < EC; ++j) if (c * EC + j > r_loc) o[j] = 0.f;
      }
      // the row-major output goes back to the thread's own row of the staging tile (below, a warp stores whole 512-byte
      // rows); the mirror image is already lane-coalesced (lanes hold consecutive rows) and leaves from registers
#pragma unroll
      for (int j = 0; j < EC; j += 4) {
        const int chunk = (c * EC + j) >> 2;                                // 16-byte chunk of the row, XOR-swizzled by the row
        *reinterpret_cast<float4*>(st + 4 * (chunk ^ lane)) = make_float4(o[j], o[j + 1], o[j + 2], o[j + 3]);
      }
      if (ep.mirror && !diag_tile) {                      // D^T into the mirror tile
        float* pt = ep.out + mat_off + (int64_t)(col0 + c * EC) * n + row;
#pragma unroll
        for (int j = 0; j < EC; ++j) pt[(int64_t)j * n] = o[j];
      }
    }
    // ---- row-major tile: warp q owns tile rows 32 q .. 32 q + 31; one row (128 floats) per store instruction
    __syncwarp();
    {
      const float* stw = reinterpret_cast<const float*>(gen_base) + (size_t)q * (32 * TG_N);
      float* po = ep.out + mat_off + (int64_t)(tile.x * TG_M + q * 32) * n + col0 + lane * 4;
#pragma unroll 4
      for (int rr = 0; rr < 32; ++rr)
        *reinterpret_cast<float4*>(po + (int64_t)rr * n) = *reinterpret_cast<const float4*>(stw + (size_t)rr * TG_N + 4 * (lane ^ rr));
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn tg_encode_fn() {
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

// operand matrices [batch][rows][cols] FP32 -> 3-D map (col, row, matrix), box {32, 128, 1}
void make_tf32_operand_tensor_map(CUtensorMap* tm, const float* base, int cols, int rows, int batch) {
  const cuuint64_t gdim[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)batch};
  const cuuint64_t gstride[2] = {(cuuint64_t)cols * 4, (cuuint64_t)rows * cols * 4};
  const cuuint32_t box[3] = {TG_KC, 128, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = tg_encode_fn()(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), gdim, gstride, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  RG_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (tf32 operand) failed (" + std::to_string((int)r) + ")");
}

// plain row-major FP32 matrix [rows][cols] -> 2-D map, box {box_cols, box_rows}, no swizzle (the substitution sweeps)
void make_f32_rows_tensor_map(CUtensorMap* tm, const float* base, int cols, int64_t rows, int box_cols, int box_rows) {
  const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)cols * 4};
  const cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = tg_encode_fn()(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstride, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  RG_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (f32 rows) failed (" + std::to_string((int)r) + ")");
}

void launch_tf32x3_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const int4* tiles, int ntiles, int batch,
                        const Tf32GemmEpilogue& ep, cudaStream_t s, const CUtensorMap* tmC) {
  RG_CHECK(ep.c_chunks == 0 || tmC, "tf32 gemm: the C phase needs its tensor map");
  RG_CHECK(ep.out != nullptr, "tf32 gemm: no output");
  if (ntiles <= 0 || batch <= 0) return;
  const size_t smem = (size_t)TG_SMEM_BYTES + 1024 + 128;
  dim3 grid(ntiles, batch);
  ensure_dyn_smem(reinterpret_cast<const void*>(tf32x3_gemm_nt_kernel), smem);
  tf32x3_gemm_nt_kernel<<<grid, TG_THREADS, smem, s>>>(tmA, tmB, tmC ? *tmC : tmA, tiles, ep);
}

}  // namespace rg
