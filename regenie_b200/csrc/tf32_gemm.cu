// Batched "NT" GEMM tiles  D = A B^T  in 3xTF32 on the Hopper tensor cores (wgmma + TMA + mbarrier):
// the arithmetic engine of the mixed-precision ridge solver (chol_mixed.cu).
//
// Every FP32 operand lives in global memory as two planes, hi = rn_tf32(x) and lo = x - hi (exact in FP32, itself
// truncated to TF32 by the tensor core), so that
//     a b  ~  a_hi b_hi + a_hi b_lo + a_lo b_hi          (relative error ~2^-21, FP32 accumulation)
// which is what an FP32 factorisation needs; the FP64 iterative refinement on top (chol_mixed.cu) removes the rest.
//
// Operand buffers are [batch][2 planes][n rows][n cols] FP32, row-major: a tile of A is 128 rows of one matrix, a
// tile of B 128 rows of another (or the same) matrix, the contraction runs along the contiguous column index
// ("K-major" on both sides), exactly the shape of a left-looking Cholesky update  L_i,0:k L_k,0:k^T, of a triangular
// solve against a stored inverse  P_ik M_k^T, and of the triangular-inverse products.
//
// One CTA per (tile, matrix of the batch):
//   warps 0..3 : one consumer warpgroup: two wgmma m64n128k8 accumulators (tile rows 0-63, 64-127, 12 MMAs each per
//                stage), then the epilogue: accumulators -> shared memory -> optional  C_in - acc  in FP64 -> hi/lo
//                planes (and / or the transposed tile, and / or a plain FP32 plane), one thread per tile row
//   warp 4     : TMA producer - 3-D boxes {32 floats, 128 rows, 2 planes} with 128B swizzle, mbarrier ring
#include "kernels.cuh"
#include "wgmma_sm90.cuh"

namespace rg {

namespace {

using namespace sm90;

constexpr int TG_M = 128, TG_N = 128;
constexpr int TG_KC = 32;                          // floats per K chunk = one 128-byte swizzle atom
// one 64 KiB stage per CTA and several co-resident CTAs per SM: the tiles of this solver are short (K <= 1024) and the
// launches small, so latency is hidden across CTAs
constexpr int TG_STAGES = 1;
constexpr int TG_PLANE_BYTES = TG_M * 128;         // 16 KiB
constexpr int TG_OP_BYTES = 2 * TG_PLANE_BYTES;    // hi + lo
constexpr int TG_STAGE_BYTES = 2 * TG_OP_BYTES;    // A + B = 64 KiB (also holds the 128 x 128 FP32 result tile)
constexpr int TG_THREADS = 160;

}  // namespace

// grid: (ntiles, batch); tile entry = (A row tile, B row tile, first K chunk, number of K chunks)
__global__ void __launch_bounds__(TG_THREADS, 2)
tf32x3_gemm_nt_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                      const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmI,
                      const int4* __restrict__ tiles, Tf32GemmEpilogue ep) {
  extern __shared__ uint8_t tg_smem_raw[];
  const uint32_t raw = smem_u32(tg_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;            // 128B swizzle needs 1024-byte aligned stage buffers
  uint8_t* gen_base = tg_smem_raw + (base - raw);
  uint64_t* bars = reinterpret_cast<uint64_t*>(gen_base + TG_STAGES * TG_STAGE_BYTES);
  const uint32_t full_bar = smem_u32(bars);
  const uint32_t empty_bar = smem_u32(bars + TG_STAGES);

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role
  const int4 tile = tiles[blockIdx.x];
  const int mat = blockIdx.y;
  // optional leading chunks:  acc = C_tile * I  (C = FP32 hi/lo planes of the matrix the product is subtracted from,
  // I = identity planes), then the main chunks with A negated:  acc = C - A B^T  without a single epilogue load
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
    if (ncc > 0) {
      prefetch_tmap(&tmC);
      prefetch_tmap(&tmI);
    }
  }
  __syncthreads();

  if (warp == 4) {
    if (lane == 0) {
      const int cmat = 2 * (ep.c_mat_div > 0 ? mat / ep.c_mat_div : mat);
      // chunk kc: (kc < ncc) C tile x identity, else A / B row tiles at column (tile.z + kc - ncc) * TG_KC
      for (int kc = 0; kc < nkc; ++kc) {
        const int s = kc % TG_STAGES;
        const uint32_t ph = (kc / TG_STAGES) & 1;
        mbar_wait(empty_bar + 8 * s, ph ^ 1);
        mbar_expect_tx(full_bar + 8 * s, TG_STAGE_BYTES);
        if (kc < ncc) {
          tma_load_3d(base + s * TG_STAGE_BYTES, &tmC, full_bar + 8 * s, tile.y * TG_N + kc * TG_KC, tile.x * TG_M, cmat);
          tma_load_3d(base + s * TG_STAGE_BYTES + TG_OP_BYTES, &tmI, full_bar + 8 * s, kc * TG_KC, 0, 0);
        } else {
          const int col = (tile.z + kc - ncc) * TG_KC;
          tma_load_3d(base + s * TG_STAGE_BYTES, &tmA, full_bar + 8 * s, col, tile.x * TG_M, 2 * mat);
          tma_load_3d(base + s * TG_STAGE_BYTES + TG_OP_BYTES, &tmB, full_bar + 8 * s, col, tile.y * TG_N, 2 * mat);
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
    const uint64_t a_hi = desc_k128(base + s * TG_STAGE_BYTES);
    const uint64_t a_lo = desc_k128(base + s * TG_STAGE_BYTES + TG_PLANE_BYTES);
    const uint64_t b_hi = desc_k128(base + s * TG_STAGE_BYTES + TG_OP_BYTES);
    const uint64_t b_lo = desc_k128(base + s * TG_STAGE_BYTES + TG_OP_BYTES + TG_PLANE_BYTES);
    wgmma_fence();
    if (kc < ncc) {
#pragma unroll
      for (int k = 0; k < TG_KC / 8; ++k) {             // (C_lo + C_hi) * 1: the lo plane of the identity is zero
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
    if (warp == 0 && lane == 0) mbar_arrive(empty_bar + 8 * s);
  }
  fence_regs(acc0);
  fence_regs(acc1);

  // ===== epilogue =====
  // the result tile goes to shared memory (stage 0, free now) as 128 rows of 128 floats, 16-byte chunk c of row r at
  // chunk c ^ (r % 32); every thread then owns one tile row, as the row-major staging below expects
  named_sync(1, 128);                                    // all MMAs of the warpgroup have read their operands
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
      // row-major outputs go back to the thread's own row of the staging tile (below, a warp stores whole 512-byte
      // rows); the transposed copies are already lane-coalesced (lanes hold consecutive rows) and leave from registers
#pragma unroll
      for (int j = 0; j < EC; j += 4) {
        const int chunk = (c * EC + j) >> 2;                                // 16-byte chunk of the row, XOR-swizzled by the row
        *reinterpret_cast<float4*>(st + 4 * (chunk ^ lane)) = make_float4(o[j], o[j + 1], o[j + 2], o[j + 3]);
      }
      if (ep.out_t) {                                     // D^T as hi / lo planes: lanes of a warp hold consecutive rows
        float* th = ep.out_t + 2 * mat_off + (int64_t)(col0 + c * EC) * n + row;
        float* tl = th + n * n;
#pragma unroll
        for (int j = 0; j < EC; ++j) {
          uint32_t t;
          asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(o[j]));
          const float hi = __uint_as_float(t);
          th[(int64_t)j * n] = hi;
          tl[(int64_t)j * n] = o[j] - hi;
        }
      }
      if (ep.out_plain && ep.mirror && !diag_tile) {      // mirror image of the plain plane (symmetric results)
        float* pt = ep.out_plain + mat_off + (int64_t)(col0 + c * EC) * n + row;
#pragma unroll
        for (int j = 0; j < EC; ++j) pt[(int64_t)j * n] = o[j];
      }
    }
    // ---- row-major planes: warp q owns tile rows 32 q .. 32 q + 31; one row (128 floats) per store instruction
    __syncwarp();
    {
      const float* stw = reinterpret_cast<const float*>(gen_base) + (size_t)q * (32 * TG_N);
      float* oh = ep.out ? ep.out + 2 * mat_off + (int64_t)(tile.x * TG_M + q * 32) * n + col0 + lane * 4 : nullptr;
      float* ol = oh ? oh + n * n : nullptr;
      float* po = ep.out_plain ? ep.out_plain + mat_off + (int64_t)(tile.x * TG_M + q * 32) * n + col0 + lane * 4 : nullptr;
#pragma unroll 4
      for (int rr = 0; rr < 32; ++rr) {
        const float4 v = *reinterpret_cast<const float4*>(stw + (size_t)rr * TG_N + 4 * (lane ^ rr));
        if (oh) {
          float4 h;
          uint32_t t;
          asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(v.x)); h.x = __uint_as_float(t);
          asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(v.y)); h.y = __uint_as_float(t);
          asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(v.z)); h.z = __uint_as_float(t);
          asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(v.w)); h.w = __uint_as_float(t);
          *reinterpret_cast<float4*>(oh + (int64_t)rr * n) = h;
          *reinterpret_cast<float4*>(ol + (int64_t)rr * n) = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
        }
        if (po) *reinterpret_cast<float4*>(po + (int64_t)rr * n) = v;
      }
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

// planes: [batch][2][n][n] FP32 -> 3-D map (col, row, 2*batch + plane), box {32, 128, 2}
void make_tf32_planes_tensor_map(CUtensorMap* tm, const float* planes, int n, int batch) {
  const cuuint64_t gdim[3] = {(cuuint64_t)n, (cuuint64_t)n, (cuuint64_t)(2 * batch)};
  const cuuint64_t gstride[2] = {(cuuint64_t)n * 4, (cuuint64_t)n * n * 4};
  const cuuint32_t box[3] = {TG_KC, 128, 2};
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = tg_encode_fn()(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(planes), gdim, gstride, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  RG_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (tf32 planes) failed (" + std::to_string((int)r) + ")");
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

// identity planes [1][2][128][128] (hi = I, lo = 0) for the C phase
void make_tf32_identity_planes(DevBuf<float>& buf, CUtensorMap* tm) {
  std::vector<float> h((size_t)2 * 128 * 128, 0.f);
  for (int i = 0; i < 128; ++i) h[(size_t)i * 128 + i] = 1.f;
  buf.alloc(h.size());
  RG_CUDA(cudaMemcpy(buf.p, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
  make_tf32_planes_tensor_map(tm, buf.p, 128, 1);
}

void launch_tf32x3_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const int4* tiles, int ntiles, int batch,
                        const Tf32GemmEpilogue& ep, cudaStream_t s, const CUtensorMap* tmC, const CUtensorMap* tmI) {
  RG_CHECK(ep.c_chunks == 0 || (tmC && tmI), "tf32 gemm: the C phase needs its tensor maps");
  if (ntiles <= 0 || batch <= 0) return;
  const size_t smem = (size_t)TG_STAGES * TG_STAGE_BYTES + 1024 + 128;
  dim3 grid(ntiles, batch);
  ensure_dyn_smem(reinterpret_cast<const void*>(tf32x3_gemm_nt_kernel), smem);
  tf32x3_gemm_nt_kernel<<<grid, TG_THREADS, smem, s>>>(tmA, tmB, tmC ? *tmC : tmA, tmI ? *tmI : tmB, tiles, ep);
}

}  // namespace rg
