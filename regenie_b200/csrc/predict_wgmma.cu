// Out-of-fold level-0 predictions on the tensor cores, exactly.
//
//   pred[t, q] = sum_i gamma[i,q] g0(i,t) + sum_i (gamma mu)[i,q] miss(i,t) - x_t . cvec_q
// (reference: `beta.transpose() * Gmat.block(...)`, src/Step1_Models.cpp:503 - 2 P R bs N flops/block).
// The genotype operand is the same plane pair Z = [G0; Miss] the Gram kernel consumes: its bytes are 8 x dosage as int8
// (bed_expand_fp8_kernel).  The real-valued coefficients are split into FIVE balanced radix-254 digits
//   gamma[i,q] = (s_q / 127) * sum_l d_l[i,q] 254^-l,   d_l in {-127..127}  (int8),
// so the s8 x s8 -> s32 MMAs accumulate exact integer sums (|sum| <= K2 * 16 * 127 < 2^24 for K2 <= 4096) and the FP64
// epilogue reassembles the prediction to s_q 254^-5 = 9.4e-13 s_q per coefficient (the last limb is rounded to within 1/2,
// and one unit of it is worth (s_q / 127) 254^-4), far inside the 1e-5 parity budget.
//
// Orientation: samples are the MMA M dimension, the 5 x 50 digit rows are N (256, zero padded), the SNP/plane index
// is K.  The digit rows are K-major in shared memory (wgmma B operand).  The genotype tile arrives samples-contiguous
// (MN-major), which 8-bit wgmma cannot read from shared memory, so the A operand comes from registers.  Each consumer
// warpgroup owns one 64-sample half of the tile and all 256 digit rows (m64n256k32).  The two threads of a lane pair
// (lane, lane ^ 4) share 4 consecutive samples: each loads them at 4 consecutive k (one of the two k quads of the
// fragment) as four 32-bit words, transposes the 4 x 4 bytes with byte permutes, keeps its own two samples and trades
// the other two with its partner.  The fragments of stage s + 1 are built while the MMAs of stage s run.
#include <stdlib.h>

#include "kernels.cuh"
#include "wgmma_sm90.cuh"

namespace rg {

namespace {

using namespace sm90;

constexpr int PT_BM = 128;            // samples per CTA
constexpr int PT_BK = 128;            // Z rows per stage
constexpr int PI_BN = 256;            // digit rows (5 limbs x 50 outputs, zero padded)
constexpr int PI_STAGES = 4;
constexpr int PI_A_BYTES = PT_BK * PT_BM;          // 16 KiB: 128 k-rows x 128 samples
constexpr int PI_B_BYTES = PI_BN * PT_BK;          // 32 KiB: 256 digit rows x 128 k bytes
constexpr int PI_STAGE_BYTES = PI_A_BYTES + PI_B_BYTES;
constexpr int PI_THREADS = 288;                    // 2 consumer warpgroups (samples 0-63 / 64-127), 1 TMA warp
constexpr int PI_QH = kLimbQI8 / 2;                // outputs per epilogue thread (25)
constexpr int PI_LDE = PI_BN + 1;                  // row stride (int32) of the staged accumulator tile
static_assert(kLimbsI8 * kLimbQI8 <= PI_BN && kLimbQI8 % 2 == 0, "INT8 prediction layout");
static_assert(PT_BM * PI_LDE * 4 <= PI_STAGES * PI_STAGE_BYTES, "the accumulator tile reuses the stage buffers");

// 4 words W_i = bytes (k = i; samples 0..3)  ->  V_j = bytes (k = 0..3; sample j)
__device__ __forceinline__ void transpose4x4(const uint32_t (&w)[4], uint32_t (&v)[4]) {
  const uint32_t t0 = __byte_perm(w[0], w[1], 0x5140), t1 = __byte_perm(w[0], w[1], 0x7362);
  const uint32_t t2 = __byte_perm(w[2], w[3], 0x5140), t3 = __byte_perm(w[2], w[3], 0x7362);
  v[0] = __byte_perm(t0, t2, 0x5410);
  v[1] = __byte_perm(t0, t2, 0x7632);
  v[2] = __byte_perm(t1, t3, 0x5410);
  v[3] = __byte_perm(t1, t3, 0x7632);
}

}  // namespace

// digit rows  dig[f][g][l*50 + qq][k]  (int8), scales s[f][q].  grid: (Qp, K folds), block 256.
__global__ void __launch_bounds__(256)
l0_gamma_limbs_i8_kernel(const double* __restrict__ gam, const double* __restrict__ gmu, int Qp, int Q, int bs,
                         int rows_p, double* __restrict__ scale, uint8_t* __restrict__ dig, int ngroups) {
  __shared__ double red[256];
  const int q = blockIdx.x, f = blockIdx.y;
  if (q >= Q) return;
  const double* gcol = gam + (int64_t)f * rows_p * Qp + q;
  const double* mcol = gmu + (int64_t)f * rows_p * Qp + q;
  double mx = 0.0;
  for (int i = threadIdx.x; i < bs; i += 256)
    mx = fmax(mx, fmax(fabs(gcol[(int64_t)i * Qp]), fabs(mcol[(int64_t)i * Qp])));
  red[threadIdx.x] = mx;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + o]);
    __syncthreads();
  }
  const double s = red[0] > 0.0 ? red[0] : 1.0;
  if (threadIdx.x == 0) scale[(int64_t)f * Qp + q] = s;
  const int g = q / kLimbQI8, qq = q % kLimbQI8;
  const int K2 = 2 * rows_p;
  uint8_t* base = dig + ((int64_t)f * ngroups + g) * (int64_t)PI_BN * K2;
  for (int k = threadIdx.x; k < K2; k += 256) {
    const int plane = k >= rows_p, i = plane ? k - rows_p : k;
    double v = 0.0;
    if (i < bs) v = (plane ? mcol[(int64_t)i * Qp] : gcol[(int64_t)i * Qp]) / s * 127.0;
#pragma unroll
    for (int l = 0; l < kLimbsI8; ++l) {
      const double d = rint(v);                    // |v| <= 127: the remainder (<= 1/2) x 254 stays in range
      base[(int64_t)(l * kLimbQI8 + qq) * K2 + k] = (uint8_t)(int8_t)(int)d;
      v = (v - d) * 254.0;
    }
  }
}

// grid: (Npad / 128 sample tiles, q groups); 288 threads.
__global__ void __launch_bounds__(PI_THREADS, 1)
l0_predict_i8_kernel(const __grid_constant__ CUtensorMap tmZ, const __grid_constant__ CUtensorMap tmD, PredictTcArgs a) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gen_base = smem_raw + (base - raw);
  const uint32_t sA = base;                                         // [NST][16 KiB]
  const uint32_t sB = base + PI_STAGES * PI_A_BYTES;                // [NST][32 KiB]
  uint64_t* bars = reinterpret_cast<uint64_t*>(gen_base + PI_STAGES * PI_STAGE_BYTES);
  const uint32_t full_bar = smem_u32(bars);
  const uint32_t empty_bar = smem_u32(bars + PI_STAGES);
  double* s_scale = reinterpret_cast<double*>(bars + 2 * PI_STAGES);   // [kLimbQI8]
  double* s_cvec = s_scale + kLimbQI8;                                  // [kLimbQI8][C]

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role
  const int tile = blockIdx.x, g = blockIdx.y;
  const int f = a.tile_fold[tile];
  const int nkb = (2 * a.rows_p) / PT_BK;
  const int q0 = g * kLimbQI8;
  const int nq = min(kLimbQI8, a.Q - q0);

  if (warp == 8 && lane == 0) {
    for (int s = 0; s < PI_STAGES; ++s) { mbar_init(full_bar + 8 * s, 1); mbar_init(empty_bar + 8 * s, 2); }
    fence_barrier_init();
    prefetch_tmap(&tmZ);
    prefetch_tmap(&tmD);
  }
  for (int e = threadIdx.x; e < kLimbQI8; e += PI_THREADS)
    s_scale[e] = (e < nq) ? a.scale[(int64_t)f * a.Qp + q0 + e] / 127.0 : 0.0;
  for (int e = threadIdx.x; e < kLimbQI8 * a.C; e += PI_THREADS) {
    const int qq = e / a.C, c = e % a.C;
    s_cvec[e] = (qq < nq) ? a.cvec[((int64_t)f * a.Qp + q0 + qq) * a.C + c] : 0.0;
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      // ===== TMA producer: A = 128 plane rows x 128 samples; B = 256 digit rows x 128 k bytes =====
      const int drow0 = (f * a.ngroups + g) * PI_BN;
      for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % PI_STAGES;
        const uint32_t ph = (kb / PI_STAGES) & 1;
        mbar_wait(empty_bar + 8 * s, ph ^ 1);
        mbar_expect_tx(full_bar + 8 * s, PI_STAGE_BYTES);
        tma_load_2d(sA + s * PI_A_BYTES, &tmZ, full_bar + 8 * s, tile * PT_BM, kb * PT_BK);
        tma_load_2d(sB + s * PI_B_BYTES, &tmD, full_bar + 8 * s, kb * PT_BK, drow0);
        tma_load_2d(sB + s * PI_B_BYTES + 16384, &tmD, full_bar + 8 * s, kb * PT_BK, drow0 + 128);
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg = samples 64 wg .. 64 wg + 63 x all 256 digit rows =====
  // Thread (warp w of the warpgroup, lane l, r = l / 4, t4 = l % 4) holds fragment rows 16 w + r and 16 w + r + 8, which
  // are samples 64 wg + 16 w + 2 r and the next one.  The pair (r, r ^ 1) shares the 4 samples from sq = 64 wg + 16 w +
  // 4 (r / 2): the even thread loads them at the k quad 4 t4 .. +3 of each MMA, the odd one at 16 + 4 t4 .. +3.
  const int wg = warp >> 2, w = warp & 3, r = lane >> 2, t4 = lane & 3;
  const bool odd = r & 1;
  const int sq = 64 * wg + 16 * w + 4 * (r >> 1);
  // The 8 lanes reading one 16-byte sample chunk take the 4 k rows of their quad in rotated orders (rot = 0..3), so each
  // load instruction of the warp meets 8 distinct swizzle phases, i.e. 32 distinct banks.  rsel undoes the rotation.
  const int rot = 2 * odd + (t4 >> 1);
  const uint32_t rsel = (0x32103210u >> (16 - 4 * rot)) & 0xFFFFu;
  int aoff[4];                                      // byte offset of load i inside a 32-k slice of the A stage
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int kr = 16 * odd + 4 * t4 + ((i + rot) & 3);          // row of the 128B-swizzled tile
    aoff[i] = kr * 128 + ((((sq >> 4) ^ (kr & 7)) << 4) | (sq & 15));
  }
  const uint8_t* gA = gen_base;                     // generic view of the A stages

  // A fragment of MMA kk of stage s: {row, row + 8} x {k 4 t4 .. +3, k 16 + 4 t4 .. +3} of the stage's 32-k slice kk
  auto build = [&](int s, int kk, uint32_t (&af)[4]) {
    uint32_t wv[4], v[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
      wv[i] = *reinterpret_cast<const uint32_t*>(gA + s * PI_A_BYTES + kk * 32 * 128 + aoff[i]);
    transpose4x4(wv, v);                            // v[j] = sample sq + j at the quad's k, rotated by rot bytes
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = __byte_perm(v[j], 0, rsel);
    const uint32_t x0 = __shfl_xor_sync(0xffffffffu, odd ? v[0] : v[2], 4);
    const uint32_t x1 = __shfl_xor_sync(0xffffffffu, odd ? v[1] : v[3], 4);
    af[0] = odd ? x0 : v[0];
    af[1] = odd ? x1 : v[1];
    af[2] = odd ? v[2] : x0;
    af[3] = odd ? v[3] : x1;
  };
  // One commit group per MMA, two fragment register sets: while MMA u runs, MMA u - 1 is retired (freeing its fragment
  // registers, and at the first MMA of a stage the previous stage's buffers) and the fragment of MMA u + 1 is built.
  // Double-buffering whole stages would need 32 fragment registers beside the 128 accumulators, more than the 168 a
  // thread gets at 288 threads per SM.
  int32_t acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0;
  fence_regs(acc);
  uint32_t afr[2][4];
  mbar_wait(full_bar, 0);
  build(0, 0, afr[0]);
  for (int kb = 0; kb < nkb; ++kb) {
    const int s = kb % PI_STAGES;
    const uint64_t db = desc_k128(sB + s * PI_B_BYTES);
#pragma unroll
    for (int kk = 0; kk < PT_BK / 32; ++kk) {
      wgmma_fence();
      // +32 bytes (K of one MMA) inside the 128-byte swizzle atom: +2 in 16-byte units
      wgmma_s8_rs_n256(acc, afr[kk & 1], db + (uint64_t)(2 * kk));
      wgmma_commit();
      wgmma_wait<1>();
      if (kk == 0 && kb > 0 && w == 0 && lane == 0) mbar_arrive(empty_bar + 8 * ((kb - 1) % PI_STAGES));
      if (kk + 1 < PT_BK / 32) {
        build(s, kk + 1, afr[(kk + 1) & 1]);
      } else if (kb + 1 < nkb) {
        mbar_wait(full_bar + 8 * ((kb + 1) % PI_STAGES), ((kb + 1) / PI_STAGES) & 1);
        build((kb + 1) % PI_STAGES, 0, afr[0]);
      }
    }
  }
  wgmma_wait<0>();
  fence_regs(acc);

  // ===== epilogue: accumulators -> shared memory tile E[sample][digit row] (the stage buffers are free once every
  // consumer is past its last MMA) -> thread = (sample, half of the outputs).  Limb sums are exact int32 multiples of 8;
  // FP64 Horner from the lowest limb up.
  named_sync(1, 256);
  int32_t* E = reinterpret_cast<int32_t*>(gen_base);
#pragma unroll
  for (int i = 0; i < 128; ++i) {
    const int smp = 64 * wg + 16 * w + 2 * r + ((i >> 1) & 1);
    const int col = 8 * (i >> 2) + 2 * t4 + (i & 1);
    E[smp * PI_LDE + col] = acc[i];
  }
  named_sync(1, 256);
  {
    const int ct = threadIdx.x;                    // 0..255
    const int smp = ct & 127, half = ct >> 7;
    const int t = tile * PT_BM + smp;
    const int32_t* er = E + smp * PI_LDE + half * PI_QH;
    const double inv254 = 1.0 / 254.0;
    double accd[PI_QH];
#pragma unroll
    for (int j = 0; j < PI_QH; ++j) accd[j] = 0.0;
#pragma unroll
    for (int l = kLimbsI8 - 1; l >= 0; --l) {
#pragma unroll
      for (int j = 0; j < PI_QH; ++j) accd[j] = fma(accd[j], inv254, (double)(er[l * kLimbQI8 + j] >> 3));
    }
    double xr[kMaxCov];
    for (int c = 0; c < a.C; ++c) xr[c] = a.xy[(int64_t)t * a.cpp + c];
#pragma unroll
    for (int j = 0; j < PI_QH; ++j) {
      const int qq = half * PI_QH + j;
      if (qq < nq) {
        const int q = q0 + qq;
        const int r = q / a.P, p = q % a.P;
        double val = accd[j] * s_scale[qq];
        for (int c = 0; c < a.C; ++c) val -= xr[c] * s_cvec[qq * a.C + c];
        val *= (double)a.mask[(int64_t)p * a.npad + t];
        a.W[p][(int64_t)(a.col0 + r) * a.npad + t] = val;
      }
    }
  }
}

// Column sums of the raw predictions for the standardisation: part[chunk][q] = (sum, sum of squares) over
// a chunk of 8192 samples, fixed-order tree reduction.  grid: (Q, nchunks), block 256.
__global__ void __launch_bounds__(256)
l0_colsum_kernel(double* const* __restrict__ W, int64_t npad, int col0, int P, int Qp,
                 double* __restrict__ part) {
  __shared__ double r1[256], r2[256];
  const int q = blockIdx.x, r = q / P, p = q % P;
  const int64_t t0 = (int64_t)blockIdx.y * 8192;
  const double* w = W[p] + (int64_t)(col0 + r) * npad;
  double s1 = 0.0, s2 = 0.0;
  for (int64_t t = t0 + threadIdx.x; t < min(t0 + 8192, npad); t += 256) {
    const double v = w[t];
    s1 += v;
    s2 = fma(v, v, s2);
  }
  r1[threadIdx.x] = s1; r2[threadIdx.x] = s2;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) { r1[threadIdx.x] += r1[threadIdx.x + o]; r2[threadIdx.x] += r2[threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    part[((int64_t)blockIdx.y * Qp + q) * 2 + 0] = r1[0];
    part[((int64_t)blockIdx.y * Qp + q) * 2 + 1] = r2[0];
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

void launch_l0_gamma_limbs_i8(const double* gam, const double* gmu, int Qp, int Q, int bs, int rows_p, int K,
                              double* scale, uint8_t* dig, int ngroups, cudaStream_t s) {
  dim3 grid(Qp, K);
  l0_gamma_limbs_i8_kernel<<<grid, 256, 0, s>>>(gam, gmu, Qp, Q, bs, rows_p, scale, dig, ngroups);
}

void launch_l0_predict_i8(const CUtensorMap& tmZ, const CUtensorMap& tmD, const PredictTcArgs& a, int ntiles,
                          cudaStream_t s) {
  RG_CHECK(2 * a.rows_p <= 4096, "INT8 prediction: 2 * rows_p <= 4096 (int32 Horner bound)");
  const size_t smem = (size_t)PI_STAGES * PI_STAGE_BYTES + 1024 + 128 + ((size_t)kLimbQI8 * (1 + a.C)) * sizeof(double);
  ensure_dyn_smem(reinterpret_cast<const void*>(l0_predict_i8_kernel), smem);
  l0_predict_i8_kernel<<<dim3(ntiles, a.ngroups), PI_THREADS, smem, s>>>(tmZ, tmD, a);
}

}  // namespace rg
