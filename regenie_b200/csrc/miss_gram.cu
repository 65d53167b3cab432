// The Miss rows of the per-fold integer Gram Z_f Z_f^T (gram_wgmma.cu) as sparse sums over the missing calls.
//
// Z = [G0; Miss].  Row rows_p + i of Z Z^T is Miss_i [G0; Miss]^T, and Miss_i is zero except at the samples where SNP i
// has no call, so per fold f
//   (Miss G0^T)_f[i, j]  = sum over s in miss(i) & f of G0[j, s]
//   (Miss Miss^T)_f[i, j] = #{ s in miss(i) & f : Miss[j, s] }
// With array-typed data (call rate 98-99 % and up) that is a few hundred samples per (SNP, fold) instead of the fold's
// whole length, and those rows are 2/3 of the Gram's dense 128 x 256 tiles at rows_p = 1024.
//
//   miss_list_kernel       per (SNP row, fold): count the missing calls, take a segment of the lane's list buffer with
//                          one atomic, write the samples into it.  The running total doubles as the path flag: when it
//                          exceeds the buffer (a missing rate above the crossover), the dense Miss tiles run instead.
//   miss_transpose_kernel  the block as sample-major 2-bit rows Gt[Npad][rows_p / 16], so that a missing call reads
//                          rows_p / 4 contiguous bytes.
//   miss_sparse_kernel     one warp per (SNP row, fold) walks its segment and adds Gt rows with SWAR on packed fields;
//                          writes the FP32 values at every position the dense Miss tiles write.
// All sums are integer sums, so the result is bit-identical to the dense tiles whatever the order of the samples.
#include "kernels.cuh"

namespace rg {

namespace {

// bit 2k set where the 2-bit code k of w is 3 (missing)
__device__ __forceinline__ uint32_t miss_bits(uint32_t w) { return w & (w >> 1) & 0x55555555u; }

constexpr int kListThreads = 256;
constexpr int kChunkWords = 64;      // Gt words per column chunk of the sparse kernel: lane owns words lane, lane + 32
constexpr int kSparseWarps = 4;
constexpr int kCodeStride = kChunkWords + 1;   // shared accumulators [code][word], padded against bank conflicts

}  // namespace

// grid (rows_p, K), block kListThreads
__global__ void __launch_bounds__(kListThreads)
miss_list_kernel(const uint32_t* __restrict__ gp, int64_t wpr, int rows_p, const int2* __restrict__ fold_k,
                 unsigned long long* __restrict__ total, unsigned long long cap, int2* __restrict__ seg,
                 int32_t* __restrict__ list) {
  const int i = blockIdx.x, f = blockIdx.y;
  const int2 fk = fold_k[f];
  const int64_t w0 = (int64_t)fk.x * (kSamplePad / 16), w1 = (int64_t)(fk.x + fk.y) * (kSamplePad / 16);
  const uint32_t* row = gp + (int64_t)i * wpr;
  __shared__ int warp_cnt[kListThreads / 32];
  __shared__ unsigned long long base_s;
  __shared__ int pos_s;
  int n = 0;
  for (int64_t w = w0 + threadIdx.x; w < w1; w += kListThreads) n += __popc(miss_bits(__ldg(row + w)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int cnt = 0;
    for (int k = 0; k < kListThreads / 32; ++k) cnt += warp_cnt[k];
    const unsigned long long base = cnt ? atomicAdd(total, (unsigned long long)cnt) : 0ull;
    seg[(int64_t)f * rows_p + i] = make_int2((int)(base + cnt <= cap ? base : 0), base + cnt <= cap ? cnt : 0);
    base_s = base + cnt <= cap ? base : ~0ull;
    pos_s = 0;
  }
  __syncthreads();
  const unsigned long long base = base_s;
  if (base == ~0ull) return;                  // the list is full: this block runs on the dense tiles
  for (int64_t w = w0 + threadIdx.x; w < w1; w += kListThreads) {
    uint32_t m = miss_bits(__ldg(row + w));
    if (!m) continue;
    int p = atomicAdd(&pos_s, __popc(m));
    for (; m; m &= m - 1) list[base + p++] = (int32_t)(w * 16 + (__ffs(m) - 1) / 2);
  }
}

// gp [rows_p][wpr] -> Gt [wpr * 16][rows_p / 16].  grid (ceil(wpr / 32), rows_p / 128), block 256: a tile of 128 SNP
// rows x 32 words (512 samples); each thread builds the 8 output words (128 SNPs) of two samples.
__global__ void __launch_bounds__(256)
miss_transpose_kernel(const uint32_t* __restrict__ gp, int64_t wpr, int rows_p,
                      const unsigned long long* __restrict__ total, unsigned long long cap, uint32_t* __restrict__ gt) {
  if (*total > cap) return;
  __shared__ uint32_t t[128][33];
  const int64_t wb = (int64_t)blockIdx.x * 32;
  const int r0 = blockIdx.y * 128;
  for (int k = threadIdx.x; k < 128 * 32; k += 256) {
    const int r = k >> 5, c = k & 31;
    t[r][c] = (wb + c < wpr) ? __ldg(gp + (int64_t)(r0 + r) * wpr + wb + c) : 0u;
  }
  __syncthreads();
  const int gw = rows_p / 16;
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int sl = threadIdx.x + 256 * q;
    const int c = sl >> 4, sh = 2 * (sl & 15);
    if (wb + c >= wpr) continue;
    uint32_t o[8];
#pragma unroll
    for (int jw = 0; jw < 8; ++jw) {
      uint32_t v = 0;
#pragma unroll
      for (int r = 0; r < 16; ++r) v |= ((t[jw * 16 + r][c] >> sh) & 3u) << (2 * r);
      o[jw] = v;
    }
    uint4* dst = reinterpret_cast<uint4*>(gt + (wb * 16 + sl) * gw + blockIdx.y * 8);
    dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
    dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
  }
}

// grid (rows_p / kSparseWarps, K), block 32 kSparseWarps.  Warp w of block b owns Miss row i = kSparseWarps b + w in fold
// blockIdx.y and writes zz row rows_p + i over the columns the dense tile list covers for it.
//
// Accumulation: a Gt word holds 16 codes.  G0 values (code 3 read as 0) and missing bits go into 4-bit fields, the even
// and the odd codes of the word in separate registers (at most 2 per call: 7 calls fit), those into 8-bit fields every
// 7 calls (126 calls fit), and those into 32-bit sums in shared memory every 126 calls.
__global__ void __launch_bounds__(32 * kSparseWarps)
miss_sparse_kernel(const uint32_t* __restrict__ gt, int rows_p, const int2* __restrict__ seg,
                   const int32_t* __restrict__ list, const unsigned long long* __restrict__ total,
                   unsigned long long cap, float* __restrict__ zz, int64_t fold_stride) {
  if (*total > cap) return;
  __shared__ uint32_t acc_s[kSparseWarps][2][16 * kCodeStride];
  __shared__ int smp_s[kSparseWarps][128];        // the samples of the current 126 calls, loaded coalesced
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * kSparseWarps + warp, f = blockIdx.y;
  uint32_t* sG = acc_s[warp][0];
  uint32_t* sM = acc_s[warp][1];
  int* sSmp = smp_s[warp];
  const int2 sg = seg[(int64_t)f * rows_p + i];
  const int32_t* lst = list + sg.x;
  const int cnt = sg.y;
  const int gw = rows_p / 16;
  const int r = rows_p + i;
  const int colmax = min(2 * rows_p, 256 * ((r / 128) / 2 + 1));     // gram_tile_list: tiles (mi, nj) with 2 nj <= mi
  float* out = zz + (int64_t)f * fold_stride + (int64_t)r * (2 * rows_p);
  constexpr int off[4] = {0, 2, 1, 3};

  for (int w0 = 0; w0 < gw; w0 += kChunkWords) {
    for (int k = lane; k < 16 * kCodeStride; k += 32) { sG[k] = 0; sM[k] = 0; }
    __syncwarp();
    for (int b0 = 0; b0 < cnt; b0 += 126) {
      const int n = min(cnt - b0, 126);
#pragma unroll
      for (int k = 0; k < 4; ++k) sSmp[32 * k + lane] = 32 * k + lane < n ? __ldg(lst + b0 + 32 * k + lane) : -1;
      __syncwarp();
      uint32_t g8[2][4] = {}, m8[2][4] = {};
      for (int g0 = 0; g0 < n; g0 += 7) {
        uint32_t g4[2][2] = {}, m4[2][2] = {};
        int smp[7];
#pragma unroll
        for (int u = 0; u < 7; ++u) smp[u] = sSmp[g0 + u];
#pragma unroll
        for (int u = 0; u < 7; ++u) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int w = w0 + lane + 32 * h;
            const uint32_t x = (smp[u] >= 0 && w < gw) ? __ldg(gt + (int64_t)smp[u] * gw + w) : 0u;
            const uint32_t m = miss_bits(x);
            const uint32_t gx = x & ~(m * 3u);                  // G0: the missing code reads as 0
            g4[h][0] += gx & 0x33333333u;                       // nibble n: code 2n
            g4[h][1] += (gx >> 2) & 0x33333333u;                // nibble n: code 2n + 1
            m4[h][0] += m & 0x11111111u;
            m4[h][1] += (m >> 2) & 0x11111111u;
          }
        }
        // byte b of field q holds code 4 b + off[q]
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          g8[h][0] += g4[h][0] & 0x0F0F0F0Fu;
          g8[h][1] += (g4[h][0] >> 4) & 0x0F0F0F0Fu;
          g8[h][2] += g4[h][1] & 0x0F0F0F0Fu;
          g8[h][3] += (g4[h][1] >> 4) & 0x0F0F0F0Fu;
          m8[h][0] += m4[h][0] & 0x0F0F0F0Fu;
          m8[h][1] += (m4[h][0] >> 4) & 0x0F0F0F0Fu;
          m8[h][2] += m4[h][1] & 0x0F0F0F0Fu;
          m8[h][3] += (m4[h][1] >> 4) & 0x0F0F0F0Fu;
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
          for (int b = 0; b < 4; ++b) {
            const int k = (4 * b + off[q]) * kCodeStride + lane + 32 * h;
            sG[k] += (g8[h][q] >> (8 * b)) & 0xFFu;
            sM[k] += (m8[h][q] >> (8 * b)) & 0xFFu;
          }
      __syncwarp();
    }
    __syncwarp();
    // column j of the chunk = SNP 16 w + code: Miss G0^T at column j, Miss Miss^T at column rows_p + j
    const int j0 = 16 * w0, j1 = min(rows_p, 16 * (w0 + kChunkWords));
    for (int j = j0 + lane; j < j1; j += 32) {
      const int k = (j & 15) * kCodeStride + (j >> 4) - w0;
      out[j] = (float)sG[k];
      if (rows_p + j < colmax) out[rows_p + j] = (float)sM[k];
    }
    __syncwarp();
  }
}

void launch_miss_list(const uint32_t* gp, int64_t npad, int rows_p, const int2* fold_k, int K, unsigned long long* total,
                      int64_t cap, int2* seg, int32_t* list, cudaStream_t s) {
  RG_CUDA(cudaMemsetAsync(total, 0, sizeof(unsigned long long), s));
  miss_list_kernel<<<dim3(rows_p, K), kListThreads, 0, s>>>(gp, npad / 16, rows_p, fold_k, total, (unsigned long long)cap,
                                                            seg, list);
}

void launch_miss_transpose(const uint32_t* gp, int64_t npad, int rows_p, const unsigned long long* total, int64_t cap,
                           uint32_t* gt, cudaStream_t s) {
  const int64_t wpr = npad / 16;
  miss_transpose_kernel<<<dim3((unsigned)ceil_div(wpr, 32), rows_p / 128), 256, 0, s>>>(gp, wpr, rows_p, total,
                                                                                          (unsigned long long)cap, gt);
}

void launch_miss_sparse(const uint32_t* gt, int rows_p, const int2* seg, const int32_t* list, int K,
                        const unsigned long long* total, int64_t cap, float* zz, int64_t fold_stride, cudaStream_t s) {
  miss_sparse_kernel<<<dim3(rows_p / kSparseWarps, K), 32 * kSparseWarps, 0, s>>>(gt, rows_p, seg, list, total,
                                                                                   (unsigned long long)cap, zz, fold_stride);
}

}  // namespace rg
