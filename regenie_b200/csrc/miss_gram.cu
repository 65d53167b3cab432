// The Miss rows of the per-fold integer Gram Z_f Z_f^T (gram_wgmma.cu) as sparse sums over the missing calls.
//
// Z = [G0; Miss].  Row rows_p + i of Z Z^T is Miss_i [G0; Miss]^T, and Miss_i is zero except at the samples where SNP i
// has no call, so per fold f
//   (Miss G0^T)_f[i, j]  = sum over s in miss(i) & f of G0[j, s]
//   (Miss Miss^T)_f[i, j] = #{ s in miss(i) & f : Miss[j, s] }
// With array-typed data (call rate 98-99 % and up) that is a few hundred samples per (SNP, fold) instead of the fold's
// whole length, and those rows are 2/3 of the Gram's dense 128 x 256 tiles at rows_p = 1024.
//
// The lists and the sample-major rows come from the relayout pass (bed_kernels.cu, launch_bed_relayout_miss), which
// reads the PLINK rows once for gp, Gt and the lists: per (SNP row, column tile of at most 512 samples inside one fold)
// a segment (offset, count) of the lane's list buffer, reserved with one atomic per 128-row tile.  The block's running
// total doubles as the path flag: when it exceeds the buffer (a missing rate above the crossover), the dense Miss tiles
// run instead.  Gt[Npad][rows_p / 16] is the block as sample-major 2-bit rows, so that a missing call reads rows_p / 4
// contiguous bytes.
//
//   miss_sparse_kernel     one warp per (SNP row, fold) walks the segments of the fold's column tiles and adds Gt rows
//                          with SWAR on packed fields; writes the FP32 values at every position the dense Miss tiles
//                          write.
// All sums are integer sums, so the result is bit-identical to the dense tiles whatever the order of the samples.
#include "kernels.cuh"

namespace rg {

namespace {

constexpr int kChunkWords = 64;      // Gt words per column chunk of the sparse kernel: lane owns words lane, lane + 32
constexpr int kSparseWarps = 4;
constexpr int kCodeStride = kChunkWords + 1;   // shared accumulators [code][word], padded against bank conflicts
constexpr int kBatch = 126;          // calls per batch: the 8-bit fields hold 126 calls

// Fills smp[0 .. kBatch) with the next calls of one (SNP row, fold), -1 past the last one, and returns how many it
// took.  The calls lie in the segments sg[ct] of column tiles ct = ct .. ct1 - 1, `used` of tile ct taken already;
// 32 tiles are looked at per step, their counts scanned across the warp, and each lane copies its own tile's part.
__device__ __forceinline__ int miss_fill_batch(const int2* __restrict__ sg, int& ct, int ct1, int& used,
                                               const int32_t* __restrict__ list, int* smp, int lane) {
  int n = 0;
  while (n < kBatch && ct < ct1) {
    int2 e = ct + lane < ct1 ? __ldg(sg + ct + lane) : make_int2(0, 0);
    if (lane == 0) { e.x += used; e.y -= used; }
    int inc = e.y;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += u;
    }
    const int room = kBatch - n, exc = inc - e.y;
    const int take = max(0, min(e.y, room - exc));
    for (int k = 0; k < take; ++k) smp[n + exc + k] = __ldg(list + e.x + k);
    const int all = __shfl_sync(0xffffffffu, inc, 31);
    if (all <= room) {
      n += all;
      ct = min(ct + 32, ct1);
      used = 0;
    } else {                                  // the batch is full inside the tile of lane l
      const int l = __ffs(__ballot_sync(0xffffffffu, inc > room)) - 1;
      used = (l == 0 ? used : 0) + __shfl_sync(0xffffffffu, take, l);
      ct += l;
      n = kBatch;
    }
  }
  for (int k = n + lane; k < 128; k += 32) smp[k] = -1;
  __syncwarp();
  return n;
}

}  // namespace

// grid (rows_p / kSparseWarps, K), block 32 kSparseWarps.  Warp w of block b owns Miss row i = kSparseWarps b + w in fold
// blockIdx.y and writes zz row rows_p + i over the columns the dense tile list covers for it.
//
// Accumulation: a Gt word holds 16 codes.  G0 values (code 3 read as 0) and missing bits go into 4-bit fields, the even
// and the odd codes of the word in separate registers (at most 2 per call: 7 calls fit), those into 8-bit fields every
// 7 calls (126 calls fit), and those into 32-bit sums in shared memory every 126 calls.
__global__ void __launch_bounds__(32 * kSparseWarps)
miss_sparse_kernel(const uint32_t* __restrict__ gt, int rows_p, const int2* __restrict__ seg, int nct,
                   const int2* __restrict__ fold_ct, const int32_t* __restrict__ list,
                   const unsigned long long* __restrict__ total, unsigned long long cap, float* __restrict__ zz,
                   int64_t fold_stride) {
  if (*total > cap) return;
  __shared__ uint32_t acc_s[kSparseWarps][2][16 * kCodeStride];
  __shared__ int smp_s[kSparseWarps][128];        // the samples of the current batch
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * kSparseWarps + warp, f = blockIdx.y;
  uint32_t* sG = acc_s[warp][0];
  uint32_t* sM = acc_s[warp][1];
  int* sSmp = smp_s[warp];
  const int2* sg = seg + (int64_t)i * nct;
  const int2 fct = fold_ct[f];
  const int gw = rows_p / 16;
  const int r = rows_p + i;
  const int colmax = min(2 * rows_p, 256 * ((r / 128) / 2 + 1));     // gram_tile_list: tiles (mi, nj) with 2 nj <= mi
  float* out = zz + (int64_t)f * fold_stride + (int64_t)r * (2 * rows_p);
  constexpr int off[4] = {0, 2, 1, 3};

  for (int w0 = 0; w0 < gw; w0 += kChunkWords) {
    for (int k = lane; k < 16 * kCodeStride; k += 32) { sG[k] = 0; sM[k] = 0; }
    __syncwarp();
    int ct = fct.x, used = 0;
    for (;;) {
      const int n = miss_fill_batch(sg, ct, fct.y, used, list, sSmp, lane);
      if (n == 0) break;
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

void launch_miss_sparse(const uint32_t* gt, int rows_p, const int2* seg, int nct, const int2* fold_ct,
                        const int32_t* list, int K, const unsigned long long* total, int64_t cap, float* zz,
                        int64_t fold_stride, cudaStream_t s) {
  miss_sparse_kernel<<<dim3(rows_p / kSparseWarps, K), 32 * kSparseWarps, 0, s>>>(
      gt, rows_p, seg, nct, fold_ct, list, total, (unsigned long long)cap, zz, fold_stride);
}

}  // namespace rg
