// Genotype-block layout kernel: PLINK 2-bit rows -> internal padded 2-bit rows (the tensor-core Gram and prediction
// kernels build their int8 operand bytes from these on chip).  Replaces the decode half of readChunkFromBedFileToG
// (reference src/Geno.cpp:1702-1768, LUT src/Geno.cpp:2833-2857); mean imputation is NOT
// materialised: missing calls stay a separate indicator plane and the mean enters as an exact
// rank-structured correction (see DESIGN.md "missing data").
//
// The Step-1 variant (kMiss) also writes, from the same tile in shared memory, what the sparse Miss rows of the level-0
// Gram read (miss_gram.cu): the block as sample-major 2-bit rows and the lists of the missing calls.
#include "kernels.cuh"

namespace rg {

// PLINK code v=(byte>>2k)&3 : 0 -> 2, 1 -> missing, 2 -> 1, 3 -> 0   (ref-last, src/Geno.cpp:2843)
// internal code: dosage 0/1/2, 3 = missing.  Packed LUTs, 2 bits per PLINK code.
__device__ __forceinline__ uint32_t plink_to_code(uint32_t v, int ref_first) {
  // ref-last : v=0->2(10) 1->3(11) 2->1(01) 3->0(00)  => 0b00011110
  // ref-first: v=0->0(00) 1->3(11) 2->1(01) 3->2(10)  => 0b10011100   (2-g, src/Geno.cpp:1746)
  const uint32_t lut = ref_first ? 0x9Cu : 0x1Eu;
  return (lut >> (2 * v)) & 3u;
}

// One output 32-bit word (16 samples) of one row.  Almost every word maps to 16 CONSECUTIVE samples of the file row
// (folds only shift whole ranges; --remove breaks a word here and there): those take the fast path - five source bytes,
// one funnel shift, the code translation as bit logic on all 16 lanes, a keep mask for samples outside the analysis.
// word_base[w] = file index of the word's first sample, -1 = nothing to read, -2 = not contiguous.
__device__ __forceinline__ uint32_t bed_word(const uint8_t* __restrict__ packed, int64_t row_stride, int row, int bs,
                                             int64_t w, const int32_t* __restrict__ file_idx_pad,
                                             const int32_t* __restrict__ word_base,
                                             const uint32_t* __restrict__ word_keep, int ref_first) {
  uint32_t out = 0;
  const int base = (row < bs) ? __ldg(word_base + w) : -1;
  if (base >= 0) {
    const uint8_t* p = packed + (int64_t)row * row_stride + (base >> 2);
    const int64_t left = row_stride - (base >> 2);            // bytes available in this row
    uint64_t x = 0;
#pragma unroll
    for (int b = 0; b < 5; ++b)
      if (b < left) x |= (uint64_t)__ldg(p + b) << (8 * b);
    const uint32_t v = (uint32_t)(x >> (2 * (base & 3)));
    const uint32_t H = (v >> 1) & 0x55555555u, Lo = v & 0x55555555u;
    const uint32_t oh = ref_first ? Lo : (~H & 0x55555555u);  // see plink_to_code
    out = ((oh << 1) | (H ^ Lo)) & __ldg(word_keep + w);
  } else if (base == -2) {
    const uint8_t* prow = packed + (int64_t)row * row_stride;
    const int4* fi4 = reinterpret_cast<const int4*>(file_idx_pad + w * 16);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int4 f = __ldg(fi4 + q);
      const int fi[4] = {f.x, f.y, f.z, f.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        uint32_t code = 0;
        if (fi[k] >= 0) {
          const uint32_t b = __ldg(prow + (fi[k] >> 2));
          code = plink_to_code((b >> (2 * (fi[k] & 3))) & 3u, ref_first);
        }
        out |= code << (2 * (q * 4 + k));
      }
    }
  }
  return out;
}

namespace {

constexpr int kTileRows = 128;     // SNP rows per CTA
constexpr int kTileWords = 32;     // 2-bit words per row of a CTA: 512 samples
constexpr int kRelayoutThreads = 256;

__device__ __forceinline__ int warp_inclusive_scan(int v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  return v;
}

}  // namespace

// grid (column tiles, rows_p / 128), block 256: a tile of 128 SNP rows x up to 32 words (512 samples).  Every thread
// decodes 16 words (a warp: one row's 32 words at a time) and writes them to gp.
//
// kMiss (Step 1, sparse Miss rows): column tile ct = ctile[ct] (first word, words, fold) lies inside one fold.  From the
// tile in shared memory the CTA counts the missing calls per row, reserves one range of the list buffer for all 128
// rows with one atomic on the block's running total, and writes
//   seg[row][ct]  = (offset, count) of the row's calls in this tile (in sample order),
//   list          = the samples (indices into the padded layout),
//   gt            = the tile as sample-major 2-bit rows Gt[Npad][rows_p / 16] (a missing call reads rows_p / 4
//                   contiguous bytes).
// Once the total exceeds cap the block runs on the dense Miss tiles: a CTA whose range does not fit writes neither
// its lists nor gt (nothing reads them).
template <bool kMiss>
__global__ void __launch_bounds__(kRelayoutThreads)
bed_relayout_kernel(const uint8_t* __restrict__ packed, int64_t row_stride, int bs,
                    const int32_t* __restrict__ file_idx_pad, const int32_t* __restrict__ word_base,
                    const uint32_t* __restrict__ word_keep, int ref_first, uint32_t* __restrict__ gp, int64_t wpr,
                    BedMissOut mo) {
  const int r0 = blockIdx.y * kTileRows;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t w0;
  int nw;
  if constexpr (kMiss) {
    const int4 ct = __ldg(mo.ctile + blockIdx.x);
    w0 = ct.x;
    nw = ct.y;
  } else {
    w0 = (int64_t)blockIdx.x * kTileWords;
    nw = (int)(wpr - w0 < kTileWords ? wpr - w0 : kTileWords);
  }
  __shared__ uint32_t t[kMiss ? kTileRows : 1][kTileWords + 1];
#pragma unroll 2
  for (int r = warp; r < kTileRows; r += kRelayoutThreads / 32) {
    const int row = r0 + r;
    uint32_t v = 0;
    if (lane < nw) {
      v = bed_word(packed, row_stride, row, bs, w0 + lane, file_idx_pad, word_base, word_keep, ref_first);
      gp[(int64_t)row * wpr + w0 + lane] = v;
    }
    if constexpr (kMiss) t[r][lane] = v;
  }
  if constexpr (kMiss) {
    __shared__ int cnt_s[kTileRows], pre_s[kTileRows];
    __shared__ unsigned long long base_s;
    __syncthreads();
    for (int r = warp; r < kTileRows; r += kRelayoutThreads / 32) {
      const int n = __reduce_add_sync(0xffffffffu, (unsigned)__popc(miss_bits(t[r][lane])));
      if (lane == 0) cnt_s[r] = n;
    }
    __syncthreads();
    if (warp == 0) {
      int c[4], sum = 0;
#pragma unroll
      for (int q = 0; q < 4; ++q) { c[q] = cnt_s[4 * lane + q]; sum += c[q]; }
      const int inc = warp_inclusive_scan(sum, lane);
      int p = inc - sum;
#pragma unroll
      for (int q = 0; q < 4; ++q) { pre_s[4 * lane + q] = p; p += c[q]; }
      if (lane == 31) {
        const unsigned long long base = inc ? atomicAdd(mo.total, (unsigned long long)inc) : 0ull;
        base_s = base + inc <= mo.cap ? base : ~0ull;
      }
    }
    __syncthreads();
    const unsigned long long base = base_s;
    if (base == ~0ull) return;                  // the list is full: this block runs on the dense tiles
    if (threadIdx.x < kTileRows)
      mo.seg[(int64_t)(r0 + threadIdx.x) * mo.nct + blockIdx.x] =
          make_int2((int)(base + pre_s[threadIdx.x]), cnt_s[threadIdx.x]);
    for (int r = warp; r < kTileRows; r += kRelayoutThreads / 32) {
      if (!cnt_s[r]) continue;
      uint32_t m = miss_bits(t[r][lane]);
      const int n = __popc(m);
      int64_t p = (int64_t)base + pre_s[r] + warp_inclusive_scan(n, lane) - n;
      for (; m; m &= m - 1) mo.list[p++] = (int32_t)((w0 + lane) * 16 + (__ffs(m) - 1) / 2);
    }
    // Gt: thread (c, jw) transposes the 16 x 16 block of 2-bit codes of rows 16 jw .. 16 jw + 15 and word c in
    // registers (four SWAR swap stages); the 8 lanes of one word store one sample's 8 words (32 bytes) at a time
    const int gw = mo.rows_p / 16;
    const int jw = lane & 7, c = 4 * warp + (lane >> 3);
    if (c < nw) {
      uint32_t a[16];
#pragma unroll
      for (int r = 0; r < 16; ++r) a[r] = t[16 * jw + r][c];
      uint32_t m = 0x0000FFFFu;
#pragma unroll
      for (int j = 8; j != 0; j >>= 1, m ^= m << (2 * j))
#pragma unroll
        for (int k = 0; k < 16; k = (k + j + 1) & ~j) {
          const uint32_t x = ((a[k] >> (2 * j)) ^ a[k + j]) & m;   // codes k, c + j <-> k + j, c
          a[k] ^= x << (2 * j);
          a[k + j] ^= x;
        }
      uint32_t* dst = mo.gt + (w0 + c) * 16 * gw + blockIdx.y * 8 + jw;
#pragma unroll
      for (int q = 0; q < 16; ++q) dst[(int64_t)q * gw] = a[q];
    }
  }
}

void launch_bed_relayout(const uint8_t* packed, int64_t row_stride, int bs, int rows_p,
                         const int32_t* file_idx_pad, const int32_t* word_base, const uint32_t* word_keep, int ref_first,
                         uint32_t* gp, int64_t npad,
                         cudaStream_t s) {
  RG_CHECK(rows_p % kTileRows == 0, "bed_relayout: rows_p must be a multiple of 128");
  const int64_t wpr = npad / 16;
  dim3 grid((unsigned)ceil_div(wpr, kTileWords), (unsigned)(rows_p / kTileRows));
  bed_relayout_kernel<false><<<grid, kRelayoutThreads, 0, s>>>(packed, row_stride, bs, file_idx_pad, word_base,
                                                               word_keep, ref_first, gp, wpr, BedMissOut{});
}

void launch_bed_relayout_miss(const uint8_t* packed, int64_t row_stride, int bs, int rows_p,
                              const int32_t* file_idx_pad, const int32_t* word_base, const uint32_t* word_keep,
                              int ref_first, uint32_t* gp, int64_t npad, const BedMissOut& mo, cudaStream_t s) {
  RG_CHECK(rows_p % kTileRows == 0 && mo.rows_p == rows_p, "bed_relayout_miss: rows_p must be a multiple of 128");
  RG_CUDA(cudaMemsetAsync(mo.total, 0, sizeof(unsigned long long), s));
  dim3 grid((unsigned)mo.nct, (unsigned)(rows_p / kTileRows));
  bed_relayout_kernel<true><<<grid, kRelayoutThreads, 0, s>>>(packed, row_stride, bs, file_idx_pad, word_base,
                                                              word_keep, ref_first, gp, npad / 16, mo);
}

}  // namespace rg
