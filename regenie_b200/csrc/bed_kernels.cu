// Genotype-block layout kernel: PLINK 2-bit rows -> internal padded 2-bit rows (the tensor-core Gram and prediction
// kernels build their int8 operand bytes from these on chip).  Replaces the decode half of readChunkFromBedFileToG
// (reference src/Geno.cpp:1702-1768, LUT src/Geno.cpp:2833-2857); mean imputation is NOT
// materialised: missing calls stay a separate indicator plane and the mean enters as an exact
// rank-structured correction (see DESIGN.md "missing data").
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

// One thread per output 32-bit word (16 samples) of one row.  Almost every word maps to 16 CONSECUTIVE samples of the
// file row (folds only shift whole ranges; --remove breaks a word here and there): those take the fast path - five
// source bytes, one funnel shift, the code translation as bit logic on all 16 lanes, a keep mask for samples outside
// the analysis.  word_base[w] = file index of the word's first sample, -1 = nothing to read, -2 = not contiguous.
__global__ void bed_relayout_kernel(const uint8_t* __restrict__ packed, int64_t row_stride, int bs,
                                    const int32_t* __restrict__ file_idx_pad, const int32_t* __restrict__ word_base,
                                    const uint32_t* __restrict__ word_keep, int ref_first,
                                    uint32_t* __restrict__ gp, int64_t words_per_row) {
  const int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int row = blockIdx.y;
  if (w >= words_per_row) return;
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
  gp[(int64_t)row * words_per_row + w] = out;
}

void launch_bed_relayout(const uint8_t* packed, int64_t row_stride, int bs, int rows_p,
                         const int32_t* file_idx_pad, const int32_t* word_base, const uint32_t* word_keep, int ref_first,
                         uint32_t* gp, int64_t npad,
                         cudaStream_t s) {
  const int64_t wpr = npad / 16;
  dim3 grid((unsigned)ceil_div(wpr, 256), rows_p);
  bed_relayout_kernel<<<grid, 256, 0, s>>>(packed, row_stride, bs, file_idx_pad, word_base, word_keep, ref_first, gp, wpr);
}

}  // namespace rg
