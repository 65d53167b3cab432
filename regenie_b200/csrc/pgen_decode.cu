// On-device decode of PLINK 2 .pgen hard-call records into PLINK 1 2-bit rows (SURVEY §8 (f)3).
//
// The reference decodes .pgen variants one at a time through pgenlib on the host (PgenReader::Read, src/Geno.cpp:1773-1821,
// :2538-2594, :2596-2712) into an FP64 column.  Here the host only slices the file (host/pgen.cpp: PgenFile::gather); the
// record bytes cross PCIe as they are - a rare variant is a difflist of a few hundred bytes instead of N / 4 - and two
// kernels expand them in HBM into the rows every .bed kernel of this library already takes:
//   pgen_fill_kernel   thread = one 32-bit word (16 samples) of a row: the dense part of the record (2-bit values, 1-bit
//                      values + code byte, or a constant), for an LD-compressed record the dense part of its base;
//                      PLINK 2 value -> PLINK 1 code (and the 0 <-> 2 swap of type 3) as bit logic on the whole word.
//                      HBM-bound: N / 4 bytes written per variant, at most N / 4 read.
//   pgen_patch_kernel  warp = one row: the difflist of the base (if it has one), then the record's own, lane = one group of
//                      64 entries (the per-group byte counts of the format make the groups independent); entries land with
//                      a 32-bit atomic and / or pair because neighbouring samples share a word.
// The arithmetic lives in pgen_core.h, which also compiles for the host: tests/test_host_cpu.py runs it (lanes one after the
// other) against oracle/pgen.py on the reference's example.pgen and on synthetic files holding every record type.
#include "context.cuh"
#include "pgen_core.h"

namespace rg {

struct PgenMeta {                 // device views into the block's metadata blob
  const uint8_t* bytes;
  const uint64_t* off;
  const uint32_t* len;
  const int32_t* own;
  const int32_t* base;
  const uint8_t* type;
};

__device__ __forceinline__ rgp::Rec pgen_rec(const PgenMeta& m, int r) {
  return rgp::Rec{m.bytes + m.off[r], m.len[r], (uint32_t)m.type[r]};
}

__device__ __forceinline__ void pgen_report(unsigned long long* err, uint32_t tag, int row, int code) {
  atomicCAS(err, 0ull, ((unsigned long long)tag << 32) | ((unsigned long long)row << 4) | (unsigned long long)code);
}

constexpr int kFillThreads = 256;
constexpr int kPatchWarps = 8;

__global__ void __launch_bounds__(kFillThreads)
pgen_fill_kernel(PgenMeta m, uint32_t n, uint32_t words, uint32_t* __restrict__ rows, unsigned long long* err, uint32_t tag) {
  const int j = blockIdx.y;
  const int o = m.own[j];
  const uint32_t ot = m.type[o];
  const rgp::Rec r = pgen_rec(m, (ot & 6) == 2 ? m.base[j] : o);
  int e = rgp::kOk;
  uint32_t* row = rows + (size_t)j * words;
  for (uint32_t w = blockIdx.x * kFillThreads + threadIdx.x; w < words; w += gridDim.x * kFillThreads)
    row[w] = rgp::fill_word(r, n, w, ot == 3, &e);
  if (e) pgen_report(err, tag, j, e);
}

__global__ void __launch_bounds__(kPatchWarps * 32)
pgen_patch_kernel(PgenMeta m, uint32_t n, uint32_t words, uint32_t* __restrict__ rows, int bs, unsigned long long* err,
                  uint32_t tag) {
  const int j = blockIdx.x * kPatchWarps + (threadIdx.x >> 5);
  if (j >= bs) return;                                      // a whole warp leaves together
  const uint32_t lane = threadIdx.x & 31;
  const int o = m.own[j];
  const rgp::Rec own = pgen_rec(m, o);
  const bool ld = (own.type & 6) == 2, inv = own.type == 3;
  uint32_t* row = rows + (size_t)j * words;
  int e = rgp::kOk;
  if (ld) {
    const rgp::Rec b = pgen_rec(m, m.base[j]);
    const uint32_t pos = rgp::difflist_pos(b.type, n);
    if (pos != 0xFFFFFFFFu) rgp::patch_difflist(b, pos, n, inv, row, lane, 32, &e);
    __syncwarp();                                           // the record's own entries override the base's
  }
  const uint32_t pos = rgp::difflist_pos(own.type, n);
  if (pos != 0xFFFFFFFFu) rgp::patch_difflist(own, pos, n, inv, row, lane, 32, &e);
  if (e) pgen_report(err, tag, j, e);
}

static const char* pgen_err_text(int code) {
  switch (code) {
    case rgp::kErrTruncated: return "record is truncated";
    case rgp::kErrSampleIdx: return "sample index out of range";
    case rgp::kErrListLen: return "difflist longer than the sample count";
    default: return "unsupported record type";
  }
}

// 0 = nothing recorded; otherwise throws with the block / variant of the first malformed record and clears the slot
void pgen_check_errors(rg_ctx* h) {
  if (!h->pgen_err.p) return;
  unsigned long long v = 0;
  RG_CUDA(cudaMemcpy(&v, h->pgen_err.p, 8, cudaMemcpyDeviceToHost));
  if (!v) return;
  RG_CUDA(cudaMemset(h->pgen_err.p, 0, 8));
  throw Error{"malformed .pgen record (" + std::string(pgen_err_text((int)(v & 15))) + ") at variant " +
              std::to_string((v >> 4) & 0xFFFFFFFull) + " of block " + std::to_string((v >> 32) - 1) + "."};
}

static void pgen_decode(rg_ctx* h, const rg_pgen_block* b, const uint8_t** rows_dev, int64_t* row_stride) {
  RG_CHECK(h->kind == 1 || h->kind == 2, "bad handle");
  RG_CHECK(b->bs > 0 && b->bs <= h->bs_max, "block size out of range");
  RG_CHECK(b->n_file > 0 && b->n_file < (1ll << 31), "bad sample count");
  RG_CHECK(b->n_rec > 0 && b->n_rec <= 2 * b->bs && b->n_bytes >= 0 && b->n_bytes < (1ll << 40), "bad record table");
  RG_CHECK(b->bytes && b->rec_off && b->rec_len && b->rec_type && b->own && b->base, "null argument");
  for (int r = 0; r < b->n_rec; ++r) {
    RG_CHECK((b->rec_off[r] & 3) == 0, "records must start at multiples of 4 bytes");
    RG_CHECK(b->rec_off[r] + (uint64_t)b->rec_len[r] <= (uint64_t)b->n_bytes, "record runs past the end of the buffer");
    RG_CHECK(b->rec_type[r] < 8, "record type out of range (multiallelic / dosage tracks are not supported)");
  }
  for (int j = 0; j < b->bs; ++j) {
    RG_CHECK(b->own[j] >= 0 && b->own[j] < b->n_rec, "record index out of range");
    if ((b->rec_type[b->own[j]] & 6) == 2) {
      RG_CHECK(b->base[j] >= 0 && b->base[j] < b->n_rec, "LD-compressed record without a base");
      RG_CHECK((b->rec_type[b->base[j]] & 6) != 2, "the base of an LD-compressed record is LD-compressed itself");
    }
  }
  RG_CUDA(cudaSetDevice(h->device));

  // where the rows go: Step 1 - the input buffer and stream of the lane the next rg_l0_block_bed call takes
  cudaStream_t s = h->stream;
  rg::DevBuf<uint8_t>* rows = &h->pgen_rows;
  rg::DevBuf<uint8_t>* in = &h->pgen_in;
  if (h->kind == 1) {
    RG_CHECK(!h->lanes.empty(), "handle has no lanes");
    rg_ctx::Lane& L = *h->lanes[h->next_lane];
    s = L.stream;
    rows = &L.packed_dev;
    in = &L.pgen_in;
  }
  const uint32_t n = (uint32_t)b->n_file;
  const uint32_t words = (uint32_t)round_up(ceil_div(n, 16), 4);          // rows are multiples of 16 bytes
  const size_t stride = (size_t)words * 4;
  if (!h->pgen_err.p) {
    h->pgen_err.alloc(1);
    RG_CUDA(cudaMemset(h->pgen_err.p, 0, 8));
  }
  // the host rows of a .bed call may have used the same buffer with another stride: size it for the larger of the two
  rows->alloc(std::max((size_t)h->bs_max * stride, rows->n));

  // one blob: [off u64 n_rec][len u32 n_rec][own i32 bs][base i32 bs][type u8 n_rec] | pad to 16 | record bytes
  const size_t o_len = (size_t)b->n_rec * 8, o_own = o_len + (size_t)b->n_rec * 4, o_base = o_own + (size_t)b->bs * 4,
               o_type = o_base + (size_t)b->bs * 4, o_bytes = (size_t)round_up((int64_t)(o_type + b->n_rec), 16);
  std::vector<uint8_t> meta(o_bytes);
  memcpy(meta.data(), b->rec_off, (size_t)b->n_rec * 8);
  memcpy(meta.data() + o_len, b->rec_len, (size_t)b->n_rec * 4);
  memcpy(meta.data() + o_own, b->own, (size_t)b->bs * 4);
  memcpy(meta.data() + o_base, b->base, (size_t)b->bs * 4);
  memcpy(meta.data() + o_type, b->rec_type, (size_t)b->n_rec);
  const size_t total = o_bytes + (size_t)b->n_bytes + 16;
  if (total > in->n) in->alloc(total + total / 4 + 4096);                  // grows rarely
  RG_CUDA(cudaMemcpyAsync(in->p, meta.data(), o_bytes, cudaMemcpyHostToDevice, s));   // pageable: staged before return
  copy_to_device(in->p + o_bytes, b->bytes, (size_t)b->n_bytes, s);
  PgenMeta m;
  m.bytes = in->p + o_bytes;
  m.off = reinterpret_cast<const uint64_t*>(in->p);
  m.len = reinterpret_cast<const uint32_t*>(in->p + o_len);
  m.own = reinterpret_cast<const int32_t*>(in->p + o_own);
  m.base = reinterpret_cast<const int32_t*>(in->p + o_base);
  m.type = in->p + o_type;
  uint32_t* out = reinterpret_cast<uint32_t*>(rows->p);
  const uint32_t tag = (uint32_t)(b->block_id + 1);
  const unsigned gx = (unsigned)std::min<int64_t>(64, ceil_div(words, kFillThreads));
  pgen_fill_kernel<<<dim3(gx, (unsigned)b->bs), kFillThreads, 0, s>>>(m, n, words, out, h->pgen_err.p, tag);
  RG_CUDA(cudaGetLastError());
  pgen_patch_kernel<<<(unsigned)ceil_div(b->bs, kPatchWarps), kPatchWarps * 32, 0, s>>>(m, n, words, out, b->bs,
                                                                                       h->pgen_err.p, tag);
  RG_CUDA(cudaGetLastError());
  h->launches += 2;
  if (h->kind == 2) {
    RG_CUDA(cudaStreamSynchronize(s));
    pgen_check_errors(h);
  }
  *rows_dev = rows->p;
  *row_stride = (int64_t)stride;
}

}  // namespace rg

extern "C" {

int rg_pgen_decode(rg_handle h, const rg_pgen_block* blk, const uint8_t** rows_dev, int64_t* row_stride) {
  RG_API_BEGIN
  RG_CHECK(h && blk && rows_dev && row_stride, "null argument");
  rg::pgen_decode(h, blk, rows_dev, row_stride);
  RG_API_END
}

}  // extern "C"
