// On-device inflate of BGEN v1.2 zlib payloads (SURVEY §8 (f)2).
//
// The reference inflates every variant on the host (`uncompress`, src/Geno.cpp:1608, :2207) before it touches the
// probabilities; at BASELINE configs[3] scale (N = 500k: 1.5 MB per variant uncompressed) host zlib is what bounds the
// Step-2 BGEN path end to end.  Here the compressed bytes go over PCIe as they are (3-10x smaller) and are inflated in
// HBM: one warp per variant stream (inflate_core.h: lane 0 decodes the Huffman symbols, the warp copies the matches),
// then a second kernel checks the payload header and splits it into the two arrays the dosage kernels take
// (`probs` [bs][n_file][2], `ploidy_missing` [bs][n_file]), i.e. exactly what host/bgen.cpp produces on the host.
//
// The decoder core is verified against zlib on the CPU (tests/test_host_cpu.py: every variant of the reference's BGEN
// fixtures plus 128 synthetic streams covering stored / fixed / dynamic blocks and the error paths) and on the GPU through
// the driver (`--gpu-inflate` output is byte-identical to the host-zlib path, tests/test_driver_gpu.py).  The default stays host
// zlib until the Step-2 bench leg is switched over.
#include <stdlib.h>

#include "context.cuh"
#include "inflate_core.h"

namespace rg {

constexpr int kInflateWarps = 8;           // streams per CTA; 3.3 KB of decode tables each in shared memory
constexpr int kStatusBadHeader = 100;      // payload is not 8-bit unphased diploid biallelic layout 2

__global__ void __launch_bounds__(kInflateWarps * 32)
bgen_inflate_kernel(const uint8_t* __restrict__ comp, const uint64_t* __restrict__ offs, uint8_t* __restrict__ raw,
                    uint64_t raw_stride, uint32_t raw_len, int bs, int32_t* __restrict__ status) {
  __shared__ rgi::Tables tabs[kInflateWarps];
  const int warp = threadIdx.x >> 5;
  const int v = blockIdx.x * kInflateWarps + warp;
  if (v >= bs) return;                     // a whole warp leaves together
  const uint64_t o = offs[v];
  const int st = rgi::inflate_zlib(comp + o, (uint32_t)(offs[v + 1] - o), raw + (uint64_t)v * raw_stride, raw_len,
                                   tabs[warp], true);
  if ((threadIdx.x & 31) == 0) status[v] = st;
}

// Variant with the last 16 KB of every stream's output in shared memory (inflate_zlib_window): matches are ring-to-ring
// copies and global memory is written in coalesced runs.  Selected with RG_B200_INFLATE=window; verified against zlib on
// the CPU like the direct variant (tests/test_host_cpu.py, tools/inflate_fuzz.cpp, both lane orders), NOT yet run or timed
// on the GPU - the direct kernel above stays the default until it has been.
constexpr int kWindowWarps = 4;
constexpr size_t kWindowWarpBytes = rgi::kWinBytes + ((sizeof(rgi::Tables) + 15) / 16) * 16;
constexpr size_t kWindowSmem = kWindowWarps * kWindowWarpBytes;

__global__ void __launch_bounds__(kWindowWarps * 32)
bgen_inflate_window_kernel(const uint8_t* __restrict__ comp, const uint64_t* __restrict__ offs, uint8_t* __restrict__ raw,
                           uint64_t raw_stride, uint32_t raw_len, int bs, int32_t* __restrict__ status) {
  extern __shared__ __align__(16) uint8_t inflate_smem[];
  const int warp = threadIdx.x >> 5;
  const int v = blockIdx.x * kWindowWarps + warp;
  if (v >= bs) return;
  uint8_t* win = inflate_smem + (size_t)warp * kWindowWarpBytes;
  rgi::Tables& tab = *reinterpret_cast<rgi::Tables*>(win + rgi::kWinBytes);
  const uint64_t o = offs[v];
  const int st = rgi::inflate_zlib_window(comp + o, (uint32_t)(offs[v + 1] - o), raw + (uint64_t)v * raw_stride, raw_len, tab, win, true);
  if ((threadIdx.x & 31) == 0) status[v] = st;
}

// raw payload of one variant (BGEN v1.2 layout 2): N u32 | K u16 | Pmin u8 | Pmax u8 | N ploidy bytes | phased u8 |
// bits u8 | 2N probability bytes.  grid = (chunks, bs)
__global__ void bgen_unpack_kernel(const uint8_t* __restrict__ raw, uint64_t raw_stride, uint32_t n_file, int bs,
                                   uint8_t* __restrict__ probs, uint8_t* __restrict__ pm, int32_t* __restrict__ status) {
  const int v = blockIdx.y;
  if (v >= bs || status[v] != 0) return;
  const uint8_t* r = raw + (uint64_t)v * raw_stride;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const uint32_t n = r[0] | ((uint32_t)r[1] << 8) | ((uint32_t)r[2] << 16) | ((uint32_t)r[3] << 24);
    const uint32_t k = r[4] | ((uint32_t)r[5] << 8);
    const bool ok = n == n_file && k == 2 && r[6] == 2 && r[7] == 2 && r[8 + n_file] == 0 && r[9 + n_file] == 8;
    if (!ok) status[v] = kStatusBadHeader;
  }
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
  uint8_t* pmv = pm + (uint64_t)v * n_file;
  uint8_t* pv = probs + (uint64_t)v * n_file * 2;
  const uint8_t* rp = r + 8;
  const uint8_t* rq = r + 10 + n_file;
  for (uint32_t i = tid; i < n_file; i += nth) pmv[i] = rp[i];
  for (uint32_t i = tid; i < 2 * n_file; i += nth) pv[i] = rq[i];
}

static void bgen_inflate(rg_ctx* h, const uint8_t* comp, const uint64_t* comp_offs, int64_t n_file, int bs,
                         const uint8_t** probs_out, const uint8_t** miss_out) {
  Step2State::Input& in = step2(h).in;
  RG_CHECK(bs > 0 && bs <= h->bs_max, "block size out of range");
  RG_CHECK(n_file > 0 && n_file < (1ll << 30), "bad sample count");
  for (int v = 0; v < bs; ++v) RG_CHECK(comp_offs[v + 1] >= comp_offs[v], "stream offsets must not decrease");
  RG_CHECK(comp_offs[bs] - comp_offs[0] < (1ull << 40), "compressed block is too large");
  for (int v = 0; v < bs; ++v) RG_CHECK(comp_offs[v + 1] - comp_offs[v] < (1ull << 32), "stream is too large");
  RG_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  const uint32_t raw_len = (uint32_t)(10 + 3 * n_file);
  const uint64_t raw_stride = (uint64_t)round_up(raw_len, 16);
  const uint64_t base = comp_offs[0], total = comp_offs[bs] - base;
  std::vector<uint64_t> rel(bs + 1);
  for (int v = 0; v <= bs; ++v) rel[v] = comp_offs[v] - base;
  if ((size_t)total > in.inflate_comp.n) in.inflate_comp.alloc((size_t)(total + total / 4 + 4096));   // grows rarely
  in.inflate_offs.alloc((size_t)h->bs_max + 1);
  in.inflate_raw.alloc((size_t)h->bs_max * raw_stride);
  in.inflate_status.alloc((size_t)h->bs_max);
  in.probs_dev.alloc((size_t)h->bs_max * n_file * 2);
  in.miss_dev.alloc((size_t)h->bs_max * n_file);
  copy_to_device(in.inflate_comp.p, comp + base, (size_t)total, s);
  RG_CUDA(cudaMemcpyAsync(in.inflate_offs.p, rel.data(), rel.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
  const char* mode_env = getenv("RG_B200_INFLATE");          // read per call: the bench times both kernels in one process
  const bool use_window = mode_env && std::string(mode_env) == "window";
  if (use_window) {
    ensure_dyn_smem(reinterpret_cast<const void*>(bgen_inflate_window_kernel), kWindowSmem);
    bgen_inflate_window_kernel<<<(unsigned)ceil_div(bs, kWindowWarps), kWindowWarps * 32, kWindowSmem, s>>>(
        in.inflate_comp.p, in.inflate_offs.p, in.inflate_raw.p, raw_stride, raw_len, bs, in.inflate_status.p);
  } else {
    bgen_inflate_kernel<<<(unsigned)ceil_div(bs, kInflateWarps), kInflateWarps * 32, 0, s>>>(
        in.inflate_comp.p, in.inflate_offs.p, in.inflate_raw.p, raw_stride, raw_len, bs, in.inflate_status.p);
  }
  RG_CUDA(cudaGetLastError());
  const unsigned chunks = (unsigned)std::min<int64_t>(64, ceil_div(n_file, 1024));
  bgen_unpack_kernel<<<dim3(chunks, (unsigned)bs), 256, 0, s>>>(in.inflate_raw.p, raw_stride, (uint32_t)n_file, bs,
                                                               in.probs_dev.p, in.miss_dev.p, in.inflate_status.p);
  RG_CUDA(cudaGetLastError());
  std::vector<int32_t> st(bs);
  RG_CUDA(cudaMemcpyAsync(st.data(), in.inflate_status.p, (size_t)bs * 4, cudaMemcpyDeviceToHost, s));
  RG_CUDA(cudaStreamSynchronize(s));
  h->launches += 2;
  for (int v = 0; v < bs; ++v) {
    if (st[v] == 0) continue;
    if (st[v] == kStatusBadHeader)
      throw Error{"unsupported bgen genotype block at variant " + std::to_string(v) +
                  " of the block (rgb200 reads 8-bit unphased diploid biallelic layout 2 only)."};
    throw Error{"corrupt zlib stream in the bgen file at variant " + std::to_string(v) + " of the block (inflate status " +
                std::to_string(st[v]) + ")."};
  }
  *probs_out = in.probs_dev.p;
  *miss_out = in.miss_dev.p;
}

}  // namespace rg

extern "C" {

int rg_bgen_inflate(rg_handle h, const uint8_t* comp, const uint64_t* comp_offs, int64_t n_file, int32_t bs,
                    const uint8_t** probs_dev, const uint8_t** miss_dev) {
  RG_API_BEGIN
  RG_CHECK(h && comp && comp_offs && probs_dev && miss_dev, "null argument");
  rg::bgen_inflate(h, comp, comp_offs, n_file, bs, probs_dev, miss_dev);
  RG_API_END
}

}  // extern "C"
