// Shared declarations for the sm_90a kernels behind include/rg_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>
#include <map>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

namespace rg {

// ---------------------------------------------------------------------------------------
// error plumbing: every C-ABI entry point catches rg::Error and stores the message.
struct Error {
  std::string msg;
};
void set_last_error(const std::string& m);

#define RG_CUDA(call)                                                                      \
  do {                                                                                     \
    cudaError_t e__ = (call);                                                              \
    if (e__ != cudaSuccess) {                                                              \
      throw rg::Error{std::string(#call) + " failed: " + cudaGetErrorString(e__) + " (" +  \
                      __FILE__ + ":" + std::to_string(__LINE__) + ")"};                    \
    }                                                                                      \
  } while (0)

#define RG_CHECK(cond, message)                                   \
  do {                                                            \
    if (!(cond)) throw rg::Error{std::string(message)};           \
  } while (0)

static inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }
static inline int64_t ceil_div(int64_t x, int64_t m) { return (x + m - 1) / m; }

// ---------------------------------------------------------------------------------------
// Device-side layout constants.
//
// Samples live in a *padded fold layout*: fold f occupies [fold_pad_start[f],
// fold_pad_start[f] + fold_pad_len[f]) with fold_pad_len a multiple of kSamplePad, so every
// tensor-core K-range and every 2-bit word is fold-aligned.  Padding samples carry
// genotype code 0, X = Y = 0 and mask = 0, so they contribute to nothing.
constexpr int kSamplePad = 128;   // = one 128-byte swizzle atom of fp8 operands
constexpr int kFoldPad = 256;     // Step-1 fold ranges: two sample tiles, so a 256-sample prediction CTA never straddles folds
constexpr int kRowPad = 128;      // SNP rows padded to the UMMA M tile
constexpr int kStatChunk = 2048;  // samples per partial-sum chunk of the f64 reductions

// internal 2-bit genotype code: 0,1,2 = dosage, 3 = missing (PLINK: 00->2 01->NA 10->1 11->0)
constexpr int kCodeMissing = 3;

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  void alloc(size_t count) {
    if (count <= n && p) return;
    release();
    RG_CUDA(cudaMalloc(&p, count * sizeof(T)));
    n = count;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
  ~DevBuf() { release(); }
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
};

// Pinned host memory, grown like DevBuf.
template <typename T>
struct PinnedBuf {
  T* p = nullptr;
  size_t n = 0;
  void alloc(size_t count) {
    if (count <= n && p) return;
    release();
    RG_CUDA(cudaMallocHost(&p, count * sizeof(T)));
    n = count;
  }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    n = 0;
  }
  ~PinnedBuf() { release(); }
  PinnedBuf() = default;
  PinnedBuf(const PinnedBuf&) = delete;
  PinnedBuf& operator=(const PinnedBuf&) = delete;
};

// A non-blocking stream, created by ensure() on first use.  The destructor drains it before destroying it, so a member
// declared after the buffers its work reads is gone, with its work, before they are freed.
struct Stream {
  cudaStream_t s = nullptr;
  Stream() = default;
  Stream(Stream&& o) noexcept : s(o.s) { o.s = nullptr; }
  Stream& operator=(Stream&& o) noexcept {
    std::swap(s, o.s);
    return *this;
  }
  ~Stream() {
    if (!s) return;
    cudaStreamSynchronize(s);
    cudaStreamDestroy(s);
  }
  cudaStream_t ensure() {
    if (!s) RG_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    return s;
  }
  operator cudaStream_t() const { return s; }
};

// An event, created by ensure() on first use (without timing unless asked for).
struct Event {
  cudaEvent_t e = nullptr;
  Event() = default;
  Event(Event&& o) noexcept : e(o.e) { o.e = nullptr; }
  Event& operator=(Event&& o) noexcept {
    std::swap(e, o.e);
    return *this;
  }
  ~Event() {
    if (e) cudaEventDestroy(e);
  }
  cudaEvent_t ensure(unsigned flags = cudaEventDisableTiming) {
    if (!e) RG_CUDA(cudaEventCreateWithFlags(&e, flags));
    return e;
  }
  operator cudaEvent_t() const { return e; }
};

// Another process's device allocation mapped into this one, unmapped by the destructor.
struct IpcMapping {
  void* p = nullptr;
  explicit IpcMapping(const cudaIpcMemHandle_t& mh) {
    RG_CUDA(cudaIpcOpenMemHandle(&p, mh, cudaIpcMemLazyEnablePeerAccess));
  }
  IpcMapping(IpcMapping&& o) noexcept : p(o.p) { o.p = nullptr; }
  IpcMapping& operator=(IpcMapping&&) = delete;
  ~IpcMapping() {
    if (p) cudaIpcCloseMemHandle(p);
  }
};

// cudaFuncAttributeMaxDynamicSharedMemorySize is a property of (kernel, DEVICE): several handles on different GPUs may
// live in one process (rgb200 --gpus N, one host thread per GPU), so the "already set" memo is kept per device.
inline void ensure_dyn_smem(const void* func, size_t bytes) {
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, size_t> done;
  int dev = 0;
  RG_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  size_t& cur = done[std::make_pair(dev, func)];
  if (bytes > cur) {
    const cudaError_t e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) {
      // a refused request also sets the runtime's last error: clear it, or the next launch check of any handle in the
      // process would report it
      cudaGetLastError();
      throw Error{"cannot give a kernel " + std::to_string(bytes) + " bytes of dynamic shared memory: " +
                  cudaGetErrorString(e)};
    }
    cur = bytes;
  }
}

// Copy `bytes` from a host-or-device pointer to device memory on `stream`.
void copy_to_device(void* dst, const void* src, size_t bytes, cudaStream_t stream);
bool is_device_pointer(const void* p);

}  // namespace rg
