// Host-side helpers: error reporting for the C-ABI, TMA tensor-map encoding.
// libcuda is NOT linked: cuTensorMapEncodeTiled is resolved at run time through
// cudaGetDriverEntryPoint so the library loads (and exports its symbols) on a
// machine without a GPU driver.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <mutex>
#include <string>

namespace sta {

void set_last_error(const std::string& msg);
const char* get_last_error();

#define STA_CHECK_CUDA(expr)                                                                      \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      char _buf[512];                                                                             \
      snprintf(_buf, sizeof(_buf), "%s:%d: %s failed: %s", __FILE__, __LINE__, #expr,             \
               cudaGetErrorString(_e));                                                           \
      sta::set_last_error(_buf);                                                                  \
      return 1;                                                                                   \
    }                                                                                             \
  } while (0)

#define STA_REQUIRE(cond, msg)                                                                    \
  do {                                                                                            \
    if (!(cond)) {                                                                                \
      char _buf[512];                                                                             \
      snprintf(_buf, sizeof(_buf), "%s:%d: requirement failed: %s (%s)", __FILE__, __LINE__,      \
               #cond, msg);                                                                       \
      sta::set_last_error(_buf);                                                                  \
      return 2;                                                                                   \
    }                                                                                             \
  } while (0)

// Encode a tiled bf16 tensor map with 128-byte swizzle.  dims[0] is the innermost
// (contiguous) dimension; strides_bytes[i] is the byte stride of dims[i+1].
// Returns 0 on success.
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box);

// Same for bf16 (kind = 0), fp32 (kind = 1) or 8-bit (kind = 2: e4m3 codes) elements.
int make_tmap(CUtensorMap* out, const void* base, int kind, int rank, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box);

int num_sms();  // of the CURRENT device (cached per device)

// true for device (or managed) memory; host pointers and unknown addresses are false
inline bool on_device(const void* p) {
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

// One-time per-DEVICE setup at a call site (cudaFuncSetAttribute is per device/context, not per process):
//   static PerDeviceOnce once;  STA_CHECK_CUDA(once.run([&] { return cudaFuncSetAttribute(...); }));
struct PerDeviceOnce {
  std::atomic<unsigned long long> done{0};
  std::mutex mu;
  template <typename F>
  cudaError_t run(F&& f) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= 64) return f();  // beyond the bitmap: just repeat the (idempotent) setup
    const unsigned long long bit = 1ull << dev;
    if (done.load(std::memory_order_acquire) & bit) return cudaSuccess;
    std::lock_guard<std::mutex> lock(mu);
    if (done.load(std::memory_order_relaxed) & bit) return cudaSuccess;
    e = f();
    if (e == cudaSuccess) done.fetch_or(bit, std::memory_order_release);
    return e;
  }
};

// Launch with programmatic stream serialization (PDL) and an optional cluster size.  The kernel MUST call
// sta::pdl_wait() before its first global-memory access.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, int cluster,
                              Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[n].val.programmaticStreamSerializationAllowed = 1;
  ++n;
  if (cluster > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

}  // namespace sta
