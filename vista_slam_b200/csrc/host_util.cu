#include "host_util.h"

#include <stdlib.h>

#include <atomic>
#include <mutex>

namespace sta {

static thread_local std::string t_last_error;

void set_last_error(const std::string& msg) { t_last_error = msg; }
const char* get_last_error() { return t_last_error.c_str(); }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap(out, base, /*is_f32=*/0, rank, dims, strides_bytes, box);
}

int make_tmap(CUtensorMap* out, const void* base, int kind, int rank, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled not available (no CUDA driver?)");
    return 1;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    estr[i] = 1;
    if (i + 1 < rank) gstr[i] = strides_bytes[i];
  }
  const CUtensorMapDataType dt = kind == 1   ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                : kind == 2 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                            : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUresult r = fn(out, dt, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed: CUresult=%d (rank=%d dims0=%llu box0=%u)", (int)r, rank,
             (unsigned long long)dims[0], box[0]);
    set_last_error(buf);
    return 1;
  }
  return 0;
}

int num_sms() {
  static std::atomic<int> cache[64];  // zero-initialised; one slot per device ordinal
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev >= 0 && dev < 64) {
    const int c = cache[dev].load(std::memory_order_relaxed);
    if (c > 0) return c;
  }
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
  if (dev >= 0 && dev < 64) cache[dev].store(n, std::memory_order_relaxed);
  return n;
}

}  // namespace sta
