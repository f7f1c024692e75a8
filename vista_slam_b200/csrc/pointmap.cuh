// The depth-scale reduction (slam_utils.py:168-190 with slam.py:227) as device functions, shared by
// sta_depth_scale (pointmap.cu) and the scale edges of the device pose graph (slam_graph.cu).
//
// One pass over the data: per-thread fp32 partial sums -> warp shuffles -> one fp64 record per block; the records are
// then combined in a fixed order in fp64 (deterministic, no atomics).
#pragma once
#include <cuda_runtime.h>

namespace sta {

constexpr int kStatBlocks = 64;  // partial records per reduction
constexpr int kStatVals = 8;     // doubles per record (5 used by the intrinsics pass, 3 by the scale pass)

// 256 threads: reduces s[] over the block and stores NV doubles at rec (threads 0..NV-1).
template <int NV>
__device__ __forceinline__ void block_reduce_store(float (&s)[NV], double* rec) {
  __shared__ float red[8][NV];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s[i] += __shfl_xor_sync(0xffffffffu, s[i], o);
  }
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) red[warp][i] = s[i];
  }
  __syncthreads();
  if (threadIdx.x < NV) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += static_cast<double>(red[w][threadIdx.x]);
    rec[threadIdx.x] = t;
  }
}

// Block `blk` of kStatBlocks (256 threads each): its record of {sum w Di Dj, sum w Di^2, sum sqrt(ci cj)} with
// w = max(ci cj, 1e-6).
__device__ __forceinline__ void scale_partial(const float* __restrict__ Di, const float* __restrict__ Dj,
                                              const float* __restrict__ ci, const float* __restrict__ cj, long long n,
                                              int blk, double* rec) {
  float s[3] = {0.f, 0.f, 0.f};
  for (long long i = static_cast<long long>(blk) * 256 + threadIdx.x; i < n; i += kStatBlocks * 256) {
    const float a = Di[i], b = Dj[i], cc = ci[i] * cj[i];
    const float w = fmaxf(cc, 1e-6f);
    s[0] += w * a * b;
    s[1] += w * a * a;
    s[2] += sqrtf(cc);
  }
  block_reduce_store<3>(s, rec);
}

// The kStatBlocks records of one reduction -> {scale, scale_conf}.
__device__ __forceinline__ void scale_finalize(const double* __restrict__ partial, long long n, float* out2) {
  double t[3] = {0.0, 0.0, 0.0};
  for (int b = 0; b < kStatBlocks; ++b)
    for (int i = 0; i < 3; ++i) t[i] += partial[static_cast<long long>(b) * kStatVals + i];
  out2[0] = static_cast<float>(t[0] / t[1]);
  out2[1] = static_cast<float>(t[2] / static_cast<double>(n));
}

}  // namespace sta
