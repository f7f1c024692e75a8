// Point clouds from masked (view, row, column) grids, shared by save_data_all's world cloud (slam_graph.cu) and the
// reconstruction evaluation's clouds (recon.cu): a per-row count, one exclusive scan over the rows, and a scatter that
// ranks the kept columns of a row by warp ballots, so points keep numpy boolean indexing's (view, row, column) order.
// The unprojection is K^-1 [x y 1]^T d followed by P [p; 1], in fp32.
#pragma once
#include <cuda_runtime.h>

namespace sta {
namespace {

// 256 threads: the block's sum of one int per thread (valid in thread 0).
__device__ __forceinline__ int block_count_256(int cnt) {
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  __shared__ int wsum[8];
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = cnt;
  __syncthreads();
  int t = 0;
  if (threadIdx.x == 0)
    for (int w = 0; w < 8; ++w) t += wsum[w];
  return t;
}

// one block of 1024 threads: exclusive scan of n counts in order (offsets[n] = total), total also to count_out
__global__ void __launch_bounds__(1024) row_scan_kernel(const int* counts, long long n, long long* offsets, int64_t* count_out) {
  __shared__ long long part[1024];
  const long long per = (n + 1023) / 1024;
  const long long lo = threadIdx.x * per, hi = min(n, lo + per);
  long long t = 0;
  for (long long i = lo; i < hi; ++i) t += counts[i];
  part[threadIdx.x] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long run = 0;
    for (int i = 0; i < 1024; ++i) {
      const long long c = part[i];
      part[i] = run;
      run += c;
    }
    offsets[n] = run;
    *count_out = run;
  }
  __syncthreads();
  long long run = part[threadIdx.x];
  for (long long i = lo; i < hi; ++i) {
    offsets[i] = run;
    run += counts[i];
  }
}

// 256 threads: emit(x, o) for every column x < W of one row with keep(x), o = base + the number of kept columns before x.
template <class Keep, class Emit>
__device__ __forceinline__ void row_compact_256(int W, long long base, Keep keep, Emit emit) {
  __shared__ int wsum[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int x0 = 0; x0 < W; x0 += 256) {
    const int x = x0 + threadIdx.x;
    const bool k = x < W && keep(x);
    const unsigned bal = __ballot_sync(0xffffffffu, k);
    if (lane == 0) wsum[warp] = __popc(bal);
    __syncthreads();
    int before = __popc(bal & ((1u << lane) - 1u)), total = 0;
    for (int w = 0; w < 8; ++w) {
      if (w < warp) before += wsum[w];
      total += wsum[w];
    }
    if (k) emit(x, base + before);
    base += total;
    __syncthreads();
  }
}

// torch.inverse of 3x3 intrinsics, evaluated in fp64 from the adjugate and rounded to fp32
__device__ __forceinline__ void inv3_f32(const float* K, float* Ki) {
  const double k00 = K[0], k01 = K[1], k02 = K[2], k10 = K[3], k11 = K[4], k12 = K[5], k20 = K[6], k21 = K[7], k22 = K[8];
  const double det = k00 * (k11 * k22 - k12 * k21) - k01 * (k10 * k22 - k12 * k20) + k02 * (k10 * k21 - k11 * k20);
  Ki[0] = static_cast<float>((k11 * k22 - k12 * k21) / det);
  Ki[1] = static_cast<float>((k02 * k21 - k01 * k22) / det);
  Ki[2] = static_cast<float>((k01 * k12 - k02 * k11) / det);
  Ki[3] = static_cast<float>((k12 * k20 - k10 * k22) / det);
  Ki[4] = static_cast<float>((k00 * k22 - k02 * k20) / det);
  Ki[5] = static_cast<float>((k02 * k10 - k00 * k12) / det);
  Ki[6] = static_cast<float>((k10 * k21 - k11 * k20) / det);
  Ki[7] = static_cast<float>((k01 * k20 - k00 * k21) / det);
  Ki[8] = static_cast<float>((k00 * k11 - k01 * k10) / det);
}

// P (K^-1 [u r 1]^T d) + t with P a row-major 4x4 (rotation and translation rows), fp32
__device__ __forceinline__ void unproject_f32(const float* Ki, const float* P, float u, float r, float d, float* out) {
  const float cx = (Ki[0] * u + Ki[1] * r + Ki[2]) * d, cy = (Ki[3] * u + Ki[4] * r + Ki[5]) * d,
              cz = (Ki[6] * u + Ki[7] * r + Ki[8]) * d;
  for (int c = 0; c < 3; ++c) out[c] = P[c * 4] * cx + P[c * 4 + 1] * cy + P[c * 4 + 2] * cz + P[c * 4 + 3];
}

}  // namespace
}  // namespace sta
