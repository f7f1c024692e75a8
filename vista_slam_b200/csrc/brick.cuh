// The brick key of the sparse TSDF volume, shared by fusion.cu (which builds and meshes the volume) and raycast.cu
// (which marches rays through it).  Samples sit at (i v, j v, k v) in bricks of kBrick^3; brick (bx, by, bz) =
// floor(i / 8) per axis, each coordinate in [-2^20, 2^20 - 1], has the 63-bit key
// (bz + 2^20) << 42 | (by + 2^20) << 21 | (bx + 2^20), so sorting the keys orders the bricks by z, then y, then x.
// A brick's samples are stored [z][y][x], kBrickSamples of them.
#pragma once

#include "../../include/sta_b200.h"

namespace sta {

constexpr int kBrick = STA_FUSION_BRICK;
constexpr int kBrickSamples = kBrick * kBrick * kBrick;  // 512
constexpr int kBias = 1 << 20;                           // brick coordinates lie in [-2^20, 2^20 - 1]

__host__ __device__ __forceinline__ unsigned long long brick_key(int bx, int by, int bz) {
  return (static_cast<unsigned long long>(bz + kBias) << 42) | (static_cast<unsigned long long>(by + kBias) << 21) |
         static_cast<unsigned long long>(bx + kBias);
}

__device__ __forceinline__ void key_brick(unsigned long long k, int& bx, int& by, int& bz) {
  bx = static_cast<int>(k & 0x1fffff) - kBias;
  by = static_cast<int>((k >> 21) & 0x1fffff) - kBias;
  bz = static_cast<int>((k >> 42) & 0x1fffff) - kBias;
}

// index of key k in the B sorted keys, or -1
__device__ __forceinline__ int find_brick(const int64_t* keys, long long B, long long k) {
  long long lo = 0, hi = B;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (keys[mid] < k) lo = mid + 1;
    else hi = mid;
  }
  return lo < B && keys[lo] == k ? static_cast<int>(lo) : -1;
}

}  // namespace sta
