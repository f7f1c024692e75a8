// Ray casting of the fused TSDF volume (fusion.raycast, OnlineSLAM.render_surface): per pixel of C cameras, the first
// front-facing zero of the volume's trilinear field, with its camera depth, normal, colour and a headlit colour.
//
// The volume is sta_fusion_integrate's: sorted 63-bit brick keys (brick.cuh), tsdf / weight [B][8][8][8] and color
// [B][8][8][8][3], samples at (float(i) v, float(j) v, float(k) v).
//   raycast_box_kernel  one block: the bricks' bounding box [6] (integer min / max, order-free) into the scratch, so
//                       that no host read is needed;
//   raycast_kernel      one thread per output pixel, 16 x 8 pixel blocks, cameras as grid z.
//
// Ray.  Pixel (col, row) of camera c is o + z R ((col - cx) / fx, (row - cy) / fy, 1), R and o from c2w[c], so z is the
// camera depth and integer pixel coordinates are pixel centres (render.cu's floor(u / w + 0.5) rounding).
// Field.  Point p lies in cell floor(p / v) per axis; the cell is valid when its 8 corner samples exist with weight >=
// min_weight (fusion.cu's cube_case rule: a cell is valid iff marching cubes meshes it), and there T(p) and the colour
// are the trilinear interpolants of the corners at the fractions p / v - floor(p / v).
// March.  Over the ray's overlap with the box [8 bmin v, 8 (bmax + 1) v] per axis, from z >= near: samples at
// z_k = za + k dz with dz = (v / 2) / |R d| (half a voxel of world length).  At a sample whose cell's brick is absent
// the march jumps to the last sample before the ray leaves that brick (no valid cell has its lower corner there, so
// the jump changes nothing).  The hit is the first k with valid samples k - 1 and k, T_{k-1} > 0 >= T_k (a front
// face; - to + crossings, surfaces seen from behind, are passed through).  It is refined by kRefine bisection steps
// on [z_{k-1}, z_k] -- an invalid midpoint closes the bracket from the far side -- and the final bracket's secant
// point z is the hit.  Normal and colour are evaluated in z's cell, or in the
// bracket's near end's cell when z's cell is invalid.
// Outputs.  depth z (0 on a miss); normal: the normalised gradient of the interpolant (world frame, 0 on a miss);
// color: the interpolated colour (background on a miss); rgb: color (0.3 + 0.7 max(0, -n . r)), a headlight with r
// the unit ray direction (background on a miss).
// One thread per pixel and no atomics in the march: every call gives the same bits, and a camera's image does not
// depend on the other cameras of the call.
#include <math.h>
#include <stdint.h>

#include "../../include/sta_b200.h"
#include "brick.cuh"
#include "host_util.h"

namespace sta {
namespace {

constexpr int kMaxSide = 8192;     // cameras, rows and columns per call (render.cu's limit)
constexpr int kRefine = 16;        // bisection steps per hit: the bracket shrinks to 2^-17 v of world length
constexpr float kAmbient = 0.3f;   // headlight: rgb = color (kAmbient + (1 - kAmbient) max(0, -n . r))
constexpr int kTileX = 16, kTileY = 8, kThreads = kTileX * kTileY;
constexpr int kNoBrick = -1, kUnknown = -2;

struct RayArgs {
  const int64_t* keys;
  long long B;
  const float *tsdf, *weight, *color;
  float vox, min_weight, near;
  const float *c2w, *K;
  const int* box;  // bx, by, bz minima, then maxima
  int Ho, Wo;
  float bg0, bg1, bg2;
  float *rgb, *color_out, *depth, *normal;
};

// grid 1, 256 threads: the bounding box of the B bricks
__global__ void __launch_bounds__(256) raycast_box_kernel(const int64_t* keys, long long B, int* box) {
  __shared__ int s[6];
  if (threadIdx.x < 3) s[threadIdx.x] = 0x7fffffff;
  else if (threadIdx.x < 6) s[threadIdx.x] = -0x7fffffff - 1;
  __syncthreads();
  int lo[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, hi[3] = {-0x7fffffff - 1, -0x7fffffff - 1, -0x7fffffff - 1};
  for (long long b = threadIdx.x; b < B; b += 256) {
    int q[3];
    key_brick(static_cast<unsigned long long>(keys[b]), q[0], q[1], q[2]);
    for (int c = 0; c < 3; ++c) {
      lo[c] = min(lo[c], q[c]);
      hi[c] = max(hi[c], q[c]);
    }
  }
  for (int c = 0; c < 3; ++c) {
    atomicMin(s + c, lo[c]);
    atomicMax(s + 3 + c, hi[c]);
  }
  __syncthreads();
  if (threadIdx.x < 6) box[threadIdx.x] = s[threadIdx.x];
}

// The bricks around the current base brick (that of a cell's lower corner): slot o = the brick at offset
// (o & 1, o >> 1 & 1, o >> 2), looked up by binary search when first needed.  Slots live in shared memory, [o][thread],
// so that a corner's run-time slot index does not put the cache on the stack.
struct BrickCache {
  int bx, by, bz;
  int* slots;  // stride kThreads

  __device__ void reset(int x, int y, int z) {
    bx = x;
    by = y;
    bz = z;
#pragma unroll
    for (int o = 0; o < 8; ++o) slots[o * kThreads] = kUnknown;
  }

  __device__ int get(const RayArgs& a, int o) {
    int n = slots[o * kThreads];
    if (n == kUnknown) {
      const int x = bx + (o & 1), y = by + (o >> 1 & 1), z = bz + (o >> 2);
      n = (x >= -kBias && y >= -kBias && z >= -kBias && x < kBias && y < kBias && z < kBias)
              ? find_brick(a.keys, a.B, static_cast<long long>(brick_key(x, y, z)))
              : kNoBrick;
      slots[o * kThreads] = n;
    }
    return n;
  }
};

struct Cell {
  int i[3];     // lower corner
  float f[3];   // fractions in [0, 1)
  long long g[8];  // corner samples, corner c at (c & 1, c >> 1 & 1, c >> 2)
};

// the cell of p and whether its base brick exists; cache moved to the base brick
__device__ __forceinline__ bool locate(const RayArgs& a, BrickCache& bc, const float* p, Cell& q) {
  for (int c = 0; c < 3; ++c) {
    const float s = p[c] / a.vox, fl = floorf(s);
    // beyond the brick range (or not finite): clamp into a coordinate that no brick has
    q.i[c] = fl >= -8.f * kBias && fl < 8.f * kBias ? static_cast<int>(fl) : -8 * kBias - 8;
    q.f[c] = s - fl;
  }
  const int bx = q.i[0] >> 3, by = q.i[1] >> 3, bz = q.i[2] >> 3;
  if (bx != bc.bx || by != bc.by || bz != bc.bz) bc.reset(bx, by, bz);
  return bc.get(a, 0) >= 0;
}

// the corner samples of cell q (its base brick exists) and whether all have weight >= min_weight
__device__ __forceinline__ bool cell_valid(const RayArgs& a, BrickCache& bc, Cell& q) {
  const int lx = q.i[0] & 7, ly = q.i[1] & 7, lz = q.i[2] & 7;
  bool ok = true;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int x = lx + (c & 1), y = ly + (c >> 1 & 1), z = lz + (c >> 2);
    const int n = ok ? bc.get(a, (x >> 3) | ((y >> 3) << 1) | ((z >> 3) << 2)) : kNoBrick;
    q.g[c] = n < 0 ? -1 : static_cast<long long>(n) * kBrickSamples + (((z & 7) << 6) | ((y & 7) << 3) | (x & 7));
    ok = ok && n >= 0 && __ldg(a.weight + q.g[c]) >= a.min_weight;
  }
  return ok;
}

__device__ __forceinline__ float lerp(float u, float w, float f) { return u + f * (w - u); }

// trilinear interpolation of corner values v[8] at fractions f
__device__ __forceinline__ float trilinear(const float* v, const float* f) {
  return lerp(lerp(lerp(v[0], v[1], f[0]), lerp(v[2], v[3], f[0]), f[1]),
              lerp(lerp(v[4], v[5], f[0]), lerp(v[6], v[7], f[0]), f[1]), f[2]);
}

__device__ __forceinline__ void point_at(const float* o, const float* d, float z, float* p) {
  for (int c = 0; c < 3; ++c) p[c] = fmaf(z, d[c], o[c]);
}

// T at ray depth z; false when z's cell is invalid
__device__ __forceinline__ bool field(const RayArgs& a, BrickCache& bc, const float* o, const float* d, float z,
                                      float& T) {
  float p[3];
  point_at(o, d, z, p);
  Cell q;
  if (!locate(a, bc, p, q) || !cell_valid(a, bc, q)) return false;
  float v[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) v[c] = __ldg(a.tsdf + q.g[c]);
  T = trilinear(v, q.f);
  return true;
}

__global__ void __launch_bounds__(kThreads) raycast_kernel(const __grid_constant__ RayArgs a) {
  __shared__ int slots[8 * kThreads];
  const int t = threadIdx.y * kTileX + threadIdx.x;
  const int col = blockIdx.x * kTileX + threadIdx.x, row = blockIdx.y * kTileY + threadIdx.y, cam = blockIdx.z;
  if (col >= a.Wo || row >= a.Ho) return;
  const long long pix = (static_cast<long long>(cam) * a.Ho + row) * a.Wo + col;
  const float* M = a.c2w + cam * 16;
  const float* K = a.K + cam * 9;
  const float dc[3] = {(static_cast<float>(col) - K[2]) / K[0], (static_cast<float>(row) - K[5]) / K[4], 1.f};
  float o[3], d[3];
  for (int r = 0; r < 3; ++r) {
    d[r] = M[r * 4] * dc[0] + M[r * 4 + 1] * dc[1] + M[r * 4 + 2] * dc[2];
    o[r] = M[r * 4 + 3];
  }
  bool hit = false;
  float z = 0.f, zn = 0.f;
  BrickCache bc{0x7fffffff, 0, 0, slots + t};
  // the ray's overlap with the bricks' box, from near
  float za = a.near, zb = INFINITY;
  bool inside = a.B > 0;
  for (int c = 0; c < 3 && inside; ++c) {
    const float lo = static_cast<float>(kBrick * a.box[c]) * a.vox, hi = static_cast<float>(kBrick * (a.box[3 + c] + 1)) * a.vox;
    if (d[c] == 0.f) {
      inside = o[c] >= lo && o[c] <= hi;
    } else {
      const float t1 = (lo - o[c]) / d[c], t2 = (hi - o[c]) / d[c];
      za = fmaxf(za, fminf(t1, t2));
      zb = fminf(zb, fmaxf(t1, t2));
    }
  }
  const float dz = 0.5f * a.vox / sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  if (inside && za <= zb && isfinite(dz) && dz > 0.f) {
    bool prev = false;
    float Tp = 0.f;
    for (int k = 0;;) {
      const float zk = fmaf(static_cast<float>(k), dz, za);
      if (!(zk <= zb)) break;
      float p[3];
      point_at(o, d, zk, p);
      Cell q;
      if (!locate(a, bc, p, q)) {
        // the base brick is absent: on to the last sample before the ray leaves it
        float ex = INFINITY;
        const int b[3] = {bc.bx, bc.by, bc.bz};
        for (int c = 0; c < 3; ++c) {
          if (d[c] == 0.f) continue;
          const float face = static_cast<float>(kBrick * (b[c] + (d[c] > 0.f))) * a.vox;
          ex = fminf(ex, (face - o[c]) / d[c]);
        }
        const float kf = floorf((ex - za) / dz);
        if (!(kf < 2e9f)) break;
        k = max(k + 1, static_cast<int>(kf));
        prev = false;
        continue;
      }
      const bool valid = cell_valid(a, bc, q);
      float T = 0.f;
      if (valid) {
        float v[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) v[c] = __ldg(a.tsdf + q.g[c]);
        T = trilinear(v, q.f);
      }
      if (valid && prev && Tp > 0.f && !(T > 0.f)) {
        // bisection of [z_{k-1}, z_k], T(z0) > 0 >= T(z1)
        float z0 = fmaf(static_cast<float>(k - 1), dz, za), z1 = zk, f0 = Tp, f1 = T;
        for (int it = 0; it < kRefine; ++it) {
          const float m = 0.5f * (z0 + z1);
          float fm = 0.f;
          const bool ok = field(a, bc, o, d, m, fm);
          if (!ok || !(fm > 0.f)) {
            if (ok) f1 = fm;
            z1 = m;
          } else {
            z0 = m;
            f0 = fm;
          }
        }
        z = z0 + (z1 - z0) * (f0 / (f0 - f1));
        zn = z0;
        hit = true;
        break;
      }
      prev = valid;
      Tp = T;
      ++k;
    }
  }
  if (!hit) {
    a.depth[pix] = 0.f;
    const float bg[3] = {a.bg0, a.bg1, a.bg2};
    for (int c = 0; c < 3; ++c) {
      a.normal[pix * 3 + c] = 0.f;
      a.color_out[pix * 3 + c] = bg[c];
      a.rgb[pix * 3 + c] = bg[c];
    }
    return;
  }
  // normal and colour in z's cell, or in the near end's (valid) cell
  float p[3];
  point_at(o, d, z, p);
  Cell q;
  if (!locate(a, bc, p, q) || !cell_valid(a, bc, q)) {
    point_at(o, d, zn, p);
    locate(a, bc, p, q);
    cell_valid(a, bc, q);
  }
  float v[8], g[3];
#pragma unroll
  for (int c = 0; c < 8; ++c) v[c] = __ldg(a.tsdf + q.g[c]);
  const float* f = q.f;
  // partial derivatives in cell units (the common 1 / v drops out when normalised)
  g[0] = lerp(lerp(v[1] - v[0], v[3] - v[2], f[1]), lerp(v[5] - v[4], v[7] - v[6], f[1]), f[2]);
  g[1] = lerp(lerp(v[2] - v[0], v[3] - v[1], f[0]), lerp(v[6] - v[4], v[7] - v[5], f[0]), f[2]);
  g[2] = lerp(lerp(v[4] - v[0], v[5] - v[1], f[0]), lerp(v[6] - v[2], v[7] - v[3], f[0]), f[1]);
  const float gn = sqrtf(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
  const float dn = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  float ndr = 0.f;
  for (int c = 0; c < 3; ++c) {
    g[c] = gn > 0.f ? g[c] / gn : 0.f;
    ndr += g[c] * (d[c] / dn);
  }
  const float shade = kAmbient + (1.f - kAmbient) * fmaxf(0.f, -ndr);
  a.depth[pix] = z;
  for (int ch = 0; ch < 3; ++ch) {
    float cv[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) cv[c] = __ldg(a.color + q.g[c] * 3 + ch);
    const float col3 = trilinear(cv, f);
    a.normal[pix * 3 + ch] = g[ch];
    a.color_out[pix * 3 + ch] = col3;
    a.rgb[pix * 3 + ch] = col3 * shade;
  }
}

}  // namespace
}  // namespace sta

using namespace sta;

extern "C" {

size_t sta_raycast_scratch_bytes(int64_t num_bricks) {
  if (num_bricks < 0 || num_bricks > STA_FUSION_MAX_BRICKS) return 0;
  return 32;  // the box, 6 ints, padded to 16 bytes
}

int sta_raycast(const int64_t* keys, int64_t num_bricks, const float* tsdf, const float* weight, const float* color,
                float voxel, float min_weight, const float* c2w, const float* K, int C, int Ho, int Wo, float near,
                const float* background, void* scratch, size_t scratch_bytes, float* rgb_out, float* color_out,
                float* depth_out, float* normal_out, void* stream) {
  STA_REQUIRE(C >= 1 && C <= kMaxSide && Ho >= 1 && Ho <= kMaxSide && Wo >= 1 && Wo <= kMaxSide,
              "cameras and output size must lie in [1, 8192]");
  STA_REQUIRE(num_bricks >= 0 && num_bricks <= STA_FUSION_MAX_BRICKS, "brick count outside [0, STA_FUSION_MAX_BRICKS]");
  STA_REQUIRE(isfinite(voxel) && voxel > 0.f, "voxel size must be positive and finite");
  STA_REQUIRE(isfinite(min_weight) && min_weight >= 1.f, "min_weight must be at least 1");
  STA_REQUIRE(isfinite(near) && near > 0.f, "the near plane must be positive and finite");
  STA_REQUIRE(num_bricks == 0 || (keys && tsdf && weight && color), "null volume");
  STA_REQUIRE(c2w && K && background, "null camera or background");
  STA_REQUIRE(rgb_out && color_out && depth_out && normal_out, "null output");
  STA_REQUIRE(scratch != nullptr && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0, "null or misaligned scratch");
  STA_REQUIRE(scratch_bytes >= sta_raycast_scratch_bytes(num_bricks), "scratch smaller than sta_raycast_scratch_bytes");
  STA_REQUIRE(on_device(c2w) && on_device(K) && on_device(scratch) && on_device(rgb_out) && on_device(color_out) &&
                  on_device(depth_out) && on_device(normal_out) &&
                  (num_bricks == 0 || (on_device(keys) && on_device(tsdf) && on_device(weight) && on_device(color))),
              "every array but the background must be device memory");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int* box = static_cast<int*>(scratch);
  if (num_bricks > 0) {
    raycast_box_kernel<<<1, 256, 0, st>>>(keys, num_bricks, box);
    STA_CHECK_CUDA(cudaGetLastError());
  }
  const RayArgs a{keys,  num_bricks, tsdf,          weight,          color,         voxel,     min_weight,
                  near,  c2w,        K,             box,             Ho,            Wo,        background[0],
                  background[1],     background[2], rgb_out,         color_out,     depth_out, normal_out};
  const dim3 grid((Wo + kTileX - 1) / kTileX, (Ho + kTileY - 1) / kTileY, C);
  raycast_kernel<<<grid, dim3(kTileX, kTileY), 0, st>>>(a);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
