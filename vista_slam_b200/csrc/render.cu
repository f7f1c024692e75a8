// Map renderer (OnlineSLAM.render, tools/render_video.py): z-buffered point splats of every confident map pixel and
// depth-tested line segments (camera frusta, pose-graph edges), seen from C cameras in one launch sequence.
//
// The map is what sta_graph_export gives without the cloud, so a live graph and a folder of saved files share this path:
//   clear                  the 64-bit z-buffer [C][Ho][Wo] to all ones (empty);
//   render_points_kernel   grid (H, V): each conf > thres pixel is unprojected with the PLY's arithmetic (cloud.cuh:
//                          K^-1 from the fp64 adjugate, unproject_f32 of depth * scale), read once and projected into
//                          every camera; it covers the (2 r + 1)^2 pixels centred on floor(u / w + 0.5),
//                          floor(v / w + 0.5) and keeps at each the smaller key (float_as_uint(z) << 32) | id;
//   render_segments_kernel grid (L, C): a segment clipped to z >= near in camera space and to the image (grown by the
//                          radius) in 2D (Liang-Barsky), then a DDA over max(|du|, |dv|) steps with perspective-correct
//                          z, splatted into the same z-buffer;
//   render_resolve_kernel  per output pixel: the key's id picks the winning point's colour (img + 1) / 2 or the
//                          segment's colour; depth is the key's z.
// z >= near > 0 makes z a positive float, whose bits order as the floats do; the id (v H W + row W + col for a point,
// V H W + l for segment l) breaks ties, so the minimum -- and the image -- does not depend on the order of the atomics.
#include <algorithm>
#include <cstdint>

#include "../../include/sta_b200.h"
#include "cloud.cuh"
#include "host_util.h"

namespace sta {
namespace {

constexpr unsigned long long kEmpty = ~0ull;
constexpr int kMaxSide = 8192;

// camera-frame point of world p under the row-major 4x4 world-to-camera M
__device__ __forceinline__ void to_camera(const float* M, const float* p, float* q) {
  for (int c = 0; c < 3; ++c) q[c] = M[c * 4] * p[0] + M[c * 4 + 1] * p[1] + M[c * 4 + 2] * p[2] + M[c * 4 + 3];
}

// image position (u / w, v / w) of camera-frame q through K
__device__ __forceinline__ void to_image(const float* K, const float* q, float& x, float& y) {
  const float u = K[0] * q[0] + K[1] * q[1] + K[2] * q[2], v = K[3] * q[0] + K[4] * q[1] + K[5] * q[2],
              w = K[6] * q[0] + K[7] * q[1] + K[8] * q[2];
  x = u / w;
  y = v / w;
}

// keep the smaller key at pixel p; the plain read first skips the atomic when it cannot win (keys only decrease, so a
// stale read is never smaller than the value the atomic would see)
__device__ __forceinline__ void splat_min(unsigned long long* p, unsigned long long key) {
  if (key < __ldcg(p)) atomicMin(p, key);
}

// the (2 r + 1)^2 pixels centred on the rounded (x, y) that lie in the Ho x Wo image; non-finite positions are dropped
__device__ __forceinline__ void splat(unsigned long long* zbuf, int Ho, int Wo, int r, float x, float y,
                                      unsigned long long key) {
  const float cx = floorf(x + 0.5f), cy = floorf(y + 0.5f);
  if (!(cx >= -r && cx <= Wo - 1 + r && cy >= -r && cy <= Ho - 1 + r)) return;
  const int px = static_cast<int>(cx), py = static_cast<int>(cy);
  for (int yy = max(0, py - r); yy <= min(Ho - 1, py + r); ++yy)
    for (int xx = max(0, px - r); xx <= min(Wo - 1, px + r); ++xx)
      splat_min(zbuf + static_cast<long long>(yy) * Wo + xx, key);
}

__device__ __forceinline__ unsigned long long make_key(float z, unsigned id) {
  return (static_cast<unsigned long long>(__float_as_uint(z)) << 32) | id;
}

struct RenderArgs {
  const float *depth, *conf, *pose, *scale, *intri;
  const float *w2c, *K, *segs;
  int H, W, C, Ho, Wo, r;
  float thres, near;
  unsigned long long* zbuf;
};

// grid (H, V), 256 threads: row blockIdx.x of view blockIdx.y
__global__ void __launch_bounds__(256) render_points_kernel(const __grid_constant__ RenderArgs a) {
  const int v = blockIdx.y, row = blockIdx.x, W = a.W;
  const long long hw = static_cast<long long>(a.H) * W;
  const float* P = a.pose + v * 16;
  float Ki[9];
  inv3_f32(a.intri + v * 9, Ki);
  const float s = a.scale[v];
  const long long base = v * hw + static_cast<long long>(row) * W;
  const long long plane = static_cast<long long>(a.Ho) * a.Wo;
  for (int x = threadIdx.x; x < W; x += 256) {
    if (!(a.conf[base + x] > a.thres)) continue;
    float p[3];
    unproject_f32(Ki, P, static_cast<float>(x), static_cast<float>(row), a.depth[base + x] * s, p);
    const unsigned id = static_cast<unsigned>(base + x);
    for (int c = 0; c < a.C; ++c) {
      float q[3], u, w;
      to_camera(a.w2c + c * 16, p, q);
      if (!(q[2] >= a.near)) continue;
      to_image(a.K + c * 9, q, u, w);
      splat(a.zbuf + c * plane, a.Ho, a.Wo, a.r, u, w, make_key(q[2], id));
    }
  }
}

// Liang-Barsky: narrow [t0, t1] to where p + t d satisfies lo <= . <= hi; false when empty
__device__ __forceinline__ bool clip_axis(float p, float d, float lo, float hi, float& t0, float& t1) {
  if (d == 0.f) return p >= lo && p <= hi;
  float a = (lo - p) / d, b = (hi - p) / d;
  if (a > b) {
    const float t = a;
    a = b;
    b = t;
  }
  t0 = fmaxf(t0, a);
  t1 = fminf(t1, b);
  return t0 <= t1;
}

// grid (L, C), 128 threads: segment blockIdx.x seen from camera blockIdx.y, its DDA steps spread over the threads
__global__ void __launch_bounds__(128) render_segments_kernel(const __grid_constant__ RenderArgs a, unsigned id0) {
  const int l = blockIdx.x, c = blockIdx.y;
  const float* M = a.w2c + c * 16;
  const float* K = a.K + c * 9;
  float qa[3], qb[3];
  to_camera(M, a.segs + l * 6, qa);
  to_camera(M, a.segs + l * 6 + 3, qb);
  const bool ina = qa[2] >= a.near, inb = qb[2] >= a.near;
  if (!ina && !inb) return;
  // the part in front of the near plane: the endpoint behind it moves along the segment onto it
  if (!ina || !inb) {
    const float t = (a.near - (ina ? qa[2] : qb[2])) / (ina ? qb[2] - qa[2] : qa[2] - qb[2]);
    for (int k = 0; k < 2; ++k) {
      const float f = ina ? qa[k] : qb[k], b = ina ? qb[k] : qa[k], m = f + t * (b - f);
      qa[k] = ina ? qa[k] : m;
      qb[k] = ina ? m : qb[k];
    }
    qa[2] = ina ? qa[2] : a.near;
    qb[2] = ina ? a.near : qb[2];
  }
  float xa, ya, xb, yb;
  to_image(K, qa, xa, ya);
  to_image(K, qb, xb, yb);
  const float du = xb - xa, dv = yb - ya;
  if (!isfinite(xa) || !isfinite(ya) || !isfinite(du) || !isfinite(dv)) return;
  // clip to the pixels whose footprint can reach the image, so an off-screen endpoint cannot blow up the step count
  float t0 = 0.f, t1 = 1.f;
  const float rr = a.r + 0.5f;
  if (!clip_axis(xa, du, -rr, a.Wo - 1 + rr, t0, t1) || !clip_axis(ya, dv, -rr, a.Ho - 1 + rr, t0, t1)) return;
  const float x0 = xa + t0 * du, y0 = ya + t0 * dv;
  const float cu = (t1 - t0) * du, cv = (t1 - t0) * dv;
  const int n = static_cast<int>(ceilf(fmaxf(fabsf(cu), fabsf(cv))));
  const float za = qa[2], zb = qb[2];
  unsigned long long* zbuf = a.zbuf + c * static_cast<long long>(a.Ho) * a.Wo;
  const unsigned id = id0 + static_cast<unsigned>(l);
  for (int k = threadIdx.x; k <= n; k += blockDim.x) {
    const float f = n > 0 ? static_cast<float>(k) / static_cast<float>(n) : 0.f;
    const float x = n > 0 ? x0 + cu * static_cast<float>(k) / static_cast<float>(n) : x0;
    const float y = n > 0 ? y0 + cv * static_cast<float>(k) / static_cast<float>(n) : y0;
    // screen parameter s of the original segment; z is linear in 1/z there: z = za + za s (zb - za) / (zb + s (za - zb)),
    // exact when za == zb
    const float s = t0 + f * (t1 - t0);
    // (held at near or beyond, so that rounding at a clipped endpoint keeps the key's z positive)
    const float z = fmaxf(za + za * s * (zb - za) / (zb + s * (za - zb)), a.near);
    splat(zbuf, a.Ho, a.Wo, a.r, x, y, make_key(z, id));
  }
}

// grid-stride over the output pixels of the C cameras
__global__ void __launch_bounds__(256) render_resolve_kernel(const unsigned long long* zbuf, long long n, const float* imgs,
                                                             long long hw, unsigned num_points, const float* seg_colors,
                                                             float b0, float b1, float b2, float* rgb, float* depth,
                                                             int64_t* index) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const unsigned long long key = zbuf[i];
    if (key == kEmpty) {
      rgb[i * 3] = b0;
      rgb[i * 3 + 1] = b1;
      rgb[i * 3 + 2] = b2;
      depth[i] = 0.f;
      index[i] = -1;
      continue;
    }
    const unsigned id = static_cast<unsigned>(key & 0xffffffffu);
    if (id < num_points) {
      const long long v = id / hw, pix = id - v * hw;
      for (int c = 0; c < 3; ++c) rgb[i * 3 + c] = (imgs[(v * 3 + c) * hw + pix] + 1.f) / 2.f;
    } else {
      for (int c = 0; c < 3; ++c) rgb[i * 3 + c] = seg_colors[(id - num_points) * 3ll + c];
    }
    depth[i] = __uint_as_float(static_cast<unsigned>(key >> 32));
    index[i] = id;
  }
}

}  // namespace
}  // namespace sta

extern "C" {

size_t sta_render_scratch_bytes(int num_cams, int Ho, int Wo) {
  if (num_cams < 1 || Ho < 1 || Wo < 1) return 0;
  return static_cast<size_t>(num_cams) * Ho * Wo * sizeof(unsigned long long);
}

int sta_render(const float* depth, const float* conf, const float* pose44, const float* scale, const float* intri,
               const float* imgs, int V, int H, int W, float conf_thres, const float* w2c, const float* K, int C, int Ho,
               int Wo, int radius, float near, const float* segs, const float* seg_colors, int L, const float* background,
               void* scratch, size_t scratch_bytes, float* rgb_out, float* depth_out, int64_t* index_out, void* stream) {
  using namespace sta;
  STA_REQUIRE(C >= 1 && C <= kMaxSide && Ho >= 1 && Ho <= kMaxSide && Wo >= 1 && Wo <= kMaxSide,
              "cameras and output size must lie in [1, 8192]");
  STA_REQUIRE(radius >= 0 && radius <= STA_RENDER_MAX_RADIUS, "point radius outside [0, STA_RENDER_MAX_RADIUS]");
  STA_REQUIRE(near > 0.f, "the near plane must be positive");
  STA_REQUIRE(V >= 0 && V <= 65535 && L >= 0, "0 to 65535 views and a non-negative segment count");
  STA_REQUIRE(V == 0 || (H >= 1 && W >= 1), "map size must be positive");
  const long long points = static_cast<long long>(V) * (V > 0 ? H : 0) * (V > 0 ? W : 0);
  STA_REQUIRE(points + L < 0xffffffffll, "V H W + L ids do not fit the 32-bit key id");
  STA_REQUIRE(V == 0 || (depth && conf && pose44 && scale && intri && imgs), "null map input");
  STA_REQUIRE(L == 0 || (segs && seg_colors), "null segments");
  STA_REQUIRE(w2c && K && background, "null camera or background");
  STA_REQUIRE(rgb_out && depth_out && index_out, "null output");
  STA_REQUIRE(scratch != nullptr && (reinterpret_cast<uintptr_t>(scratch) & 7) == 0, "null or misaligned scratch");
  STA_REQUIRE(scratch_bytes >= sta_render_scratch_bytes(C, Ho, Wo), "scratch smaller than sta_render_scratch_bytes");
  STA_REQUIRE(on_device(w2c) && on_device(K) && on_device(scratch) && on_device(rgb_out) && on_device(depth_out) &&
                  on_device(index_out) && (L == 0 || (on_device(segs) && on_device(seg_colors))) &&
                  (V == 0 || (on_device(depth) && on_device(conf) && on_device(pose44) && on_device(scale) &&
                              on_device(intri) && on_device(imgs))),
              "every array but the background must be device memory");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long n = static_cast<long long>(C) * Ho * Wo;
  unsigned long long* zbuf = static_cast<unsigned long long*>(scratch);
  STA_CHECK_CUDA(cudaMemsetAsync(zbuf, 0xff, n * sizeof(unsigned long long), st));
  RenderArgs a{depth, conf, pose44, scale, intri, w2c, K, segs, H, W, C, Ho, Wo, radius, conf_thres, near, zbuf};
  if (V > 0) {
    render_points_kernel<<<dim3(H, V), 256, 0, st>>>(a);
    STA_CHECK_CUDA(cudaGetLastError());
  }
  if (L > 0) {
    render_segments_kernel<<<dim3(L, C), 128, 0, st>>>(a, static_cast<unsigned>(points));
    STA_CHECK_CUDA(cudaGetLastError());
  }
  render_resolve_kernel<<<static_cast<unsigned>(std::min<long long>((n + 255) / 256, 1 << 20)), 256, 0, st>>>(
      zbuf, n, imgs, static_cast<long long>(H) * W, static_cast<unsigned>(points), seg_colors, background[0],
      background[1], background[2], rgb_out, depth_out, index_out);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
