// ORB features on the device: cv2.ORB_create().detectAndCompute(gray, None) with OpenCV's defaults (nfeatures 500,
// scaleFactor 1.2f, nlevels 8, edgeThreshold 31, WTA_K 2, HARRIS_SCORE, patchSize 31, fastThreshold 20), as the loop
// detector of vista_slam/loop_detector.py runs it on every keyframe.
//
// Bit-exact with the numpy restatement under oracle/ (tests/test_loop_gpu.py), which is equal to cv2 4.13 on the golden
// frames (tests/test_loop_detector.py).  The pyramid (INTER_LINEAR_EXACT), FAST, the Harris sums and the centroid moments
// are integer work; every float step is one correctly-rounded operation in OpenCV's order (__fmul_rn / __fadd_rn /
// __fmaf_rn where OpenCV's SIMD blur fuses).  retainBest keeps every point tied with the n-th best, so the kept set
// does not depend on the order of the candidates; the output is sorted by (level, y, x).
//
// Stages (one stream, no host synchronisation): level 0 from uint8 or from the fp32 gray; levels 1..7 resized from the
// previous level; FAST scores; 3x3 non-max suppression, border filter and a per-level score histogram; the FAST
// threshold of retainBest(2n); Harris responses (one warp per candidate); retainBest(n) on them by counting; the
// canonical order; angles and descriptors (one warp per keypoint) on the blurred levels.
//
// A batch of F frames of one size runs the same launches with blockIdx.z = frame: frame f reads its input at f H W,
// works in scratch slice f (OrbLayout::total bytes apart) and writes output slot f (kOrbMaxKeypoints apart, count f).
// A frame's arithmetic does not depend on F.
#include "../../include/sta_b200.h"
#include "common.cuh"
#include "host_util.h"
#include "loop.h"
#include "orb_pattern.h"

#include <float.h>
#include <math.h>
#include <stdint.h>

namespace sta {

namespace {

constexpr int kFastThreshold = 20;
constexpr int kEdge = 31;
constexpr int kHalfPatch = 15;
constexpr int kNFeatures = 500;
constexpr int kMinSide = 32, kMaxSide = 4096;
constexpr int kFrame = 3;  // FAST reads a radius-3 circle

__constant__ int c_umax[kHalfPatch + 2];
__constant__ signed char c_pattern[1024];

struct LevelGeom {
  int h[kOrbLevels], w[kOrbLevels];
  long long ofs[kOrbLevels];
  int quota[kOrbLevels];
  float scale[kOrbLevels];
};

inline size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

// p moved to the slice of frame blockIdx.z, `bytes` apart
template <typename T>
__device__ __forceinline__ T* frame_slice(T* p, size_t bytes) {
  return reinterpret_cast<T*>(reinterpret_cast<uintptr_t>(p) + static_cast<uintptr_t>(blockIdx.z) * bytes);
}

__device__ __forceinline__ OrbOut frame_out(OrbOut o) {
  const int f = blockIdx.z;
  const long long m = static_cast<long long>(f) * kOrbMaxKeypoints;
  return {o.xy + m, o.level + m, o.pts + m, o.angle + m, o.response + m, o.desc + 32 * m, o.count + f};
}

float level_scale(int l) { return static_cast<float>(pow(static_cast<double>(1.2f), static_cast<double>(l))); }

LevelGeom geom_of(const OrbLayout& s) {
  LevelGeom g = {};
  for (int l = 0; l < kOrbLevels; ++l) {
    g.h[l] = s.h[l];
    g.w[l] = s.w[l];
    g.ofs[l] = s.lvl[l];
    g.quota[l] = s.quota[l];
    g.scale[l] = level_scale(l);
  }
  return g;
}

__device__ __forceinline__ int reflect101(int i, int n) {
  i = i < 0 ? -i : i;
  return i >= n ? 2 * (n - 1) - i : i;
}

__global__ void to_u8_kernel(const void* frame, int is_f32, int n, uint8_t* out, size_t fs) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  frame = frame_slice(static_cast<const char*>(frame), static_cast<size_t>(n) * (is_f32 ? 4 : 1));
  out = frame_slice(out, fs);
  if (is_f32) {
    // (gray * 255).astype(np.uint8): an fp32 multiply, then truncation
    out[i] = static_cast<uint8_t>(static_cast<int>(__fmul_rn(static_cast<const float*>(frame)[i], 255.f)));
  } else {
    out[i] = static_cast<const uint8_t*>(frame)[i];
  }
}

// interpolationLinear::getCoeffs of resize_bitExact: offset and 8-bit weight of the second tap (-1: clamp to `clampto`)
__device__ __forceinline__ void linear_coeff(int i, int src, int dst, int& ofs, int& w1) {
  const double scale = __ddiv_rn(1.0, __ddiv_rn(static_cast<double>(dst), static_cast<double>(src)));
  const double fval = __dsub_rn(__dmul_rn(scale, __dadd_rn(static_cast<double>(i), 0.5)), 0.5);
  const double fl = floor(fval);
  const int iv = static_cast<int>(fl);
  if (iv >= 0 && src > 1 && iv < src - 1) {
    ofs = iv;
    w1 = __double2int_rn(__dmul_rn(__dsub_rn(fval, fl), 256.0));
  } else {
    ofs = (iv >= 0 && src > 1) ? src - 1 : 0;
    w1 = 0;
  }
}

// cv::resize(src, dst, dsize, 0, 0, INTER_LINEAR_EXACT): (sum of 8-bit x 8-bit weighted taps + 2^15) >> 16
__global__ void resize_kernel(const uint8_t* src, int sh, int sw, uint8_t* dst, int dh, int dw, size_t fs) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= dh * dw) return;
  src = frame_slice(src, fs);
  dst = frame_slice(dst, fs);
  const int y = i / dw, x = i - y * dw;
  int xo, xw1, yo, yw1;
  linear_coeff(x, sw, dw, xo, xw1);
  linear_coeff(y, sh, dh, yo, yw1);
  const int xo1 = min(xo + 1, sw - 1), yo1 = min(yo + 1, sh - 1);
  const uint8_t* r0 = src + static_cast<long long>(yo) * sw;
  const uint8_t* r1 = src + static_cast<long long>(yo1) * sw;
  const int h0 = r0[xo] * (256 - xw1) + r0[xo1] * xw1;
  const int h1 = r1[xo] * (256 - xw1) + r1[xo1] * xw1;
  const int v = h0 * (256 - yw1) + h1 * yw1;
  dst[i] = static_cast<uint8_t>(min((v + (1 << 15)) >> 16, 255));
}

// FAST-9 score (cornerScore<16>) where the pixel is a corner, else 0.  blockIdx.y = level.
__global__ void fast_kernel(const uint8_t* pyr, LevelGeom g, uint8_t* score, size_t fs) {
  pyr = frame_slice(pyr, fs);
  score = frame_slice(score, fs);
  const int l = blockIdx.y;
  const int h = g.h[l], w = g.w[l];
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= h * w) return;
  const int y = i / w, x = i - y * w;
  uint8_t out = 0;
  if (y >= kFrame && y < h - kFrame && x >= kFrame && x < w - kFrame) {
    const uint8_t* img = pyr + g.ofs[l];
    const int dx[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
    const int dy[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};
    const int v = img[y * w + x];
    int d[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) d[k] = v - img[(y + dy[k]) * w + x + dx[k]];
    int A = -1 << 20, B = -1 << 20;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      int mn = 1 << 20, mx = -(1 << 20);
#pragma unroll
      for (int j = 0; j < 9; ++j) {
        mn = min(mn, d[(k + j) & 15]);
        mx = max(mx, d[(k + j) & 15]);
      }
      A = max(A, mn);
      B = max(B, -mx);
    }
    if (A > kFastThreshold || B > kFastThreshold) out = static_cast<uint8_t>(max(max(A, B), kFastThreshold) - 1);
  }
  score[g.ofs[l] + i] = out;
}

// Non-max suppression (strictly above all 8 neighbours), border filter, candidate list and score histogram.
__global__ void nms_kernel(const uint8_t* score, LevelGeom g, int4* cand, unsigned* hist, unsigned* counters,
                           size_t fs) {
  score = frame_slice(score, fs);
  cand = frame_slice(cand, fs);
  hist = frame_slice(hist, fs);
  counters = frame_slice(counters, fs);
  const int l = blockIdx.y;
  const int h = g.h[l], w = g.w[l];
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= h * w || h <= 2 * kEdge || w <= 2 * kEdge) return;
  const int y = i / w, x = i - y * w;
  if (y < kEdge || y >= h - kEdge || x < kEdge || x >= w - kEdge) return;
  const uint8_t* sc = score + g.ofs[l];
  const int s = sc[i];
  if (s == 0) return;
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx)
      if ((dy || dx) && sc[(y + dy) * w + x + dx] >= s) return;
  const unsigned k = atomicAdd(&counters[0], 1u);
  if (k >= kOrbMaxCandidates) {
    atomicExch(&counters[3], 1u);
    return;
  }
  cand[k] = make_int4(l, x, y, s);
  atomicAdd(&hist[l * 256 + s], 1u);
}

// retainBest(2 n_l) on the integer FAST score: the smallest kept score per level (256 = keep none).
__global__ void fast_threshold_kernel(const unsigned* hist, LevelGeom g, int* thr, size_t fs) {
  hist = frame_slice(hist, fs);
  thr = frame_slice(thr, fs);
  const int l = threadIdx.x;
  if (l >= kOrbLevels) return;
  const unsigned want = 2u * g.quota[l];
  unsigned total = 0;
  for (int s = 0; s < 256; ++s) total += hist[l * 256 + s];
  int t = 0;
  if (total > want) {
    t = 256;
    unsigned acc = 0;
    for (int s = 255; s >= 0 && want > 0; --s) {
      acc += hist[l * 256 + s];
      if (acc >= want) {
        t = s;
        break;
      }
    }
  }
  thr[l] = t;
}

// HarrisResponses(blockSize 7, k 0.04) of the candidates that pass retainBest(2n); one warp per candidate.
__global__ void harris_kernel(const uint8_t* pyr, LevelGeom g, const int4* cand, const int* thr, float* resp,
                              int* alive, unsigned* counters, size_t fs) {
  pyr = frame_slice(pyr, fs);
  cand = frame_slice(cand, fs);
  thr = frame_slice(thr, fs);
  resp = frame_slice(resp, fs);
  alive = frame_slice(alive, fs);
  counters = frame_slice(counters, fs);
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int n = min(counters[0], static_cast<unsigned>(kOrbMaxCandidates));
  if (warp >= n) return;
  const int4 c = cand[warp];
  if (c.w < thr[c.x]) return;
  const int w = g.w[c.x];
  const uint8_t* img = pyr + g.ofs[c.x];
  int a = 0, b = 0, cc = 0;
  for (int k = lane; k < 49; k += 32) {
    const int y = c.z - 3 + k / 7, x = c.y - 3 + k % 7;
    const uint8_t* p = img + y * w + x;
    const int Ix = (p[1] - p[-1]) * 2 + (p[-w + 1] - p[-w - 1]) + (p[w + 1] - p[w - 1]);
    const int Iy = (p[w] - p[-w]) * 2 + (p[w - 1] - p[-w - 1]) + (p[w + 1] - p[-w + 1]);
    a += Ix * Ix;
    b += Iy * Iy;
    cc += Ix * Iy;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
    cc += __shfl_xor_sync(0xffffffffu, cc, o);
  }
  if (lane == 0) {
    const float scale = __fdiv_rn(1.f, __fmul_rn(28.f, 255.f));
    const float s4 = __fmul_rn(__fmul_rn(__fmul_rn(scale, scale), scale), scale);
    const float fa = static_cast<float>(a), fb = static_cast<float>(b), fc = static_cast<float>(cc);
    const float sab = __fadd_rn(fa, fb);
    const float t = __fsub_rn(__fsub_rn(__fmul_rn(fa, fb), __fmul_rn(fc, fc)), __fmul_rn(__fmul_rn(0.04f, sab), sab));
    resp[warp] = __fmul_rn(t, s4);
    alive[atomicAdd(&counters[1], 1u)] = warp;
  }
}

// retainBest(n_l) on the Harris response: keep a candidate when fewer than n_l of its level respond more strongly.
__global__ void harris_select_kernel(const int4* cand, const float* resp, const int* alive, LevelGeom g, int* kept,
                                     unsigned* counters, size_t fs) {
  cand = frame_slice(cand, fs);
  resp = frame_slice(resp, fs);
  alive = frame_slice(alive, fs);
  kept = frame_slice(kept, fs);
  counters = frame_slice(counters, fs);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int m = counters[1];
  if (i >= m) return;
  const int ci = alive[i];
  const int l = cand[ci].x;
  const float r = resp[ci];
  int greater = 0;
  for (int j = 0; j < m; ++j) {
    const int cj = alive[j];
    greater += (cand[cj].x == l && resp[cj] > r) ? 1 : 0;
  }
  if (greater >= g.quota[l]) return;
  const unsigned k = atomicAdd(&counters[2], 1u);
  if (k >= kOrbMaxKeypoints) {
    atomicExch(&counters[3], 1u);
    return;
  }
  kept[k] = ci;
}

// Canonical order (level, y, x) by counting; writes the keypoint fields that need no image.
__global__ void order_kernel(const int4* cand, const float* resp, const int* kept, LevelGeom g, unsigned* counters,
                             OrbOut out, size_t fs) {
  cand = frame_slice(cand, fs);
  resp = frame_slice(resp, fs);
  kept = frame_slice(kept, fs);
  counters = frame_slice(counters, fs);
  out = frame_out(out);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int m = min(counters[2], static_cast<unsigned>(kOrbMaxKeypoints));
  if (i == 0) *out.count = m;
  if (i >= m) return;
  const int4 c = cand[kept[i]];
  const long long key = (static_cast<long long>(c.x) << 40) | (static_cast<long long>(c.z) << 20) | c.y;
  int rank = 0;
  for (int j = 0; j < m; ++j) {
    const int4 d = cand[kept[j]];
    rank += ((static_cast<long long>(d.x) << 40) | (static_cast<long long>(d.z) << 20) | d.y) < key ? 1 : 0;
  }
  out.xy[rank] = make_int2(c.y, c.z);
  out.level[rank] = c.x;
  out.response[rank] = resp[kept[i]];
  const float sc = g.scale[c.x];
  out.pts[rank] = make_float2(__fmul_rn(static_cast<float>(c.y), sc), __fmul_rn(static_cast<float>(c.z), sc));
}

// cv::fastAtan2 (degrees), each fp32 step rounded as OpenCV's scalar code does
__device__ float fast_atan2(float y, float x) {
  const float c180 = static_cast<float>(180.0 / 3.14159265358979323846);
  const float p1 = __fmul_rn(0.9997878412794807f, c180), p3 = __fmul_rn(-0.3258083974640975f, c180);
  const float p5 = __fmul_rn(0.1555786518463281f, c180), p7 = __fmul_rn(-0.04432655554792128f, c180);
  const float eps = static_cast<float>(DBL_EPSILON);
  const float ax = fabsf(x), ay = fabsf(y);
  float a, c;
  const bool big = ax >= ay;
  c = big ? __fdiv_rn(ay, __fadd_rn(ax, eps)) : __fdiv_rn(ax, __fadd_rn(ay, eps));
  const float c2 = __fmul_rn(c, c);
  a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
  if (!big) a = __fsub_rn(90.f, a);
  if (x < 0) a = __fsub_rn(180.f, a);
  if (y < 0) a = __fsub_rn(360.f, a);
  return a;
}

// ICAngles: intensity centroid over the radius-15 disc of the unsmoothed level; one warp per keypoint
__global__ void angle_kernel(const uint8_t* pyr, LevelGeom g, OrbOut out, size_t fs) {
  pyr = frame_slice(pyr, fs);
  out = frame_out(out);
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= *out.count) return;
  const int l = out.level[warp];
  const int2 p = out.xy[warp];
  const int w = g.w[l];
  const uint8_t* img = pyr + g.ofs[l] + static_cast<long long>(p.y) * w + p.x;
  int m01 = 0, m10 = 0;
  if (lane < 2 * kHalfPatch + 1) {
    const int v = lane - kHalfPatch;
    const int av = v < 0 ? -v : v;
    const int d = c_umax[av];
    for (int u = -d; u <= d; ++u) {
      const int val = img[v * w + u];
      m10 += u * val;
      m01 += v * val;
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    m01 += __shfl_xor_sync(0xffffffffu, m01, o);
    m10 += __shfl_xor_sync(0xffffffffu, m10, o);
  }
  if (lane == 0) out.angle[warp] = fast_atan2(static_cast<float>(m01), static_cast<float>(m10));
}

__constant__ float c_gauss[7];

// ORB's GaussianBlur(7x7, 2, REFLECT_101) of each level: fp32 row pass with fused multiply-adds left to right, then
// the symmetric column pass (centre, then (above + below) * tap, fused), rounded half to even.  blockIdx.y = level.
__global__ void blur_kernel(const uint8_t* pyr, LevelGeom g, uint8_t* blur, size_t fs) {
  pyr = frame_slice(pyr, fs);
  blur = frame_slice(blur, fs);
  const int l = blockIdx.y;
  const int h = g.h[l], w = g.w[l];
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= h * w) return;
  const int y = i / w, x = i - y * w;
  const uint8_t* img = pyr + g.ofs[l];
  int xs[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) xs[k] = reflect101(x + k - 3, w);
  float R[7];
#pragma unroll
  for (int r = 0; r < 7; ++r) {
    const uint8_t* row = img + static_cast<long long>(reflect101(y + r - 3, h)) * w;
    float acc = __fmul_rn(c_gauss[0], static_cast<float>(row[xs[0]]));
#pragma unroll
    for (int k = 1; k < 7; ++k) acc = __fmaf_rn(static_cast<float>(row[xs[k]]), c_gauss[k], acc);
    R[r] = acc;
  }
  float s = __fmul_rn(R[3], c_gauss[3]);
#pragma unroll
  for (int d = 1; d <= 3; ++d) s = __fmaf_rn(__fadd_rn(R[3 + d], R[3 - d]), c_gauss[3 + d], s);
  blur[g.ofs[l] + i] = static_cast<uint8_t>(min(max(__float2int_rn(s), 0), 255));
}

// rBRIEF: lane b writes descriptor byte b from 8 pair tests of the blurred level; one warp per keypoint
__global__ void desc_kernel(const uint8_t* blur, LevelGeom g, OrbOut out, size_t fs) {
  blur = frame_slice(blur, fs);
  out = frame_out(out);
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= *out.count) return;
  const int l = out.level[warp];
  const int2 p = out.xy[warp];
  const int w = g.w[l];
  const float sc = g.scale[l];
  const float inv = __fdiv_rn(1.f, sc);
  // orb.cpp scales the keypoint to level 0 and back: cvRound(pt * (1 / scale))
  const int cx = __float2int_rn(__fmul_rn(__fmul_rn(static_cast<float>(p.x), sc), inv));
  const int cy = __float2int_rn(__fmul_rn(__fmul_rn(static_cast<float>(p.y), sc), inv));
  const float ang = __fmul_rn(out.angle[warp], static_cast<float>(3.14159265358979323846 / 180.0));
  const float ca = __double2float_rn(cos(static_cast<double>(ang)));
  const float sa = __double2float_rn(sin(static_cast<double>(ang)));
  const uint8_t* center = blur + g.ofs[l] + static_cast<long long>(cy) * w + cx;
  int val = 0;
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    int v[2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int idx = (lane * 16 + t * 2 + q) * 2;
      const float px = static_cast<float>(c_pattern[idx]), py = static_cast<float>(c_pattern[idx + 1]);
      const float x = __fsub_rn(__fmul_rn(px, ca), __fmul_rn(py, sa));
      const float y = __fadd_rn(__fmul_rn(px, sa), __fmul_rn(py, ca));
      v[q] = center[__float2int_rn(y) * w + __float2int_rn(x)];
    }
    val |= (v[0] < v[1]) << t;
  }
  out.desc[warp * 32 + lane] = static_cast<uint8_t>(val);
}

int upload_constants() {
  static PerDeviceOnce once;
  return once.run([] {
    int umax[kHalfPatch + 2] = {};
    const int vmax = static_cast<int>(floor(kHalfPatch * sqrt(2.f) / 2 + 1));
    const int vmin = static_cast<int>(ceil(kHalfPatch * sqrt(2.f) / 2));
    for (int v = 0; v <= vmax; ++v) umax[v] = static_cast<int>(lrint(sqrt(static_cast<double>(kHalfPatch * kHalfPatch - v * v))));
    for (int v = kHalfPatch, v0 = 0; v >= vmin; --v) {
      while (umax[v0] == umax[v0 + 1]) ++v0;
      umax[v] = v0;
      ++v0;
    }
    // cv::getGaussianKernel(7, 2, CV_32F)
    const float gauss[7] = {0x1.1f5f62p-4f, 0x1.0c70fcp-3f, 0x1.869472p-3f, 0x1.ba95c0p-3f,
                            0x1.869472p-3f, 0x1.0c70fcp-3f, 0x1.1f5f62p-4f};
    cudaError_t e = cudaMemcpyToSymbol(c_umax, umax, sizeof(umax));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_pattern, kOrbPattern31, sizeof(kOrbPattern31));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_gauss, gauss, sizeof(gauss));
    return e;
  }) == cudaSuccess ? 0 : 1;
}

}  // namespace

bool orb_size_ok(int H, int W) { return H >= kMinSide && W >= kMinSide && H <= kMaxSide && W <= kMaxSide; }

OrbLayout orb_layout(int H, int W) {
  OrbLayout s = {};
  s.H = H;
  s.W = W;
  long long pix = 0;
  for (int l = 0; l < kOrbLevels; ++l) {
    const float sc = level_scale(l);
    s.h[l] = static_cast<int>(lrintf(static_cast<float>(H) / sc));
    s.w[l] = static_cast<int>(lrintf(static_cast<float>(W) / sc));
    s.lvl[l] = pix;
    pix += static_cast<long long>(s.h[l]) * s.w[l];
  }
  s.pix = pix;
  // computeKeyPoints: features per level in fp32
  const float factor = static_cast<float>(1.0 / static_cast<double>(1.2f));
  float nd = static_cast<float>(kNFeatures) * (1.f - factor) /
             (1.f - static_cast<float>(pow(static_cast<double>(factor), static_cast<double>(kOrbLevels))));
  int sum = 0;
  for (int l = 0; l < kOrbLevels - 1; ++l) {
    s.quota[l] = static_cast<int>(lrintf(nd));
    sum += s.quota[l];
    nd *= factor;
  }
  s.quota[kOrbLevels - 1] = kNFeatures - sum > 0 ? kNFeatures - sum : 0;
  size_t o = 0;
  s.pyr = o;      o = align256(o + pix);
  s.blur = o;     o = align256(o + pix);
  s.score = o;    o = align256(o + pix);
  s.cand = o;     o = align256(o + sizeof(int4) * kOrbMaxCandidates);
  s.resp = o;     o = align256(o + sizeof(float) * kOrbMaxCandidates);
  s.hist = o;     o = align256(o + sizeof(unsigned) * 256 * kOrbLevels);
  s.counters = o; o = align256(o + sizeof(unsigned) * 8 + sizeof(int) * kOrbLevels);
  s.alive = o;    o = align256(o + sizeof(int) * kOrbMaxCandidates);
  s.kept = o;     o = align256(o + sizeof(int) * kOrbMaxKeypoints);
  s.total = o;
  return s;
}

int orb_run(const OrbLayout& s, void* scratch, const void* frame, int is_f32, const OrbOut& out, cudaStream_t st, int F) {
  if (upload_constants()) {
    set_last_error("orb: constant upload failed");
    return 1;
  }
  char* base = static_cast<char*>(scratch);
  uint8_t* pyr = reinterpret_cast<uint8_t*>(base + s.pyr);
  uint8_t* blur = reinterpret_cast<uint8_t*>(base + s.blur);
  uint8_t* score = reinterpret_cast<uint8_t*>(base + s.score);
  int4* cand = reinterpret_cast<int4*>(base + s.cand);
  float* resp = reinterpret_cast<float*>(base + s.resp);
  unsigned* hist = reinterpret_cast<unsigned*>(base + s.hist);
  unsigned* counters = reinterpret_cast<unsigned*>(base + s.counters);
  int* thr = reinterpret_cast<int*>(counters + 8);
  int* alive = reinterpret_cast<int*>(base + s.alive);
  int* kept = reinterpret_cast<int*>(base + s.kept);
  const LevelGeom g = geom_of(s);
  const int n0 = s.H * s.W;
  const size_t fs = s.total;  // scratch slice of one frame
  STA_CHECK_CUDA(cudaMemset2DAsync(base + s.hist, fs, 0, s.alive - s.hist, F, st));
  to_u8_kernel<<<dim3((n0 + 255) / 256, 1, F), 256, 0, st>>>(frame, is_f32, n0, pyr, fs);
  for (int l = 1; l < kOrbLevels; ++l) {
    const int n = s.h[l] * s.w[l];
    resize_kernel<<<dim3((n + 255) / 256, 1, F), 256, 0, st>>>(pyr + s.lvl[l - 1], s.h[l - 1], s.w[l - 1], pyr + s.lvl[l],
                                                               s.h[l], s.w[l], fs);
  }
  const dim3 grid_lv((n0 + 255) / 256, kOrbLevels, F);
  fast_kernel<<<grid_lv, 256, 0, st>>>(pyr, g, score, fs);
  nms_kernel<<<grid_lv, 256, 0, st>>>(score, g, cand, hist, counters, fs);
  fast_threshold_kernel<<<dim3(1, 1, F), 32, 0, st>>>(hist, g, thr, fs);
  harris_kernel<<<dim3(kOrbMaxCandidates / 8, 1, F), 256, 0, st>>>(pyr, g, cand, thr, resp, alive, counters, fs);
  harris_select_kernel<<<dim3(kOrbMaxCandidates / 256, 1, F), 256, 0, st>>>(cand, resp, alive, g, kept, counters, fs);
  order_kernel<<<dim3(kOrbMaxKeypoints / 256, 1, F), 256, 0, st>>>(cand, resp, kept, g, counters, out, fs);
  angle_kernel<<<dim3(kOrbMaxKeypoints / 8, 1, F), 256, 0, st>>>(pyr, g, out, fs);
  blur_kernel<<<grid_lv, 256, 0, st>>>(pyr, g, blur, fs);
  desc_kernel<<<dim3(kOrbMaxKeypoints / 8, 1, F), 256, 0, st>>>(blur, g, out, fs);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace sta

using namespace sta;

extern "C" {

size_t sta_orb_scratch_bytes(int H, int W) { return orb_size_ok(H, W) ? orb_layout(H, W).total : 0; }

int sta_orb_layout(int H, int W, int64_t* out) {
  STA_REQUIRE(orb_size_ok(H, W), "ORB frame sides must be in [32, 4096]");
  const OrbLayout s = orb_layout(H, W);
  const size_t offs[10] = {s.total, s.pyr, s.blur, s.score, s.cand, s.resp, s.counters, s.alive, s.kept, s.hist};
  for (int i = 0; i < 10; ++i) out[i] = static_cast<int64_t>(offs[i]);
  for (int l = 0; l < kOrbLevels; ++l) {
    out[10 + 4 * l] = s.h[l];
    out[11 + 4 * l] = s.w[l];
    out[12 + 4 * l] = s.lvl[l];
    out[13 + 4 * l] = s.quota[l];
  }
  return 0;
}

int sta_op_orb(const void* frame_dev, int frame_is_f32, int H, int W, int32_t* xy_out, int32_t* level_out, float* pts_out,
               float* angle_out, float* response_out, uint8_t* desc_out, int32_t* count_out, void* scratch, void* stream) {
  STA_REQUIRE(orb_size_ok(H, W), "ORB frame sides must be in [32, 4096]");
  const OrbLayout s = orb_layout(H, W);
  OrbOut o = {reinterpret_cast<int2*>(xy_out), level_out, reinterpret_cast<float2*>(pts_out), angle_out, response_out,
              desc_out, count_out};
  return orb_run(s, scratch, frame_dev, frame_is_f32, o, static_cast<cudaStream_t>(stream));
}

// F frames [F][H][W] of one size: scratch of F sta_orb_scratch_bytes(H, W) bytes, outputs [F][STA_ORB_MAX_KEYPOINTS]
// and count_out [F]
int sta_op_orb_many(const void* frames_dev, int frames_is_f32, int F, int H, int W, int32_t* xy_out, int32_t* level_out,
                    float* pts_out, float* angle_out, float* response_out, uint8_t* desc_out, int32_t* count_out,
                    void* scratch, void* stream) {
  STA_REQUIRE(orb_size_ok(H, W), "ORB frame sides must be in [32, 4096]");
  STA_REQUIRE(F >= 1, "the frame count must be at least 1");
  const OrbLayout s = orb_layout(H, W);
  OrbOut o = {reinterpret_cast<int2*>(xy_out), level_out, reinterpret_cast<float2*>(pts_out), angle_out, response_out,
              desc_out, count_out};
  return orb_run(s, scratch, frames_dev, frames_is_f32, o, static_cast<cudaStream_t>(stream), F);
}

}  // extern "C"
