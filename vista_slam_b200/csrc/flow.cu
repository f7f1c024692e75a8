// SLAM keyframe flow tracker on the device: what FlowTracker.compute_disparity (vista_slam/flow_tracker.py:26-66) does on
// the host with OpenCV, with the reference's fixed constants --
//   cv2.goodFeaturesToTrack(maxCorners=1000, qualityLevel=0.01, minDistance=8, blockSize=7), gradient size 3, no Harris
//   cv2.calcOpticalFlowPyrLK(winSize=(21, 21), maxLevel=3, criteria=(EPS|COUNT, 30, 0.01)), flags 0, minEigThreshold 1e-4
// and the mean |dx|, |dy| of the tracked points that decides whether the frame becomes a keyframe.
//
// Bit-exact with the numpy restatement under oracle/ (tests/test_flow_gpu.py): the pyramid (pyrDown), the Scharr and Sobel
// derivatives, the 7x7 box sums and the LK window sums are integer work (the LK sums in int64, so they do not depend on
// the summation order), and every float step is one correctly-rounded fp32 operation (__fmul_rn / __fadd_rn / ...: nvcc
// would otherwise contract to FMA) in the order OpenCV's LKTrackerInvoker uses.  The greedy minimum-distance selection
// of goodFeaturesToTrack is resolved in rounds inside one CTA (see select_kernel); the result is the sequential one.
//
// Buffers (one arena per frame size): two padded pyramids (a tracker's keyframe and its first frame slot, swapped when
// that frame becomes the keyframe), the keyframe's Scharr derivatives, the corner selection scratch and the keyframe
// corners.  A tracker adds pyramid slots for the frames of its largest group track, and the LK output and statistics of
// every frame of a group it leads.
//
// Every stage runs over a batch: the pyramid kernels over frames, LK and the statistics over (frame, keyframe) items,
// the derivative and corner kernels over keyframes, each with the batch index in blockIdx.y (one CTA per keyframe in
// select_kernel, one per item in flow_stats_kernel).  The per-item pointers travel in a __grid_constant__ table of at
// most kMaxBatch entries; a larger batch is several launches.  One frame is a group of one.
#include "../../include/sta_b200.h"
#include "common.cuh"
#include "host_util.h"

#include <float.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

namespace sta {

namespace {

constexpr int kWin = 21;                 // winSize
constexpr int kPad = kWin;               // pyramid / derivative border: LK reads up to winSize outside a level
constexpr int kWinPix = kWin * kWin;     // 441 window pixels
constexpr int kPerLane = (kWinPix + 31) / 32;
constexpr int kMaxLevels = 4;            // maxLevel 3
constexpr int kMaxIters = 30;
constexpr double kEps2 = 0.01 * 0.01;    // criteria.epsilon, squared in double as calcOpticalFlowPyrLK does
constexpr double kMinEig = 1e-4;         // minEigThreshold
constexpr float kLkScale = 1.0f / (1 << 20);
constexpr int kWBits = 14;
constexpr float kEigScale2 = static_cast<float>(1.0 / (7140.0 * 7140.0));  // Sobel scale 1/(4*7*255), squared
constexpr int kMaxCorners = STA_FLOW_MAX_CORNERS;
constexpr int kMinSide = 32, kMaxSide = 2048;
constexpr int kSelectThreads = 1024;
constexpr int kMaxBatch = 64;  // frames, keyframes or LK items per launch (the LK table is 3.5 KB of parameters)

struct Levels {
  int nlev;
  int w[kMaxLevels], h[kMaxLevels];
  long long ofs[kMaxLevels];  // element offset of each padded level [h + 2 kPad][w + 2 kPad] in a pyramid
  long long total;            // elements of one pyramid
};

// buildOpticalFlowPyramid: level L exists while both of its sides are > winSize
Levels make_levels(int H, int W) {
  Levels L = {};
  int w = W, h = H;
  long long ofs = 0;
  for (int l = 0; l < kMaxLevels; ++l) {
    if (l > 0) {
      w = (w + 1) / 2;
      h = (h + 1) / 2;
      if (w <= kWin || h <= kWin) break;
    }
    L.w[l] = w;
    L.h[l] = h;
    L.ofs[l] = ofs;
    ofs += static_cast<long long>(w + 2 * kPad) * (h + 2 * kPad);
    L.nlev = l + 1;
  }
  L.total = ofs;
  return L;
}

// every buffer the tracker and the op-level entry points use, carved from one arena
struct Layout {
  Levels lv;
  size_t pyr[2], deriv, sob, eig, state, cand, acc, counters, corners, ncorners, total;
  int acc_cap;
};

enum { kCntMax = 0, kCntCand = 1, kCntAcc = 2, kNumCounters = 4 };

Layout make_layout(int H, int W) {
  Layout s;
  s.lv = make_levels(H, W);
  const long long hw = static_cast<long long>(H) * W;
  // accepted corners are >= 8 px apart, so a 5x5 block of pixels (diameter sqrt(32) < 8) holds at most one
  s.acc_cap = ((H + 4) / 5) * ((W + 4) / 5);
  size_t off = 0;
  auto take = [&](size_t bytes) {
    const size_t o = off;
    off += (bytes + 255) & ~static_cast<size_t>(255);
    return o;
  };
  s.pyr[0] = take(s.lv.total);
  s.pyr[1] = take(s.lv.total);
  s.deriv = take(s.lv.total * sizeof(short2));
  s.sob = take(hw * sizeof(short2));
  s.eig = take(hw * sizeof(float));
  s.state = take(hw);
  s.cand = take(hw * sizeof(int));
  s.acc = take(static_cast<size_t>(s.acc_cap) * sizeof(int));
  s.counters = take(kNumCounters * sizeof(unsigned));
  s.corners = take(kMaxCorners * sizeof(float2));
  s.ncorners = take(sizeof(int));
  s.total = off;
  return s;
}

// per-keyframe pointers of a derivative / corner batch: its pyramid, its arena (a Layout's derivatives, corner scratch
// and counters) and where its corners and their count go
struct KfBatch {
  const uint8_t* pyr[kMaxBatch];
  char* arena[kMaxBatch];
  float2* pts[kMaxBatch];
  int* count[kMaxBatch];
};

template <typename T>
__host__ __device__ __forceinline__ T* at(void* arena, size_t off) {
  return reinterpret_cast<T*>(static_cast<char*>(arena) + off);
}

__device__ __forceinline__ int refl101(int i, int n) {  // BORDER_REFLECT_101 for -n < i < 2n - 1
  i = abs(i);
  return i >= n ? 2 * (n - 1) - i : i;
}

// ---------------------------------------------------------------------------------------------------------------------
// pyramid
// ---------------------------------------------------------------------------------------------------------------------
// level 0 with its REFLECT_101 border; an fp32 gray in [0, 1] becomes (gray * 255).astype(uint8): one fp32 multiply,
// then truncation
// per-frame pointers of a pyramid batch: the source frame (level 0 only) and the padded pyramid it builds
struct FrameBatch {
  const void* src[kMaxBatch];
  uint8_t* pyr[kMaxBatch];
};

__global__ void __launch_bounds__(256)
level0_kernel(const __grid_constant__ FrameBatch b, int is_f32, int H, int W) {
  pdl_wait();
  pdl_launch_dependents();
  const void* frame = b.src[blockIdx.y];
  uint8_t* dst = b.pyr[blockIdx.y];
  const int pw = W + 2 * kPad, ph = H + 2 * kPad;
  const int idx = blockIdx.x * 256 + threadIdx.x;
  if (idx >= pw * ph) return;
  const int py = idx / pw, px = idx - py * pw;
  const long long src = static_cast<long long>(refl101(py - kPad, H)) * W + refl101(px - kPad, W);
  uint8_t v;
  if (is_f32) {
    v = static_cast<uint8_t>(__float2int_rz(__fmul_rn(static_cast<const float*>(frame)[src], 255.0f)));
  } else {
    v = static_cast<const uint8_t*>(frame)[src];
  }
  dst[idx] = v;
}

// pyrDown: 5x5 [1 4 6 4 1]^2 / 256 with rounding.  The source level's border already holds REFLECT_101 values, which is
// what pyrDown reads outside the level; the destination's own border is written by reflecting its coordinates.
__global__ void __launch_bounds__(256)
pyrdown_kernel(const __grid_constant__ FrameBatch b, long long src_ofs, int sw, long long dst_ofs, int dw, int dh) {
  pdl_wait();
  pdl_launch_dependents();
  const uint8_t* src = b.pyr[blockIdx.y] + src_ofs;
  uint8_t* dst = b.pyr[blockIdx.y] + dst_ofs;
  const int spw = sw + 2 * kPad;
  const int pw = dw + 2 * kPad, ph = dh + 2 * kPad;
  const int idx = blockIdx.x * 256 + threadIdx.x;
  if (idx >= pw * ph) return;
  const int py = idx / pw, px = idx - py * pw;
  const int y = refl101(py - kPad, dh), x = refl101(px - kPad, dw);
  const int k[5] = {1, 4, 6, 4, 1};
  const uint8_t* s = src + static_cast<long long>(2 * y - 2 + kPad) * spw + (2 * x - 2 + kPad);
  int tot = 0;
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    const uint8_t* r = s + i * spw;
    const int row = r[0] + 4 * r[1] + 6 * r[2] + 4 * r[3] + r[4];
    tot += k[i] * row;
  }
  dst[idx] = static_cast<uint8_t>((tot + 128) >> 8);
}

// calcSharrDeriv: int16 (dI/dx, dI/dy) with 3-10-3 smoothing (REFLECT_101: the level's border), zero outside the level
__global__ void __launch_bounds__(256)
scharr_kernel(const __grid_constant__ KfBatch b, size_t deriv_off, long long ofs, int w, int h) {
  pdl_wait();
  pdl_launch_dependents();
  const uint8_t* img = b.pyr[blockIdx.y] + ofs;
  short2* deriv = at<short2>(b.arena[blockIdx.y], deriv_off) + ofs;
  const int pw = w + 2 * kPad, ph = h + 2 * kPad;
  const int idx = blockIdx.x * 256 + threadIdx.x;
  if (idx >= pw * ph) return;
  const int py = idx / pw, px = idx - py * pw;
  const int y = py - kPad, x = px - kPad;
  if (y < 0 || y >= h || x < 0 || x >= w) {
    deriv[idx] = make_short2(0, 0);
    return;
  }
  const uint8_t* c = img + idx;
  const uint8_t *u = c - pw, *d = c + pw;
  const int t0l = (u[-1] + d[-1]) * 3 + c[-1] * 10, t0r = (u[1] + d[1]) * 3 + c[1] * 10;
  const int t1l = d[-1] - u[-1], t1c = d[0] - u[0], t1r = d[1] - u[1];
  deriv[idx] = make_short2(static_cast<short>(t0r - t0l), static_cast<short>((t1r + t1l) * 3 + t1c * 10));
}

// ---------------------------------------------------------------------------------------------------------------------
// Shi-Tomasi corners (goodFeaturesToTrack -> cornerMinEigenVal)
// ---------------------------------------------------------------------------------------------------------------------
// integer 3x3 Sobel (dx, dy) of level 0 (REFLECT_101)
// (also clears the keyframe's selection counters, which the following kernels accumulate into)
__global__ void __launch_bounds__(256)
sobel_kernel(const __grid_constant__ KfBatch b, const __grid_constant__ Layout s, int W, int H) {
  pdl_wait();
  pdl_launch_dependents();
  const uint8_t* img = b.pyr[blockIdx.y];
  short2* sob = at<short2>(b.arena[blockIdx.y], s.sob);
  if (blockIdx.x == 0 && threadIdx.x < kNumCounters) at<unsigned>(b.arena[blockIdx.y], s.counters)[threadIdx.x] = 0u;
  const int idx = blockIdx.x * 256 + threadIdx.x;
  if (idx >= W * H) return;
  const int y = idx / W, x = idx - y * W;
  const int pw = W + 2 * kPad;
  const uint8_t* c = img + static_cast<long long>(y + kPad) * pw + x + kPad;
  const uint8_t *u = c - pw, *d = c + pw;
  const int sx = (u[1] - u[-1]) + 2 * (c[1] - c[-1]) + (d[1] - d[-1]);
  const int sy = (d[-1] - u[-1]) + 2 * (d[0] - u[0]) + (d[1] - u[1]);
  sob[idx] = make_short2(static_cast<short>(sx), static_cast<short>(sy));
}

__device__ __forceinline__ unsigned float_order_key(float f) {  // monotonic float -> unsigned
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float float_from_order_key(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

// exact 7x7 box sums of dx^2, dx dy, dy^2 (REFLECT_101), scaled once: lambda_min = (a + c) - sqrt((a - c)^2 + b^2) with
// a = sum(dx^2)/2, b = sum(dx dy), c = sum(dy^2)/2; and the global maximum
__global__ void __launch_bounds__(256)
min_eigen_kernel(const __grid_constant__ KfBatch kb, const __grid_constant__ Layout s, int W, int H) {
  pdl_wait();
  pdl_launch_dependents();
  const short2* sob = at<const short2>(kb.arena[blockIdx.y], s.sob);
  float* eig = at<float>(kb.arena[blockIdx.y], s.eig);
  unsigned* counters = at<unsigned>(kb.arena[blockIdx.y], s.counters);
  const int idx = blockIdx.x * 256 + threadIdx.x;
  unsigned key = 0;
  if (idx < W * H) {
    const int y = idx / W, x = idx - y * W;
    int cx[7];
#pragma unroll
    for (int j = 0; j < 7; ++j) cx[j] = refl101(x + j - 3, W);
    int sxx = 0, sxy = 0, syy = 0;
    for (int i = 0; i < 7; ++i) {
      const short2* r = sob + static_cast<long long>(refl101(y + i - 3, H)) * W;
#pragma unroll
      for (int j = 0; j < 7; ++j) {
        const short2 v = r[cx[j]];
        sxx += v.x * v.x;
        sxy += v.x * v.y;
        syy += v.y * v.y;
      }
    }
    const float a = __fmul_rn(__fmul_rn(__int2float_rn(sxx), kEigScale2), 0.5f);
    const float b = __fmul_rn(__int2float_rn(sxy), kEigScale2);
    const float c = __fmul_rn(__fmul_rn(__int2float_rn(syy), kEigScale2), 0.5f);
    const float d = __fsub_rn(a, c);
    const float e = __fsub_rn(__fadd_rn(a, c), __fsqrt_rn(__fadd_rn(__fmul_rn(d, d), __fmul_rn(b, b))));
    eig[idx] = e;
    key = float_order_key(e);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) key = max(key, __shfl_xor_sync(0xffffffffu, key, o));
  if ((threadIdx.x & 31) == 0) atomicMax(&counters[kCntMax], key);
}

__device__ __forceinline__ float thresholded(float v, float thr) { return v > thr ? v : 0.0f; }

// threshold(eig, max * 0.01, TOZERO), then the candidates: non-zero, equal to their 3x3 dilation, not on the 1-pixel
// border.  state: 1 = candidate (undecided), 0 = not a candidate
__global__ void __launch_bounds__(256)
candidates_kernel(const __grid_constant__ KfBatch kb, const __grid_constant__ Layout s, int W, int H) {
  pdl_wait();
  pdl_launch_dependents();
  const float* eig = at<const float>(kb.arena[blockIdx.y], s.eig);
  uint8_t* state = at<uint8_t>(kb.arena[blockIdx.y], s.state);
  int* cand = at<int>(kb.arena[blockIdx.y], s.cand);
  unsigned* counters = at<unsigned>(kb.arena[blockIdx.y], s.counters);
  const int idx = blockIdx.x * 256 + threadIdx.x;
  if (idx >= W * H) return;
  const int y = idx / W, x = idx - y * W;
  const float thr = __double2float_rn(__dmul_rn(static_cast<double>(float_from_order_key(counters[kCntMax])), 0.01));
  bool is_cand = false;
  if (y > 0 && y < H - 1 && x > 0 && x < W - 1) {
    const float v = thresholded(eig[idx], thr);
    if (v != 0.0f) {
      float m = v;
#pragma unroll
      for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) m = fmaxf(m, thresholded(eig[idx + dy * W + dx], thr));
      is_cand = (v == m);
    }
  }
  state[idx] = is_cand ? 1 : 0;
  if (is_cand) cand[atomicAdd(&counters[kCntCand], 1u)] = idx;
}

__device__ __forceinline__ unsigned long long rank_key(const float* eig, int p) {
  // candidates are > 0, so the value's bits order like the value; ties go to the higher linear index (OpenCV's
  // greaterThanPtr compares addresses)
  return (static_cast<unsigned long long>(__float_as_uint(eig[p])) << 32) | static_cast<unsigned>(p);
}

// The sequential greedy selection (walk the candidates by rank, reject one closer than 8 px to an accepted corner) is
// the lexicographically-first independent set of the conflict graph, and a candidate's fate depends only on the
// higher-ranked candidates within its 15x15 neighbourhood.  So: accept a candidate with no undecided or accepted
// higher-ranked neighbour, reject one with an accepted higher-ranked neighbour, and repeat until nothing changes.  Every
// round decides at least the highest undecided candidate.  Updates are in place: a candidate only moves from undecided
// to final, and each rule reads final states only to conclude.  Then the accepted corners are listed.
// state: 1 undecided, 2 accepted, 3 rejected.  One CTA per keyframe.
__global__ void __launch_bounds__(kSelectThreads)
select_kernel(const __grid_constant__ KfBatch kb, const __grid_constant__ Layout s, int W, int H) {
  pdl_wait();
  pdl_launch_dependents();
  char* a = kb.arena[blockIdx.x];
  const float* eig = at<const float>(a, s.eig);
  volatile uint8_t* state = at<uint8_t>(a, s.state);
  const int* cand = at<const int>(a, s.cand);
  int* acc = at<int>(a, s.acc);
  unsigned* counters = at<unsigned>(a, s.counters);
  __shared__ int changed;
  const int n = static_cast<int>(counters[kCntCand]);
  for (;;) {
    if (threadIdx.x == 0) changed = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += kSelectThreads) {
      const int p = cand[i];
      if (state[p] != 1) continue;
      const unsigned long long key = rank_key(eig, p);
      const int y = p / W, x = p - y * W;
      bool blocked = false, rejected = false;
      for (int dy = -7; dy <= 7 && !rejected; ++dy) {
        const int yy = y + dy;
        if (yy < 0 || yy >= H) continue;
        for (int dx = -7; dx <= 7; ++dx) {
          const int xx = x + dx;
          if (dx * dx + dy * dy >= 64 || xx < 0 || xx >= W) continue;
          const int q = yy * W + xx;
          const uint8_t s = state[q];
          if (s == 1 || s == 2) {
            if (rank_key(eig, q) > key) {
              if (s == 2) {
                rejected = true;
                break;
              }
              blocked = true;
            }
          }
        }
      }
      if (rejected) {
        state[p] = 3;
        changed = 1;
      } else if (!blocked) {
        state[p] = 2;
        changed = 1;
      }
    }
    __syncthreads();
    const int c = changed;
    __syncthreads();
    if (!c) break;
  }
  for (int i = threadIdx.x; i < n; i += kSelectThreads) {
    const int p = cand[i];
    if (state[p] == 2) acc[atomicAdd(&counters[kCntAcc], 1u)] = p;
  }
}

// order the accepted corners by rank (a corner's position is the number of higher-ranked accepted corners) and keep the
// first 1000: the same as stopping the sequential walk at 1000
__global__ void __launch_bounds__(256)
rank_kernel(const __grid_constant__ KfBatch kb, const __grid_constant__ Layout s, int W) {
  pdl_wait();
  pdl_launch_dependents();
  const float* eig = at<const float>(kb.arena[blockIdx.y], s.eig);
  const int* acc = at<const int>(kb.arena[blockIdx.y], s.acc);
  const unsigned* counters = at<const unsigned>(kb.arena[blockIdx.y], s.counters);
  float2* pts = kb.pts[blockIdx.y];
  int* count = kb.count[blockIdx.y];
  __shared__ unsigned long long tile[256];
  const int n = static_cast<int>(counters[kCntAcc]);
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i == 0) *count = n < kMaxCorners ? n : kMaxCorners;
  if (static_cast<int>(blockIdx.x) * 256 >= n) return;
  const int p = i < n ? acc[i] : 0;
  const unsigned long long key = i < n ? rank_key(eig, p) : 0ull;
  int rank = 0;
  for (int t = 0; t < n; t += 256) {
    __syncthreads();
    tile[threadIdx.x] = t + static_cast<int>(threadIdx.x) < n ? rank_key(eig, acc[t + threadIdx.x]) : 0ull;
    __syncthreads();
    const int m = n - t < 256 ? n - t : 256;
    for (int j = 0; j < m; ++j) rank += tile[j] > key;
  }
  if (i < n && rank < kMaxCorners) {
    const int y = p / W;
    pts[rank] = make_float2(static_cast<float>(p - y * W), static_cast<float>(y));
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// pyramidal Lucas-Kanade (LKTrackerInvoker), one warp per point, coarse to fine
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void bilinear_weights(float a, float b, int* w) {
  // iw00..iw10 = cvRound(...) (half to even), iw11 = 2^14 - the others
  const float s = static_cast<float>(1 << kWBits);
  const float ia = __fsub_rn(1.0f, a), ib = __fsub_rn(1.0f, b);
  w[0] = __float2int_rn(__fmul_rn(__fmul_rn(ia, ib), s));
  w[1] = __float2int_rn(__fmul_rn(__fmul_rn(a, ib), s));
  w[2] = __float2int_rn(__fmul_rn(__fmul_rn(ia, b), s));
  w[3] = (1 << kWBits) - w[0] - w[1] - w[2];
}

__device__ __forceinline__ long long warp_sum_ll(long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// one LK item: the keyframe's pyramid I, derivatives dI, corners pts and device corner count n_dev (NULL: the kernel's
// n_host), the frame's pyramid J, and the item's output slots
struct LkItem {
  const uint8_t* I;
  const short2* dI;
  const uint8_t* J;
  const float2* pts;
  const int* n_dev;
  float2* next;
  uint8_t* status;
};
struct LkBatch {
  LkItem it[kMaxBatch];
};

__global__ void __launch_bounds__(128)
lk_kernel(const __grid_constant__ Levels lv, const __grid_constant__ LkBatch b, int n_host) {
  pdl_wait();
  pdl_launch_dependents();
  const LkItem& item = b.it[blockIdx.y];
  const uint8_t* __restrict__ I = item.I;
  const short2* __restrict__ dI = item.dI;
  const uint8_t* __restrict__ J = item.J;
  const float2* __restrict__ pts = item.pts;
  const int* n_dev = item.n_dev;
  const int lane = threadIdx.x & 31;
  const int pid = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int n = n_dev ? *n_dev : n_host;
  if (pid >= n) return;
  const float2 pt = pts[pid];
  int status = 1;
  float2 nxt = make_float2(0.0f, 0.0f);
  for (int L = lv.nlev - 1; L >= 0; --L) {
    const int w = lv.w[L], h = lv.h[L], pw = w + 2 * kPad;
    const long long base = lv.ofs[L] + static_cast<long long>(kPad) * pw + kPad;
    const uint8_t* Ib = I + base;
    const short2* dIb = dI + base;
    const uint8_t* Jb = J + base;
    const float sc = 1.0f / static_cast<float>(1 << L);
    const float px = __fmul_rn(pt.x, sc), py = __fmul_rn(pt.y, sc);
    if (L == lv.nlev - 1) {
      nxt = make_float2(px, py);
    } else {
      nxt = make_float2(__fmul_rn(nxt.x, 2.0f), __fmul_rn(nxt.y, 2.0f));
    }
    const float qx = __fsub_rn(px, 10.0f), qy = __fsub_rn(py, 10.0f);
    const int ipx = static_cast<int>(floorf(qx)), ipy = static_cast<int>(floorf(qy));
    if (ipx < -kWin || ipx >= w || ipy < -kWin || ipy >= h) {
      if (L == 0) status = 0;
      continue;
    }
    int iw[4];
    bilinear_weights(__fsub_rn(qx, static_cast<float>(ipx)), __fsub_rn(qy, static_cast<float>(ipy)), iw);
    int tI[kPerLane], tX[kPerLane], tY[kPerLane], wofs[kPerLane];
    long long s11 = 0, s12 = 0, s22 = 0;
#pragma unroll
    for (int i = 0; i < kPerLane; ++i) {
      const int k = lane + 32 * i;
      const int wy = k / kWin, wx = k - wy * kWin;
      wofs[i] = wy * pw + wx;
      tI[i] = tX[i] = tY[i] = 0;
      if (k < kWinPix) {
        const int off = (ipy + wy) * pw + ipx + wx;
        const uint8_t* s = Ib + off;
        tI[i] = (s[0] * iw[0] + s[1] * iw[1] + s[pw] * iw[2] + s[pw + 1] * iw[3] + (1 << (kWBits - 6))) >> (kWBits - 5);
        const short2* d = dIb + off;
        const short2 d00 = d[0], d01 = d[1], d10 = d[pw], d11 = d[pw + 1];
        tX[i] = (d00.x * iw[0] + d01.x * iw[1] + d10.x * iw[2] + d11.x * iw[3] + (1 << (kWBits - 1))) >> kWBits;
        tY[i] = (d00.y * iw[0] + d01.y * iw[1] + d10.y * iw[2] + d11.y * iw[3] + (1 << (kWBits - 1))) >> kWBits;
        s11 += tX[i] * tX[i];
        s12 += tX[i] * tY[i];
        s22 += tY[i] * tY[i];
      }
    }
    s11 = warp_sum_ll(s11);
    s12 = warp_sum_ll(s12);
    s22 = warp_sum_ll(s22);
    const float A11 = __fmul_rn(__ll2float_rn(s11), kLkScale), A12 = __fmul_rn(__ll2float_rn(s12), kLkScale),
                A22 = __fmul_rn(__ll2float_rn(s22), kLkScale);
    float D = __fsub_rn(__fmul_rn(A11, A22), __fmul_rn(A12, A12));
    const float dd = __fsub_rn(A11, A22);
    const float min_eig = __fdiv_rn(
        __fsub_rn(__fadd_rn(A22, A11), __fsqrt_rn(__fadd_rn(__fmul_rn(dd, dd), __fmul_rn(__fmul_rn(4.0f, A12), A12)))),
        static_cast<float>(2 * kWinPix));
    if (static_cast<double>(min_eig) < kMinEig || D < FLT_EPSILON) {
      if (L == 0) status = 0;
      continue;
    }
    D = __fdiv_rn(1.0f, D);
    float nx = __fsub_rn(nxt.x, 10.0f), ny = __fsub_rn(nxt.y, 10.0f);
    float pdx = 0.0f, pdy = 0.0f;
    for (int j = 0; j < kMaxIters; ++j) {
      const int inx = static_cast<int>(floorf(nx)), iny = static_cast<int>(floorf(ny));
      if (inx < -kWin || inx >= w || iny < -kWin || iny >= h) {
        if (L == 0) status = 0;
        break;
      }
      bilinear_weights(__fsub_rn(nx, static_cast<float>(inx)), __fsub_rn(ny, static_cast<float>(iny)), iw);
      const uint8_t* Jw = Jb + iny * pw + inx;
      long long b1 = 0, b2 = 0;
#pragma unroll
      for (int i = 0; i < kPerLane; ++i) {
        if (lane + 32 * i < kWinPix) {
          const uint8_t* s = Jw + wofs[i];
          const int diff =
              ((s[0] * iw[0] + s[1] * iw[1] + s[pw] * iw[2] + s[pw + 1] * iw[3] + (1 << (kWBits - 6))) >> (kWBits - 5)) -
              tI[i];
          b1 += diff * tX[i];
          b2 += diff * tY[i];
        }
      }
      b1 = warp_sum_ll(b1);
      b2 = warp_sum_ll(b2);
      const float fb1 = __fmul_rn(__ll2float_rn(b1), kLkScale), fb2 = __fmul_rn(__ll2float_rn(b2), kLkScale);
      const float dx = __fmul_rn(__fsub_rn(__fmul_rn(A12, fb2), __fmul_rn(A22, fb1)), D);
      const float dy = __fmul_rn(__fsub_rn(__fmul_rn(A12, fb1), __fmul_rn(A11, fb2)), D);
      nx = __fadd_rn(nx, dx);
      ny = __fadd_rn(ny, dy);
      nxt = make_float2(__fadd_rn(nx, 10.0f), __fadd_rn(ny, 10.0f));
      const double ddx = dx, ddy = dy;
      if (__dadd_rn(__dmul_rn(ddx, ddx), __dmul_rn(ddy, ddy)) <= kEps2) break;
      if (j > 0 && static_cast<double>(fabsf(__fadd_rn(dx, pdx))) < 0.01 &&
          static_cast<double>(fabsf(__fadd_rn(dy, pdy))) < 0.01) {
        nxt = make_float2(__fsub_rn(nxt.x, __fmul_rn(dx, 0.5f)), __fsub_rn(nxt.y, __fmul_rn(dy, 0.5f)));
        break;
      }
      pdx = dx;
      pdy = dy;
    }
  }
  if (lane == 0) {
    item.next[pid] = nxt;
    item.status[pid] = static_cast<uint8_t>(status);
  }
}

// keyframe corner count, tracked count, sum over tracked points of |dx| + |dy| (fp32 differences, fp64 sum in a fixed
// order) and the mean disparity sum / (2 count) of flow_tracker.py:50-51; one CTA per LK item, out[item]
__global__ void __launch_bounds__(256)
flow_stats_kernel(const __grid_constant__ LkBatch b, StaFlowStats* __restrict__ out_base) {
  pdl_wait();
  pdl_launch_dependents();
  const LkItem& item = b.it[blockIdx.x];
  const float2* __restrict__ kf = item.pts;
  const float2* __restrict__ nxt = item.next;
  const uint8_t* __restrict__ status = item.status;
  const int* __restrict__ n_dev = item.n_dev;
  StaFlowStats* out = out_base + blockIdx.x;
  __shared__ double ssum[256];
  __shared__ int scnt[256];
  const int n = *n_dev;
  double s = 0.0;
  int c = 0;
  for (int i = threadIdx.x; i < n; i += 256) {
    if (status[i]) {
      const float2 a = kf[i], b = nxt[i];
      s = __dadd_rn(s, static_cast<double>(fabsf(__fsub_rn(b.x, a.x))));
      s = __dadd_rn(s, static_cast<double>(fabsf(__fsub_rn(b.y, a.y))));
      ++c;
    }
  }
  ssum[threadIdx.x] = s;
  scnt[threadIdx.x] = c;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (static_cast<int>(threadIdx.x) < o) {
      ssum[threadIdx.x] = __dadd_rn(ssum[threadIdx.x], ssum[threadIdx.x + o]);
      scnt[threadIdx.x] += scnt[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    out->n_corners = n;
    out->n_tracked = scnt[0];
    out->abs_sum = ssum[0];
    out->mean_disparity = scnt[0] > 0 ? __ddiv_rn(ssum[0], 2.0 * scnt[0]) : 0.0;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// host-side sequences: each takes a batch of n >= 1 and launches it in chunks of kMaxBatch
// ---------------------------------------------------------------------------------------------------------------------
inline unsigned blocks_for(long long n, int per) { return static_cast<unsigned>((n + per - 1) / per); }

inline long long padded_elems(const Levels& lv, int l) {
  return static_cast<long long>(lv.w[l] + 2 * kPad) * (lv.h[l] + 2 * kPad);
}

// the pyramids of n frames of one size: src[i] ([H][W] uint8, or the fp32 gray when is_f32) -> padded pyramid pyr[i]
int build_pyramids(const Layout& s, int n, const void* const* src, int is_f32, uint8_t* const* pyr, cudaStream_t st) {
  const Levels& lv = s.lv;
  for (int c0 = 0; c0 < n; c0 += kMaxBatch) {
    const int m = n - c0 < kMaxBatch ? n - c0 : kMaxBatch;
    FrameBatch b = {};
    for (int i = 0; i < m; ++i) {
      b.src[i] = src[c0 + i];
      b.pyr[i] = pyr[c0 + i];
    }
    STA_CHECK_CUDA(launch_pdl(level0_kernel, dim3(blocks_for(padded_elems(lv, 0), 256), m), dim3(256), 0, st, 1, b, is_f32,
                              lv.h[0], lv.w[0]));
    for (int l = 1; l < lv.nlev; ++l)
      STA_CHECK_CUDA(launch_pdl(pyrdown_kernel, dim3(blocks_for(padded_elems(lv, l), 256), m), dim3(256), 0, st, 1, b,
                                lv.ofs[l - 1], lv.w[l - 1], lv.ofs[l], lv.w[l], lv.h[l]));
  }
  return 0;
}

// one keyframe of a derivative / corner batch: its pyramid, the arena (Layout) its scratch lives in, and where its
// corners [1000] and their count go
struct KfJob {
  const uint8_t* pyr;
  void* arena;
  float2* pts;
  int* count;
};

// for n keyframes: the Scharr derivatives of every level (derivs), then the corners of level 0 (corners)
int keyframe_products(const Layout& s, int n, const KfJob* jobs, bool derivs, bool corners, cudaStream_t st) {
  const Levels& lv = s.lv;
  const int W = lv.w[0], H = lv.h[0];
  const long long hw = static_cast<long long>(W) * H;
  for (int c0 = 0; c0 < n; c0 += kMaxBatch) {
    const int m = n - c0 < kMaxBatch ? n - c0 : kMaxBatch;
    KfBatch b = {};
    for (int i = 0; i < m; ++i) {
      b.pyr[i] = jobs[c0 + i].pyr;
      b.arena[i] = static_cast<char*>(jobs[c0 + i].arena);
      b.pts[i] = jobs[c0 + i].pts;
      b.count[i] = jobs[c0 + i].count;
    }
    if (derivs) {
      for (int l = 0; l < lv.nlev; ++l)
        STA_CHECK_CUDA(launch_pdl(scharr_kernel, dim3(blocks_for(padded_elems(lv, l), 256), m), dim3(256), 0, st, 1, b,
                                  s.deriv, lv.ofs[l], lv.w[l], lv.h[l]));
    }
    if (corners) {
      STA_CHECK_CUDA(launch_pdl(sobel_kernel, dim3(blocks_for(hw, 256), m), dim3(256), 0, st, 1, b, s, W, H));
      STA_CHECK_CUDA(launch_pdl(min_eigen_kernel, dim3(blocks_for(hw, 256), m), dim3(256), 0, st, 1, b, s, W, H));
      STA_CHECK_CUDA(launch_pdl(candidates_kernel, dim3(blocks_for(hw, 256), m), dim3(256), 0, st, 1, b, s, W, H));
      STA_CHECK_CUDA(launch_pdl(select_kernel, dim3(m), dim3(kSelectThreads), 0, st, 1, b, s, W, H));
      STA_CHECK_CUDA(launch_pdl(rank_kernel, dim3(blocks_for(s.acc_cap, 256), m), dim3(256), 0, st, 1, b, s, W));
    }
  }
  return 0;
}

// LK of n items (n_host points each where an item has no device count), then, if stats is not NULL, each item's
// statistics into stats[i]
int track_items(const Layout& s, int n, const LkItem* items, int n_host, StaFlowStats* stats, cudaStream_t st) {
  for (int c0 = 0; c0 < n; c0 += kMaxBatch) {
    const int m = n - c0 < kMaxBatch ? n - c0 : kMaxBatch;
    LkBatch b = {};
    for (int i = 0; i < m; ++i) b.it[i] = items[c0 + i];
    const int n_max = b.it[0].n_dev ? kMaxCorners : n_host;
    if (n_max > 0)
      STA_CHECK_CUDA(launch_pdl(lk_kernel, dim3(blocks_for(n_max, 4), m), dim3(128), 0, st, 1, s.lv, b, n_host));
    if (stats) STA_CHECK_CUDA(launch_pdl(flow_stats_kernel, dim3(m), dim3(256), 0, st, 1, b, stats + c0));
  }
  return 0;
}

bool size_ok(int H, int W) { return H >= kMinSide && W >= kMinSide && H <= kMaxSide && W <= kMaxSide; }

}  // namespace

}  // namespace sta

// ---------------------------------------------------------------------------------------------------------------------
// C ABI (include/sta_b200.h)
// ---------------------------------------------------------------------------------------------------------------------
using namespace sta;

struct StaFlowTracker {
  int H = 0, W = 0;
  Layout s;
  void* arena = nullptr;
  uint8_t* kf_pyr = nullptr;  // the keyframe's pyramid
  bool has_kf = false;        // a keyframe was set
  cudaStream_t last_stream = nullptr;
  bool has_stream = false;
  cudaEvent_t ev_switch = nullptr;
  // Frame pyramid slots: the arena's second pyramid, then more allocated when a group track first needs them, up to the
  // most frames this tracker had in one group.  Frame j of its last group track is in slots[j] (group_n frames).  A
  // promotion of frame j swaps slots[j] with kf_pyr, and the frames after it stay held in
  // slots[held_first, held_first + held_n) for the next group track to reuse.
  std::vector<uint8_t*> slots;
  std::vector<void*> slot_allocs;
  int group_n = 0, held_first = 0, held_n = 0;
  // when this tracker is the first of a group: LK output and statistics of every frame of the group, allocated at
  // creation for 16 frames (so a tracker used one frame at a time makes no cudaMalloc, which can stall other streams,
  // after sta_flow_create) and grown by larger groups
  int gcap = 0;
  void* gbuf = nullptr;  // [gcap][1000] float2 next points, [gcap][1000] uint8 status, [gcap] StaFlowStats
  StaFlowStats* gpinned = nullptr;
};

namespace {

#define FLOW_REQUIRE_SIZE(H, W)                                                                   \
  STA_REQUIRE(size_ok(H, W), "frame sides must be in [32, 2048]")

// one stream at a time: work enqueued on another stream waits for the previous one
int bind_stream(StaFlowTracker* t, cudaStream_t st) {
  if (t->has_stream && t->last_stream != st) {
    if (!t->ev_switch) STA_CHECK_CUDA(cudaEventCreateWithFlags(&t->ev_switch, cudaEventDisableTiming));
    STA_CHECK_CUDA(cudaEventRecord(t->ev_switch, t->last_stream));
    STA_CHECK_CUDA(cudaStreamWaitEvent(st, t->ev_switch, 0));
  }
  t->last_stream = st;
  t->has_stream = true;
  return 0;
}

KfJob kf_job(StaFlowTracker* t) {
  return KfJob{t->kf_pyr, t->arena, at<float2>(t->arena, t->s.corners), at<int>(t->arena, t->s.ncorners)};
}

LkItem lk_item(StaFlowTracker* t, const uint8_t* J, float2* next, uint8_t* status) {
  return LkItem{t->kf_pyr, at<const short2>(t->arena, t->s.deriv), J, at<const float2>(t->arena, t->s.corners),
                at<const int>(t->arena, t->s.ncorners), next, status};
}

size_t group_stats_offset(int cap) {
  return (static_cast<size_t>(cap) * kMaxCorners * (sizeof(float2) + 1) + 255) & ~static_cast<size_t>(255);
}

int ensure_group_buffers(StaFlowTracker* t, int F) {
  if (F <= t->gcap) return 0;
  const int cap = (F + 15) / 16 * 16;
  // the previous buffers' last use ended in the synchronisation of the group track that used them
  if (t->gbuf) cudaFree(t->gbuf);
  if (t->gpinned) cudaFreeHost(t->gpinned);
  t->gbuf = nullptr;
  t->gpinned = nullptr;
  t->gcap = 0;
  STA_CHECK_CUDA(cudaMalloc(&t->gbuf, group_stats_offset(cap) + cap * sizeof(StaFlowStats)));
  STA_CHECK_CUDA(cudaMallocHost(reinterpret_cast<void**>(&t->gpinned), cap * sizeof(StaFlowStats)));
  t->gcap = cap;
  return 0;
}

int ensure_slots(StaFlowTracker* t, int m) {
  const int have = static_cast<int>(t->slots.size());
  if (m <= have) return 0;
  const size_t bytes = (static_cast<size_t>(t->s.lv.total) + 255) & ~static_cast<size_t>(255);
  void* p = nullptr;
  STA_CHECK_CUDA(cudaMalloc(&p, bytes * (m - have)));
  t->slot_allocs.push_back(p);
  for (int i = 0; i < m - have; ++i) t->slots.push_back(static_cast<uint8_t*>(p) + bytes * i);
  return 0;
}

// the trackers of a group: non-null, of one frame size, and either one entry per tracker (distinct) or a tracker's
// frames consecutive.  Refusals only, no CUDA call.
int check_group(StaFlowTracker* const* ts, int F, bool distinct) {
  STA_REQUIRE(ts != nullptr && F >= 1, "empty group");
  for (int f = 0; f < F; ++f) {
    STA_REQUIRE(ts[f] != nullptr, "null tracker");
    STA_REQUIRE(ts[f]->H == ts[0]->H && ts[f]->W == ts[0]->W, "the trackers of a group must share one frame size");
    if (f > 0 && ts[f] == ts[f - 1]) {
      STA_REQUIRE(!distinct, "a tracker appears twice in the group");
      continue;
    }
    for (int g = 0; g < f; ++g)
      STA_REQUIRE(ts[g] != ts[f], distinct ? "a tracker appears twice in the group"
                                           : "a tracker's frames must be consecutive in the group");
  }
  return 0;
}

}  // namespace

extern "C" {

size_t sta_flow_scratch_bytes(int H, int W) { return size_ok(H, W) ? make_layout(H, W).total : 0; }

int sta_flow_create(int H, int W, StaFlowTracker** out) {
  STA_REQUIRE(out != nullptr, "null output pointer");
  *out = nullptr;
  FLOW_REQUIRE_SIZE(H, W);
  StaFlowTracker* t = new StaFlowTracker();
  t->H = H;
  t->W = W;
  t->s = make_layout(H, W);
  const cudaError_t e = cudaMalloc(&t->arena, t->s.total);
  if (e != cudaSuccess) {
    set_last_error(std::string("sta_flow_create: ") + cudaGetErrorString(e));
    sta_flow_destroy(t);
    return 1;
  }
  t->kf_pyr = at<uint8_t>(t->arena, t->s.pyr[0]);
  t->slots.push_back(at<uint8_t>(t->arena, t->s.pyr[1]));
  if (int rc = ensure_group_buffers(t, 1)) {
    sta_flow_destroy(t);
    return rc;
  }
  *out = t;
  return 0;
}

void sta_flow_destroy(StaFlowTracker* t) {
  if (!t) return;
  if (t->arena || t->gbuf || !t->slot_allocs.empty()) cudaDeviceSynchronize();
  if (t->arena) cudaFree(t->arena);
  for (void* p : t->slot_allocs) cudaFree(p);
  if (t->gbuf) cudaFree(t->gbuf);
  if (t->gpinned) cudaFreeHost(t->gpinned);
  if (t->ev_switch) cudaEventDestroy(t->ev_switch);
  delete t;
}

int sta_flow_set_keyframe_group(StaFlowTracker* const* ts, int n, const void* frames_dev, int frames_is_f32,
                                void* stream) {
  if (int rc = check_group(ts, n, true)) return rc;
  STA_REQUIRE(frames_dev != nullptr, "null frames");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const Layout& s = ts[0]->s;
  const size_t frame_bytes = static_cast<size_t>(ts[0]->H) * ts[0]->W * (frames_is_f32 ? sizeof(float) : 1);
  std::vector<const void*> src(n);
  std::vector<uint8_t*> dst(n);
  std::vector<KfJob> jobs(n);
  for (int i = 0; i < n; ++i) {
    if (int rc = bind_stream(ts[i], st)) return rc;
    src[i] = static_cast<const char*>(frames_dev) + frame_bytes * i;
    dst[i] = ts[i]->kf_pyr;
    jobs[i] = kf_job(ts[i]);
  }
  if (int rc = build_pyramids(s, n, src.data(), frames_is_f32, dst.data(), st)) return rc;
  if (int rc = keyframe_products(s, n, jobs.data(), true, true, st)) return rc;
  STA_CHECK_CUDA(cudaGetLastError());
  for (int i = 0; i < n; ++i) {
    ts[i]->has_kf = true;
    ts[i]->group_n = ts[i]->held_n = 0;
  }
  return 0;
}

int sta_flow_track_group(StaFlowTracker* const* ts, int F, const int* held_host, const void* frames_dev,
                         int frames_is_f32, StaFlowStats* stats_out, void* stream) {
  if (int rc = check_group(ts, F, false)) return rc;
  STA_REQUIRE(stats_out != nullptr, "null argument");
  // per frame: its index among its tracker's frames, and whether it is held
  std::vector<int> j_of(F);
  int n_new = 0;
  for (int f = 0; f < F; ++f) {
    StaFlowTracker* t = ts[f];
    STA_REQUIRE(t->has_kf, "no keyframe: call sta_flow_set_keyframe_group first");
    j_of[f] = (f > 0 && ts[f - 1] == t) ? j_of[f - 1] + 1 : 0;
    const bool held = held_host && held_host[f];
    if (held) {
      STA_REQUIRE(j_of[f] == 0 || held_host[f - 1], "a tracker's held frames must come first");
      STA_REQUIRE(j_of[f] < t->held_n, "more held frames than the tracker holds");
    } else {
      ++n_new;
    }
  }
  STA_REQUIRE(n_new == 0 || frames_dev != nullptr, "null frames");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const Layout& s = ts[0]->s;
  for (int f = 0; f < F; ++f) {
    StaFlowTracker* t = ts[f];
    if (j_of[f] != 0) continue;
    if (int rc = bind_stream(t, st)) return rc;
    int m = 1;
    while (f + m < F && ts[f + m] == t) ++m;
    // the held frames move to the front of the slots, in order
    const int k = held_host ? static_cast<int>(std::count(held_host + f, held_host + f + m, 1)) : 0;
    if (k > 0) std::rotate(t->slots.begin(), t->slots.begin() + t->held_first, t->slots.end());
    if (int rc = ensure_slots(t, m)) return rc;
  }
  if (int rc = ensure_group_buffers(ts[0], F)) return rc;
  float2* gnext = static_cast<float2*>(ts[0]->gbuf);
  uint8_t* gstatus = reinterpret_cast<uint8_t*>(gnext + static_cast<size_t>(ts[0]->gcap) * kMaxCorners);
  StaFlowStats* gstats = at<StaFlowStats>(ts[0]->gbuf, group_stats_offset(ts[0]->gcap));
  const size_t frame_bytes = static_cast<size_t>(s.lv.w[0]) * s.lv.h[0] * (frames_is_f32 ? sizeof(float) : 1);
  std::vector<const void*> src;
  std::vector<uint8_t*> dst;
  std::vector<LkItem> items(F);
  for (int f = 0; f < F; ++f) {
    StaFlowTracker* t = ts[f];
    uint8_t* J = t->slots[j_of[f]];
    if (!(held_host && held_host[f])) {
      src.push_back(static_cast<const char*>(frames_dev) + frame_bytes * src.size());
      dst.push_back(J);
    }
    items[f] = lk_item(t, J, gnext + static_cast<size_t>(f) * kMaxCorners, gstatus + static_cast<size_t>(f) * kMaxCorners);
  }
  for (int f = 0; f < F; ++f) {
    ts[f]->held_n = 0;
    ts[f]->group_n = j_of[f] + 1;
  }
  if (n_new > 0)
    if (int rc = build_pyramids(s, n_new, src.data(), frames_is_f32, dst.data(), st)) return rc;
  if (int rc = track_items(s, F, items.data(), 0, gstats, st)) return rc;
  STA_CHECK_CUDA(cudaMemcpyAsync(ts[0]->gpinned, gstats, F * sizeof(StaFlowStats), cudaMemcpyDeviceToHost, st));
  STA_CHECK_CUDA(cudaStreamSynchronize(st));
  for (int f = 0; f < F; ++f) stats_out[f] = ts[0]->gpinned[f];
  return 0;
}

int sta_flow_promote_group(StaFlowTracker* const* ts, int n, const int* frame_host, void* stream) {
  if (int rc = check_group(ts, n, true)) return rc;
  STA_REQUIRE(frame_host != nullptr, "null argument");
  for (int i = 0; i < n; ++i)
    STA_REQUIRE(frame_host[i] >= 0 && frame_host[i] < ts[i]->group_n, "no such frame in the tracker's last group track");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  std::vector<KfJob> jobs(n);
  for (int i = 0; i < n; ++i) {
    StaFlowTracker* t = ts[i];
    if (int rc = bind_stream(t, st)) return rc;
    const int j = frame_host[i];
    std::swap(t->kf_pyr, t->slots[j]);
    t->held_first = j + 1;
    t->held_n = t->group_n - j - 1;
    t->group_n = 0;
    jobs[i] = kf_job(t);
  }
  if (int rc = keyframe_products(ts[0]->s, n, jobs.data(), true, true, st)) return rc;
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int sta_flow_keyframe_points(StaFlowTracker* t, float* pts_out_dev, int* count_out_dev, void* stream) {
  STA_REQUIRE(t != nullptr && pts_out_dev != nullptr && count_out_dev != nullptr, "null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(t, st)) return rc;
  STA_CHECK_CUDA(cudaMemcpyAsync(pts_out_dev, at<float2>(t->arena, t->s.corners), kMaxCorners * sizeof(float2),
                                 cudaMemcpyDeviceToDevice, st));
  STA_CHECK_CUDA(cudaMemcpyAsync(count_out_dev, at<int>(t->arena, t->s.ncorners), sizeof(int), cudaMemcpyDeviceToDevice, st));
  return 0;
}

int sta_flow_keyframe_level0(StaFlowTracker* t, uint8_t* gray_out_dev, int16_t* deriv_out_dev, void* stream) {
  STA_REQUIRE(t != nullptr, "null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_stream(t, st)) return rc;
  const int pw = t->W + 2 * kPad;
  const size_t inner = static_cast<size_t>(kPad) * pw + kPad;
  if (gray_out_dev)
    STA_CHECK_CUDA(cudaMemcpy2DAsync(gray_out_dev, t->W, t->kf_pyr + inner, pw, t->W, t->H, cudaMemcpyDeviceToDevice, st));
  if (deriv_out_dev)
    STA_CHECK_CUDA(cudaMemcpy2DAsync(deriv_out_dev, t->W * sizeof(short2), at<short2>(t->arena, t->s.deriv) + inner,
                                     pw * sizeof(short2), t->W * sizeof(short2), t->H, cudaMemcpyDeviceToDevice, st));
  return 0;
}

int sta_op_good_features(const uint8_t* gray_u8, int H, int W, float* pts_out, int* count_out, void* scratch,
                         void* stream) {
  FLOW_REQUIRE_SIZE(H, W);
  STA_REQUIRE(gray_u8 && pts_out && count_out && scratch, "null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const Layout s = make_layout(H, W);
  uint8_t* pyr = at<uint8_t>(scratch, s.pyr[0]);
  const void* src = gray_u8;
  if (int rc = build_pyramids(s, 1, &src, 0, &pyr, st)) return rc;
  const KfJob job{pyr, scratch, reinterpret_cast<float2*>(pts_out), count_out};
  if (int rc = keyframe_products(s, 1, &job, false, true, st)) return rc;
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int sta_op_lk_track(const uint8_t* prev_u8, const uint8_t* next_u8, int H, int W, const float* pts, int n,
                    float* next_pts_out, uint8_t* status_out, void* scratch, void* stream) {
  FLOW_REQUIRE_SIZE(H, W);
  STA_REQUIRE(n >= 0, "negative point count");
  STA_REQUIRE(prev_u8 && next_u8 && scratch && (n == 0 || (pts && next_pts_out && status_out)), "null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const Layout s = make_layout(H, W);
  uint8_t* pyr[2] = {at<uint8_t>(scratch, s.pyr[0]), at<uint8_t>(scratch, s.pyr[1])};
  const void* src[2] = {prev_u8, next_u8};
  if (int rc = build_pyramids(s, 2, src, 0, pyr, st)) return rc;
  const KfJob job{pyr[0], scratch, nullptr, nullptr};
  if (int rc = keyframe_products(s, 1, &job, true, false, st)) return rc;
  const LkItem item{pyr[0], at<const short2>(scratch, s.deriv), pyr[1], reinterpret_cast<const float2*>(pts), nullptr,
                    reinterpret_cast<float2*>(next_pts_out), status_out};
  if (int rc = track_items(s, 1, &item, n, nullptr, st)) return rc;
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
