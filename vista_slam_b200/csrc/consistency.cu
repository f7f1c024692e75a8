// Multi-view depth consistency of a map (slam_utils.view_consistency_check, OnlineSLAM.view_consistency and the
// min_consistent_views filter of render / extract_mesh / save_data_all): for every pixel of view i, the number of views
// j in [i - 4, i + 4] (j != i, clipped to the sequence) whose depth, bilinearly sampled where the pixel's world point
// lands in j, agrees with the point's camera z in j within an absolute threshold.
//
// consistency_kernel: grid (ceil(H W / 256), n), one thread per pixel of view blockIdx.y.  The CTA first builds its
// view's K^-1 (cloud.cuh's fp64 adjugate) and pose and, per neighbour, the inverse pose (fp64 cofactors, rounded) and K
// in shared memory; each thread then unprojects its pixel with unproject_f32 and walks the neighbours in index order.
// Views are the slow grid dimension, so the CTAs resident at once read the same few neighbour depth maps from L2.
//
// The float32 steps after the projection follow the reference's (vista_slam/utils/slam_utils.py:346-419) with the CPU
// grid_sample of torch: u / w, the normalisation (u / (W - 1)) * 2 - 1, the unnormalisation (g + 1) * ((W - 1) / 2),
// bilinear weights from floor, zero padding, and the four corners summed as fma(se, fma(sw, fma(ne, nw * v_nw)))
// (the contraction the vectorised CPU kernel makes).  A coordinate that is NaN or infinite -- including one whose
// unnormalisation overflows -- gives NaN weights, so the sample is NaN and never agrees; a finite one outside the
// image samples 0.  z is the camera z clamped below at 1e-6 (NaN stays NaN); u / w divides by the unclamped third
// component.  No atomics: each thread writes its own count, so every call gives the same bits.
#include <math.h>
#include <stdint.h>

#include "../../include/sta_b200.h"
#include "cloud.cuh"
#include "host_util.h"

namespace sta {
namespace {

constexpr int kHalfWindow = 4;
constexpr int kMaxNeighbours = 2 * kHalfWindow;

// rows 0..2 of the inverse of the row-major 4x4 M, from fp64 cofactors, rounded to fp32 (torch.inverse of a pose)
__device__ __forceinline__ void inv4_rows3_f32(const float* M, float* out) {
  double m[16];
  for (int k = 0; k < 16; ++k) m[k] = M[k];
  // 2x2 minors of rows 0-1 (s) and rows 2-3 (c)
  const double s0 = m[0] * m[5] - m[4] * m[1], s1 = m[0] * m[6] - m[4] * m[2], s2 = m[0] * m[7] - m[4] * m[3];
  const double s3 = m[1] * m[6] - m[5] * m[2], s4 = m[1] * m[7] - m[5] * m[3], s5 = m[2] * m[7] - m[6] * m[3];
  const double c5 = m[10] * m[15] - m[14] * m[11], c4 = m[9] * m[15] - m[13] * m[11], c3 = m[9] * m[14] - m[13] * m[10];
  const double c2 = m[8] * m[15] - m[12] * m[11], c1 = m[8] * m[14] - m[12] * m[10], c0 = m[8] * m[13] - m[12] * m[9];
  const double det = s0 * c5 - s1 * c4 + s2 * c3 + s3 * c2 - s4 * c1 + s5 * c0;
  // inverse = adj / det; the adjugate's rows 0..2 (the fourth is not needed: cam_j keeps x, y, z)
  const double a[12] = {
      m[5] * c5 - m[6] * c4 + m[7] * c3,   -m[1] * c5 + m[2] * c4 - m[3] * c3,
      m[13] * s5 - m[14] * s4 + m[15] * s3, -m[9] * s5 + m[10] * s4 - m[11] * s3,
      -m[4] * c5 + m[6] * c2 - m[7] * c1,  m[0] * c5 - m[2] * c2 + m[3] * c1,
      -m[12] * s5 + m[14] * s2 - m[15] * s1, m[8] * s5 - m[10] * s2 + m[11] * s1,
      m[4] * c4 - m[5] * c2 + m[7] * c0,   -m[0] * c4 + m[1] * c2 - m[3] * c0,
      m[12] * s4 - m[13] * s2 + m[15] * s0, -m[8] * s4 + m[9] * s2 - m[11] * s0};
  for (int k = 0; k < 12; ++k) out[k] = static_cast<float>(a[k] / det);
}

struct ConsistencyArgs {
  const float *depth, *intri, *pose;
  int n, H, W;
  float thres;
  int32_t* count;
};

// depth at (row y, column x) of map d when the corner is inside the image, else 0 (grid_sample's zero padding); x and y
// are floor values, so the comparisons decide what the CPU kernel's int conversion and bounds masks decide
__device__ __forceinline__ float corner(const float* d, int H, int W, float x, float y) {
  if (!(x >= 0.f && x <= static_cast<float>(W - 1) && y >= 0.f && y <= static_cast<float>(H - 1))) return 0.f;
  return __ldg(d + static_cast<int>(y) * W + static_cast<int>(x));
}

// grid (ceil(H W / 256), n), 256 threads
__global__ void __launch_bounds__(256) consistency_kernel(const __grid_constant__ ConsistencyArgs a) {
  __shared__ float Ki[9], Ti[16], Tinv[kMaxNeighbours][12], Kj[kMaxNeighbours][9];
  __shared__ int nbr[kMaxNeighbours];
  const int i = blockIdx.y, H = a.H, W = a.W;
  const int lo = max(0, i - kHalfWindow), hi = min(a.n - 1, i + kHalfWindow);
  const int nn = hi - lo;  // neighbours: the window without i
  const int t = threadIdx.x;
  if (t < nn) {
    const int j = lo + t + (lo + t >= i ? 1 : 0);
    nbr[t] = j;
    inv4_rows3_f32(a.pose + static_cast<long long>(j) * 16, Tinv[t]);
  } else if (t >= 32 && t < 32 + kMaxNeighbours && t - 32 < nn) {
    const int j = lo + (t - 32) + (lo + (t - 32) >= i ? 1 : 0);
    for (int k = 0; k < 9; ++k) Kj[t - 32][k] = a.intri[static_cast<long long>(j) * 9 + k];
  } else if (t == 64) {
    inv3_f32(a.intri + static_cast<long long>(i) * 9, Ki);
  } else if (t >= 96 && t < 112) {
    Ti[t - 96] = a.pose[static_cast<long long>(i) * 16 + (t - 96)];
  }
  __syncthreads();
  const long long hw = static_cast<long long>(H) * W;
  const long long p = static_cast<long long>(blockIdx.x) * 256 + t;
  if (p >= hw) return;
  const int y = static_cast<int>(p / W), x = static_cast<int>(p - static_cast<long long>(y) * W);
  float wp[3];
  unproject_f32(Ki, Ti, static_cast<float>(x), static_cast<float>(y), __ldg(a.depth + i * hw + p), wp);
  const float wm1 = static_cast<float>(W - 1), hm1 = static_cast<float>(H - 1);
  const float sx = wm1 / 2.f, sy = hm1 / 2.f;
  int count = 0;
  for (int k = 0; k < nn; ++k) {
    const float* M = Tinv[k];
    const float* K = Kj[k];
    float c[3];
    for (int r = 0; r < 3; ++r) c[r] = M[r * 4] * wp[0] + M[r * 4 + 1] * wp[1] + M[r * 4 + 2] * wp[2] + M[r * 4 + 3];
    const float z = c[2] < 1e-6f ? 1e-6f : c[2];  // torch.clamp(min=1e-6): NaN stays NaN
    const float uu = K[0] * c[0] + K[1] * c[1] + K[2] * c[2], vv = K[3] * c[0] + K[4] * c[1] + K[5] * c[2],
                ww = K[6] * c[0] + K[7] * c[1] + K[8] * c[2];
    const float u = __fdiv_rn(uu, ww), v = __fdiv_rn(vv, ww);
    // normalise as the reference does, then unnormalise as grid_sample(align_corners=True) does
    const float gx = __fsub_rn(__fmul_rn(__fdiv_rn(u, wm1), 2.f), 1.f);
    const float gy = __fsub_rn(__fmul_rn(__fdiv_rn(v, hm1), 2.f), 1.f);
    const float px = __fmul_rn(__fadd_rn(gx, 1.f), sx), py = __fmul_rn(__fadd_rn(gy, 1.f), sy);
    const float xw = floorf(px), yn = floorf(py);
    const float fw = __fsub_rn(px, xw), fe = __fsub_rn(1.f, fw), fn = __fsub_rn(py, yn), fs = __fsub_rn(1.f, fn);
    const float* d = a.depth + nbr[k] * hw;
    const float vnw = corner(d, H, W, xw, yn), vne = corner(d, H, W, xw + 1.f, yn);
    const float vsw = corner(d, H, W, xw, yn + 1.f), vse = corner(d, H, W, xw + 1.f, yn + 1.f);
    float s = __fmul_rn(vnw, __fmul_rn(fs, fe));
    s = __fmaf_rn(vne, __fmul_rn(fs, fw), s);
    s = __fmaf_rn(vsw, __fmul_rn(fn, fe), s);
    s = __fmaf_rn(vse, __fmul_rn(fn, fw), s);
    count += (fabsf(__fsub_rn(s, z)) < a.thres && z > 0.f) ? 1 : 0;
  }
  a.count[i * hw + p] = count;
}

}  // namespace
}  // namespace sta

extern "C" {

int sta_view_consistency(const float* depth, const float* intri, const float* pose44, int n, int H, int W,
                         float threshold, int32_t* count_out, void* stream) {
  using namespace sta;
  STA_REQUIRE(n >= 1 && n <= 65535, "the view count must lie in [1, 65535]");
  STA_REQUIRE(H >= 2 && W >= 2, "H and W must be at least 2 (grid_sample divides by H - 1 and W - 1)");
  STA_REQUIRE(static_cast<long long>(n) * H * W < (1ll << 31), "n H W must be below 2^31");
  STA_REQUIRE(isfinite(threshold), "the threshold must be finite");
  STA_REQUIRE(depth && intri && pose44 && count_out, "null input or output");
  STA_REQUIRE(on_device(depth) && on_device(intri) && on_device(pose44) && on_device(count_out),
              "every array must be device memory");
  const long long hw = static_cast<long long>(H) * W;
  const ConsistencyArgs a{depth, intri, pose44, n, H, W, threshold, count_out};
  consistency_kernel<<<dim3(static_cast<unsigned>((hw + 255) / 256), n), 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
