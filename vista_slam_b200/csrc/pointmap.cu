// Pointmap consumers that follow the STA heads in OnlineSLAM (SURVEY.md section 8(f), rank 2): bandwidth-bound
// reductions over the fp32 pointmaps / confidences the DPT head has just written.
//
//   estimate_intrinsic_from_pts3d            vista_slam/utils/slam_utils.py:8-79   (called at slam.py:184)
//   depths = pcls[..., 2]                    vista_slam/slam.py:185
//   conf.mean()                              vista_slam/pose_graph.py:41
//   estimate_scale_with_depth_and_confidence vista_slam/utils/slam_utils.py:168-190 (called at slam.py:224)
//   (ci * cj).sqrt().mean()                  vista_slam/slam.py:227
//
// One pass over the data: per-thread fp32 partial sums -> warp shuffles -> one fp64 record per block; a second
// tiny kernel combines the records in a fixed order in fp64 (deterministic, no atomics) and writes K / scale.
// The scale reduction lives in pointmap.cuh, which the device pose graph (slam_graph.cu) shares.
// 16 bytes read + 4 bytes written per pixel: the kernel is HBM-bound (100 MB at cfg-2, ~16 us).
#include "common.cuh"
#include "host_util.h"
#include "ops.h"
#include "pointmap.cuh"

namespace sta {

namespace {

// grid (kStatBlocks, V), 256 threads
__global__ void __launch_bounds__(256)
pointmap_stats_kernel(const float* __restrict__ pts3d, const float* __restrict__ conf, int H, int W,
                      float* __restrict__ depth_out, double* __restrict__ partial) {
  pdl_wait();
  pdl_launch_dependents();
  const int v = blockIdx.y;
  const int px = H * W;
  const float cx = W * 0.5f, cy = H * 0.5f;
  const float* pv = pts3d + static_cast<long long>(v) * px * 3;
  const float* cv = conf + static_cast<long long>(v) * px;
  float s[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
  for (int i = blockIdx.x * 256 + threadIdx.x; i < px; i += kStatBlocks * 256) {
    const float X = pv[3 * i], Y = pv[3 * i + 1], Z = pv[3 * i + 2];
    const float c = cv[i];
    if (depth_out) depth_out[static_cast<long long>(v) * px + i] = Z;
    const int row = i / W, col = i - row * W;
    const float u = static_cast<float>(col) - cx, vv = static_cast<float>(row) - cy;
    const float w = fmaxf(c, 1e-6f);  // torch.clamp(confidence, min=1e-6)
    float xz = X / Z, yz = Y / Z;     // IEEE division: x/0 = inf, 0/0 = nan -> nan_to_num(..., 0, 0, 0)
    if (!isfinite(xz)) xz = 0.f;
    if (!isfinite(yz)) yz = 0.f;
    s[0] += w * xz * u;
    s[1] += w * xz * xz;
    s[2] += w * yz * vv;
    s[3] += w * yz * yz;
    s[4] += c;
  }
  block_reduce_store<5>(s, partial + (static_cast<long long>(v) * kStatBlocks + blockIdx.x) * kStatVals);
}

// one block of 32 threads; shared == 0: one K per view, 1: one K for all views, 2: one K per edge e < V/2 from
// its two views (e, e + V/2) -- the [ij ; ji] concatenation of slam.py:181-184 for a batch of edges
__global__ void pointmap_finalize_kernel(const double* __restrict__ partial, int V, int H, int W, int shared,
                                         float* __restrict__ K_out, float* __restrict__ conf_mean_out) {
  pdl_wait();
  pdl_launch_dependents();
  const float cx = W * 0.5f, cy = H * 0.5f;
  double tot[4] = {0.0, 0.0, 0.0, 0.0};
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    double t[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (int b = 0; b < kStatBlocks; ++b)
      for (int i = 0; i < 5; ++i) t[i] += partial[(static_cast<long long>(v) * kStatBlocks + b) * kStatVals + i];
    if (conf_mean_out) conf_mean_out[v] = static_cast<float>(t[4] / (static_cast<double>(H) * W));
    if (shared == 2 && v < V / 2) {
      double u[4];
      for (int i = 0; i < 4; ++i) {
        double t2 = 0.0;
        for (int b = 0; b < kStatBlocks; ++b) t2 += partial[(static_cast<long long>(v + V / 2) * kStatBlocks + b) * kStatVals + i];
        u[i] = t[i] + t2;
      }
      float* K = K_out + v * 9;
      K[0] = static_cast<float>(u[0] / u[1]); K[1] = 0.f; K[2] = cx;
      K[3] = 0.f; K[4] = static_cast<float>(u[2] / u[3]); K[5] = cy;
      K[6] = 0.f; K[7] = 0.f; K[8] = 1.f;
    }
    if (!shared) {
      float* K = K_out + v * 9;
      K[0] = static_cast<float>(t[0] / t[1]); K[1] = 0.f; K[2] = cx;
      K[3] = 0.f; K[4] = static_cast<float>(t[2] / t[3]); K[5] = cy;
      K[6] = 0.f; K[7] = 0.f; K[8] = 1.f;
    }
  }
  if (shared == 1 && threadIdx.x == 0) {
    for (int v = 0; v < V; ++v) {  // fixed order
      for (int i = 0; i < 4; ++i) {
        double t = 0.0;
        for (int b = 0; b < kStatBlocks; ++b) t += partial[(static_cast<long long>(v) * kStatBlocks + b) * kStatVals + i];
        tot[i] += t;
      }
    }
    K_out[0] = static_cast<float>(tot[0] / tot[1]); K_out[1] = 0.f; K_out[2] = cx;
    K_out[3] = 0.f; K_out[4] = static_cast<float>(tot[2] / tot[3]); K_out[5] = cy;
    K_out[6] = 0.f; K_out[7] = 0.f; K_out[8] = 1.f;
  }
}

// grid (kStatBlocks), 256 threads
__global__ void __launch_bounds__(256)
scale_stats_kernel(const float* __restrict__ Di, const float* __restrict__ Dj, const float* __restrict__ ci,
                   const float* __restrict__ cj, long long n, double* __restrict__ partial) {
  pdl_wait();
  pdl_launch_dependents();
  scale_partial(Di, Dj, ci, cj, n, blockIdx.x, partial + static_cast<long long>(blockIdx.x) * kStatVals);
}

__global__ void scale_finalize_kernel(const double* __restrict__ partial, long long n, float* __restrict__ out2) {
  pdl_wait();
  pdl_launch_dependents();
  if (threadIdx.x != 0) return;
  scale_finalize(partial, n, out2);
}

}  // namespace

size_t pointmap_scratch_bytes(int V) {
  return static_cast<size_t>(V > 1 ? V : 1) * kStatBlocks * kStatVals * sizeof(double);
}

int launch_pointmap_consumers(const float* pts3d, const float* conf, int V, int H, int W, int shared, float* K_out,
                              float* depth_out, float* conf_mean_out, void* scratch, cudaStream_t stream) {
  STA_REQUIRE(pts3d && conf && K_out && scratch, "null pointer");
  STA_REQUIRE(V > 0 && V <= 65535 && H > 0 && W > 0 && static_cast<long long>(H) * W < (1ll << 30), "bad shape");
  STA_REQUIRE(shared >= 0 && shared <= 2 && (shared != 2 || V % 2 == 0), "shared: 0 per view, 1 all views, 2 per edge (V even)");
  STA_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 7) == 0, "scratch must be 8-byte aligned");
  double* partial = static_cast<double*>(scratch);
  STA_CHECK_CUDA(launch_pdl(pointmap_stats_kernel, dim3(kStatBlocks, V), dim3(256), 0, stream, 1, pts3d, conf, H, W,
                            depth_out, partial));
  STA_CHECK_CUDA(launch_pdl(pointmap_finalize_kernel, dim3(1), dim3(32), 0, stream, 1,
                            static_cast<const double*>(partial), V, H, W, shared, K_out, conf_mean_out));
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_depth_scale(const float* Di, const float* Dj, const float* ci, const float* cj, long long n, float* out2,
                       void* scratch, cudaStream_t stream) {
  STA_REQUIRE(Di && Dj && ci && cj && out2 && scratch, "null pointer");
  STA_REQUIRE(n > 0, "empty depth maps");
  STA_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 7) == 0, "scratch must be 8-byte aligned");
  double* partial = static_cast<double*>(scratch);
  STA_CHECK_CUDA(launch_pdl(scale_stats_kernel, dim3(kStatBlocks), dim3(256), 0, stream, 1, Di, Dj, ci, cj, n, partial));
  STA_CHECK_CUDA(launch_pdl(scale_finalize_kernel, dim3(1), dim3(32), 0, stream, 1, static_cast<const double*>(partial), n,
                            out2));
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace sta
