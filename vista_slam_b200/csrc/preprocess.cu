// SLAM image preprocessing on the device (SURVEY.md section 8(f), rank 3): what
// SLAM_image_only.process_image (vista_slam/datasets/slam_images_only.py:22-34) does on the host with PIL per frame --
// centred crop with edge margins, high-quality Lanczos down-scaling, centre crop to the network resolution
// (datasets/base/base_view_graph_dataset.py:171-225, utils/cropping.py:54-84,102-118), ToTensor + Normalize(0.5, 0.5)
// (utils/image.py:13) and ToTensor + Grayscale (slam_images_only.py:20).
//
// Bit-exact with PIL's 8-bit resampler (Pillow src/libImaging/Resample.c): the per-output-pixel coefficient windows are
// computed on the host in double precision exactly as precompute_coeffs / normalize_coeffs_8bpc do (22-bit fixed
// point), the two passes (horizontal, then vertical) accumulate in int32 and round through clip8, and the float
// outputs are single correctly-rounded fp32 operations (no FMA contraction).  Byte work: HBM / latency bound; a
// 640x480 frame is 0.9 MB in, 0.8 MB out.
#include "common.cuh"
#include "host_util.h"
#include "ops.h"

#include <math.h>

#include <map>
#include <mutex>
#include <tuple>
#include <vector>

namespace sta {

namespace {

constexpr int kPrecisionBits = 32 - 8 - 2;

struct Geometry {
  int l, t, W1, H1;  // crop window of the source frame
  int rw, rh;        // size after the Lanczos resize
  int l2, t2;        // final centre crop offset
  int ow, oh;        // network resolution (possibly transposed for portrait frames)
};

// base_view_graph_dataset.py:181-223 (aug_crop <= 1).  Returns 0 on success.
int make_geometry(int H, int W, int res_w, int res_h, int w_edge, int h_edge, Geometry* g) {
  const int cx = W / 2, cy = H / 2;
  const int mx = cx < W - cx ? cx : W - cx, my = cy < H - cy ? cy : H - cy;
  STA_REQUIRE(static_cast<double>(mx) > W / 5.0 && static_cast<double>(my) > H / 5.0, "bad principal point");
  int l = cx - mx, t = cy - my, r = cx + mx, b = cy + my;
  l = l > w_edge ? l : w_edge;
  t = t > h_edge ? t : h_edge;
  r = r < W - w_edge ? r : W - w_edge;
  b = b < H - h_edge ? b : H - h_edge;
  STA_REQUIRE(r > l && b > t, "edge margins leave no image");
  g->l = l; g->t = t; g->W1 = r - l; g->H1 = b - t;
  STA_REQUIRE(res_w >= res_h, "resolution must be (width >= height)");
  int ow = res_w, oh = res_h;
  const double ratio = static_cast<double>(g->H1) / g->W1;
  if (g->H1 > 1.1 * g->W1) {
    ow = res_h; oh = res_w;  // portrait frame
  } else if (0.9 < ratio && ratio < 1.1 && res_w != res_h) {
    set_last_error("square frame with a non-square resolution: the reference picks the orientation at random");
    return 2;
  }
  const double sx = static_cast<double>(ow) / g->W1, sy = static_cast<double>(oh) / g->H1;
  const double scale_final = (sx > sy ? sx : sy) + 1e-8;             // cropping.py:68
  g->rw = static_cast<int>(floor(g->W1 * scale_final));              // cropping.py:69
  g->rh = static_cast<int>(floor(g->H1 * scale_final));
  g->l2 = static_cast<int>(nearbyint(g->rw / 2.0 - ow / 2.0));       // np.round: half to even
  g->t2 = static_cast<int>(nearbyint(g->rh / 2.0 - oh / 2.0));
  g->ow = ow; g->oh = oh;
  STA_REQUIRE(g->l2 >= 0 && g->t2 >= 0 && g->l2 + ow <= g->rw && g->t2 + oh <= g->rh, "internal: final crop outside");
  return 0;
}

double lanczos(double x) {
  if (-3.0 <= x && x < 3.0) {
    auto sinc = [](double v) {
      if (v == 0.0) return 1.0;
      v = v * M_PI;
      return sin(v) / v;
    };
    return sinc(x) * sinc(x / 3);
  }
  return 0.0;
}

// Resample.c precompute_coeffs (box = whole axis) + normalize_coeffs_8bpc
void precompute_coeffs(int in_size, int out_size, int* ksize_out, std::vector<int>* bounds, std::vector<int>* kk) {
  const float in0 = 0.0f, in1 = static_cast<float>(in_size);
  const double scale = static_cast<double>(in1 - in0) / out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = 3.0 * filterscale;
  const int ksize = static_cast<int>(ceil(support)) * 2 + 1;
  bounds->assign(static_cast<size_t>(out_size) * 2, 0);
  kk->assign(static_cast<size_t>(out_size) * ksize, 0);
  std::vector<double> w(ksize);
  const double ss = 1.0 / filterscale;
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = in0 + (xx + 0.5) * scale;
    int xmin = static_cast<int>(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = static_cast<int>(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      w[x] = lanczos((x + xmin - center + 0.5) * ss);
      ww += w[x];
    }
    for (int x = 0; x < xmax; ++x) {
      const double k = (ww != 0.0) ? w[x] / ww : w[x];
      (*kk)[static_cast<size_t>(xx) * ksize + x] =
          (k < 0) ? static_cast<int>(-0.5 + k * (1 << kPrecisionBits)) : static_cast<int>(0.5 + k * (1 << kPrecisionBits));
    }
    (*bounds)[2 * xx] = xmin;
    (*bounds)[2 * xx + 1] = xmax;
  }
  *ksize_out = ksize;
}

__device__ __forceinline__ int clip8(int v) {
  v >>= kPrecisionBits;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// horizontal pass: src frame rows [t, t + H1), columns [l, l + W1)  ->  tmp [H1][rw][3] uint8; frame blockIdx.y of
// [F][src_h][src_w][3] into tmp [F][H1][rw][3]
__global__ void __launch_bounds__(256)
resample_h_kernel(const uint8_t* __restrict__ src, int src_h, int src_w, int l, int t, int H1, int rw, int ksize,
                  const int* __restrict__ bounds, const int* __restrict__ kk, uint8_t* __restrict__ tmp) {
  pdl_wait();
  pdl_launch_dependents();
  src += static_cast<long long>(blockIdx.y) * src_h * src_w * 3;
  tmp += static_cast<long long>(blockIdx.y) * H1 * rw * 3;
  const int idx = blockIdx.x * 256 + threadIdx.x;
  if (idx >= H1 * rw) return;
  const int y = idx / rw, xx = idx - y * rw;
  const int xmin = bounds[2 * xx], xmax = bounds[2 * xx + 1];
  const int* k = kk + static_cast<long long>(xx) * ksize;
  const uint8_t* p = src + (static_cast<long long>(t + y) * src_w + l + xmin) * 3;
  int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
  for (int x = 0; x < xmax; ++x) {
    const int kv = k[x];
    s0 += p[3 * x] * kv;
    s1 += p[3 * x + 1] * kv;
    s2 += p[3 * x + 2] * kv;
  }
  uint8_t* o = tmp + static_cast<long long>(idx) * 3;
  o[0] = static_cast<uint8_t>(clip8(s0));
  o[1] = static_cast<uint8_t>(clip8(s1));
  o[2] = static_cast<uint8_t>(clip8(s2));
}

// vertical pass restricted to the final crop + ToTensor / Normalize / Grayscale:
// tmp [H1][rw][3] -> rgb [3][oh][ow] fp32 in [-1, 1], gray [oh][ow] fp32 in [0, 1], u8 [oh][ow][3] (optional);
// frame blockIdx.y of [F] of each
__global__ void __launch_bounds__(256)
resample_v_finish_kernel(const uint8_t* __restrict__ tmp, int H1, int rw, int l2, int t2, int ow, int oh, int ksize,
                         const int* __restrict__ bounds, const int* __restrict__ kk, int vertical_identity,
                         float* __restrict__ rgb, float* __restrict__ gray, uint8_t* __restrict__ u8) {
  pdl_wait();
  pdl_launch_dependents();
  const long long plane = static_cast<long long>(ow) * oh, f = blockIdx.y;
  tmp += f * H1 * rw * 3;
  rgb += f * 3 * plane;
  if (gray) gray += f * plane;
  if (u8) u8 += f * plane * 3;
  const int idx = blockIdx.x * 256 + threadIdx.x;
  if (idx >= ow * oh) return;
  const int py = idx / ow, px = idx - py * ow;
  const int yy = py + t2, xx = px + l2;
  int c0, c1, c2;
  if (vertical_identity) {  // PIL skips a pass whose size does not change
    const uint8_t* p = tmp + (static_cast<long long>(yy) * rw + xx) * 3;
    c0 = p[0]; c1 = p[1]; c2 = p[2];
  } else {
    const int ymin = bounds[2 * yy], ymax = bounds[2 * yy + 1];
    const int* k = kk + static_cast<long long>(yy) * ksize;
    const uint8_t* p = tmp + (static_cast<long long>(ymin) * rw + xx) * 3;
    int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
    for (int y = 0; y < ymax; ++y) {
      const int kv = k[y];
      const uint8_t* q = p + static_cast<long long>(y) * rw * 3;
      s0 += q[0] * kv;
      s1 += q[1] * kv;
      s2 += q[2] * kv;
    }
    c0 = clip8(s0); c1 = clip8(s1); c2 = clip8(s2);
  }
  // ToTensor: uint8 / 255 (IEEE division); Normalize: (x - 0.5) / 0.5; Grayscale: 0.2989 r + 0.587 g + 0.114 b,
  // every operation rounded separately as the elementwise torch kernels do
  const float f0 = __fdiv_rn(static_cast<float>(c0), 255.0f), f1 = __fdiv_rn(static_cast<float>(c1), 255.0f),
              f2 = __fdiv_rn(static_cast<float>(c2), 255.0f);
  rgb[idx] = __fdiv_rn(__fsub_rn(f0, 0.5f), 0.5f);
  rgb[plane + idx] = __fdiv_rn(__fsub_rn(f1, 0.5f), 0.5f);
  rgb[2 * plane + idx] = __fdiv_rn(__fsub_rn(f2, 0.5f), 0.5f);
  if (gray) gray[idx] = __fadd_rn(__fadd_rn(__fmul_rn(0.2989f, f0), __fmul_rn(0.587f, f1)), __fmul_rn(0.114f, f2));
  if (u8) {
    u8[3 * idx] = static_cast<uint8_t>(c0);
    u8[3 * idx + 1] = static_cast<uint8_t>(c1);
    u8[3 * idx + 2] = static_cast<uint8_t>(c2);
  }
}

// per (device, frame geometry): coefficient tables and the intermediate images of up to tmp_frames frames; SLAM
// streams have one frame size
struct Plan {
  Geometry g;
  int ksize_h = 0, ksize_v = 0;
  int *d_bh = nullptr, *d_kh = nullptr, *d_bv = nullptr, *d_kv = nullptr;
  uint8_t* d_tmp = nullptr;
  int tmp_frames = 0;
};
typedef std::tuple<int, int, int, int, int, int, int> PlanKey;

int get_plan(int H, int W, int res_w, int res_h, int w_edge, int h_edge, Plan** out) {
  static std::mutex mu;
  static std::map<PlanKey, Plan> plans;
  int dev = 0;
  STA_CHECK_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  const PlanKey key(dev, H, W, res_w, res_h, w_edge, h_edge);
  auto it = plans.find(key);
  if (it != plans.end()) {
    *out = &it->second;
    return 0;
  }
  if (plans.size() >= 64) {
    set_last_error("too many distinct frame geometries (64) for the preprocessing plan cache");
    return 2;
  }
  Plan p;
  if (int rc = make_geometry(H, W, res_w, res_h, w_edge, h_edge, &p.g)) return rc;
  std::vector<int> bh, kh, bv, kv;
  precompute_coeffs(p.g.W1, p.g.rw, &p.ksize_h, &bh, &kh);
  precompute_coeffs(p.g.H1, p.g.rh, &p.ksize_v, &bv, &kv);
  auto upload = [](const std::vector<int>& v, int** d) -> int {
    STA_CHECK_CUDA(cudaMalloc(d, v.size() * sizeof(int)));
    STA_CHECK_CUDA(cudaMemcpy(*d, v.data(), v.size() * sizeof(int), cudaMemcpyHostToDevice));
    return 0;
  };
  if (upload(bh, &p.d_bh) || upload(kh, &p.d_kh) || upload(bv, &p.d_bv) || upload(kv, &p.d_kv)) return 1;
  STA_CHECK_CUDA(cudaMalloc(&p.d_tmp, static_cast<size_t>(p.g.H1) * p.g.rw * 3));
  p.tmp_frames = 1;
  *out = &plans.emplace(key, p).first->second;
  return 0;
}

// room for F intermediate images; the old buffer's last use is on `stream` (a geometry is used on one stream at a time)
int grow_tmp(Plan* p, int F, cudaStream_t stream) {
  if (F <= p->tmp_frames) return 0;
  STA_CHECK_CUDA(cudaStreamSynchronize(stream));
  STA_CHECK_CUDA(cudaFree(p->d_tmp));
  p->d_tmp = nullptr;
  p->tmp_frames = 0;
  STA_CHECK_CUDA(cudaMalloc(&p->d_tmp, static_cast<size_t>(F) * p->g.H1 * p->g.rw * 3));
  p->tmp_frames = F;
  return 0;
}

}  // namespace

// host-only test hooks (no GPU work): the geometry and the PIL coefficient windows the kernels are driven by
int preprocess_geometry(int H, int W, int res_w, int res_h, int w_edge, int h_edge, int* out10) {
  Geometry g;
  if (int rc = make_geometry(H, W, res_w, res_h, w_edge, h_edge, &g)) return rc;
  const int v[10] = {g.l, g.t, g.l + g.W1, g.t + g.H1, g.rw, g.rh, g.l2, g.t2, g.ow, g.oh};
  for (int i = 0; i < 10; ++i) out10[i] = v[i];
  return 0;
}
int preprocess_coeffs(int in_size, int out_size, int* ksize_out, int* bounds_out, int* kk_out, long long kk_capacity) {
  STA_REQUIRE(in_size > 0 && out_size > 0 && ksize_out && bounds_out && kk_out, "bad arguments");
  int ksize = 0;
  std::vector<int> b, k;
  precompute_coeffs(in_size, out_size, &ksize, &b, &k);
  STA_REQUIRE(static_cast<long long>(k.size()) <= kk_capacity, "coefficient buffer too small");
  *ksize_out = ksize;
  for (size_t i = 0; i < b.size(); ++i) bounds_out[i] = b[i];
  for (size_t i = 0; i < k.size(); ++i) kk_out[i] = k[i];
  return 0;
}

int launch_preprocess_rgb8(const uint8_t* rgb_dev, int F, int H, int W, int res_w, int res_h, int w_edge, int h_edge,
                           float* rgb_out, float* gray_out, uint8_t* u8_out, int* out_hw_host, int query_only,
                           cudaStream_t stream) {
  STA_REQUIRE(H > 0 && W > 0 && res_w > 0 && res_h > 0 && w_edge >= 0 && h_edge >= 0, "bad arguments");
  STA_REQUIRE(F >= 1 && F <= 65535, "frame count must be in [1, 65535]");
  if (query_only) {
    Geometry g;
    if (int rc = make_geometry(H, W, res_w, res_h, w_edge, h_edge, &g)) return rc;
    if (out_hw_host) { out_hw_host[0] = g.oh; out_hw_host[1] = g.ow; }
    return 0;
  }
  STA_REQUIRE(rgb_dev && rgb_out, "null pointer");
  Plan* p = nullptr;
  if (int rc = get_plan(H, W, res_w, res_h, w_edge, h_edge, &p)) return rc;
  if (int rc = grow_tmp(p, F, stream)) return rc;
  const Geometry& g = p->g;
  if (out_hw_host) { out_hw_host[0] = g.oh; out_hw_host[1] = g.ow; }
  // horizontal pass (an identity pass still copies the crop window: same code, the coefficients are then 1 << 22)
  const int n1 = g.H1 * g.rw;
  STA_CHECK_CUDA(launch_pdl(resample_h_kernel, dim3((n1 + 255) / 256, F), dim3(256), 0, stream, 1, rgb_dev, H, W, g.l, g.t,
                            g.H1, g.rw, p->ksize_h, static_cast<const int*>(p->d_bh), static_cast<const int*>(p->d_kh),
                            p->d_tmp));
  const int n2 = g.ow * g.oh;
  STA_CHECK_CUDA(launch_pdl(resample_v_finish_kernel, dim3((n2 + 255) / 256, F), dim3(256), 0, stream, 1,
                            static_cast<const uint8_t*>(p->d_tmp), g.H1, g.rw, g.l2, g.t2, g.ow, g.oh, p->ksize_v,
                            static_cast<const int*>(p->d_bv), static_cast<const int*>(p->d_kv), g.rh == g.H1 ? 1 : 0, rgb_out,
                            gray_out, u8_out));
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace sta
