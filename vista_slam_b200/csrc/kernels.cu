// Bandwidth-bound and tiny kernels of the STA forward pass (sm_90a, plain SIMT with
// 128-bit vector accesses): LayerNorm, patch im2col, token positions, casts,
// bilinear x2 upsampling, strided im2col, pose head (MLP + 3x3 SVD orthogonalisation),
// and the RoPE sin/cos table.
#include <math.h>
#include <stdlib.h>

#include <mutex>
#include <vector>

#include "common.cuh"
#include "host_util.h"
#include "ops.h"

namespace sta {

// ---------------------------------------------------------------------------
// LayerNorm over the last dim (C % 128 == 0, C <= 1024), fp32 in, bf16 out.
// One warp per row; two-pass statistics in registers (matches torch's fp32 LN).
// Optionally writes a second output with different affine parameters (decoder:
// norm1(x) and norm_y(x) share statistics, sta_blocks.py:227-228), and can drop
// the first row of every `drop_first_of` rows (pose token) from the output.
// Reference: nn.LayerNorm(eps=1e-6) sta_model.py:43.
// ---------------------------------------------------------------------------
// the row's values (v[i] = columns 4 (lane + 32 i) .. + 3), its mean and 1 / sqrt(var + eps)
template <int V>
__device__ __forceinline__ void ln_row_stats(const float4* xp, float eps, float4 (&v)[V], float& mean, float& rstd) {
  constexpr int C = 128 * V;
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    v[i] = xp[(threadIdx.x & 31) + 32 * i];
    sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  mean = sum * (1.0f / C);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    sq += (a * a + b * b) + (c * c + d * d);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  rstd = rsqrtf(sq * (1.0f / C) + eps);
}

template <int C>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, int rows, float eps, const float* __restrict__ g1,
                 const float* __restrict__ b1, __nv_bfloat16* __restrict__ out1, const float* __restrict__ g2,
                 const float* __restrict__ b2, __nv_bfloat16* __restrict__ out2, int drop_first_of, int split) {
  pdl_wait();
  pdl_launch_dependents();
  constexpr int V = C / 128;  // float4 per lane
  const long long ldo = split ? 3 * C : C;  // split-precision mode: rows are (hi | lo | hi)
  // Blocks are scheduled in increasing blockIdx and walk the rows from the END: the residual GEMM that produced x wrote
  // its rows in increasing order, so its last rows are the ones still resident in L2, and the consumer GEMM (increasing
  // rows) then finds this kernel's most recent outputs -- the first rows -- in L2 as well.
  const int blk = static_cast<int>(gridDim.x) - 1 - static_cast<int>(blockIdx.x);
  const int row = blk * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  long long orow = row;
  if (drop_first_of > 0) {
    const int s = row / drop_first_of;
    const int t = row - s * drop_first_of;
    if (t == 0) return;
    orow = static_cast<long long>(s) * (drop_first_of - 1) + (t - 1);
  }
  float4 v[V];
  float mean, rstd;
  ln_row_stats<V>(reinterpret_cast<const float4*>(x + static_cast<long long>(row) * C), eps, v, mean, rstd);
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const int c4 = lane + 32 * i;
    const float n0 = (v[i].x - mean) * rstd, n1 = (v[i].y - mean) * rstd, n2 = (v[i].z - mean) * rstd,
                n3 = (v[i].w - mean) * rstd;
    {
      const float4 g = __ldg(reinterpret_cast<const float4*>(g1) + c4);
      const float4 bb = __ldg(reinterpret_cast<const float4*>(b1) + c4);
      const float y0 = n0 * g.x + bb.x, y1 = n1 * g.y + bb.y, y2 = n2 * g.z + bb.z, y3 = n3 * g.w + bb.w;
      uint2 q;
      q.x = pack_bf16x2(y0, y1);
      q.y = pack_bf16x2(y2, y3);
      reinterpret_cast<uint2*>(out1 + orow * ldo)[c4] = q;
      if (split) {
        reinterpret_cast<uint2*>(out1 + orow * ldo + C)[c4] = make_uint2(pack_bf16x2_resid(y0, y1), pack_bf16x2_resid(y2, y3));
        reinterpret_cast<uint2*>(out1 + orow * ldo + 2 * C)[c4] = q;
      }
    }
    if (out2) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(g2) + c4);
      const float4 bb = __ldg(reinterpret_cast<const float4*>(b2) + c4);
      const float y0 = n0 * g.x + bb.x, y1 = n1 * g.y + bb.y, y2 = n2 * g.z + bb.z, y3 = n3 * g.w + bb.w;
      uint2 q;
      q.x = pack_bf16x2(y0, y1);
      q.y = pack_bf16x2(y2, y3);
      reinterpret_cast<uint2*>(out2 + orow * ldo)[c4] = q;
      if (split) {
        reinterpret_cast<uint2*>(out2 + orow * ldo + C)[c4] = make_uint2(pack_bf16x2_resid(y0, y1), pack_bf16x2_resid(y2, y3));
        reinterpret_cast<uint2*>(out2 + orow * ldo + 2 * C)[c4] = q;
      }
    }
  }
}

int launch_layernorm(const float* x, int rows, int C, float eps, const float* g1, const float* b1, bf16* out1,
                     const float* g2, const float* b2, bf16* out2, int drop_first_of, cudaStream_t stream, int split) {
  if (rows <= 0) return 0;
  const int grid = (rows + 7) / 8;
  if (C == 1024)
    STA_CHECK_CUDA(launch_pdl(layernorm_kernel<1024>, dim3(grid), dim3(256), 0, stream, 1, x, rows, eps, g1, b1, out1, g2, b2, out2,
                              drop_first_of, split));
  else if (C == 768)
    STA_CHECK_CUDA(launch_pdl(layernorm_kernel<768>, dim3(grid), dim3(256), 0, stream, 1, x, rows, eps, g1, b1, out1, g2, b2, out2,
                              drop_first_of, split));
  else {
    set_last_error("layernorm: C must be 768 or 1024");
    return 2;
  }
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------
// FP8 mode (common.cuh fp8_scale): e4m3 rows [rows][C] with one power-of-two scale per row and 128 columns
// ([rows][C / 128] fp32).  A warp's 32 lanes hold one 128-column group, 4 values each.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void quant_group_store(float y0, float y1, float y2, float y3, uint32_t* q, float* s) {
  float am = fmaxf(fmaxf(fabsf(y0), fabsf(y1)), fmaxf(fabsf(y2), fabsf(y3)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, o));
  float sc, inv;
  fp8_scale(am, sc, inv);
  *q = static_cast<uint32_t>(cvt_e4m3x2(y0 * inv, y1 * inv)) | (static_cast<uint32_t>(cvt_e4m3x2(y2 * inv, y3 * inv)) << 16);
  if ((threadIdx.x & 31) == 0) *s = sc;
}

// LayerNorm straight to e4m3 (the FP8 mode's trunk linears read it), statistics as layernorm_kernel; optional second
// output with other affine parameters (decoder norm1 / norm_y).
template <int C>
__global__ void __launch_bounds__(256)
layernorm_fp8_kernel(const float* __restrict__ x, int rows, float eps, const float* __restrict__ g1,
                     const float* __restrict__ b1, uint8_t* __restrict__ q1, float* __restrict__ s1,
                     const float* __restrict__ g2, const float* __restrict__ b2, uint8_t* __restrict__ q2,
                     float* __restrict__ s2) {
  pdl_wait();
  pdl_launch_dependents();
  constexpr int V = C / 128;
  const int blk = static_cast<int>(gridDim.x) - 1 - static_cast<int>(blockIdx.x);  // rows from the end: layernorm_kernel
  const int row = blk * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float4 v[V];
  float mean, rstd;
  ln_row_stats<V>(reinterpret_cast<const float4*>(x + static_cast<long long>(row) * C), eps, v, mean, rstd);
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const int c4 = lane + 32 * i;
    const float n0 = (v[i].x - mean) * rstd, n1 = (v[i].y - mean) * rstd, n2 = (v[i].z - mean) * rstd,
                n3 = (v[i].w - mean) * rstd;
    {
      const float4 g = __ldg(reinterpret_cast<const float4*>(g1) + c4);
      const float4 bb = __ldg(reinterpret_cast<const float4*>(b1) + c4);
      quant_group_store(n0 * g.x + bb.x, n1 * g.y + bb.y, n2 * g.z + bb.z, n3 * g.w + bb.w,
                        reinterpret_cast<uint32_t*>(q1 + static_cast<long long>(row) * C) + c4, s1 + static_cast<long long>(row) * V + i);
    }
    if (q2) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(g2) + c4);
      const float4 bb = __ldg(reinterpret_cast<const float4*>(b2) + c4);
      quant_group_store(n0 * g.x + bb.x, n1 * g.y + bb.y, n2 * g.z + bb.z, n3 * g.w + bb.w,
                        reinterpret_cast<uint32_t*>(q2 + static_cast<long long>(row) * C) + c4, s2 + static_cast<long long>(row) * V + i);
    }
  }
}

int launch_layernorm_fp8(const float* x, int rows, int C, float eps, const float* g1, const float* b1, uint8_t* q1, float* s1,
                         const float* g2, const float* b2, uint8_t* q2, float* s2, cudaStream_t stream) {
  if (rows <= 0) return 0;
  STA_REQUIRE(x && g1 && b1 && q1 && s1 && (!q2 || (g2 && b2 && s2)), "layernorm_fp8: null pointer");
  const int grid = (rows + 7) / 8;
  if (C == 1024)
    STA_CHECK_CUDA(launch_pdl(layernorm_fp8_kernel<1024>, dim3(grid), dim3(256), 0, stream, 1, x, rows, eps, g1, b1, q1, s1, g2,
                              b2, q2, s2));
  else if (C == 768)
    STA_CHECK_CUDA(launch_pdl(layernorm_fp8_kernel<768>, dim3(grid), dim3(256), 0, stream, 1, x, rows, eps, g1, b1, q1, s1, g2,
                              b2, q2, s2));
  else {
    set_last_error("layernorm_fp8: C must be 768 or 1024");
    return 2;
  }
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// bf16 [rows][C] -> e4m3 + scales (the attention output ahead of the FP8 mode's proj GEMMs): one warp per row and
// 128-column group
__global__ void __launch_bounds__(256)
quant_fp8_kernel(const __nv_bfloat16* __restrict__ in, long long groups, uint8_t* __restrict__ q,
                 float* __restrict__ s) {
  pdl_wait();
  pdl_launch_dependents();
  const long long gi = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (gi >= groups) return;
  const int lane = threadIdx.x & 31;
  const uint2 u = reinterpret_cast<const uint2*>(in + gi * 128)[lane];
  quant_group_store(bf16_lo(u.x), bf16_hi(u.x), bf16_lo(u.y), bf16_hi(u.y), reinterpret_cast<uint32_t*>(q + gi * 128) + lane,
                    s + gi);
}

int launch_quant_fp8(const bf16* in, long long rows, int C, uint8_t* q, float* s, cudaStream_t stream) {
  if (rows <= 0) return 0;
  STA_REQUIRE(C > 0 && C % 128 == 0, "quant_fp8: C must be a positive multiple of 128");
  STA_REQUIRE(in && q && s, "quant_fp8: null pointer");
  const long long groups = rows * (C / 128);
  STA_CHECK_CUDA(launch_pdl(quant_fp8_kernel, dim3(static_cast<unsigned>((groups + 7) / 8)), dim3(256), 0, stream, 1, in, groups, q, s));
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------
// PatchEmbed im2col: NCHW image -> [B*h*w][768] bf16 rows, K order (c, ph, pw)
// = Conv2d(3, 1024, 16, 16) weight flattening (sta_blocks.py:262, patch_embed.py:17-27).
// One thread produces 8 consecutive pw values (one 16-byte store).
// ---------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
patch_im2col_kernel(const T* __restrict__ img, int B, int H, int W, __nv_bfloat16* __restrict__ out, int split) {
  pdl_wait();
  pdl_launch_dependents();
  const int h = H / 16, w = W / 16;
  const long long total = static_cast<long long>(B) * h * w * 96;  // 768 / 8 chunks per patch
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int chunk = static_cast<int>(idx % 96);
  const long long patch = idx / 96;
  const int px = static_cast<int>(patch % w);
  const int py = static_cast<int>((patch / w) % h);
  const int b = static_cast<int>(patch / (static_cast<long long>(w) * h));
  const int c = chunk / 32;
  const int ph = (chunk % 32) / 2;
  const int pw0 = (chunk % 2) * 8;
  const T* src = img + ((static_cast<long long>(b) * 3 + c) * H + (py * 16 + ph)) * W + px * 16 + pw0;
  float f[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = static_cast<float>(src[i]);
  uint4 q;
  q.x = pack_bf16x2(f[0], f[1]);
  q.y = pack_bf16x2(f[2], f[3]);
  q.z = pack_bf16x2(f[4], f[5]);
  q.w = pack_bf16x2(f[6], f[7]);
  if (!split) {
    reinterpret_cast<uint4*>(out)[idx] = q;
  } else {  // rows of 3 x 768: (hi | lo | hi)
    uint4* orow = reinterpret_cast<uint4*>(out) + patch * (3 * 96) + chunk;
    orow[0] = q;
    orow[96] = make_uint4(pack_bf16x2_resid(f[0], f[1]), pack_bf16x2_resid(f[2], f[3]), pack_bf16x2_resid(f[4], f[5]),
                          pack_bf16x2_resid(f[6], f[7]));
    orow[192] = q;
  }
}

int launch_patch_im2col(const void* img, int img_is_bf16, int B, int H, int W, bf16* out, cudaStream_t stream, int split) {
  STA_REQUIRE(H % 16 == 0 && W % 16 == 0, "image height and width must be multiples of the patch size 16");
  const long long total = static_cast<long long>(B) * (H / 16) * (W / 16) * 96;
  const int grid = static_cast<int>((total + 255) / 256);
  if (img_is_bf16)
    STA_CHECK_CUDA(launch_pdl(patch_im2col_kernel<__nv_bfloat16>, dim3(grid), dim3(256), 0, stream, 1,
                              static_cast<const __nv_bfloat16*>(img), B, H, W, out, split));
  else
    STA_CHECK_CUDA(launch_pdl(patch_im2col_kernel<float>, dim3(grid), dim3(256), 0, stream, 1, static_cast<const float*>(img), B, H, W,
                              out, split));
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------
// token positions (y, x): PositionGetter sta_blocks.py:235-247; the decoder's pose
// token sits at (-1, -1), sta_model.py:214-219.
// ---------------------------------------------------------------------------
__global__ void make_positions_kernel(int* pos, int B, int h, int w, int with_pose) {
  pdl_wait();
  pdl_launch_dependents();
  const int per = h * w + (with_pose ? 1 : 0);
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(B) * per) return;
  int t = static_cast<int>(idx % per);
  int y, x;
  if (with_pose) {
    if (t == 0) { y = -1; x = -1; } else { --t; y = t / w; x = t % w; }
  } else {
    y = t / w;
    x = t % w;
  }
  pos[2 * idx] = y;
  pos[2 * idx + 1] = x;
}
int launch_make_positions(int* pos, int B, int h, int w, int with_pose_token, cudaStream_t stream) {
  const long long total = static_cast<long long>(B) * (h * w + (with_pose_token ? 1 : 0));
  STA_CHECK_CUDA(launch_pdl(make_positions_kernel, dim3(static_cast<int>((total + 255) / 256)), dim3(256), 0, stream, 1, pos, B, h, w,
                            with_pose_token));
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

__global__ void pos_from_int64_kernel(const long long* __restrict__ in, long long n, int* __restrict__ out) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx < n) out[idx] = static_cast<int>(in[idx]);
}
int launch_pos_from_int64(const long long* pos64, int rows, int* pos32, cudaStream_t stream) {
  const long long n = 2LL * rows;
  pos_from_int64_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, stream>>>(pos64, n, pos32);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------
// fp32 -> bf16 cast of [rows][C] (C % 8 == 0), optionally dropping the first row of
// every `drop_first_of` rows (tok[:, 1:, :] at sta_model.py:271,275).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
cast_f32_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, long long rows, int C,
                     int drop_first_of, int split) {
  pdl_wait();
  pdl_launch_dependents();
  const int cpr = C / 8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= rows * cpr) return;
  const long long row = idx / cpr;
  const int ch = static_cast<int>(idx - row * cpr);
  long long orow = row;
  if (drop_first_of > 0) {
    const long long s = row / drop_first_of;
    const long long t = row - s * drop_first_of;
    if (t == 0) return;
    orow = s * (drop_first_of - 1) + (t - 1);
  }
  const float4* ip = reinterpret_cast<const float4*>(in + row * C + ch * 8);
  const float4 a = ip[0], b = ip[1];
  uint4 q;
  q.x = pack_bf16x2(a.x, a.y);
  q.y = pack_bf16x2(a.z, a.w);
  q.z = pack_bf16x2(b.x, b.y);
  q.w = pack_bf16x2(b.z, b.w);
  if (!split) {
    *reinterpret_cast<uint4*>(out + orow * C + ch * 8) = q;
  } else {
    __nv_bfloat16* o = out + orow * 3 * C + ch * 8;
    *reinterpret_cast<uint4*>(o) = q;
    *reinterpret_cast<uint4*>(o + C) = make_uint4(pack_bf16x2_resid(a.x, a.y), pack_bf16x2_resid(a.z, a.w),
                                                  pack_bf16x2_resid(b.x, b.y), pack_bf16x2_resid(b.z, b.w));
    *reinterpret_cast<uint4*>(o + 2 * C) = q;
  }
}
int launch_cast_f32_bf16(const float* in, bf16* out, long long rows, int C, int drop_first_of, cudaStream_t stream,
                         int split) {
  STA_REQUIRE(C % 8 == 0, "C must be a multiple of 8");
  const long long total = rows * (C / 8);
  if (total == 0) return 0;
  STA_CHECK_CUDA(launch_pdl(cast_f32_bf16_kernel, dim3(static_cast<int>((total + 255) / 256)), dim3(256), 0, stream, 1, in, out, rows,
                            C, drop_first_of, split));
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// x[s, 0, :] = init_pose_token  (sta_model.py:206-212)
__global__ void fill_pose_token_kernel(float* x, const float* __restrict__ tok, int samples, long long sample_stride,
                                       int C) {
  pdl_wait();
  pdl_launch_dependents();
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(samples) * C) return;
  const int s = static_cast<int>(idx / C);
  const int c = static_cast<int>(idx - static_cast<long long>(s) * C);
  x[s * sample_stride + c] = tok[c];
}
int launch_fill_pose_token(float* x, const float* tok, int samples, int tokens_per_sample, int C,
                           cudaStream_t stream) {
  const long long total = static_cast<long long>(samples) * C;
  STA_CHECK_CUDA(launch_pdl(fill_pose_token_kernel, dim3(static_cast<int>((total + 255) / 256)), dim3(256), 0, stream, 1, x, tok,
                            samples, static_cast<long long>(tokens_per_sample) * C, C));
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

__global__ void copy_f32_kernel(const float4* __restrict__ in, float4* __restrict__ out, long long n4) {
  pdl_wait();
  pdl_launch_dependents();
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx < n4) out[idx] = in[idx];
}
int launch_copy_f32(const float* in, float* out, long long n, cudaStream_t stream) {
  STA_REQUIRE(n % 4 == 0, "copy length must be a multiple of 4 floats");
  const long long n4 = n / 4;
  if (n4 == 0) return 0;
  STA_CHECK_CUDA(launch_pdl(copy_f32_kernel, dim3(static_cast<int>((n4 + 255) / 256)), dim3(256), 0, stream, 1,
                            reinterpret_cast<const float4*>(in), reinterpret_cast<float4*>(out), n4));
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------
// bilinear x2 upsampling, align_corners=True, NHWC bf16 (dpt_block.py:215-216,320).
// src coordinate = dst * (in - 1) / (out - 1); weights in fp32 like ATen's
// upsample_bilinear2d (area_pixel_compute_scale with align_corners).
// One block: one output row (blockIdx.y) of one image (blockIdx.z), a run of kUpsPix * (256 / (C/8)) pixels; one
// thread: 8 channels of kUpsPix pixels, so the row weights are computed once and all index math is 32-bit.
// ---------------------------------------------------------------------------
constexpr int kUpsPix = 4;
__global__ void __launch_bounds__(256)
upsample2x_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int nimg, int H, int W, int C,
                  int OH, int OW, int split) {
  pdl_wait();
  pdl_launch_dependents();
  // the interpolation grid is always the full 2H x 2W one; (OH, OW) <= (2H, 2W) only crops the output
  const int FH = 2 * H, FW = 2 * W;
  const int cpp = C >> 3;            // 16-byte channel groups per pixel
  const int ppb = 256 / cpp;         // pixels per block pass
  const int ch = threadIdx.x % cpp;
  const int pl = threadIdx.x / cpp;
  if (pl >= ppb) return;
  const int oy = blockIdx.y, n = blockIdx.z;
  const float sy = (FH > 1) ? static_cast<float>(H - 1) / static_cast<float>(FH - 1) : 0.f;
  const float sx = (FW > 1) ? static_cast<float>(W - 1) / static_cast<float>(FW - 1) : 0.f;
  const float fy = sy * oy;
  const int y0 = static_cast<int>(fy);
  const int y1 = y0 + (y0 < H - 1 ? 1 : 0);
  const float ly = fy - y0, hy = 1.f - ly;
  const int PC = split ? 3 * C : C;  // physical channels per pixel (split-precision mode: hi | lo | hi)
  const __nv_bfloat16* row0 = in + (static_cast<long long>(n) * H + y0) * W * PC + ch * 8;
  const __nv_bfloat16* row1 = in + (static_cast<long long>(n) * H + y1) * W * PC + ch * 8;
  __nv_bfloat16* orow = out + (static_cast<long long>(n) * OH + oy) * OW * PC + ch * 8;
  const int ox_base = blockIdx.x * (ppb * kUpsPix) + pl;
  if (split) {
    // parity mode (not performance critical): interpolate hi + lo in fp32, store (hi | lo | hi)
    for (int k = 0; k < kUpsPix; ++k) {
      const int ox = ox_base + k * ppb;
      if (ox >= OW) break;
      const float fx = sx * ox;
      int x0 = static_cast<int>(fx);
      x0 = x0 < W - 1 ? x0 : W - 1;
      const int x1 = x0 + (x0 < W - 1 ? 1 : 0);
      const float lx = fx - x0, hx = 1.f - lx;
      float r[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        auto val = [&](const __nv_bfloat16* rp, int x) {
          return __bfloat162float(rp[x * PC + i]) + __bfloat162float(rp[x * PC + C + i]);
        };
        r[i] = hy * (hx * val(row0, x0) + lx * val(row0, x1)) + ly * (hx * val(row1, x0) + lx * val(row1, x1));
      }
      __nv_bfloat16* o = orow + static_cast<long long>(ox) * PC;
      const uint4 hi = make_uint4(pack_bf16x2(r[0], r[1]), pack_bf16x2(r[2], r[3]), pack_bf16x2(r[4], r[5]),
                                  pack_bf16x2(r[6], r[7]));
      *reinterpret_cast<uint4*>(o) = hi;
      *reinterpret_cast<uint4*>(o + C) = make_uint4(pack_bf16x2_resid(r[0], r[1]), pack_bf16x2_resid(r[2], r[3]),
                                                    pack_bf16x2_resid(r[4], r[5]), pack_bf16x2_resid(r[6], r[7]));
      *reinterpret_cast<uint4*>(o + 2 * C) = hi;
    }
    return;
  }
  uint4 q00[kUpsPix], q01[kUpsPix], q10[kUpsPix], q11[kUpsPix];
  float lxs[kUpsPix];
#pragma unroll
  for (int k = 0; k < kUpsPix; ++k) {
    const int ox = ox_base + k * ppb;
    const float fx = sx * ox;
    int x0 = static_cast<int>(fx);
    x0 = x0 < W - 1 ? x0 : W - 1;  // also keeps the loads of out-of-range pixels (ox >= OW) in bounds
    const int x1 = x0 + (x0 < W - 1 ? 1 : 0);
    lxs[k] = fx - x0;
    q00[k] = *reinterpret_cast<const uint4*>(row0 + x0 * C);
    q01[k] = *reinterpret_cast<const uint4*>(row0 + x1 * C);
    q10[k] = *reinterpret_cast<const uint4*>(row1 + x0 * C);
    q11[k] = *reinterpret_cast<const uint4*>(row1 + x1 * C);
  }
#pragma unroll
  for (int k = 0; k < kUpsPix; ++k) {
    const int ox = ox_base + k * ppb;
    if (ox >= OW) break;
    const float lx = lxs[k], hx = 1.f - lx;
    const uint32_t a00[4] = {q00[k].x, q00[k].y, q00[k].z, q00[k].w}, a01[4] = {q01[k].x, q01[k].y, q01[k].z, q01[k].w};
    const uint32_t a10[4] = {q10[k].x, q10[k].y, q10[k].z, q10[k].w}, a11[4] = {q11[k].x, q11[k].y, q11[k].z, q11[k].w};
    uint32_t r[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float lo = hy * (hx * bf16_lo(a00[i]) + lx * bf16_lo(a01[i])) + ly * (hx * bf16_lo(a10[i]) + lx * bf16_lo(a11[i]));
      const float hi = hy * (hx * bf16_hi(a00[i]) + lx * bf16_hi(a01[i])) + ly * (hx * bf16_hi(a10[i]) + lx * bf16_hi(a11[i]));
      r[i] = pack_bf16x2(lo, hi);
    }
    *reinterpret_cast<uint4*>(orow + static_cast<long long>(ox) * C) = make_uint4(r[0], r[1], r[2], r[3]);
  }
}
int launch_upsample2x(const bf16* in, bf16* out, int nimg, int H, int W, int C, int OH, int OW, cudaStream_t stream,
                      int split) {
  STA_REQUIRE(C % 8 == 0 && C / 8 <= 256, "C must be a multiple of 8, at most 2048");
  STA_REQUIRE(OH <= 2 * H && OW <= 2 * W && OH > 0 && OW > 0, "output crop must fit inside the 2x grid");
  STA_REQUIRE(OH <= 65535 && nimg <= 65535, "grid limits");
  if (nimg == 0) return 0;
  const int ppb = 256 / (C / 8);
  const int gx = (OW + ppb * kUpsPix - 1) / (ppb * kUpsPix);
  STA_CHECK_CUDA(launch_pdl(upsample2x_kernel, dim3(gx, OH, nimg), dim3(256), 0, stream, 1, in, out, nimg, H, W, C, OH, OW, split));
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------
// im2col for the one strided conv (act_postprocess[3][1]: 3x3, stride 2, pad 1,
// dpt_block.py:403-410): NHWC [n][H][W][C] -> [n*OH*OW][9*C], K order (kh, kw, c).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
im2col_3x3_s2_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int nimg, int H, int W,
                     int C) {
  pdl_wait();
  pdl_launch_dependents();
  const int OH = (H + 1) / 2, OW = (W + 1) / 2;  // floor((H + 2 - 3) / 2) + 1
  const int cpp = C / 8;
  const long long total = static_cast<long long>(nimg) * OH * OW * 9 * cpp;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int ch = static_cast<int>(idx % cpp);
  long long t = idx / cpp;
  const int tap = static_cast<int>(t % 9);
  t /= 9;
  const int ox = static_cast<int>(t % OW);
  t /= OW;
  const int oy = static_cast<int>(t % OH);
  const int n = static_cast<int>(t / OH);
  const int iy = oy * 2 + tap / 3 - 1, ix = ox * 2 + tap % 3 - 1;
  uint4 q = make_uint4(0, 0, 0, 0);
  if (iy >= 0 && iy < H && ix >= 0 && ix < W)
    q = *reinterpret_cast<const uint4*>(in + ((static_cast<long long>(n) * H + iy) * W + ix) * C + ch * 8);
  reinterpret_cast<uint4*>(out)[idx] = q;
}
int launch_im2col_3x3_s2(const bf16* in, bf16* out, int nimg, int H, int W, int C, cudaStream_t stream) {
  STA_REQUIRE(C % 8 == 0, "C must be a multiple of 8");
  const long long total = static_cast<long long>(nimg) * ((H + 1) / 2) * ((W + 1) / 2) * 9 * (C / 8);
  if (total == 0) return 0;
  STA_CHECK_CUDA(launch_pdl(im2col_3x3_s2_kernel, dim3(static_cast<int>((total + 255) / 256)), dim3(256), 0, stream, 1, in, out, nimg,
                            H, W, C));
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------
// Pose head (heads/pose_head.py:7-119), one CTA (256 threads) per sample, all fp32:
//   [dec_norm] -> 3 x (Linear + ReLU) (768 -> 512 -> 512 -> 512) -> fc_t (3), fc_rot (9),
//   sigmoid(fc_conf); R = svd_orthogonalize(fc_rot) (pose_head.py:38-57):
//     A = normalize_rows(M)^T ; A = U S V^T ; R = V diag(1, 1, det(V U^T)) U^T
//   computed with a one-sided Jacobi SVD of the 3x3 in registers (thread 0).
// ---------------------------------------------------------------------------
__device__ __forceinline__ float block_sum_256(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) t += red[i];
  __syncthreads();
  return t;
}

// y[o] = act(W[o,:] . x + b[o]).  Each warp produces 4 output rows at a time with 128-bit weight loads and
// fully unrolled (independent) loads, so ~24 L2 requests per lane are in flight instead of one.
template <int IN_DIM>
__device__ __forceinline__ void dense_layer(const float* __restrict__ W, const float* __restrict__ b,
                                            const float* x_s, float* y_s, int out_dim, int relu) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int IT = IN_DIM / 128;  // float4 per lane per row
  float4 xv[IT];
#pragma unroll
  for (int k = 0; k < IT; ++k) xv[k] = *reinterpret_cast<const float4*>(x_s + 4 * (lane + 32 * k));
  for (int o = warp * 4; o < out_dim; o += 32) {
    float4 wv[4][IT];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int k = 0; k < IT; ++k)
        wv[r][k] = __ldg(reinterpret_cast<const float4*>(W + static_cast<long long>(o + r) * IN_DIM) + lane + 32 * k);
    float acc[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      float a = 0.f;
#pragma unroll
      for (int k = 0; k < IT; ++k)
        a += wv[r][k].x * xv[k].x + wv[r][k].y * xv[k].y + wv[r][k].z * xv[k].z + wv[r][k].w * xv[k].w;
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) a += __shfl_xor_sync(0xffffffffu, a, s);
      acc[r] = a;
    }
    if (lane < 4) {
      float v = (lane == 0 ? acc[0] : lane == 1 ? acc[1] : lane == 2 ? acc[2] : acc[3]) + b[o + lane];
      y_s[o + lane] = relu ? fmaxf(v, 0.f) : v;
    }
  }
  __syncthreads();
}

// One-sided (Hestenes) Jacobi SVD of a 3x3 matrix A (row-major): A = U S V^T.
// Returns R = V diag(1,1,det(V U^T)) U^T.  Zero singular values are handled by
// completing U with a cross product.
__device__ void svd_orthogonalize_3x3(const float* A, float* R) {
  float B[3][3], V[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      B[i][j] = A[3 * i + j];
      V[i][j] = (i == j) ? 1.f : 0.f;
    }
  for (int sweep = 0; sweep < 12; ++sweep) {
    float off = 0.f;
#pragma unroll
    for (int pq = 0; pq < 3; ++pq) {
      const int pc = (pq == 2) ? 1 : 0;
      const int qc = (pq == 0) ? 1 : 2;
      float alpha = 0.f, beta = 0.f, gamma = 0.f;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        alpha += B[i][pc] * B[i][pc];
        beta += B[i][qc] * B[i][qc];
        gamma += B[i][pc] * B[i][qc];
      }
      off = fmaxf(off, fabsf(gamma) / fmaxf(sqrtf(alpha * beta), 1e-30f));
      if (fabsf(gamma) > 1e-30f) {
        const float zeta = (beta - alpha) / (2.f * gamma);
        const float t = copysignf(1.f, zeta) / (fabsf(zeta) + sqrtf(1.f + zeta * zeta));
        const float c = rsqrtf(1.f + t * t), s = c * t;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const float bp = B[i][pc], bq = B[i][qc];
          B[i][pc] = c * bp - s * bq;
          B[i][qc] = s * bp + c * bq;
          const float vp = V[i][pc], vq = V[i][qc];
          V[i][pc] = c * vp - s * vq;
          V[i][qc] = s * vp + c * vq;
        }
      }
    }
    if (off < 1e-7f) break;
  }
  // columns of B are sigma_j * u_j ; sort so the smallest singular value is last
  float sig[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) sig[j] = sqrtf(B[0][j] * B[0][j] + B[1][j] * B[1][j] + B[2][j] * B[2][j]);
  int order[3] = {0, 1, 2};
  if (sig[order[0]] < sig[order[1]]) { int t = order[0]; order[0] = order[1]; order[1] = t; }
  if (sig[order[1]] < sig[order[2]]) { int t = order[1]; order[1] = order[2]; order[2] = t; }
  if (sig[order[0]] < sig[order[1]]) { int t = order[0]; order[0] = order[1]; order[1] = t; }
  float U[3][3], Vs[3][3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int src = order[j];
    const float inv = sig[src] > 1e-20f ? 1.f / sig[src] : 0.f;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      U[i][j] = B[i][src] * inv;
      Vs[i][j] = V[i][src];
    }
  }
  // rank deficient: complete U to an orthonormal basis.  Rank 0: u0 = e0.  Rank <= 1: u1 = the coordinate axis least
  // aligned with u0, made orthogonal to it.  Rank <= 2: u2 = u0 x u1.
  if (sig[order[0]] <= 1e-20f) {
    U[0][0] = 1.f; U[1][0] = 0.f; U[2][0] = 0.f;
  }
  if (sig[order[1]] <= 1e-20f) {
    const float a0 = fabsf(U[0][0]), a1 = fabsf(U[1][0]), a2 = fabsf(U[2][0]);
    const int k = (a0 <= a1 && a0 <= a2) ? 0 : (a1 <= a2 ? 1 : 2);
    float v[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) v[i] = (i == k ? 1.f : 0.f) - U[k][0] * U[i][0];
    const float inv = rsqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);  // |v|^2 = 1 - u0_k^2 >= 2/3
#pragma unroll
    for (int i = 0; i < 3; ++i) U[i][1] = v[i] * inv;
  }
  if (sig[order[2]] <= 1e-20f) {
    U[0][2] = U[1][0] * U[2][1] - U[2][0] * U[1][1];
    U[1][2] = U[2][0] * U[0][1] - U[0][0] * U[2][1];
    U[2][2] = U[0][0] * U[1][1] - U[1][0] * U[0][1];
  }
  // det(V U^T) = det(V) det(U)
  auto det3 = [](float M[3][3]) {
    return M[0][0] * (M[1][1] * M[2][2] - M[1][2] * M[2][1]) - M[0][1] * (M[1][0] * M[2][2] - M[1][2] * M[2][0]) +
           M[0][2] * (M[1][0] * M[2][1] - M[1][1] * M[2][0]);
  };
  const float d = det3(Vs) * det3(U);
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      R[3 * i + j] = Vs[i][0] * U[j][0] + Vs[i][1] * U[j][1] + d * Vs[i][2] * U[j][2];
}

__global__ void __launch_bounds__(256)
pose_head_kernel(const float* __restrict__ x, long long sample_stride, int apply_ln, float eps, PoseHeadWeights w,
                 float* __restrict__ pose44, float* __restrict__ conf) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ __align__(16) float buf0[768];
  __shared__ __align__(16) float buf1[512];
  __shared__ float red[8];
  __shared__ float outv[16];
  const int s = blockIdx.x;
  const float* xr = x + s * sample_stride;
  float v[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) v[i] = xr[threadIdx.x + 256 * i];
  if (apply_ln) {
    const float mean = block_sum_256(v[0] + v[1] + v[2], red) * (1.f / 768.f);
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < 3; ++i) sq += (v[i] - mean) * (v[i] - mean);
    const float rstd = rsqrtf(block_sum_256(sq, red) * (1.f / 768.f) + eps);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const int c = threadIdx.x + 256 * i;
      v[i] = (v[i] - mean) * rstd * w.ln_g[c] + w.ln_b[c];
    }
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) buf0[threadIdx.x + 256 * i] = v[i];
  __syncthreads();
  dense_layer<768>(w.w0, w.b0, buf0, buf1, 512, 1);
  dense_layer<512>(w.w1, w.b1, buf1, buf0, 512, 1);
  dense_layer<512>(w.w2, w.b2, buf0, buf1, 512, 1);
  // 13 small outputs: t(3), rot(9), conf(1)
  {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int o = warp; o < 13; o += 8) {
      const float* wr;
      float bias;
      if (o < 3) { wr = w.wt + o * 512; bias = w.bt[o]; }
      else if (o < 12) { wr = w.wr + (o - 3) * 512; bias = w.br[o - 3]; }
      else { wr = w.wc; bias = w.bc[0]; }
      float acc = 0.f;
      for (int i = lane; i < 512; i += 32) acc = fmaf(__ldg(wr + i), buf1[i], acc);
#pragma unroll
      for (int sft = 16; sft > 0; sft >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, sft);
      if (lane == 0) outv[o] = acc + bias;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // rows of M are L2-normalised (F.normalize eps 1e-12), then transposed
    float Mn[9], A[9], R[9];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const float a = outv[3 + 3 * i], b = outv[4 + 3 * i], c = outv[5 + 3 * i];
      const float inv = 1.f / fmaxf(sqrtf(a * a + b * b + c * c), 1e-12f);
      Mn[3 * i] = a * inv; Mn[3 * i + 1] = b * inv; Mn[3 * i + 2] = c * inv;
    }
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) A[3 * i + j] = Mn[3 * j + i];
    svd_orthogonalize_3x3(A, R);
    float* P = pose44 + 16 * s;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      P[4 * i + 0] = R[3 * i + 0];
      P[4 * i + 1] = R[3 * i + 1];
      P[4 * i + 2] = R[3 * i + 2];
      P[4 * i + 3] = outv[i];
    }
    P[12] = 0.f; P[13] = 0.f; P[14] = 0.f; P[15] = 1.f;
    conf[s] = 1.f / (1.f + expf(-outv[12]));
  }
}

int launch_pose_head(const float* x, long long sample_stride, int samples, int apply_ln, float eps,
                     const PoseHeadWeights& w, float* pose44, float* conf, cudaStream_t stream) {
  if (samples <= 0) return 0;
  STA_CHECK_CUDA(launch_pdl(pose_head_kernel, dim3(samples), dim3(256), 0, stream, 1, x, sample_stride, apply_ln, eps, w, pose44,
                            conf));
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------
// RoPE table: tab[(pos + 1) * 16 + i] = (cos, sin)(pos * 100^(-i/16)), pos in [-1, 1023]
// (pos_embed.py:128-146 with base = 100, F0 = 1, D/4 = 16 frequencies per axis).
// Built once per device in fp32 exactly like the reference (inv_freq = 1 / base^(i/16)).
// ---------------------------------------------------------------------------
static constexpr int kRopeMaxPos = 1023;
const float* rope_table(int* max_pos) {
  static std::mutex mu;
  static std::vector<float*> tabs(64, nullptr);
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  std::lock_guard<std::mutex> lock(mu);
  if (max_pos) *max_pos = kRopeMaxPos;
  if (tabs[dev]) return tabs[dev];
  const int npos = kRopeMaxPos + 2;
  std::vector<float> h(static_cast<size_t>(npos) * 32);
  for (int p = 0; p < npos; ++p) {
    const float pos = static_cast<float>(p - 1);
    for (int i = 0; i < 16; ++i) {
      const float inv_freq = 1.0f / powf(100.0f, static_cast<float>(i) / 16.0f);
      const float ang = pos * inv_freq;
      h[(static_cast<size_t>(p) * 16 + i) * 2 + 0] = cosf(ang);
      h[(static_cast<size_t>(p) * 16 + i) * 2 + 1] = sinf(ang);
    }
  }
  float* d = nullptr;
  if (cudaMalloc(&d, h.size() * sizeof(float)) != cudaSuccess) return nullptr;
  if (cudaMemcpy(d, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) return nullptr;
  tabs[dev] = d;
  return d;
}

}  // namespace sta
