// Host launcher for the wgmma GEMM / implicit-GEMM convolution (gemm.cuh).
#include "gemm.cuh"
#include "host_util.h"
#include "ops.h"

namespace sta {

// x[m][n] (+)= bias[n] + sum_ks partial[ks][m][n]  -- second pass of the split-K route (fixed summation order)
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ partial, long long slice_elems, int ksplit, const float* __restrict__ bias,
                     float* __restrict__ out, long long ldo, int M, int N, int accumulate) {
  pdl_wait();
  pdl_launch_dependents();
  const int n4 = N / 4;
  const long long total = static_cast<long long>(M) * n4;
  for (long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * 256) {
    const int m = static_cast<int>(i / n4), c = static_cast<int>(i - static_cast<long long>(m) * n4) * 4;
    float4 acc = bias ? __ldg(reinterpret_cast<const float4*>(bias + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float* pp = partial + static_cast<long long>(m) * N + c;
    for (int ks = 0; ks < ksplit; ++ks) {
      const float4 v = *reinterpret_cast<const float4*>(pp + ks * slice_elems);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    float4* o = reinterpret_cast<float4*>(out + static_cast<long long>(m) * ldo + c);
    if (accumulate) {
      const float4 r = *o;
      acc.x += r.x; acc.y += r.y; acc.z += r.z; acc.w += r.w;
    }
    *o = acc;
  }
}

template <int AMODE, int EPI, bool TMA>
static int launch_inst(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const GemmParams& p,
                       int num_tiles, cudaStream_t stream) {
  using Cfg = GemmCfg<AMODE, EPI, TMA>;
  auto kern = gemm_wg_kernel<AMODE, EPI, TMA>;
  static PerDeviceOnce once;  // the opt-in is per device, not per process
  STA_CHECK_CUDA(once.run(
      [&] { return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM_BYTES); }));
  // persistent: one CTA per SM at most
  const int items = num_tiles < num_sms() ? num_tiles : num_sms();
  if (items < 1) return 0;
  STA_CHECK_CUDA(launch_pdl(kern, dim3(items), dim3(Cfg::THREADS), Cfg::SMEM_BYTES, stream, 1, tmA, tmB, tmC, p));
  return 0;
}

template <int EPI>
static int launch_wide(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const GemmParams& p,
                       int num_tiles, cudaStream_t stream) {
  using Cfg = GemmWideCfg<EPI>;
  auto kern = gemm_wide_kernel<EPI>;
  static PerDeviceOnce once;
  STA_CHECK_CUDA(once.run(
      [&] { return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM_BYTES); }));
  const int items = num_tiles < num_sms() ? num_tiles : num_sms();
  if (items < 1) return 0;
  STA_CHECK_CUDA(launch_pdl(kern, dim3(items), dim3(Cfg::THREADS), Cfg::SMEM_BYTES, stream, 1, tmA, tmB, tmC, p));
  return 0;
}

// Wave efficiency of a persistent grid: tiles over the tile slots of the waves it takes.
static double wave_efficiency(long long tiles, int sms) {
  const long long waves = (tiles + sms - 1) / sms;
  return static_cast<double>(tiles) / static_cast<double>(waves * sms);
}

// The 128 x 256 kernel needs less shared-memory traffic per MAC than the 128 x 128 kernel, but its epilogue is not
// hidden behind another tile's MMAs and it has half as many tiles.  Per-layer times at cfg-2 on the 700 W H100
// (DESIGN.md section 5): it wins where the 128 x 128 kernel is bound by that traffic -- many column tiles (enc qkv
// N = 3072: 0.301 -> 0.249 ms, enc fc1 N = 4096: 0.377 -> 0.330 ms, dec qkv N = 2304: 0.174 -> 0.153 ms) or a long k loop
// (enc fc2 K = 4096: 0.376 -> 0.296 ms) -- and loses where both are short (enc proj N = K = 1024: 0.128 -> 0.134 ms).
// So it is taken for N >= 2048 or K >= 2048, and only when its wave efficiency is at most 5 points below the 128 x 128
// kernel's: the decoder's N = 768 layers (87.7 % against 97.5 % at M = 24608 on 132 SMs) and the one-keyframe SLAM
// shapes (a few tiles on a mostly idle GPU) keep 128 x 128 tiles.
int gemm_auto_tile_n(int M, int N, int K, int epi, int num_sms) {
  if (M <= 0 || N % 256 != 0 || num_sms <= 0 || (N < 2048 && K < 2048)) return 128;
  if (epi != EPI_BF16 && epi != EPI_GELU && epi != EPI_F32 && epi != EPI_ROPE) return 128;
  const long long m_tiles = (M + 127) / 128;
  const double wide = wave_efficiency(m_tiles * (N / 256), num_sms);
  const double narrow = wave_efficiency(m_tiles * (N / 128), num_sms);
  return wide >= narrow - 0.05 ? 256 : 128;
}

int launch_gemm(const GemmLaunch& g, cudaStream_t stream) {
  GemmParams p = g.p;
  const bool fp8 = g.amode == A_FP8;
  STA_REQUIRE(p.N % 32 == 0, "N must be a multiple of 32");
  STA_REQUIRE(!fp8 || (p.N % 128 == 0 && p.K % 128 == 0 && p.K > 0 && p.M > 0 && !p.split),
              "e4m3 operands need N and K multiples of 128");
  STA_REQUIRE(!fp8 || (p.a_scale != nullptr && p.w_scale != nullptr), "e4m3 operands need their scales");
  STA_REQUIRE(!fp8 || g.epi == EPI_F32 || g.epi == EPI_ROPE || g.epi == EPI_GELU_FP8,
              "e4m3 operands: EPI_F32, EPI_ROPE or EPI_GELU_FP8");
  STA_REQUIRE(g.epi != EPI_GELU_FP8 || (fp8 && p.out_scale != nullptr), "EPI_GELU_FP8 needs e4m3 operands and out_scale");
  STA_REQUIRE(!p.split || g.epi == EPI_F32 || g.epi == EPI_HEAD || g.epi == EPI_PIXSHUF || p.ldo >= 3LL * p.N,
              "split-precision bf16 outputs need ldo >= 3N");
  STA_REQUIRE(g.A != nullptr && g.Wt != nullptr, "null operand");
  STA_REQUIRE((reinterpret_cast<uintptr_t>(g.A) & 15) == 0 && (reinterpret_cast<uintptr_t>(g.Wt) & 15) == 0,
              "operands must be 16-byte aligned");

  // 128 x 128 tiles: two m64n128 wgmmas per consumer warpgroup and k16 step
  const int bn = 128;

  // TMA-store epilogue (epilogue_tile_tma) for the linear layers: bf16 / GELU / RoPE outputs without skip
  // tensors, fp32 outputs that either have no residual or accumulate in place (out += ..., bulk reduce-add).
  // GELU and RoPE have no other epilogue.
  const int esz = (g.epi == EPI_F32) ? 4 : (g.epi == EPI_GELU_FP8) ? 1 : 2;
  bool tma = p.N % bn == 0 && (g.amode == A_LINEAR || fp8) && p.out != nullptr && p.out2 == nullptr &&
             (reinterpret_cast<uintptr_t>(p.out) & 15) == 0 && (p.ldo * esz) % 16 == 0;
  p.c_reduce = 0;
  if (g.epi == EPI_BF16) {
    tma = tma && p.resid == nullptr && p.resid2 == nullptr;
  } else if (g.epi == EPI_F32) {
    tma = tma && p.rowmap_n == 0 && (p.resid == nullptr || p.resid == p.out);
    p.c_reduce = (p.resid != nullptr) ? 1 : 0;
  } else if (g.epi == EPI_GELU || g.epi == EPI_ROPE || g.epi == EPI_GELU_FP8) {
    STA_REQUIRE(tma, "GELU / RoPE epilogues need a linear layer with N % 128 == 0, a 16-byte aligned output and row "
                     "stride, and no out2");
  } else {
    tma = false;
  }
  STA_REQUIRE(!fp8 || tma, "e4m3 operands need the TMA-store epilogue (16-byte aligned output, fp32 residual in place)");
  const int bk = fp8 ? 128 : 64;  // k-block: one 128-byte operand row

  // Small problems (one keyframe / a few edges in SLAM mode) are bound by streaming the weights through too few SMs:
  // the fp32 residual-stream layers (out += A W^T + b) with fewer tiles than SMs split K across CTAs: every split
  // stores its partial tile to scratch and a second tiny kernel sums them in a fixed order (deterministic, unlike
  // reduce-adds racing).
  int ksplit = 1;
  if (tma && g.epi == EPI_F32 && g.splitk_ws != nullptr) {
    const int tiles = ((p.M + 127) / 128) * (p.N / bn), nkb = (p.K + bk - 1) / bk;
    if (tiles < num_sms()) {
      int ks = num_sms() / tiles;
      if (ks > 8) ks = 8;
      if (ks > nkb / 2) ks = nkb / 2;
      const size_t need = static_cast<size_t>(ks) * ((p.M + 127) / 128) * 128 * p.N * sizeof(float);
      if (ks >= 2 && need <= g.splitk_ws_bytes && (reinterpret_cast<uintptr_t>(g.splitk_ws) & 15) == 0) ksplit = ks;
    }
  }
  // 128 x 256 tiles (gemm_wide_kernel) for the plain linear layers with the TMA-store epilogue
  STA_REQUIRE(g.tile_n == 0 || g.tile_n == 128 || g.tile_n == 256, "tile_n must be 0, 128 or 256");
  const bool wide_ok = tma && g.amode == A_LINEAR && !p.split && ksplit == 1 && p.N % 256 == 0 &&
                       (g.epi == EPI_BF16 || g.epi == EPI_GELU || g.epi == EPI_F32 || g.epi == EPI_ROPE);
  STA_REQUIRE(g.tile_n != 256 || wide_ok,
              "tile_n = 256 needs a linear layer with the TMA-store epilogue, N % 256 == 0, no split-K and no "
              "split precision");
  const bool wide = wide_ok && (g.tile_n == 256 || (g.tile_n == 0 && gemm_auto_tile_n(p.M, p.N, p.K, g.epi, num_sms()) == 256));
  const int bn_tile = wide ? 256 : bn;
  CUtensorMap tmA, tmB;
  int m_tiles;
  if (g.amode == A_CONV3) {
    STA_REQUIRE(p.Cin % 64 == 0, "conv input channels must be a multiple of 64");
    STA_REQUIRE(p.K == 9 * p.Cin, "conv K must be 9*Cin");
    // 16 x 8-pixel tiles fed from one 18 x 10-pixel box per channel chunk
    p.tiles_h = (p.H + 15) / 16;
    p.tiles_w = (p.W + 7) / 8;
    p.M = p.nimg * p.H * p.W;
    m_tiles = p.nimg * p.tiles_h * p.tiles_w;
    uint64_t dims[4] = {(uint64_t)p.Cin, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.nimg};
    uint64_t strides[3] = {(uint64_t)p.Cin * 2, (uint64_t)p.W * p.Cin * 2, (uint64_t)p.H * p.W * p.Cin * 2};
    uint32_t box[4] = {64, (uint32_t)kHaloPitch, 18u, 1};
    if (make_tmap_bf16(&tmA, g.A, 4, dims, strides, box)) return 1;
  } else {
    const int oes = fp8 ? 1 : 2;  // operand bytes
    STA_REQUIRE(g.lda * oes % 16 == 0, "lda must be a multiple of 16 bytes");
    m_tiles = (p.M + 127) / 128;
    uint64_t dims[2] = {(uint64_t)p.K, (uint64_t)p.M};
    uint64_t strides[1] = {(uint64_t)g.lda * oes};
    uint32_t box[2] = {(uint32_t)bk, 128};
    if (make_tmap(&tmA, g.A, fp8 ? 2 : 0, 2, dims, strides, box)) return 1;
  }
  {
    const int oes = fp8 ? 1 : 2;
    STA_REQUIRE(g.ldw * oes % 16 == 0, "ldw must be a multiple of 16 bytes");
    uint64_t dims[2] = {(uint64_t)p.K, (uint64_t)p.N};
    uint64_t strides[1] = {(uint64_t)g.ldw * oes};
    uint32_t box[2] = {(uint32_t)bk, (uint32_t)bn_tile};
    if (make_tmap(&tmB, g.Wt, fp8 ? 2 : 0, 2, dims, strides, box)) return 1;
  }
  const int n_tiles = (p.N + bn_tile - 1) / bn_tile;
  const int num_tiles = m_tiles * n_tiles * ksplit;

  CUtensorMap tmC = tmA;
  p.ksplit = 1;
  p.split_rows = 0;
  // split-K: the GEMM stores bias-free partial tiles into scratch slices, splitk_reduce_kernel finishes the layer
  const float* final_bias = p.bias;
  float* final_out = static_cast<float*>(p.out);
  const int final_accumulate = p.c_reduce;
  if (tma && ksplit > 1) {
    p.ksplit = ksplit;
    p.split_rows = m_tiles * 128;
    p.bias = nullptr;
    p.c_reduce = 0;
    uint64_t dims[2] = {(uint64_t)p.N, (uint64_t)ksplit * p.split_rows};
    uint64_t strides[1] = {(uint64_t)p.N * 4};
    uint32_t box[2] = {32, 16};  // one 16-row group of a warp's accumulator fragments
    if (make_tmap(&tmC, g.splitk_ws, 1, 2, dims, strides, box)) return 1;
  } else if (tma) {
    ksplit = 1;
    // split-precision mode: bf16 rows are (hi | lo | hi), 3N wide
    uint64_t dims[2] = {(uint64_t)p.N * ((p.split && esz == 2) ? 3 : 1), (uint64_t)p.M};
    uint64_t strides[1] = {(uint64_t)p.ldo * esz};
    uint32_t box[2] = {(uint32_t)(128 / esz), 16};  // one 16-row group of a warp's accumulator fragments
    if (make_tmap(&tmC, p.out, esz == 4 ? 1 : esz == 1 ? 2 : 0, 2, dims, strides, box)) return 1;
  }
  STA_REQUIRE(tma || ksplit == 1, "split-K needs the TMA epilogue");

  int rc = -1;
  if (wide) {
    if (g.epi == EPI_GELU) rc = launch_wide<EPI_GELU>(tmA, tmB, tmC, p, num_tiles, stream);
    else if (g.epi == EPI_F32) rc = launch_wide<EPI_F32>(tmA, tmB, tmC, p, num_tiles, stream);
    else if (g.epi == EPI_ROPE) rc = launch_wide<EPI_ROPE>(tmA, tmB, tmC, p, num_tiles, stream);
    else rc = launch_wide<EPI_BF16>(tmA, tmB, tmC, p, num_tiles, stream);
  }
#define STA_GEMM_CASE(AM_, EP_, TMA_) \
  if (rc < 0 && g.amode == AM_ && g.epi == EP_ && tma == TMA_) rc = launch_inst<AM_, EP_, TMA_>(tmA, tmB, tmC, p, num_tiles, stream);

  STA_GEMM_CASE(A_LINEAR, EPI_GELU, true)
  STA_GEMM_CASE(A_LINEAR, EPI_F32, true)
  STA_GEMM_CASE(A_LINEAR, EPI_ROPE, true)
  STA_GEMM_CASE(A_LINEAR, EPI_BF16, true)
  STA_GEMM_CASE(A_LINEAR, EPI_BF16, false)
  STA_GEMM_CASE(A_LINEAR, EPI_F32, false)
  STA_GEMM_CASE(A_LINEAR, EPI_PIXSHUF, false)
  STA_GEMM_CASE(A_CONV3, EPI_BF16, false)
  STA_GEMM_CASE(A_CONV3, EPI_HEAD, false)
  STA_GEMM_CASE(A_FP8, EPI_F32, true)
  STA_GEMM_CASE(A_FP8, EPI_ROPE, true)
  STA_GEMM_CASE(A_FP8, EPI_GELU_FP8, true)
#undef STA_GEMM_CASE
  if (rc == 0 && ksplit > 1) {
    const long long total = static_cast<long long>(p.M) * (p.N / 4);
    int blocks = static_cast<int>((total + 255) / 256);
    if (blocks > 4 * num_sms()) blocks = 4 * num_sms();
    STA_CHECK_CUDA(launch_pdl(splitk_reduce_kernel, dim3(blocks), dim3(256), 0, stream, 1,
                              static_cast<const float*>(g.splitk_ws), static_cast<long long>(p.split_rows) * p.N, ksplit,
                              final_bias, final_out, p.ldo, p.M, p.N, final_accumulate));
  }
  if (rc >= 0) return rc;
  set_last_error("launch_gemm: unsupported (amode, epilogue) combination");
  return 2;
}

}  // namespace sta
