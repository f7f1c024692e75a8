// Persistent warp-specialised wgmma GEMM / implicit-GEMM 3x3 convolution for sm_90a.
//
//   D[M,N] = A[M,K] * W[N,K]^T  (bf16 operands, fp32 accumulation in registers)
//
// Roles: warpgroup 0 = TMA producer (warp 0 lane 0 issues the loads; the warpgroup drops to 40 registers), warpgroups 1
// and 2 = consumers (232 registers each) that ping-pong whole 128 x BN tiles: consumer g takes tiles g, g + 2, .. of
// the CTA's sequence, holds the tile's fp32 accumulators in registers (two m64n128k16 wgmmas per k16 step), and the two
// take turns on the tensor cores, so one runs its fused epilogue (straight from the wgmma fragments) while the other runs
// its mainloop.  The producer keeps a STAGES-deep operand ring filled in tile order.  Operand tiles are 128B-swizzled
// K-major [rows][64] boxes written by TMA; the 3x3 convolution loads one halo tile per channel chunk through a 4-D NHWC
// tensor map (out-of-bounds = zero padding) and feeds every filter tap from shifted views of it, so no im2col buffer
// exists.
//
// Reference ops covered (vista_slam/sta_model): nn.Linear in blocks/sta_blocks.py:67-70,
// 88-90,179-183; PatchEmbed conv sta_blocks.py:262 (after im2col); the DPT convs of
// heads/dpt_block.py:33-68,93-111,174-182,319-323,356-403.
#pragma once
#include "common.cuh"

namespace sta {

// A_CONV3: 3x3 convolution, halo-staged: ONE box of 18 x 10 pixels x 64 channels per channel chunk feeds all nine taps --
//          a tap is a row-shifted view of the staged tile (tile 16 rows x 8 pixels, descriptor base offset = the tap's
//          shift).  Shared-memory write traffic of the A operand is 22.5 KB per channel chunk instead of 9 x 16 KB with one
//          box per tap; the N = 128 head convolutions are bound by exactly that traffic.
// A_FP8:   linear layer with e4m3 operands (A [M][K] and W [N][K] bytes, K contiguous) and power-of-two block scales: one
//          per row and 128 columns of A (a_scale [M][K / 128]) and one per 128 x 128 block of W (w_scale [N / 128][K / 128]).
//          A 128-byte row holds 128 e4m3 values, so the TMA boxes, the swizzle and the ring are those of the bf16 kernel
//          with BK = 128.  Each 128-wide k-block accumulates in a fresh wgmma accumulator (four m64n128k32 MMAs per
//          64-row half) that is folded into the fp32 tile as acc = fma(blk, a_scale[row] * w_scale, acc).
enum AMode : int { A_LINEAR = 0, A_CONV3 = 1, A_FP8 = 2 };
enum Epi : int {
  EPI_BF16 = 0,     // out_bf16 = [relu](acc + bias [+ resid_bf16] [+ resid2_bf16]); optional relu copy in out2
  EPI_GELU = 1,     // out_bf16 = gelu_erf(acc + bias)
  EPI_F32 = 2,      // out_f32[row'] = acc + bias [+ resid_f32[row']]   (row' optionally skips one pose-token row per sample)
  EPI_ROPE = 3,     // out_bf16 = rope2d(acc + bias) on columns < rope_cols, plain on the rest
  EPI_PIXSHUF = 4,  // ConvTranspose2d(k = stride): scatter to the k x k sub-pixels, NHWC bf16
  EPI_HEAD = 5,     // relu(acc + bias) -> 1x1 conv (128 -> 4) -> pointmap/confidence post-process (fp32 out)
  EPI_GELU_FP8 = 6, // out_e4m3 = gelu_erf(acc + bias) / s, out_scale[row][n_tile] = s (one power-of-two scale per 128 columns)
};

struct GemmParams {
  int M, N, K;
  // A_CONV3 geometry (input and output NHWC, same H x W)
  int nimg, H, W, Cin, tiles_h, tiles_w;
  // epilogue
  const float* bias;
  void* out;
  long long ldo;  // output row stride in elements (also residual row stride)
  void* out2;
  const void* resid;
  const void* resid2;
  int relu_main;
  int rowmap_n;  // EPI_F32: if > 0, out row = (r / n) * (n + 1) + 1 + r % n
  // EPI_ROPE
  const float* rope_tab;  // [(pos + 1)][16] x (cos, sin)
  const int* pos;         // [M][2] (y, x)
  int rope_cols;
  int rope_max_pos;
  int rope_smem_rows;  // > 0: table rows for positions [-1, rope_smem_rows - 2] are staged in shared memory
  // EPI_PIXSHUF
  int ps_k, ps_cout, ps_h, ps_w;
  // EPI_HEAD
  const float* head_w;  // [128][4]
  const float* head_b;  // [4]
  float* pts3d;         // [pixels][3]
  float* conf;          // [pixels]
  // split-K (TMA epilogue, EPI_F32 only): a work item is (m, n, ks); split ks accumulates k-blocks
  // [ks * nkb / ksplit, (ks + 1) * nkb / ksplit) and stores its fp32 partial tile at output row ks * split_rows + row
  int ksplit;      // >= 1
  int split_rows;  // rows of one partial slice (multiple of 128)
  int c_reduce;         // TMA epilogue, EPI_F32: out += result (in-place fp32 residual stream) via bulk reduce-add
  // split-precision parity mode (common.cuh): the operands are already (hi | lo | hi) x (hi | hi | lo) expanded along K
  // (K here is the physical 3K); bf16 outputs / bf16 skip tensors use the (hi | lo | hi) row layout with logical
  // width N (ldo = 3N).  fp32 outputs are unaffected.
  int split;
  // A_FP8 operand scales (see AMode) and the EPI_GELU_FP8 output scales [M][N / 128]
  const float* a_scale;
  const float* w_scale;
  float* out_scale;
};

// TMA = true: the epilogue writes through per-warp swizzled boxes + TMA tensor stores (epilogue_tile_tma), else the
// coalesced per-warp path (epilogue_tile).
// A_CONV3: pixels per staged halo row.  10 = the 8-pixel tile plus its two halo columns (dense box, 8-row descriptor groups
// 1280 B apart -- groups then start at any 128-byte multiple, which the absolute-address swizzle permits).
constexpr int kHaloPitch = 10;
constexpr int kRopeLd = 36;  // floats per staged sin/cos table row (32 + 4 pad: conflict-free row-per-lane reads)
template <int AMODE, int EPI, bool TMA>
struct GemmCfg {
  static constexpr bool CONV = (AMODE == A_CONV3);
  static constexpr bool FP8 = (AMODE == A_FP8);
  static constexpr int BM = 128;
  static constexpr int BN = 128;  // two m64n128k16 wgmmas per k16 step cover a consumer warpgroup's whole tile
  static constexpr int ESZ = FP8 ? 1 : 2;  // operand bytes
  static constexpr int BK = 128 / ESZ;     // one 128-byte K-major row per k-block
  static constexpr uint32_t A_BYTES = BM * BK * ESZ;
  static constexpr uint32_t B_BYTES = BN * BK * ESZ;
  static constexpr uint32_t BAR_BYTES = 256;
  static constexpr int EPI_WARPS = 8;  // the two consumer warpgroups
  // Register split (setmaxnreg): the producer warpgroup only issues TMA loads; a consumer thread holds a 128 x 128 fp32
  // accumulator tile's 128 values plus the epilogue's working set.
  static constexpr uint32_t PRODUCER_REGS = 40;
  static constexpr uint32_t CONSUMER_REGS = 232;
  static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS <= 64 * 1024, "register file");
  // Per-warp epilogue staging.  TMA-store epilogue: two 16-row x 128-byte SWIZZLE_128B boxes, alternated so that one
  // is written while the bulk store of the other reads it.  Coalesced epilogue: one fp32 box of the warp's 32 accumulator
  // rows x 32 columns (box_off: 16-byte chunks XOR-swizzled by row, so fragment writes and row reads are conflict-free).
  static constexpr uint32_t TMA_BOX_BYTES = 16 * 128;
  static constexpr uint32_t STG_WARP_BYTES = TMA ? 2 * TMA_BOX_BYTES : 32 * 32 * sizeof(float);
  static constexpr uint32_t STG_BYTES = EPI_WARPS * STG_WARP_BYTES;
  static constexpr int ROPE_SMEM_ROWS = 64;  // positions -1 .. 62
  static constexpr uint32_t ROPE_SMEM_BYTES = (EPI == EPI_ROPE) ? ROPE_SMEM_ROWS * kRopeLd * sizeof(float) : 0;
  static constexpr uint32_t MAX_SMEM = 227 * 1024;
  // convolution: the ring holds B tiles only; three 18 x 10 x 64-channel halo input tiles besides it
  static constexpr uint32_t HALO_TX_BYTES = 18 * kHaloPitch * 128;                 // bytes one box delivers
  static constexpr uint32_t HALO_BYTES = (HALO_TX_BYTES + 1023u) & ~1023u;        // stage stride (swizzle-pattern aligned)
  static constexpr int HALO_STAGES = 3;
  static constexpr uint32_t HALO_TOTAL = CONV ? HALO_STAGES * HALO_BYTES : 0;
  static constexpr uint32_t STAGE_BYTES = CONV ? B_BYTES : A_BYTES + B_BYTES;
  static constexpr int STAGES_FIT = (MAX_SMEM - BAR_BYTES - STG_BYTES - ROPE_SMEM_BYTES - HALO_TOTAL) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > 8 ? 8 : STAGES_FIT;
  // layout: operand ring | halo tiles | staging (1024-byte aligned) | barriers | RoPE
  static constexpr uint32_t OFF_HALO = STAGES * STAGE_BYTES;
  static constexpr uint32_t OFF_STG = OFF_HALO + HALO_TOTAL;
  static constexpr uint32_t OFF_BAR = OFF_STG + STG_BYTES;
  static constexpr uint32_t OFF_ROPE = OFF_BAR + BAR_BYTES;
  static constexpr uint32_t SMEM_BYTES = OFF_ROPE + ROPE_SMEM_BYTES;
  static constexpr int THREADS = 128 + 32 * EPI_WARPS;
  static constexpr int EPI_THREADS = 32 * EPI_WARPS;
  static_assert(STAGES <= 8 && STAGES >= 3, "barrier area holds at most 8 stages");
  static_assert(OFF_STG % 1024 == 0 && OFF_HALO % 1024 == 0 && STG_WARP_BYTES % 16 == 0, "staging alignment");
  static_assert(!TMA || STG_WARP_BYTES % 1024 == 0, "SWIZZLE_128B boxes are 1024-byte aligned");
  static_assert(SMEM_BYTES <= MAX_SMEM, "shared memory");
};

// ---------------------------------------------------------------------------
// Accumulator fragments.  A consumer warpgroup holds its 128 x 128 tile as acc[h][64]: acc[h] is the m64n128 wgmma
// fragment of tile rows [64 h, 64 h + 64).  Warp wq (of the warpgroup), lane = 4 r + t holds, in acc[h][4 j + 2 half + e],
// row 64 h + 16 wq + 8 half + r, column 8 j + 2 t + e (j = 0..15).  So a thread holds rows r, r + 8, r + 64, r + 72 of
// its warp's 16-row groups, and the four lanes of a quad hold all 128 columns of those rows.
// ---------------------------------------------------------------------------

template <int AMODE>
__device__ __forceinline__ void tile_row(const GemmParams& p, int m_tile, int r_local, long long& orow, bool& valid) {
  if constexpr (AMODE == A_CONV3) {  // 16 rows x 8 pixels per 128-row tile
    const int tpi = p.tiles_h * p.tiles_w;
    const int n = m_tile / tpi;
    const int t = m_tile - n * tpi;
    const int th = t / p.tiles_w;
    const int tw = t - th * p.tiles_w;
    const int h = th * 16 + (r_local >> 3);
    const int w = tw * 8 + (r_local & 7);
    valid = (h < p.H) && (w < p.W) && (n < p.nimg);
    orow = (static_cast<long long>(n) * p.H + h) * p.W + w;
  } else {
    const int r = m_tile * 128 + r_local;
    valid = r < p.M;
    orow = r;
  }
}

__device__ __forceinline__ uint2 pack4_bf16(const float4& v) {
  return make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
}
__device__ __forceinline__ void add_bf16x4(float4& v, uint2 q) {
  v.x += bf16_lo(q.x); v.y += bf16_hi(q.x); v.z += bf16_lo(q.y); v.w += bf16_hi(q.y);
}
// bf16 store of 4 values at p; in split mode also the residual part at p + w and the second hi copy at p + 2w
__device__ __forceinline__ void store4_bf16(__nv_bfloat16* p, const float4& v, int split, long long w) {
  const uint2 hi = pack4_bf16(v);
  *reinterpret_cast<uint2*>(p) = hi;
  if (split) {
    *reinterpret_cast<uint2*>(p + w) = make_uint2(pack_bf16x2_resid(v.x, v.y), pack_bf16x2_resid(v.z, v.w));
    *reinterpret_cast<uint2*>(p + 2 * w) = hi;
  }
}

// ---------------------------------------------------------------------------
// Coalesced epilogue of one warp's 32 accumulator rows (all 128 columns of the tile), run straight from the fragments.
//
// Box row rho (0..31) of the per-warp fp32 box is tile row 16 wq + rho (rho < 16) or 64 + 16 wq + rho - 16.  Each 32-column
// chunk is written into the box from the fragments and read back in a COALESCED mapping -- lane -> (box row
// 4*it + lane/8, 4 columns at (lane%8)*4) -- in which bias, residuals, activation and the global stores happen: a warp-wide
// access covers 4 rows x 128 contiguous bytes (fp32) or 4 rows x 64 bytes (bf16).
// ---------------------------------------------------------------------------
__device__ __forceinline__ int box_row_to_tile_row(int wq, int rho) { return 16 * wq + rho + 48 * (rho >> 4); }

// float offset of (row, col) in the per-warp [32][32] fp32 box: 16-byte chunk col / 4 of a row lives at (col / 4) ^ (row & 7)
__device__ __forceinline__ int box_off(int row, int col) { return row * 32 + ((((col >> 2) ^ row) & 7) << 2) + (col & 3); }

// fragments of 32-column chunk c -> the per-warp box
__device__ __forceinline__ void stage_chunk(float* box, const float (&acc)[2][64], int c) {
  const int lane = threadIdx.x & 31;
  const int r = lane >> 2, t = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int half = 0; half < 2; ++half)
#pragma unroll
      for (int jl = 0; jl < 4; ++jl) {
        const int i = 4 * (4 * c + jl) + 2 * half;
        *reinterpret_cast<float2*>(box + box_off(16 * h + 8 * half + r, 8 * jl + 2 * t)) = make_float2(acc[h][i], acc[h][i + 1]);
      }
}

template <int AMODE, int EPI>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, const float (&acc)[2][64], int m_tile, int n_tile,
                                              int wq, float* box) {
  using Cfg = GemmCfg<AMODE, EPI, false>;
  constexpr int BN = Cfg::BN;
  constexpr int NCH = BN / 32;  // 32-column chunks
  const int lane = threadIdx.x & 31;
  const int colbase = n_tile * BN;

  if constexpr (EPI == EPI_HEAD) {
    // head.2 epilogue: ReLU -> head.4 (1x1, 128 -> 4) -> postprocess (dpt_block.py:319-323,
    // postprocess.py:10-62).  Row mapping: lane = box row, so each thread walks the 128 channels of one pixel in order,
    // with columns [0, 64) and [64, 128) summed in two chains that are added at the end.  Nothing but 16 bytes per
    // pixel is written.
    long long orow;
    bool valid;
    tile_row<AMODE>(p, m_tile, box_row_to_tile_row(wq, lane), orow, valid);
    float psum[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      __syncwarp();  // the previous chunk's reads of the box are done
      stage_chunk(box, acc, c);
      __syncwarp();
      const int col = colbase + 32 * c;
      const int part = c / (NCH / 2);
      const float4* wp = reinterpret_cast<const float4*>(p.head_w) + col;
#pragma unroll 1
      for (int i4 = 0; i4 < 8; ++i4) {
        const float4 a = *reinterpret_cast<const float4*>(box + box_off(lane, 4 * i4));
        const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int i = 4 * i4 + e;
          float v = fmaxf(av[e] + __ldg(p.bias + col + i), 0.0f);
          float4 w4 = __ldg(wp + i);
          psum[part][0] = fmaf(v, w4.x, psum[part][0]);
          psum[part][1] = fmaf(v, w4.y, psum[part][1]);
          psum[part][2] = fmaf(v, w4.z, psum[part][2]);
          psum[part][3] = fmaf(v, w4.w, psum[part][3]);
        }
      }
    }
    __syncwarp();
    const float x = psum[0][0] + psum[1][0] + __ldg(p.head_b + 0);
    const float y = psum[0][1] + psum[1][1] + __ldg(p.head_b + 1);
    const float z = psum[0][2] + psum[1][2] + __ldg(p.head_b + 2);
    const float cf = psum[0][3] + psum[1][3] + __ldg(p.head_b + 3);
    if (valid) {
      const float d = sqrtf(x * x + y * y + z * z);
      const float dc = fmaxf(d, 1e-8f);
      const float e = expm1f(d);
      p.pts3d[orow * 3 + 0] = (x / dc) * e;
      p.pts3d[orow * 3 + 1] = (y / dc) * e;
      p.pts3d[orow * 3 + 2] = (z / dc) * e;
      p.conf[orow] = 1.0f + expf(cf);
    }
    return;
  } else {
    // ---- coalesced mapping bookkeeping: this lane touches box rows 4*it + (lane>>3), it = 0..7 ----
    const int crow = lane >> 3;
    const int cc = (lane & 7) * 4;  // first of this lane's 4 columns inside the 32-column chunk
    long long orow_c[8];
    uint32_t vmask = 0;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      bool v;
      tile_row<AMODE>(p, m_tile, box_row_to_tile_row(wq, it * 4 + crow), orow_c[it], v);
      vmask |= (v ? 1u : 0u) << it;
      if constexpr (EPI == EPI_F32) {
        if (p.rowmap_n > 0) {
          const long long s = orow_c[it] / p.rowmap_n;
          orow_c[it] = s * (p.rowmap_n + 1) + 1 + (orow_c[it] - s * p.rowmap_n);
        }
      }
      if constexpr (EPI == EPI_PIXSHUF) {
        // token -> (n, h, w); keep ((n*ps_h + h)*k) * (ps_w*k) + w*k  (pixel index of sub-pixel (0,0))
        const int hw = p.ps_h * p.ps_w;
        const int n = static_cast<int>(orow_c[it] / hw);
        const int rem = static_cast<int>(orow_c[it] - static_cast<long long>(n) * hw);
        const int h = rem / p.ps_w;
        const int w = rem - h * p.ps_w;
        orow_c[it] = (static_cast<long long>(n) * p.ps_h + h) * p.ps_k * (p.ps_w * p.ps_k) + w * p.ps_k;
      }
    }

    // flush one staged 32-column chunk (global columns [col, col+32)) in the coalesced mapping
    auto flush = [&](int col, const float* stg) {
      float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
      long long pix_off = 0;
      int co = 0;
      if constexpr (EPI == EPI_PIXSHUF) {
        const int kk = col / p.ps_cout;
        co = col - kk * p.ps_cout;
        const int kh = kk / p.ps_k;
        const int kw = kk - kh * p.ps_k;
        pix_off = static_cast<long long>(kh) * (p.ps_w * p.ps_k) + kw;
        b4 = __ldg(reinterpret_cast<const float4*>(p.bias + co + cc));
      } else {
        if (p.bias) b4 = __ldg(reinterpret_cast<const float4*>(p.bias + col + cc));
      }
      // Residual loads are issued ahead of the stores, four rows at a time: the in-place residual stream
      // (resid == out) would otherwise force load -> store -> load ordering (possible aliasing) and serialise
      // ~1 us DRAM round trips.
#pragma unroll
      for (int hb = 0; hb < 2; ++hb) {
        [[maybe_unused]] float4 rf[4];
        [[maybe_unused]] uint2 ra[4], rb[4];
        if constexpr (EPI == EPI_F32) {
          if (p.resid) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const int it = hb * 4 + k;
              rf[k] = ((vmask >> it) & 1u)
                          ? *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.resid) +
                                                             orow_c[it] * p.ldo + col + cc)
                          : make_float4(0.f, 0.f, 0.f, 0.f);
            }
          }
        }
        if constexpr (EPI == EPI_BF16) {
          if (p.resid) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const int it = hb * 4 + k;
              ra[k] = ((vmask >> it) & 1u)
                          ? *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(p.resid) +
                                                            orow_c[it] * p.ldo + col + cc)
                          : make_uint2(0u, 0u);
            }
          }
          if (p.resid2) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const int it = hb * 4 + k;
              rb[k] = ((vmask >> it) & 1u)
                          ? *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(p.resid2) +
                                                            orow_c[it] * p.ldo + col + cc)
                          : make_uint2(0u, 0u);
            }
          }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          // straight-line body: only the global loads / stores are predicated on row validity, so the
          // compiler can interleave the four rows of a batch
          const int it = hb * 4 + k;
          const bool ok = (vmask >> it) & 1u;
          float4 v = *reinterpret_cast<const float4*>(stg + box_off(it * 4 + crow, cc));
          v.x += b4.x; v.y += b4.y; v.z += b4.z; v.w += b4.w;
          if constexpr (EPI == EPI_F32) {
            float* op = reinterpret_cast<float*>(p.out) + orow_c[it] * p.ldo + col + cc;
            if (p.resid) { v.x += rf[k].x; v.y += rf[k].y; v.z += rf[k].z; v.w += rf[k].w; }
            if (ok) *reinterpret_cast<float4*>(op) = v;
          } else if constexpr (EPI == EPI_PIXSHUF) {
            __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(p.out) +
                                (orow_c[it] + pix_off) * (p.split ? 3 * p.ps_cout : p.ps_cout) + co + cc;
            if (ok) store4_bf16(op, v, p.split, p.ps_cout);
          } else {  // EPI_BF16
            const long long off = orow_c[it] * p.ldo + col + cc;
            if (p.resid) {
              add_bf16x4(v, ra[k]);
              if (p.split && ok)  // residual (lo) part of the skip tensor
                add_bf16x4(v, *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(p.resid) + off + p.N));
            }
            if (p.resid2) {
              add_bf16x4(v, rb[k]);
              if (p.split && ok)
                add_bf16x4(v, *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(p.resid2) + off + p.N));
            }
            if (p.relu_main) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
            if (p.out && ok) store4_bf16(reinterpret_cast<__nv_bfloat16*>(p.out) + off, v, p.split, p.N);
            if (p.out2 && ok) {
              v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
              store4_bf16(reinterpret_cast<__nv_bfloat16*>(p.out2) + off, v, p.split, p.N);
            }
          }
        }
      }
    };

    // L2 prefetch of the residual rows this lane will add (fp32 residual stream / bf16 skip tensors)
    if constexpr (EPI == EPI_F32 || EPI == EPI_BF16) {
      if (p.resid) {
        constexpr int esz = (EPI == EPI_F32) ? 4 : 2;
#pragma unroll
        for (int it = 0; it < 8; ++it) {
          if ((vmask >> it) & 1u) {
#pragma unroll
            for (int c = 0; c < NCH; ++c) {
              if (colbase + 32 * c < p.N) {
                const char* a = reinterpret_cast<const char*>(p.resid) + (orow_c[it] * p.ldo + colbase + 32 * c + cc) * esz;
                asm volatile("prefetch.global.L2 [%0];" ::"l"(a));
                if constexpr (EPI == EPI_BF16) {
                  if (p.resid2) {
                    const char* a2 = reinterpret_cast<const char*>(p.resid2) + (orow_c[it] * p.ldo + colbase + 32 * c + cc) * esz;
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(a2));
                  }
                }
              }
            }
          }
        }
      }
    }
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      if (colbase + 32 * c < p.N) {  // warp-uniform
        __syncwarp();  // the previous chunk's reads of the box are done
        stage_chunk(box, acc, c);
        __syncwarp();
        flush(colbase + 32 * c, box);
      }
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------
// TMA-store epilogue for the linear layers with N % 128 == 0 (EPI_BF16 / EPI_GELU / EPI_ROPE / EPI_F32), run in
// registers on the wgmma fragments.
//
// Bias, GELU, ReLU and the RoPE rotation work on the fragments in place: a RoPE pair (i, i + 16) of a 32-column half-head
// is fragment columns 8 j + 2 t and 8 (j + 2) + 2 t, both in the same thread.  The results go to a per-warp 16-row x
// 128-byte shared-memory box in the SWIZZLE_128B layout (a 16-byte chunk is one fragment column group j, so the stores are
// conflict-free) and leave with ONE bulk tensor store per box issued by lane 0: no per-lane global stores, rows >= M are
// clipped by the tensor map, and the in-place fp32 residual stream (x += proj(..)) becomes a bulk reduce-add performed by
// the L2, so the epilogue never loads the residual.  The warp's two boxes alternate (ubuf counts the boxes written).
// ---------------------------------------------------------------------------
template <int EPI>
__device__ __forceinline__ void epilogue_tile_tma(const GemmParams& p, const CUtensorMap* tmC, float (&acc)[2][64],
                                                  int m_tile, int n_tile, int row_off, int wq, uint8_t* stg,
                                                  const float* rope_s, uint32_t& ubuf) {
  using Cfg = GemmCfg<A_LINEAR, EPI, true>;
  constexpr bool OUT_F32 = (EPI == EPI_F32);
  const int lane = threadIdx.x & 31;
  const int r = lane >> 2, t = lane & 3;
  const int col0 = n_tile * Cfg::BN;
  const int row0 = m_tile * 128 + 16 * wq;  // first row of this warp's 16-row group h = 0 (token index); h = 1 is + 64

  // bias (adding 0 without one, as the accumulators always went through the same add)
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float2 b = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 8 * j + 2 * t)) : make_float2(0.f, 0.f);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      acc[h][4 * j] += b.x; acc[h][4 * j + 1] += b.y; acc[h][4 * j + 2] += b.x; acc[h][4 * j + 3] += b.y;
    }
  }
  if constexpr (EPI == EPI_GELU || EPI == EPI_GELU_FP8) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[h][i] = gelu_erf(acc[h][i]);
  }
  if constexpr (EPI == EPI_BF16) {
    if (p.relu_main) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[h][i] = fmaxf(acc[h][i], 0.0f);
    }
  }
  [[maybe_unused]] uint32_t pyx[2][2];  // [h][half]: (pos_y + 1) | (pos_x + 1) << 16 of this thread's four token rows
  [[maybe_unused]] bool staged = true;
  if constexpr (EPI == EPI_ROPE) {
    // 2-D RoPE (pos_embed/pos_embed.py:149-185, curope/kernels.cu:17-82): a 32-column chunk q is one half of a 64-wide
    // head -- the y-half (rotated by pos_y, q even) or the x-half (pos_x, q odd); inside it the pairs are (i, i + 16).
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int row = row0 + 64 * h + 8 * half + r;
        pyx[h][half] = 0x00010001u;
        if (row < p.M) {
          const int2 pp = *reinterpret_cast<const int2*>(p.pos + 2 * static_cast<long long>(row));
          if (pp.x < -1 || pp.x > p.rope_max_pos || pp.y < -1 || pp.y > p.rope_max_pos)
            __trap();  // token position outside the RoPE table (no printf: see mbar_wait)
          pyx[h][half] = static_cast<uint32_t>(pp.x + 1) | (static_cast<uint32_t>(pp.y + 1) << 16);
        }
      }
    // does the shared-memory table hold every position of the warp?
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int half = 0; half < 2; ++half)
        staged = staged && static_cast<int>(max(pyx[h][half] & 0xFFFFu, pyx[h][half] >> 16)) < p.rope_smem_rows;
    staged = __all_sync(0xFFFFFFFFu, staged);
  }
  // RoPE of 32-column chunk q in the rows of acc[h]; run just before the chunk is written out, so the rotated values
  // die right away.  The table rows come from shared memory when every position of the warp is staged there, else all
  // from global memory (one address space per rotation keeps it within the register budget).
  auto rope_chunk = [&](int h, int q) {
    if constexpr (EPI == EPI_ROPE) {
      if (col0 + 32 * q >= p.rope_cols) return;  // warp-uniform: the V columns are not rotated
      auto rotate = [&](auto table_row) {
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int ps = static_cast<int>((q & 1) ? pyx[h][half] >> 16 : pyx[h][half] & 0xFFFFu);
          const float4* tb = table_row(ps);
#pragma unroll
          for (int jj = 0; jj < 2; ++jj) {
            const float4 tt = tb[4 * jj + t];  // (cos f, sin f, cos f+1, sin f+1), f = 8 jj + 2 t
            const int ia = 4 * (4 * q + jj) + 2 * half;  // columns 8 jj + 2 t + {0, 1} of the half-head
            const int ib = ia + 8;                       // ... + 16
            const float a0 = acc[h][ia], b0 = acc[h][ib], a1 = acc[h][ia + 1], b1 = acc[h][ib + 1];
            acc[h][ia] = fmaf(-b0, tt.y, a0 * tt.x);
            acc[h][ib] = fmaf(a0, tt.y, b0 * tt.x);
            acc[h][ia + 1] = fmaf(-b1, tt.w, a1 * tt.z);
            acc[h][ib + 1] = fmaf(a1, tt.w, b1 * tt.z);
          }
        }
      };
      if (staged) rotate([&](int ps) { return reinterpret_cast<const float4*>(rope_s + ps * kRopeLd); });
      else rotate([&](int ps) { return reinterpret_cast<const float4*>(p.rope_tab + static_cast<long long>(ps) * 32); });
    }
  };

  // ---- registers -> swizzled boxes -> bulk tensor stores ----
  // A box row is 128 bytes: 64 bf16 columns (fragment groups j = 8 c .. 8 c + 7) or 32 fp32 columns (j = 4 c .. 4 c + 3).
  // Split-precision parity mode, bf16 outputs: hi = bf16(v) is stored at columns [col, ..) and [2N + col, ..), and
  // lo = bf16(v - hi) from the same registers at [N + col, ..).
  constexpr int NCH = OUT_F32 ? 4 : 2;
  const uint32_t sb = smem_u32(stg);
  const uint32_t sx = r;  // 128B swizzle: 16-byte chunk k of box row R lives at k ^ (R & 7), and R & 7 = r
  auto next_box = [&]() -> uint32_t {
    if (lane == 0) tma_store_wait_read1();  // the store that read this box two boxes ago is done with it
    __syncwarp();
    return sb + (ubuf++ & 1u) * Cfg::TMA_BOX_BYTES;
  };
  auto issue = [&](uint32_t box, int col, int row, bool second_copy) {
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
      const void* src = stg + (box - sb);
      if constexpr (OUT_F32) {
        if (p.c_reduce) tma_reduce_add_2d(tmC, src, col, row);
        else tma_store_2d(tmC, src, col, row);
      } else {
        tma_store_2d(tmC, src, col, row);
        if (second_copy) tma_store_2d(tmC, src, col + 2 * p.N, row);
      }
      tma_store_commit();
    }
  };
  if constexpr (EPI == EPI_GELU_FP8) {
    // One 16-row x 128-byte box per 64-row half holds the tile's 128 e4m3 columns.  A row's 128 columns sit in one quad,
    // so its amax takes two shuffles; lane t = 0 of the quad writes the row's scale.  Column 8 j + 2 t of box row R is
    // byte 8 (j & 1) + 2 t of 16-byte chunk (j >> 1) ^ (R & 7).
    const int nsb = p.N / 128;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t box = next_box();
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        float am = 0.0f;
#pragma unroll
        for (int j = 0; j < 16; ++j)
          am = fmaxf(am, fmaxf(fabsf(acc[h][4 * j + 2 * half]), fabsf(acc[h][4 * j + 2 * half + 1])));
        am = fmaxf(am, __shfl_xor_sync(0xFFFFFFFFu, am, 1));
        am = fmaxf(am, __shfl_xor_sync(0xFFFFFFFFu, am, 2));
        float s, inv;
        fp8_scale(am, s, inv);
        const int row = row0 + 64 * h + 8 * half + r;
        if (t == 0 && row < p.M) p.out_scale[static_cast<long long>(row) * nsb + n_tile] = s;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const uint16_t q = cvt_e4m3x2(acc[h][4 * j + 2 * half] * inv, acc[h][4 * j + 2 * half + 1] * inv);
          asm volatile("st.shared.b16 [%0], %1;" ::"r"(box + (8 * half + r) * 128 + (((j >> 1) ^ sx) << 4) + 8 * (j & 1) + 2 * t),
                       "h"(q)
                       : "memory");
        }
      }
      issue(box, col0, row0 + 64 * h + row_off, false);
    }
  } else {
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + 64 * h + row_off;
      if constexpr (OUT_F32) {
        const uint32_t box = next_box();
#pragma unroll
        for (int half = 0; half < 2; ++half)
#pragma unroll
          for (int jl = 0; jl < 4; ++jl) {
            const int i = 4 * (4 * c + jl) + 2 * half;
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(box + (8 * half + r) * 128 +
                                                                   (((2 * jl + (t >> 1)) ^ sx) << 4) + (t & 1) * 8),
                         "f"(acc[h][i]), "f"(acc[h][i + 1])
                         : "memory");
          }
        issue(box, col0 + 32 * c, row, false);
      } else {
        const int npass = p.split ? 2 : 1;
#pragma unroll 1
        for (int pass = 0; pass < npass; ++pass) {
          if (pass == 0) {
            rope_chunk(h, 2 * c);
            rope_chunk(h, 2 * c + 1);
          }
          const uint32_t box = next_box();
#pragma unroll
          for (int half = 0; half < 2; ++half)
#pragma unroll
            for (int jl = 0; jl < 8; ++jl) {
              const int i = 4 * (8 * c + jl) + 2 * half;
              const uint32_t v = pass ? pack_bf16x2_resid(acc[h][i], acc[h][i + 1]) : pack_bf16x2(acc[h][i], acc[h][i + 1]);
              asm volatile("st.shared.b32 [%0], %1;" ::"r"(box + (8 * half + r) * 128 + ((jl ^ sx) << 4) + 4 * t), "r"(v)
                           : "memory");
            }
          issue(box, col0 + 64 * c + pass * p.N, row, p.split && pass == 0);
        }
      }
    }
  }
  }
}

template <int AMODE, int EPI, bool TMA>
__global__ void __launch_bounds__(GemmCfg<AMODE, EPI, TMA>::THREADS, 1)
gemm_wg_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmC, const GemmParams p) {
  using Cfg = GemmCfg<AMODE, EPI, TMA>;
  constexpr bool CONV = Cfg::CONV;
  static_assert(!TMA || (AMODE == A_LINEAR && (EPI == EPI_BF16 || EPI == EPI_GELU || EPI == EPI_F32 || EPI == EPI_ROPE)) ||
                    (AMODE == A_FP8 && (EPI == EPI_F32 || EPI == EPI_ROPE || EPI == EPI_GELU_FP8)),
                "TMA-store epilogue: linear layers only");
  static_assert(AMODE != A_FP8 || TMA, "e4m3 operands: TMA-store epilogues only");
  static_assert(TMA || EPI == EPI_BF16 || EPI == EPI_F32 || EPI == EPI_PIXSHUF || EPI == EPI_HEAD,
                "GELU and RoPE have the TMA-store epilogue only");
  constexpr int BN = Cfg::BN;
  constexpr int STAGES = Cfg::STAGES;
  constexpr uint32_t A_BYTES = Cfg::A_BYTES;
  constexpr uint32_t B_BYTES = Cfg::B_BYTES;
  constexpr uint32_t kOrderBar = 1;  // named barriers 1, 2: "consumer warpgroup 0 / 1 may issue its mainloop"

  extern __shared__ __align__(1024) uint8_t smem[];
  [[maybe_unused]] uint8_t* sA = smem;
  uint8_t* sB = smem + (CONV ? 0u : STAGES * A_BYTES);
  [[maybe_unused]] uint8_t* sH = smem + Cfg::OFF_HALO;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;
  [[maybe_unused]] uint64_t* hfull = bars + 2 * STAGES;  // halo tiles (A_CONV3)
  [[maybe_unused]] uint64_t* hempty = hfull + Cfg::HALO_STAGES;
  static_assert((2 * STAGES + 2 * Cfg::HALO_STAGES) * 8 <= Cfg::BAR_BYTES, "barrier area");
  uint8_t* stg_all = smem + Cfg::OFF_STG;
  [[maybe_unused]] float* rope_s = reinterpret_cast<float*>(smem + Cfg::OFF_ROPE);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int m_tiles = CONV ? p.nimg * p.tiles_h * p.tiles_w : (p.M + 127) / 128;
  const int n_tiles = (p.N + BN - 1) / BN;
  const int ksplit = TMA ? p.ksplit : 1;
  const int num_tiles = m_tiles * n_tiles * ksplit;  // work items (m, n, ks), ks fastest
  const int cpb = CONV ? (p.Cin / 64) : 1;  // 64-channel chunks per filter tap
  const int nkb = CONV ? 9 * cpb : (p.K + Cfg::BK - 1) / Cfg::BK;

  if (threadIdx.x == 0) {
    if ((smem_u32(smem) & 1023u) != 0) device_fatal("dynamic shared memory is not 1024-byte aligned");
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);  // the producer's expect_tx arrival
      mbar_init(&empty[s], 4);  // one arrival per warp of the consumer warpgroup that read the stage
    }
    if constexpr (CONV) {
      for (int s = 0; s < Cfg::HALO_STAGES; ++s) {
        mbar_init(&hfull[s], 1);
        mbar_init(&hempty[s], 4);
      }
    }
    fence_mbar_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if constexpr (TMA) tma_prefetch_desc(&tmC);
  }
  if constexpr (EPI == EPI_ROPE) {
    // the sin/cos table is a constant of the library (not produced by the previous kernel): stage the rows for
    // small positions in shared memory before the PDL wait
    if (warp >= 4) {
      const int nfl = p.rope_smem_rows * 32;
      for (int i = (threadIdx.x - 128) * 4; i < nfl; i += Cfg::EPI_THREADS * 4)
        *reinterpret_cast<float4*>(rope_s + (i >> 5) * kRopeLd + (i & 31)) =
            __ldg(reinterpret_cast<const float4*>(p.rope_tab + i));
    }
  }
  __syncthreads();
  pdl_wait();               // previous kernel's outputs (A operand, residuals) are complete and visible
  pdl_launch_dependents();  // the next kernel may start its prologue

  if (warp < 4) {
    // ===================== TMA producer (warp 0, lane 0; warps 1-3 only give their registers away) =====================
    setmaxnreg_dec<Cfg::PRODUCER_REGS>();
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      [[maybe_unused]] int hstage = 0;
      [[maybe_unused]] uint32_t hphase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int ks = tile % ksplit, mn = tile / ksplit;
        const int m_tile = mn / n_tiles;
        const int n_tile = mn % n_tiles;
        const int kb0 = ks * nkb / ksplit, kb1 = (ks + 1) * nkb / ksplit;
        const int b_row0 = n_tile * BN;
        if constexpr (CONV) {
          const int tpi = p.tiles_h * p.tiles_w;
          const int cn = m_tile / tpi;
          const int t = m_tile - cn * tpi;
          const int th = t / p.tiles_w;
          const int ch0 = th * 16;
          const int cw0 = (t - th * p.tiles_w) * 8;
          // channel chunk outermost: one halo tile, then the nine taps' weight tiles
          for (int cc = 0; cc < cpb; ++cc) {
            mbar_wait(&hempty[hstage], hphase ^ 1);
            mbar_arrive_expect_tx(&hfull[hstage], Cfg::HALO_TX_BYTES);
            tma_load_4d(sH + hstage * Cfg::HALO_BYTES, &tmA, &hfull[hstage], cc * 64, cw0 - 1, ch0 - 1, cn);
            if (++hstage == Cfg::HALO_STAGES) { hstage = 0; hphase ^= 1; }
            for (int tap = 0; tap < 9; ++tap) {
              mbar_wait(&empty[stage], phase ^ 1);
              mbar_arrive_expect_tx(&full[stage], B_BYTES);
              tma_load_2d(sB + stage * B_BYTES, &tmB, &full[stage], (tap * cpb + cc) * 64, b_row0);
              if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
          }
        } else {
          for (int kb = kb0; kb < kb1; ++kb) {
            mbar_wait(&empty[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full[stage], A_BYTES + B_BYTES);
            tma_load_2d(sA + stage * A_BYTES, &tmA, &full[stage], kb * Cfg::BK, m_tile * 128);
            tma_load_2d(sB + stage * B_BYTES, &tmB, &full[stage], kb * Cfg::BK, b_row0);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    // ============ consumer warpgroups, ping-pong: whole tiles, mainloops in turn, epilogue under the other's mainloop ============
    // Warpgroup wg takes tiles j = wg, wg + 2, .. of this CTA's sequence.  The ring is filled in tile order, so a
    // warpgroup skips the stages of the other's tiles.  Turn-taking (two named barriers): before tile j > 0 wait for
    // the other warpgroup to have issued tile j - 1; after issuing the last k-block of tile j hand the turn over if
    // tile j + 1 exists -- so every wait meets exactly one arrival.
    setmaxnreg_inc<Cfg::CONSUMER_REGS>();
    const int wg = (warp - 4) >> 2;
    const int wq = warp & 3;  // warp inside the warpgroup: rows [16 wq, +16) of each 64-row half of the tile
    uint8_t* stg = stg_all + (warp - 4) * Cfg::STG_WARP_BYTES;
    [[maybe_unused]] uint32_t ubuf = 0;
    int kdone = 0;  // k-blocks (ring stages) of the CTA's earlier tiles
    [[maybe_unused]] int hdone = 0;  // halo tiles of the CTA's earlier tiles
    int j = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++j) {
      const int ks = tile % ksplit, mn = tile / ksplit;
      const int kb0 = ks * nkb / ksplit, kb1 = (ks + 1) * nkb / ksplit;
      if ((j & 1) != wg) {
        kdone += kb1 - kb0;
        hdone += cpb;
        continue;
      }
      const int m_tile = mn / n_tiles;
      const int n_tile = mn % n_tiles;
      int stage = kdone % STAGES;
      uint32_t phase = (kdone / STAGES) & 1;
      kdone += kb1 - kb0;
      [[maybe_unused]] int hstage = hdone % Cfg::HALO_STAGES;
      [[maybe_unused]] uint32_t hphase = (hdone / Cfg::HALO_STAGES) & 1;
      hdone += cpb;

      float acc[2][64];
#pragma unroll
      for (int i = 0; i < 64; ++i) { acc[0][i] = 0.0f; acc[1][i] = 0.0f; }
      if (j > 0) named_bar_sync(kOrderBar + wg, 256);
      // one k-block: four k16 steps, each two m64n128k16 wgmmas (tile rows 0-63 and 64-127); the previous k-block's
      // wgmma group may still run, its stage is released once this one is issued
      int prev = -1;
      auto kblock = [&](uint64_t adesc0, uint64_t adesc1, uint64_t bdesc) {
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_m64n128k16_ss(acc[0], adesc0 + 2 * k, bdesc + 2 * k, 1u);
          wgmma_m64n128k16_ss(acc[1], adesc1 + 2 * k, bdesc + 2 * k, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        fence_regs(acc[0]);
        fence_regs(acc[1]);
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      };
      // the other warpgroup may issue once this tile's last k-block is issued (not finished)
      auto hand_over = [&]() {
        if (tile + static_cast<int>(gridDim.x) < num_tiles) named_bar_arrive(kOrderBar + (wg ^ 1), 256);
      };
      if constexpr (Cfg::FP8) {
        // The two 64-row halves of a k-block run one after the other through one 64-register block accumulator (beside
        // the 128 tile accumulators); the scales are loaded before the stage wait and used after the MMAs.  The turn
        // passes once the wait on the tile's last stage is done (every stage of the tile is then filled, which is what
        // keeps the other warpgroup's parity waits within one ring round), so the other warpgroup's MMAs overlap this
        // one's last k-block and folds.
        const int nks = p.K / 128;
        const int r = lane >> 2;
        const int rbase = m_tile * 128 + 16 * wq + r;  // + 64 h + 8 half
        for (int kb = kb0; kb < kb1; ++kb) {
          float as[2][2];
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              const int row = rbase + 64 * h + 8 * half;
              as[h][half] = row < p.M ? __ldg(p.a_scale + static_cast<long long>(row) * nks + kb) : 0.0f;
            }
          const float wsc = __ldg(p.w_scale + n_tile * nks + kb);
          mbar_wait(&full[stage], phase);
          if (kb == kb1 - 1) hand_over();
          const uint32_t a = smem_u32(sA + stage * A_BYTES);
          const uint64_t bdesc = make_smem_desc_sw128(smem_u32(sB + stage * B_BYTES));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float blk[64];
            const uint64_t adesc = make_smem_desc_sw128(a + h * 64 * 128);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_m64n128k32_e4m3(blk, adesc + 2 * k, bdesc + 2 * k, k > 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(blk);
            const float s0 = as[h][0] * wsc, s1 = as[h][1] * wsc;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              acc[h][4 * j] = fmaf(blk[4 * j], s0, acc[h][4 * j]);
              acc[h][4 * j + 1] = fmaf(blk[4 * j + 1], s0, acc[h][4 * j + 1]);
              acc[h][4 * j + 2] = fmaf(blk[4 * j + 2], s1, acc[h][4 * j + 2]);
              acc[h][4 * j + 3] = fmaf(blk[4 * j + 3], s1, acc[h][4 * j + 3]);
            }
          }
          if (lane == 0) mbar_arrive(&empty[stage]);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      } else if constexpr (CONV) {
        for (int cc = 0; cc < cpb; ++cc) {
          mbar_wait(&hfull[hstage], hphase);
          // output pixel (y, x) of the 16 x 8 tile reads halo pixel (y + kh, x + kw); halo rows are kHaloPitch pixels.
          // Tile rows 0-63 are the output rows y = 0..7, tile rows 64-127 are y = 8..15 (8 halo rows further).
          const uint32_t hbase = smem_u32(sH + hstage * Cfg::HALO_BYTES);
          for (int tap = 0; tap < 9; ++tap) {
            mbar_wait(&full[stage], phase);
            const int kh = tap / 3, kw = tap - kh * 3;
            const uint32_t tb = hbase + (kh * kHaloPitch + kw) * 128;
            kblock(make_smem_desc_sw128_rows(tb, kHaloPitch * 128),
                   make_smem_desc_sw128_rows(tb + 8 * kHaloPitch * 128, kHaloPitch * 128),
                   make_smem_desc_sw128(smem_u32(sB + stage * B_BYTES)));
          }
          if (cc == cpb - 1) hand_over();
          wgmma_wait<0>();  // every read of this halo tile has completed
          fence_regs(acc[0]);
          fence_regs(acc[1]);
          if (lane == 0) mbar_arrive(&hempty[hstage]);
          if (++hstage == Cfg::HALO_STAGES) { hstage = 0; hphase ^= 1; }
        }
      } else {
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&full[stage], phase);
          const uint32_t a = smem_u32(sA + stage * A_BYTES);
          kblock(make_smem_desc_sw128(a), make_smem_desc_sw128(a + 64 * 128),
                 make_smem_desc_sw128(smem_u32(sB + stage * B_BYTES)));
        }
        hand_over();
      }
      wgmma_wait<0>();
      fence_regs(acc[0]);
      fence_regs(acc[1]);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);

      if constexpr (TMA) {
        epilogue_tile_tma<EPI>(p, &tmC, acc, m_tile, n_tile, ks * p.split_rows, wq, stg, rope_s, ubuf);
        // After the warpgroup's last tile: the bulk stores read this CTA's shared memory.  (Waiting here rather than
        // after the tile loop matters: with the wait after the loop, ptxas kept the consumer code inside the
        // 168-register launch budget instead of the setmaxnreg budget, and the RoPE epilogue spilled.)
        if (tile + 2 * static_cast<int>(gridDim.x) >= num_tiles && lane == 0) tma_store_wait_all();
      } else {
        epilogue_tile<AMODE, EPI>(p, acc, m_tile, n_tile, wq, reinterpret_cast<float*>(stg));
      }
    }
  }
}

// ---------------------------------------------------------------------------
// Wide linear GEMM: 128 x 256 tiles, both consumer warpgroups on the same tile.
//
// Warpgroup g computes tile rows [64 g, 64 g + 64) x 256 columns with one m64n256k16 wgmma per k16 step.  Against the
// 128 x 128 ping-pong kernel, a k16 step reads 2 x 2 KB of A and 8 KB of B from shared memory for 2 x 64 x 256 x 16 MACs
// (instead of 2 x 2 KB + 2 x 4 KB for two 64 x 128 halves of half the columns per warpgroup), and TMA writes 48 KB per
// k-block of 128 x 256 x 64 MACs instead of 32 KB per 128 x 128 x 64: the shared-memory traffic per MAC drops from about
// 160 to 128 bytes per clock at full tensor rate, the SM's shared-memory bandwidth.  The price is that the epilogue is no
// longer hidden behind the other warpgroup's mainloop; the producer keeps the ring filled meanwhile, so the next tile's
// first k-blocks are waiting when it ends.
//
// Fragment: warp wq of warpgroup g, lane = 4 r + t holds in acc[4 j + 2 half + e] tile row 64 g + 16 wq + 8 half + r,
// column 8 j + 2 t + e (j = 0..31).  Each output element sees the same k16 steps in the same order as in the 128 x 128
// kernel, and the epilogue runs the same operations on it, so the two kernels give bit-identical results.
// Linear layers only (A_LINEAR, not split-precision), TMA-store epilogue, N % 256 == 0, no split-K.
// ---------------------------------------------------------------------------
template <int EPI>
struct GemmWideCfg {
  static constexpr int BM = 128;
  static constexpr int BN = 256;
  static constexpr int BK = 64;
  static constexpr uint32_t A_BYTES = BM * BK * 2;
  static constexpr uint32_t B_BYTES = BN * BK * 2;
  static constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr uint32_t BAR_BYTES = 256;
  static constexpr int EPI_WARPS = 8;
  static constexpr uint32_t PRODUCER_REGS = 40;
  static constexpr uint32_t CONSUMER_REGS = 232;
  static constexpr uint32_t TMA_BOX_BYTES = 16 * 128;
  // Per-warp staging: two alternating 16-row x 128-byte boxes, or one with the RoPE table, which leaves room for a
  // fourth ring stage (enc qkv at cfg-2 on the 700 W H100: 0.241 ms with 4 stages and one box, 0.254 ms with 3 and two).
  static constexpr int STG_BOXES = (EPI == EPI_ROPE) ? 1 : 2;
  static constexpr uint32_t STG_WARP_BYTES = STG_BOXES * TMA_BOX_BYTES;
  static constexpr uint32_t STG_BYTES = EPI_WARPS * STG_WARP_BYTES;
  static constexpr int ROPE_SMEM_ROWS = 64;
  static constexpr uint32_t ROPE_SMEM_BYTES = (EPI == EPI_ROPE) ? ROPE_SMEM_ROWS * kRopeLd * sizeof(float) : 0;
  static constexpr uint32_t MAX_SMEM = 227 * 1024;
  static constexpr int STAGES_FIT = (MAX_SMEM - BAR_BYTES - STG_BYTES - ROPE_SMEM_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > 4 ? 4 : STAGES_FIT;
  // layout: operand ring (A tiles, then B tiles) | staging | barriers | RoPE
  static constexpr uint32_t OFF_STG = STAGES * STAGE_BYTES;
  static constexpr uint32_t OFF_BAR = OFF_STG + STG_BYTES;
  static constexpr uint32_t OFF_ROPE = OFF_BAR + BAR_BYTES;
  static constexpr uint32_t SMEM_BYTES = OFF_ROPE + ROPE_SMEM_BYTES;
  static constexpr int THREADS = 128 + 32 * EPI_WARPS;
  static constexpr int EPI_THREADS = 32 * EPI_WARPS;
  static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS <= 64 * 1024, "register file");
  static_assert(STAGES == 4 && 2 * STAGES * 8 <= BAR_BYTES, "ring");
  static_assert(OFF_STG % 1024 == 0 && STG_WARP_BYTES % 1024 == 0, "SWIZZLE_128B boxes are 1024-byte aligned");
  static_assert(SMEM_BYTES <= MAX_SMEM, "shared memory");
};

// TMA-store epilogue of one warp's 16 rows x 256 columns (EPI_BF16 / EPI_GELU / EPI_ROPE / EPI_F32): the operations of
// epilogue_tile_tma, element for element, on the wide fragment.  A warp writes four bf16 boxes (64 columns each) or eight
// fp32 boxes (32 columns each) per tile, through its staging boxes in turn.
template <int EPI>
__device__ __forceinline__ void epilogue_wide_tma(const GemmParams& p, const CUtensorMap* tmC, float (&acc)[128],
                                                  int row0, int col0, uint8_t* stg, const float* rope_s, uint32_t& ubuf) {
  using Cfg = GemmWideCfg<EPI>;
  constexpr bool OUT_F32 = (EPI == EPI_F32);
  const int lane = threadIdx.x & 31;
  const int r = lane >> 2, t = lane & 3;

#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float2 b = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 8 * j + 2 * t)) : make_float2(0.f, 0.f);
    acc[4 * j] += b.x; acc[4 * j + 1] += b.y; acc[4 * j + 2] += b.x; acc[4 * j + 3] += b.y;
  }
  if constexpr (EPI == EPI_GELU) {
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = gelu_erf(acc[i]);
  }
  if constexpr (EPI == EPI_BF16) {
    if (p.relu_main) {
#pragma unroll
      for (int i = 0; i < 128; ++i) acc[i] = fmaxf(acc[i], 0.0f);
    }
  }
  [[maybe_unused]] uint32_t pyx[2];  // [half]: (pos_y + 1) | (pos_x + 1) << 16 of this thread's two token rows
  [[maybe_unused]] bool staged = true;
  if constexpr (EPI == EPI_ROPE) {
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int row = row0 + 8 * half + r;
      pyx[half] = 0x00010001u;
      if (row < p.M) {
        const int2 pp = *reinterpret_cast<const int2*>(p.pos + 2 * static_cast<long long>(row));
        if (pp.x < -1 || pp.x > p.rope_max_pos || pp.y < -1 || pp.y > p.rope_max_pos)
          __trap();  // token position outside the RoPE table (no printf: see mbar_wait)
        pyx[half] = static_cast<uint32_t>(pp.x + 1) | (static_cast<uint32_t>(pp.y + 1) << 16);
      }
      staged = staged && static_cast<int>(max(pyx[half] & 0xFFFFu, pyx[half] >> 16)) < p.rope_smem_rows;
    }
    staged = __all_sync(0xFFFFFFFFu, staged);
  }
  // RoPE of 32-column chunk q (fragment groups j = 4 q .. 4 q + 3; pair (i, i + 16) is j and j + 2), as in
  // epilogue_tile_tma
  auto rope_chunk = [&](int q) {
    if constexpr (EPI == EPI_ROPE) {
      if (col0 + 32 * q >= p.rope_cols) return;  // warp-uniform: the V columns are not rotated
      auto rotate = [&](auto table_row) {
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int ps = static_cast<int>((q & 1) ? pyx[half] >> 16 : pyx[half] & 0xFFFFu);
          const float4* tb = table_row(ps);
#pragma unroll
          for (int jj = 0; jj < 2; ++jj) {
            const float4 tt = tb[4 * jj + t];
            const int ia = 4 * (4 * q + jj) + 2 * half;
            const int ib = ia + 8;
            const float a0 = acc[ia], b0 = acc[ib], a1 = acc[ia + 1], b1 = acc[ib + 1];
            acc[ia] = fmaf(-b0, tt.y, a0 * tt.x);
            acc[ib] = fmaf(a0, tt.y, b0 * tt.x);
            acc[ia + 1] = fmaf(-b1, tt.w, a1 * tt.z);
            acc[ib + 1] = fmaf(a1, tt.w, b1 * tt.z);
          }
        }
      };
      if (staged) rotate([&](int ps) { return reinterpret_cast<const float4*>(rope_s + ps * kRopeLd); });
      else rotate([&](int ps) { return reinterpret_cast<const float4*>(p.rope_tab + static_cast<long long>(ps) * 32); });
    }
  };

  const uint32_t sb = smem_u32(stg);
  const uint32_t sx = r;  // 128B swizzle: 16-byte chunk k of box row R lives at k ^ (R & 7), and R & 7 = r
  auto next_box = [&]() -> uint32_t {
    if constexpr (Cfg::STG_BOXES == 1) {
      if (lane == 0) tma_store_wait_read();  // the store of the previous box is done reading it
      __syncwarp();
      return sb;
    } else {
      if (lane == 0) tma_store_wait_read1();  // the store that read this box two boxes ago is done with it
      __syncwarp();
      return sb + (ubuf++ & 1u) * Cfg::TMA_BOX_BYTES;
    }
  };
  auto issue = [&](uint32_t box, int col) {
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
      const void* src = stg + (box - sb);
      if constexpr (OUT_F32) {
        if (p.c_reduce) tma_reduce_add_2d(tmC, src, col, row0);
        else tma_store_2d(tmC, src, col, row0);
      } else {
        tma_store_2d(tmC, src, col, row0);
      }
      tma_store_commit();
    }
  };
  if constexpr (OUT_F32) {
#pragma unroll
    for (int c = 0; c < 8; ++c) {  // box c: columns [32 c, 32 c + 32) = fragment groups j = 4 c .. 4 c + 3
      const uint32_t box = next_box();
#pragma unroll
      for (int half = 0; half < 2; ++half)
#pragma unroll
        for (int jl = 0; jl < 4; ++jl) {
          const int i = 4 * (4 * c + jl) + 2 * half;
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(box + (8 * half + r) * 128 +
                                                                 (((2 * jl + (t >> 1)) ^ sx) << 4) + (t & 1) * 8),
                       "f"(acc[i]), "f"(acc[i + 1])
                       : "memory");
        }
      issue(box, col0 + 32 * c);
    }
  } else {
#pragma unroll
    for (int c = 0; c < 4; ++c) {  // box c: columns [64 c, 64 c + 64) = fragment groups j = 8 c .. 8 c + 7
      rope_chunk(2 * c);
      rope_chunk(2 * c + 1);
      const uint32_t box = next_box();
#pragma unroll
      for (int half = 0; half < 2; ++half)
#pragma unroll
        for (int jl = 0; jl < 8; ++jl) {
          const int i = 4 * (8 * c + jl) + 2 * half;
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(box + (8 * half + r) * 128 + ((jl ^ sx) << 4) + 4 * t),
                       "r"(pack_bf16x2(acc[i], acc[i + 1]))
                       : "memory");
        }
      issue(box, col0 + 64 * c);
    }
  }
}

template <int EPI>
__global__ void __launch_bounds__(GemmWideCfg<EPI>::THREADS, 1)
gemm_wide_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmC, const GemmParams p) {
  using Cfg = GemmWideCfg<EPI>;
  static_assert(EPI == EPI_BF16 || EPI == EPI_GELU || EPI == EPI_F32 || EPI == EPI_ROPE, "wide tiles: TMA-store epilogues");
  constexpr int STAGES = Cfg::STAGES;
  constexpr uint32_t A_BYTES = Cfg::A_BYTES;
  constexpr uint32_t B_BYTES = Cfg::B_BYTES;

  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* empty = full + STAGES;
  uint8_t* stg_all = smem + Cfg::OFF_STG;
  [[maybe_unused]] float* rope_s = reinterpret_cast<float*>(smem + Cfg::OFF_ROPE);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n_tiles = p.N / Cfg::BN;
  const int num_tiles = ((p.M + 127) / 128) * n_tiles;  // (m, n), n fastest
  const int nkb = (p.K + Cfg::BK - 1) / Cfg::BK;

  if (threadIdx.x == 0) {
    if ((smem_u32(smem) & 1023u) != 0) device_fatal("dynamic shared memory is not 1024-byte aligned");
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);   // the producer's expect_tx arrival
      mbar_init(&empty[s], 8);  // one arrival per consumer warp: both warpgroups read every stage
    }
    fence_mbar_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmC);
  }
  if constexpr (EPI == EPI_ROPE) {  // constant table: staged before the PDL wait, as in gemm_wg_kernel
    if (warp >= 4) {
      const int nfl = p.rope_smem_rows * 32;
      for (int i = (threadIdx.x - 128) * 4; i < nfl; i += Cfg::EPI_THREADS * 4)
        *reinterpret_cast<float4*>(rope_s + (i >> 5) * kRopeLd + (i & 31)) =
            __ldg(reinterpret_cast<const float4*>(p.rope_tab + i));
    }
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();

  if (warp < 4) {
    // ===================== TMA producer (warp 0, lane 0) =====================
    setmaxnreg_dec<Cfg::PRODUCER_REGS>();
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_tile = tile / n_tiles;
        const int n_tile = tile - m_tile * n_tiles;
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full[stage], A_BYTES + B_BYTES);
          tma_load_2d(sA + stage * A_BYTES, &tmA, &full[stage], kb * Cfg::BK, m_tile * 128);
          tma_load_2d(sB + stage * B_BYTES, &tmB, &full[stage], kb * Cfg::BK, n_tile * Cfg::BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ============ consumer warpgroups: both on every tile, warpgroup wg on rows [64 wg, 64 wg + 64) ============
    setmaxnreg_inc<Cfg::CONSUMER_REGS>();
    const int wg = (warp - 4) >> 2;
    const int wq = warp & 3;
    uint8_t* stg = stg_all + (warp - 4) * Cfg::STG_WARP_BYTES;
    uint32_t ubuf = 0;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_tile = tile / n_tiles;
      const int n_tile = tile - m_tile * n_tiles;
      float acc[128];
#pragma unroll
      for (int i = 0; i < 128; ++i) acc[i] = 0.0f;
      // one k-block: four k16 steps of one m64n256k16 wgmma; the previous k-block's wgmma group may still run, its
      // stage is released once this one is issued
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint64_t adesc = make_smem_desc_sw128(smem_u32(sA + stage * A_BYTES) + wg * 64 * 128);
        const uint64_t bdesc = make_smem_desc_sw128(smem_u32(sB + stage * B_BYTES));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_m64n256k16_ss(acc, adesc + 2 * k, bdesc + 2 * k, 1u);
        wgmma_commit();
        wgmma_wait<1>();
        fence_regs(acc);
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);

      epilogue_wide_tma<EPI>(p, &tmC, acc, m_tile * 128 + 64 * wg + 16 * wq, n_tile * Cfg::BN, stg, rope_s, ubuf);
      // after the CTA's last tile: the bulk stores read this CTA's shared memory
      if (tile + static_cast<int>(gridDim.x) >= num_tiles && lane == 0) tma_store_wait_all();
    }
  }
}

}  // namespace sta
