// Persistent warp-specialised wgmma GEMM / implicit-GEMM 3x3 convolution for sm_90a.
//
//   D[M,N] = A[M,K] * W[N,K]^T  (bf16 operands, fp32 accumulation in registers)
//
// Roles: warp 0 = TMA producer (warps 1-3 idle), warps 4-11 = two consumer warpgroups.  Consumer warpgroup g
// computes rows [64 g, 64 g + 64) of the 128 x BN tile with wgmma (m64 n128 k16, accumulators in registers) while
// the producer keeps a STAGES-deep operand ring filled; the finished accumulators are written to a padded fp32 tile
// in shared memory, from which the same eight warps run the fused epilogue (-> global).  The producer prefetches
// the next tile's operands during the epilogue.  Operand tiles are 128B-swizzled K-major [rows][64] boxes written
// by TMA; the 3x3 convolution loads one halo tile per channel chunk through a 4-D NHWC tensor map (out-of-bounds =
// zero padding) and feeds every filter tap from shifted views of it, so no im2col buffer exists.
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
enum AMode : int { A_LINEAR = 0, A_CONV3 = 1 };
enum Epi : int {
  EPI_BF16 = 0,     // out_bf16 = [relu](acc + bias [+ resid_bf16] [+ resid2_bf16]); optional relu copy in out2
  EPI_GELU = 1,     // out_bf16 = gelu_erf(acc + bias)
  EPI_F32 = 2,      // out_f32[row'] = acc + bias [+ resid_f32[row']]   (row' optionally skips one pose-token row per sample)
  EPI_ROPE = 3,     // out_bf16 = rope2d(acc + bias) on columns < rope_cols, plain on the rest
  EPI_PIXSHUF = 4,  // ConvTranspose2d(k = stride): scatter to the k x k sub-pixels, NHWC bf16
  EPI_HEAD = 5,     // relu(acc + bias) -> 1x1 conv (128 -> 4) -> pointmap/confidence post-process (fp32 out)
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
};

// TMA = true: the epilogue writes through shared memory + TMA tensor stores (epilogue_tile_tma), else the
// coalesced per-warp path (epilogue_tile).
// A_CONV3: pixels per staged halo row.  10 = the 8-pixel tile plus its two halo columns (dense box, 8-row descriptor groups
// 1280 B apart -- groups then start at any 128-byte multiple, which the absolute-address swizzle permits).
constexpr int kHaloPitch = 10;
constexpr int kRopeLd = 36;  // floats per staged sin/cos table row (32 + 4 pad: conflict-free row-per-lane reads)
template <int AMODE, int EPI, bool TMA>
struct GemmCfg {
  static constexpr bool CONV = (AMODE == A_CONV3);
  static constexpr int BM = 128;
  static constexpr int BN = 128;  // one consumer warpgroup covers the 128 columns of a tile (wgmma m64n128k16)
  static constexpr int BK = 64;
  static constexpr uint32_t A_BYTES = BM * BK * 2;
  static constexpr uint32_t B_BYTES = BN * BK * 2;
  static constexpr uint32_t BAR_BYTES = 256;
  static constexpr int EPI_WARPS = 8;   // the two consumer warpgroups
  static constexpr int PARTS = EPI_WARPS / 4;  // column parts of a tile, one per epilogue warp of a lane quarter
  static constexpr uint32_t EPI_SMEM_BYTES = (EPI == EPI_HEAD) ? 3 * 128 * 4 * sizeof(float) : 0;  // partial sums
  // finished accumulators: [128 rows][BN + 4] fp32 (the pad makes row-per-lane 16-byte reads conflict-free)
  static constexpr int ACC_LD = BN + 4;
  static constexpr uint32_t ACC_BYTES = BM * ACC_LD * sizeof(float);
  // per-warp staging of the TMA-store epilogue: one 4 KB SWIZZLE_128B box
  static constexpr uint32_t STG_WARP_BYTES = 4096;
  static constexpr uint32_t STG_BYTES = TMA ? EPI_WARPS * STG_WARP_BYTES : 0;
  static constexpr int ROPE_SMEM_ROWS = 64;  // positions -1 .. 62
  static constexpr uint32_t ROPE_SMEM_BYTES = (EPI == EPI_ROPE) ? ROPE_SMEM_ROWS * kRopeLd * sizeof(float) : 0;
  static constexpr uint32_t MAX_SMEM = 227 * 1024;
  // convolution: the ring holds B tiles only; three 18 x 10 x 64-channel halo input tiles besides it
  static constexpr uint32_t HALO_TX_BYTES = 18 * kHaloPitch * 128;                 // bytes one box delivers
  static constexpr uint32_t HALO_BYTES = (HALO_TX_BYTES + 1023u) & ~1023u;        // stage stride (swizzle-pattern aligned)
  static constexpr int HALO_STAGES = 3;
  static constexpr uint32_t HALO_TOTAL = CONV ? HALO_STAGES * HALO_BYTES : 0;
  static constexpr uint32_t STAGE_BYTES = CONV ? B_BYTES : A_BYTES + B_BYTES;
  static constexpr int STAGES_FIT =
      (MAX_SMEM - BAR_BYTES - EPI_SMEM_BYTES - STG_BYTES - ACC_BYTES - ROPE_SMEM_BYTES - HALO_TOTAL) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > 8 ? 8 : STAGES_FIT;
  // layout: operand ring | halo tiles | staging (1024-byte aligned) | accumulator tile | barriers | EPI_HEAD partials | RoPE
  static constexpr uint32_t OFF_HALO = STAGES * STAGE_BYTES;
  static constexpr uint32_t OFF_STG = OFF_HALO + HALO_TOTAL;
  static constexpr uint32_t OFF_ACC = OFF_STG + STG_BYTES;
  static constexpr uint32_t OFF_BAR = OFF_ACC + ACC_BYTES;
  static constexpr uint32_t OFF_EPI = OFF_BAR + BAR_BYTES;
  static constexpr uint32_t OFF_ROPE = OFF_EPI + EPI_SMEM_BYTES;
  static constexpr uint32_t SMEM_BYTES = OFF_ROPE + ROPE_SMEM_BYTES;
  static constexpr int THREADS = 128 + 32 * EPI_WARPS;
  static constexpr int EPI_THREADS = 32 * EPI_WARPS;
  static_assert(STAGES <= 8 && STAGES >= 3, "barrier area holds at most 8 stages");
  static_assert(OFF_STG % 1024 == 0 && OFF_HALO % 1024 == 0 && OFF_ACC % 16 == 0, "staging alignment");
  static_assert(SMEM_BYTES <= MAX_SMEM, "shared memory");
};

// ---------------------------------------------------------------------------
// Epilogue for one 128 x BN accumulator tile held in shared memory ([128][BN + 4] fp32); executed by the 8 consumer
// warps.  warp (quarter, part): rows [32*quarter, +32), columns [part*BN/2, +BN/2).
//
// Every 32x32 fp32 chunk is read in a COALESCED mapping -- lane -> (row = 4*it + lane/8, 4 columns at (lane%8)*4) --
// in which bias, residuals, activation and the global stores happen: a warp-wide access covers 4 rows x 128
// contiguous bytes (fp32) or 4 rows x 64 bytes (bf16).
// ---------------------------------------------------------------------------
// 32 consecutive fp32 accumulators of one row (16-byte aligned)
__device__ __forceinline__ void acc_ld32(const float* src, uint32_t (&r)[32]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 v = reinterpret_cast<const float4*>(src)[j];
    r[4 * j] = __float_as_uint(v.x); r[4 * j + 1] = __float_as_uint(v.y);
    r[4 * j + 2] = __float_as_uint(v.z); r[4 * j + 3] = __float_as_uint(v.w);
  }
}

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

// accs: the accumulator tile at this warp's first row (32 * quarter) and first column (part * BN / PARTS)
template <int AMODE, int EPI>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, const float* accs, int m_tile, int n_tile,
                                              int quarter, int part, float* epi_smem) {
  using Cfg = GemmCfg<AMODE, EPI, false>;
  constexpr int BN = Cfg::BN;
  constexpr int PARTS = Cfg::PARTS;
  constexpr int LD = Cfg::ACC_LD;  // accumulator tile row stride (floats)
  constexpr int CH = BN / PARTS;  // columns per epilogue warp
  const int lane = threadIdx.x & 31;
  const int colbase = n_tile * BN + part * CH;

  if constexpr (EPI == EPI_HEAD) {
    // head.2 epilogue: ReLU -> head.4 (1x1, 128 -> 4) -> postprocess (dpt_block.py:319-323,
    // postprocess.py:10-62).  Row mapping: each thread owns 32 of the 128 channels of one pixel; the four
    // column parts are combined through shared memory.  Nothing but 16 bytes per pixel is written.
    const int r_local = quarter * 32 + lane;
    long long orow;
    bool valid;
    tile_row<AMODE>(p, m_tile, r_local, orow, valid);
    float psum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
    for (int c = 0; c < CH; c += 32) {
      const int col = colbase + c;
      uint32_t acc[32];
      acc_ld32(accs + lane * LD + c, acc);
      const float4* wp = reinterpret_cast<const float4*>(p.head_w) + col;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        float v = fmaxf(__uint_as_float(acc[i]) + __ldg(p.bias + col + i), 0.0f);
        float4 w4 = __ldg(wp + i);
        psum[0] = fmaf(v, w4.x, psum[0]);
        psum[1] = fmaf(v, w4.y, psum[1]);
        psum[2] = fmaf(v, w4.z, psum[2]);
        psum[3] = fmaf(v, w4.w, psum[3]);
      }
    }
    if (part != 0)
      reinterpret_cast<float4*>(epi_smem)[(part - 1) * 128 + r_local] = make_float4(psum[0], psum[1], psum[2], psum[3]);
    named_bar_sync(1, Cfg::EPI_THREADS);
    if (part == 0) {
      float4 o = reinterpret_cast<float4*>(epi_smem)[r_local];
#pragma unroll
      for (int q = 1; q < PARTS - 1; ++q) {
        const float4 t = reinterpret_cast<float4*>(epi_smem)[q * 128 + r_local];
        o.x += t.x; o.y += t.y; o.z += t.z; o.w += t.w;
      }
      const float x = psum[0] + o.x + __ldg(p.head_b + 0);
      const float y = psum[1] + o.y + __ldg(p.head_b + 1);
      const float z = psum[2] + o.z + __ldg(p.head_b + 2);
      const float cf = psum[3] + o.w + __ldg(p.head_b + 3);
      if (valid) {
        const float d = sqrtf(x * x + y * y + z * z);
        const float dc = fmaxf(d, 1e-8f);
        const float e = expm1f(d);
        p.pts3d[orow * 3 + 0] = (x / dc) * e;
        p.pts3d[orow * 3 + 1] = (y / dc) * e;
        p.pts3d[orow * 3 + 2] = (z / dc) * e;
        p.conf[orow] = 1.0f + expf(cf);
      }
    }
    named_bar_sync(1, Cfg::EPI_THREADS);
    return;
  } else {
    // ---- coalesced mapping bookkeeping: this lane touches rows 4*it + (lane>>3), it = 0..7 ----
    const int crow = lane >> 3;
    const int cc = (lane & 7) * 4;  // first of this lane's 4 columns inside the 32-column chunk
    long long orow_c[8];
    uint32_t vmask = 0;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      bool v;
      tile_row<AMODE>(p, m_tile, quarter * 32 + it * 4 + crow, orow_c[it], v);
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
      if (col >= p.N) return;
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
          float4 v = *reinterpret_cast<const float4*>(stg + (it * 4 + crow) * LD + cc);
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
            for (int c = 0; c < CH; c += 32) {
              if (colbase + c < p.N) {
                const char* a = reinterpret_cast<const char*>(p.resid) + (orow_c[it] * p.ldo + colbase + c + cc) * esz;
                asm volatile("prefetch.global.L2 [%0];" ::"l"(a));
                if constexpr (EPI == EPI_BF16) {
                  if (p.resid2) {
                    const char* a2 = reinterpret_cast<const char*>(p.resid2) + (orow_c[it] * p.ldo + colbase + c + cc) * esz;
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(a2));
                  }
                }
              }
            }
          }
        }
      }
    }
#pragma unroll 1
    for (int c = 0; c < CH; c += 32) flush(colbase + c, accs + c);
  }
}

// ---------------------------------------------------------------------------
// TMA-store epilogue for the linear layers with N % 128 == 0 (EPI_BF16 / EPI_GELU / EPI_ROPE / EPI_F32).
//
// The math stays in a row-per-thread mapping -- one accumulator ROW per thread, 32 consecutive columns per load --
// so bias, GELU and the RoPE rotation (whose (i, i+16) partners sit in the same thread) need no shuffles.  The
// results go to a per-warp 32-row x 128-byte shared-memory box in the SWIZZLE_128B layout (conflict-free 16-byte
// stores) and leave with ONE bulk tensor store per box issued by lane 0: no per-lane global stores, rows >= M are
// clipped by the tensor map, and the in-place fp32 residual stream (x += proj(..)) becomes a bulk reduce-add
// performed by the L2, so the epilogue never loads the residual.
// accrow: this thread's accumulator row at the warp's first column.
// ---------------------------------------------------------------------------
template <int EPI>
__device__ __forceinline__ void epilogue_tile_tma(const GemmParams& p, const CUtensorMap* tmC, const float* accrow, int m_tile,
                                                  int colbase, int row_off, int quarter, uint8_t* cbuf,
                                                  const float* rope_s) {
  using Cfg = GemmCfg<A_LINEAR, EPI, true>;
  constexpr int CH = Cfg::BN / Cfg::PARTS;  // columns per epilogue warp
  constexpr int NCH = CH / 32;    // 32-column chunks
  constexpr bool OUT_F32 = (EPI == EPI_F32);
  const int lane = threadIdx.x & 31;
  const int row0 = m_tile * 128 + quarter * 32;  // first row of this warp's box (token index)
  const int srow0 = row0 + row_off;              // ... in the output tensor (split-K partial slices)
  const uint32_t cb = smem_u32(cbuf);
  const uint32_t srow = cb + lane * 128;  // this thread's row inside the box
  const uint32_t sx = lane & 7;           // 128B swizzle: 16-byte chunk j lives at j ^ (row & 7)

  [[maybe_unused]] int py = 0, px = 0;
  if constexpr (EPI == EPI_ROPE) {
    if (row0 + lane < p.M) {
      const int2 pp = *reinterpret_cast<const int2*>(p.pos + 2 * static_cast<long long>(row0 + lane));
      py = pp.x;
      px = pp.y;
      if (py < -1 || py > p.rope_max_pos || px < -1 || px > p.rope_max_pos)
        __trap();  // token position outside the RoPE table (no printf: see mbar_wait)
    }
  }

  // Split-precision parity mode, bf16 outputs: the tile is drained twice -- pass 0 stores hi = bf16(v) at columns
  // [col, ..) and [2N + col, ..), pass 1 re-reads v and stores lo = bf16(v - hi) at [N + col, ..) -- so the
  // production register footprint is unchanged.
  const int npass = (!OUT_F32 && p.split) ? 2 : 1;
  const bool has_bias = p.bias != nullptr;
#pragma unroll 1
  for (int pass = 0; pass < npass; ++pass) {
  // bias of chunk c is loaded one chunk ahead (warp-uniform addresses: L1 broadcast), so its latency never sits
  // between the accumulator load and the math
  float4 bcur[8];
#pragma unroll
  for (int j = 0; j < 8; ++j)
    bcur[j] = has_bias ? __ldg(reinterpret_cast<const float4*>(p.bias + colbase) + j) : make_float4(0.f, 0.f, 0.f, 0.f);

#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    uint32_t acc[32];
    acc_ld32(accrow + c * 32, acc);
    float* v = reinterpret_cast<float*>(acc);
    const int col = colbase + c * 32;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      v[4 * j] += bcur[j].x; v[4 * j + 1] += bcur[j].y; v[4 * j + 2] += bcur[j].z; v[4 * j + 3] += bcur[j].w;
    }
    if (c + 1 < NCH && has_bias) {
#pragma unroll
      for (int j = 0; j < 8; ++j) bcur[j] = __ldg(reinterpret_cast<const float4*>(p.bias + col + 32) + j);
    }
    if constexpr (EPI == EPI_GELU) {
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = gelu_erf(v[i]);
    }
    if constexpr (EPI == EPI_BF16) {
      if (p.relu_main) {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i], 0.0f);
      }
    }
    if constexpr (EPI == EPI_ROPE) {
      // 2-D RoPE (pos_embed/pos_embed.py:149-185, curope/kernels.cu:17-82): a 32-column chunk is one half of a
      // 64-wide head -- the y-half (rotated by pos_y) or the x-half (pos_x); inside it the pairs are (i, i + 16).
      if (col < p.rope_cols) {  // warp-uniform: the V columns are not rotated
        const int ps = (((col >> 5) & 1) ? px : py) + 1;
        const float4* tb = (ps < p.rope_smem_rows)
                               ? reinterpret_cast<const float4*>(rope_s + ps * kRopeLd)
                               : reinterpret_cast<const float4*>(p.rope_tab + static_cast<long long>(ps) * 32);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float4 t = tb[j];  // (cos f, sin f, cos f+1, sin f+1), f = 2j
          const float a0 = v[2 * j], b0 = v[2 * j + 16], a1 = v[2 * j + 1], b1 = v[2 * j + 17];
          v[2 * j] = fmaf(-b0, t.y, a0 * t.x);
          v[2 * j + 16] = fmaf(a0, t.y, b0 * t.x);
          v[2 * j + 1] = fmaf(-b1, t.w, a1 * t.z);
          v[2 * j + 17] = fmaf(a1, t.w, b1 * t.z);
        }
      }
    }
    // ---- registers -> swizzled box -> bulk tensor store ----
    if constexpr (OUT_F32) {
      // one box per chunk: 32 rows x 32 fp32 columns
      if (lane == 0) tma_store_wait_read();
      __syncwarp();
#pragma unroll
      for (int j = 0; j < 8; ++j)
        asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(srow + ((j ^ sx) << 4)), "f"(v[4 * j]),
                     "f"(v[4 * j + 1]), "f"(v[4 * j + 2]), "f"(v[4 * j + 3])
                     : "memory");
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {
        if (p.c_reduce) tma_reduce_add_2d(tmC, cbuf, col, srow0);
        else tma_store_2d(tmC, cbuf, col, srow0);
        tma_store_commit();
      }
    } else {
      // one box per two chunks: 32 rows x 64 bf16 columns
      const int sub = c & 1;
      if (sub == 0) {
        if (lane == 0) tma_store_wait_read();
        __syncwarp();
      }
      if (pass == 1) {  // residual part: lo = v - bf16(v)
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = bf16_resid(v[i]);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(srow + (((sub * 4 + j) ^ sx) << 4)),
                     "r"(pack_bf16x2(v[8 * j], v[8 * j + 1])), "r"(pack_bf16x2(v[8 * j + 2], v[8 * j + 3])),
                     "r"(pack_bf16x2(v[8 * j + 4], v[8 * j + 5])), "r"(pack_bf16x2(v[8 * j + 6], v[8 * j + 7]))
                     : "memory");
      if (sub == 1) {
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
          tma_store_2d(tmC, cbuf, col - 32 + pass * p.N, srow0);
          if (p.split && pass == 0) tma_store_2d(tmC, cbuf, col - 32 + 2 * p.N, srow0);  // second hi copy
          tma_store_commit();
        }
      }
    }
  }
  }  // pass
}

template <int AMODE, int EPI, bool TMA>
__global__ void __launch_bounds__(GemmCfg<AMODE, EPI, TMA>::THREADS, 1)
gemm_wg_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmC, const GemmParams p) {
  using Cfg = GemmCfg<AMODE, EPI, TMA>;
  constexpr bool CONV = Cfg::CONV;
  static_assert(!TMA || (AMODE == A_LINEAR && (EPI == EPI_BF16 || EPI == EPI_GELU || EPI == EPI_F32 || EPI == EPI_ROPE)),
                "TMA-store epilogue: linear layers only");
  static_assert(TMA || EPI == EPI_BF16 || EPI == EPI_F32 || EPI == EPI_PIXSHUF || EPI == EPI_HEAD,
                "GELU and RoPE have the TMA-store epilogue only");
  constexpr int BN = Cfg::BN;
  constexpr int STAGES = Cfg::STAGES;
  constexpr uint32_t A_BYTES = Cfg::A_BYTES;
  constexpr uint32_t B_BYTES = Cfg::B_BYTES;
  constexpr int EW = Cfg::EPI_WARPS;

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
  [[maybe_unused]] float* epi_smem = reinterpret_cast<float*>(smem + Cfg::OFF_EPI);
  [[maybe_unused]] uint8_t* stg_all = smem + Cfg::OFF_STG;
  float* acc_s = reinterpret_cast<float*>(smem + Cfg::OFF_ACC);
  [[maybe_unused]] float* rope_s = reinterpret_cast<float*>(smem + Cfg::OFF_ROPE);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int m_tiles = CONV ? p.nimg * p.tiles_h * p.tiles_w : (p.M + 127) / 128;
  const int n_tiles = (p.N + BN - 1) / BN;
  const int ksplit = TMA ? p.ksplit : 1;
  const int num_tiles = m_tiles * n_tiles * ksplit;  // work items (m, n, ks), ks fastest
  const int cpb = CONV ? (p.Cin / 64) : 1;  // 64-channel chunks per filter tap
  const int nkb = CONV ? 9 * cpb : (p.K + 63) / 64;

  if (threadIdx.x == 0) {
    if ((smem_u32(smem) & 1023u) != 0) device_fatal("dynamic shared memory is not 1024-byte aligned");
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);    // the producer's expect_tx arrival
      mbar_init(&empty[s], EW);  // one arrival per consumer warp
    }
    if constexpr (CONV) {
      for (int s = 0; s < Cfg::HALO_STAGES; ++s) {
        mbar_init(&hfull[s], 1);
        mbar_init(&hempty[s], EW);
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

  if (warp == 0) {
    // ===================== TMA producer =====================
    if (lane == 0) {
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
            tma_load_2d(sA + stage * A_BYTES, &tmA, &full[stage], kb * 64, m_tile * 128);
            tma_load_2d(sB + stage * B_BYTES, &tmB, &full[stage], kb * 64, b_row0);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ============ consumer warpgroups: mainloop (wgmma) + epilogue ============
    const int wg = (warp - 4) >> 2;     // rows [64 wg, 64 wg + 64) of the tile in the mainloop
    const int wq = (warp - 4) & 3;      // warp inside the warpgroup: 16 of those rows
    const int quarter = warp & 3;       // epilogue mapping: rows [32 quarter, +32) ...
    const int part = (warp - 4) >> 2;   // ... columns [part * BN / 2, +BN / 2)
    int stage = 0;
    uint32_t phase = 0;
    [[maybe_unused]] int hstage = 0;
    [[maybe_unused]] uint32_t hphase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int ks = tile % ksplit, mn = tile / ksplit;
      const int m_tile = mn / n_tiles;
      const int n_tile = mn % n_tiles;
      const int kb0 = ks * nkb / ksplit, kb1 = (ks + 1) * nkb / ksplit;
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.0f;
      // one k-block: four k16 steps; the previous k-block's wgmma group may still run, its stage is released
      // once this one is issued
      int prev = -1;
      auto kblock = [&](uint64_t adesc, uint64_t bdesc) {
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_m64n128k16_ss(acc, adesc + 2 * k, bdesc + 2 * k, 1u);
        wgmma_commit();
        wgmma_wait<1>();
        fence_regs(acc);
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      };
      if constexpr (CONV) {
        for (int cc = 0; cc < cpb; ++cc) {
          mbar_wait(&hfull[hstage], hphase);
          // output pixel (y, x) of the 16 x 8 tile reads halo pixel (y + kh, x + kw); halo rows are kHaloPitch pixels,
          // and this warpgroup's 64 rows are the output rows y = 8 wg .. 8 wg + 7
          const uint32_t hbase = smem_u32(sH + hstage * Cfg::HALO_BYTES) + wg * 8 * kHaloPitch * 128;
          for (int tap = 0; tap < 9; ++tap) {
            mbar_wait(&full[stage], phase);
            const int kh = tap / 3, kw = tap - kh * 3;
            kblock(make_smem_desc_sw128_rows(hbase + (kh * kHaloPitch + kw) * 128, kHaloPitch * 128),
                   make_smem_desc_sw128(smem_u32(sB + stage * B_BYTES)));
          }
          wgmma_wait<0>();  // every read of this halo tile has completed
          fence_regs(acc);
          if (lane == 0) mbar_arrive(&hempty[hstage]);
          if (++hstage == Cfg::HALO_STAGES) { hstage = 0; hphase ^= 1; }
        }
      } else {
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&full[stage], phase);
          kblock(make_smem_desc_sw128(smem_u32(sA + stage * A_BYTES) + wg * 64 * 128),
                 make_smem_desc_sw128(smem_u32(sB + stage * B_BYTES)));
        }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);

      // accumulators -> shared tile (wgmma layout: register 4j + {0,1} = row g, columns 8j + 2t + {0,1}; 4j + {2,3} = row g + 8)
      named_bar_sync(1, Cfg::EPI_THREADS);  // the previous tile's epilogue has finished reading the tile
      {
        const int r0 = wg * 64 + wq * 16 + (lane >> 2);
        const int c0 = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          *reinterpret_cast<float2*>(acc_s + r0 * Cfg::ACC_LD + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(acc_s + (r0 + 8) * Cfg::ACC_LD + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
      named_bar_sync(1, Cfg::EPI_THREADS);
      const int cols_w = BN / Cfg::PARTS;
      if constexpr (TMA) {
        epilogue_tile_tma<EPI>(p, &tmC, acc_s + (quarter * 32 + lane) * Cfg::ACC_LD + part * cols_w, m_tile,
                               n_tile * BN + part * cols_w, ks * p.split_rows, quarter,
                               stg_all + (warp - 4) * Cfg::STG_WARP_BYTES, rope_s);
      } else {
        epilogue_tile<AMODE, EPI>(p, acc_s + quarter * 32 * Cfg::ACC_LD + part * cols_w, m_tile, n_tile, quarter, part,
                                  epi_smem);
      }
    }
    if constexpr (TMA) {
      if (lane == 0) tma_store_wait_all();  // the bulk stores read this CTA's shared memory
    }
  }
}

}  // namespace sta
