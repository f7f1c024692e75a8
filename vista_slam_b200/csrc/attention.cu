// Flash-attention forward (head_dim 64, non-causal) on wgmma for sm_90a.
//
// Replaces, for every (sample, head, 128-query tile):
//   * xformers memory_efficient_attention at vista_slam/sta_model/blocks/sta_blocks.py:143
//     (encoder / decoder self-attention), and
//   * the materialised softmax(q k^T * scale) v of CrossAttention, sta_blocks.py:201-205
//     (K/V taken from the partner sample: kv_batch_shift).
//
// Q, K, V are read straight out of the projection GEMM outputs with 3-D TMA tensor maps
// (64 head columns x tokens x samples); nothing is re-laid-out.
//
// Persistent CTAs (min(items, SMs)), each walking the items blockIdx.x, blockIdx.x + gridDim.x, ..; 128 + 128 * CWG
// threads:
//   warp 0        TMA producer: per item the Q tile (double-buffered, so the next item's Q lands under this one), then
//                 K and V tiles of 128 keys through a 3-stage ring that runs on across items (separate full barriers so
//                 that Q K^T starts before V has landed)
//   warps 4..     CWG consumer warpgroups (1 or 2), 64 query rows each: S = Q K^T (wgmma m64n128k16, fp32 in registers),
//                 online softmax in registers (exp2 with the scale folded in, running maximum per row), P rounded to bf16
//                 and kept in registers as the A operand of O += P V (wgmma m64n64k16, V consumed MN-major exactly as TMA
//                 wrote it).  The final O / l is stored straight from the accumulator registers.
// Software pipeline of a consumer warpgroup: S_{j+1} = Q K_{j+1}^T and O += P_j V_j are issued together, and the softmax
// of tile j + 1 runs while P_j V_j is on the tensor cores (only S_{j+1} is waited for); P_{j+1} is rounded to bf16 and O
// rescaled by c_{j+1} once P_j V_j has completed.  Every row still goes through the same operations in the same order as a serial loop, so
// the schedule does not change a bit of the output.  With two warpgroups the issue of those MMAs alternates (named
// barriers), so that one warpgroup's exponentials run while the other's MMAs occupy the tensor cores.
// Ragged tails: a last key tile of <= 16 keys takes one k16 step of P V instead of eight (the others would add exact
// zeros), and a warpgroup whose 64 rows all lie past nq does no MMA or softmax for that item.
// Two warpgroups per CTA share every K / V tile (half the K / V traffic); one warpgroup per CTA doubles the item count
// for problems that would not fill the GPU with 128-row tiles (launch_attention chooses).
#include "common.cuh"
#include "host_util.h"

#include <limits.h>
#include <math.h>
#include <stdio.h>
#include <type_traits>
#include "ops.h"

namespace sta {

namespace {

// CWG consumer warpgroups of 64 query rows each (query tile = 64 * CWG rows); warp 0 is the TMA producer (warps 1-3 idle)
template <int CWG>
constexpr int att_threads() { return 128 + 128 * CWG; }
constexpr int KV_STAGES = 3;
constexpr uint32_t TILE_BYTES = 128 * 64 * 2;  // 16 KB: [128 rows][64 bf16]
// Q (up to 128 rows) x2 | K x3 | V x3 | barriers
constexpr uint32_t ATT_OFF_K = 2 * TILE_BYTES;
constexpr uint32_t ATT_OFF_V = ATT_OFF_K + KV_STAGES * TILE_BYTES;
constexpr uint32_t ATT_OFF_BAR = ATT_OFF_V + KV_STAGES * TILE_BYTES;
constexpr uint32_t ATT_SMEM = ATT_OFF_BAR + 256;
// Register split of the two-warpgroup kernel (setmaxnreg, as in gemm.cuh): the producer warpgroup only issues TMA loads;
// a consumer thread holds S (64, then the fp32 weights P), the bf16 P fragments of the P V in flight (32) and O (32).
constexpr uint32_t ATT_PRODUCER_REGS = 40;
constexpr uint32_t ATT_CONSUMER_REGS = 232;
static_assert(128 * ATT_PRODUCER_REGS + 256 * ATT_CONSUMER_REGS <= 64 * 1024, "register file");
constexpr uint32_t kTurnBar = 1;  // named barriers 1, 2: "consumer warpgroup 0 / 1 may issue its MMAs"

struct AttnParams {
  int nq, nk, batch, heads, qtiles, kv_batch_shift, items;
  float scale_log2;
  __nv_bfloat16* out;
  long long ldo;
};

// Item = (64 * CWG-query tile, head, sample), the tile index fastest, so that the CTAs working side by side share one
// (sample, head)'s K / V tiles in L2.
struct AttnItem {
  int q0, head, b, kvb;
};
template <int CWG>
__device__ __forceinline__ AttnItem attn_item(const AttnParams& p, int item) {
  AttnItem it;
  it.q0 = (item % p.qtiles) * 64 * CWG;
  it.head = (item / p.qtiles) % p.heads;
  it.b = item / (p.qtiles * p.heads);
  it.kvb = (it.b + p.kv_batch_shift) % p.batch;
  return it;
}

// Online softmax of one 64-row x 128-key score tile (wgmma accumulator layout: this thread holds rows g, g + 8 and
// columns 8c + 2t + {0,1}; register 4c + {0,1} = row g, 4c + {2,3} = row g + 8).  Updates the running maxima and this
// thread's part of the row sums, returns the rescale factors of O and leaves P = 2^(S scale - m) in s (fp32; pack_p
// rounds it to bf16 once the registers of the previous P are free).
// NKK = 1 serves a tile of <= 16 keys: columns 16.. are masked to -inf, so their maximum and weights (exact zeros, which
// add nothing to l) are left out; only the first k16 group of P is formed.  The result is bit-identical to NKK = 8.
template <int NKK>
__device__ __forceinline__ void softmax_tile(float (&s)[64], int kvalid, float scale_log2, float& m0, float& m1,
                                             float& l0, float& l1, float& c0, float& c1) {
  const int t = threadIdx.x & 3;
  if (kvalid < 128) {
#pragma unroll
    for (int i = 0; i < 8 * NKK; ++i)
      if (8 * (i >> 2) + 2 * t + (i & 1) >= kvalid) s[i] = -INFINITY;
  }
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int c = 0; c < 2 * NKK; ++c) {
    mx0 = fmaxf(mx0, fmaxf(s[4 * c], s[4 * c + 1]));
    mx1 = fmaxf(mx1, fmaxf(s[4 * c + 2], s[4 * c + 3]));
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  const float mn0 = fmaxf(m0, mx0 * scale_log2), mn1 = fmaxf(m1, mx1 * scale_log2);  // finite: >= 1 valid key
  c0 = ex2_approx(m0 - mn0);                                                          // first tile: 2^-inf = 0
  c1 = ex2_approx(m1 - mn1);
  m0 = mn0;
  m1 = mn1;
  l0 *= c0;
  l1 *= c1;
#pragma unroll
  for (int kk = 0; kk < NKK; ++kk) {
    float* e = s + 8 * kk;
#pragma unroll
    for (int i = 0; i < 8; ++i) e[i] = ex2_approx(fmaf(e[i], scale_log2, (i & 2) ? -m1 : -m0));
    l0 += (e[0] + e[1]) + (e[4] + e[5]);
    l1 += (e[2] + e[3]) + (e[6] + e[7]);
  }
}
// P as bf16 A fragments of the P V wgmma: keys 16 kk .. 16 kk + 15 = accumulator columns 2 kk, 2 kk + 1
template <int NKK>
__device__ __forceinline__ void pack_p(const float (&s)[64], uint32_t (&pa)[8][4]) {
#pragma unroll
  for (int kk = 0; kk < NKK; ++kk) {
    const float* e = s + 8 * kk;
    pa[kk][0] = pack_bf16x2(e[0], e[1]);
    pa[kk][1] = pack_bf16x2(e[2], e[3]);
    pa[kk][2] = pack_bf16x2(e[4], e[5]);
    pa[kk][3] = pack_bf16x2(e[6], e[7]);
  }
}

// TAIL16: the last key tile holds <= 16 keys (nk % 128 in 1..16).
template <int CWG, bool TAIL16>
__global__ void __launch_bounds__(att_threads<CWG>(), 1)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, const AttnParams p, int q_col0, int k_col0, int v_col0) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sK = smem + ATT_OFF_K;
  uint8_t* sV = smem + ATT_OFF_V;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + ATT_OFF_BAR);
  uint64_t* q_full = bars;
  uint64_t* q_empty = bars + 2;
  uint64_t* k_full = bars + 4;
  uint64_t* v_full = k_full + KV_STAGES;
  uint64_t* kv_empty = v_full + KV_STAGES;

  constexpr int QROWS = 64 * CWG;
  const int nkt = (p.nk + 127) / 128;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    if ((smem_u32(smem) & 1023u) != 0) device_fatal("dynamic shared memory is not 1024-byte aligned");
    for (int i = 0; i < 2; ++i) {
      mbar_init(&q_full[i], 1);
      mbar_init(&q_empty[i], 4 * CWG);  // one arrival per consumer warp
    }
    for (int s = 0; s < KV_STAGES; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&v_full[s], 1);
      mbar_init(&kv_empty[s], 4 * CWG);
    }
    fence_mbar_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();

  if (warp < 4) {
    // ===================== TMA producer (warp 0, lane 0; warps 1-3 only give their registers away) =====================
    if constexpr (CWG == 2) setmaxnreg_dec<ATT_PRODUCER_REGS>();
    if (warp == 0 && lane == 0) {
      int st = 0;  // the ring position runs on across items
      uint32_t ph = 0;
      int qi = 0;
      for (int item = blockIdx.x; item < p.items; item += gridDim.x, ++qi) {
        const AttnItem it = attn_item<CWG>(p, item);
        const int qb = qi & 1;
        mbar_wait(&q_empty[qb], ((qi >> 1) & 1) ^ 1);
        mbar_arrive_expect_tx(&q_full[qb], QROWS * 128);
        tma_load_3d(sQ + qb * TILE_BYTES, &tmQ, &q_full[qb], q_col0 + it.head * 64, it.q0, it.b);  // rows >= nq: zeros
        for (int j = 0; j < nkt; ++j) {
          mbar_wait(&kv_empty[st], ph ^ 1);
          mbar_arrive_expect_tx(&k_full[st], TILE_BYTES);
          tma_load_3d(sK + st * TILE_BYTES, &tmK, &k_full[st], k_col0 + it.head * 64, j * 128, it.kvb);
          mbar_arrive_expect_tx(&v_full[st], TILE_BYTES);
          tma_load_3d(sV + st * TILE_BYTES, &tmV, &v_full[st], v_col0 + it.head * 64, j * 128, it.kvb);
          if (++st == KV_STAGES) { st = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ============ consumer warpgroups: 64 query rows each ============
    if constexpr (CWG == 2) setmaxnreg_inc<ATT_CONSUMER_REGS>();
    const int wg = (warp - 4) >> 2, wq = (warp - 4) & 3;
    const int g = lane >> 2, t = lane & 3;
    auto release = [&](uint64_t* bar) {
      __syncwarp();
      if (lane == 0) mbar_arrive(bar);
    };
    // Turn-taking of the two warpgroups (CWG == 2): every item has nkt + 1 MMA issues per warpgroup (S_0, then
    // S_{j+1} with P_j V_j, then the last P V), and the warpgroups issue in turn, warpgroup 0 first.  Warpgroup 0 waits
    // before every issue but its first, warpgroup 1 before every issue; each hands the turn over after issuing, except
    // warpgroup 1 after the CTA's last issue -- so every wait meets exactly one arrival.  A warpgroup with no rows in an
    // item still takes its turns.
    bool first_turn = true;
    auto turn_begin = [&]() {
      if constexpr (CWG == 2)
        if (!first_turn || wg == 1) named_bar_sync(kTurnBar + wg, 256);
      first_turn = false;
    };
    auto turn_end = [&](bool cta_last) {
      if constexpr (CWG == 2)
        if (wg == 0 || !cta_last) named_bar_arrive(kTurnBar + (wg ^ 1), 256);
    };
    int st = 0;  // ring position of the item's first K / V tile
    uint32_t ph = 0;
    int qi = 0;
#pragma unroll 1
    for (int item = blockIdx.x; item < p.items; item += gridDim.x, ++qi) {
      const AttnItem it = attn_item<CWG>(p, item);
      const bool last_item = item >= p.items - static_cast<int>(gridDim.x);
      const int qb = qi & 1;
      mbar_wait(&q_full[qb], (qi >> 1) & 1);
      if (it.q0 + wg * 64 >= p.nq) {
        // no valid row: release the Q buffer and each K / V stage once it has been loaded, and pass the turns
        release(&q_empty[qb]);
        for (int j = 0; j <= nkt; ++j) {
          turn_begin();
          turn_end(last_item && j == nkt);
          if (j < nkt) {
            mbar_wait(&v_full[st], ph);
            release(&kv_empty[st]);
            if (++st == KV_STAGES) { st = 0; ph ^= 1; }
          }
        }
        continue;
      }
      const uint64_t qdesc = make_smem_desc_sw128(smem_u32(sQ + qb * TILE_BYTES) + wg * 64 * 128);
      float o[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] = 0.0f;
      float m0 = -INFINITY, m1 = -INFINITY;  // running maxima of the two rows (log2 units)
      float l0 = 0.0f, l1 = 0.0f;            // this thread's part of the running row sums
      float c0, c1;                          // rescale factors of the latest softmax tile
      float s[64];
      uint32_t pa[8][4];
      // ---- S = Q K^T (64 x 128 keys, K-major operands exactly as TMA wrote them) ----
      auto issue_s = [&](int st, uint32_t ph) {
#pragma unroll
        for (int i = 0; i < 64; ++i) s[i] = 0.0f;
        mbar_wait(&k_full[st], ph);
        const uint64_t kdesc = make_smem_desc_sw128(smem_u32(sK + st * TILE_BYTES));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_m64n128k16_ss(s, qdesc + 2 * k, kdesc + 2 * k, 1u);
        wgmma_commit();
      };
      // ---- O += P V (V [keys][64] is the MN-major B operand: 16 keys = two 8-row groups = 2 KB per k16 step) ----
      auto issue_pv = [&](int st, uint32_t ph, auto nkk) {
        mbar_wait(&v_full[st], ph);
        const uint32_t vbase = smem_u32(sV + st * TILE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < decltype(nkk)::value; ++kk)
          wgmma_m64n64k16_rs_mn(o, pa[kk], make_smem_desc_sw128(vbase + kk * 2048));
        wgmma_commit();
      };
      auto rescale_o = [&]() {
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          o[4 * c] *= c0; o[4 * c + 1] *= c0;
          o[4 * c + 2] *= c1; o[4 * c + 3] *= c1;
        }
      };
      // key tile j >= 1: S_j and P_{j-1} V_{j-1} on the tensor cores, the softmax of tile j under P_{j-1} V_{j-1}; then
      // P_j is packed and O rescaled by c_j, ready for P_j V_j
      auto step = [&](int j, auto nkk) {
        constexpr int NKK = decltype(nkk)::value;
        const int pst = st;
        const uint32_t pph = ph;
        if (++st == KV_STAGES) { st = 0; ph ^= 1; }
        turn_begin();
        issue_s(st, ph);
        issue_pv(pst, pph, std::integral_constant<int, 8>());
        turn_end(false);
        wgmma_wait<1>();  // S_j has landed; P_{j-1} V_{j-1} may still run
        fence_regs(s);
        const int kvalid = p.nk - j * 128;
        softmax_tile<NKK>(s, kvalid, p.scale_log2, m0, m1, l0, l1, c0, c1);
        fence_regs(s);
        // The item's last S has landed: release its Q buffer.  This branch sits between the softmax and the wait for
        // P_{j-1} V_{j-1} on purpose: it ends the basic block, and ptxas keeps the wait in the next one.  Within one
        // block it schedules the wait above the softmax's MUFU.EX2 and nothing overlaps the MMAs (tests/
        // test_attention_sass_cpu.py checks the compiled order).  The test is on kvalid rather than j == nkt - 1 so that
        // the peeled last step keeps the branch too.
        if (kvalid <= 128) release(&q_empty[qb]);
        wgmma_wait<0>();
        fence_regs(o);
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) fence_regs(pa[kk]);
        release(&kv_empty[pst]);
        pack_p<NKK>(s, pa);
        rescale_o();
      };
      constexpr int LAST_NKK = TAIL16 ? 1 : 8;  // k16 steps of the last key tile's P V

      turn_begin();
      issue_s(st, ph);
      turn_end(false);
      wgmma_wait<0>();
      fence_regs(s);
      if (nkt == 1) release(&q_empty[qb]);
      // (a single tile of <= 16 keys takes the full softmax here: its P fragments past the first are exact zeros)
      softmax_tile<8>(s, p.nk, p.scale_log2, m0, m1, l0, l1, c0, c1);
      pack_p<8>(s, pa);
      rescale_o();
#pragma unroll 1
      for (int j = 1; j < nkt - 1; ++j) step(j, std::integral_constant<int, 8>());
      if (nkt > 1) step(nkt - 1, std::integral_constant<int, LAST_NKK>());
      turn_begin();
      issue_pv(st, ph, std::integral_constant<int, LAST_NKK>());
      turn_end(last_item);
      wgmma_wait<0>();
      fence_regs(o);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) fence_regs(pa[kk]);
      release(&kv_empty[st]);
      if (++st == KV_STAGES) { st = 0; ph ^= 1; }

      l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
      l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
      const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
      const int row = it.q0 + wg * 64 + wq * 16 + g;
      __nv_bfloat16* oa = p.out + (static_cast<long long>(it.b) * p.nq + row) * p.ldo + it.head * 64 + 2 * t;
      __nv_bfloat16* ob = oa + 8 * p.ldo;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        if (row < p.nq) *reinterpret_cast<uint32_t*>(oa + 8 * c) = pack_bf16x2(o[4 * c] * inv0, o[4 * c + 1] * inv0);
        if (row + 8 < p.nq) *reinterpret_cast<uint32_t*>(ob + 8 * c) = pack_bf16x2(o[4 * c + 2] * inv1, o[4 * c + 3] * inv1);
      }
    }
  }
}

// ---------------------------------------------------------------------------
// Split-precision parity mode (common.cuh): exact-softmax attention in fp32 on the CUDA cores.  Q, K, V rows are
// (hi | lo | hi) bf16; every value is reconstructed as hi + lo (16-17 significant bits), scores, the online softmax
// (full-precision exp2f) and P V are fp32, the output is stored as (hi | lo | hi).  One thread per query row (its q
// and output accumulator live in registers), 32-key tiles of K and V staged in shared memory as fp32.  Not a
// performance path: it exists so that the whole model can be checked against the fp32 reference below the bf16
// noise floor (tests, tools/parity_report.py).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
attention_x3_kernel(const __nv_bfloat16* __restrict__ q, long long ldq, int q_col0, const __nv_bfloat16* __restrict__ k,
                    long long ldk, int k_col0, const __nv_bfloat16* __restrict__ v, long long ldv, int v_col0,
                    __nv_bfloat16* __restrict__ out, long long ldo, int nq, int nk, int batch, int kv_batch_shift,
                    float scale_log2) {
  __shared__ __align__(16) float Ks[32][64];
  __shared__ __align__(16) float Vs[32][64];
  pdl_wait();
  pdl_launch_dependents();
  const int head = blockIdx.y, b = blockIdx.z;
  const int kvb = (b + kv_batch_shift) % batch;
  const int tid = threadIdx.x;
  const int row = blockIdx.x * 128 + tid;
  const bool valid = row < nq;
  float qv[64], o[64];
  {
    const __nv_bfloat16* qp = q + (static_cast<long long>(b) * nq + (valid ? row : 0)) * ldq + q_col0 + head * 64;
    const long long lo_off = ldq / 3;
#pragma unroll
    for (int d = 0; d < 64; ++d) {
      qv[d] = valid ? (__bfloat162float(qp[d]) + __bfloat162float(qp[lo_off + d])) * scale_log2 : 0.f;
      o[d] = 0.f;
    }
  }
  float m = -INFINITY, l = 0.f;
  const __nv_bfloat16* kb = k + static_cast<long long>(kvb) * nk * ldk + k_col0 + head * 64;
  const __nv_bfloat16* vb = v + static_cast<long long>(kvb) * nk * ldv + v_col0 + head * 64;
  const long long klo = ldk / 3, vlo = ldv / 3;
  for (int j0 = 0; j0 < nk; j0 += 32) {
    __syncthreads();
    {  // stage 32 keys x 64 dims of K and V as fp32: thread -> (key = tid / 4, 16 dims)
      const int key = tid >> 2, d0 = (tid & 3) * 16;
      const int j = j0 + key;
#pragma unroll
      for (int d = 0; d < 16; ++d) {
        float kf = 0.f, vf = 0.f;
        if (j < nk) {
          const __nv_bfloat16* kr = kb + static_cast<long long>(j) * ldk + d0 + d;
          const __nv_bfloat16* vr = vb + static_cast<long long>(j) * ldv + d0 + d;
          kf = __bfloat162float(kr[0]) + __bfloat162float(kr[klo]);
          vf = __bfloat162float(vr[0]) + __bfloat162float(vr[vlo]);
        }
        Ks[key][d0 + d] = kf;
        Vs[key][d0 + d] = vf;
      }
    }
    __syncthreads();
    const int nv = (nk - j0 < 32) ? (nk - j0) : 32;
    float sc[32];
    float tmax = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < 32; ++jj) {
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
      for (int d = 0; d < 64; d += 4) {
        const float4 kk = *reinterpret_cast<const float4*>(&Ks[jj][d]);
        a0 = fmaf(qv[d], kk.x, a0);
        a1 = fmaf(qv[d + 1], kk.y, a1);
        a2 = fmaf(qv[d + 2], kk.z, a2);
        a3 = fmaf(qv[d + 3], kk.w, a3);
      }
      const float sv = (jj < nv) ? (a0 + a1) + (a2 + a3) : -INFINITY;
      sc[jj] = sv;
      tmax = fmaxf(tmax, sv);
    }
    const float m_new = fmaxf(m, tmax);  // finite: every tile holds at least one valid key
    const float corr = exp2f(m - m_new);  // first tile: exp2f(-inf) = 0
    l *= corr;
#pragma unroll
    for (int d = 0; d < 64; ++d) o[d] *= corr;
    m = m_new;
#pragma unroll
    for (int jj = 0; jj < 32; ++jj) {
      const float pj = exp2f(sc[jj] - m);  // masked keys: exp2f(-inf) = 0
      l += pj;
#pragma unroll
      for (int d = 0; d < 64; d += 4) {
        const float4 vv = *reinterpret_cast<const float4*>(&Vs[jj][d]);
        o[d] = fmaf(pj, vv.x, o[d]);
        o[d + 1] = fmaf(pj, vv.y, o[d + 1]);
        o[d + 2] = fmaf(pj, vv.z, o[d + 2]);
        o[d + 3] = fmaf(pj, vv.w, o[d + 3]);
      }
    }
  }
  if (valid) {
    const float inv_l = 1.0f / l;
    __nv_bfloat16* op = out + (static_cast<long long>(b) * nq + row) * ldo + head * 64;
    const long long w = ldo / 3;
#pragma unroll
    for (int d = 0; d < 64; d += 8) {
      float r[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) r[i] = o[d + i] * inv_l;
      const uint4 hi = make_uint4(pack_bf16x2(r[0], r[1]), pack_bf16x2(r[2], r[3]), pack_bf16x2(r[4], r[5]),
                                  pack_bf16x2(r[6], r[7]));
      *reinterpret_cast<uint4*>(op + d) = hi;
      *reinterpret_cast<uint4*>(op + w + d) = make_uint4(pack_bf16x2_resid(r[0], r[1]), pack_bf16x2_resid(r[2], r[3]),
                                                         pack_bf16x2_resid(r[4], r[5]), pack_bf16x2_resid(r[6], r[7]));
      *reinterpret_cast<uint4*>(op + 2 * w + d) = hi;
    }
  }
}

int make_qkv_map(CUtensorMap* m, const bf16* base, long long ld, int ntok, int batch, uint32_t rows = 128) {
  uint64_t dims[3] = {(uint64_t)ld, (uint64_t)ntok, (uint64_t)batch};
  uint64_t strides[2] = {(uint64_t)ld * 2, (uint64_t)ld * 2 * (uint64_t)ntok};
  uint32_t box[3] = {64, rows, 1};
  return make_tmap_bf16(m, base, 3, dims, strides, box);
}

}  // namespace

template <int CWG, bool TAIL16>
static int launch_attention_inst(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const AttnParams& p,
                                 const AttnLaunch& a, cudaStream_t stream) {
  static PerDeviceOnce once;  // the opt-in is per device, not per process
  STA_CHECK_CUDA(once.run([&] {
    return cudaFuncSetAttribute(attention_fwd_kernel<CWG, TAIL16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ATT_SMEM);
  }));
  const int ctas = p.items < num_sms() ? p.items : num_sms();  // persistent: one CTA per SM walks the items
  STA_CHECK_CUDA(launch_pdl(attention_fwd_kernel<CWG, TAIL16>, dim3(static_cast<unsigned>(ctas)), dim3(att_threads<CWG>()), ATT_SMEM,
                            stream, 1, tmQ, tmK, tmV, p, a.q_col0, a.k_col0, a.v_col0));
  return 0;
}

int launch_attention(const AttnLaunch& a, cudaStream_t stream) {
  STA_REQUIRE(a.batch > 0 && a.heads > 0 && a.nq > 0 && a.nk > 0, "empty attention problem");
  STA_REQUIRE(a.ldq % 8 == 0 && a.ldk % 8 == 0 && a.ldv % 8 == 0 && a.ldo % 8 == 0, "row strides must be 16B multiples");
  STA_REQUIRE(a.q_col0 % 8 == 0 && a.k_col0 % 8 == 0 && a.v_col0 % 8 == 0, "column offsets must be 16B multiples");
  if (a.split)
    STA_REQUIRE(a.ldq % 3 == 0 && a.ldk % 3 == 0 && a.ldv % 3 == 0 && a.ldo % 3 == 0 && (a.ldo / 3) % 8 == 0,
                "split-precision rows are (hi | lo | hi): strides must be 3 x the logical width");
  // Out-of-range values would not fail loudly: the TMA loads zero-fill coordinates outside a tensor map (a negative
  // sample gives all-zero scores and values), while the split kernel reads whatever lies in front of or after a row.
  // In split mode the *_col0 are hi-column offsets within the logical width ld / 3.
  const long long wdiv = a.split ? 3 : 1, hcols = 64LL * a.heads;
  STA_REQUIRE(a.kv_batch_shift >= 0 && a.kv_batch_shift < a.batch, "kv_batch_shift must lie in [0, batch)");
  STA_REQUIRE(a.q_col0 >= 0 && a.q_col0 + hcols <= a.ldq / wdiv, "q head columns run past the row width");
  STA_REQUIRE(a.k_col0 >= 0 && a.k_col0 + hcols <= a.ldk / wdiv, "k head columns run past the row width");
  STA_REQUIRE(a.v_col0 >= 0 && a.v_col0 + hcols <= a.ldv / wdiv, "v head columns run past the row width");
  STA_REQUIRE(hcols <= a.ldo / wdiv, "output rows are narrower than 64 x heads");
  // the wgmma kernel takes the row maximum of the raw scores and scales afterwards: that is the maximum only for scale > 0
  STA_REQUIRE(std::isfinite(a.scale) && a.scale > 0.0f, "scale must be finite and positive");
  if (a.split) {
    STA_REQUIRE(a.heads <= 65535 && a.batch <= 65535, "grid limits");
    STA_CHECK_CUDA(launch_pdl(attention_x3_kernel, dim3((a.nq + 127) / 128, a.heads, a.batch), dim3(128), 0, stream, 1, a.q,
                              a.ldq, a.q_col0, a.k, a.ldk, a.k_col0, a.v, a.ldv, a.v_col0, a.out, a.ldo, a.nq, a.nk, a.batch,
                              a.kv_batch_shift, a.scale * 1.4426950408889634f));
    return 0;
  }
  AttnParams p;
  p.nq = a.nq;
  p.nk = a.nk;
  p.batch = a.batch;
  p.heads = a.heads;
  p.kv_batch_shift = a.kv_batch_shift;
  p.scale_log2 = a.scale * 1.4426950408889634f;
  p.out = a.out;
  p.ldo = a.ldo;
  // Query tile: 128 rows (two consumer warpgroups share every K / V tile) unless that grid leaves SMs idle (small
  // problems: SLAM-mode keyframes, low resolutions), then 64 rows (one warpgroup) for twice the CTAs.
  const long long items128 = static_cast<long long>((a.nq + 127) / 128) * a.heads * a.batch;
  const int qrows = items128 < num_sms() ? 64 : 128;
  p.qtiles = (a.nq + qrows - 1) / qrows;
  CUtensorMap tmQ, tmK, tmV;
  if (make_qkv_map(&tmQ, a.q, a.ldq, a.nq, a.batch, static_cast<uint32_t>(qrows))) return 1;
  if (make_qkv_map(&tmK, a.k, a.ldk, a.nk, a.batch)) return 1;
  if (make_qkv_map(&tmV, a.v, a.ldv, a.nk, a.batch)) return 1;
  const long long items = static_cast<long long>(p.qtiles) * a.heads * a.batch;
  STA_REQUIRE(items <= INT_MAX - num_sms(), "grid limits");  // the CTAs step through item indices by the grid size
  p.items = static_cast<int>(items);
  const bool tail16 = (a.nk - 1) % 128 < 16;
  if (qrows == 64)
    return tail16 ? launch_attention_inst<1, true>(tmQ, tmK, tmV, p, a, stream)
                  : launch_attention_inst<1, false>(tmQ, tmK, tmV, p, a, stream);
  return tail16 ? launch_attention_inst<2, true>(tmQ, tmK, tmV, p, a, stream)
                : launch_attention_inst<2, false>(tmQ, tmK, tmV, p, a, stream);
}

}  // namespace sta
