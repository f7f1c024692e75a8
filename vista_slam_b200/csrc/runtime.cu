// STA model runtime: packed weights, workspace and the kernel sequence of the forward pass,
// exported through the C ABI declared in include/sta_b200.h.
//
// Mirrors (behaviour, not code) vista_slam/sta_model/sta_model.py:
//   _encode_image :163-174, _decode_stereo :177-244, forward :247-291,
//   DPT head heads/dpt_head.py:34-66 + heads/dpt_block.py, pose head heads/pose_head.py:109-119.
#include <stdint.h>
#include <string.h>

#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/sta_b200.h"
#include "host_util.h"
#include "ops.h"

namespace sta {

// ---------------------------------------------------------------------------
// weight packing kernels (run once per tensor at load time)
// ---------------------------------------------------------------------------
// dst[r * ldd + c] = bf16(src[r * cols + c]).  Split-precision mode (common.cuh): a weight row of logical width kw
// is stored as (hi | hi | lo), each part kw wide (ldd = 3 * kw).
__device__ __forceinline__ void put_weight(__nv_bfloat16* d, float v, int split, long long kw) {
  const __nv_bfloat16 hi = __float2bfloat16(v);
  d[0] = hi;
  if (split) {
    d[kw] = hi;
    d[2 * kw] = __float2bfloat16(v - __bfloat162float(hi));
  }
}
__global__ void pack_linear_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int rows, int cols,
                                   long long ldd, int split) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(rows) * cols) return;
  const int r = static_cast<int>(idx / cols), c = static_cast<int>(idx % cols);
  put_weight(dst + r * ldd + c, src[idx], split, ldd / 3);
}
// Conv2d weight [Cout][Cin][3][3] -> [Cout][(kh*3+kw)][Cin_pad]  (split mode: [..][3 * Cin_pad] = hi | hi | lo per tap)
__global__ void pack_conv3_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int Cout, int Cin,
                                  int Cin_pad, int split) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(Cout) * Cin * 9) return;
  const int tap = static_cast<int>(idx % 9);
  const int ci = static_cast<int>((idx / 9) % Cin);
  const int co = static_cast<int>(idx / (9LL * Cin));
  put_weight(dst + (static_cast<long long>(co) * 9 + tap) * (split ? 3 * Cin_pad : Cin_pad) + ci, src[idx], split, Cin_pad);
}
// ConvTranspose2d weight [Cin][Cout][k][k] -> [(kh*k+kw)*Cout_pad + co][Cin_pad]
__global__ void pack_convT_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int Cin, int Cout,
                                  int k, int Cin_pad, int Cout_pad, int split) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(Cin) * Cout * k * k) return;
  const int kk = static_cast<int>(idx % (k * k));
  const int co = static_cast<int>((idx / (k * k)) % Cout);
  const int ci = static_cast<int>(idx / (static_cast<long long>(k) * k * Cout));
  put_weight(dst + (static_cast<long long>(kk) * Cout_pad + co) * (split ? 3 * Cin_pad : Cin_pad) + ci, src[idx], split,
             Cin_pad);
}
// FP8 mode: one 128 x 128 block (blockIdx.y, blockIdx.x) of a trunk weight [rows][cols] fp32 -> e4m3 codes (row stride
// ldd) and the block's power-of-two scale at sdst[blockIdx.y * sld + blockIdx.x] (common.cuh fp8_scale)
__global__ void __launch_bounds__(256)
pack_linear_fp8_kernel(const float* __restrict__ src, int cols, uint8_t* __restrict__ dst, long long ldd, float* __restrict__ sdst,
                       int sld) {
  __shared__ float red[8];
  const int r = blockIdx.y * 128 + (threadIdx.x >> 1), c0 = blockIdx.x * 128 + (threadIdx.x & 1) * 64;
  const float* sp = src + static_cast<long long>(r) * cols + c0;
  float am = 0.f;
  for (int c = 0; c < 64; ++c) am = fmaxf(am, fabsf(sp[c]));
  for (int o = 16; o > 0; o >>= 1) am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = am;
  __syncthreads();
  am = red[0];
  for (int w = 1; w < 8; ++w) am = fmaxf(am, red[w]);
  float s, inv;
  fp8_scale(am, s, inv);
  uint16_t* dp = reinterpret_cast<uint16_t*>(dst + static_cast<long long>(r) * ldd + c0);
  for (int c = 0; c < 64; c += 2) dp[c / 2] = cvt_e4m3x2(sp[c] * inv, sp[c + 1] * inv);
  if (threadIdx.x == 0) sdst[blockIdx.y * sld + blockIdx.x] = s;
}
// [rows][cols] fp32 -> [cols][rows] fp32
__global__ void transpose_f32_kernel(const float* __restrict__ src, float* __restrict__ dst, int rows, int cols) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * cols) return;
  const int r = idx / cols, c = idx % cols;
  dst[c * rows + r] = src[idx];
}
// decoder positions: [2B][N+1][2] int32 from two int64 [B][N][2] arrays, pose token at (-1,-1)
__global__ void build_dec_pos_kernel(const long long* __restrict__ p1, const long long* __restrict__ p2, int B, int N,
                                     int* __restrict__ out) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = 2LL * B * (N + 1);
  if (idx >= total) return;
  const int t = static_cast<int>(idx % (N + 1));
  const int s = static_cast<int>(idx / (N + 1));
  int y = -1, x = -1;
  if (t > 0) {
    const long long* p = (s < B) ? p1 + (static_cast<long long>(s) * N + (t - 1)) * 2
                                 : p2 + (static_cast<long long>(s - B) * N + (t - 1)) * 2;
    y = static_cast<int>(p[0]);
    x = static_cast<int>(p[1]);
  }
  out[2 * idx] = y;
  out[2 * idx + 1] = x;
}
__global__ void pos_to_int64_kernel(const int* __restrict__ in, long long n, long long* __restrict__ out) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx < n) out[idx] = in[idx];
}
// LayerNorm with fp32 output (all rows) -- only used by the per-layer-output compatibility path.
__global__ void __launch_bounds__(256)
layernorm_f32_kernel(const float* __restrict__ x, int rows, int C, float eps, const float* __restrict__ g,
                     const float* __restrict__ b, float* __restrict__ out) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + static_cast<long long>(row) * C;
  float sum = 0.f;
  for (int c = lane; c < C; c += 32) sum += xr[c];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / C;
  float sq = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float d = xr[c] - mean;
    sq += d * d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / C + eps);
  float* orow = out + static_cast<long long>(row) * C;
  for (int c = lane; c < C; c += 32) orow[c] = (xr[c] - mean) * rstd * g[c] + b[c];
}

// ---------------------------------------------------------------------------
// model
// ---------------------------------------------------------------------------
struct Lin {
  bf16* w = nullptr;  // [N][K]
  float* b = nullptr; // [N] or null
  int N = 0, K = 0;   // K is the PHYSICAL reduction length: 3 x the logical one in split-precision mode
  // FP8 mode, trunk linears (w is then null): e4m3 codes [N][K] and one scale per 128 x 128 block [N / 128][K / 128]
  uint8_t* q = nullptr;
  float* qs = nullptr;
};
// FP8 mode: e4m3 activation rows [rows][C] and their scales [rows][C / 128]
struct Fp8Act {
  uint8_t* q = nullptr;
  float* s = nullptr;
};
struct LNp {
  float *g = nullptr, *b = nullptr;
};
struct EncBlock {
  LNp n1, n2;
  Lin qkv, proj, fc1, fc2;
};
struct DecBlock {
  LNp n1, n2, n3, ny;
  Lin qkv, proj, cq, ckv, cproj, fc1, fc2;
};
struct Rcu {
  Lin c1, c2;  // 3x3 256 -> 256
};
struct Refine {
  Rcu r1, r2;
  Lin out;  // 1x1
};

enum PackKind { PK_F32, PK_LINEAR, PK_CONV3, PK_CONVT, PK_TRANSPOSE_F32, PK_IGNORE, PK_LINEAR_FP8 };
struct Slot {
  PackKind kind;
  std::vector<int64_t> shape;  // expected source shape
  void* dst = nullptr;
  long long ldd = 0;            // PK_LINEAR / PK_LINEAR_FP8: destination row stride
  float* sdst = nullptr;        // PK_LINEAR_FP8: block scales, row stride ldd / 128
  int cin_pad = 0, cout_pad = 0, k = 0;
  bool loaded = false;
};

struct Workspace {
  char* base = nullptr;  // null: a dry run that only counts bytes (ws_need)
  size_t bytes = 0;
  size_t off = 0;
  bool overflow = false;  // a take went past `bytes`: the entry point refuses before its first launch (check_ws)
  int bmul = 1;  // bf16 activations are 3x wide in split-precision mode
  int fp8 = 0;   // FP8 mode: the trunk linears read e4m3 activations (Fp8Act) instead of bf16 ones
  template <typename T>
  T* take(size_t n) {
    off = (off + 255) & ~static_cast<size_t>(255);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += n * sizeof(T);
    if (off > bytes) overflow = true;
    return p;
  }
  bf16* takeb(size_t n) { return take<bf16>(n * bmul); }  // bf16 activation buffer with n LOGICAL elements
  Fp8Act takeq(size_t rows, int C) {
    Fp8Act a;
    a.q = take<uint8_t>(rows * C);
    a.s = take<float>(rows * (C / 128));
    return a;
  }
};

struct EncBufs {
  bf16 *patches, *lnb, *qkv, *att, *hid;  // lnb, hid: null in FP8 mode
  int* pos;
  Fp8Act ln8, att8, hid8;  // FP8 mode only
};
struct DecBufs {
  float* xd;
  bf16 *ln1, *lny, *qkv, *att, *qc, *kvc, *hid;  // ln1, lny, hid: null in FP8 mode
  Fp8Act ln8, lny8, att8, hid8;                  // FP8 mode only
  bf16* hook[4];  // the DPT hooks (dpt_head.py:112): bf16 encoder features (the decoder input), decoder outputs 6, 9, 12
  int* pos;
};
struct DptBufs {
  bf16 *a0, *l1, *a1, *l2, *l3, *a3, *col4, *l4;
  bf16 *r_raw[4], *r_relu[4];
  bf16 *t1, *t2, *s_raw, *s_relu, *o, *up, *path;  // sized for the largest level
  bf16 *hc1, *hup;
};

}  // namespace sta

using namespace sta;

struct StaModel {
  // Precision of the tensor-core operands: 0 = bf16 (production), 1 = split-precision "x3" parity mode -- every bf16
  // activation is (hi | lo | hi), every bf16 weight (hi | hi | lo) (common.cuh), the same gemm_wg_kernel mainloop runs
  // over 3K, attention runs in fp32 on the CUDA cores.  ~17 significant operand bits instead of 8; ~3.5x slower.
  int split = 0;
  int bmul() const { return split ? 3 : 1; }
  // 2 = FP8 mode (STA_PRECISION_FP8): the linears of the 24 encoder and 12 decoder blocks run on e4m3 operands with
  // power-of-two block scales (gemm.cuh A_FP8), everything else as in bf16 mode.
  int fp8 = 0;
  // ---- weights ----
  char* arena = nullptr;
  size_t arena_bytes = 0, arena_off = 0;
  std::unordered_map<std::string, Slot> slots;
  int missing = 0;

  float* pose_tok = nullptr;
  Lin patch, dec_embed;
  EncBlock enc[24];
  DecBlock dec[12];
  LNp dec_norm;
  // DPT
  Lin act0, act0T, act1, act1T, act2, act3, act3c;
  Lin rn[4];
  Refine ref[4];  // ref[0] = refinenet1 ... ref[3] = refinenet4
  Lin head0, head2;
  float *head4_w = nullptr, *head4_b = nullptr;
  PoseHeadWeights pose = {};

  // ---- workspace ----
  Workspace ws;
  float* stage = nullptr;  // staging for host->device weight uploads
  size_t stage_bytes = 0;
  char* io = nullptr;      // device staging for sta_forward_pairs_host
  size_t io_bytes = 0;
  static constexpr int kMaxHostChunks = 32;
  cudaStream_t s_in = nullptr, s_out = nullptr;  // copy streams of the host entry point
  static constexpr int kMaxParts = 4;  // DPT parts per view in the host entry point (D2H of a part overlaps the next part)
  cudaEvent_t ev_in[kMaxHostChunks] = {}, ev_done[kMaxHostChunks] = {}, ev_part[kMaxHostChunks][2 * kMaxParts] = {},
              ev_start = nullptr;
  int64_t launches = 0;
  int max_pairs_per_chunk = 16;
  // What sta_regress_pairs_begin leaves for _finish (K = 0: nothing): the shape, the decoder buffers holding the hooks and
  // the workspace offset past _begin's buffers.  Every other model entry point clears it (check_ready).
  struct PairsBegun { int K = 0, H = 0, W = 0; DecBufs d = {}; size_t ws_off = 0; } rp;
  // The handle owns ONE workspace / io buffer / graph set: calls are ordered on whatever stream they are given.  When the
  // caller switches streams, the new stream first waits for the work this handle enqueued on the previous one.
  cudaStream_t last_stream = nullptr;
  bool has_last_stream = false;
  cudaEvent_t ev_switch = nullptr;

  // ---- CUDA-graph replay of the launch-bound small-batch entry points (SLAM mode) ----
  struct GraphEntry {
    std::vector<long long> key;
    cudaGraphExec_t exec = nullptr;  // null: seen once (ran eagerly), capture on the next call
    int64_t launches = 0;
    bool unsupported = false;  // capture / instantiate failed once: stay eager for this key
  };
  float* splitk_ws = nullptr;  // fp32 partial tiles of the split-K route for small problems (gemm.cu)
  static constexpr size_t kSplitKBytes = static_cast<size_t>(48) << 20;
  std::vector<GraphEntry> graphs;
  cudaStream_t s_cap = nullptr;  // capture stream (the caller's stream may be the legacy default stream)
  int64_t graph_replays = 0;

  // ---- optional per-kernel-family timing (CUDA events on the launch stream) ----
  bool prof_on = false;
  struct ProfRec { int cat; cudaEvent_t e0, e1; };
  std::vector<ProfRec> prof_recs;
  std::vector<cudaEvent_t> prof_pool;
  double prof_ms[4] = {0, 0, 0, 0};
  int64_t prof_cnt[4] = {0, 0, 0, 0};
  double prof_flops[4] = {0, 0, 0, 0};
  // ---- buffer taps of the tests (sta_set_taps): name -> the caller's StaTap ----
  std::unordered_map<std::string, StaTap*> taps;
  cudaEvent_t prof_event() {
    cudaEvent_t e;
    if (!prof_pool.empty()) {
      e = prof_pool.back();
      prof_pool.pop_back();
    } else {
      cudaEventCreate(&e);
    }
    return e;
  }

  template <typename T>
  T* alloc(size_t n) {
    arena_off = (arena_off + 255) & ~static_cast<size_t>(255);
    T* p = reinterpret_cast<T*>(arena + arena_off);
    arena_off += n * sizeof(T);
    return p;
  }
};

namespace {

#define RUN(expr)            \
  do {                       \
    int _rc = (expr);        \
    if (_rc) return _rc;     \
  } while (0)

constexpr float kLnEps = 1e-6f;
constexpr int kEncDim = 1024, kDecDim = 768, kEncHeads = 16, kDecHeads = 12;

void add_slot(StaModel* m, const std::string& name, PackKind kind, std::vector<int64_t> shape, void* dst,
              long long ldd = 0, int cin_pad = 0, int cout_pad = 0, int k = 0) {
  Slot s;
  s.kind = kind;
  s.shape = std::move(shape);
  s.dst = dst;
  s.ldd = ldd;
  s.cin_pad = cin_pad;
  s.cout_pad = cout_pad;
  s.k = k;
  m->slots[name] = s;
  if (kind != PK_IGNORE) m->missing++;
}

// linear [N][K] (+bias) registered under prefix.weight / prefix.bias; optional zero padding of N
// FP8 mode: the e4m3 slot of a trunk weight [rows][K] whose first row is row0 of L's packed matrix
void add_fp8_slot(StaModel* m, const std::string& name, const Lin* L, int row0, int rows) {
  add_slot(m, name, PK_LINEAR_FP8, {rows, L->K}, L->q + static_cast<size_t>(row0) * L->K, L->K);
  m->slots[name].sdst = L->qs + static_cast<size_t>(row0 / 128) * (L->K / 128);
}
void alloc_fp8(StaModel* m, Lin* L) {
  L->q = m->alloc<uint8_t>(static_cast<size_t>(L->N) * L->K);
  L->qs = m->alloc<float>(static_cast<size_t>(L->N / 128) * (L->K / 128));
}
// trunk = a linear of the encoder / decoder blocks: e4m3 in FP8 mode
void reg_linear(StaModel* m, const std::string& prefix, Lin* L, int N, int K, bool bias = true, int N_pad = 0,
                std::vector<int64_t> wshape = {}, bool trunk = false) {
  const int Np = N_pad > 0 ? N_pad : N;
  L->N = Np;
  L->K = K * m->bmul();
  if (wshape.empty()) wshape = {N, K};
  if (trunk && m->fp8) {
    alloc_fp8(m, L);
    add_fp8_slot(m, prefix + ".weight", L, 0, N);
  } else {
    L->w = m->alloc<bf16>(static_cast<size_t>(Np) * L->K);
    add_slot(m, prefix + ".weight", PK_LINEAR, wshape, L->w, L->K);
  }
  if (bias) {
    L->b = m->alloc<float>(Np);
    add_slot(m, prefix + ".bias", PK_F32, {N}, L->b);
  }
}
void reg_ln(StaModel* m, const std::string& prefix, LNp* p, int C) {
  p->g = m->alloc<float>(C);
  p->b = m->alloc<float>(C);
  add_slot(m, prefix + ".weight", PK_F32, {C}, p->g);
  add_slot(m, prefix + ".bias", PK_F32, {C}, p->b);
}
void reg_conv3(StaModel* m, const std::string& prefix, Lin* L, int Cout, int Cin, bool bias, int Cin_pad = 0) {
  const int Cp = Cin_pad > 0 ? Cin_pad : Cin;
  L->N = Cout;
  L->K = 9 * Cp * m->bmul();
  L->w = m->alloc<bf16>(static_cast<size_t>(Cout) * L->K);
  add_slot(m, prefix + ".weight", PK_CONV3, {Cout, Cin, 3, 3}, L->w, 0, Cp);
  if (bias) {
    L->b = m->alloc<float>(Cout);
    add_slot(m, prefix + ".bias", PK_F32, {Cout}, L->b);
  }
}
void reg_convT(StaModel* m, const std::string& prefix, Lin* L, int C, int k, int C_pad) {
  L->N = k * k * C_pad;
  L->K = C_pad * m->bmul();
  L->w = m->alloc<bf16>(static_cast<size_t>(L->N) * L->K);
  add_slot(m, prefix + ".weight", PK_CONVT, {C, C, k, k}, L->w, 0, C_pad, C_pad, k);
  L->b = m->alloc<float>(C_pad);  // indexed by output channel
  add_slot(m, prefix + ".bias", PK_F32, {C}, L->b);
}
void reg_f32(StaModel* m, const std::string& name, float** dst, std::vector<int64_t> shape) {
  size_t n = 1;
  for (auto d : shape) n *= static_cast<size_t>(d);
  *dst = m->alloc<float>(n);
  add_slot(m, name, PK_F32, shape, *dst);
}

int build_registry(StaModel* m) {
  reg_f32(m, "init_pose_token", &m->pose_tok, {1, 1, kDecDim});
  reg_linear(m, "patch_embed.proj", &m->patch, kEncDim, 768, true, 0, {kEncDim, 3, 16, 16});
  for (int i = 0; i < 24; ++i) {
    const std::string p = "enc_blocks." + std::to_string(i) + ".";
    EncBlock& b = m->enc[i];
    reg_ln(m, p + "norm1", &b.n1, kEncDim);
    reg_linear(m, p + "attn.qkv", &b.qkv, 3 * kEncDim, kEncDim, true, 0, {}, true);
    reg_linear(m, p + "attn.proj", &b.proj, kEncDim, kEncDim, true, 0, {}, true);
    reg_ln(m, p + "norm2", &b.n2, kEncDim);
    reg_linear(m, p + "mlp.fc1", &b.fc1, 4 * kEncDim, kEncDim, true, 0, {}, true);
    reg_linear(m, p + "mlp.fc2", &b.fc2, kEncDim, 4 * kEncDim, true, 0, {}, true);
  }
  add_slot(m, "enc_norm.weight", PK_IGNORE, {kEncDim}, nullptr);  // never applied (normalize=False everywhere)
  add_slot(m, "enc_norm.bias", PK_IGNORE, {kEncDim}, nullptr);
  reg_linear(m, "decoder_embed", &m->dec_embed, kDecDim, kEncDim);
  for (int i = 0; i < 12; ++i) {
    const std::string p = "dec_block." + std::to_string(i) + ".";
    DecBlock& b = m->dec[i];
    reg_ln(m, p + "norm1", &b.n1, kDecDim);
    reg_linear(m, p + "attn.qkv", &b.qkv, 3 * kDecDim, kDecDim, true, 0, {}, true);
    reg_linear(m, p + "attn.proj", &b.proj, kDecDim, kDecDim, true, 0, {}, true);
    reg_linear(m, p + "cross_attn.projq", &b.cq, kDecDim, kDecDim, true, 0, {}, true);
    // projk and projv are fused into one [1536][768] matrix (both act on norm_y(y))
    b.ckv.N = 2 * kDecDim;
    b.ckv.K = kDecDim * m->bmul();
    if (m->fp8) {
      alloc_fp8(m, &b.ckv);
      add_fp8_slot(m, p + "cross_attn.projk.weight", &b.ckv, 0, kDecDim);
      add_fp8_slot(m, p + "cross_attn.projv.weight", &b.ckv, kDecDim, kDecDim);
      b.ckv.b = m->alloc<float>(2 * kDecDim);
    } else {
      b.ckv.w = m->alloc<bf16>(static_cast<size_t>(2) * kDecDim * b.ckv.K);
      b.ckv.b = m->alloc<float>(2 * kDecDim);
      add_slot(m, p + "cross_attn.projk.weight", PK_LINEAR, {kDecDim, kDecDim}, b.ckv.w, b.ckv.K);
      add_slot(m, p + "cross_attn.projv.weight", PK_LINEAR, {kDecDim, kDecDim},
               b.ckv.w + static_cast<size_t>(kDecDim) * b.ckv.K, b.ckv.K);
    }
    add_slot(m, p + "cross_attn.projk.bias", PK_F32, {kDecDim}, b.ckv.b);
    add_slot(m, p + "cross_attn.projv.bias", PK_F32, {kDecDim}, b.ckv.b + kDecDim);
    reg_linear(m, p + "cross_attn.proj", &b.cproj, kDecDim, kDecDim, true, 0, {}, true);
    reg_ln(m, p + "norm2", &b.n2, kDecDim);
    reg_ln(m, p + "norm3", &b.n3, kDecDim);
    reg_linear(m, p + "mlp.fc1", &b.fc1, 4 * kDecDim, kDecDim, true, 0, {}, true);
    reg_linear(m, p + "mlp.fc2", &b.fc2, kDecDim, 4 * kDecDim, true, 0, {}, true);
    reg_ln(m, p + "norm_y", &b.ny, kDecDim);
  }
  reg_ln(m, "dec_norm", &m->dec_norm, kDecDim);

  const std::string d = "downstream_head_pts.dpt.";
  const int rn_cin[4] = {96, 192, 384, 768};
  const int rn_cin_pad[4] = {128, 192, 384, 768};
  for (int i = 0; i < 4; ++i) {
    reg_conv3(m, d + "scratch.layer_rn." + std::to_string(i), &m->rn[i], 256, rn_cin[i], false, rn_cin_pad[i]);
    // the same Parameter is also registered as scratch.layer{i+1}_rn (dpt_block.py:33-75)
    add_slot(m, d + "scratch.layer" + std::to_string(i + 1) + "_rn.weight", PK_IGNORE, {256, rn_cin[i], 3, 3}, nullptr);
  }
  for (int i = 0; i < 4; ++i) {
    const std::string p = d + "scratch.refinenet" + std::to_string(i + 1) + ".";
    Refine& r = m->ref[i];
    reg_linear(m, p + "out_conv", &r.out, 256, 256, true, 0, {256, 256, 1, 1});
    if (i == 3) {  // refinenet4 is called with one input: resConfUnit1 is never used (dpt_block.py:189-197)
      for (const char* c : {"conv1", "conv2"}) {
        add_slot(m, p + "resConfUnit1." + c + ".weight", PK_IGNORE, {256, 256, 3, 3}, nullptr);
        add_slot(m, p + "resConfUnit1." + c + ".bias", PK_IGNORE, {256}, nullptr);
      }
    } else {
      reg_conv3(m, p + "resConfUnit1.conv1", &r.r1.c1, 256, 256, true);
      reg_conv3(m, p + "resConfUnit1.conv2", &r.r1.c2, 256, 256, true);
    }
    reg_conv3(m, p + "resConfUnit2.conv1", &r.r2.c1, 256, 256, true);
    reg_conv3(m, p + "resConfUnit2.conv2", &r.r2.c2, 256, 256, true);
  }
  reg_conv3(m, d + "head.0", &m->head0, 128, 256, true);
  reg_conv3(m, d + "head.2", &m->head2, 128, 128, true);
  m->head4_w = m->alloc<float>(128 * 4);
  add_slot(m, d + "head.4.weight", PK_TRANSPOSE_F32, {4, 128, 1, 1}, m->head4_w);
  reg_f32(m, d + "head.4.bias", &m->head4_b, {4});
  reg_linear(m, d + "act_postprocess.0.0", &m->act0, 96, kEncDim, true, 128, {96, kEncDim, 1, 1});
  reg_convT(m, d + "act_postprocess.0.1", &m->act0T, 96, 4, 128);
  reg_linear(m, d + "act_postprocess.1.0", &m->act1, 192, kDecDim, true, 0, {192, kDecDim, 1, 1});
  reg_convT(m, d + "act_postprocess.1.1", &m->act1T, 192, 2, 192);
  reg_linear(m, d + "act_postprocess.2.0", &m->act2, 384, kDecDim, true, 0, {384, kDecDim, 1, 1});
  reg_linear(m, d + "act_postprocess.3.0", &m->act3, 768, kDecDim, true, 0, {768, kDecDim, 1, 1});
  reg_conv3(m, d + "act_postprocess.3.1", &m->act3c, 768, 768, true);

  float* tmp = nullptr;
  auto regp = [&](const std::string& name, const float** dst, std::vector<int64_t> shape) {
    reg_f32(m, name, &tmp, shape);
    *dst = tmp;
  };
  m->pose.ln_g = m->dec_norm.g;
  m->pose.ln_b = m->dec_norm.b;
  regp("head_pose_s.mlp.0.weight", &m->pose.w0, {512, kDecDim});
  regp("head_pose_s.mlp.0.bias", &m->pose.b0, {512});
  regp("head_pose_s.mlp.2.weight", &m->pose.w1, {512, 512});
  regp("head_pose_s.mlp.2.bias", &m->pose.b1, {512});
  regp("head_pose_s.mlp.4.weight", &m->pose.w2, {512, 512});
  regp("head_pose_s.mlp.4.bias", &m->pose.b2, {512});
  regp("head_pose_s.fc_t.weight", &m->pose.wt, {3, 512});
  regp("head_pose_s.fc_t.bias", &m->pose.bt, {3});
  regp("head_pose_s.fc_conf.0.weight", &m->pose.wc, {1, 512});
  regp("head_pose_s.fc_conf.0.bias", &m->pose.bc, {1});
  regp("head_pose_s.fc_rot.weight", &m->pose.wr, {9, 512});
  regp("head_pose_s.fc_rot.bias", &m->pose.br, {9});
  return 0;
}

// ---------------------------------------------------------------------------
// launch helpers (all increment the model's launch counter)
// ---------------------------------------------------------------------------
struct Ctx {
  StaModel* m;
  cudaStream_t st;
};

enum ProfCat { PROF_GEMM = 0, PROF_CONV = 1, PROF_ATTN = 2, PROF_LN = 3 };
// RAII scope: records an event pair around one launch when profiling is enabled
struct ProfScope {
  StaModel* m;
  cudaStream_t st;
  int cat;
  cudaEvent_t e0 = nullptr;
  ProfScope(const Ctx& c, int cat_, double flops) : m(c.m), st(c.st), cat(cat_) {
    if (!m->prof_on) return;
    m->prof_flops[cat] += flops;
    e0 = m->prof_event();
    cudaEventRecord(e0, st);
  }
  ~ProfScope() {
    if (!e0) return;
    cudaEvent_t e1 = m->prof_event();
    cudaEventRecord(e1, st);
    m->prof_recs.push_back({cat, e0, e1});
  }
};

int gemm(const Ctx& c, int amode, int epi, const void* A, long long lda, const Lin& L, GemmParams p) {
  GemmLaunch g;
  g.amode = amode;
  g.epi = epi;
  g.A = A;
  g.lda = lda;
  g.splitk_ws = c.m->splitk_ws;
  g.splitk_ws_bytes = c.m->splitk_ws ? StaModel::kSplitKBytes : 0;
  g.Wt = L.w;
  if (amode == A_FP8) {
    g.Wt = L.q;
    p.w_scale = L.qs;
  }
  g.ldw = L.K;
  p.N = L.N;
  p.K = L.K;
  if (!p.bias) p.bias = L.b;
  p.split = c.m->split;
  if (p.split && (epi == EPI_BF16 || epi == EPI_GELU || epi == EPI_ROPE)) p.ldo *= 3;  // (hi | lo | hi) output rows
  g.p = p;
  c.m->launches++;
  const double rows = (amode == A_CONV3) ? static_cast<double>(p.nimg) * p.H * p.W : static_cast<double>(p.M);
  ProfScope ps(c, amode == A_CONV3 ? PROF_CONV : PROF_GEMM, 2.0 * rows * L.N * L.K);
  return launch_gemm(g, c.st);
}
int set_rope(GemmParams& p, const int* pos, int rope_cols) {
  p.pos = pos;
  p.rope_cols = rope_cols;
  p.rope_tab = rope_table(&p.rope_max_pos);
  if (!p.rope_tab) {
    set_last_error("failed to build the RoPE table");
    return 1;
  }
  p.rope_smem_rows = 64;  // positions -1..62 from shared memory, larger ones from the global table
  return 0;
}
// plain linear on rows
int linear(const Ctx& c, int epi, const bf16* A, int M, const Lin& L, void* out, const void* resid = nullptr,
           const int* pos = nullptr, int rope_cols = 0, int rowmap_n = 0) {
  GemmParams p = {};
  p.M = M;
  p.out = out;
  p.ldo = L.N;
  p.resid = resid;
  p.rowmap_n = rowmap_n;
  if (epi == EPI_ROPE) RUN(set_rope(p, pos, rope_cols));
  return gemm(c, A_LINEAR, epi, A, L.K, L, p);
}
// FP8 mode: a trunk linear on e4m3 rows a.  EPI_F32: out += a W^T + b in place (the residual stream); EPI_ROPE: bf16 q/k/v
// rows for the attention kernel; EPI_GELU_FP8: e4m3 rows + scales into *q.
int linear_fp8(const Ctx& c, int epi, const Fp8Act& a, int M, const Lin& L, void* out, const int* pos = nullptr,
               int rope_cols = 0, const Fp8Act* q = nullptr) {
  GemmParams p = {};
  p.M = M;
  p.out = out;
  p.ldo = L.N;
  p.a_scale = a.s;
  if (epi == EPI_F32) p.resid = out;
  if (epi == EPI_ROPE) RUN(set_rope(p, pos, rope_cols));
  if (epi == EPI_GELU_FP8) {
    p.out = q->q;
    p.out_scale = q->s;
  }
  return gemm(c, A_FP8, epi, a.q, L.K, L, p);
}
int conv3(const Ctx& c, const bf16* in, int nimg, int H, int W, int Cin, const Lin& L, bf16* out, bf16* out_relu,
          const bf16* resid, const bf16* resid2, int relu_main) {
  GemmParams p = {};
  p.nimg = nimg;
  p.H = H;
  p.W = W;
  p.Cin = Cin * c.m->bmul();  // physical channels of the NHWC input
  p.out = out;
  p.out2 = out_relu;
  p.ldo = L.N;
  p.resid = resid;
  p.resid2 = resid2;
  p.relu_main = relu_main;
  return gemm(c, A_CONV3, EPI_BF16, in, 0, L, p);
}
int ln(const Ctx& c, const float* x, int rows, int C, const LNp& a, bf16* out1, const LNp* b2 = nullptr,
       bf16* out2 = nullptr, int drop_first_of = 0) {
  c.m->launches++;
  ProfScope ps(c, PROF_LN, 0.0);
  return launch_layernorm(x, rows, C, kLnEps, a.g, a.b, out1, b2 ? b2->g : nullptr, b2 ? b2->b : nullptr, out2,
                          drop_first_of, c.st, c.m->split);
}
int ln_fp8(const Ctx& c, const float* x, int rows, int C, const LNp& a, const Fp8Act& o1, const LNp* b2 = nullptr,
           const Fp8Act* o2 = nullptr) {
  c.m->launches++;
  ProfScope ps(c, PROF_LN, 0.0);
  return launch_layernorm_fp8(x, rows, C, kLnEps, a.g, a.b, o1.q, o1.s, b2 ? b2->g : nullptr, b2 ? b2->b : nullptr,
                              o2 ? o2->q : nullptr, o2 ? o2->s : nullptr, c.st);
}
// FP8 mode: bf16 attention output -> e4m3 (counted with the LayerNorms: both are row-wise bandwidth-bound passes)
int quant_fp8(const Ctx& c, const bf16* in, long long rows, int C, const Fp8Act& o) {
  c.m->launches++;
  ProfScope ps(c, PROF_LN, 0.0);
  return launch_quant_fp8(in, rows, C, o.q, o.s, c.st);
}
int attn(const Ctx& c, const bf16* q, long long ldq, int qc, const bf16* k, long long ldk, int kc, const bf16* v,
         long long ldv, int vc, bf16* out, long long ldo, int batch, int heads, int nq, int nk, int shift) {
  AttnLaunch a;
  const int bm = c.m->bmul();  // the ld* arguments are logical widths
  a.q = q; a.ldq = ldq * bm; a.q_col0 = qc;
  a.k = k; a.ldk = ldk * bm; a.k_col0 = kc;
  a.v = v; a.ldv = ldv * bm; a.v_col0 = vc;
  a.out = out; a.ldo = ldo * bm;
  a.batch = batch; a.heads = heads; a.nq = nq; a.nk = nk;
  a.kv_batch_shift = shift;
  a.split = c.m->split;
  a.scale = 0.125f;  // head_dim ** -0.5, sta_blocks.py:86
  c.m->launches++;
  ProfScope ps(c, PROF_ATTN, 4.0 * batch * heads * static_cast<double>(nq) * nk * 64);
  return launch_attention(a, c.st);
}

// Buffer taps (sta_set_taps): after the launch named fmt % i, copy `bytes` of its output at src to the tap of that name.
// The name is only formatted while taps are set.
int tap(const Ctx& c, const void* src, size_t bytes, const char* fmt, int i = 0) {
  StaModel* m = c.m;
  if (m->taps.empty()) return 0;
  char name[48];
  snprintf(name, sizeof(name), fmt, i);
  const auto it = m->taps.find(name);
  if (it == m->taps.end()) return 0;
  StaTap* t = it->second;
  if (t->dst) {
    if (t->written + static_cast<int64_t>(bytes) > t->capacity) {
      set_last_error(std::string("tap ") + name + ": capacity too small");
      return 2;
    }
    STA_CHECK_CUDA(cudaMemcpyAsync(static_cast<char*>(t->dst) + t->written, src, bytes, cudaMemcpyDeviceToDevice, c.st));
  }
  t->written += static_cast<int64_t>(bytes);
  t->fired++;
  return 0;
}
// bf16 activation rows of n logical elements, in bytes
size_t bf_bytes(const Ctx& c, size_t n) { return n * c.m->bmul() * sizeof(bf16); }
// FP8 activation rows: codes as fmt.q, scales as fmt.s
int tap_fp8(const Ctx& c, const Fp8Act& a, size_t rows, int C, const char* fmt, int i) {
  if (c.m->taps.empty()) return 0;
  const std::string f(fmt);
  RUN(tap(c, a.q, rows * C, (f + ".q").c_str(), i));
  return tap(c, a.s, rows * (C / 128) * sizeof(float), (f + ".s").c_str(), i);
}

// ---------------------------------------------------------------------------
// workspace: every entry point carves its buffers with the take functions below before its first launch, and
// ws_need sizes the allocation by a dry run of the same functions
// ---------------------------------------------------------------------------
EncBufs take_enc(Workspace& ws, int nimg, int N) {
  const size_t T = static_cast<size_t>(nimg) * N;
  EncBufs e;
  e.patches = ws.takeb(T * 768);
  e.lnb = ws.fp8 ? nullptr : ws.takeb(T * 1024);
  e.qkv = ws.takeb(T * 3072);
  e.att = ws.takeb(T * 1024);
  e.hid = ws.fp8 ? nullptr : ws.takeb(T * 4096);
  e.pos = ws.take<int>(T * 2);
  if (ws.fp8) {
    e.ln8 = ws.takeq(T, 1024);
    e.att8 = ws.takeq(T, 1024);
    e.hid8 = ws.takeq(T, 4096);
  }
  return e;
}
// The DPT head's four token inputs for nimg images of N tokens: [nimg*N][1024 | 768 | 768 | 768]
void take_hooks(Workspace& ws, int nimg, int N, bf16* hook[4]) {
  const size_t T = static_cast<size_t>(nimg) * N;
  hook[0] = ws.takeb(T * 1024);
  for (int q = 1; q < 4; ++q) hook[q] = ws.takeb(T * 768);
}
DecBufs take_dec(Workspace& ws, int S, int N) {
  const size_t Td = static_cast<size_t>(S) * (N + 1);
  DecBufs d;
  d.xd = ws.take<float>(Td * 768);
  d.ln1 = ws.fp8 ? nullptr : ws.takeb(Td * 768);
  d.lny = ws.fp8 ? nullptr : ws.takeb(Td * 768);
  d.qkv = ws.takeb(Td * 2304);
  d.att = ws.takeb(Td * 768);
  d.qc = ws.takeb(Td * 768);
  d.kvc = ws.takeb(Td * 1536);
  d.hid = ws.fp8 ? nullptr : ws.takeb(Td * 3072);
  take_hooks(ws, S, N, d.hook);
  d.pos = ws.take<int>(Td * 2);
  if (ws.fp8) {
    d.ln8 = ws.takeq(Td, 768);
    d.lny8 = ws.takeq(Td, 768);
    d.att8 = ws.takeq(Td, 768);
    d.hid8 = ws.takeq(Td, 3072);
  }
  return d;
}
// DPT head over up to nimg images of an h x w token grid
DptBufs take_dpt(Workspace& ws, int nimg, int h, int w) {
  const size_t N = static_cast<size_t>(h) * w, T = nimg * N;
  const size_t h4 = (h + 1) / 2, w4 = (w + 1) / 2;
  const size_t LP[4] = {16 * N, 4 * N, N, h4 * w4};  // pixels per image of the four levels
  DptBufs b;
  b.a0 = ws.takeb(T * 128);
  b.l1 = ws.takeb(nimg * LP[0] * 128);
  b.a1 = ws.takeb(T * 192);
  b.l2 = ws.takeb(nimg * LP[1] * 192);
  b.l3 = ws.takeb(T * 384);
  b.a3 = ws.takeb(T * 768);
  b.col4 = ws.takeb(nimg * LP[3] * 6912);
  b.l4 = ws.takeb(nimg * LP[3] * 768);
  for (int i = 0; i < 4; ++i) {
    b.r_raw[i] = ws.takeb(nimg * LP[i] * 256);
    b.r_relu[i] = ws.takeb(nimg * LP[i] * 256);
  }
  const size_t big = nimg * LP[0] * 256;
  b.t1 = ws.takeb(big);
  b.t2 = ws.takeb(big);
  b.s_raw = ws.takeb(big);
  b.s_relu = ws.takeb(big);
  b.o = ws.takeb(big);
  b.up = ws.takeb(nimg * 64 * N * 256);    // up, path: up to 8h x 8w
  b.path = ws.takeb(nimg * 64 * N * 256);
  b.hc1 = ws.takeb(nimg * 64 * N * 128);
  b.hup = ws.takeb(nimg * 256 * N * 128);  // full resolution
  return b;
}

// Staging rule of the graphed entry points: a graphed body may only touch memory whose address is a function of its
// graph key (run_graphed), so it writes workspace buffers, which flush() copies to the caller's tensors after the
// replay.  An eager body writes the caller's tensors directly and there is nothing to copy.  An output the caller did
// not ask for (null) stays null.
struct Staging {
  Workspace& ws;
  bool graphed;
  struct Copy { float* user; const float* staged; size_t n; };
  std::vector<Copy> copies;
  float* out(float* user, size_t n) {  // the buffer a body writes for the caller's user[0, n)
    if (!graphed || !user) return user;
    float* p = ws.take<float>(n);
    copies.push_back({user, p, n});
    return p;
  }
  int flush(cudaStream_t st) const {
    for (const Copy& c : copies)
      STA_CHECK_CUDA(cudaMemcpyAsync(c.user, c.staged, c.n * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return 0;
  }
};

// Outputs of the keyframe step for n edges, [view][edge] (view 0 = the i -> j direction): the DPT pointmaps and
// confidences, then what the pointmap consumers write and their scratch.  Null: not asked for.
struct PairOuts {
  float *pts, *conf, *intri, *depth, *cmean;
  void* scratch;
};
PairOuts stage_pair_outs(Staging& s, const PairOuts& u, int n, long long px) {
  const size_t V = 2 * static_cast<size_t>(n);
  PairOuts o;
  o.pts = s.out(u.pts, V * px * 3);
  o.conf = s.out(u.conf, V * px);
  o.intri = s.out(u.intri, static_cast<size_t>(n) * 9);
  o.depth = s.out(u.depth, V * px);
  o.cmean = s.out(u.cmean, V);
  o.scratch = s.graphed && u.intri ? s.ws.take<double>(pointmap_scratch_bytes(V) / sizeof(double)) : u.scratch;
  return o;
}

// Workspace bytes for nimg images of an h x w token grid: a dry run of the take functions.  The envelope covers every
// entry point: encoder + fp32 residual stream + decoder + DPT head (sta_forward_pairs), and on top of the decoder the
// keyframe step's staged poses (_begin), compact hook copies and staged outputs (_finish with every edge kept and every
// output asked for).
size_t ws_need(int nimg, int h, int w, int bmul, int fp8) {
  Workspace dry;
  dry.bmul = bmul;
  dry.fp8 = fp8;
  const int N = h * w;
  float any;  // stands for a caller's tensor: staging only asks whether there is one
  bf16* hook[4];
  take_enc(dry, nimg, N);
  dry.take<float>(static_cast<size_t>(nimg) * N * kEncDim);
  take_dec(dry, nimg, N);
  take_dpt(dry, nimg, h, w);
  Staging staged{dry, true};
  staged.out(&any, static_cast<size_t>(nimg) * 16);
  staged.out(&any, nimg);
  take_hooks(dry, nimg, N, hook);
  stage_pair_outs(staged, {&any, &any, &any, &any, &any, &any}, nimg / 2, 256LL * N);
  return dry.off;
}

void drop_graphs(StaModel* m);

int ensure_ws(StaModel* m, int nimg, int h, int w) {
  const size_t need = ws_need(nimg, h, w, m->bmul(), m->fp8);
  m->ws.bmul = m->bmul();
  m->ws.fp8 = m->fp8;
  if (m->ws.bytes < need) {
    STA_CHECK_CUDA(cudaDeviceSynchronize());
    drop_graphs(m);  // they point into the old workspace
    if (m->ws.base) STA_CHECK_CUDA(cudaFree(m->ws.base));
    m->ws.base = nullptr;
    m->ws.bytes = 0;
    STA_CHECK_CUDA(cudaMalloc(&m->ws.base, need));
    m->ws.bytes = need;
  }
  m->ws.off = 0;
  m->ws.overflow = false;
  return 0;
}
int check_ws(const Workspace& ws) {
  STA_REQUIRE(!ws.overflow, "internal: the workspace is smaller than the buffers this call carves");
  return 0;
}

// ---------------------------------------------------------------------------
// Small-batch calls (one keyframe, a handful of edges) are launch-bound: ~170-400 kernels of a few microseconds each.
// run_graphed() runs `body(ctx)` eagerly the first time a key is seen (lazy initialisation such as
// cudaFuncSetAttribute / the RoPE table happens there), captures it into a CUDA graph on the second call (on a private
// stream -- the caller's may be the legacy default stream -- with the programmatic-dependent-launch edges kept) and
// replays the instantiated graph on the caller's stream from then on.  `body` must only touch memory whose
// addresses are a function of the key (workspace offsets for that shape, weights): user pointers are handled by
// the caller outside the graph (Staging).  Graphs die with the workspace they point into.  Sizes that are not
// launch-bound (`graphed` false) always run eagerly.
// ---------------------------------------------------------------------------
constexpr long long kGraphMaxTokens = 8192;  // only launch-bound problem sizes

void drop_graphs(StaModel* m) {
  for (auto& g : m->graphs)
    if (g.exec) cudaGraphExecDestroy(g.exec);
  m->graphs.clear();
}

template <typename Body>
int run_graphed(StaModel* m, cudaStream_t st, bool graphed, const std::vector<long long>& key, Body&& body) {
  // per-kernel timing events and buffer taps need eager launches
  if (!graphed || m->prof_on || !m->taps.empty()) return body(Ctx{m, st});
  StaModel::GraphEntry* ent = nullptr;
  for (auto& g : m->graphs)
    if (g.key == key) ent = &g;
  if (!ent) {
    if (m->graphs.size() >= 32) drop_graphs(m);
    m->graphs.emplace_back();
    m->graphs.back().key = key;
    return body(Ctx{m, st});  // first sighting: eager
  }
  if (ent->unsupported) return body(Ctx{m, st});
  if (!ent->exec) {
    if (!m->s_cap) STA_CHECK_CUDA(cudaStreamCreateWithFlags(&m->s_cap, cudaStreamNonBlocking));
    const int64_t l0 = m->launches;
    STA_CHECK_CUDA(cudaStreamBeginCapture(m->s_cap, cudaStreamCaptureModeThreadLocal));
    const int rc = body(Ctx{m, m->s_cap});
    cudaGraph_t graph = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(m->s_cap, &graph);
    if (rc != 0) {
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();
      return rc;
    }
    cudaGraphExec_t exec = nullptr;
    if (ce != cudaSuccess || graph == nullptr || cudaGraphInstantiate(&exec, graph, 0) != cudaSuccess) {
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();  // clear; fall back to eager launches for this key
      ent->unsupported = true;
      m->launches = l0;
      return body(Ctx{m, st});
    }
    cudaGraphDestroy(graph);
    ent->exec = exec;
    ent->launches = m->launches - l0;
    m->launches = l0;
  }
  STA_CHECK_CUDA(cudaGraphLaunch(ent->exec, st));
  m->launches += ent->launches;
  m->graph_replays++;
  return 0;
}

// ---------------------------------------------------------------------------
// encoder over nimg images whose patches (e.patches) and positions (e.pos) are prepared.
// x: fp32 residual stream [nimg*N][1024], provided by the caller (user buffer or workspace);
// on return it holds the un-normalised encoder features (normalize=False, sta_model.py:172).
// ---------------------------------------------------------------------------
int run_encoder(const Ctx& c, int nimg, int N, float* x, EncBufs& e) {
  StaModel* m = c.m;
  const int T = nimg * N;
  const size_t xb = static_cast<size_t>(T) * kEncDim * sizeof(float);
  RUN(linear(c, EPI_F32, e.patches, T, m->patch, x));
  RUN(tap(c, x, xb, "enc.embed"));
  for (int l = 0; l < 24; ++l) {
    const EncBlock& b = m->enc[l];
    if (m->fp8) {
      RUN(ln_fp8(c, x, T, kEncDim, b.n1, e.ln8));
      RUN(tap_fp8(c, e.ln8, T, kEncDim, "enc.%d.ln1", l));
      RUN(linear_fp8(c, EPI_ROPE, e.ln8, T, b.qkv, e.qkv, e.pos, 2 * kEncDim));
      RUN(tap(c, e.qkv, bf_bytes(c, T * 3 * kEncDim), "enc.%d.qkv", l));
      RUN(attn(c, e.qkv, 3 * kEncDim, 0, e.qkv, 3 * kEncDim, kEncDim, e.qkv, 3 * kEncDim, 2 * kEncDim, e.att, kEncDim,
               nimg, kEncHeads, N, N, 0));
      RUN(tap(c, e.att, bf_bytes(c, T * kEncDim), "enc.%d.att", l));
      RUN(quant_fp8(c, e.att, T, kEncDim, e.att8));
      RUN(tap_fp8(c, e.att8, T, kEncDim, "enc.%d.att8", l));
      RUN(linear_fp8(c, EPI_F32, e.att8, T, b.proj, x));
      RUN(tap(c, x, xb, "enc.%d.x_attn", l));
      RUN(ln_fp8(c, x, T, kEncDim, b.n2, e.ln8));
      RUN(tap_fp8(c, e.ln8, T, kEncDim, "enc.%d.ln2", l));
      RUN(linear_fp8(c, EPI_GELU_FP8, e.ln8, T, b.fc1, nullptr, nullptr, 0, &e.hid8));
      RUN(tap_fp8(c, e.hid8, T, 4 * kEncDim, "enc.%d.hid", l));
      RUN(linear_fp8(c, EPI_F32, e.hid8, T, b.fc2, x));
      RUN(tap(c, x, xb, "enc.%d.x", l));
      continue;
    }
    RUN(ln(c, x, T, kEncDim, b.n1, e.lnb));
    RUN(tap(c, e.lnb, bf_bytes(c, T * kEncDim), "enc.%d.ln1", l));
    RUN(linear(c, EPI_ROPE, e.lnb, T, b.qkv, e.qkv, nullptr, e.pos, 2 * kEncDim));
    RUN(tap(c, e.qkv, bf_bytes(c, T * 3 * kEncDim), "enc.%d.qkv", l));
    RUN(attn(c, e.qkv, 3 * kEncDim, 0, e.qkv, 3 * kEncDim, kEncDim, e.qkv, 3 * kEncDim, 2 * kEncDim, e.att, kEncDim,
             nimg, kEncHeads, N, N, 0));
    RUN(tap(c, e.att, bf_bytes(c, T * kEncDim), "enc.%d.att", l));
    RUN(linear(c, EPI_F32, e.att, T, b.proj, x, x));
    RUN(tap(c, x, xb, "enc.%d.x_attn", l));
    RUN(ln(c, x, T, kEncDim, b.n2, e.lnb));
    RUN(tap(c, e.lnb, bf_bytes(c, T * kEncDim), "enc.%d.ln2", l));
    RUN(linear(c, EPI_GELU, e.lnb, T, b.fc1, e.hid));
    RUN(tap(c, e.hid, bf_bytes(c, T * 4 * kEncDim), "enc.%d.hid", l));
    RUN(linear(c, EPI_F32, e.hid, T, b.fc2, x, x));
    RUN(tap(c, x, xb, "enc.%d.x", l));
  }
  return 0;
}

// ---------------------------------------------------------------------------
// symmetric decoder over S = 2B samples (samples [0,B) = view 1, [B,2B) = view 2).
// d.hook[0] (bf16 encoder features of all S samples) and d.pos must be filled.
// outs: optional 2 x 13 fp32 per-layer outputs (compat path), may be null.
// ---------------------------------------------------------------------------
int run_decoder(const Ctx& c, int B, int N, DecBufs& d, float* const* out1, float* const* out2) {
  StaModel* m = c.m;
  const int S = 2 * B, M = N + 1, T = S * N, Td = S * M;
  const long long half = static_cast<long long>(B) * M * kDecDim;
  const size_t xb = static_cast<size_t>(Td) * kDecDim * sizeof(float);
  const size_t hb = bf_bytes(c, static_cast<size_t>(T) * kDecDim);  // a decoder hook: the pose rows dropped
  auto emit = [&](int idx) -> int {
    if (out1 && out1[idx]) {
      m->launches++;
      RUN(launch_copy_f32(d.xd, out1[idx], half, c.st));
      RUN(tap(c, out1[idx], half * sizeof(float), "dec.out"));
    }
    if (out2 && out2[idx]) {
      m->launches++;
      RUN(launch_copy_f32(d.xd + half, out2[idx], half, c.st));
      RUN(tap(c, out2[idx], half * sizeof(float), "dec.out"));
    }
    return 0;
  };
  RUN(linear(c, EPI_F32, d.hook[0], T, m->dec_embed, d.xd, nullptr, nullptr, 0, N));
  RUN(tap(c, d.xd, xb, "dec.embed"));
  m->launches++;
  RUN(launch_fill_pose_token(d.xd, m->pose_tok, S, M, kDecDim, c.st));
  RUN(tap(c, d.xd, xb, "dec.pose_tok"));
  RUN(emit(0));
  for (int l = 0; l < 12; ++l) {
    const DecBlock& b = m->dec[l];
    const size_t lnb = bf_bytes(c, static_cast<size_t>(Td) * kDecDim);
    if (m->fp8) {  // the same sequence with e4m3 operands for every linear
      RUN(ln_fp8(c, d.xd, Td, kDecDim, b.n1, d.ln8, &b.ny, &d.lny8));
      RUN(tap_fp8(c, d.ln8, Td, kDecDim, "dec.%d.ln1", l));
      RUN(tap_fp8(c, d.lny8, Td, kDecDim, "dec.%d.lny", l));
      RUN(linear_fp8(c, EPI_ROPE, d.ln8, Td, b.qkv, d.qkv, d.pos, 2 * kDecDim));
      RUN(tap(c, d.qkv, 3 * lnb, "dec.%d.qkv", l));
      RUN(attn(c, d.qkv, 3 * kDecDim, 0, d.qkv, 3 * kDecDim, kDecDim, d.qkv, 3 * kDecDim, 2 * kDecDim, d.att, kDecDim, S,
               kDecHeads, M, M, 0));
      RUN(tap(c, d.att, lnb, "dec.%d.att", l));
      RUN(quant_fp8(c, d.att, Td, kDecDim, d.att8));
      RUN(tap_fp8(c, d.att8, Td, kDecDim, "dec.%d.att8", l));
      RUN(linear_fp8(c, EPI_F32, d.att8, Td, b.proj, d.xd));
      RUN(tap(c, d.xd, xb, "dec.%d.x_self", l));
      RUN(linear_fp8(c, EPI_ROPE, d.lny8, Td, b.ckv, d.kvc, d.pos, kDecDim));
      RUN(tap(c, d.kvc, 2 * lnb, "dec.%d.kvc", l));
      RUN(ln_fp8(c, d.xd, Td, kDecDim, b.n2, d.ln8));
      RUN(tap_fp8(c, d.ln8, Td, kDecDim, "dec.%d.ln2", l));
      RUN(linear_fp8(c, EPI_ROPE, d.ln8, Td, b.cq, d.qc, d.pos, kDecDim));
      RUN(tap(c, d.qc, lnb, "dec.%d.qc", l));
      RUN(attn(c, d.qc, kDecDim, 0, d.kvc, 2 * kDecDim, 0, d.kvc, 2 * kDecDim, kDecDim, d.att, kDecDim, S, kDecHeads, M,
               M, B));
      RUN(tap(c, d.att, lnb, "dec.%d.catt", l));
      RUN(quant_fp8(c, d.att, Td, kDecDim, d.att8));
      RUN(tap_fp8(c, d.att8, Td, kDecDim, "dec.%d.catt8", l));
      RUN(linear_fp8(c, EPI_F32, d.att8, Td, b.cproj, d.xd));
      RUN(tap(c, d.xd, xb, "dec.%d.x_cross", l));
      RUN(ln_fp8(c, d.xd, Td, kDecDim, b.n3, d.ln8));
      RUN(tap_fp8(c, d.ln8, Td, kDecDim, "dec.%d.ln3", l));
      RUN(linear_fp8(c, EPI_GELU_FP8, d.ln8, Td, b.fc1, nullptr, nullptr, 0, &d.hid8));
      RUN(tap_fp8(c, d.hid8, Td, 4 * kDecDim, "dec.%d.hid", l));
      RUN(linear_fp8(c, EPI_F32, d.hid8, Td, b.fc2, d.xd));
      RUN(tap(c, d.xd, xb, "dec.%d.x", l));
    } else {
    // self-attention on norm1(x); norm_y(x) is what the partner view cross-attends to
    RUN(ln(c, d.xd, Td, kDecDim, b.n1, d.ln1, &b.ny, d.lny));
    RUN(tap(c, d.ln1, lnb, "dec.%d.ln1", l));
    RUN(tap(c, d.lny, lnb, "dec.%d.lny", l));
    RUN(linear(c, EPI_ROPE, d.ln1, Td, b.qkv, d.qkv, nullptr, d.pos, 2 * kDecDim));
    RUN(tap(c, d.qkv, 3 * lnb, "dec.%d.qkv", l));
    RUN(attn(c, d.qkv, 3 * kDecDim, 0, d.qkv, 3 * kDecDim, kDecDim, d.qkv, 3 * kDecDim, 2 * kDecDim, d.att, kDecDim, S,
             kDecHeads, M, M, 0));
    RUN(tap(c, d.att, lnb, "dec.%d.att", l));
    RUN(linear(c, EPI_F32, d.att, Td, b.proj, d.xd, d.xd));
    RUN(tap(c, d.xd, xb, "dec.%d.x_self", l));
    // cross-attention: q from norm2(x), k/v from norm_y(partner input) -- kv sample = (s + B) % 2B
    RUN(linear(c, EPI_ROPE, d.lny, Td, b.ckv, d.kvc, nullptr, d.pos, kDecDim));
    RUN(tap(c, d.kvc, 2 * lnb, "dec.%d.kvc", l));
    RUN(ln(c, d.xd, Td, kDecDim, b.n2, d.ln1));
    RUN(tap(c, d.ln1, lnb, "dec.%d.ln2", l));
    RUN(linear(c, EPI_ROPE, d.ln1, Td, b.cq, d.qc, nullptr, d.pos, kDecDim));
    RUN(tap(c, d.qc, lnb, "dec.%d.qc", l));
    RUN(attn(c, d.qc, kDecDim, 0, d.kvc, 2 * kDecDim, 0, d.kvc, 2 * kDecDim, kDecDim, d.att, kDecDim, S, kDecHeads, M, M,
             B));
    RUN(tap(c, d.att, lnb, "dec.%d.catt", l));
    RUN(linear(c, EPI_F32, d.att, Td, b.cproj, d.xd, d.xd));
    RUN(tap(c, d.xd, xb, "dec.%d.x_cross", l));
    // MLP
    RUN(ln(c, d.xd, Td, kDecDim, b.n3, d.ln1));
    RUN(tap(c, d.ln1, lnb, "dec.%d.ln3", l));
    RUN(linear(c, EPI_GELU, d.ln1, Td, b.fc1, d.hid));
    RUN(tap(c, d.hid, 4 * lnb, "dec.%d.hid", l));
    RUN(linear(c, EPI_F32, d.hid, Td, b.fc2, d.xd, d.xd));
    RUN(tap(c, d.xd, xb, "dec.%d.x", l));
    }
    if (l + 1 == 6 || l + 1 == 9) {  // DPT hooks [0, 7, 10, 13] -> decoder outputs 6, 9, 12 (dpt_head.py:112)
      const int q = l + 1 == 6 ? 1 : 2;
      m->launches++;
      RUN(launch_cast_f32_bf16(d.xd, d.hook[q], Td, kDecDim, M, c.st, m->split));
      RUN(tap(c, d.hook[q], hb, "dec.hook%d", q));
    }
    if (l + 1 < 12) RUN(emit(l + 1));
  }
  // dec_norm on the last output; bf16 copy without the pose token feeds the DPT head
  RUN(ln(c, d.xd, Td, kDecDim, m->dec_norm, d.hook[3], nullptr, nullptr, M));
  RUN(tap(c, d.hook[3], hb, "dec.hook3"));
  if ((out1 && out1[12]) || (out2 && out2[12])) {
    // compat path: fp32 LayerNorm-ed last layer
    const int rows_half = B * M;
    if (out1 && out1[12]) {
      m->launches++;
      layernorm_f32_kernel<<<(rows_half + 7) / 8, 256, 0, c.st>>>(d.xd, rows_half, kDecDim, kLnEps, m->dec_norm.g,
                                                                  m->dec_norm.b, out1[12]);
      RUN(tap(c, out1[12], half * sizeof(float), "dec.out"));
    }
    if (out2 && out2[12]) {
      m->launches++;
      layernorm_f32_kernel<<<(rows_half + 7) / 8, 256, 0, c.st>>>(d.xd + half, rows_half, kDecDim, kLnEps,
                                                                  m->dec_norm.g, m->dec_norm.b, out2[12]);
      RUN(tap(c, out2[12], half * sizeof(float), "dec.out"));
    }
    STA_CHECK_CUDA(cudaGetLastError());
  }
  return 0;
}

// bf16 decoder input of B feature pairs: the B view-1 samples, then the B view-2 samples
int cast_features(const Ctx& c, const float* feat1, const float* feat2, int B, int N, DecBufs& d) {
  const long long T = static_cast<long long>(B) * N;
  c.m->launches += 2;
  RUN(launch_cast_f32_bf16(feat1, d.hook[0], T, kEncDim, 0, c.st, c.m->split));
  RUN(tap(c, d.hook[0], bf_bytes(c, T * kEncDim), "dec.hook0"));
  RUN(launch_cast_f32_bf16(feat2, d.hook[0] + T * kEncDim * c.m->bmul(), T, kEncDim, 0, c.st, c.m->split));
  return tap(c, d.hook[0] + T * kEncDim * c.m->bmul(), bf_bytes(c, T * kEncDim), "dec.hook0");
}

// Decoder positions, the symmetric decoder over 2B samples (d.hook[0] must be filled) and the pose heads on the
// dec_norm-ed pose tokens of both views: view 1 into pose / pose_conf, view 2 `view_stride` entries further.
int decode_with_poses(const Ctx& c, int B, int h, int w, DecBufs& d, float* pose, float* pose_conf, int view_stride) {
  StaModel* m = c.m;
  const long long rows = static_cast<long long>(h * w + 1) * kDecDim;  // decoder rows of one sample
  m->launches += 3;
  RUN(launch_make_positions(d.pos, 2 * B, h, w, 1, c.st));
  RUN(tap(c, d.pos, 2 * static_cast<size_t>(B) * (h * w + 1) * 2 * sizeof(int), "pos.dec"));
  RUN(run_decoder(c, B, h * w, d, nullptr, nullptr));
  for (int v = 0; v < 2; ++v) {
    float* p = pose + static_cast<long long>(v) * view_stride * 16;
    float* pc = pose_conf + static_cast<long long>(v) * view_stride;
    RUN(launch_pose_head(d.xd + v * B * rows, rows, B, 1, kLnEps, m->pose, p, pc, c.st));
    RUN(tap(c, p, static_cast<size_t>(B) * 16 * sizeof(float), "pose"));
    RUN(tap(c, pc, static_cast<size_t>(B) * sizeof(float), "pose_conf"));
  }
  return 0;
}

// ---------------------------------------------------------------------------
// DPT head over images [first, first + nimg) of the four bf16 token inputs hook[q] ([images * N][1024 | 768 | 768 |
// 768], take_hooks), into pts3d / conf (the outputs of those nimg images).  b: take_dpt for at least nimg images.
// ---------------------------------------------------------------------------
int run_dpt(const Ctx& c, const DptBufs& b, int h, int w, const bf16* const hook[4], int first, int nimg, float* pts3d,
            float* conf) {
  StaModel* m = c.m;
  const int N = h * w, T = nimg * N;
  const int h4 = (h + 1) / 2, w4 = (w + 1) / 2;
  const int LH[4] = {4 * h, 2 * h, h, h4}, LW[4] = {4 * w, 2 * w, w, w4};
  const size_t tok0 = static_cast<size_t>(first) * N * m->bmul();  // first token row, times the bf16 row width factor
  const bf16 *hook0 = hook[0] + tok0 * 1024, *hook1 = hook[1] + tok0 * 768, *hook2 = hook[2] + tok0 * 768,
             *hook3 = hook[3] + tok0 * 768;

  // ---- act_postprocess (dpt_block.py:356-410) ----
  const size_t T4 = static_cast<size_t>(nimg) * h4 * w4;
  RUN(linear(c, EPI_BF16, hook0, T, m->act0, b.a0));
  RUN(tap(c, b.a0, bf_bytes(c, static_cast<size_t>(T) * 128), "dpt.a0"));
  {
    GemmParams p = {};
    p.M = T; p.out = b.l1; p.ps_k = 4; p.ps_cout = 128; p.ps_h = h; p.ps_w = w;
    RUN(gemm(c, A_LINEAR, EPI_PIXSHUF, b.a0, m->act0T.K, m->act0T, p));
    RUN(tap(c, b.l1, bf_bytes(c, static_cast<size_t>(T) * 16 * 128), "dpt.l1"));
  }
  RUN(linear(c, EPI_BF16, hook1, T, m->act1, b.a1));
  RUN(tap(c, b.a1, bf_bytes(c, static_cast<size_t>(T) * 192), "dpt.a1"));
  {
    GemmParams p = {};
    p.M = T; p.out = b.l2; p.ps_k = 2; p.ps_cout = 192; p.ps_h = h; p.ps_w = w;
    RUN(gemm(c, A_LINEAR, EPI_PIXSHUF, b.a1, m->act1T.K, m->act1T, p));
    RUN(tap(c, b.l2, bf_bytes(c, static_cast<size_t>(T) * 4 * 192), "dpt.l2"));
  }
  RUN(linear(c, EPI_BF16, hook2, T, m->act2, b.l3));
  RUN(tap(c, b.l3, bf_bytes(c, static_cast<size_t>(T) * 384), "dpt.l3"));
  RUN(linear(c, EPI_BF16, hook3, T, m->act3, b.a3));
  RUN(tap(c, b.a3, bf_bytes(c, static_cast<size_t>(T) * 768), "dpt.a3"));
  m->launches++;
  RUN(launch_im2col_3x3_s2(b.a3, b.col4, nimg, h, w, 768 * m->bmul(), c.st));  // pure channel-vector copy
  RUN(tap(c, b.col4, bf_bytes(c, T4 * 9 * 768), "dpt.col4"));
  RUN(linear(c, EPI_BF16, b.col4, nimg * h4 * w4, m->act3c, b.l4));
  RUN(tap(c, b.l4, bf_bytes(c, T4 * 768), "dpt.l4"));
  // ---- layer_rn: 3x3 conv to 256 channels, no bias (dpt_block.py:33-75); raw + relu copies ----
  const bf16* lin[4] = {b.l1, b.l2, b.l3, b.l4};
  const int lc[4] = {128, 192, 384, 768};
  for (int i = 0; i < 4; ++i) {
    RUN(conv3(c, lin[i], nimg, LH[i], LW[i], lc[i], m->rn[i], b.r_raw[i], b.r_relu[i], nullptr, nullptr, 0));
    const size_t rb = bf_bytes(c, static_cast<size_t>(nimg) * LH[i] * LW[i] * 256);
    RUN(tap(c, b.r_raw[i], rb, "dpt.rn%d.raw", i));
    RUN(tap(c, b.r_relu[i], rb, "dpt.rn%d.relu", i));
  }

  // ---- refinenet4 .. refinenet1 (dpt_block.py:189-218, dpt_head.py:58-61) ----
  const bf16* path = nullptr;  // output of the previous (coarser) fusion block at this level's resolution
  for (int lvl = 3; lvl >= 0; --lvl) {
    const Refine& r = m->ref[lvl];
    const int Hh = LH[lvl], Ww = LW[lvl];
    const size_t lb = bf_bytes(c, static_cast<size_t>(nimg) * Hh * Ww * 256);  // one 256-channel map of this level
    const bf16* s_raw;
    const bf16* s_relu;
    if (lvl == 3) {
      s_raw = b.r_raw[3];
      s_relu = b.r_relu[3];
    } else {
      // res = RCU1(layer); s = path + res
      RUN(conv3(c, b.r_relu[lvl], nimg, Hh, Ww, 256, r.r1.c1, b.t1, nullptr, nullptr, nullptr, 1));
      RUN(tap(c, b.t1, lb, "dpt.ref%d.t1", lvl));
      RUN(conv3(c, b.t1, nimg, Hh, Ww, 256, r.r1.c2, b.s_raw, b.s_relu, b.r_raw[lvl], path, 0));
      RUN(tap(c, b.s_raw, lb, "dpt.ref%d.s_raw", lvl));
      RUN(tap(c, b.s_relu, lb, "dpt.ref%d.s_relu", lvl));
      s_raw = b.s_raw;
      s_relu = b.s_relu;
    }
    // out = RCU2(s)
    RUN(conv3(c, s_relu, nimg, Hh, Ww, 256, r.r2.c1, b.t2, nullptr, nullptr, nullptr, 1));
    RUN(tap(c, b.t2, lb, "dpt.ref%d.t2", lvl));
    RUN(conv3(c, b.t2, nimg, Hh, Ww, 256, r.r2.c2, b.o, nullptr, s_raw, nullptr, 0));
    RUN(tap(c, b.o, lb, "dpt.ref%d.o", lvl));
    // bilinear x2 (align_corners=True), cropped to the next level's size for refinenet4 (dpt_head.py:58)
    // The reference applies out_conv (1x1) AFTER the upsample (dpt_block.py:215-217).  Both are linear and the
    // bilinear weights sum to one, so conv1x1(up(x)) == up(conv1x1(x)) exactly in real arithmetic; doing the
    // 1x1 at the low resolution costs a quarter of the FLOPs and HBM bytes.
    int OH = 2 * Hh, OW = 2 * Ww;
    if (lvl == 3) { OH = LH[2]; OW = LW[2]; }
    RUN(linear(c, EPI_BF16, b.o, nimg * Hh * Ww, r.out, b.up));
    RUN(tap(c, b.up, lb, "dpt.ref%d.up", lvl));
    m->launches++;
    RUN(launch_upsample2x(b.up, b.path, nimg, Hh, Ww, 256, OH, OW, c.st, m->split));
    RUN(tap(c, b.path, bf_bytes(c, static_cast<size_t>(nimg) * OH * OW * 256), "dpt.ref%d.path", lvl));
    path = b.path;
  }
  // ---- head (dpt_block.py:318-324) + postprocess (postprocess.py:10-62) ----
  const int H8 = 8 * h, W8 = 8 * w;
  const size_t px8 = static_cast<size_t>(nimg) * H8 * W8;
  RUN(conv3(c, b.path, nimg, H8, W8, 256, m->head0, b.hc1, nullptr, nullptr, nullptr, 0));
  RUN(tap(c, b.hc1, bf_bytes(c, px8 * 128), "dpt.hc1"));
  m->launches++;
  RUN(launch_upsample2x(b.hc1, b.hup, nimg, H8, W8, 128, 2 * H8, 2 * W8, c.st, m->split));
  RUN(tap(c, b.hup, bf_bytes(c, 4 * px8 * 128), "dpt.hup"));
  {
    GemmParams p = {};
    p.nimg = nimg; p.H = 2 * H8; p.W = 2 * W8; p.Cin = 128 * m->bmul();
    p.head_w = m->head4_w; p.head_b = m->head4_b; p.pts3d = pts3d; p.conf = conf;
    RUN(gemm(c, A_CONV3, EPI_HEAD, b.hup, 0, m->head2, p));
    RUN(tap(c, pts3d, 4 * px8 * 3 * sizeof(float), "dpt.pts3d"));
    RUN(tap(c, conf, 4 * px8 * sizeof(float), "dpt.conf"));
  }
  return 0;
}

// Every model entry point starts here.  All but sta_regress_pairs_finish end a begin/finish pair: they may carve the
// workspace that holds _begin's decoder hooks again.
int check_ready(StaModel* m, bool finishing_pairs = false) {
  if (!m) {
    set_last_error("null model handle");
    return 2;
  }
  if (!finishing_pairs) m->rp = {};
  if (m->missing != 0) {
    char buf[128];
    snprintf(buf, sizeof(buf), "model is missing %d state-dict tensors", m->missing);
    set_last_error(buf);
    return 2;
  }
  return 0;
}
// B images of positive multiples of the 16-pixel patch, whose token grid fits the RoPE table
int check_grid(int B, int H, int W) {
  STA_REQUIRE(B > 0 && H % 16 == 0 && W % 16 == 0 && H > 0 && W > 0, "image size must be a positive multiple of 16");
  STA_REQUIRE(H / 16 <= 1024 && W / 16 <= 1024, "token grid exceeds the RoPE table");
  return 0;
}
int check_edges(const StaModel* m, int K) {
  STA_REQUIRE(K > 0 && K <= m->max_pairs_per_chunk, "edge batch must be in [1, 16]");
  return 0;
}
// The pointmap consumers run when any of their outputs is asked for; they then need the scratch buffer and intri_out.
int check_consumers(const void* scratch, const float* intri_out, const float* depth_out, const float* conf_mean_out) {
  if (intri_out || depth_out || conf_mean_out)
    STA_REQUIRE(scratch != nullptr && intri_out != nullptr,
                "the pointmap consumers need the scratch buffer and intri_out (depth_out / conf_mean_out are optional)");
  return 0;
}

// The keyframe step after the decoder, for n edges whose token inputs hold [view][edge] images: the DPT head on each
// view, then the pointmap consumers if they were asked for (o.intri is set exactly then, check_consumers).
int pair_heads(const Ctx& c, const DptBufs& b, const bf16* const hook[4], int n, int H, int W, const PairOuts& o) {
  const long long px = static_cast<long long>(H) * W;
  for (int v = 0; v < 2; ++v)
    RUN(run_dpt(c, b, H / 16, W / 16, hook, v * n, n, o.pts + v * n * px * 3, o.conf + v * n * px));
  if (!o.intri) return 0;
  c.m->launches += 2;
  return launch_pointmap_consumers(o.pts, o.conf, 2 * n, H, W, 2, o.intri, o.depth, o.cmean, o.scratch, c.st);
}

// DPT parts per view in the host entry point: two halves, so that the device-to-host copy of the first half overlaps
// the DPT of the second.
int host_dpt_parts(int B) { return B >= 2 ? 2 : 1; }

// one stream per handle at a time: order a call on `st` after everything this handle enqueued on its previous stream
int enter_stream(StaModel* m, cudaStream_t st) {
  if (m->has_last_stream && m->last_stream != st) {
    if (!m->ev_switch) STA_CHECK_CUDA(cudaEventCreateWithFlags(&m->ev_switch, cudaEventDisableTiming));
    STA_CHECK_CUDA(cudaEventRecord(m->ev_switch, m->last_stream));
    STA_CHECK_CUDA(cudaStreamWaitEvent(st, m->ev_switch, 0));
  }
  m->last_stream = st;
  m->has_last_stream = true;
  return 0;
}

int forward_chunk(const Ctx& c, const void* img1, const void* img2, int img_is_bf16, int B, int H, int W,
                  float* pts3d, float* conf, float* pose, float* pose_conf, int B_total,
                  cudaEvent_t* ev_parts = nullptr) {
  StaModel* m = c.m;
  const int h = H / 16, w = W / 16, N = h * w, S = 2 * B;
  RUN(ensure_ws(m, S, h, w));
  Workspace& ws = m->ws;
  float* x = ws.take<float>(static_cast<size_t>(S) * N * kEncDim);
  EncBufs e = take_enc(ws, S, N);
  DecBufs d = take_dec(ws, S, N);
  const DptBufs dpt = take_dpt(ws, B, h, w);  // one view; the parts of the host entry point reuse it
  RUN(check_ws(ws));
  // encode both views as one batch of 2B images: [view 1 batch ; view 2 batch]
  m->launches += 3;
  const size_t bm = m->bmul();  // physical / logical width of the bf16 activation rows
  const size_t pb = bf_bytes(c, static_cast<size_t>(B) * N * 768);  // one view's patches
  RUN(launch_patch_im2col(img1, img_is_bf16, B, H, W, e.patches, c.st, m->split));
  RUN(tap(c, e.patches, pb, "patches"));
  RUN(launch_patch_im2col(img2, img_is_bf16, B, H, W, e.patches + static_cast<size_t>(B) * N * 768 * bm, c.st, m->split));
  RUN(tap(c, e.patches + static_cast<size_t>(B) * N * 768 * bm, pb, "patches"));
  RUN(launch_make_positions(e.pos, S, h, w, 0, c.st));
  RUN(tap(c, e.pos, static_cast<size_t>(S) * N * 2 * sizeof(int), "pos.enc"));
  RUN(run_encoder(c, S, N, x, e));
  m->launches += 1;
  RUN(launch_cast_f32_bf16(x, d.hook[0], static_cast<long long>(S) * N, kEncDim, 0, c.st, m->split));
  RUN(tap(c, d.hook[0], bf_bytes(c, static_cast<size_t>(S) * N * kEncDim), "dec.hook0"));
  // pose outputs are laid out [2][B_total]: view 1 block then view 2 block
  RUN(decode_with_poses(c, B, h, w, d, pose, pose_conf, B_total));
  // DPT heads: view 1 images then view 2 images (outputs are [2][B_total] blocks).  The host entry point passes events:
  // each view is then processed in `halves` parts (host_dpt_parts) and an event is recorded after every part, so that the
  // D2H copy of one part runs under the head of the next and only the last quarter of the outputs is exposed.
  const long long px = static_cast<long long>(H) * W;
  const int halves = ev_parts ? host_dpt_parts(B) : 1;
  for (int v = 0; v < 2; ++v) {
    for (int hf = 0; hf < halves; ++hf) {
      const int i0 = hf * (B / halves), nb = (hf == halves - 1) ? B - i0 : B / halves;
      const long long o = static_cast<long long>(v) * B_total + i0;
      RUN(run_dpt(c, dpt, h, w, d.hook, v * B + i0, nb, pts3d + o * px * 3, conf + o * px));
      if (ev_parts) STA_CHECK_CUDA(cudaEventRecord(ev_parts[v * halves + hf], c.st));
    }
  }
  return 0;
}

}  // namespace

// ===========================================================================
// C ABI
// ===========================================================================
extern "C" {

const char* sta_last_error(void) { return get_last_error(); }
int sta_version(void) { return 2; }

int sta_device_synchronize(void) {
  STA_CHECK_CUDA(cudaDeviceSynchronize());
  return 0;
}

int sta_create(StaModel** out) { return sta_create_ex(out, STA_PRECISION_BF16); }

int sta_create_ex(StaModel** out, int precision) {
  if (precision != STA_PRECISION_BF16 && precision != STA_PRECISION_X3 && precision != STA_PRECISION_FP8) {
    set_last_error("sta_create_ex: unknown precision (0 = bf16, 1 = split-precision x3 parity mode, 2 = fp8)");
    return 2;
  }
  if (!out) {
    set_last_error("sta_create: null output pointer");
    return 2;
  }
  *out = nullptr;
  int dev = 0;
  STA_CHECK_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  STA_CHECK_CUDA(cudaGetDeviceProperties(&prop, dev));
  if (prop.major != 9 || prop.minor != 0) {
    char buf[160];
    snprintf(buf, sizeof(buf), "sta_b200 needs a Hopper sm_90 GPU (found %s, sm_%d%d); there is no fallback path",
             prop.name, prop.major, prop.minor);
    set_last_error(buf);
    return 3;
  }
  StaModel* m = new StaModel();
  m->split = (precision == STA_PRECISION_X3) ? 1 : 0;
  m->fp8 = (precision == STA_PRECISION_FP8) ? 1 : 0;
  // 438.5 M params: ~877 MB bf16 + fp32 vectors + padding (3x the bf16 part in split-precision mode)
  m->arena_bytes = static_cast<size_t>(m->split ? 2800 : 960) << 20;
  if (m->fp8) {  // 415 M trunk weights at one byte: the exact size, from a dry run of the registry (no arena yet)
    build_registry(m);
    m->arena_bytes = (m->arena_off + 255) & ~static_cast<size_t>(255);
    m->slots.clear();
    m->missing = 0;
    m->arena_off = 0;
  }
  cudaError_t e = cudaMalloc(&m->arena, m->arena_bytes);
  if (e != cudaSuccess) {
    set_last_error(std::string("cudaMalloc(weight arena) failed: ") + cudaGetErrorString(e));
    delete m;
    return 1;
  }
  cudaMemset(m->arena, 0, m->arena_bytes);
  if (cudaMalloc(&m->splitk_ws, StaModel::kSplitKBytes) != cudaSuccess) {
    cudaGetLastError();
    m->splitk_ws = nullptr;  // the split-K route is simply not taken
  }
  build_registry(m);
  if (m->arena_off > m->arena_bytes) {
    set_last_error("internal: weight arena too small");
    cudaFree(m->arena);
    delete m;
    return 1;
  }
  *out = m;
  return 0;
}

void sta_destroy(StaModel* m) {
  if (!m) return;
  cudaDeviceSynchronize();
  if (m->arena) cudaFree(m->arena);
  if (m->ws.base) cudaFree(m->ws.base);
  if (m->stage) cudaFree(m->stage);
  if (m->io) cudaFree(m->io);
  if (m->splitk_ws) cudaFree(m->splitk_ws);
  drop_graphs(m);
  if (m->s_cap) cudaStreamDestroy(m->s_cap);
  if (m->ev_switch) cudaEventDestroy(m->ev_switch);
  if (m->s_in) {
    cudaStreamDestroy(m->s_in);
    cudaStreamDestroy(m->s_out);
    for (int i = 0; i < StaModel::kMaxHostChunks; ++i) {
      cudaEventDestroy(m->ev_in[i]);
      cudaEventDestroy(m->ev_done[i]);
      for (int k = 0; k < 2 * StaModel::kMaxParts; ++k) cudaEventDestroy(m->ev_part[i][k]);
    }
    cudaEventDestroy(m->ev_start);
  }
  for (auto& r : m->prof_recs) {
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  for (auto e : m->prof_pool) cudaEventDestroy(e);
  delete m;
}

int sta_missing_tensors(StaModel* m) { return m ? m->missing : -1; }
int64_t sta_launch_count(StaModel* m) { return m ? m->launches : 0; }
int64_t sta_device_bytes(StaModel* m) {
  return m ? static_cast<int64_t>(m->arena_bytes + m->ws.bytes + m->stage_bytes + m->io_bytes) : 0;
}
int sta_profile(StaModel* m, int enable) {
  if (!m) return 2;
  m->prof_on = enable != 0;
  return 0;
}
int sta_profile_read(StaModel* m, double* ms4, int64_t* counts4, double* flops4) {
  if (!m || !ms4 || !counts4 || !flops4) {
    set_last_error("sta_profile_read: null argument");
    return 2;
  }
  STA_CHECK_CUDA(cudaDeviceSynchronize());
  for (auto& r : m->prof_recs) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, r.e0, r.e1) == cudaSuccess) {
      m->prof_ms[r.cat] += ms;
      m->prof_cnt[r.cat]++;
    }
    m->prof_pool.push_back(r.e0);
    m->prof_pool.push_back(r.e1);
  }
  m->prof_recs.clear();
  for (int i = 0; i < 4; ++i) {
    ms4[i] = m->prof_ms[i];
    counts4[i] = m->prof_cnt[i];
    flops4[i] = m->prof_flops[i];
    m->prof_ms[i] = 0;
    m->prof_cnt[i] = 0;
    m->prof_flops[i] = 0;
  }
  return 0;
}
int sta_set_taps(StaModel* m, StaTap* taps, int n) {
  if (!m || n < 0 || (n > 0 && !taps)) {
    set_last_error("sta_set_taps: null model, or n > 0 taps at a null array");
    return 2;
  }
  m->taps.clear();
  for (int i = 0; i < n; ++i) {
    if (!taps[i].name || m->taps.count(taps[i].name)) {
      set_last_error("sta_set_taps: a tap without a name, or two taps with one name");
      m->taps.clear();
      return 2;
    }
    m->taps[taps[i].name] = &taps[i];
  }
  return 0;
}
int sta_weight_arena(StaModel* m, void** ptr, int64_t* bytes) {
  if (!m || !ptr || !bytes) {
    set_last_error("sta_weight_arena: null argument");
    return 2;
  }
  *ptr = m->arena;
  *bytes = static_cast<int64_t>((m->arena_off + 255) & ~static_cast<size_t>(255));
  return 0;
}
int sta_weight_slot(StaModel* m, const char* name, void** data_out, int64_t* ld_out, float** scales_out) {
  if (!m || !name || !data_out || !ld_out || !scales_out) {
    set_last_error("sta_weight_slot: null argument");
    return 2;
  }
  const auto it = m->slots.find(name);
  if (it == m->slots.end()) {
    set_last_error(std::string("sta_weight_slot: no slot named ") + name);
    return 4;
  }
  const Slot& s = it->second;
  *data_out = s.dst;
  *ld_out = static_cast<int64_t>(s.ldd);
  *scales_out = s.kind == PK_LINEAR_FP8 ? s.sdst : nullptr;
  return 0;
}
int sta_mark_all_loaded(StaModel* m) {  // after the arena was filled by a broadcast from another rank
  if (!m) return 2;
  for (auto& kv : m->slots) kv.second.loaded = true;
  m->missing = 0;
  return 0;
}

int sta_load_tensor(StaModel* m, const char* name, const float* data, const int64_t* shape, int ndim,
                    int data_on_device) {
  if (!m || !name || !data) {
    set_last_error("sta_load_tensor: null argument");
    return 2;
  }
  auto it = m->slots.find(name);
  if (it == m->slots.end()) {
    set_last_error(std::string("unexpected key in state_dict: ") + name);
    return 4;
  }
  Slot& s = it->second;
  bool ok = static_cast<int>(s.shape.size()) == ndim;
  size_t numel = 1;
  for (int i = 0; ok && i < ndim; ++i) {
    ok = (shape[i] == s.shape[i]);
    numel *= static_cast<size_t>(shape[i]);
  }
  if (!ok) {
    set_last_error(std::string("size mismatch for ") + name);
    return 5;
  }
  if (s.kind == PK_IGNORE) return 0;
  const float* src = data;
  if (!data_on_device) {
    if (m->stage_bytes < numel * sizeof(float)) {
      STA_CHECK_CUDA(cudaDeviceSynchronize());
      if (m->stage) STA_CHECK_CUDA(cudaFree(m->stage));
      m->stage = nullptr;
      m->stage_bytes = 0;
      size_t want = numel * sizeof(float);
      if (want < (static_cast<size_t>(32) << 20)) want = static_cast<size_t>(32) << 20;
      STA_CHECK_CUDA(cudaMalloc(&m->stage, want));
      m->stage_bytes = want;
    }
    STA_CHECK_CUDA(cudaMemcpy(m->stage, data, numel * sizeof(float), cudaMemcpyHostToDevice));
    src = m->stage;
  }
  const int threads = 256;
  const int blocks = static_cast<int>((numel + threads - 1) / threads);
  switch (s.kind) {
    case PK_F32:
      STA_CHECK_CUDA(cudaMemcpy(s.dst, src, numel * sizeof(float), cudaMemcpyDeviceToDevice));
      break;
    case PK_LINEAR: {
      const int rows = static_cast<int>(s.shape[0]);
      const int cols = static_cast<int>(numel / rows);
      pack_linear_kernel<<<blocks, threads>>>(src, static_cast<bf16*>(s.dst), rows, cols, s.ldd, m->split);
      break;
    }
    case PK_LINEAR_FP8: {
      const int rows = static_cast<int>(s.shape[0]), cols = static_cast<int>(s.shape[1]);
      STA_REQUIRE(rows % 128 == 0 && cols % 128 == 0, "fp8 weights come in 128 x 128 blocks");
      pack_linear_fp8_kernel<<<dim3(cols / 128, rows / 128), 256>>>(src, cols, static_cast<uint8_t*>(s.dst), s.ldd, s.sdst,
                                                                    static_cast<int>(s.ldd / 128));
      break;
    }
    case PK_CONV3:
      pack_conv3_kernel<<<blocks, threads>>>(src, static_cast<bf16*>(s.dst), static_cast<int>(s.shape[0]),
                                             static_cast<int>(s.shape[1]), s.cin_pad, m->split);
      break;
    case PK_CONVT:
      pack_convT_kernel<<<blocks, threads>>>(src, static_cast<bf16*>(s.dst), static_cast<int>(s.shape[0]),
                                             static_cast<int>(s.shape[1]), s.k, s.cin_pad, s.cout_pad, m->split);
      break;
    case PK_TRANSPOSE_F32:
      transpose_f32_kernel<<<blocks, threads>>>(src, static_cast<float*>(s.dst), static_cast<int>(s.shape[0]),
                                                static_cast<int>(numel / s.shape[0]));
      break;
    default:
      break;
  }
  STA_CHECK_CUDA(cudaGetLastError());
  STA_CHECK_CUDA(cudaDeviceSynchronize());  // the staging buffer is reused by the next call
  if (!s.loaded) {
    s.loaded = true;
    m->missing--;
  }
  return 0;
}

int sta_encode(StaModel* m, const void* img_dev, int img_is_bf16, int B, int H, int W, float* feat_out_dev,
               int64_t* pos_out_dev, void* stream) {
  RUN(check_ready(m));
  RUN(check_grid(B, H, W));
  STA_REQUIRE(feat_out_dev != nullptr, "null pointer");
  Ctx c{m, static_cast<cudaStream_t>(stream)};
  RUN(enter_stream(m, c.st));
  const int h = H / 16, w = W / 16, N = h * w;
  RUN(ensure_ws(m, B, h, w));
  EncBufs e = take_enc(m->ws, B, N);
  // launch-bound sizes: the encoder proper is replayed as a CUDA graph (staged features; the caller's tensor is
  // long-lived: slam.py:145 keeps it for the whole run)
  const bool graphed = static_cast<long long>(B) * N <= kGraphMaxTokens;
  Staging staged{m->ws, graphed};
  float* x = staged.out(feat_out_dev, static_cast<size_t>(B) * N * kEncDim);
  RUN(check_ws(m->ws));
  m->launches += 1;
  RUN(launch_patch_im2col(img_dev, img_is_bf16, B, H, W, e.patches, c.st, m->split));
  RUN(tap(c, e.patches, bf_bytes(c, static_cast<size_t>(B) * N * 768), "patches"));
  auto body = [&](const Ctx& cc) -> int {
    m->launches += 1;
    RUN(launch_make_positions(e.pos, B, h, w, 0, cc.st));
    RUN(tap(cc, e.pos, static_cast<size_t>(B) * N * 2 * sizeof(int), "pos.enc"));
    return run_encoder(cc, B, N, x, e);
  };
  RUN(run_graphed(m, c.st, graphed, {1, B, H, W}, body));
  RUN(staged.flush(c.st));
  if (pos_out_dev) {
    const long long n = 2LL * B * N;
    m->launches++;
    pos_to_int64_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, c.st>>>(
        e.pos, n, reinterpret_cast<long long*>(pos_out_dev));
    STA_CHECK_CUDA(cudaGetLastError());
  }
  return 0;
}

int sta_decode(StaModel* m, const float* feat1_dev, const float* feat2_dev, const int64_t* pos1_dev,
               const int64_t* pos2_dev, int B, int N, float* const* out1_dev, float* const* out2_dev, void* stream) {
  RUN(check_ready(m));
  STA_REQUIRE(B > 0 && N > 0, "empty batch");
  Ctx c{m, static_cast<cudaStream_t>(stream)};
  RUN(enter_stream(m, c.st));
  // workspace sized as an (N x 1) token grid: only token counts matter for the decoder buffers
  RUN(ensure_ws(m, 2 * B, N, 1));
  DecBufs d = take_dec(m->ws, 2 * B, N);
  RUN(check_ws(m->ws));
  RUN(cast_features(c, feat1_dev, feat2_dev, B, N, d));
  m->launches++;
  {
    const long long total = 2LL * B * (N + 1);
    build_dec_pos_kernel<<<static_cast<int>((total + 255) / 256), 256, 0, c.st>>>(
        reinterpret_cast<const long long*>(pos1_dev), reinterpret_cast<const long long*>(pos2_dev), B, N, d.pos);
    STA_CHECK_CUDA(cudaGetLastError());
  }
  return run_decoder(c, B, N, d, out1_dev, out2_dev);
}

int sta_head_pose(StaModel* m, const float* tok_dev, int B, float* pose_out_dev, float* conf_out_dev, void* stream) {
  RUN(check_ready(m));
  m->launches++;
  return launch_pose_head(tok_dev, kDecDim, B, 0, kLnEps, m->pose, pose_out_dev, conf_out_dev,
                          static_cast<cudaStream_t>(stream));
}

int sta_head_pts(StaModel* m, const float* enc_feat_dev, const float* dec6_dev, const float* dec9_dev,
                 const float* dec12_dev, int B, int H, int W, float* pts3d_out_dev, float* conf_out_dev,
                 void* stream) {
  RUN(check_ready(m));
  STA_REQUIRE(B > 0 && H % 16 == 0 && W % 16 == 0, "image size must be a multiple of 16");
  Ctx c{m, static_cast<cudaStream_t>(stream)};
  RUN(enter_stream(m, c.st));
  const int h = H / 16, w = W / 16, N = h * w;
  RUN(ensure_ws(m, B, h, w));
  Workspace& ws = m->ws;
  bf16* hook[4];
  take_hooks(ws, B, N, hook);
  const DptBufs dpt = take_dpt(ws, B, h, w);
  RUN(check_ws(ws));
  const float* src[4] = {enc_feat_dev, dec6_dev, dec9_dev, dec12_dev};
  m->launches += 4;
  for (int q = 0; q < 4; ++q)
    RUN(launch_cast_f32_bf16(src[q], hook[q], static_cast<long long>(B) * N, q ? 768 : 1024, 0, c.st, m->split));
  return run_dpt(c, dpt, h, w, hook, 0, B, pts3d_out_dev, conf_out_dev);
}

int64_t sta_graph_replays(StaModel* m) { return m ? m->graph_replays : 0; }

int sta_regress_pairs(StaModel* m, const float* feat_i_dev, const float* feat_j_dev, int K, int H, int W,
                      float* pose_out_dev, float* pose_conf_out_dev, float* pts3d_out_dev, float* conf_out_dev,
                      float* intri_out_dev, float* depth_out_dev, float* conf_mean_out_dev, void* scratch, void* stream) {
  RUN(check_ready(m));
  RUN(check_edges(m, K));
  RUN(check_grid(K, H, W));
  STA_REQUIRE(feat_i_dev && feat_j_dev && pose_out_dev && pose_conf_out_dev && pts3d_out_dev && conf_out_dev,
              "null pointer");
  RUN(check_consumers(scratch, intri_out_dev, depth_out_dev, conf_mean_out_dev));
  Ctx c{m, static_cast<cudaStream_t>(stream)};
  RUN(enter_stream(m, c.st));
  const int h = H / 16, w = W / 16, N = h * w, S = 2 * K;
  const long long px = static_cast<long long>(H) * W;
  RUN(ensure_ws(m, S, h, w));
  Workspace& ws = m->ws;
  DecBufs d = take_dec(ws, S, N);
  // Launch-bound sizes: decoder, pose heads, DPT heads and consumers are replayed as one CUDA graph (staged outputs).
  const bool graphed = static_cast<long long>(S) * (N + 1) <= kGraphMaxTokens;
  Staging staged{ws, graphed};
  float* o_pose = staged.out(pose_out_dev, static_cast<size_t>(S) * 16);
  float* o_pconf = staged.out(pose_conf_out_dev, S);
  const PairOuts o =
      stage_pair_outs(staged, {pts3d_out_dev, conf_out_dev, intri_out_dev, depth_out_dev, conf_mean_out_dev, scratch}, K, px);
  const DptBufs dpt = take_dpt(ws, K, h, w);
  RUN(check_ws(ws));
  RUN(cast_features(c, feat_i_dev, feat_j_dev, K, N, d));
  auto body = [&](const Ctx& cc) -> int {
    RUN(decode_with_poses(cc, K, h, w, d, o_pose, o_pconf, K));
    return pair_heads(cc, dpt, d.hook, K, H, W, o);
  };
  RUN(run_graphed(m, c.st, graphed, {2, K, H, W, intri_out_dev ? 1 : 0, depth_out_dev ? 1 : 0, conf_mean_out_dev ? 1 : 0},
                  body));
  return staged.flush(c.st);
}

// ---------------------------------------------------------------------------
// Gated keyframe step (SURVEY.md 8(f) rank 1 with the early-out of slam.py:169-170): phase 1 runs the decoder and the
// pose heads for all K candidate edges and leaves the decoder hooks in the workspace; the caller reads the K pose
// confidences ONCE, decides which edges survive (`conf >= thres or i - j == 1`) and phase 2 runs the DPT heads and the
// pointmap consumers for the survivors only.  Any other model call on this handle in between ends the pair (check_ready).
// ---------------------------------------------------------------------------
int sta_regress_pairs_begin(StaModel* m, const float* feat_i_dev, const float* feat_j_dev, int K, int H, int W,
                            float* pose_out_dev, float* pose_conf_out_dev, void* stream) {
  RUN(check_ready(m));
  RUN(check_edges(m, K));
  RUN(check_grid(K, H, W));
  STA_REQUIRE(feat_i_dev && feat_j_dev && pose_out_dev && pose_conf_out_dev, "null pointer");
  Ctx c{m, static_cast<cudaStream_t>(stream)};
  RUN(enter_stream(m, c.st));
  const int h = H / 16, w = W / 16, N = h * w, S = 2 * K;
  RUN(ensure_ws(m, S, h, w));
  Workspace& ws = m->ws;
  DecBufs d = take_dec(ws, S, N);
  const bool graphed = static_cast<long long>(S) * (N + 1) <= kGraphMaxTokens;
  Staging staged{ws, graphed};
  float* o_pose = staged.out(pose_out_dev, static_cast<size_t>(S) * 16);
  float* o_pconf = staged.out(pose_conf_out_dev, S);
  RUN(check_ws(ws));
  RUN(cast_features(c, feat_i_dev, feat_j_dev, K, N, d));
  auto body = [&](const Ctx& cc) -> int { return decode_with_poses(cc, K, h, w, d, o_pose, o_pconf, K); };
  RUN(run_graphed(m, c.st, graphed, {3, K, H, W}, body));
  RUN(staged.flush(c.st));
  m->rp = {K, H, W, d, ws.off};
  return 0;
}

int sta_regress_pairs_finish(StaModel* m, const int* edge_idx_host, int n_sel, float* pts3d_out_dev, float* conf_out_dev,
                             float* intri_out_dev, float* depth_out_dev, float* conf_mean_out_dev, void* scratch,
                             void* stream) {
  RUN(check_ready(m, /*finishing_pairs=*/true));
  STA_REQUIRE(m->rp.K > 0, "sta_regress_pairs_finish without a preceding sta_regress_pairs_begin on this handle, or "
                           "another call on the handle came between them");
  const int K = m->rp.K, H = m->rp.H, W = m->rp.W;
  STA_REQUIRE(n_sel >= 0 && n_sel <= K, "more selected edges than candidates");
  if (n_sel == 0) return 0;
  STA_REQUIRE(edge_idx_host && pts3d_out_dev && conf_out_dev, "null pointer");
  for (int k = 0; k < n_sel; ++k) STA_REQUIRE(edge_idx_host[k] >= 0 && edge_idx_host[k] < K, "edge index out of range");
  RUN(check_consumers(scratch, intri_out_dev, depth_out_dev, conf_mean_out_dev));
  Ctx c{m, static_cast<cudaStream_t>(stream)};
  RUN(enter_stream(m, c.st));
  const int h = H / 16, w = W / 16, N = h * w, S2 = 2 * n_sel;
  const long long px = static_cast<long long>(H) * W;
  const DecBufs& d = m->rp.d;
  Workspace& ws = m->ws;
  ws.off = m->rp.ws_off;  // _begin's buffers stay untouched
  const bool graphed = 2LL * K * (N + 1) <= kGraphMaxTokens;
  // compact copies of the survivors' hooks: [view][edge] order, view 0 = the (i -> j) direction
  bf16* sel[4];
  take_hooks(ws, S2, N, sel);
  Staging staged{ws, graphed};
  const PairOuts o = stage_pair_outs(
      staged, {pts3d_out_dev, conf_out_dev, intri_out_dev, depth_out_dev, conf_mean_out_dev, scratch}, n_sel, px);
  const DptBufs dpt = take_dpt(ws, n_sel, h, w);
  RUN(check_ws(ws));
  const size_t bm = m->bmul();
  const size_t width[4] = {1024 * bm, 768 * bm, 768 * bm, 768 * bm};
  for (int v = 0; v < 2; ++v)
    for (int k = 0; k < n_sel; ++k)
      for (int q = 0; q < 4; ++q) {
        const size_t rows = static_cast<size_t>(N) * width[q];
        STA_CHECK_CUDA(cudaMemcpyAsync(sel[q] + (static_cast<size_t>(v) * n_sel + k) * rows,
                                       d.hook[q] + (static_cast<size_t>(v) * K + edge_idx_host[k]) * rows, rows * sizeof(bf16),
                                       cudaMemcpyDeviceToDevice, c.st));
      }
  auto body = [&](const Ctx& cc) -> int { return pair_heads(cc, dpt, sel, n_sel, H, W, o); };
  RUN(run_graphed(m, c.st, graphed,
                  {4, K, n_sel, H, W, intri_out_dev ? 1 : 0, depth_out_dev ? 1 : 0, conf_mean_out_dev ? 1 : 0}, body));
  return staged.flush(c.st);
}

int sta_forward_pairs(StaModel* m, const void* img1_dev, const void* img2_dev, int img_is_bf16, int B, int H, int W,
                      float* pts3d_out_dev, float* conf_out_dev, float* pose_out_dev, float* pose_conf_out_dev,
                      void* stream) {
  RUN(check_ready(m));
  RUN(check_grid(B, H, W));
  Ctx c{m, static_cast<cudaStream_t>(stream)};
  RUN(enter_stream(m, c.st));
  const size_t esz = img_is_bf16 ? 2 : 4;
  const long long px = static_cast<long long>(H) * W;
  for (int b0 = 0; b0 < B; b0 += m->max_pairs_per_chunk) {
    const int nb = (B - b0 < m->max_pairs_per_chunk) ? (B - b0) : m->max_pairs_per_chunk;
    const char* i1 = static_cast<const char*>(img1_dev) + static_cast<size_t>(b0) * 3 * px * esz;
    const char* i2 = static_cast<const char*>(img2_dev) + static_cast<size_t>(b0) * 3 * px * esz;
    RUN(forward_chunk(c, i1, i2, img_is_bf16, nb, H, W, pts3d_out_dev + static_cast<long long>(b0) * px * 3,
                      conf_out_dev + static_cast<long long>(b0) * px, pose_out_dev + static_cast<long long>(b0) * 16,
                      pose_conf_out_dev + b0, B));
  }
  return 0;
}

int sta_forward_pairs_host(StaModel* m, const void* img1_host, const void* img2_host, int img_is_bf16, int B, int H,
                           int W, float* pts3d_out_host, float* conf_out_host, float* pose_out_host,
                           float* pose_conf_out_host, void* stream) {
  RUN(check_ready(m));
  RUN(check_grid(B, H, W));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RUN(enter_stream(m, st));
  const size_t esz = img_is_bf16 ? 2 : 4;
  const size_t px = static_cast<size_t>(H) * W;
  const size_t img_bytes = static_cast<size_t>(B) * 3 * px * esz;
  const size_t pts_bytes = 2 * static_cast<size_t>(B) * px * 3 * sizeof(float);
  const size_t conf_bytes = 2 * static_cast<size_t>(B) * px * sizeof(float);
  const size_t pose_bytes = 2 * static_cast<size_t>(B) * 16 * sizeof(float);
  const size_t pconf_bytes = 2 * static_cast<size_t>(B) * sizeof(float);
  auto up = [](size_t v) { return (v + 255) & ~static_cast<size_t>(255); };
  const size_t need = 2 * up(img_bytes) + up(pts_bytes) + up(conf_bytes) + up(pose_bytes) + up(pconf_bytes);
  if (m->io_bytes < need) {
    STA_CHECK_CUDA(cudaDeviceSynchronize());
    if (m->io) STA_CHECK_CUDA(cudaFree(m->io));
    m->io = nullptr;
    m->io_bytes = 0;
    STA_CHECK_CUDA(cudaMalloc(&m->io, need));
    m->io_bytes = need;
  }
  if (!m->s_in) {
    STA_CHECK_CUDA(cudaStreamCreateWithFlags(&m->s_in, cudaStreamNonBlocking));
    STA_CHECK_CUDA(cudaStreamCreateWithFlags(&m->s_out, cudaStreamNonBlocking));
    for (int i = 0; i < StaModel::kMaxHostChunks; ++i) {
      STA_CHECK_CUDA(cudaEventCreateWithFlags(&m->ev_in[i], cudaEventDisableTiming));
      STA_CHECK_CUDA(cudaEventCreateWithFlags(&m->ev_done[i], cudaEventDisableTiming));
      for (int k = 0; k < 2 * StaModel::kMaxParts; ++k)
        STA_CHECK_CUDA(cudaEventCreateWithFlags(&m->ev_part[i][k], cudaEventDisableTiming));
    }
    STA_CHECK_CUDA(cudaEventCreateWithFlags(&m->ev_start, cudaEventDisableTiming));
  }
  char* p = m->io;
  char* d_img1 = p; p += up(img_bytes);
  char* d_img2 = p; p += up(img_bytes);
  float* d_pts = reinterpret_cast<float*>(p); p += up(pts_bytes);
  float* d_conf = reinterpret_cast<float*>(p); p += up(conf_bytes);
  float* d_pose = reinterpret_cast<float*>(p); p += up(pose_bytes);
  float* d_pconf = reinterpret_cast<float*>(p);

  // Pipeline over chunks of pairs: the H2D copy of chunk c+1 and the D2H copy of chunk c-1 overlap the compute
  // of chunk c (separate copy streams, pinned host memory makes them truly asynchronous).
  // one chunk of up to 16 pairs (the exposed H2D of a 16-pair chunk is meant to cost less than running the GEMMs at half
  // the tile count); larger batches pipeline chunks
  int cp = B;
  if (cp > m->max_pairs_per_chunk) cp = m->max_pairs_per_chunk;
  int nchunks = (B + cp - 1) / cp;
  if (nchunks > StaModel::kMaxHostChunks) {
    nchunks = StaModel::kMaxHostChunks;
    cp = (B + nchunks - 1) / nchunks;
    STA_REQUIRE(cp <= m->max_pairs_per_chunk, "batch too large for the host entry point; split it");
    nchunks = (B + cp - 1) / cp;
  }
  // the copy streams must not start before previously enqueued work on `st` that may still use the io buffers
  STA_CHECK_CUDA(cudaEventRecord(m->ev_start, st));
  STA_CHECK_CUDA(cudaStreamWaitEvent(m->s_in, m->ev_start, 0));
  STA_CHECK_CUDA(cudaStreamWaitEvent(m->s_out, m->ev_start, 0));
  const size_t img_pair = 3 * px * esz;
  for (int c = 0; c < nchunks; ++c) {
    const int b0 = c * cp, nb = (B - b0 < cp) ? (B - b0) : cp;
    STA_CHECK_CUDA(cudaMemcpyAsync(d_img1 + b0 * img_pair, static_cast<const char*>(img1_host) + b0 * img_pair,
                                   nb * img_pair, cudaMemcpyHostToDevice, m->s_in));
    STA_CHECK_CUDA(cudaMemcpyAsync(d_img2 + b0 * img_pair, static_cast<const char*>(img2_host) + b0 * img_pair,
                                   nb * img_pair, cudaMemcpyHostToDevice, m->s_in));
    STA_CHECK_CUDA(cudaEventRecord(m->ev_in[c], m->s_in));
  }
  Ctx cx{m, st};
  for (int c = 0; c < nchunks; ++c) {
    const int b0 = c * cp, nb = (B - b0 < cp) ? (B - b0) : cp;
    STA_CHECK_CUDA(cudaStreamWaitEvent(st, m->ev_in[c], 0));
    RUN(forward_chunk(cx, d_img1 + b0 * img_pair, d_img2 + b0 * img_pair, img_is_bf16, nb, H, W,
                      d_pts + static_cast<size_t>(b0) * px * 3, d_conf + static_cast<size_t>(b0) * px,
                      d_pose + static_cast<size_t>(b0) * 16, d_pconf + b0, B, m->ev_part[c]));
    STA_CHECK_CUDA(cudaEventRecord(m->ev_done[c], st));
    const int halves = host_dpt_parts(nb);  // mirrors forward_chunk
    for (int v = 0; v < 2; ++v) {
      for (int hf = 0; hf < halves; ++hf) {
        const int i0 = hf * (nb / halves), ni = (hf == halves - 1) ? nb - i0 : nb / halves;
        STA_CHECK_CUDA(cudaStreamWaitEvent(m->s_out, m->ev_part[c][v * halves + hf], 0));
        const size_t o = static_cast<size_t>(v) * B + b0 + i0;
        STA_CHECK_CUDA(cudaMemcpyAsync(pts3d_out_host + o * px * 3, d_pts + o * px * 3, ni * px * 3 * sizeof(float),
                                       cudaMemcpyDeviceToHost, m->s_out));
        STA_CHECK_CUDA(cudaMemcpyAsync(conf_out_host + o * px, d_conf + o * px, ni * px * sizeof(float),
                                       cudaMemcpyDeviceToHost, m->s_out));
      }
    }
    STA_CHECK_CUDA(cudaStreamWaitEvent(m->s_out, m->ev_done[c], 0));
    for (int v = 0; v < 2; ++v) {
      const size_t o = static_cast<size_t>(v) * B + b0;
      STA_CHECK_CUDA(cudaMemcpyAsync(pose_out_host + o * 16, d_pose + o * 16, nb * 16 * sizeof(float),
                                     cudaMemcpyDeviceToHost, m->s_out));
      STA_CHECK_CUDA(cudaMemcpyAsync(pose_conf_out_host + o, d_pconf + o, nb * sizeof(float), cudaMemcpyDeviceToHost,
                                     m->s_out));
    }
  }
  STA_CHECK_CUDA(cudaStreamSynchronize(m->s_out));
  STA_CHECK_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// ---------------------------------------------------------------------------
// op-level entry points (parity tests drive the same kernels the model uses)
// ---------------------------------------------------------------------------
int sta_op_gemm(const StaGemmDesc* d, void* stream) {
  if (!d) {
    set_last_error("sta_op_gemm: null descriptor");
    return 2;
  }
  GemmLaunch g;
  g.amode = d->conv3x3 ? A_CONV3 : A_LINEAR;
  g.epi = d->epi;
  g.A = static_cast<const bf16*>(d->A);
  g.lda = d->lda;
  g.Wt = static_cast<const bf16*>(d->W);
  g.ldw = d->ldw;
  g.splitk_ws = d->splitk_ws;
  g.splitk_ws_bytes = d->splitk_ws ? static_cast<size_t>(d->splitk_ws_bytes) : 0;
  GemmParams p = {};
  p.M = d->M; p.N = d->N; p.K = d->K;
  p.nimg = d->nimg; p.H = d->H; p.W = d->Wd; p.Cin = d->Cin;
  p.bias = d->bias;
  p.out = d->out; p.ldo = d->ldo; p.out2 = d->out2;
  p.resid = d->resid; p.resid2 = d->resid2;
  p.relu_main = d->relu_main;
  p.rowmap_n = d->rowmap_n;
  p.pos = d->pos; p.rope_cols = d->rope_cols;
  if (d->epi == EPI_ROPE) {
    p.rope_tab = rope_table(&p.rope_max_pos);
    if (!p.rope_tab) {
      set_last_error("failed to build the RoPE table");
      return 1;
    }
    p.rope_smem_rows = 64;
  }
  p.ps_k = d->ps_k; p.ps_cout = d->ps_cout; p.ps_h = d->ps_h; p.ps_w = d->ps_w;
  p.head_w = d->head_w; p.head_b = d->head_b; p.pts3d = d->pts3d; p.conf = d->conf;
  p.split = d->split_precision;
  g.p = p;
  g.tile_n = d->tile_n;
  return launch_gemm(g, static_cast<cudaStream_t>(stream));
}

int sta_gemm_auto_tile_n(int M, int N, int K, int epi, int num_sms) { return gemm_auto_tile_n(M, N, K, epi, num_sms); }

int sta_op_gemm_fp8(const StaGemmFp8Desc* d, void* stream) {
  if (!d) {
    set_last_error("sta_op_gemm_fp8: null descriptor");
    return 2;
  }
  STA_REQUIRE(d->epi == STA_EPI_F32 || d->epi == STA_EPI_ROPE || d->epi == STA_EPI_GELU_FP8,
              "sta_op_gemm_fp8: epi must be STA_EPI_F32, STA_EPI_ROPE or STA_EPI_GELU_FP8");
  GemmLaunch g;
  g.amode = A_FP8;
  g.epi = d->epi;
  g.A = d->A;
  g.lda = d->lda;
  g.Wt = d->W;
  g.ldw = d->ldw;
  g.splitk_ws = d->splitk_ws;
  g.splitk_ws_bytes = d->splitk_ws ? static_cast<size_t>(d->splitk_ws_bytes) : 0;
  GemmParams p = {};
  p.M = d->M; p.N = d->N; p.K = d->K;
  p.bias = d->bias;
  p.out = d->out; p.ldo = d->ldo;
  p.resid = d->resid;
  p.a_scale = d->a_scale; p.w_scale = d->w_scale; p.out_scale = d->out_scale;
  if (d->epi == STA_EPI_ROPE) RUN(set_rope(p, d->pos, d->rope_cols));
  g.p = p;
  return launch_gemm(g, static_cast<cudaStream_t>(stream));
}
int sta_op_layernorm_fp8(const float* x, int rows, int C, float eps, const float* g1, const float* b1, void* q1, float* s1,
                         const float* g2, const float* b2, void* q2, float* s2, void* stream) {
  return launch_layernorm_fp8(x, rows, C, eps, g1, b1, static_cast<uint8_t*>(q1), s1, g2, b2, static_cast<uint8_t*>(q2), s2,
                              static_cast<cudaStream_t>(stream));
}
int sta_op_quant_fp8(const void* in_bf16, int64_t rows, int C, void* q, float* s, void* stream) {
  return launch_quant_fp8(static_cast<const bf16*>(in_bf16), rows, C, static_cast<uint8_t*>(q), s,
                          static_cast<cudaStream_t>(stream));
}

static int op_attention(const void* q, int64_t ldq, int q_col0, const void* k, int64_t ldk, int k_col0, const void* v,
                        int64_t ldv, int v_col0, void* out, int64_t ldo, int batch, int heads, int nq, int nk,
                        int kv_batch_shift, float scale, int split, void* stream) {
  AttnLaunch a;
  a.q = static_cast<const bf16*>(q); a.ldq = ldq; a.q_col0 = q_col0;
  a.k = static_cast<const bf16*>(k); a.ldk = ldk; a.k_col0 = k_col0;
  a.v = static_cast<const bf16*>(v); a.ldv = ldv; a.v_col0 = v_col0;
  a.out = static_cast<bf16*>(out); a.ldo = ldo;
  a.batch = batch; a.heads = heads; a.nq = nq; a.nk = nk;
  a.kv_batch_shift = kv_batch_shift;
  a.scale = scale;
  a.split = split;
  return launch_attention(a, static_cast<cudaStream_t>(stream));
}
int sta_op_attention(const void* q, int64_t ldq, int q_col0, const void* k, int64_t ldk, int k_col0, const void* v,
                     int64_t ldv, int v_col0, void* out, int64_t ldo, int batch, int heads, int nq, int nk,
                     int kv_batch_shift, float scale, void* stream) {
  return op_attention(q, ldq, q_col0, k, ldk, k_col0, v, ldv, v_col0, out, ldo, batch, heads, nq, nk, kv_batch_shift,
                      scale, 0, stream);
}
int sta_op_attention_split(const void* q, int64_t ldq, int q_col0, const void* k, int64_t ldk, int k_col0,
                           const void* v, int64_t ldv, int v_col0, void* out, int64_t ldo, int batch, int heads, int nq,
                           int nk, int kv_batch_shift, float scale, void* stream) {
  return op_attention(q, ldq, q_col0, k, ldk, k_col0, v, ldv, v_col0, out, ldo, batch, heads, nq, nk, kv_batch_shift,
                      scale, 1, stream);
}

int sta_op_layernorm(const float* x, int rows, int C, float eps, const float* g1, const float* b1, void* out1_bf16,
                     const float* g2, const float* b2, void* out2_bf16, int drop_first_of, void* stream) {
  return launch_layernorm(x, rows, C, eps, g1, b1, static_cast<bf16*>(out1_bf16), g2, b2,
                          static_cast<bf16*>(out2_bf16), drop_first_of, static_cast<cudaStream_t>(stream));
}
int sta_op_patch_im2col(const void* img, int img_is_bf16, int B, int H, int W, void* out_bf16, void* stream) {
  return launch_patch_im2col(img, img_is_bf16, B, H, W, static_cast<bf16*>(out_bf16), static_cast<cudaStream_t>(stream));
}
int sta_op_upsample2x(const void* in_bf16, void* out_bf16, int nimg, int H, int W, int C, void* stream) {
  return launch_upsample2x(static_cast<const bf16*>(in_bf16), static_cast<bf16*>(out_bf16), nimg, H, W, C, 2 * H, 2 * W,
                           static_cast<cudaStream_t>(stream));
}
int sta_op_im2col_3x3_s2(const void* in_bf16, void* out_bf16, int nimg, int H, int W, int C, void* stream) {
  return launch_im2col_3x3_s2(static_cast<const bf16*>(in_bf16), static_cast<bf16*>(out_bf16), nimg, H, W, C,
                              static_cast<cudaStream_t>(stream));
}
int sta_op_cast_f32_bf16(const float* in, void* out_bf16, int64_t rows, int C, int drop_first_of, void* stream) {
  return launch_cast_f32_bf16(in, static_cast<bf16*>(out_bf16), rows, C, drop_first_of,
                              static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------
// pointmap consumers (pointmap.cu)
// ---------------------------------------------------------------------------
size_t sta_pointmap_scratch_bytes(int V) { return pointmap_scratch_bytes(V); }
int sta_pointmap_consumers(const float* pts3d, const float* conf, int V, int H, int W, int shared, float* K_out,
                           float* depth_out, float* conf_mean_out, void* scratch, void* stream) {
  return launch_pointmap_consumers(pts3d, conf, V, H, W, shared, K_out, depth_out, conf_mean_out, scratch,
                                   static_cast<cudaStream_t>(stream));
}
int sta_depth_scale(const float* Di, const float* Dj, const float* ci, const float* cj, int64_t n, float* out2,
                    void* scratch, void* stream) {
  return launch_depth_scale(Di, Dj, ci, cj, static_cast<long long>(n), out2, scratch, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------
// Sim(3) pose-graph LM step (pose_graph.cu)
// ---------------------------------------------------------------------------
size_t sta_pose_graph_scratch_bytes(int num_nodes, int num_edges, int num_opt) {
  return pose_graph_scratch_bytes(num_nodes, num_edges, num_opt);
}
int sta_pose_graph_lm_step(const float* nodes, int num_nodes, const int64_t* edges, const float* meas, const float* weights,
                           int num_edges, const int64_t* opt_idx, int num_opt, double damping, double dmin, double dmax,
                           float* nodes_out, double* info_out, void* scratch, void* stream) {
  return launch_pose_graph_lm_step(nodes, num_nodes, reinterpret_cast<const long long*>(edges), meas, weights, num_edges,
                                   reinterpret_cast<const long long*>(opt_idx), num_opt, damping, dmin, dmax, nodes_out,
                                   info_out, scratch, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------
// image preprocessing (preprocess.cu)
// ---------------------------------------------------------------------------
int sta_preprocess_shape(int H, int W, int res_w, int res_h, int w_edge, int h_edge, int* out_hw) {
  return launch_preprocess_rgb8(nullptr, 1, H, W, res_w, res_h, w_edge, h_edge, nullptr, nullptr, nullptr, out_hw, 1,
                                nullptr);
}
int sta_preprocess_geometry(int H, int W, int res_w, int res_h, int w_edge, int h_edge, int* out10) {
  if (!out10) {
    set_last_error("sta_preprocess_geometry: null output");
    return 2;
  }
  return preprocess_geometry(H, W, res_w, res_h, w_edge, h_edge, out10);
}
int sta_preprocess_coeffs(int in_size, int out_size, int* ksize, int* bounds, int* kk, int64_t kk_capacity) {
  return preprocess_coeffs(in_size, out_size, ksize, bounds, kk, static_cast<long long>(kk_capacity));
}
int sta_preprocess_rgb8(const uint8_t* rgb_dev, int H, int W, int res_w, int res_h, int w_edge, int h_edge,
                        float* rgb_out_dev, float* gray_out_dev, uint8_t* u8_out_dev, void* stream) {
  return sta_preprocess_rgb8_many(rgb_dev, 1, H, W, res_w, res_h, w_edge, h_edge, rgb_out_dev, gray_out_dev, u8_out_dev,
                                  stream);
}
int sta_preprocess_rgb8_many(const uint8_t* rgb_dev, int F, int H, int W, int res_w, int res_h, int w_edge, int h_edge,
                             float* rgb_out_dev, float* gray_out_dev, uint8_t* u8_out_dev, void* stream) {
  return launch_preprocess_rgb8(rgb_dev, F, H, W, res_w, res_h, w_edge, h_edge, rgb_out_dev, gray_out_dev, u8_out_dev,
                                nullptr, 0, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
