/*
 * sta_b200.h -- C ABI of libsta_b200.so, the H100 (sm_90a) implementation of the
 * ViSTA-SLAM "Symmetric Two-view Association" (STA) frontend forward pass.
 *
 * The library is the drop-in boundary underneath the reference's Python module
 * vista_slam/sta_model/sta_model.py::SymmetricTwoViewAssociation.  Every model-level
 * entry point below names the reference method it replaces (file:line in
 * zhangganlin/vista-slam).  Conventions:
 *   - plain C: pointers, sizes, opaque handle; no C++/torch types, no exceptions;
 *   - every function returns 0 on success, non-zero on failure; sta_last_error()
 *     then returns a thread-local human-readable message;
 *   - all "dev" pointers are CUDA device pointers on the current device, "host"
 *     pointers are host memory; `stream` is a cudaStream_t passed as void* (NULL =
 *     default stream); calls are asynchronous with respect to the host unless noted;
 *   - the caller owns all input/output buffers, the handle owns weights + workspace;
 *   - the CUDA kernels are the only implementation: there is no CPU fallback.
 */
#ifndef STA_B200_H_
#define STA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct StaModel StaModel; /* opaque */

/* ---- library ---- */
const char* sta_last_error(void);
int sta_version(void);                 /* ABI version, currently 2 */
int sta_device_synchronize(void);      /* cudaDeviceSynchronize + error check */

/* ---- model lifetime (replaces STA() + load_state_dict + .to(cuda), slam.py:95-106) ---- */
int sta_create(StaModel** out);
/* Same with an explicit operand precision.  STA_PRECISION_BF16 (what sta_create uses, and what every benchmark
 * number is measured with): bf16 tensor-core operands, fp32 accumulation.  STA_PRECISION_X3: split-precision PARITY
 * mode -- every bf16 activation is carried as (hi | lo | hi) and every bf16 weight as (hi | hi | lo), so the same
 * wgmma kernels compute a_hi w_hi + a_lo w_hi + a_hi w_lo over K' = 3K (about 17 significant operand bits),
 * and attention runs in fp32 on the CUDA cores.  It exists to check the kernels against the fp32 reference at
 * north_star's tolerance (pointmaps 1e-3, pose 1e-4); ~3x the weight memory, several times slower.
 * STA_PRECISION_FP8: an opt-in mode that changes the numerics -- the linear layers of the 24 encoder and 12 decoder
 * blocks (qkv, proj, fc1, fc2; qkv, proj, projq, projk|projv, cross proj, fc1, fc2) run on e4m3 operands with power-of-two
 * scales, one per row and 128 columns of the activations and one per 128 x 128 block of the weights, each 128-wide
 * k-block accumulated on its own and folded into fp32 with both scales.  Everything else (patch embedding,
 * decoder_embed, attention, the DPT head, the pose head) is as in bf16 mode.  The trunk weights take half the bytes.
 * With random-init weights its outputs move about 6-10x as far from fp32 as bf16's do; how that carries over to the
 * trained checkpoint or to SLAM accuracy is not measured, so check it on your own data. */
enum { STA_PRECISION_BF16 = 0, STA_PRECISION_X3 = 1, STA_PRECISION_FP8 = 2 };
int sta_create_ex(StaModel** out, int precision);
void sta_destroy(StaModel* m);

/* Upload one state-dict tensor (fp32, contiguous, host or device memory) under its
 * reference state_dict name (SURVEY.md App. C, e.g. "enc_blocks.0.attn.qkv.weight").
 * The library converts/packs it into its own bf16 / fp32 device layout.
 * Names the forward pass does not use (enc_norm.*, refinenet4.resConfUnit1.*, the
 * aliased scratch.layerN_rn.*) are accepted and ignored.  Returns non-zero for an
 * unknown name or a shape mismatch (strict=True semantics, sta_model.py:143). */
int sta_load_tensor(StaModel* m, const char* name, const float* data, const int64_t* shape, int ndim,
                    int data_on_device);
/* Number of tensors still missing before the model can run (0 = ready). */
int sta_missing_tensors(StaModel* m);
/* The packed weights live in ONE device arena.  For multi-GPU runs rank 0 loads the state dict,
 * every rank exposes its arena, the host broadcasts it (torch.distributed / ncclBroadcast over NVLink)
 * and the receiving ranks call sta_mark_all_loaded. */
int sta_weight_arena(StaModel* m, void** dev_ptr_out, int64_t* bytes_out);
int sta_mark_all_loaded(StaModel* m);
/* Read-only: where the state-dict tensor `name` lands in the arena.  data_out: its packed destination (device memory;
 * NULL for a name the forward pass ignores), ld_out: its row stride in elements for the linear packings (0 otherwise),
 * scales_out: for an FP8-mode trunk weight (e4m3 codes, row stride ld_out bytes) its 128 x 128 block scales, fp32
 * [rows / 128][ld_out / 128], else NULL.  Returns non-zero for an unknown name. */
int sta_weight_slot(StaModel* m, const char* name, void** data_out, int64_t* ld_out, float** scales_out);

/* ---- model-level forward entry points ---- */

/* _encode_image(image, true_shape, normalize=False), sta_model.py:163-174.
 * img_dev: [B,3,H,W] fp32 (img_is_bf16 = 0) or bf16 (1), values in [-1,1].
 * feat_out_dev: [B, (H/16)*(W/16), 1024] fp32.  pos_out_dev: [B, N, 2] int64 (y, x) or NULL. */
int sta_encode(StaModel* m, const void* img_dev, int img_is_bf16, int B, int H, int W, float* feat_out_dev,
               int64_t* pos_out_dev, void* stream);

/* _decode_stereo(feat1, feat2, pos1, pos2), sta_model.py:177-244.
 * feat*_dev: [B,N,1024] fp32; pos*_dev: [B,N,2] int64 (values in [-1,1023]).
 * out1_dev / out2_dev: arrays (host memory) of 13 device pointers, each [B,N+1,768] fp32 or NULL to
 * skip that layer's output; entry 12 is LayerNorm-ed (dec_norm), as in the reference. */
int sta_decode(StaModel* m, const float* feat1_dev, const float* feat2_dev, const int64_t* pos1_dev,
               const int64_t* pos2_dev, int B, int N, float* const* out1_dev, float* const* out2_dev, void* stream);

/* head_pose_s(tok), heads/pose_head.py:109-119.  tok_dev: [B,768] fp32 (already dec_norm-ed).
 * pose_out_dev: [B,4,4] fp32, conf_out_dev: [B] fp32. */
int sta_head_pose(StaModel* m, const float* tok_dev, int B, float* pose_out_dev, float* conf_out_dev, void* stream);

/* head_pts([enc_feat] + [dec_k[:,1:]]_k, true_shape), sta_model.py:135-137 + utils/misc.py:48-76 +
 * heads/dpt_head.py:34-66.  Only the four hooked layers are read:
 *   enc_feat_dev [B,N,1024], dec6_dev, dec9_dev, dec12_dev [B,N,768] fp32 (pose token already dropped).
 * pts3d_out_dev: [B,H,W,3] fp32, conf_out_dev: [B,H,W] fp32. */
int sta_head_pts(StaModel* m, const float* enc_feat_dev, const float* dec6_dev, const float* dec9_dev,
                 const float* dec12_dev, int B, int H, int W, float* pts3d_out_dev, float* conf_out_dev,
                 void* stream);

/* forward(views) for ONE support view over a batch of B pairs (sta_model.py:247-291): 2 encodes +
 * symmetric decode + 2 DPT heads + 2 pose heads, fused fast path (no per-layer outputs).
 * img1 = main view, img2 = support view, each [B,3,H,W].  Outputs, index 0 = main view, 1 = support:
 * pts3d_out_dev [2,B,H,W,3], conf_out_dev [2,B,H,W], pose_out_dev [2,B,4,4], pose_conf_out_dev [2,B]. */
int sta_forward_pairs(StaModel* m, const void* img1_dev, const void* img2_dev, int img_is_bf16, int B, int H, int W,
                      float* pts3d_out_dev, float* conf_out_dev, float* pose_out_dev, float* pose_conf_out_dev,
                      void* stream);

/* Same as sta_forward_pairs but with HOST buffers (pinned or pageable): copies the images to the
 * device, runs the forward, copies the four outputs back and synchronises the stream.
 * This is the end-to-end entry point bench.py times as "e2e". */
int sta_forward_pairs_host(StaModel* m, const void* img1_host, const void* img2_host, int img_is_bf16, int B, int H,
                           int W, float* pts3d_out_host, float* conf_out_host, float* pose_out_host,
                           float* pose_conf_out_host, void* stream);

/* Counters: number of kernel launches issued by this library on behalf of `m` since creation. */
int64_t sta_launch_count(StaModel* m);
/* Bytes of device memory currently held (weights + workspace). */
int64_t sta_device_bytes(StaModel* m);

/* Per-kernel-family device timing with CUDA events on the launch stream (adds two event records per
 * launch while enabled).  Families: 0 = wgmma GEMM (linear), 1 = wgmma GEMM (implicit 3x3 conv),
 * 2 = attention, 3 = LayerNorm.  sta_profile_read synchronises, returns the accumulated milliseconds,
 * launch counts and executed FLOPs per family since the last read, and resets the counters. */
int sta_profile(StaModel* m, int enable);
int sta_profile_read(StaModel* m, double* ms4, int64_t* counts4, double* flops4);

/* Buffer taps (tests): read a forward's intermediate buffers launch by launch.  After each launch of run_encoder,
 * run_decoder, decode_with_poses, run_dpt and forward_chunk whose tap name is set, the runtime enqueues a
 * device-to-device copy of that launch's output, in its physical layout (bf16 rows 3x wide in the x3 mode; FP8 codes
 * and scales as two taps, ".q" and ".s"), on the call's stream to dst + written (bytes), then advances `written` and
 * increments `fired`.  Repeated firings within a call append.  A null dst only counts.  A copy past `capacity` fails the
 * entry point with sta_last_error naming the tap.  The caller owns the array, zeroes written / fired, and keeps it
 * alive until n = 0 clears the taps.  While any tap is set the graphed entry points run eagerly; the copies are not
 * counted by sta_launch_count.  The names are listed in tests/test_forward_taps_gpu.py (TAP_PATTERNS). */
typedef struct {
  const char* name;
  void* dst;
  int64_t capacity;
  int64_t written;
  int32_t fired;
} StaTap;
int sta_set_taps(StaModel* m, StaTap* taps, int n);

/* ---- op-level entry points (used by the parity tests; same kernels the model uses) ---- */

enum { STA_EPI_BF16 = 0, STA_EPI_GELU = 1, STA_EPI_F32 = 2, STA_EPI_ROPE = 3, STA_EPI_PIXSHUF = 4, STA_EPI_HEAD = 5,
       STA_EPI_GELU_FP8 = 6 };

typedef struct StaGemmDesc {
  int conv3x3;          /* 0: A is [M][lda] bf16;  1: A is NHWC [nimg][H][W][Cin] bf16 (3x3, pad 1, stride 1) */
  int epi;              /* STA_EPI_* */
  const void* A;
  int64_t lda;
  const void* W;        /* [N][ldw] bf16; for conv3x3 K = 9*Cin ordered (kh, kw, cin) */
  int64_t ldw;
  int M, N, K;
  int nimg, H, Wd, Cin; /* conv3x3 geometry */
  const float* bias;    /* [N] fp32 or NULL */
  void* out;            /* bf16 (EPI_BF16/GELU/ROPE/PIXSHUF) or fp32 (EPI_F32) */
  int64_t ldo;
  void* out2;           /* EPI_BF16: optional relu copy */
  const void* resid;    /* EPI_BF16: bf16 [.][ldo];  EPI_F32: fp32 [.][ldo] */
  const void* resid2;   /* EPI_BF16 only */
  int relu_main;
  int rowmap_n;         /* EPI_F32: insert one skipped row before every n output rows */
  const int32_t* pos;   /* EPI_ROPE: [M][2] int32 (y, x) */
  int rope_cols;        /* EPI_ROPE: columns [0, rope_cols) are rotated */
  int ps_k, ps_cout, ps_h, ps_w; /* EPI_PIXSHUF */
  const float* head_w;  /* EPI_HEAD: [128][4] fp32 */
  const float* head_b;  /* EPI_HEAD: [4] */
  float* pts3d;         /* EPI_HEAD: [pixels][3] */
  float* conf;          /* EPI_HEAD: [pixels] */
  void* splitk_ws;      /* optional fp32 scratch (16-byte aligned): lets small EPI_F32 problems split K across CTAs */
  int64_t splitk_ws_bytes;
  int split_precision;  /* 1: operands are already expanded along K as A (hi|lo|hi) x W (hi|hi|lo) (K = 3x logical);
                           bf16 outputs / skip tensors use (hi|lo|hi) rows of logical width N (ldo >= 3N) */
  int tile_n;           /* 0: automatic (sta_gemm_auto_tile_n);  128: 128 x 128 tiles;  256: 128 x 256 tiles (linear
                           layers with the TMA-store epilogue, N % 256 == 0, no split-K, not split precision; an error
                           elsewhere).  Both tile shapes give bit-identical results. */
} StaGemmDesc;

int sta_op_gemm(const StaGemmDesc* d, void* stream);
/* The tile columns (256 or 128) the automatic choice takes for a linear layer (M x N, depth K) with epilogue epi that
 * runs the TMA-store epilogue without split-K on a GPU with num_sms SMs.  A function of these arguments only. */
int sta_gemm_auto_tile_n(int M, int N, int K, int epi, int num_sms);

/* The FP8 mode's GEMM (STA_PRECISION_FP8): out = A W^T + bias on e4m3 codes ("fn" format, max 448) with power-of-two
 * scales: A [M][lda] with a_scale [M][K/128] (one per row and 128 columns), W [N][ldw] with w_scale [N/128][K/128] (one
 * per 128 x 128 block).  N and K multiples of 128, lda and ldw multiples of 16.  Each 128-wide k-block is accumulated on
 * its own and folded as acc = fma(blk, a_scale[m][kb] * w_scale[n/128][kb], acc).  Epilogues:
 *   STA_EPI_F32       out fp32 [M][ldo]; resid NULL (out = ...) or resid == out (out += ..., in place)
 *   STA_EPI_ROPE      out bf16 [M][ldo], 2-D RoPE on columns [0, rope_cols) with pos [M][2] int32 (y, x)
 *   STA_EPI_GELU_FP8  out e4m3 [M][ldo] = gelu(.) / s with out_scale [M][N/128] = s, the scales defined as for the inputs
 * (a group's scale is 2^e with e the smallest integer for which amax <= 448 * 2^e, 1 for an all-zero group). */
typedef struct StaGemmFp8Desc {
  int epi;
  const void* A;
  int64_t lda;
  const float* a_scale;
  const void* W;
  int64_t ldw;
  const float* w_scale;
  int M, N, K;
  const float* bias;    /* [N] fp32 or NULL */
  void* out;
  int64_t ldo;
  const void* resid;    /* STA_EPI_F32: NULL or out */
  float* out_scale;     /* STA_EPI_GELU_FP8 */
  const int32_t* pos;   /* STA_EPI_ROPE */
  int rope_cols;
  void* splitk_ws;      /* optional fp32 scratch, as in StaGemmDesc */
  int64_t splitk_ws_bytes;
} StaGemmFp8Desc;
int sta_op_gemm_fp8(const StaGemmFp8Desc* d, void* stream);
/* The FP8 mode's quantisers: e4m3 codes [rows][C] plus scales [rows][C/128] as for the GEMM's A operand.
 * sta_op_layernorm_fp8: LayerNorm of fp32 x (C = 768 or 1024) straight to e4m3, optionally a second output with other
 * affine parameters (g2 / b2 / q2 / s2, or NULL).  sta_op_quant_fp8: bf16 rows -> e4m3 (C a multiple of 128). */
int sta_op_layernorm_fp8(const float* x, int rows, int C, float eps, const float* g1, const float* b1, void* q1, float* s1,
                         const float* g2, const float* b2, void* q2, float* s2, void* stream);
int sta_op_quant_fp8(const void* in_bf16, int64_t rows, int C, void* q, float* s, void* stream);

/* softmax(q k^T * scale) v, head_dim 64.  q/k/v: [batch][n*][ld*] bf16 with head h at columns
 * *_col0 + 64*h; out: [batch][nq][ldo] bf16.  kv sample for query sample b is (b + kv_batch_shift) % batch. */
int sta_op_attention(const void* q, int64_t ldq, int q_col0, const void* k, int64_t ldk, int k_col0, const void* v,
                     int64_t ldv, int v_col0, void* out, int64_t ldo, int batch, int heads, int nq, int nk,
                     int kv_batch_shift, float scale, void* stream);
/* The same in the split-precision parity mode (STA_PRECISION_X3): q/k/v/out rows are (hi | lo | hi) bf16, ld* are the
 * physical strides (3x the logical width) and *_col0 are offsets of the hi columns; out stores (hi | lo | hi).
 * Requires 0 <= kv_batch_shift < batch, *_col0 + 64*heads <= ld* (ld* / 3 in split mode), 64*heads <= ldo (ldo / 3)
 * and a finite scale > 0 (both entry points). */
int sta_op_attention_split(const void* q, int64_t ldq, int q_col0, const void* k, int64_t ldk, int k_col0,
                           const void* v, int64_t ldv, int v_col0, void* out, int64_t ldo, int batch, int heads, int nq,
                           int nk, int kv_batch_shift, float scale, void* stream);

int sta_op_layernorm(const float* x, int rows, int C, float eps, const float* g1, const float* b1, void* out1_bf16,
                     const float* g2, const float* b2, void* out2_bf16, int drop_first_of, void* stream);
int sta_op_patch_im2col(const void* img, int img_is_bf16, int B, int H, int W, void* out_bf16, void* stream);
int sta_op_upsample2x(const void* in_bf16, void* out_bf16, int nimg, int H, int W, int C, void* stream);
int sta_op_im2col_3x3_s2(const void* in_bf16, void* out_bf16, int nimg, int H, int W, int C, void* stream);
int sta_op_cast_f32_bf16(const float* in, void* out_bf16, int64_t rows, int C, int drop_first_of, void* stream);


/* ---- keyframe step (SURVEY.md 8(f) rank 1): OnlineSLAM.regress_two_views (vista_slam/slam.py:153-189) for K edges
 * (i, j_k) at once, from cached encoder features: symmetric decoder on the K feature pairs, head_pose_s on both
 * pose tokens, head_pts on both views, then estimate_intrinsic_from_pts3d(shared_intrinsic=True) per edge,
 * depths = pts3d[..., 2] and conf.mean().  Token positions are the regular (y, x) grid of PositionGetter
 * (sta_blocks.py:235-247), which is what slam.py:145 caches.  All outputs are [2][K]...: block 0 = the (i -> j)
 * direction ("ij"), block 1 = "ji".  intri_out [K][3][3], depth_out, conf_mean_out [2][K] may be NULL; scratch as for
 * sta_pointmap_consumers with V = 2K (only needed when intri_out / depth_out / conf_mean_out is given).
 * No host synchronisation: the caller decides when to read rel_pose_conf (slam.py:169). ---- */
int sta_regress_pairs(StaModel* m, const float* feat_i_dev, const float* feat_j_dev, int K, int H, int W,
                      float* pose_out_dev, float* pose_conf_out_dev, float* pts3d_out_dev, float* conf_out_dev,
                      float* intri_out_dev, float* depth_out_dev, float* conf_mean_out_dev, void* scratch, void* stream);

/* The same step in two phases, keeping the reference's early-out (slam.py:169-170: `rel_pose_conf < thres and i - j != 1`
 * skips both DPT heads): _begin runs the symmetric decoder and the pose heads for all K candidate edges
 * (pose_out [2][K][4][4], pose_conf_out [2][K]; block 0 = the i -> j direction) and keeps the decoder hooks in the
 * handle's workspace; the caller reads the K confidences (ONE device-to-host copy per keyframe instead of one per edge),
 * and _finish runs the DPT heads + pointmap consumers only for the n_sel surviving edges edge_idx_host[0..n_sel)
 * (indices into the K candidates; host memory).  Outputs of _finish are compact: pts3d_out [2][n_sel][H][W][3],
 * conf_out [2][n_sel][H][W], intri_out [n_sel][3][3], depth_out / conf_mean_out optional, scratch for V = 2 n_sel.
 * _begin records its shape and where it left the hooks in the handle.  Any other model call on this handle ends the
 * pair: a later _finish is then refused with an error, before any launch. */
int sta_regress_pairs_begin(StaModel* m, const float* feat_i_dev, const float* feat_j_dev, int K, int H, int W,
                            float* pose_out_dev, float* pose_conf_out_dev, void* stream);
int sta_regress_pairs_finish(StaModel* m, const int* edge_idx_host, int n_sel, float* pts3d_out_dev, float* conf_out_dev,
                             float* intri_out_dev, float* depth_out_dev, float* conf_mean_out_dev, void* scratch,
                             void* stream);

/* Launch-bound sizes (<= 8192 tokens per call: one keyframe, a few edges) of sta_encode and sta_regress_pairs are
 * captured into CUDA graphs per (entry point, batch, H, W) on their second use and replayed afterwards (not while
 * sta_profile is enabled).  Number of graph replays so far (tests / diagnostics): */
int64_t sta_graph_replays(StaModel* m);

/* ---- pointmap consumers (SURVEY.md 8(f) rank 2): what OnlineSLAM.regress_two_views / connect_view_i_j compute from
 * the head outputs right after the boundary.  Device pointers, fp32; `scratch` is a caller-owned device buffer of
 * sta_pointmap_scratch_bytes(V) bytes (8-byte aligned).  No host synchronisation. ---- */
size_t sta_pointmap_scratch_bytes(int V);
/* estimate_intrinsic_from_pts3d (vista_slam/utils/slam_utils.py:8-79, call site slam.py:184) fused with
 * depths = pts3d[..., 2] (slam.py:185) and conf.mean() per view (pose_graph.py:41).
 * pts3d [V][H][W][3], conf [V][H][W]; shared = 0 -> K_out [V][3][3]; 1 -> one K_out [3][3] over all views;
 * 2 -> K_out [V/2][3][3], edge e from its two views (e, e + V/2), i.e. shared_intrinsic=True per (ij, ji) pair;
 * depth_out [V][H][W] and conf_mean_out [V] may be NULL. */
int sta_pointmap_consumers(const float* pts3d, const float* conf, int V, int H, int W, int shared, float* K_out,
                           float* depth_out, float* conf_mean_out, void* scratch, void* stream);
/* estimate_scale_with_depth_and_confidence (slam_utils.py:168-190, call site slam.py:224) and
 * scale_conf = (ci * cj).sqrt().mean() (slam.py:227): out2 = {scale, scale_conf}; n elements per map. */
int sta_depth_scale(const float* Di, const float* Dj, const float* ci, const float* cj, int64_t n, float* out2,
                    void* scratch, void* stream);


/* ---- Sim(3) pose-graph Levenberg-Marquardt step (SURVEY.md 8(f) rank 4): one iteration of the optimisation in
 * OnlineSLAM.pose_graph_optimize (vista_slam/slam.py:108-140) over PoseGraphOpt (vista_slam/pose_graph.py:70-154):
 * residuals r_e = Log(T_e X_i^-1 X_j) of the edges with at least one optimised endpoint, their Jacobians w.r.t. left
 * perturbations X <- Exp(delta) X (what PyPose's LieTensor parameters use), A = J^T W J with W = diag(weights_e) and the LM
 * damping of pp.optim.LM.step (diagonal clamped to [dmin, dmax], then scaled by 1 + damping), a dense Cholesky solve of
 * A d = -J^T W r, and the update.  Device pointers: nodes / nodes_out [num_nodes][8] and meas [num_edges][8] fp32 Sim3 in
 * PyPose's layout (tx ty tz | qx qy qz qw | s), edges [num_edges][2] int64 (i, j), weights [num_edges][7] fp32,
 * opt_idx [num_opt] int64 (the optimised nodes, all others stay fixed).  info_out (device) [4] fp64 = {loss before,
 * loss after, |delta|_2, Cholesky ok (1/0)}; loss = sum r^T W r.  fp64 inside, deterministic, no host synchronisation: the
 * caller reads info_out to accept or reject the step (as pp.optim.LM does).  scratch: sta_pose_graph_scratch_bytes.
 * The dense route keeps the 7 num_opt right-hand side in one CTA's shared memory (200 KB): it refuses num_opt above
 * STA_PG_DENSE_MAX_OPT, and its scratch holds the dense (7 num_opt)^2 fp64 matrix.  Larger graphs take the
 * block-sparse route below. ---- */
enum { STA_PG_DENSE_MAX_OPT = 3657 };
size_t sta_pose_graph_scratch_bytes(int num_nodes, int num_edges, int num_opt);
int sta_pose_graph_lm_step(const float* nodes, int num_nodes, const int64_t* edges, const float* meas, const float* weights,
                           int num_edges, const int64_t* opt_idx, int num_opt, double damping, double dmin, double dmax,
                           float* nodes_out, double* info_out, void* scratch, void* stream);

/* ---- the same dense LM step on a group of G independent graphs, in one launch sequence: each graph has its own nodes,
 * edges, measurements, weights, optimised set, damping and nodes_out (the device pointers and layouts of
 * sta_pose_graph_lm_step), and its info row info_out[4 k .. 4 k + 3] (device, G x 4 fp64, the layout above).  Each
 * graph's nodes_out and info row are bit-identical to its own sta_pose_graph_lm_step, whichever graphs share the group
 * and in whatever order: no reduction crosses graphs.  No host synchronisation; read all G info rows back with one copy.
 * The descriptor table is read on the call (it travels as a kernel parameter), so it may be rebuilt for every step.
 * Refused with a status before any launch: a null table, info_out or scratch, G outside [1, STA_PG_GROUP_MAX], a null
 * pointer or an empty graph (no nodes, edges or optimised nodes), num_opt > num_nodes, num_opt above
 * STA_PG_DENSE_MAX_OPT, and scratch_bytes below sta_pose_graph_group_scratch_bytes.  The scratch holds the descriptor
 * table and each graph's scratch one after another; the scratch-size function returns 0 for a table it would refuse.
 * A group of one runs sta_pose_graph_lm_step's launch sequence. ---- */
enum { STA_PG_GROUP_MAX = 16 };
typedef struct StaPgGraph {
  const float* nodes;     /* [num_nodes][8] */
  const int64_t* edges;   /* [num_edges][2] */
  const float* meas;      /* [num_edges][8] */
  const float* weights;   /* [num_edges][7] */
  const int64_t* opt_idx; /* [num_opt] */
  float* nodes_out;       /* [num_nodes][8] */
  int num_nodes, num_edges, num_opt;
  double damping;
} StaPgGraph;
size_t sta_pose_graph_group_scratch_bytes(const StaPgGraph* graphs, int G);
int sta_pose_graph_lm_step_group(const StaPgGraph* graphs, int G, double dmin, double dmax, double* info_out, void* scratch,
                                 size_t scratch_bytes, void* stream);

/* ---- block-sparse route of the same LM step, for any number of optimised nodes: identical residuals, Jacobians,
 * normal equations (A, g and loss before equal the dense route's), damping, update and losses; A d = -g is solved by a
 * block Cholesky factorisation with 7x7 blocks under a nested-dissection ordering, scheduled by elimination-tree levels.
 * A plan holds the symbolic analysis of one edge list and one optimised set (fixed over the iterations of one
 * optimisation), device copies of both and the per-iteration scratch.  sta_pg_plan_create takes HOST arrays
 * edges [num_edges][2] and opt_idx [num_opt] (int64) and refuses, before anything reaches the device: an empty
 * problem, edge endpoints outside [0, num_nodes), optimised indices out of range or repeated.  It allocates and
 * uploads synchronously; the plan is used on the device that was current at creation. ---- */
typedef struct StaPgPlan StaPgPlan; /* opaque */
int sta_pg_plan_create(const int64_t* edges_host, int num_edges, int num_nodes, const int64_t* opt_idx_host, int num_opt,
                       StaPgPlan** out);
void sta_pg_plan_destroy(StaPgPlan* plan);
/* out4 = {nonzero 7x7 blocks of L, elimination-tree levels, device bytes of the plan, block updates L_Ij L_Kj^T per
 * factorisation} */
int sta_pg_plan_info(const StaPgPlan* plan, int64_t* out4);
/* The host analysis alone (no GPU needed): stats5 = {nonzero blocks of L, nonzero blocks of A's lower triangle, levels,
 * block updates, device bytes a plan would take}.  Optional outputs (NULL to skip), sized from stats5 by a first call:
 * order [num_opt] (positions of opt_idx in elimination order), level [num_opt] (elimination-tree level per position),
 * colptr [num_opt + 1] and blk_row [L blocks] (block pattern of L by column, diagonal block first, then rows ascending),
 * upd_ptr [L blocks + 1] and upd [2 updates] (per block of L, the pairs of block indices (L_Ij, L_Kj), j ascending). */
int sta_pg_plan_analyze(const int64_t* edges_host, int num_edges, int num_nodes, const int64_t* opt_idx_host, int num_opt,
                        int64_t* stats5, int* order, int* level, int* colptr, int* blk_row, int64_t* upd_ptr, int* upd);
/* One LM step on the plan's edges and optimised set.  Device pointers as in sta_pose_graph_lm_step (nodes / nodes_out
 * [num_nodes][8], meas [num_edges][8], weights [num_edges][7]); info_out has the same layout.  No host synchronisation;
 * steps on one plan must not overlap (the scratch is the plan's). */
int sta_pose_graph_lm_step_sparse(const StaPgPlan* plan, const float* nodes, const float* meas, const float* weights,
                                  double damping, double dmin, double dmax, float* nodes_out, double* info_out, void* stream);
/* The last step's update d (device, fp64 [num_opt][7] in opt_idx order), for checking the solve: stream-ordered copy. */
int sta_pg_plan_last_delta(const StaPgPlan* plan, double* delta_out, void* stream);

/* ---- the block-sparse LM step over a group of G plans (1 <= G <= STA_PG_GROUP_MAX), in one launch sequence whose
 * length does not grow with G: one launch per kernel and elimination-tree level covers every member, the grid's y
 * dimension selecting the member.  Each active member's nodes_out and info row (info_out[4 k .. 4 k + 3], device,
 * G x 4 fp64) are bit-identical to sta_pose_graph_lm_step_sparse on its own plan, whatever the other members, their
 * order and which of them are active: no reduction crosses plans.  An inactive member (active = 0) is neither read nor
 * written, its info row included.  No host synchronisation; steps and dampings may change on every call.
 * The group plan borrows the member plans' device arrays and scratch and uploads only its own small tables (creation
 * synchronises once): the member plans must outlive it, steps on one group plan must not overlap, and a member plan may
 * be stepped on its own between group steps, in stream order.  A member's sta_pg_plan_last_delta gives its last
 * update, from whichever entry point ran it.
 * Refused with a status before any launch: a null pointer, G outside [1, STA_PG_GROUP_MAX], a plan named twice
 * (its scratch would be shared), a plan created on a device other than the current one, and, at a step, a null
 * info_out or steps table, an active member with a null nodes, meas, weights or nodes_out, or a current device other
 * than the group plan's. ---- */
typedef struct StaPgGroupPlan StaPgGroupPlan; /* opaque */
int sta_pg_group_plan_create(const StaPgPlan* const* plans, int G, StaPgGroupPlan** out);
void sta_pg_group_plan_destroy(StaPgGroupPlan* gp);
/* out4 = {G, elimination-tree levels (the most of any member), kernel launches per step, device bytes of the group plan} */
int sta_pg_group_plan_info(const StaPgGroupPlan* gp, int64_t* out4);
typedef struct StaPgSparseStep {
  const float* nodes;   /* [num_nodes][8] of the member's plan */
  const float* meas;    /* [num_edges][8] */
  const float* weights; /* [num_edges][7] */
  float* nodes_out;     /* [num_nodes][8] */
  double damping;
  int active;           /* 0: the member sits this step out */
} StaPgSparseStep;
int sta_pose_graph_lm_step_sparse_group(const StaPgGroupPlan* gp, const StaPgSparseStep* steps /* [G] */, double dmin,
                                        double dmax, double* info_out, void* stream);

/* ---- image preprocessing (SURVEY.md 8(f) rank 3): SLAM_image_only.process_image
 * (vista_slam/datasets/slam_images_only.py:22-34 -> datasets/base/base_view_graph_dataset.py:171-225 ->
 * utils/cropping.py:54-84,102-118 with PIL LANCZOS -> utils/image.py:13) on the device, bit-exact with PIL's 8-bit
 * resampler and torchvision's ToTensor / Normalize(0.5, 0.5) / Grayscale.  rgb [H][W][3] uint8 (RGB order) on the
 * device; res_w >= res_h is the dataset `resolution` (portrait frames get the transposed one, as in the reference).
 * Outputs: rgb_out [3][oh][ow] fp32 in [-1, 1] (the STA input), gray_out [oh][ow] fp32 in [0, 1] or NULL,
 * u8_out [oh][ow][3] (the resized crop itself) or NULL.  sta_preprocess_shape returns (oh, ow) without touching
 * the GPU.  Coefficient tables and the intermediate image are cached per (device, frame geometry); calls for one
 * geometry must not overlap on different streams. ---- */
int sta_preprocess_shape(int H, int W, int res_w, int res_h, int w_edge, int h_edge, int* out_hw);
/* Host-only test hooks (no GPU): the crop/resize geometry {crop l, t, r, b, resized w, h, final l, t, out w, h} and
 * the fixed-point Lanczos windows of one axis (Resample.c precompute_coeffs + normalize_coeffs_8bpc): *ksize taps per
 * output sample, bounds [out_size][2] = (first input sample, tap count), kk [out_size][*ksize] int32 (22-bit). */
int sta_preprocess_geometry(int H, int W, int res_w, int res_h, int w_edge, int h_edge, int* out10);
int sta_preprocess_coeffs(int in_size, int out_size, int* ksize, int* bounds, int* kk, int64_t kk_capacity);
int sta_preprocess_rgb8(const uint8_t* rgb_dev, int H, int W, int res_w, int res_h, int w_edge, int h_edge,
                        float* rgb_out_dev, float* gray_out_dev, uint8_t* u8_out_dev, void* stream);
/* F same-size frames in one launch pair, each bit-identical to its own sta_preprocess_rgb8 (its F = 1 case): rgb
 * [F][H][W][3] -> rgb_out [F][3][oh][ow], gray_out [F][oh][ow] or NULL, u8_out [F][oh][ow][3] or NULL.  F in
 * [1, 65535]; the cached intermediate image grows to the largest F of its geometry. */
int sta_preprocess_rgb8_many(const uint8_t* rgb_dev, int F, int H, int W, int res_w, int res_h, int w_edge, int h_edge,
                             float* rgb_out_dev, float* gray_out_dev, uint8_t* u8_out_dev, void* stream);

/* ---- keyframe flow tracker: FlowTracker.compute_disparity (vista_slam/flow_tracker.py:26-66) on the device, with the
 * reference's fixed constants: cv2.goodFeaturesToTrack(maxCorners=1000, qualityLevel=0.01, minDistance=8, blockSize=7)
 * and cv2.calcOpticalFlowPyrLK(winSize=(21,21), maxLevel=3, criteria=(EPS|COUNT, 30, 0.01)).  A frame is [H][W] uint8
 * (frame_is_f32 = 0) or the [H][W] fp32 gray in [0,1] that sta_preprocess_rgb8 writes (1), converted as
 * (gray * 255).astype(uint8).  Frame sides must be in [32, 2048]; the size checks come before any CUDA call.
 * A tracker handle owns, for one frame size, the keyframe's pyramid, derivatives and corners, corner scratch, the
 * pyramids of the frames of its group tracks (one from creation on, more allocated on first use for larger groups) and
 * the LK output and statistics of the groups it leads (16 frames' from creation on).  One stream at a time: work on a
 * new stream waits for the previous one. ---- */
enum { STA_FLOW_MAX_CORNERS = 1000 };
typedef struct StaFlowTracker StaFlowTracker; /* opaque */
typedef struct StaFlowStats {
  int32_t n_corners;     /* keyframe corners */
  int32_t n_tracked;     /* points with status 1 */
  double abs_sum;        /* sum over tracked points of |dx| + |dy| of the fp32 differences next - keyframe, in fp64 */
  double mean_disparity; /* abs_sum / (2 n_tracked): the reference's mean of |dx| and |dy|; 0 when n_tracked = 0 */
} StaFlowStats;
int sta_flow_create(int H, int W, StaFlowTracker** out);
void sta_flow_destroy(StaFlowTracker* t);
/* The tracker works on groups: many frames and many trackers (SLAM sessions, or a run of frames of one tracker), one
 * frame being a group of one; every per-frame result is independent of the group.  All trackers of a group share one
 * frame size; frames are [n][H][W] uint8 or fp32 gray as above.  Refused before any launch: n or F < 1, a null pointer,
 * mixed tracker sizes, and the per-call conditions below.
 * sta_flow_set_keyframe_group: initialize_keyframe of frame i on ts[i] (n distinct trackers): its pyramid, Scharr
 * derivatives and corners; asynchronous.
 * sta_flow_track_group: frame f belongs to ts[f]; a tracker's frames are consecutive and in its own order, and every
 * one is tracked against the tracker's current keyframe (which must exist) in one launch per stage, with the
 * statistics reduced per frame, then the one host synchronisation: stats_out [F] (host).  held_host [F] (or NULL:
 * none) marks the frames whose pyramids the tracker still holds from its last group track: the frames after the one
 * sta_flow_promote_group promoted, reused in order as a prefix of its frames here (at most as many as it holds).
 * frames_dev holds only the other frames, in group order (NULL when there are none).
 * sta_flow_promote_group: frame frame_host[i] (its index among ts[i]'s frames of its last group track) becomes the
 * keyframe of ts[i] (n distinct trackers) without a rebuild; their derivatives and corners are enqueued as one
 * sequence; asynchronous.  Refused for a tracker with no group track since its last keyframe. */
int sta_flow_set_keyframe_group(StaFlowTracker* const* ts, int n, const void* frames_dev, int frames_is_f32,
                                void* stream);
int sta_flow_track_group(StaFlowTracker* const* ts, int F, const int* held_host, const void* frames_dev,
                         int frames_is_f32, StaFlowStats* stats_out, void* stream);
int sta_flow_promote_group(StaFlowTracker* const* ts, int n, const int* frame_host, void* stream);
/* Device copies of the keyframe corners: pts_out [STA_FLOW_MAX_CORNERS][2] fp32 (x, y) in selection order, the first
 * *count_out valid; and of the keyframe's level-0 image [H][W] uint8 and derivatives [H][W][2] int16 (either may be
 * NULL). */
int sta_flow_keyframe_points(StaFlowTracker* t, float* pts_out_dev, int* count_out_dev, void* stream);
int sta_flow_keyframe_level0(StaFlowTracker* t, uint8_t* gray_out_dev, int16_t* deriv_out_dev, void* stream);
/* Op-level entry points (the same kernels).  scratch: a device buffer of sta_flow_scratch_bytes(H, W) bytes (256-byte
 * aligned); 0 for a refused size.  good_features: pts_out [STA_FLOW_MAX_CORNERS][2], count_out [1] (device).
 * lk_track: pts [n][2] -> next_pts_out [n][2], status_out [n] uint8 (device). */
size_t sta_flow_scratch_bytes(int H, int W);
int sta_op_good_features(const uint8_t* gray_u8, int H, int W, float* pts_out, int* count_out, void* scratch, void* stream);
int sta_op_lk_track(const uint8_t* prev_u8, const uint8_t* next_u8, int H, int W, const float* pts, int n,
                    float* next_pts_out, uint8_t* status_out, void* scratch, void* stream);

/* ---- loop detection: LoopDetector (vista_slam/loop_detector.py) on the device -- cv2.ORB_create().detectAndCompute
 * with OpenCV's defaults, the DBoW3 vocabulary transform with BowVector::normalize(L1), L1Scoring::score and
 * detect_loop.  Frames are [H][W] uint8 (frame_is_f32 = 0) or the fp32 gray in [0,1] of sta_preprocess_rgb8 (1),
 * converted as (gray * 255).astype(uint8); sides must be in [32, 4096].
 * A vocabulary is a DBoW3 text file (*.txt, load_fromtxt) or a binary stream (toStream, plain or QuickLZ), with 32-byte
 * binary descriptors and L1 scoring; anything else is refused.  It is parsed on the host and uploaded once to the
 * current device.  A detector owns ORB scratch for one frame size and the database of every view's vector. ---- */
typedef struct StaVocab StaVocab;             /* opaque */
typedef struct StaLoopDetector StaLoopDetector; /* opaque */
enum { STA_ORB_MAX_KEYPOINTS = 4096 };
int sta_vocab_load(const char* path, StaVocab** out);
/* out6 = {k, L, scoring, weighting, nodes, words} */
int sta_vocab_info(const StaVocab* v, int64_t* out6);
void sta_vocab_destroy(StaVocab* v);
int sta_loop_create(StaVocab* v, int loop_dist_min, int loop_nms, int loop_cand_thresh_neighbor, StaLoopDetector** out);
void sta_loop_destroy(StaLoopDetector* d);
int sta_loop_views(const StaLoopDetector* d);
/* compute_bow_feat and detect_loop over F >= 1 frames [F][H][W] of one size, of one detector or of several that share
 * one StaVocab (SLAM sessions stepped together; refused before any launch otherwise).  Frame f belongs to dets[f]; a
 * detector's frames are consecutive and in its own order; one detector's frame is a group of one.  Every per-frame
 * result is independent of the group.
 * sta_loop_add_frames_group: compute_bow_feat for every frame: ORB over the F frames, one transform, one build CTA per
 * frame and one append launch into each frame's own database (a view's vector is None when ORB finds no keypoint);
 * asynchronous, unless dets[0]'s previous add has had no detect since: then the stream is synchronised first.
 * sta_loop_detect_group: detect_loop for the frames of the last add of dets[0] (the same dets and F, no view added to
 * them since), farthest_host[f] in [0, view index of frame f in its detector]: similarities against every earlier view
 * of its detector in one score launch over all rows, the candidate scan in one thread per row, and the one host
 * synchronisation: n_out [2F] = {candidates, length of the frame's vector (-1: None)} per row, row f's first
 * cap_per_view candidates at js_out / sims_out + f cap_per_view (host) in the reference's order (descending
 * similarity, ties in descending j).  An ORB overflow is reported with the frame's index in the group.  The ORB
 * scratch, staging and result buffers of a group are dets[0]'s.  Afterwards sta_loop_similarities returns the last
 * row when every row was dets[0]'s, and is refused on the group's detectors until their own next detect otherwise. */
int sta_loop_add_frames_group(StaLoopDetector* const* dets, int F, const void* frames_dev, int frames_is_f32,
                              int H, int W, void* stream);
int sta_loop_detect_group(StaLoopDetector* const* dets, int F, const int* farthest_host, int* n_out,
                          int64_t* js_out, double* sims_out, int cap_per_view, void* stream);
/* Test read-backs (synchronise): a view's vector (len -1 for None) and the last similarity row of the last detect (NaN
 * where either vector is None; n at most that row's view index). */
int sta_loop_view(StaLoopDetector* d, int view, int32_t* words_out, double* vals_out, int cap, int* len_out, void* stream);
int sta_loop_similarities(StaLoopDetector* d, double* sims_out, int n, void* stream);
/* Op-level entry points (the same kernels).  ORB: scratch of sta_orb_scratch_bytes(H, W) bytes (256-byte aligned; 0 for
 * a refused size); outputs [STA_ORB_MAX_KEYPOINTS] in (level, y, x) order, count_out [1] (all device): xy in level
 * pixels (int32 x, y), level, pts in level-0 pixels (fp32 x, y), angle (degrees), Harris response, desc [32].
 * sta_orb_layout: out[0..9] = {total, pyramid, blurred, fast scores, candidates, responses, counters, alive, kept,
 * histogram} byte offsets in the scratch, then per level {h, w, pixel offset, feature quota}. */
size_t sta_orb_scratch_bytes(int H, int W);
int sta_orb_layout(int H, int W, int64_t* out42);
int sta_op_orb(const void* frame_dev, int frame_is_f32, int H, int W, int32_t* xy_out, int32_t* level_out, float* pts_out,
               float* angle_out, float* response_out, uint8_t* desc_out, int32_t* count_out, void* scratch, void* stream);
/* The same for F frames [F][H][W] of one size: scratch of F sta_orb_scratch_bytes(H, W) bytes (frame f's slice at f times
 * that), outputs [F][STA_ORB_MAX_KEYPOINTS] (desc [F][STA_ORB_MAX_KEYPOINTS][32]), count_out [F]; each frame's outputs
 * and scratch equal sta_op_orb's on that frame. */
int sta_op_orb_many(const void* frames_dev, int frames_is_f32, int F, int H, int W, int32_t* xy_out, int32_t* level_out,
                    float* pts_out, float* angle_out, float* response_out, uint8_t* desc_out, int32_t* count_out,
                    void* scratch, void* stream);
/* Per descriptor [n][32] (device): word id and weight of the leaf it descends to. */
int sta_op_bow_transform(const StaVocab* v, const uint8_t* desc_dev, int n, int32_t* word_out, double* weight_out,
                         void* stream);
/* The normalised BowVector of n <= STA_ORB_MAX_KEYPOINTS (word, weight) pairs: words_out / vals_out [n], len_out [1]. */
int sta_op_bow_vector(const StaVocab* v, const int32_t* word, const double* weight, int n, int32_t* words_out,
                      double* vals_out, int32_t* len_out, void* stream);
/* L1 score of one vector (qw, qv, *q_len_dev; -1 = None) against nviews CSR vectors (db_start int64, db_len -1 = None). */
int sta_op_bow_score(const int32_t* qw, const double* qv, const int32_t* q_len_dev, const int32_t* db_word,
                     const double* db_val, const int64_t* db_start, const int32_t* db_len, int nviews, double* sims_out,
                     void* stream);

/* ---- device pose graph: the bookkeeping of OnlineSLAM (vista_slam/slam.py:191-241 over pose_graph.py:5-54) and the
 * gather of save_data_all / get_view (slam.py:299-412) on the device.  A graph handle owns fixed-capacity device tables,
 * all poses starting as the identity (PoseGraphNodes.reset):
 *   per node  pose [max_nodes][8] fp32 Sim3 in PyPose's layout (tx ty tz | qx qy qz qw | s), depth and conf
 *             [max_nodes][H][W] fp32, intri [max_nodes][3][3], conf mean [max_nodes] fp32, node_to_view and
 *             node_to_connected_view [max_nodes] int64 (-1 = unused);
 *   per view  best node [max_views] int64 (-1) and its conf mean [max_views] fp32 (-100);
 *   per edge  endpoints [max_edges][2] int64 (-1), measurement [max_edges][8] fp32 Sim3, weight [max_edges][7] fp32 (1).
 * The map store is 8 H W max_nodes bytes: 1.44 GB at OnlineSLAM's defaults (3600 nodes) and 224 x 224.
 * sta_graph_tables: the 12 device pointers in that order (pose, depth, conf, intri, conf mean, node_to_view,
 * node_to_connected_view, best node, best mean, edges, measurements, weights). ---- */
typedef struct StaGraph StaGraph; /* opaque */
enum { STA_GRAPH_MAX_KEYFRAME_EDGES = 32, STA_GRAPH_FLAG_NOT_SO3 = 1, STA_GRAPH_MAX_GROUP_KEYFRAMES = 32 };
int sta_graph_create(int max_nodes, int max_edges, int max_views, int H, int W, StaGraph** out);
void sta_graph_destroy(StaGraph* g);
int sta_graph_tables(const StaGraph* g, void** out12);
/* Back to the state of sta_graph_create; clears the flags. */
int sta_graph_reset(StaGraph* g, void* stream);
/* Flags the device has raised (STA_GRAPH_FLAG_NOT_SO3: a pose rotation was not orthonormal with det +1 to 1e-3, which
 * pp.mat2SE3(atol=1e-3) refuses).  The flags live in mapped host memory: this reads them without synchronising, so a
 * flag raised by a launch is visible once the caller has synchronised with it. */
int sta_graph_flags(const StaGraph* g, int* flags_out);
/* Insert the n kept edges (i = view, j = js_host[k]) of one keyframe in the reference's order (connect_view_i_j per edge:
 * node of i, its scale edge to i's first node when k > 0, node of j, its scale edge to first_j_host[k] when that is
 * >= 0, then the pose edge (i, j)).  Node slots are node0 + 2k (i) and node0 + 2k + 1 (j); edges fill edge0, edge0 + 1, ...
 * Host integers: js_host, cand_host (row of edge k in pose_dev / pose_conf_dev), first_j_host (first node of view j when
 * edge k is inserted, -1 if none).  Device inputs, as regress_views_gated leaves them: pose_dev [*][4][4], pose_conf_dev
 * [*], confs_dev / depths_dev [2][n][H][W] (row 0 view i, row 1 view j), intri_dev [n][3][3], conf_mean_dev [2][n].
 * Two launches, no host synchronisation.  Refused before any launch: a capacity overflow, a map size other than the
 * graph's, host memory as input, n outside [1, STA_GRAPH_MAX_KEYFRAME_EDGES]. */
int sta_graph_add_keyframe(StaGraph* g, int view, int n, const int64_t* js_host, const int* cand_host,
                           const int* first_j_host, int node0, int edge0, int H, int W, const float* pose_dev,
                           const float* pose_conf_dev, const float* confs_dev, const float* depths_dev, const float* intri_dev,
                           const float* conf_mean_dev, void* stream);
/* One keyframe of sta_graph_add_keyframes: sta_graph_add_keyframe's arguments (js / cand / first_j host arrays of n
 * entries, the device inputs as there). */
typedef struct StaGraphKeyframe {
  StaGraph* graph;
  int view, n, node0, edge0, H, W;
  const int64_t* js;
  const int* cand;
  const int* first_j;
  const float *pose, *pose_conf, *confs, *depths, *intri, *conf_mean;
} StaGraphKeyframe;
/* Insert count keyframes, of one graph or of several, with two launches in all and no host synchronisation: every
 * table and the flags end as count consecutive sta_graph_add_keyframe calls in table order would leave them, bit for
 * bit.  A graph's keyframes go in in table order, and each must continue its graph's previous keyframe in the table
 * (node0 = previous node0 + 2 n, edge0 = previous edge0 + its scale edges + n); a keyframe's scale edge to a node that
 * an earlier keyframe of the call inserts reads that keyframe's inputs.  scratch (device, 8-byte aligned) holds the
 * scale reductions' records: sta_graph_add_keyframes_scratch_bytes(kfs, count) bytes, which is 0 for a table the call
 * would refuse (the reason is then in sta_last_error), so it also checks a table without launching.  Refused before any launch, with every table untouched: any refusal of
 * sta_graph_add_keyframe for any keyframe, a keyframe that does not continue its graph's previous one, count outside
 * [1, STA_GRAPH_MAX_GROUP_KEYFRAMES], a null or too small scratch.  sta_graph_add_keyframe is a group of one over
 * the same kernels, with the graph's own scratch. */
size_t sta_graph_add_keyframes_scratch_bytes(const StaGraphKeyframe* kfs, int count);
int sta_graph_add_keyframes(const StaGraphKeyframe* kfs, int count, void* scratch, size_t scratch_bytes, void* stream);
/* Re-derive node poses after their parents' poses changed: for t = 0 .. count - 1 in order, with (node, parent, edge) =
 * triples_host[3t .. 3t + 2], pose[node] = pose[parent] * measurement[edge], the Sim(3) product sta_graph_add_keyframe
 * uses when it inserts a node.  Listed in insertion order (a keyframe's first j node before its i node), the triples of
 * nodes inserted since a pose snapshot bring them to the poses they would have had if inserted after the snapshot's
 * poses were written, bit for bit.  One single-thread launch per 256 triples, no host synchronisation.  Refused before
 * any launch: a node or parent outside [0, max_nodes), a node that is its own parent, an edge outside [0, max_edges). */
int sta_graph_replay_nodes(StaGraph* g, int count, const int* triples_host, void* stream);
/* Track F frames against the graph without changing it.  Frame f was regressed as the pair (frame, keyframe view k)
 * (sta_regress_pairs_begin / _finish): pose_dev [F][4][4] its i -> j pose T, depth_dev / conf_dev [F][H][W] its k-side
 * maps.  anchors_host[f] is the first node of view k.  Per frame:
 *   s = the scale edge reduction of sta_graph_add_keyframe (depth_k, depth_anchor, conf_k, conf_anchor), same grid;
 *   T as Sim(3) [t | q | 1] (meas_out [F][8]), s (scale_edge_out [F]), valid_out [F] = 1 unless T's rotation fails
 *   the orthonormality check that raises STA_GRAPH_FLAG_NOT_SO3 for a keyframe (the flag is not raised here);
 *   pose = pose[anchor] * Sim3(0, id, s) * Sim3(T): pose_out [F][4][4] with the scale dropped and scale_out [F], as
 *   sta_graph_export gives keyframes.  This is bit for bit the pose sta_graph_add_keyframe gives node i of a keyframe
 *   whose first kept edge is (i, k) with the same inputs.
 * scratch: sta_graph_track_frames_scratch_bytes(F) bytes, 8-byte aligned (0 for F outside the range).  Two launches,
 * the anchors passed as kernel parameters, no host synchronisation.  Refused before any launch: F outside
 * [1, STA_GRAPH_MAX_TRACK_FRAMES], a null argument, an anchor outside [0, max_nodes), host memory, a small scratch. */
enum { STA_GRAPH_MAX_TRACK_FRAMES = 4096 };
size_t sta_graph_track_frames_scratch_bytes(int num_frames);
int sta_graph_track_frames(StaGraph* g, int num_frames, const int* anchors_host, const float* pose_dev,
                           const float* depth_dev, const float* conf_dev, float* meas_out, float* scale_edge_out,
                           unsigned char* valid_out, float* pose_out, float* scale_out, void* scratch,
                           size_t scratch_bytes, void* stream);
/* Recompose F stored frames (meas_dev [F][8] and scale_edge_dev [F] as sta_graph_track_frames wrote them) on their
 * anchors' current poses, in the same order: pose_out [F][4][4] (scale dropped), scale_out [F].  One launch, no host
 * synchronisation; refused as sta_graph_track_frames. */
int sta_graph_frame_poses(StaGraph* g, int num_frames, const int* anchors_host, const float* meas_dev,
                          const float* scale_edge_dev, float* pose_out, float* scale_out, void* stream);
/* Per view v in [view0, view0 + num_views), through its best node (every view must have one): pose_out [V][4][4] (rotation
 * and translation, scale dropped), scale_out [V], depth_out / conf_out [V][H][W] (unscaled), intri_out [V][3][3].
 * With points_out: the world point cloud of save_data_all -- depth s unprojected with K^-1, then R p + t, points with
 * conf > conf_thres in (view, row, column) order, colours (img + 1) / 2 from imgs_dev [V][3][H][W] -- into points_out /
 * colors_out [V H W][3] and *count_out (device int64).  scratch: sta_graph_export_scratch_bytes(V, H), 8-byte aligned.
 * One launch without the cloud, three with it (count, exclusive scan, scatter); no host synchronisation. */
size_t sta_graph_export_scratch_bytes(int num_views, int H);
int sta_graph_export(StaGraph* g, int view0, int num_views, float conf_thres, const float* imgs_dev, float* pose_out,
                     float* scale_out, float* depth_out, float* conf_out, float* intri_out, float* points_out,
                     float* colors_out, int64_t* count_out, void* scratch, void* stream);

/* ---- map rendering (OnlineSLAM.render, tools/render_video.py) ---- */
enum { STA_RENDER_MAX_RADIUS = 4 };
/* Render a map from C cameras into a z-buffer.  The map is sta_graph_export's output without the cloud: depth / conf
 * [V][H][W] (unscaled), pose44 [V][4][4] (scale dropped), scale [V], intri [V][3][3], and imgs [V][3][H][W] in [-1, 1].
 * Every pixel with conf > conf_thres becomes the PLY's world point (K^-1 from the fp64 adjugate, then
 * P (K^-1 [col row 1]^T depth s) in fp32); segs [L][2][3] are world-space line segments coloured seg_colors [L][3].
 * Cameras: w2c [C][4][4] world-to-camera, K [C][3][3].  A point with camera z >= near covers the (2 radius + 1)^2
 * pixels centred on floor(u / w + 0.5), floor(v / w + 0.5); a segment is clipped to z >= near and to the image and
 * drawn by DDA with perspective-correct z.  Each pixel keeps the smallest key (float bits of z << 32) | id, id =
 * v H W + row W + col for a point and V H W + l for segment l, so ties go to the lower id and the result does not depend
 * on scheduling.  Outputs per camera: rgb_out [C][Ho][Wo][3] ((img + 1) / 2, the segment's colour, or background, a
 * host float[3]), depth_out [C][Ho][Wo] (the winner's camera z, or 0), index_out [C][Ho][Wo] (its id, or -1).
 * scratch: sta_render_scratch_bytes(C, Ho, Wo), 8-byte aligned.  Four launches (clear, points, segments, resolve), no
 * host synchronisation.  Refused before any launch: C, Ho or Wo outside [1, 8192], radius outside
 * [0, STA_RENDER_MAX_RADIUS], near <= 0, V outside [0, 65535], V H W + L >= 2^32 - 1, a null input or output, a small
 * or misaligned scratch, host memory. */
size_t sta_render_scratch_bytes(int num_cams, int Ho, int Wo);
int sta_render(const float* depth, const float* conf, const float* pose44, const float* scale, const float* intri,
               const float* imgs, int V, int H, int W, float conf_thres, const float* w2c, const float* K, int C, int Ho,
               int Wo, int radius, float near, const float* segs, const float* seg_colors, int L, const float* background,
               void* scratch, size_t scratch_bytes, float* rgb_out, float* depth_out, int64_t* index_out, void* stream);

/* ---- TSDF fusion and meshing of the map (fusion.fuse_views, OnlineSLAM.extract_mesh) ---- */
enum { STA_FUSION_BRICK = 8, STA_FUSION_BRICK_BITS = 21, STA_FUSION_MAX_BRICKS = 1 << 20 };
/* The map is sta_render's (depth / conf [V][H][W] unscaled, pose44 [V][4][4], scale [V], intri [V][3][3], imgs
 * [V][3][H][W] in [-1, 1]).  Samples sit at (i v, j v, k v), each coordinate float(i) * v in fp32, in bricks of
 * STA_FUSION_BRICK^3; brick (bx, by, bz) = floor(i / 8) per axis, each in [-2^20, 2^20 - 1], has the 63-bit key
 * (bz + 2^20) << 42 | (by + 2^20) << 21 | (bx + 2^20).  A pixel is used when conf > conf_thres and d = depth scale > 0.
 *
 * sta_fusion_bricks: the sorted distinct keys of the bricks that the cube [p - trunc, p + trunc] of some used pixel's
 * PLY point p touches (floor((p -+ trunc) / 8v) per axis); a point with a non-finite coordinate or a brick outside
 * the range is skipped.  Two calls: with key_capacity 0 it writes counts_out[0] = the number of (tile, brick) keys
 * (an upper bound of the brick count); with key_capacity = that count it writes the keys to keys_out [key_capacity]
 * and counts_out[1] = the brick count B.  scratch: sta_fusion_bricks_scratch_bytes(V, H, W, key_capacity), 16-byte
 * aligned.  No host synchronisation.
 *
 * sta_fusion_integrate: KinectFusion's projective TSDF with unit weights of every view, in increasing index, into the
 * B bricks of keys: for sample x and view v, c = w2c[v] x (fp32); skipped unless c_z > 0, the pixel
 * (floor(u + 0.5), floor(r + 0.5)) of intri[v] c / c_z is inside the image and used, and sdf = d - c_z >= -trunc;
 * then T <- (T W + min(1, sdf / trunc)) / (W + 1), rgb alike with (img + 1) / 2, W <- W + 1.  Outputs tsdf_out,
 * weight_out [B][8][8][8] ([b][z][y][x]) and color_out [B][8][8][8][3]; unobserved samples are 0.  Views are culled
 * per brick conservatively, and there are no floating-point atomics, so the result is the same bit for bit on every
 * call.  scratch: sta_fusion_integrate_scratch_bytes(B, V), 16-byte aligned.
 *
 * sta_fusion_mesh: marching cubes (mc_table.h) over every cube whose 8 samples exist with weight >= min_weight; inside
 * is T < 0.  One vertex per crossing lattice edge used by an emitted face, at a + T_a / (T_a - T_b) (b - a) with its
 * colour interpolated alike, in (brick, sample, axis) order; faces in (brick, cube, triangle) order, counter-clockwise
 * seen from T > 0.  Two calls: with zero capacities it writes counts_out[0] = vertices, counts_out[1] = faces; with
 * capacities at least those it also writes vertices_out / vertex_colors_out [Nv][3] and faces_out [Nf][3].
 * scratch: sta_fusion_mesh_scratch_bytes(B), 16-byte aligned.
 *
 * Refused before any CUDA call: sizes outside [1, 65535], voxel <= 0 or not finite, trunc outside (0, 4 voxel],
 * min_weight < 1, B outside [0, STA_FUSION_MAX_BRICKS], a key capacity outside [0, 2^31), a null input or output, a
 * small or misaligned scratch, host memory. */
size_t sta_fusion_bricks_scratch_bytes(int V, int H, int W, int64_t key_capacity);
int sta_fusion_bricks(const float* depth, const float* conf, const float* pose44, const float* scale, const float* intri,
                      int V, int H, int W, float conf_thres, float voxel, float trunc, int64_t key_capacity,
                      void* scratch, size_t scratch_bytes, int64_t* keys_out, int64_t* counts_out, void* stream);
size_t sta_fusion_integrate_scratch_bytes(int64_t num_bricks, int V);
int sta_fusion_integrate(const float* depth, const float* conf, const float* scale, const float* intri, const float* imgs,
                         const float* w2c, int V, int H, int W, float conf_thres, const int64_t* keys, int64_t num_bricks,
                         float voxel, float trunc, void* scratch, size_t scratch_bytes, float* tsdf_out,
                         float* weight_out, float* color_out, void* stream);
size_t sta_fusion_mesh_scratch_bytes(int64_t num_bricks);
int sta_fusion_mesh(const int64_t* keys, int64_t num_bricks, const float* tsdf, const float* weight, const float* color,
                    float voxel, float min_weight, int64_t max_vertices, int64_t max_faces, void* scratch,
                    size_t scratch_bytes, float* vertices_out, float* vertex_colors_out, int32_t* faces_out,
                    int64_t* counts_out, void* stream);

/* ---- ray casting of the fused volume (fusion.raycast, OnlineSLAM.render_surface) ---- */
/* Ray-cast a volume exactly as sta_fusion_integrate returns it -- keys [B] (sorted, distinct), tsdf / weight
 * [B][8][8][8] ([b][z][y][x]) and color [B][8][8][8][3], samples at (float(i) v, float(j) v, float(k) v) -- from C
 * cameras: c2w [C][4][4] camera-to-world, K [C][3][3] (fx = K[0], cx = K[2], fy = K[4], cy = K[5]).  Pixel (col, row)
 * is the ray o + z R ((col - cx) / fx, (row - cy) / fy, 1), z the camera depth.  A point lies in cell floor(p / v);
 * a cell is valid when its 8 corner samples exist with weight >= min_weight (sta_fusion_mesh's rule), and there the
 * field and colour are the trilinear interpolants.  The march covers the ray's overlap with the bricks' bounding box
 * (computed on the device) from z >= near, in steps of half a voxel of world length, and jumps over absent bricks.
 * The hit is the first pair of consecutive valid samples with T > 0 then T <= 0 (surfaces seen from behind are passed
 * through), refined by 16 bisection steps and a final secant.  Outputs per pixel: depth_out [C][Ho][Wo] (the hit's z, 0 on
 * a miss), normal_out [C][Ho][Wo][3] (normalised gradient of the interpolant, world frame, 0 on a miss), color_out
 * [C][Ho][Wo][3] (the interpolated colour) and rgb_out [C][Ho][Wo][3] (color (0.3 + 0.7 max(0, -n . r)), r the unit ray
 * direction), both background (a host float[3]) on a miss.  One thread per pixel, no atomics in the march: the same
 * bits on every call and for a camera alone or among others.  scratch: sta_raycast_scratch_bytes(B), 16-byte aligned.
 * Two launches (the box, the march), no host synchronisation.  Refused before any launch: C, Ho or Wo outside
 * [1, 8192], B outside [0, STA_FUSION_MAX_BRICKS], voxel <= 0 or not finite, min_weight < 1, near <= 0 or not finite,
 * a null input or output, a small or misaligned scratch, host memory. */
size_t sta_raycast_scratch_bytes(int64_t num_bricks);
int sta_raycast(const int64_t* keys, int64_t num_bricks, const float* tsdf, const float* weight, const float* color,
                float voxel, float min_weight, const float* c2w, const float* K, int C, int Ho, int Wo, float near,
                const float* background, void* scratch, size_t scratch_bytes, float* rgb_out, float* color_out,
                float* depth_out, float* normal_out, void* stream);

/* ---- multi-view depth consistency of the map (slam_utils.view_consistency_check, OnlineSLAM.view_consistency) ---- */
/* vista_slam/utils/slam_utils.py:346-419 for n views: depth [n][H][W], intri [n][3][3], pose44 [n][4][4]
 * camera-to-world, all fp32.  count_out [n][H][W] (device int32): for pixel (x, y) of view i, the number of views j in
 * [max(0, i - 4), min(n - 1, i + 4)], j != i, for which |sample - z| < threshold and z > 0, where p = T_i (K_i^-1
 * [x y 1]^T d_i), c = T_j^-1 p, z = max(c_z, 1e-6), (u, v) = (K_j c)_xy / (K_j c)_z with the unclamped c, and sample is
 * depth j bilinearly at (u, v) with zero padding (grid_sample, align_corners=True).  A non-finite coordinate never
 * agrees; a finite one outside the image samples 0.  One launch, no atomics (the same bits on every call), no host
 * synchronisation.  Refused before any launch: n outside [1, 65535], H or W < 2, n H W >= 2^31, a non-finite threshold,
 * a null pointer, host memory. */
int sta_view_consistency(const float* depth, const float* intri, const float* pose44, int n, int H, int W,
                         float threshold, int32_t* count_out, void* stream);

/* ---- reconstruction evaluation (vista_slam/eval/eval_recon.py:108-206): world clouds, open3d's voxel_down_sample, the
 * moments of open3d's point-to-point ICP and the nearest-neighbour distances of the Chamfer metric.  Points are fp64
 * [n][3] device arrays.  Every reduction runs in a fixed order without floating-point atomics, so repeated runs are
 * bit-identical.  Host pointers are refused before any launch. ---- */

/* Stable LSD radix sort of (key, index) pairs by the low nbits (0..64) of the keys, 8 bits per pass; idx null means
 * 0 .. n-1.  The outputs may be the inputs.  n < 2^31.  scratch: sta_sort_scratch_bytes(n), 16-byte aligned. */
size_t sta_sort_scratch_bytes(int64_t n);
int sta_op_radix_sort(const uint64_t* keys, const uint32_t* idx, int64_t n, int nbits, uint64_t* keys_out, uint32_t* idx_out,
                      void* scratch, void* stream);
/* Both clouds of eval_recon in numpy boolean-indexing order (view, row, column):
 *   ground truth  gt_depth > 0, unprojected with the shared gt_intri [3][3] and moved by gt_pose [N][4][4];
 *   estimate      conf > thres and gt_depth > 0, depth (times scale[v] when scale [N] is given) unprojected with
 *                 intri [N][3][3] and moved by pose [N][4][4].
 * All inputs fp32; K^-1 from the fp64 adjugate, the rest in fp32; the points are written as fp64 into gt_out / est_out
 * (room for N H W points each), the two counts into count_out [2] (device int64).  scratch:
 * sta_eval_clouds_scratch_bytes(N, H), 8-byte aligned.  No host synchronisation. */
size_t sta_eval_clouds_scratch_bytes(int N, int H);
int sta_eval_clouds(int N, int H, int W, const float* gt_depth, const float* gt_pose, const float* gt_intri, const float* depth,
                    const float* scale, const float* pose, const float* intri, const float* conf, float thres, double* gt_out,
                    double* est_out, int64_t* count_out, void* scratch, void* stream);
/* open3d voxel_down_sample: min_bound = min - v/2, key = floor((p - min_bound) / v) per axis in fp64, each voxel's
 * point = the fp64 sum of its points in input order / their count, in ascending (kx, ky, kz) order.  out: room for n
 * points; *count_host: the number written.  Refused: v <= 0, and v * INT_MAX < the padded extent (open3d's condition).
 * Synchronises twice: to read the cloud's box (key widths, refusal) and the voxel count.  scratch:
 * sta_voxel_scratch_bytes(n), 16-byte aligned. */
size_t sta_voxel_scratch_bytes(int64_t n);
int sta_voxel_down(const double* pts, int64_t n, double voxel, double* out, int64_t* count_host, void* scratch, void* stream);
/* Nearest-neighbour index over one cloud (n may be 0): the points sorted by a 63-bit Morton code, leaves of 32 points
 * under a complete binary tree of fp64 boxes.  The index copies what it needs; create synchronises the stream. */
typedef struct StaNnIndex StaNnIndex; /* opaque */
int sta_nn_create(const double* pts, int64_t n, StaNnIndex** out, void* stream);
void sta_nn_destroy(StaNnIndex* ix);
/* Per query: the nearest indexed point strictly within radius (d^2 < r^2, d^2 = (dx dx + dy dy) + dz dz with every
 * operation rounded on its own).  dist_out [nq]: its distance, or radius when there is none; idx_out [nq]: its input
 * index, or -1.  Exact whatever the tree's shape.  scratch: sta_nn_query_scratch_bytes(nq), 16-byte aligned. */
size_t sta_nn_query_scratch_bytes(int64_t nq);
int sta_nn_query(const StaNnIndex* ix, const double* q, int64_t nq, double radius, double* dist_out, int64_t* idx_out,
                 void* scratch, void* stream);
/* Moments of one point-to-point ICP step over corr [n] (index into dst, -1 = none), into out17 (device):
 * [0] count, [1] sum d^2, [2..4] sum src, [5..7] sum dst, [8..16] the centred cross-covariance sum
 * sum (dst - mean_dst)(src - mean_src)^T, row-major (means from the first pass: two passes, not raw moments).
 * scratch: sta_reduce_scratch_bytes(). */
size_t sta_reduce_scratch_bytes(void);
int sta_op_moments(const double* src, const double* dst, const int64_t* corr, int64_t n, double* out17, void* scratch,
                   void* stream);
/* sta_nn_query of the source points in the target's index (target_pts: the cloud the index was built from), then
 * sta_op_moments.  scratch: sta_icp_scratch_bytes(n), 16-byte aligned. */
size_t sta_icp_scratch_bytes(int64_t n);
int sta_icp_moments(const StaNnIndex* target, const double* target_pts, const double* src, int64_t n, double radius,
                    double* out17, void* scratch, void* stream);
/* In place: p <- M[:, :3] p + M[:, 3] with M the row-major 3x4 m12_host, fp64 without FMA contraction. */
int sta_transform_points(double* pts, int64_t n, const double* m12_host, void* stream);
/* *out_dev = sum of min(max(d, 0), clip)^2 over n values.  scratch: sta_reduce_scratch_bytes(). */
int sta_sum_sq_clipped(const double* d, int64_t n, double clip, double* out_dev, void* scratch, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* STA_B200_H_ */
