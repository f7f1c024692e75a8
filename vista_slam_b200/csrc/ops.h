// Internal C++ launch API shared by the model runtime and the op-level C-ABI
// test entry points (both in runtime.cu).  All functions return 0 on success and set
// sta::get_last_error() otherwise; all work is enqueued on `stream`.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include "gemm.cuh"

namespace sta {

typedef __nv_bfloat16 bf16;

struct GemmLaunch {
  int amode = A_LINEAR;
  int epi = EPI_BF16;
  // A operand.  A_LINEAR: [M][lda] bf16 (K contiguous).  A_CONV3: NHWC [nimg][H][W][Cin] bf16.  A_FP8: [M][lda] e4m3.
  const void* A = nullptr;
  long long lda = 0;
  // weights: [N][ldw] bf16 (A_FP8: e4m3), K contiguous (K = 9*Cin ordered (kh, kw, cin) for A_CONV3)
  const void* Wt = nullptr;
  long long ldw = 0;
  GemmParams p = {};
  // optional fp32 scratch for split-K partials (small, weight-streaming-bound problems); unused if null
  void* splitk_ws = nullptr;
  size_t splitk_ws_bytes = 0;
  // tile columns: 0 = automatic (gemm_auto_tile_n), 128 = the 128 x 128 kernel, 256 = the 128 x 256 kernel (error where
  // it does not apply).  Both give bit-identical results.
  int tile_n = 0;
};

int launch_gemm(const GemmLaunch& g, cudaStream_t stream);
// Tile columns the automatic choice takes for a linear layer (M x N, depth K) with epilogue epi that runs the TMA-store
// epilogue without split-K on a GPU with num_sms SMs: 256 or 128.  A function of these arguments only.
int gemm_auto_tile_n(int M, int N, int K, int epi, int num_sms);

// ---- attention (attention.cu) ----
struct AttnLaunch {
  // q rows: [batch][nq][ldq] bf16, head h at columns q_col0 + 64*h
  const bf16* q = nullptr; long long ldq = 0; int q_col0 = 0;
  const bf16* k = nullptr; long long ldk = 0; int k_col0 = 0;
  const bf16* v = nullptr; long long ldv = 0; int v_col0 = 0;
  bf16* out = nullptr; long long ldo = 0;   // [batch][nq][ldo], head h at columns 64*h
  int batch = 0, heads = 0, nq = 0, nk = 0;
  int kv_batch_shift = 0;   // k/v sample for query sample b is (b + shift) % batch  (cross-view attention)
  float scale = 0.125f;
  // split-precision parity mode (common.cuh): q/k/v/out rows are (hi | lo | hi) with ld* the physical (3x) strides;
  // an fp32 SIMT kernel with exact exp2f computes softmax(q k^T) v from hi + lo and stores (hi | lo | hi).
  int split = 0;
};
int launch_attention(const AttnLaunch& a, cudaStream_t stream);

// ---- bandwidth-bound kernels (kernels.cu) ----
int launch_layernorm(const float* x, int rows, int C, float eps, const float* g1, const float* b1, bf16* out1,
                     const float* g2, const float* b2, bf16* out2, int drop_first_of, cudaStream_t stream, int split = 0);
// FP8 mode: e4m3 rows plus one power-of-two scale per row and 128 columns (common.cuh fp8_scale)
int launch_layernorm_fp8(const float* x, int rows, int C, float eps, const float* g1, const float* b1, uint8_t* q1, float* s1,
                         const float* g2, const float* b2, uint8_t* q2, float* s2, cudaStream_t stream);
int launch_quant_fp8(const bf16* in, long long rows, int C, uint8_t* q, float* s, cudaStream_t stream);
int launch_patch_im2col(const void* img, int img_is_bf16, int B, int H, int W, bf16* out, cudaStream_t stream, int split = 0);
int launch_make_positions(int* pos, int B, int h, int w, int with_pose_token, cudaStream_t stream);
int launch_pos_from_int64(const long long* pos64, int rows, int* pos32, cudaStream_t stream);
int launch_cast_f32_bf16(const float* in, bf16* out, long long rows, int C, int drop_first_of, cudaStream_t stream,
                         int split = 0);
int launch_fill_pose_token(float* x, const float* tok, int samples, int tokens_per_sample, int C,
                           cudaStream_t stream);
int launch_upsample2x(const bf16* in, bf16* out, int nimg, int H, int W, int C, int OH, int OW, cudaStream_t stream,
                      int split = 0);
// preprocess.cu: SLAM_image_only.process_image on the device (PIL-exact Lanczos resize + ToTensor/Normalize/Grayscale),
// F same-size frames per launch pair
int launch_preprocess_rgb8(const uint8_t* rgb_dev, int F, int H, int W, int res_w, int res_h, int w_edge, int h_edge,
                           float* rgb_out, float* gray_out, uint8_t* u8_out, int* out_hw_host, int query_only,
                           cudaStream_t stream);
int preprocess_geometry(int H, int W, int res_w, int res_h, int w_edge, int h_edge, int* out10);
int preprocess_coeffs(int in_size, int out_size, int* ksize_out, int* bounds_out, int* kk_out, long long kk_capacity);
// pointmap.cu: reductions over the head outputs (slam_utils.py:8-79,168-190)
size_t pointmap_scratch_bytes(int V);
int launch_pointmap_consumers(const float* pts3d, const float* conf, int V, int H, int W, int shared, float* K_out,
                              float* depth_out, float* conf_mean_out, void* scratch, cudaStream_t stream);
int launch_depth_scale(const float* Di, const float* Dj, const float* ci, const float* cj, long long n, float* out2,
                       void* scratch, cudaStream_t stream);
// pose_graph.cu: one Sim(3) pose-graph LM step (pose_graph.py:70-154, slam.py:108-140)
size_t pose_graph_scratch_bytes(int num_nodes, int num_edges, int num_opt);
int launch_pose_graph_lm_step(const float* nodes, int num_nodes, const long long* edges, const float* meas, const float* weights,
                              int num_edges, const long long* opt_idx, int num_opt, double damping, double dmin, double dmax,
                              float* nodes_out, double* info_out, void* scratch, cudaStream_t stream);
int launch_im2col_3x3_s2(const bf16* in, bf16* out, int nimg, int H, int W, int C, cudaStream_t stream);
int launch_copy_f32(const float* in, float* out, long long n, cudaStream_t stream);

struct PoseHeadWeights {
  const float *ln_g, *ln_b;  // dec_norm
  const float *w0, *b0, *w1, *b1, *w2, *b2;
  const float *wt, *bt, *wr, *br, *wc, *bc;
};
// x: fp32 rows; pose-token row of sample s is x[s * sample_stride .. +768); apply_ln = LayerNorm(dec_norm) first
int launch_pose_head(const float* x, long long sample_stride, int samples, int apply_ln, float eps,
                     const PoseHeadWeights& w, float* pose44, float* conf, cudaStream_t stream);

const float* rope_table(int* max_pos);  // device table [(pos+1)][16][2], pos in [-1, max_pos]

}  // namespace sta
