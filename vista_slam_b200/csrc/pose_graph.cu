// Sim(3) pose-graph Levenberg-Marquardt step on the GPU (SURVEY.md section 8(f) rank 4).
//
// Replaces, for one LM iteration of OnlineSLAM.pose_graph_optimize (vista_slam/slam.py:108-140):
//   * PoseGraphOpt.forward (vista_slam/pose_graph.py:100-149): r_e = Log(T_e X_i^-1 X_j) in R^7 for every edge with at
//     least one optimised endpoint (get_related_edge_idxs, :150-154), optimised / fixed node split (:73-98);
//   * the autograd Jacobian PyPose builds for it (left perturbation X <- Exp(delta) X, LieTensor.add_):
//     dr/d delta_j = J_l^-1(r) Ad_{T_e X_i^-1},  dr/d delta_i = -dr/d delta_j;
//   * pp.optim.LM.step: A = J^T W J (W = diag(conf_e), 7 per edge), diagonal clamped to [min, max] and scaled by
//     (1 + damping), dense Cholesky solve of A d = -J^T W r (the reference's solver is a dense torch Cholesky),
//     X <- Exp(d) X, loss = r^T W r before and after.
// Everything is fp64 inside (node / measurement tensors are fp32 like the reference's), deterministic (no atomics: every
// output element has one owner thread and a fixed summation order), and there is no host synchronisation: the caller reads
// the two losses to accept / reject the step, exactly where pp.optim.LM does.
//
// Kernels: pg_edge_kernel (one thread per edge: group algebra in closed form, J_l via phi_1(ad) by scaling-and-squaring,
// 7x7 Gauss-Jordan), pg_assemble_kernel (one CTA per optimised node: its block row of A and of g), pg_damp_kernel,
// blocked right-looking Cholesky (diag / trsm / syrk kernels, 32-wide panels), pg_solve_kernel (forward + backward
// substitution, one CTA), pg_update_kernel, pg_loss_kernel.  The problem is small (<= a few thousand edges, A of order
// 7 * optimised nodes): this is latency-bound work; the design goal is zero host round trips and determinism.
// pg_edge_kernel, pg_update_kernel, pg_loss_kernel and the Sim(3) algebra live in pose_graph.cuh, shared with the
// block-sparse route (pose_graph_sparse.cu) that PoseGraphOpt takes above STA_PG_DENSE_MAX_OPT optimised nodes.
//
// Groups: one launch sequence steps G >= 2 independent graphs (sta_pose_graph_lm_step_group; a group of one runs the
// one-graph sequence, which stays the faster one for a single graph, by 1-2 % at 500-3600 optimised nodes).  Kernel
// bodies are device functions shared by the one-graph and the group kernels.  Every kernel takes the group's descriptor table and finds its graph from a grid dimension (the last one
// it uses); blocks past their graph's node, edge, order or tile count return at once, and the panel loop runs to the
// largest order.  A graph's blocks do the arithmetic of a one-graph launch in the same order -- no reduction crosses
// graphs -- so each graph's result is independent of the group around it, bit for bit.  The descriptors (pointers, sizes,
// damping and the graph's scratch carve) travel as ONE kernel-parameter struct of at most PG_GROUP_MAX entries to
// pg_group_setup_kernel, which stores them at the head of the scratch for the kernels after it: replacing them every
// iteration costs no host synchronisation and no host-to-device copy, and those launches keep small parameters.  The
// Cholesky panel kernels, launched three times per 32 columns, take their graph's A, info and order as a kernel
// parameter of their own (PgPanels) instead.
#include <math.h>

#include <algorithm>

#include "../../include/sta_b200.h"
#include "common.cuh"
#include "host_util.h"
#include "ops.h"
#include "pose_graph.cuh"

namespace sta {

namespace {

constexpr int PG_GROUP_MAX = STA_PG_GROUP_MAX;
constexpr int PG_SOLVE_SMEM_MAX = 200 * 1024;  // the one-CTA solve keeps the 7 num_opt right-hand side in shared memory

struct PgScratch {
  double *r, *J, *A, *g, *delta, *r2, *info;
  int *related, *opt_map;
};

// one graph of a group: its inputs, outputs, damping and scratch carve
struct PgDesc {
  const float* nodes;
  const long long* edges;
  const float* meas;
  const float* weights;
  const long long* opt_idx;
  float* nodes_out;
  double* info_out;
  PgScratch s;
  int num_nodes, num_edges, num_opt, n7;
  double damping;
};
struct PgGroupParams {
  PgDesc g[PG_GROUP_MAX];
};
static_assert(sizeof(PgGroupParams) + 16 <= 4096, "the group descriptors must fit the kernel-parameter space");
// what the Cholesky panel kernels and the solve read per graph, passed to them by value (576 bytes): a syrk step runs up
// to hundreds of thousands of blocks, and reading A and the order from the constant bank spares each one a dependent
// global load
struct PgPanels {
  double* A[PG_GROUP_MAX];
  double* info[PG_GROUP_MAX];
  double* g[PG_GROUP_MAX];
  double* delta[PG_GROUP_MAX];
  int n[PG_GROUP_MAX];
};

// the descriptors into the scratch head, and each graph's Cholesky-ok flag (info[3]) set
__global__ void pg_group_setup_kernel(const __grid_constant__ PgGroupParams p, int G, PgDesc* __restrict__ descs) {
  const int k = threadIdx.x;
  if (k >= G) return;
  descs[k] = p.g[k];
  p.g[k].s.info[3] = 1.0;
}

// A = 0 (order n7, row-major), grid (x, graph)
__global__ void __launch_bounds__(256) pg_zero_kernel(const PgDesc* __restrict__ gd) {
  const PgDesc& d = gd[blockIdx.y];
  const long long n = static_cast<long long>(d.n7) * d.n7;
  double* A = d.s.A;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) A[i] = 0.0;
}

// phase 0 marks every node fixed, phase 1 numbers the optimised ones (pose_graph.py:90-91)
__device__ __forceinline__ void pg_opt_map(int i, const long long* __restrict__ opt_idx, int num_opt, int num_nodes,
                                           int* __restrict__ opt_map, int phase) {
  if (phase == 0) {
    if (i < num_nodes) opt_map[i] = -1;
  } else if (i < num_opt) {
    const long long v = opt_idx[i];
    if (v >= 0 && v < num_nodes) opt_map[v] = i;
  }
}
__global__ void pg_opt_map_kernel(const long long* __restrict__ opt_idx, int num_opt, int num_nodes, int* __restrict__ opt_map,
                                  int phase) {
  pg_opt_map(blockIdx.x * blockDim.x + threadIdx.x, opt_idx, num_opt, num_nodes, opt_map, phase);
}
// grid (x, graph)
__global__ void pg_opt_map_group_kernel(const PgDesc* __restrict__ gd, int phase) {
  const PgDesc& d = gd[blockIdx.y];
  pg_opt_map(blockIdx.x * blockDim.x + threadIdx.x, d.opt_idx, d.num_opt, d.num_nodes, d.s.opt_map, phase);
}

// grid (x, graph): residuals and Jacobians at the nodes (second = 0), or residuals alone at the candidate (second = 1)
__global__ void __launch_bounds__(64) pg_edge_group_kernel(const PgDesc* __restrict__ gd, int second) {
  const PgDesc& d = gd[blockIdx.y];
  pg_edge(blockIdx.x * blockDim.x + threadIdx.x, second ? d.nodes_out : d.nodes, d.edges, d.meas, d.s.opt_map, d.num_edges,
          second ? d.s.r2 : d.s.r, second ? nullptr : d.s.J, d.s.related);
}

// ---------------------------------------------------------------------------
// one CTA per optimised node a: block row a of A = J^T W J and of g = J^T W r.  64 threads: thread (p, q) = entry of
// the 7x7 blocks (49), threads 49..55 = the 7 entries of g.  Edges are visited in index order: fixed summation order.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void pg_assemble(int a, const long long* __restrict__ edges, const float* __restrict__ weights,
                                            const int* __restrict__ opt_map, const int* __restrict__ related,
                                            const double* __restrict__ r, const double* __restrict__ J, int E, int n7,
                                            double* __restrict__ A, double* __restrict__ g) {
  const int t = threadIdx.x;
  const int p = t / 7, q = t - 7 * p;
  double diag = 0.0, gv = 0.0;
  for (int e = 0; e < E; ++e) {
    if (!related[e]) continue;
    const int oi = opt_map[edges[2 * e]], oj = opt_map[edges[2 * e + 1]];
    if (oi != a && oj != a) continue;
    const double* Je = J + 49ll * e;
    const float* w = weights + 7 * e;
    for (int side = 0; side < 2; ++side) {  // side 0: a is the first endpoint (J_a = -J), side 1: the second (J_a = +J)
      if ((side == 0 ? oi : oj) != a) continue;
      const int b = side == 0 ? oj : oi;
      if (t < 49) {
        double s = 0.0;
        for (int k = 0; k < 7; ++k) s = fma(Je[7 * k + p] * static_cast<double>(w[k]), Je[7 * k + q], s);
        diag += s;                                             // J_a^T W J_a
        if (b >= 0) A[(7ll * a + p) * n7 + 7 * b + q] -= s;     // J_a^T W J_b with J_b = -J_a (single owner thread)
      } else if (t < 56) {
        const int pp = t - 49;
        double s = 0.0;
        for (int k = 0; k < 7; ++k) s = fma(Je[7 * k + pp] * static_cast<double>(w[k]), r[7ll * e + k], s);
        gv += side == 0 ? -s : s;
      }
    }
  }
  if (t < 49) A[(7ll * a + p) * n7 + 7 * a + q] += diag;
  else if (t < 56) g[7 * a + (t - 49)] = gv;
}
__global__ void __launch_bounds__(64)
pg_assemble_kernel(const long long* __restrict__ edges, const float* __restrict__ weights, const int* __restrict__ opt_map,
                   const int* __restrict__ related, const double* __restrict__ r, const double* __restrict__ J, int E, int n7,
                   double* __restrict__ A, double* __restrict__ g) {
  pg_assemble(blockIdx.x, edges, weights, opt_map, related, r, J, E, n7, A, g);
}
// grid (optimised node, graph)
__global__ void __launch_bounds__(64) pg_assemble_group_kernel(const PgDesc* __restrict__ gd) {
  const PgDesc& d = gd[blockIdx.y];
  if (static_cast<int>(blockIdx.x) >= d.num_opt) return;
  pg_assemble(blockIdx.x, d.edges, d.weights, d.s.opt_map, d.s.related, d.s.r, d.s.J, d.num_edges, d.n7, d.s.A, d.s.g);
}

// grid (graph): loss before (second = 0), or loss after and |delta| (second = 1), then the graph's info row out
__global__ void __launch_bounds__(256) pg_loss_group_kernel(const PgDesc* __restrict__ gd, int second) {
  const PgDesc& d = gd[blockIdx.x];
  if (!second) {
    pg_loss(d.s.r, d.weights, d.s.related, d.num_edges, nullptr, 0, d.s.info, 0);
    return;
  }
  pg_loss(d.s.r2, d.weights, d.s.related, d.num_edges, d.s.delta, d.n7, d.s.info, 1);
  if (threadIdx.x == 0)  // info[1], info[2] are this thread's own writes; info[0] and info[3] come from earlier launches
    for (int k = 0; k < 4; ++k) d.info_out[k] = d.s.info[k];
}

// LM damping of pp.optim.LM.step: A.diagonal().clamp_(min, max); A.diagonal() += damping * A.diagonal()
__device__ __forceinline__ void pg_damp(int i, double* A, int n7, double dmin, double dmax, double damping) {
  if (i >= n7) return;
  double d = A[static_cast<long long>(i) * n7 + i];
  d = fmin(fmax(d, dmin), dmax);
  A[static_cast<long long>(i) * n7 + i] = d * (1.0 + damping);
}
__global__ void pg_damp_kernel(double* A, int n7, double dmin, double dmax, double damping) {
  pg_damp(blockIdx.x * blockDim.x + threadIdx.x, A, n7, dmin, dmax, damping);
}
// grid (x, graph)
__global__ void pg_damp_group_kernel(const PgDesc* __restrict__ gd, double dmin, double dmax) {
  const PgDesc& d = gd[blockIdx.y];
  pg_damp(blockIdx.x * blockDim.x + threadIdx.x, d.s.A, d.n7, dmin, dmax, d.damping);
}

// ---------------------------------------------------------------------------
// dense blocked right-looking Cholesky (lower), fp64, 32-wide panels.  info[3] is set to 0 on a non-positive pivot.
// Panel k0 of a graph of order n exists while k0 < n; its trsm / syrk tiles while rows remain below it.
// ---------------------------------------------------------------------------
constexpr int NB = 32;
__device__ __forceinline__ int pg_tiles_below(int n, int k0) {  // row tiles below panel k0 (0: no trsm / syrk)
  const int rest = n - k0 - NB;
  return rest > 0 ? (rest + NB - 1) / NB : 0;
}
__device__ __forceinline__ void chol_diag(double* A, int n, int k0, double* info) {
  __shared__ double S[NB][NB + 1];
  const int nb = min(NB, n - k0);
  const int r = threadIdx.y, c = threadIdx.x;
  if (r < nb && c < nb) S[r][c] = A[static_cast<long long>(k0 + r) * n + k0 + c];
  __syncthreads();
  for (int k = 0; k < nb; ++k) {
    if (r == k && c == k) {
      const double d = S[k][k];
      if (!(d > 0.0)) { info[3] = 0.0; S[k][k] = 1.0; } else S[k][k] = sqrt(d);
    }
    __syncthreads();
    if (c == k && r > k && r < nb) S[r][k] /= S[k][k];
    __syncthreads();
    if (r > k && r < nb && c > k && c <= r) S[r][c] -= S[r][k] * S[c][k];
    __syncthreads();
  }
  if (r < nb && c < nb && c <= r) A[static_cast<long long>(k0 + r) * n + k0 + c] = S[r][c];
}
// rows below the panel: X L_kk^T = A_ik  (one thread per row; row tile blockIdx.x)
__device__ __forceinline__ void chol_trsm(double* A, int n, int k0) {
  __shared__ double L[NB][NB + 1];
  const int nb = min(NB, n - k0);
  for (int idx = threadIdx.x; idx < NB * NB; idx += NB) {
    const int r = idx / NB, c = idx % NB;
    L[r][c] = (r < nb && c <= r) ? A[static_cast<long long>(k0 + r) * n + k0 + c] : 0.0;
  }
  __syncthreads();
  const int row = k0 + nb + blockIdx.x * NB + threadIdx.x;
  if (row >= n) return;
  double x[NB];
  double* ar = A + static_cast<long long>(row) * n + k0;
  for (int c = 0; c < nb; ++c) x[c] = ar[c];
  for (int c = 0; c < nb; ++c) {
    double s = x[c];
    for (int cc = 0; cc < c; ++cc) s -= x[cc] * L[c][cc];
    x[c] = s / L[c][c];
  }
  for (int c = 0; c < nb; ++c) ar[c] = x[c];
}
// trailing update: A_ij -= L_ik L_jk^T for tiles j <= i below / right of the panel (tiles (blockIdx.x, blockIdx.y))
__device__ __forceinline__ void chol_syrk(double* A, int n, int k0) {
  __shared__ double Li[NB][NB + 1], Lj[NB][NB + 1];
  const int nb = min(NB, n - k0);
  const int base = k0 + nb;
  const int i = base + blockIdx.y * NB + threadIdx.y, j = base + blockIdx.x * NB + threadIdx.x;
  const int li = base + blockIdx.y * NB + threadIdx.y, lj = base + blockIdx.x * NB + threadIdx.y;
  Li[threadIdx.y][threadIdx.x] = (li < n && threadIdx.x < nb) ? A[static_cast<long long>(li) * n + k0 + threadIdx.x] : 0.0;
  Lj[threadIdx.y][threadIdx.x] = (lj < n && threadIdx.x < nb) ? A[static_cast<long long>(lj) * n + k0 + threadIdx.x] : 0.0;
  __syncthreads();
  if (i >= n || j >= n || j > i) return;
  double s = 0.0;
  for (int c = 0; c < NB; ++c) s = fma(Li[threadIdx.y][c], Lj[threadIdx.x][c], s);
  A[static_cast<long long>(i) * n + j] -= s;
}
__global__ void __launch_bounds__(NB * NB) chol_diag_kernel(double* A, int n, int k0, double* info) {
  chol_diag(A, n, k0, info);
}
__global__ void __launch_bounds__(NB) chol_trsm_kernel(double* A, int n, int k0) { chol_trsm(A, n, k0); }
__global__ void __launch_bounds__(NB * NB) chol_syrk_kernel(double* A, int n, int k0) {
  if (blockIdx.x > blockIdx.y) return;  // (bj, bi) with bj <= bi
  chol_syrk(A, n, k0);
}
// group forms: grid (graph), (row tile, graph), (col tile, row tile, graph)
__global__ void __launch_bounds__(NB * NB) chol_diag_group_kernel(const __grid_constant__ PgPanels P, int k0) {
  const int n = P.n[blockIdx.x];
  if (k0 >= n) return;
  chol_diag(P.A[blockIdx.x], n, k0, P.info[blockIdx.x]);
}
__global__ void __launch_bounds__(NB) chol_trsm_group_kernel(const __grid_constant__ PgPanels P, int k0) {
  const int n = P.n[blockIdx.y];
  if (static_cast<int>(blockIdx.x) >= pg_tiles_below(n, k0)) return;
  chol_trsm(P.A[blockIdx.y], n, k0);
}
__global__ void __launch_bounds__(NB * NB) chol_syrk_group_kernel(const __grid_constant__ PgPanels P, int k0) {
  if (blockIdx.x > blockIdx.y) return;
  const int n = P.n[blockIdx.z];
  if (static_cast<int>(blockIdx.y) >= pg_tiles_below(n, k0)) return;
  chol_syrk(P.A[blockIdx.z], n, k0);
}
// x = -(L L^T)^-1 g, one CTA per graph: blocked forward then backward substitution with the right-hand side in shared
// memory (sized for the group's largest order)
__device__ __forceinline__ void pg_solve(const double* __restrict__ A, const double* __restrict__ g, int n,
                                         double* __restrict__ x) {
  extern __shared__ double b[];
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int i = tid; i < n; i += nt) b[i] = -g[i];
  __syncthreads();
  for (int k0 = 0; k0 < n; k0 += NB) {  // L y = b
    const int nb = min(NB, n - k0);
    if (tid == 0) {
      for (int c = 0; c < nb; ++c) {
        double s = b[k0 + c];
        const double* lr = A + static_cast<long long>(k0 + c) * n + k0;
        for (int cc = 0; cc < c; ++cc) s -= lr[cc] * b[k0 + cc];
        b[k0 + c] = s / lr[c];
      }
    }
    __syncthreads();
    for (int i = k0 + nb + tid; i < n; i += nt) {
      const double* lr = A + static_cast<long long>(i) * n + k0;
      double s = b[i];
      for (int c = 0; c < nb; ++c) s -= lr[c] * b[k0 + c];
      b[i] = s;
    }
    __syncthreads();
  }
  const int nblk = (n + NB - 1) / NB;
  for (int kb = nblk - 1; kb >= 0; --kb) {  // L^T x = y
    const int k0 = kb * NB, nb = min(NB, n - k0);
    if (tid == 0) {
      for (int c = nb - 1; c >= 0; --c) {
        double s = b[k0 + c];
        for (int cc = c + 1; cc < nb; ++cc) s -= A[static_cast<long long>(k0 + cc) * n + k0 + c] * b[k0 + cc];
        b[k0 + c] = s / A[static_cast<long long>(k0 + c) * n + k0 + c];
      }
    }
    __syncthreads();
    for (int i = tid; i < k0; i += nt) {  // b_i -= sum_c L[k0 + c][i] x[k0 + c]
      double s = b[i];
      for (int c = 0; c < nb; ++c) s -= A[static_cast<long long>(k0 + c) * n + i] * b[k0 + c];
      b[i] = s;
    }
    __syncthreads();
  }
  for (int i = tid; i < n; i += nt) x[i] = b[i];
}
// grid (graph)
__global__ void __launch_bounds__(1024) pg_solve_group_kernel(const __grid_constant__ PgPanels P) {
  pg_solve(P.A[blockIdx.x], P.g[blockIdx.x], P.n[blockIdx.x], P.delta[blockIdx.x]);
}
__global__ void __launch_bounds__(1024) pg_solve_kernel(const double* __restrict__ A, const double* __restrict__ g, int n,
                                                        double* __restrict__ x) {
  pg_solve(A, g, n, x);
}

// grid (x, graph): nodes_out = Exp(delta_a) node for the optimised nodes, copies of the fixed ones
__global__ void pg_update_group_kernel(const PgDesc* __restrict__ gd) {
  const PgDesc& d = gd[blockIdx.y];
  pg_update(blockIdx.x * blockDim.x + threadIdx.x, d.nodes, d.s.opt_map, d.s.delta, d.num_nodes, d.nodes_out);
}

size_t carve(char* base, int Nn, int E, int n_opt, PgScratch* s) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    off = (off + 255) & ~static_cast<size_t>(255);
    char* p = base ? base + off : nullptr;
    off += bytes;
    return p;
  };
  const size_t n7 = 7ull * n_opt;
  char* r = take(7ull * E * 8);
  char* J = take(49ull * E * 8);
  char* A = take(n7 * n7 * 8);
  char* g = take(n7 * 8);
  char* d = take(n7 * 8);
  char* r2 = take(7ull * E * 8);
  char* info = take(4 * 8);
  char* rel = take(4ull * E);
  char* om = take(4ull * Nn);
  if (s) {
    s->r = reinterpret_cast<double*>(r); s->J = reinterpret_cast<double*>(J); s->A = reinterpret_cast<double*>(A);
    s->g = reinterpret_cast<double*>(g); s->delta = reinterpret_cast<double*>(d); s->r2 = reinterpret_cast<double*>(r2);
    s->info = reinterpret_cast<double*>(info); s->related = reinterpret_cast<int*>(rel); s->opt_map = reinterpret_cast<int*>(om);
  }
  return off + 256;
}

// scratch of a group: the descriptor table, then each graph's carve, one after another.  Every part starts on a 256-byte
// boundary: a carve's size is not a multiple of 8 when it ends with an odd node count's opt_map.
size_t align256(size_t n) { return (n + 255) & ~static_cast<size_t>(255); }
size_t group_head_bytes(int G) { return align256(static_cast<size_t>(G) * sizeof(PgDesc)); }
size_t group_scratch_bytes(const StaPgGraph* graphs, int G) {
  size_t off = group_head_bytes(G);
  for (int k = 0; k < G; ++k)
    off += align256(carve(nullptr, graphs[k].num_nodes, graphs[k].num_edges, graphs[k].num_opt, nullptr));
  return off;
}

// refusals, before anything reaches the device
int check_group(const StaPgGraph* graphs, int G) {
  STA_REQUIRE(graphs != nullptr, "null graph table");
  STA_REQUIRE(G >= 1 && G <= PG_GROUP_MAX, "a group holds 1 to STA_PG_GROUP_MAX graphs");
  for (int k = 0; k < G; ++k) {
    const StaPgGraph& q = graphs[k];
    STA_REQUIRE(q.nodes && q.edges && q.meas && q.weights && q.opt_idx && q.nodes_out, "null pointer");
    STA_REQUIRE(q.num_nodes > 0 && q.num_edges > 0 && q.num_opt > 0 && q.num_opt <= q.num_nodes, "empty problem");
    STA_REQUIRE(q.num_opt <= STA_PG_DENSE_MAX_OPT,
                "more than 3657 optimised nodes: the one-CTA solve needs the RHS in shared memory");
  }
  return 0;
}

// the launch sequence of one LM step over graphs[0..G), G >= 2 (checked), info rows at info_out + 4 k
int launch_group(const StaPgGraph* graphs, int G, double dmin, double dmax, double* info_out, void* scratch,
                 cudaStream_t st) {
  PgGroupParams p = {};
  PgPanels panels = {};
  char* base = static_cast<char*>(scratch);
  PgDesc* descs = reinterpret_cast<PgDesc*>(base);
  size_t off = group_head_bytes(G);
  int max_nodes = 0, max_edges = 0, max_opt = 0, max_n7 = 0;
  for (int k = 0; k < G; ++k) {
    const StaPgGraph& q = graphs[k];
    PgDesc& d = p.g[k];
    d.nodes = q.nodes;
    d.edges = reinterpret_cast<const long long*>(q.edges);
    d.meas = q.meas;
    d.weights = q.weights;
    d.opt_idx = reinterpret_cast<const long long*>(q.opt_idx);
    d.nodes_out = q.nodes_out;
    d.info_out = info_out + 4 * k;
    off += align256(carve(base + off, q.num_nodes, q.num_edges, q.num_opt, &d.s));
    d.num_nodes = q.num_nodes;
    d.num_edges = q.num_edges;
    d.num_opt = q.num_opt;
    d.n7 = 7 * q.num_opt;
    d.damping = q.damping;
    panels.A[k] = d.s.A;
    panels.info[k] = d.s.info;
    panels.g[k] = d.s.g;
    panels.delta[k] = d.s.delta;
    panels.n[k] = d.n7;
    max_nodes = std::max(max_nodes, d.num_nodes);
    max_edges = std::max(max_edges, d.num_edges);
    max_opt = std::max(max_opt, d.num_opt);
    max_n7 = std::max(max_n7, d.n7);
  }
  const unsigned g = static_cast<unsigned>(G);
  pg_group_setup_kernel<<<1, 32, 0, st>>>(p, G, descs);
  pg_opt_map_group_kernel<<<dim3((max_nodes + 255) / 256, g), 256, 0, st>>>(descs, 0);
  pg_opt_map_group_kernel<<<dim3((max_opt + 255) / 256, g), 256, 0, st>>>(descs, 1);
  const long long a_elems = static_cast<long long>(max_n7) * max_n7;
  pg_zero_kernel<<<dim3(static_cast<unsigned>(std::min<long long>((a_elems + 255) / 256, 2048)), g), 256, 0, st>>>(descs);
  pg_edge_group_kernel<<<dim3((max_edges + 63) / 64, g), 64, 0, st>>>(descs, 0);
  pg_assemble_group_kernel<<<dim3(max_opt, g), 64, 0, st>>>(descs);
  pg_loss_group_kernel<<<g, 256, 0, st>>>(descs, 0);
  pg_damp_group_kernel<<<dim3((max_n7 + 255) / 256, g), 256, 0, st>>>(descs, dmin, dmax);
  for (int k0 = 0; k0 < max_n7; k0 += NB) {
    chol_diag_group_kernel<<<g, dim3(NB, NB), 0, st>>>(panels, k0);
    const int rest = max_n7 - k0 - NB;
    if (rest > 0) {
      const unsigned nt = static_cast<unsigned>((rest + NB - 1) / NB);
      chol_trsm_group_kernel<<<dim3(nt, g), NB, 0, st>>>(panels, k0);
      chol_syrk_group_kernel<<<dim3(nt, nt, g), dim3(NB, NB), 0, st>>>(panels, k0);
    }
  }
  static PerDeviceOnce once;
  STA_CHECK_CUDA(once.run([&] {
    return cudaFuncSetAttribute(pg_solve_group_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PG_SOLVE_SMEM_MAX);
  }));
  pg_solve_group_kernel<<<g, 1024, static_cast<size_t>(max_n7) * sizeof(double), st>>>(panels);
  pg_update_group_kernel<<<dim3((max_nodes + 127) / 128, g), 128, 0, st>>>(descs);
  pg_edge_group_kernel<<<dim3((max_edges + 63) / 64, g), 64, 0, st>>>(descs, 1);
  pg_loss_group_kernel<<<g, 256, 0, st>>>(descs, 1);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace

size_t pose_graph_scratch_bytes(int num_nodes, int num_edges, int num_opt) {
  if (num_nodes < 0 || num_edges < 0 || num_opt < 0) return 0;
  return carve(nullptr, num_nodes, num_edges, num_opt, nullptr);
}

// the one-graph step, also what a group of one runs
int launch_pose_graph_lm_step(const float* nodes, int num_nodes, const long long* edges, const float* meas, const float* weights,
                              int num_edges, const long long* opt_idx, int num_opt, double damping, double dmin, double dmax,
                              float* nodes_out, double* info_out, void* scratch, cudaStream_t st) {
  STA_REQUIRE(nodes && edges && meas && weights && opt_idx && nodes_out && info_out && scratch, "null pointer");
  STA_REQUIRE(num_nodes > 0 && num_edges > 0 && num_opt > 0 && num_opt <= num_nodes, "empty problem");
  STA_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 7) == 0, "scratch must be 8-byte aligned");
  const int n7 = 7 * num_opt;
  STA_REQUIRE(static_cast<size_t>(n7) * 8 <= PG_SOLVE_SMEM_MAX,
              "more than 3657 optimised nodes: the one-CTA solve needs the RHS in shared memory");
  PgScratch s;
  carve(static_cast<char*>(scratch), num_nodes, num_edges, num_opt, &s);
  const int E = num_edges;
  pg_opt_map_kernel<<<(num_nodes + 255) / 256, 256, 0, st>>>(opt_idx, num_opt, num_nodes, s.opt_map, 0);
  pg_opt_map_kernel<<<(num_opt + 255) / 256, 256, 0, st>>>(opt_idx, num_opt, num_nodes, s.opt_map, 1);
  STA_CHECK_CUDA(cudaMemsetAsync(s.A, 0, static_cast<size_t>(n7) * n7 * sizeof(double), st));
  const double one = 1.0;
  STA_CHECK_CUDA(cudaMemcpyAsync(s.info + 3, &one, sizeof(double), cudaMemcpyHostToDevice, st));  // Cholesky-ok flag
  pg_edge_kernel<<<(E + 63) / 64, 64, 0, st>>>(nodes, edges, meas, s.opt_map, E, s.r, s.J, s.related);
  pg_assemble_kernel<<<num_opt, 64, 0, st>>>(edges, weights, s.opt_map, s.related, s.r, s.J, E, n7, s.A, s.g);
  pg_loss_kernel<<<1, 256, 0, st>>>(s.r, weights, s.related, E, nullptr, 0, s.info, 0);
  pg_damp_kernel<<<(n7 + 255) / 256, 256, 0, st>>>(s.A, n7, dmin, dmax, damping);
  for (int k0 = 0; k0 < n7; k0 += NB) {
    chol_diag_kernel<<<1, dim3(NB, NB), 0, st>>>(s.A, n7, k0, s.info);
    const int rest = n7 - k0 - NB;
    if (rest > 0) {
      const int nt = (rest + NB - 1) / NB;
      chol_trsm_kernel<<<nt, NB, 0, st>>>(s.A, n7, k0);
      chol_syrk_kernel<<<dim3(nt, nt), dim3(NB, NB), 0, st>>>(s.A, n7, k0);
    }
  }
  static PerDeviceOnce once;
  STA_CHECK_CUDA(once.run([&] {
    return cudaFuncSetAttribute(pg_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PG_SOLVE_SMEM_MAX);
  }));
  pg_solve_kernel<<<1, 1024, static_cast<size_t>(n7) * sizeof(double), st>>>(s.A, s.g, n7, s.delta);
  pg_update_kernel<<<(num_nodes + 127) / 128, 128, 0, st>>>(nodes, s.opt_map, s.delta, num_nodes, nodes_out);
  pg_edge_kernel<<<(E + 63) / 64, 64, 0, st>>>(nodes_out, edges, meas, s.opt_map, E, s.r2, nullptr, s.related);
  pg_loss_kernel<<<1, 256, 0, st>>>(s.r2, weights, s.related, E, s.delta, n7, s.info, 1);
  STA_CHECK_CUDA(cudaMemcpyAsync(info_out, s.info, 4 * sizeof(double), cudaMemcpyDeviceToDevice, st));
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace sta

extern "C" {

size_t sta_pose_graph_group_scratch_bytes(const StaPgGraph* graphs, int G) {
  if (sta::check_group(graphs, G) != 0) return 0;
  return sta::group_scratch_bytes(graphs, G);
}

int sta_pose_graph_lm_step_group(const StaPgGraph* graphs, int G, double dmin, double dmax, double* info_out, void* scratch,
                                 size_t scratch_bytes, void* stream) {
  const int rc = sta::check_group(graphs, G);
  if (rc != 0) return rc;
  STA_REQUIRE(info_out && scratch, "null pointer");
  STA_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 7) == 0, "scratch must be 8-byte aligned");
  STA_REQUIRE(scratch_bytes >= sta::group_scratch_bytes(graphs, G), "scratch smaller than sta_pose_graph_group_scratch_bytes");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (G == 1) {  // the one-graph launch sequence (its scratch is a prefix of the group's)
    const StaPgGraph& q = graphs[0];
    return sta::launch_pose_graph_lm_step(q.nodes, q.num_nodes, reinterpret_cast<const long long*>(q.edges), q.meas, q.weights,
                                          q.num_edges, reinterpret_cast<const long long*>(q.opt_idx), q.num_opt, q.damping,
                                          dmin, dmax, q.nodes_out, info_out, scratch, st);
  }
  return sta::launch_group(graphs, G, dmin, dmax, info_out, scratch, st);
}

}  // extern "C"
