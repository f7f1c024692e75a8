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
#include <math.h>

#include "common.cuh"
#include "host_util.h"
#include "ops.h"
#include "pose_graph.cuh"

namespace sta {

namespace {

// ---------------------------------------------------------------------------
// one CTA per optimised node a: block row a of A = J^T W J and of g = J^T W r.  64 threads: thread (p, q) = entry of
// the 7x7 blocks (49), threads 49..55 = the 7 entries of g.  Edges are visited in index order: fixed summation order.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(64)
pg_assemble_kernel(const long long* __restrict__ edges, const float* __restrict__ weights, const int* __restrict__ opt_map,
                   const int* __restrict__ related, const double* __restrict__ r, const double* __restrict__ J, int E, int n7,
                   double* __restrict__ A, double* __restrict__ g) {
  const int a = blockIdx.x;
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

// LM damping of pp.optim.LM.step: A.diagonal().clamp_(min, max); A.diagonal() += damping * A.diagonal()
__global__ void pg_damp_kernel(double* A, int n7, double dmin, double dmax, double damping) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n7) return;
  double d = A[static_cast<long long>(i) * n7 + i];
  d = fmin(fmax(d, dmin), dmax);
  A[static_cast<long long>(i) * n7 + i] = d * (1.0 + damping);
}

// ---------------------------------------------------------------------------
// dense blocked right-looking Cholesky (lower), fp64, 32-wide panels.  info[3] is set to 0 on a non-positive pivot.
// ---------------------------------------------------------------------------
constexpr int NB = 32;
__global__ void __launch_bounds__(NB * NB) chol_diag_kernel(double* A, int n, int k0, double* info) {
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
// rows below the panel: X L_kk^T = A_ik  (one thread per row)
__global__ void __launch_bounds__(NB) chol_trsm_kernel(double* A, int n, int k0) {
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
// trailing update: A_ij -= L_ik L_jk^T for tiles j <= i below / right of the panel
__global__ void __launch_bounds__(NB * NB) chol_syrk_kernel(double* A, int n, int k0) {
  if (blockIdx.x > blockIdx.y) return;  // (bj, bi) with bj <= bi
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
// x = -(L L^T)^-1 g, one CTA: blocked forward then backward substitution with the right-hand side in shared memory
__global__ void __launch_bounds__(1024) pg_solve_kernel(const double* __restrict__ A, const double* __restrict__ g, int n,
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


__global__ void pg_opt_map_kernel(const long long* __restrict__ opt_idx, int num_opt, int num_nodes, int* __restrict__ opt_map,
                                  int phase) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (phase == 0) {
    if (i < num_nodes) opt_map[i] = -1;
  } else if (i < num_opt) {
    const long long v = opt_idx[i];
    if (v >= 0 && v < num_nodes) opt_map[v] = i;  // pose_graph.py:90-91
  }
}

struct PgScratch {
  double *r, *J, *A, *g, *delta, *r2, *info;
  int *related, *opt_map;
};
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

}  // namespace

size_t pose_graph_scratch_bytes(int num_nodes, int num_edges, int num_opt) {
  if (num_nodes < 0 || num_edges < 0 || num_opt < 0) return 0;
  return carve(nullptr, num_nodes, num_edges, num_opt, nullptr);
}

int launch_pose_graph_lm_step(const float* nodes, int num_nodes, const long long* edges, const float* meas, const float* weights,
                              int num_edges, const long long* opt_idx, int num_opt, double damping, double dmin, double dmax,
                              float* nodes_out, double* info_out, void* scratch, cudaStream_t st) {
  STA_REQUIRE(nodes && edges && meas && weights && opt_idx && nodes_out && info_out && scratch, "null pointer");
  STA_REQUIRE(num_nodes > 0 && num_edges > 0 && num_opt > 0 && num_opt <= num_nodes, "empty problem");
  STA_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 7) == 0, "scratch must be 8-byte aligned");
  const int n7 = 7 * num_opt;
  STA_REQUIRE(static_cast<size_t>(n7) * 8 <= 200 * 1024, "more than 3657 optimised nodes: the one-CTA solve needs the RHS in shared memory");
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
    return cudaFuncSetAttribute(pg_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
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
