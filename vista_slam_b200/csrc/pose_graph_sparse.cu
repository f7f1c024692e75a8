// Block-sparse route of the Sim(3) pose-graph LM step: the residuals, Jacobians, normal equations, damping, update and
// losses of sta_pose_graph_lm_step (pose_graph.cu), with A d = -g solved by a supernode-free block Cholesky (7x7 blocks)
// whose cost follows the nonzeros of the factor instead of (7 n)^3, and with no bound on the number of optimised nodes.
//
// Plan (host, once per edge list and optimised set, i.e. once per PoseGraphOpt.optimize):
//   * block graph of the optimised nodes (one vertex per node, one edge per pair joined by a related edge);
//   * fill-reducing ordering by nested dissection along node order: split the current node set at its median index,
//     take as separator the smaller of the two boundaries (the nodes of one half with a neighbour in the other; the right
//     one on a tie), recurse on the two parts, separator last; sets of at most kLeaf nodes keep node order.  Pose graphs
//     number their nodes along the trajectory, so a boundary is a few keyframes' nodes plus the loop closures crossing it;
//   * elimination tree, block pattern of L (column K: diagonal block first, then its rows ascending), and levels
//     (level = height in the elimination tree: a column only depends on its descendants, which sit on lower levels);
//   * for every block (I, K) of L its update list: the columns j < K with L_Ij and L_Kj nonzero, ascending;
//   * for every optimised node its incident related edges in edge order, and for every off-diagonal block of A the
//     related edges joining its two nodes in edge order.
// Numeric step (per LM iteration, no host synchronisation, a launch sequence fixed by the plan):
//   pg_edge_kernel -> sp_assemble_kernel (one owner CTA per block of L: the dense route's per-edge arithmetic in edge
//   order, so A, g and the loss equal pg_assemble_kernel's; the diagonal owners apply pg_damp_kernel's damping) ->
//   pg_loss_kernel -> per level: sp_update_kernel (one CTA per block of the level's columns, updates in list order) and
//   sp_factor_kernel (one CTA per column: 7x7 Cholesky of the diagonal block, then the off-diagonal rows) -> level-scheduled
//   forward / backward solves (one CTA per block row / column) -> pg_update_kernel -> pg_edge_kernel -> pg_loss_kernel.
// fp64 throughout, no atomics, every output element has one owner and a fixed summation order: deterministic.  No
// inter-CTA waiting: levels are ordered by stream order only.
#include <math.h>

#include <algorithm>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/sta_b200.h"
#include "host_util.h"
#include "pose_graph.cuh"

namespace sta {
namespace {

constexpr int kLeaf = 8;  // nested dissection stops at this many nodes
size_t align_up(size_t n) { return (n + 255) & ~static_cast<size_t>(255); }

struct PgSymbolic {
  int num_nodes = 0, num_edges = 0, n = 0;
  long long nnzb_a = 0;                      // lower-triangle blocks of A (diagonal included)
  std::vector<int> opt_map;                  // [num_nodes] local optimised index or -1
  std::vector<int> order;                    // position -> local optimised node
  std::vector<int> colptr, blk_row, blk_col; // blocks of L, column-major, diagonal first in its column
  std::vector<int> row_ptr, row_blk;         // off-diagonal blocks of each block row, ascending column
  std::vector<int> level;                    // [n] per position
  int nlev = 0;
  std::vector<int> lvl_col_ptr, lvl_col;     // positions grouped by level
  std::vector<int> lvl_blk_ptr, lvl_blk;     // blocks grouped by the level of their column
  std::vector<long long> upd_ptr;            // [nnzb + 1]
  std::vector<int> upd;                      // pairs (block L_Ij, block L_Kj)
  std::vector<int> inc_ptr, inc;             // per local node: 2 e + side over its related edges, edge order
  std::vector<int> oasm_ptr, oasm;           // per block of L: the edges summed into it (off-diagonal blocks only)
  long long nnzb() const { return static_cast<long long>(blk_row.size()); }
  long long nupd() const { return static_cast<long long>(upd.size()) / 2; }
};

void nd_order(const std::vector<std::vector<int>>& adj, const std::vector<int>& nodes, std::vector<int>& side,
              std::vector<int>& out) {
  const size_t m = nodes.size();
  if (m <= static_cast<size_t>(kLeaf)) {
    out.insert(out.end(), nodes.begin(), nodes.end());
    return;
  }
  const size_t h = m / 2;
  for (size_t k = 0; k < m; ++k) side[nodes[k]] = k < h ? 0 : 1;
  std::vector<char> bnd(m, 0);
  size_t nl = 0, nr = 0;
  for (size_t k = 0; k < m; ++k) {
    const int other = k < h ? 1 : 0;
    for (int u : adj[nodes[k]])
      if (side[u] == other) { bnd[k] = 1; break; }
    if (bnd[k]) (k < h ? nl : nr) += 1;
  }
  for (size_t k = 0; k < m; ++k) side[nodes[k]] = -1;
  const bool sep_left = nl < nr;
  std::vector<int> first, second, sep;
  for (size_t k = 0; k < m; ++k) {
    const bool left = k < h;
    if (bnd[k] && left == sep_left) sep.push_back(nodes[k]);
    else (left ? first : second).push_back(nodes[k]);
  }
  nd_order(adj, first, side, out);
  nd_order(adj, second, side, out);
  out.insert(out.end(), sep.begin(), sep.end());
}

int find_block(const PgSymbolic& S, int I, int K) {  // index of block (I, K), I >= K, or -1
  const int* b = S.blk_row.data() + S.colptr[K];
  const int* e = S.blk_row.data() + S.colptr[K + 1];
  if (I == K) return S.colptr[K];
  const int* f = std::lower_bound(b + 1, e, I);
  return (f != e && *f == I) ? static_cast<int>(f - S.blk_row.data()) : -1;
}

// Validates the problem and builds the symbolic plan.  Returns 0, or 2 with the error set (nothing launched).
int pg_analyze(const long long* edges, int E, int Nn, const long long* opt, int No, PgSymbolic& S) {
  STA_REQUIRE(Nn > 0 && E > 0 && No > 0 && No <= Nn, "empty problem");
  STA_REQUIRE(edges != nullptr && opt != nullptr, "null pointer");
  for (int e = 0; e < E; ++e)
    for (int s = 0; s < 2; ++s) {
      const long long v = edges[2 * e + s];
      if (v < 0 || v >= Nn) {
        set_last_error("edge " + std::to_string(e) + " has endpoint " + std::to_string(v) + " outside [0, num_nodes = " +
                       std::to_string(Nn) + ")");
        return 2;
      }
    }
  S = PgSymbolic();
  S.num_nodes = Nn;
  S.num_edges = E;
  S.n = No;
  S.opt_map.assign(Nn, -1);
  for (int a = 0; a < No; ++a) {
    const long long v = opt[a];
    if (v < 0 || v >= Nn) {
      set_last_error("optimised index " + std::to_string(v) + " outside [0, num_nodes = " + std::to_string(Nn) + ")");
      return 2;
    }
    if (S.opt_map[v] >= 0) {
      set_last_error("optimised index " + std::to_string(v) + " repeated");
      return 2;
    }
    S.opt_map[v] = a;
  }
  const int n = No;
  // block graph
  std::vector<std::vector<int>> adj(n);
  for (int e = 0; e < E; ++e) {
    const int a = S.opt_map[edges[2 * e]], b = S.opt_map[edges[2 * e + 1]];
    if (a >= 0 && b >= 0 && a != b) {
      adj[a].push_back(b);
      adj[b].push_back(a);
    }
  }
  long long npairs = 0;
  for (auto& v : adj) {
    std::sort(v.begin(), v.end());
    v.erase(std::unique(v.begin(), v.end()), v.end());
    npairs += static_cast<long long>(v.size());
  }
  S.nnzb_a = n + npairs / 2;
  // ordering
  {
    std::vector<int> all(n), side(n, -1);
    for (int a = 0; a < n; ++a) all[a] = a;
    S.order.reserve(n);
    nd_order(adj, all, side, S.order);
  }
  std::vector<int> pos(n);
  for (int k = 0; k < n; ++k) pos[S.order[k]] = k;
  // symbolic factorisation: struct(K) = {adjacent positions > K} u struct(children) \ {K}
  std::vector<std::vector<int>> st(n), children(n);
  std::vector<int> mark(n, -1);
  S.level.assign(n, 0);
  for (int K = 0; K < n; ++K) {
    std::vector<int>& s = st[K];
    mark[K] = K;
    for (int u : adj[S.order[K]]) {
      const int P = pos[u];
      if (P > K && mark[P] != K) { mark[P] = K; s.push_back(P); }
    }
    for (int c : children[K])
      for (int P : st[c])
        if (mark[P] != K) { mark[P] = K; s.push_back(P); }
    std::sort(s.begin(), s.end());
    if (!s.empty()) {
      children[s[0]].push_back(K);
      S.level[s[0]] = std::max(S.level[s[0]], S.level[K] + 1);
    }
  }
  S.colptr.assign(n + 1, 0);
  for (int K = 0; K < n; ++K) S.colptr[K + 1] = S.colptr[K] + 1 + static_cast<int>(st[K].size());
  const int nnzb = S.colptr[n];
  S.blk_row.resize(nnzb);
  S.blk_col.resize(nnzb);
  for (int K = 0; K < n; ++K) {
    int b = S.colptr[K];
    S.blk_row[b] = K;
    S.blk_col[b] = K;
    for (int I : st[K]) { ++b; S.blk_row[b] = I; S.blk_col[b] = K; }
  }
  // block rows (forward solve)
  S.row_ptr.assign(n + 1, 0);
  for (int b = 0; b < nnzb; ++b)
    if (S.blk_row[b] != S.blk_col[b]) ++S.row_ptr[S.blk_row[b] + 1];
  for (int I = 0; I < n; ++I) S.row_ptr[I + 1] += S.row_ptr[I];
  S.row_blk.resize(S.row_ptr[n]);
  {
    std::vector<int> cur(S.row_ptr.begin(), S.row_ptr.end() - 1);
    for (int b = 0; b < nnzb; ++b)  // column-major walk: each row's blocks come out in ascending column
      if (S.blk_row[b] != S.blk_col[b]) S.row_blk[cur[S.blk_row[b]]++] = b;
  }
  // levels
  S.nlev = 0;
  for (int K = 0; K < n; ++K) S.nlev = std::max(S.nlev, S.level[K] + 1);
  S.lvl_col_ptr.assign(S.nlev + 1, 0);
  S.lvl_blk_ptr.assign(S.nlev + 1, 0);
  for (int K = 0; K < n; ++K) {
    ++S.lvl_col_ptr[S.level[K] + 1];
    S.lvl_blk_ptr[S.level[K] + 1] += S.colptr[K + 1] - S.colptr[K];
  }
  for (int l = 0; l < S.nlev; ++l) {
    S.lvl_col_ptr[l + 1] += S.lvl_col_ptr[l];
    S.lvl_blk_ptr[l + 1] += S.lvl_blk_ptr[l];
  }
  S.lvl_col.resize(n);
  S.lvl_blk.resize(nnzb);
  {
    std::vector<int> cc(S.lvl_col_ptr.begin(), S.lvl_col_ptr.end() - 1), cb(S.lvl_blk_ptr.begin(), S.lvl_blk_ptr.end() - 1);
    for (int K = 0; K < n; ++K) {
      S.lvl_col[cc[S.level[K]]++] = K;
      for (int b = S.colptr[K]; b < S.colptr[K + 1]; ++b) S.lvl_blk[cb[S.level[K]]++] = b;
    }
  }
  // update lists: column j contributes L_Ij L_Kj^T to block (I, K) for every I >= K in struct(j); j ascending
  std::vector<long long> cnt(nnzb + 1, 0);
  for (int pass = 0; pass < 2; ++pass) {
    std::vector<long long> cur;
    if (pass == 1) {
      S.upd_ptr.assign(nnzb + 1, 0);
      for (int b = 0; b < nnzb; ++b) S.upd_ptr[b + 1] = S.upd_ptr[b] + cnt[b];
      S.upd.resize(2 * S.upd_ptr[nnzb]);
      cur.assign(S.upd_ptr.begin(), S.upd_ptr.end() - 1);
    }
    for (int j = 0; j < n; ++j) {
      const int s0 = S.colptr[j] + 1, s1 = S.colptr[j + 1];
      for (int x = s0; x < s1; ++x) {
        const int K = S.blk_row[x];
        int w = S.colptr[K];  // walks column K: struct(j) n [K, n) lies in {K} u struct(K)
        for (int y = x; y < s1; ++y) {
          const int I = S.blk_row[y];
          while (S.blk_row[w] != I) ++w;
          if (pass == 0) {
            ++cnt[w];
          } else {
            const long long u = cur[w]++;
            S.upd[2 * u] = y;      // L_Ij
            S.upd[2 * u + 1] = x;  // L_Kj
          }
        }
      }
    }
  }
  // assembly lists
  S.inc_ptr.assign(n + 1, 0);
  S.oasm_ptr.assign(nnzb + 1, 0);
  std::vector<int> eblk(E, -1);
  for (int e = 0; e < E; ++e) {
    const int a = S.opt_map[edges[2 * e]], b = S.opt_map[edges[2 * e + 1]];
    if (a >= 0) ++S.inc_ptr[a + 1];
    if (b >= 0) ++S.inc_ptr[b + 1];
    if (a >= 0 && b >= 0 && a != b) {
      eblk[e] = find_block(S, std::max(pos[a], pos[b]), std::min(pos[a], pos[b]));
      ++S.oasm_ptr[eblk[e] + 1];
    }
  }
  for (int a = 0; a < n; ++a) S.inc_ptr[a + 1] += S.inc_ptr[a];
  for (int b = 0; b < nnzb; ++b) S.oasm_ptr[b + 1] += S.oasm_ptr[b];
  S.inc.resize(S.inc_ptr[n]);
  S.oasm.resize(S.oasm_ptr[nnzb]);
  {
    std::vector<int> ci(S.inc_ptr.begin(), S.inc_ptr.end() - 1), co(S.oasm_ptr.begin(), S.oasm_ptr.end() - 1);
    for (int e = 0; e < E; ++e) {
      const int a = S.opt_map[edges[2 * e]], b = S.opt_map[edges[2 * e + 1]];
      if (a >= 0) S.inc[ci[a]++] = 2 * e;
      if (b >= 0) S.inc[ci[b]++] = 2 * e + 1;
      if (eblk[e] >= 0) S.oasm[co[eblk[e]]++] = e;
    }
  }
  return 0;
}

// ---------------------------------------------------------------------------
// device plan: one arena holding the plan arrays and the per-iteration scratch
// ---------------------------------------------------------------------------
struct PgDev {
  long long* edges;
  int *opt_map, *order, *colptr, *blk_row, *blk_col, *row_ptr, *row_blk, *lvl_col, *lvl_blk, *inc_ptr, *inc, *oasm_ptr,
      *oasm, *related;
  long long* upd_ptr;
  int2* upd;
  double *r, *J, *r2, *L, *g, *y, *delta, *info;
};

size_t carve_plan(char* base, const PgSymbolic& S, PgDev* d) {
  size_t off = 0;
  auto take = [&](auto** p, size_t count) {
    off = (off + 255) & ~static_cast<size_t>(255);
    if (base) *p = reinterpret_cast<std::remove_reference_t<decltype(*p)>>(base + off);
    off += count * sizeof(**p);
  };
  PgDev t;
  PgDev& x = d ? *d : t;
  const size_t E = S.num_edges, n = S.n, nb = S.blk_row.size();
  take(&x.edges, 2 * E);
  take(&x.opt_map, S.num_nodes);
  take(&x.order, n);
  take(&x.colptr, n + 1);
  take(&x.blk_row, nb);
  take(&x.blk_col, nb);
  take(&x.row_ptr, n + 1);
  take(&x.row_blk, S.row_blk.size());
  take(&x.lvl_col, n);
  take(&x.lvl_blk, nb);
  take(&x.inc_ptr, n + 1);
  take(&x.inc, S.inc.size());
  take(&x.oasm_ptr, nb + 1);
  take(&x.oasm, S.oasm.size());
  take(&x.related, E);
  take(&x.upd_ptr, nb + 1);
  take(&x.upd, S.upd.size() / 2);
  take(&x.r, 7 * E);
  take(&x.J, 49 * E);
  take(&x.r2, 7 * E);
  take(&x.L, 49 * nb);
  take(&x.g, 7 * n);
  take(&x.y, 7 * n);
  take(&x.delta, 7 * n);
  take(&x.info, 4);
  return off + 256;
}

// ---------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------
__global__ void sp_info_init_kernel(double* info) { info[3] = 1.0; }  // Cholesky-ok flag

// one CTA per block of L.  Diagonal block of node a: pg_assemble_kernel's loop restricted to a's incident edges (same
// order, same arithmetic: diag += s, A_aa -= s for a self-edge, then A_aa + diag), then pg_damp_kernel's damping, and g_a
// on threads 49..55.  Off-diagonal block (I, K) = A[order[I]][order[K]]: minus the sum of s over the edges joining the two
// nodes, in edge order, as row owner order[I] computes it in pg_assemble_kernel.  Fill blocks come out zero.
__device__ __forceinline__ void sp_assemble(int b, const long long* __restrict__ edges, const float* __restrict__ weights,
                                            const int* __restrict__ opt_map, const double* __restrict__ r,
                                            const double* __restrict__ J, const int* __restrict__ order,
                                            const int* __restrict__ blk_row, const int* __restrict__ blk_col,
                                            const int* __restrict__ inc_ptr, const int* __restrict__ inc,
                                            const int* __restrict__ oasm_ptr, const int* __restrict__ oasm, double dmin,
                                            double dmax, double damping, double* __restrict__ L, double* __restrict__ g) {
  const int t = threadIdx.x;
  const int p = t / 7, q = t - 7 * p;
  const int I = blk_row[b], K = blk_col[b];
  if (I != K) {
    if (t >= 49) return;
    double acc = 0.0;
    for (int k = oasm_ptr[b]; k < oasm_ptr[b + 1]; ++k) {
      const int e = oasm[k];
      const double* Je = J + 49ll * e;
      const float* w = weights + 7 * e;
      double s = 0.0;
      for (int m = 0; m < 7; ++m) s = fma(Je[7 * m + p] * static_cast<double>(w[m]), Je[7 * m + q], s);
      acc -= s;
    }
    L[49ll * b + t] = acc;
    return;
  }
  const int a = order[K];
  double diag = 0.0, off = 0.0, gv = 0.0;
  for (int k = inc_ptr[a]; k < inc_ptr[a + 1]; ++k) {
    const int e = inc[k] >> 1, side = inc[k] & 1;
    const int oi = opt_map[edges[2 * e]], oj = opt_map[edges[2 * e + 1]];
    const double* Je = J + 49ll * e;
    const float* w = weights + 7 * e;
    const int other = side == 0 ? oj : oi;
    if (t < 49) {
      double s = 0.0;
      for (int m = 0; m < 7; ++m) s = fma(Je[7 * m + p] * static_cast<double>(w[m]), Je[7 * m + q], s);
      diag += s;
      if (other == a) off -= s;
    } else if (t < 56) {
      const int pp = t - 49;
      double s = 0.0;
      for (int m = 0; m < 7; ++m) s = fma(Je[7 * m + pp] * static_cast<double>(w[m]), r[7ll * e + m], s);
      gv += side == 0 ? -s : s;
    }
  }
  if (t < 49) {
    double v = off + diag;
    if (p == q) {
      v = fmin(fmax(v, dmin), dmax);
      v = v * (1.0 + damping);
    }
    L[49ll * b + t] = v;
  } else if (t < 56) {
    g[7 * a + (t - 49)] = gv;
  }
}
__global__ void __launch_bounds__(64)
sp_assemble_kernel(const long long* __restrict__ edges, const float* __restrict__ weights, const int* __restrict__ opt_map,
                   const double* __restrict__ r, const double* __restrict__ J, const int* __restrict__ order,
                   const int* __restrict__ blk_row, const int* __restrict__ blk_col, const int* __restrict__ inc_ptr,
                   const int* __restrict__ inc, const int* __restrict__ oasm_ptr, const int* __restrict__ oasm, double dmin,
                   double dmax, double damping, double* __restrict__ L, double* __restrict__ g) {
  sp_assemble(blockIdx.x, edges, weights, opt_map, r, J, order, blk_row, blk_col, inc_ptr, inc, oasm_ptr, oasm, dmin, dmax,
              damping, L, g);
}

// one CTA per block (I, K) of the level's columns: A_IK -= sum_j L_Ij L_Kj^T over its update list, in list order
__device__ __forceinline__ void sp_update(int b, const long long* __restrict__ upd_ptr, const int2* __restrict__ upd,
                                          double* L) {
  const int t = threadIdx.x;
  if (t >= 49) return;
  const int p = t / 7, q = t - 7 * p;
  double acc = L[49ll * b + t];
  for (long long u = upd_ptr[b]; u < upd_ptr[b + 1]; ++u) {
    const int2 xy = upd[u];
    const double* Li = L + 49ll * xy.x + 7 * p;
    const double* Lk = L + 49ll * xy.y + 7 * q;
    double s = 0.0;
    for (int m = 0; m < 7; ++m) s = fma(Li[m], Lk[m], s);
    acc -= s;
  }
  L[49ll * b + t] = acc;
}
__global__ void __launch_bounds__(64)
sp_update_kernel(const int* __restrict__ lvl_blk, const long long* __restrict__ upd_ptr, const int2* __restrict__ upd,
                 double* L) {
  sp_update(lvl_blk[blockIdx.x], upd_ptr, upd, L);
}

// one CTA per column K of the level: Cholesky of the 7x7 diagonal block (chol_diag_kernel's recurrence on its lower
// triangle; a non-positive pivot clears info[3] and is replaced by 1), then X L_KK^T = A_IK for every off-diagonal block,
// one thread per block row (chol_trsm_kernel's recurrence)
__device__ __forceinline__ void sp_factor(int K, const int* __restrict__ colptr, double* L, double* info) {
  __shared__ double S[7][8];
  const int t = threadIdx.x;
  const int b0 = colptr[K], nb = colptr[K + 1] - b0;
  double* D = L + 49ll * b0;
  if (t < 49) S[t / 7][t % 7] = D[t];
  __syncthreads();
  if (t == 0) {
    for (int k = 0; k < 7; ++k) {
      const double d = S[k][k];
      if (!(d > 0.0)) { info[3] = 0.0; S[k][k] = 1.0; } else S[k][k] = sqrt(d);
      for (int r = k + 1; r < 7; ++r) S[r][k] /= S[k][k];
      for (int r = k + 1; r < 7; ++r)
        for (int c = k + 1; c <= r; ++c) S[r][c] -= S[r][k] * S[c][k];
    }
  }
  __syncthreads();
  if (t < 49 && t % 7 <= t / 7) D[t] = S[t / 7][t % 7];
  for (int rr = t; rr < 7 * (nb - 1); rr += blockDim.x) {
    double* ar = L + 49ll * (b0 + 1 + rr / 7) + 7 * (rr % 7);
    double x[7];
    for (int c = 0; c < 7; ++c) x[c] = ar[c];
    for (int c = 0; c < 7; ++c) {
      double s = x[c];
      for (int cc = 0; cc < c; ++cc) s -= x[cc] * S[c][cc];
      x[c] = s / S[c][c];
    }
    for (int c = 0; c < 7; ++c) ar[c] = x[c];
  }
}
__global__ void __launch_bounds__(128)
sp_factor_kernel(const int* __restrict__ lvl_col, const int* __restrict__ colptr, double* L, double* info) {
  sp_factor(lvl_col[blockIdx.x], colptr, L, info);
}

// forward solve L y = -g (positions), one CTA per block row I of the level: rows of earlier levels are final
__device__ __forceinline__ void sp_forward(int I, const int* __restrict__ order, const int* __restrict__ colptr,
                                           const int* __restrict__ row_ptr, const int* __restrict__ row_blk,
                                           const int* __restrict__ blk_col, const double* __restrict__ L,
                                           const double* __restrict__ g, double* y) {
  __shared__ double b[7];
  const int t = threadIdx.x;
  if (t < 7) {
    double s = -g[7 * order[I] + t];
    for (int k = row_ptr[I]; k < row_ptr[I + 1]; ++k) {
      const int bk = row_blk[k];
      const double* Lb = L + 49ll * bk + 7 * t;
      const double* yk = y + 7ll * blk_col[bk];
      for (int q = 0; q < 7; ++q) s -= Lb[q] * yk[q];
    }
    b[t] = s;
  }
  __syncthreads();
  if (t == 0) {
    const double* D = L + 49ll * colptr[I];
    for (int c = 0; c < 7; ++c) {
      double s = b[c];
      for (int cc = 0; cc < c; ++cc) s -= D[7 * c + cc] * b[cc];
      b[c] = s / D[7 * c + c];
    }
  }
  __syncthreads();
  if (t < 7) y[7ll * I + t] = b[t];
}
__global__ void __launch_bounds__(32)
sp_forward_kernel(const int* __restrict__ lvl_col, const int* __restrict__ order, const int* __restrict__ colptr,
                  const int* __restrict__ row_ptr, const int* __restrict__ row_blk, const int* __restrict__ blk_col,
                  const double* __restrict__ L, const double* __restrict__ g, double* y) {
  sp_forward(lvl_col[blockIdx.x], order, colptr, row_ptr, row_blk, blk_col, L, g, y);
}

// backward solve L^T x = y, one CTA per column K of the level (levels descending): x overwrites y in place, and
// delta[order[K]] = x_K
__device__ __forceinline__ void sp_backward(int K, const int* __restrict__ order, const int* __restrict__ colptr,
                                            const int* __restrict__ blk_row, const double* __restrict__ L, double* y,
                                            double* __restrict__ delta) {
  __shared__ double b[7];
  const int t = threadIdx.x;
  if (t < 7) {
    double s = y[7ll * K + t];
    for (int k = colptr[K] + 1; k < colptr[K + 1]; ++k) {
      const double* Lb = L + 49ll * k + t;
      const double* xi = y + 7ll * blk_row[k];
      for (int q = 0; q < 7; ++q) s -= Lb[7 * q] * xi[q];
    }
    b[t] = s;
  }
  __syncthreads();
  if (t == 0) {
    const double* D = L + 49ll * colptr[K];
    for (int c = 6; c >= 0; --c) {
      double s = b[c];
      for (int cc = c + 1; cc < 7; ++cc) s -= D[7 * cc + c] * b[cc];
      b[c] = s / D[7 * c + c];
    }
  }
  __syncthreads();
  if (t < 7) {
    y[7ll * K + t] = b[t];
    delta[7ll * order[K] + t] = b[t];
  }
}
__global__ void __launch_bounds__(32)
sp_backward_kernel(const int* __restrict__ lvl_col, const int* __restrict__ order, const int* __restrict__ colptr,
                   const int* __restrict__ blk_row, const double* __restrict__ L, double* y, double* __restrict__ delta) {
  sp_backward(lvl_col[blockIdx.x], order, colptr, blk_row, L, y, delta);
}

// ---------------------------------------------------------------------------
// group form: one launch sequence steps the active members of a group plan.  blockIdx.y selects the member's descriptor
// (the last grid dimension of the loss kernels' grid (member)); CTAs past the member's edge, block, column or node
// count, and levels at or above its level count, return at once.  A member's CTAs run the solo kernels' bodies on its
// own plan arrays and scratch, so its result does not depend on the group around it.
// ---------------------------------------------------------------------------
constexpr int SP_GROUP_MAX = STA_PG_GROUP_MAX;

// a member plan as the kernels see it (uploaded once with the group plan)
struct SpMember {
  PgDev d;
  const int4* lvl;  // [nlev] {first block, blocks, first column, columns} of each level in lvl_blk / lvl_col
  int nlev, num_nodes, num_edges, n7, nnzb;
};
// one active member's step inputs (a kernel parameter of the setup kernel, every step)
struct SpStepArgs {
  const float* nodes;
  const float* meas;
  const float* weights;
  float* nodes_out;
  double* info_out;
  double damping;
  int member;
};
struct SpGroupParams {
  SpStepArgs s[SP_GROUP_MAX];
};
static_assert(sizeof(SpGroupParams) + 32 <= 4096, "the step arguments must fit the kernel-parameter space");
struct SpDesc {
  SpMember m;
  SpStepArgs s;
};

// the active members' descriptors into the group plan's table, and each one's Cholesky-ok flag (info[3]) set
__global__ void sp_group_setup_kernel(const __grid_constant__ SpGroupParams p, int A, const SpMember* __restrict__ members,
                                      SpDesc* __restrict__ descs) {
  const int k = threadIdx.x;
  if (k >= A) return;
  descs[k].m = members[p.s[k].member];
  descs[k].s = p.s[k];
  members[p.s[k].member].d.info[3] = 1.0;
}

// grid (x, member): residuals and Jacobians at the nodes (second = 0), or residuals alone at the candidate (second = 1)
__global__ void __launch_bounds__(64) sp_edge_group_kernel(const SpDesc* __restrict__ gd, int second) {
  const SpDesc& g = gd[blockIdx.y];
  const PgDev& d = g.m.d;
  pg_edge(blockIdx.x * blockDim.x + threadIdx.x, second ? g.s.nodes_out : g.s.nodes, d.edges, g.s.meas, d.opt_map,
          g.m.num_edges, second ? d.r2 : d.r, second ? nullptr : d.J, d.related);
}

// grid (block of L, member)
__global__ void __launch_bounds__(64) sp_assemble_group_kernel(const SpDesc* __restrict__ gd, double dmin, double dmax) {
  const SpDesc& g = gd[blockIdx.y];
  if (static_cast<int>(blockIdx.x) >= g.m.nnzb) return;
  const PgDev& d = g.m.d;
  sp_assemble(blockIdx.x, d.edges, g.s.weights, d.opt_map, d.r, d.J, d.order, d.blk_row, d.blk_col, d.inc_ptr, d.inc,
              d.oasm_ptr, d.oasm, dmin, dmax, g.s.damping, d.L, d.g);
}

// grid (member): loss before (second = 0), or loss after and |delta| (second = 1), then the member's info row out
__global__ void __launch_bounds__(256) sp_loss_group_kernel(const SpDesc* __restrict__ gd, int second) {
  const SpDesc& g = gd[blockIdx.x];
  const PgDev& d = g.m.d;
  if (!second) {
    pg_loss(d.r, g.s.weights, d.related, g.m.num_edges, nullptr, 0, d.info, 0);
    return;
  }
  pg_loss(d.r2, g.s.weights, d.related, g.m.num_edges, d.delta, g.m.n7, d.info, 1);
  if (threadIdx.x == 0)  // info[1], info[2] are this thread's own writes; info[0] and info[3] come from earlier launches
    for (int k = 0; k < 4; ++k) g.s.info_out[k] = d.info[k];
}

// grid (block of the level, member), levels >= 1
__global__ void __launch_bounds__(64) sp_update_group_kernel(const SpDesc* __restrict__ gd, int l) {
  const SpDesc& g = gd[blockIdx.y];
  if (l >= g.m.nlev) return;
  const int4 v = g.m.lvl[l];
  if (static_cast<int>(blockIdx.x) >= v.y) return;
  sp_update(g.m.d.lvl_blk[v.x + blockIdx.x], g.m.d.upd_ptr, g.m.d.upd, g.m.d.L);
}

// grid (column of the level, member)
__global__ void __launch_bounds__(128) sp_factor_group_kernel(const SpDesc* __restrict__ gd, int l) {
  const SpDesc& g = gd[blockIdx.y];
  if (l >= g.m.nlev) return;
  const int4 v = g.m.lvl[l];
  if (static_cast<int>(blockIdx.x) >= v.w) return;
  sp_factor(g.m.d.lvl_col[v.z + blockIdx.x], g.m.d.colptr, g.m.d.L, g.m.d.info);
}

// grid (column of the level, member)
__global__ void __launch_bounds__(32) sp_forward_group_kernel(const SpDesc* __restrict__ gd, int l) {
  const SpDesc& g = gd[blockIdx.y];
  if (l >= g.m.nlev) return;
  const int4 v = g.m.lvl[l];
  if (static_cast<int>(blockIdx.x) >= v.w) return;
  const PgDev& d = g.m.d;
  sp_forward(d.lvl_col[v.z + blockIdx.x], d.order, d.colptr, d.row_ptr, d.row_blk, d.blk_col, d.L, d.g, d.y);
}

// grid (column of the level, member)
__global__ void __launch_bounds__(32) sp_backward_group_kernel(const SpDesc* __restrict__ gd, int l) {
  const SpDesc& g = gd[blockIdx.y];
  if (l >= g.m.nlev) return;
  const int4 v = g.m.lvl[l];
  if (static_cast<int>(blockIdx.x) >= v.w) return;
  const PgDev& d = g.m.d;
  sp_backward(d.lvl_col[v.z + blockIdx.x], d.order, d.colptr, d.blk_row, d.L, d.y, d.delta);
}

// grid (x, member): nodes_out = Exp(delta_a) node for the optimised nodes, copies of the fixed ones
__global__ void sp_node_update_group_kernel(const SpDesc* __restrict__ gd) {
  const SpDesc& g = gd[blockIdx.y];
  pg_update(blockIdx.x * blockDim.x + threadIdx.x, g.s.nodes, g.m.d.opt_map, g.m.d.delta, g.m.num_nodes, g.s.nodes_out);
}

}  // namespace
}  // namespace sta

struct StaPgPlan {
  sta::PgSymbolic S;
  sta::PgDev d = {};
  void* arena = nullptr;
  size_t bytes = 0;
  int device = 0;
};

// a group plan: the member plans (borrowed, not owned), the maxima that size its grids, and one device allocation holding
// the members' descriptors, their level tables and the per-step descriptor table
struct StaPgGroupPlan {
  std::vector<const StaPgPlan*> plans;
  std::vector<int> max_blk, max_col;  // [levels] the largest block / column count any member has at each level
  int nlev = 0, max_edges = 0, max_nnzb = 0, max_nodes = 0;
  void* arena = nullptr;
  sta::SpMember* members = nullptr;
  sta::SpDesc* descs = nullptr;
  size_t bytes = 0;
  int device = 0;
};

using namespace sta;

namespace {
int group_launches(int nlev) { return 4 * nlev + 6; }  // setup, edge, assemble, loss, 2 nlev - 1 factor, 2 nlev solve, 3 after
}  // namespace

extern "C" {

int sta_pg_plan_analyze(const int64_t* edges, int num_edges, int num_nodes, const int64_t* opt_idx, int num_opt,
                        int64_t* stats5, int* order, int* level, int* colptr, int* blk_row, int64_t* upd_ptr, int* upd) {
  PgSymbolic S;
  const int rc = pg_analyze(reinterpret_cast<const long long*>(edges), num_edges, num_nodes,
                            reinterpret_cast<const long long*>(opt_idx), num_opt, S);
  if (rc) return rc;
  if (stats5) {
    stats5[0] = S.nnzb();
    stats5[1] = S.nnzb_a;
    stats5[2] = S.nlev;
    stats5[3] = S.nupd();
    stats5[4] = static_cast<int64_t>(carve_plan(nullptr, S, nullptr));
  }
  if (order) std::copy(S.order.begin(), S.order.end(), order);
  if (level) std::copy(S.level.begin(), S.level.end(), level);
  if (colptr) std::copy(S.colptr.begin(), S.colptr.end(), colptr);
  if (blk_row) std::copy(S.blk_row.begin(), S.blk_row.end(), blk_row);
  if (upd_ptr) std::copy(S.upd_ptr.begin(), S.upd_ptr.end(), upd_ptr);
  if (upd) std::copy(S.upd.begin(), S.upd.end(), upd);
  return 0;
}

int sta_pg_plan_create(const int64_t* edges, int num_edges, int num_nodes, const int64_t* opt_idx, int num_opt,
                       StaPgPlan** out) {
  STA_REQUIRE(out != nullptr, "null output pointer");
  *out = nullptr;
  StaPgPlan* P = new StaPgPlan();
  const int rc = pg_analyze(reinterpret_cast<const long long*>(edges), num_edges, num_nodes,
                            reinterpret_cast<const long long*>(opt_idx), num_opt, P->S);
  if (rc) {
    delete P;
    return rc;
  }
  const PgSymbolic& S = P->S;
  P->bytes = carve_plan(nullptr, S, nullptr);
  cudaError_t e = cudaGetDevice(&P->device);
  if (e == cudaSuccess) e = cudaMalloc(&P->arena, P->bytes);
  if (e == cudaSuccess) carve_plan(static_cast<char*>(P->arena), S, &P->d);
  auto up = [&](void* dst, const void* src, size_t bytes) {
    if (e == cudaSuccess && bytes) e = cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice);
  };
  const PgDev& d = P->d;
  up(d.edges, edges, sizeof(long long) * 2 * num_edges);
  up(d.opt_map, S.opt_map.data(), sizeof(int) * S.opt_map.size());
  up(d.order, S.order.data(), sizeof(int) * S.order.size());
  up(d.colptr, S.colptr.data(), sizeof(int) * S.colptr.size());
  up(d.blk_row, S.blk_row.data(), sizeof(int) * S.blk_row.size());
  up(d.blk_col, S.blk_col.data(), sizeof(int) * S.blk_col.size());
  up(d.row_ptr, S.row_ptr.data(), sizeof(int) * S.row_ptr.size());
  up(d.row_blk, S.row_blk.data(), sizeof(int) * S.row_blk.size());
  up(d.lvl_col, S.lvl_col.data(), sizeof(int) * S.lvl_col.size());
  up(d.lvl_blk, S.lvl_blk.data(), sizeof(int) * S.lvl_blk.size());
  up(d.inc_ptr, S.inc_ptr.data(), sizeof(int) * S.inc_ptr.size());
  up(d.inc, S.inc.data(), sizeof(int) * S.inc.size());
  up(d.oasm_ptr, S.oasm_ptr.data(), sizeof(int) * S.oasm_ptr.size());
  up(d.oasm, S.oasm.data(), sizeof(int) * S.oasm.size());
  up(d.upd_ptr, S.upd_ptr.data(), sizeof(long long) * S.upd_ptr.size());
  up(d.upd, S.upd.data(), sizeof(int) * S.upd.size());
  if (e != cudaSuccess) {
    set_last_error(std::string("sta_pg_plan_create: ") + cudaGetErrorString(e));
    sta_pg_plan_destroy(P);
    return 1;
  }
  *out = P;
  return 0;
}

void sta_pg_plan_destroy(StaPgPlan* plan) {
  if (!plan) return;
  if (plan->arena) {
    cudaDeviceSynchronize();
    cudaFree(plan->arena);
  }
  delete plan;
}

int sta_pg_plan_info(const StaPgPlan* plan, int64_t* out4) {
  STA_REQUIRE(plan && out4, "null argument");
  out4[0] = plan->S.nnzb();
  out4[1] = plan->S.nlev;
  out4[2] = static_cast<int64_t>(plan->bytes);
  out4[3] = plan->S.nupd();
  return 0;
}

int sta_pose_graph_lm_step_sparse(const StaPgPlan* plan, const float* nodes, const float* meas, const float* weights,
                                  double damping, double dmin, double dmax, float* nodes_out, double* info_out, void* stream) {
  STA_REQUIRE(plan && nodes && meas && weights && nodes_out && info_out, "null pointer");
  int dev = -1;
  STA_CHECK_CUDA(cudaGetDevice(&dev));
  STA_REQUIRE(dev == plan->device, "the plan was created on another device");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const PgSymbolic& S = plan->S;
  const PgDev& d = plan->d;
  const int E = S.num_edges, Nn = S.num_nodes, n7 = 7 * S.n;
  sp_info_init_kernel<<<1, 1, 0, st>>>(d.info);
  pg_edge_kernel<<<(E + 63) / 64, 64, 0, st>>>(nodes, d.edges, meas, d.opt_map, E, d.r, d.J, d.related);
  sp_assemble_kernel<<<static_cast<unsigned>(S.nnzb()), 64, 0, st>>>(d.edges, weights, d.opt_map, d.r, d.J, d.order,
                                                                       d.blk_row, d.blk_col, d.inc_ptr, d.inc, d.oasm_ptr,
                                                                       d.oasm, dmin, dmax, damping, d.L, d.g);
  pg_loss_kernel<<<1, 256, 0, st>>>(d.r, weights, d.related, E, nullptr, 0, d.info, 0);
  for (int l = 0; l < S.nlev; ++l) {
    const int b0 = S.lvl_blk_ptr[l], nb = S.lvl_blk_ptr[l + 1] - b0;
    const int c0 = S.lvl_col_ptr[l], nc = S.lvl_col_ptr[l + 1] - c0;
    if (l > 0) sp_update_kernel<<<nb, 64, 0, st>>>(d.lvl_blk + b0, d.upd_ptr, d.upd, d.L);  // leaves have no updates
    sp_factor_kernel<<<nc, 128, 0, st>>>(d.lvl_col + c0, d.colptr, d.L, d.info);
  }
  for (int l = 0; l < S.nlev; ++l) {
    const int c0 = S.lvl_col_ptr[l], nc = S.lvl_col_ptr[l + 1] - c0;
    sp_forward_kernel<<<nc, 32, 0, st>>>(d.lvl_col + c0, d.order, d.colptr, d.row_ptr, d.row_blk, d.blk_col, d.L, d.g, d.y);
  }
  for (int l = S.nlev - 1; l >= 0; --l) {
    const int c0 = S.lvl_col_ptr[l], nc = S.lvl_col_ptr[l + 1] - c0;
    sp_backward_kernel<<<nc, 32, 0, st>>>(d.lvl_col + c0, d.order, d.colptr, d.blk_row, d.L, d.y, d.delta);
  }
  pg_update_kernel<<<(Nn + 127) / 128, 128, 0, st>>>(nodes, d.opt_map, d.delta, Nn, nodes_out);
  pg_edge_kernel<<<(E + 63) / 64, 64, 0, st>>>(nodes_out, d.edges, meas, d.opt_map, E, d.r2, nullptr, d.related);
  pg_loss_kernel<<<1, 256, 0, st>>>(d.r2, weights, d.related, E, d.delta, n7, d.info, 1);
  STA_CHECK_CUDA(cudaMemcpyAsync(info_out, d.info, 4 * sizeof(double), cudaMemcpyDeviceToDevice, st));
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int sta_pg_plan_last_delta(const StaPgPlan* plan, double* delta_out, void* stream) {
  STA_REQUIRE(plan && delta_out, "null argument");
  STA_CHECK_CUDA(cudaMemcpyAsync(delta_out, plan->d.delta, sizeof(double) * 7 * plan->S.n, cudaMemcpyDeviceToDevice,
                                 static_cast<cudaStream_t>(stream)));
  return 0;
}

int sta_pg_group_plan_create(const StaPgPlan* const* plans, int G, StaPgGroupPlan** out) {
  STA_REQUIRE(out != nullptr, "null output pointer");
  *out = nullptr;
  STA_REQUIRE(plans != nullptr, "null plan table");
  STA_REQUIRE(G >= 1 && G <= SP_GROUP_MAX, "a group holds 1 to STA_PG_GROUP_MAX plans");
  for (int k = 0; k < G; ++k) {
    STA_REQUIRE(plans[k] != nullptr, "null plan");
    for (int j = 0; j < k; ++j)
      STA_REQUIRE(plans[j] != plans[k], "a plan is named twice in the group (its scratch would be shared)");
  }
  int dev = -1;
  STA_CHECK_CUDA(cudaGetDevice(&dev));
  for (int k = 0; k < G; ++k) STA_REQUIRE(plans[k]->device == dev, "a plan was created on another device");
  StaPgGroupPlan* gp = new StaPgGroupPlan();
  gp->device = dev;
  gp->plans.assign(plans, plans + G);
  // layout: members [G], descs [G], then each member's level table
  size_t off = align_up(sizeof(SpMember) * G);
  const size_t descs_off = off;
  off += align_up(sizeof(SpDesc) * G);
  std::vector<size_t> lvl_off(G);
  for (int k = 0; k < G; ++k) {
    const PgSymbolic& S = plans[k]->S;
    lvl_off[k] = off;
    off += align_up(sizeof(int4) * S.nlev);
    gp->nlev = std::max(gp->nlev, S.nlev);
    gp->max_edges = std::max(gp->max_edges, S.num_edges);
    gp->max_nodes = std::max(gp->max_nodes, S.num_nodes);
    gp->max_nnzb = std::max(gp->max_nnzb, static_cast<int>(S.nnzb()));
  }
  gp->bytes = off;
  gp->max_blk.assign(gp->nlev, 0);
  gp->max_col.assign(gp->nlev, 0);
  std::vector<char> host(off, 0);
  cudaError_t e = cudaMalloc(&gp->arena, off);
  char* base = static_cast<char*>(gp->arena);
  for (int k = 0; k < G && e == cudaSuccess; ++k) {
    const PgSymbolic& S = plans[k]->S;
    int4* lv = reinterpret_cast<int4*>(host.data() + lvl_off[k]);
    for (int l = 0; l < S.nlev; ++l) {
      lv[l] = make_int4(S.lvl_blk_ptr[l], S.lvl_blk_ptr[l + 1] - S.lvl_blk_ptr[l], S.lvl_col_ptr[l],
                        S.lvl_col_ptr[l + 1] - S.lvl_col_ptr[l]);
      gp->max_blk[l] = std::max(gp->max_blk[l], lv[l].y);
      gp->max_col[l] = std::max(gp->max_col[l], lv[l].w);
    }
    SpMember& m = reinterpret_cast<SpMember*>(host.data())[k];
    m.d = plans[k]->d;
    m.lvl = reinterpret_cast<const int4*>(base + lvl_off[k]);
    m.nlev = S.nlev;
    m.num_nodes = S.num_nodes;
    m.num_edges = S.num_edges;
    m.n7 = 7 * S.n;
    m.nnzb = static_cast<int>(S.nnzb());
  }
  if (e == cudaSuccess) e = cudaMemcpy(gp->arena, host.data(), off, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    set_last_error(std::string("sta_pg_group_plan_create: ") + cudaGetErrorString(e));
    sta_pg_group_plan_destroy(gp);
    return 1;
  }
  gp->members = reinterpret_cast<SpMember*>(base);
  gp->descs = reinterpret_cast<SpDesc*>(base + descs_off);
  *out = gp;
  return 0;
}

void sta_pg_group_plan_destroy(StaPgGroupPlan* gp) {
  if (!gp) return;
  if (gp->arena) {
    cudaDeviceSynchronize();
    cudaFree(gp->arena);
  }
  delete gp;
}

int sta_pg_group_plan_info(const StaPgGroupPlan* gp, int64_t* out4) {
  STA_REQUIRE(gp && out4, "null argument");
  out4[0] = static_cast<int64_t>(gp->plans.size());
  out4[1] = gp->nlev;
  out4[2] = group_launches(gp->nlev);
  out4[3] = static_cast<int64_t>(gp->bytes);
  return 0;
}

int sta_pose_graph_lm_step_sparse_group(const StaPgGroupPlan* gp, const StaPgSparseStep* steps, double dmin, double dmax,
                                        double* info_out, void* stream) {
  STA_REQUIRE(gp && steps && info_out, "null pointer");
  const int G = static_cast<int>(gp->plans.size());
  SpGroupParams p = {};
  int A = 0;
  for (int k = 0; k < G; ++k) {
    const StaPgSparseStep& q = steps[k];
    if (!q.active) continue;
    STA_REQUIRE(q.nodes && q.meas && q.weights && q.nodes_out, "null pointer in an active member");
    p.s[A++] = SpStepArgs{q.nodes, q.meas, q.weights, q.nodes_out, info_out + 4 * k, q.damping, k};
  }
  int dev = -1;
  STA_CHECK_CUDA(cudaGetDevice(&dev));
  STA_REQUIRE(dev == gp->device, "the group plan was created on another device");
  if (A == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const unsigned a = static_cast<unsigned>(A);
  SpDesc* descs = gp->descs;
  sp_group_setup_kernel<<<1, 32, 0, st>>>(p, A, gp->members, descs);
  sp_edge_group_kernel<<<dim3((gp->max_edges + 63) / 64, a), 64, 0, st>>>(descs, 0);
  sp_assemble_group_kernel<<<dim3(gp->max_nnzb, a), 64, 0, st>>>(descs, dmin, dmax);
  sp_loss_group_kernel<<<a, 256, 0, st>>>(descs, 0);
  for (int l = 0; l < gp->nlev; ++l) {
    if (l > 0) sp_update_group_kernel<<<dim3(gp->max_blk[l], a), 64, 0, st>>>(descs, l);  // leaves have no updates
    sp_factor_group_kernel<<<dim3(gp->max_col[l], a), 128, 0, st>>>(descs, l);
  }
  for (int l = 0; l < gp->nlev; ++l) sp_forward_group_kernel<<<dim3(gp->max_col[l], a), 32, 0, st>>>(descs, l);
  for (int l = gp->nlev - 1; l >= 0; --l) sp_backward_group_kernel<<<dim3(gp->max_col[l], a), 32, 0, st>>>(descs, l);
  sp_node_update_group_kernel<<<dim3((gp->max_nodes + 127) / 128, a), 128, 0, st>>>(descs);
  sp_edge_group_kernel<<<dim3((gp->max_edges + 63) / 64, a), 64, 0, st>>>(descs, 1);
  sp_loss_group_kernel<<<a, 256, 0, st>>>(descs, 1);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
