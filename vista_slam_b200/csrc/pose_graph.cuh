// Sim(3) device algebra and the per-edge / update / loss kernels of the pose-graph LM step, shared by the dense route
// (pose_graph.cu) and the block-sparse route (pose_graph_sparse.cu): the same residuals, Jacobians, update and losses on
// both.  Tangent order [tau | phi | sigma], Sim3 data (tx ty tz | qx qy qz qw | s) as PyPose stores it.
#pragma once
#include <math.h>

#include <cuda_runtime.h>

namespace sta {
namespace {

struct Sim3d {
  double t[3];
  double q[4];  // x, y, z, w
  double s;
};

__device__ __forceinline__ void quat_mul(const double* a, const double* b, double* o) {
  o[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  o[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  o[1] = a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0];
  o[2] = a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3];
}
__device__ __forceinline__ void quat_rot(const double* q, const double* v, double* o) {
  // v + 2 w (u x v) + 2 u x (u x v)
  const double cx = q[1] * v[2] - q[2] * v[1], cy = q[2] * v[0] - q[0] * v[2], cz = q[0] * v[1] - q[1] * v[0];
  const double dx = q[1] * cz - q[2] * cy, dy = q[2] * cx - q[0] * cz, dz = q[0] * cy - q[1] * cx;
  o[0] = v[0] + 2.0 * (q[3] * cx + dx);
  o[1] = v[1] + 2.0 * (q[3] * cy + dy);
  o[2] = v[2] + 2.0 * (q[3] * cz + dz);
}
__device__ __forceinline__ void quat_to_rot(const double* q, double* R) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w);     R[2] = 2 * (x * z + y * w);
  R[3] = 2 * (x * y + z * w);     R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
  R[6] = 2 * (x * z - y * w);     R[7] = 2 * (y * z + x * w);     R[8] = 1 - 2 * (x * x + y * y);
}
__device__ __forceinline__ Sim3d sim3_load(const float* p) {
  Sim3d X;
  X.t[0] = p[0]; X.t[1] = p[1]; X.t[2] = p[2];
  double n = 0.0;
  for (int i = 0; i < 4; ++i) { X.q[i] = p[3 + i]; n += X.q[i] * X.q[i]; }
  n = 1.0 / sqrt(n);
  for (int i = 0; i < 4; ++i) X.q[i] *= n;
  X.s = p[7];
  return X;
}
__device__ __forceinline__ Sim3d sim3_mul(const Sim3d& A, const Sim3d& B) {  // x -> s R x + t composition
  Sim3d C;
  double rt[3];
  quat_rot(A.q, B.t, rt);
  for (int i = 0; i < 3; ++i) C.t[i] = A.s * rt[i] + A.t[i];
  quat_mul(A.q, B.q, C.q);
  C.s = A.s * B.s;
  return C;
}
__device__ __forceinline__ Sim3d sim3_inv(const Sim3d& X) {
  Sim3d Y;
  Y.q[0] = -X.q[0]; Y.q[1] = -X.q[1]; Y.q[2] = -X.q[2]; Y.q[3] = X.q[3];
  Y.s = 1.0 / X.s;
  double rt[3];
  quat_rot(Y.q, X.t, rt);
  for (int i = 0; i < 3; ++i) Y.t[i] = -Y.s * rt[i];
  return Y;
}

// W = C I + A Phi + B Phi^2 = int_0^1 exp(u (sigma I + Phi)) du  (translation part of the Sim(3) exponential)
__device__ void w_coeffs(double sigma, double theta, double& C, double& A, double& B) {
  // int_0^1 e^{u sigma} u^k du = sum_n sigma^n / (n! (n + k + 1)): series below |sigma| = 1e-2 (the closed forms cancel)
  const double es = exp(sigma);
  const bool small_s = fabs(sigma) < 1e-2;
  const double s1 = sigma, s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2;
  C = small_s ? 1.0 + s1 / 2 + s2 / 6 + s3 / 24 + s4 / 120 : expm1(sigma) / sigma;
  if (theta < 1e-4) {  // theta^2 corrections (<= 4e-10) are far below the fp32 resolution of the inputs
    if (small_s) {
      A = 0.5 + s1 / 3 + s2 / 8 + s3 / 30 + s4 / 144;
      B = 1.0 / 6 + s1 / 8 + s2 / 20 + s3 / 72 + s4 / 336;
    } else {
      A = (es * (sigma - 1.0) + 1.0) / s2;
      B = (es * (s2 - 2.0 * sigma + 2.0) - 2.0) / (2.0 * s3);
    }
  } else {
    const double den = s2 + theta * theta, sn = sin(theta), cs = cos(theta);
    A = (es * (sigma * sn - theta * cs) + theta) / (theta * den);
    B = (C - (es * (sigma * cs + theta * sn) - sigma) / den) / (theta * theta);
  }
}
__device__ void w_matrix(const double* phi, double sigma, double* W) {
  const double th = sqrt(phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2]);
  double C, A, B;
  w_coeffs(sigma, th, C, A, B);
  const double x = phi[0], y = phi[1], z = phi[2];
  // Phi = [[0,-z,y],[z,0,-x],[-y,x,0]];  Phi^2 = phi phi^T - |phi|^2 I
  const double t2 = th * th;
  W[0] = C + B * (x * x - t2); W[1] = -A * z + B * x * y;   W[2] = A * y + B * x * z;
  W[3] = A * z + B * x * y;    W[4] = C + B * (y * y - t2); W[5] = -A * x + B * y * z;
  W[6] = -A * y + B * x * z;   W[7] = A * x + B * y * z;    W[8] = C + B * (z * z - t2);
}
__device__ void sim3_log(const Sim3d& X, double* xi) {
  double q[4] = {X.q[0], X.q[1], X.q[2], X.q[3]};
  if (q[3] < 0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
  const double k = (n < 1e-12) ? 2.0 : 2.0 * atan2(n, q[3]) / n;
  xi[3] = k * q[0]; xi[4] = k * q[1]; xi[5] = k * q[2];
  xi[6] = log(X.s);
  double W[9];
  w_matrix(xi + 3, xi[6], W);
  // tau = W^-1 t (3x3 inverse by cofactors)
  const double c0 = W[4] * W[8] - W[5] * W[7], c1 = W[5] * W[6] - W[3] * W[8], c2 = W[3] * W[7] - W[4] * W[6];
  const double det = W[0] * c0 + W[1] * c1 + W[2] * c2, id = 1.0 / det;
  const double* t = X.t;
  xi[0] = id * (c0 * t[0] + (W[2] * W[7] - W[1] * W[8]) * t[1] + (W[1] * W[5] - W[2] * W[4]) * t[2]);
  xi[1] = id * (c1 * t[0] + (W[0] * W[8] - W[2] * W[6]) * t[1] + (W[2] * W[3] - W[0] * W[5]) * t[2]);
  xi[2] = id * (c2 * t[0] + (W[1] * W[6] - W[0] * W[7]) * t[1] + (W[0] * W[4] - W[1] * W[3]) * t[2]);
}
__device__ Sim3d sim3_exp(const double* xi) {
  Sim3d X;
  const double* phi = xi + 3;
  const double th = sqrt(phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2]);
  const double k = (th < 1e-8) ? 0.5 - th * th / 48.0 : sin(0.5 * th) / th;
  X.q[0] = k * phi[0]; X.q[1] = k * phi[1]; X.q[2] = k * phi[2]; X.q[3] = cos(0.5 * th);
  X.s = exp(xi[6]);
  double W[9];
  w_matrix(phi, xi[6], W);
  for (int i = 0; i < 3; ++i) X.t[i] = W[3 * i] * xi[0] + W[3 * i + 1] * xi[1] + W[3 * i + 2] * xi[2];
  return X;
}

// 7x7 helpers (row-major)
__device__ void mat7_mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < 7; ++i)
    for (int j = 0; j < 7; ++j) {
      double s = 0.0;
      for (int k = 0; k < 7; ++k) s = fma(A[7 * i + k], B[7 * k + j], s);
      C[7 * i + j] = s;
    }
}
// Ad_X, tangent order [tau | phi | sigma]
__device__ void sim3_adj(const Sim3d& X, double* A) {
  double R[9];
  quat_to_rot(X.q, R);
  for (int i = 0; i < 49; ++i) A[i] = 0.0;
  const double* t = X.t;
  const double H[9] = {0, -t[2], t[1], t[2], 0, -t[0], -t[1], t[0], 0};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      A[7 * i + j] = X.s * R[3 * i + j];
      A[7 * i + 3 + j] = H[3 * i] * R[j] + H[3 * i + 1] * R[3 + j] + H[3 * i + 2] * R[6 + j];
      A[7 * (3 + i) + 3 + j] = R[3 * i + j];
    }
  for (int i = 0; i < 3; ++i) A[7 * i + 6] = -t[i];
  A[48] = 1.0;
}
// ad_xi
__device__ void sim3_ad(const double* xi, double* a) {
  for (int i = 0; i < 49; ++i) a[i] = 0.0;
  const double* tau = xi;
  const double* phi = xi + 3;
  const double Hp[9] = {0, -phi[2], phi[1], phi[2], 0, -phi[0], -phi[1], phi[0], 0};
  const double Ht[9] = {0, -tau[2], tau[1], tau[2], 0, -tau[0], -tau[1], tau[0], 0};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      a[7 * i + j] = Hp[3 * i + j] + (i == j ? xi[6] : 0.0);
      a[7 * i + 3 + j] = Ht[3 * i + j];
      a[7 * (3 + i) + 3 + j] = Hp[3 * i + j];
    }
  for (int i = 0; i < 3; ++i) a[7 * i + 6] = -tau[i];
}
// P = phi_1(M) = sum_n M^n / (n+1)!  by scaling and squaring: phi_1(2M) = (exp(M) + I) phi_1(M) / 2, exp(2M) = exp(M)^2
__device__ void phi1_7(const double* M, double* P) {
  double nrm = 0.0;
  for (int i = 0; i < 7; ++i) {
    double s = 0.0;
    for (int j = 0; j < 7; ++j) s += fabs(M[7 * i + j]);
    nrm = fmax(nrm, s);
  }
  int k = 0;
  double sc = 1.0;
  while (nrm * sc > 0.5 && k < 30) { sc *= 0.5; ++k; }
  double Ms[49], T[49], U[49], E[49];
  for (int i = 0; i < 49; ++i) { Ms[i] = M[i] * sc; P[i] = 0.0; T[i] = 0.0; }
  for (int i = 0; i < 7; ++i) { P[8 * i] = 1.0; T[8 * i] = 1.0; }
  for (int n = 1; n <= 14; ++n) {  // T = Ms^n / (n+1)!
    mat7_mul(T, Ms, U);
    const double f = 1.0 / (n + 1);
    for (int i = 0; i < 49; ++i) { T[i] = U[i] * f; P[i] += T[i]; }
  }
  mat7_mul(Ms, P, E);  // exp(Ms) = I + Ms phi_1(Ms)
  for (int i = 0; i < 7; ++i) E[8 * i] += 1.0;
  for (int s = 0; s < k; ++s) {
    for (int i = 0; i < 49; ++i) T[i] = 0.5 * E[i];
    for (int i = 0; i < 7; ++i) T[8 * i] += 0.5;
    mat7_mul(T, P, U);
    for (int i = 0; i < 49; ++i) P[i] = U[i];
    mat7_mul(E, E, U);
    for (int i = 0; i < 49; ++i) E[i] = U[i];
  }
}
// in-place Gauss-Jordan inverse with partial pivoting; returns false if singular
__device__ bool mat7_inv(double* A, double* Inv) {
  for (int i = 0; i < 49; ++i) Inv[i] = 0.0;
  for (int i = 0; i < 7; ++i) Inv[8 * i] = 1.0;
  for (int c = 0; c < 7; ++c) {
    int piv = c;
    double best = fabs(A[7 * c + c]);
    for (int r = c + 1; r < 7; ++r)
      if (fabs(A[7 * r + c]) > best) { best = fabs(A[7 * r + c]); piv = r; }
    if (best < 1e-300) return false;
    if (piv != c)
      for (int j = 0; j < 7; ++j) {
        double t = A[7 * c + j]; A[7 * c + j] = A[7 * piv + j]; A[7 * piv + j] = t;
        t = Inv[7 * c + j]; Inv[7 * c + j] = Inv[7 * piv + j]; Inv[7 * piv + j] = t;
      }
    const double d = 1.0 / A[7 * c + c];
    for (int j = 0; j < 7; ++j) { A[7 * c + j] *= d; Inv[7 * c + j] *= d; }
    for (int r = 0; r < 7; ++r) {
      if (r == c) continue;
      const double f = A[7 * r + c];
      if (f == 0.0) continue;
      for (int j = 0; j < 7; ++j) { A[7 * r + j] -= f * A[7 * c + j]; Inv[7 * r + j] -= f * Inv[7 * c + j]; }
    }
  }
  return true;
}

// ---------------------------------------------------------------------------
// one thread per edge: residual (and, if J != null, dr/d delta_j; dr/d delta_i = -that)
// ---------------------------------------------------------------------------
// (the bodies are device functions so that the dense route's group kernels run the same code per graph)
__device__ __forceinline__ void pg_edge(int e, const float* __restrict__ nodes, const long long* __restrict__ edges,
                                        const float* __restrict__ meas, const int* __restrict__ opt_map, int E,
                                        double* __restrict__ r_out, double* __restrict__ J_out, int* __restrict__ related) {
  if (e >= E) return;
  const long long i = edges[2 * e], j = edges[2 * e + 1];
  const bool rel = opt_map[i] >= 0 || opt_map[j] >= 0;  // pose_graph.py:150-154
  related[e] = rel ? 1 : 0;
  if (!rel) {
    for (int k = 0; k < 7; ++k) r_out[7 * e + k] = 0.0;
    return;
  }
  const Sim3d T = sim3_load(meas + 8 * e), Xi = sim3_load(nodes + 8 * i), Xj = sim3_load(nodes + 8 * j);
  const Sim3d A = sim3_mul(T, sim3_inv(Xi));
  const Sim3d Err = sim3_mul(A, Xj);
  double r[7];
  sim3_log(Err, r);
  for (int k = 0; k < 7; ++k) r_out[7 * e + k] = r[k];
  if (J_out == nullptr) return;
  double ad[49], Jl[49], Jinv[49], Ad[49], J[49];
  sim3_ad(r, ad);
  phi1_7(ad, Jl);
  if (!mat7_inv(Jl, Jinv)) {
    for (int k = 0; k < 49; ++k) Jinv[k] = (k % 8 == 0) ? 1.0 : 0.0;
  }
  sim3_adj(A, Ad);
  mat7_mul(Jinv, Ad, J);
  for (int k = 0; k < 49; ++k) J_out[49 * e + k] = J[k];
}
__global__ void __launch_bounds__(64)
pg_edge_kernel(const float* __restrict__ nodes, const long long* __restrict__ edges, const float* __restrict__ meas,
               const int* __restrict__ opt_map, int E, double* __restrict__ r_out, double* __restrict__ J_out,
               int* __restrict__ related) {
  pg_edge(blockIdx.x * blockDim.x + threadIdx.x, nodes, edges, meas, opt_map, E, r_out, J_out, related);
}

// nodes_out = Exp(delta_a) * node for optimised nodes (LieTensor.add_), copy for fixed ones
__device__ __forceinline__ void pg_update(int v, const float* __restrict__ nodes, const int* __restrict__ opt_map,
                                          const double* __restrict__ delta, int num_nodes, float* __restrict__ out) {
  if (v >= num_nodes) return;
  const int a = opt_map[v];
  if (a < 0) {
    for (int k = 0; k < 8; ++k) out[8 * v + k] = nodes[8 * v + k];
    return;
  }
  const Sim3d X = sim3_load(nodes + 8 * v);
  const Sim3d Y = sim3_mul(sim3_exp(delta + 7 * a), X);
  const double qn = 1.0 / sqrt(Y.q[0] * Y.q[0] + Y.q[1] * Y.q[1] + Y.q[2] * Y.q[2] + Y.q[3] * Y.q[3]);
  for (int k = 0; k < 3; ++k) out[8 * v + k] = static_cast<float>(Y.t[k]);
  for (int k = 0; k < 4; ++k) out[8 * v + 3 + k] = static_cast<float>(Y.q[k] * qn);
  out[8 * v + 7] = static_cast<float>(Y.s);
}
__global__ void pg_update_kernel(const float* __restrict__ nodes, const int* __restrict__ opt_map, const double* __restrict__ delta,
                                 int num_nodes, float* __restrict__ out) {
  pg_update(blockIdx.x * blockDim.x + threadIdx.x, nodes, opt_map, delta, num_nodes, out);
}

// loss = sum_e r_e^T W_e r_e (related edges), |delta|_2 -> info; fixed-order reduction in one CTA of 256 threads
__device__ __forceinline__ void pg_loss(const double* __restrict__ r, const float* __restrict__ weights,
                                        const int* __restrict__ related, int E, const double* __restrict__ delta, int n7,
                                        double* __restrict__ info, int slot) {
  __shared__ double red[256];
  double s = 0.0;
  for (int e = threadIdx.x; e < E; e += 256) {
    if (!related[e]) continue;
    for (int k = 0; k < 7; ++k) s += r[7ll * e + k] * r[7ll * e + k] * static_cast<double>(weights[7 * e + k]);
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) info[slot] = red[0];
  if (delta != nullptr) {
    __syncthreads();
    double d = 0.0;
    for (int i = threadIdx.x; i < n7; i += 256) d += delta[i] * delta[i];
    red[threadIdx.x] = d;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
      __syncthreads();
    }
    if (threadIdx.x == 0) info[2] = sqrt(red[0]);
  }
}
__global__ void __launch_bounds__(256) pg_loss_kernel(const double* __restrict__ r, const float* __restrict__ weights,
                                                      const int* __restrict__ related, int E, const double* __restrict__ delta,
                                                      int n7, double* __restrict__ info, int slot) {
  pg_loss(r, weights, related, E, delta, n7, info, slot);
}

}  // namespace
}  // namespace sta
