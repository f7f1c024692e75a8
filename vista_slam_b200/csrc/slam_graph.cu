// Device-resident pose graph of OnlineSLAM (vista_slam/slam.py:20-447 over vista_slam/pose_graph.py:5-54): the node
// and edge tables, the per-node depth / confidence / intrinsics store, the per-view best node, the graph update of one
// keyframe (connect_view_i_j, slam.py:191-241, for all its kept edges) and the per-view gather + world point cloud of
// save_data_all / get_view (slam.py:299-412).
//
// The reference keeps the maps on the host (pose_graph.py:37) and reads a confidence mean back per node (:41) and per
// scale edge (slam.py:227); here everything stays on the device and a keyframe costs two launches with no host
// synchronisation:
//   graph_ingest_kernel  copies the 2n maps of the n kept edges into the node store and runs the 2n - 1 scale-edge
//                        reductions (pointmap.cuh, the reduction of sta_depth_scale);
//   graph_link_kernel    finishes the reductions, then one thread walks the edges in the reference's order: node tables,
//                        best node (strict > against -100), rotation -> quaternion, node poses and edge records.
#include <string>

#include "../../include/sta_b200.h"
#include "cloud.cuh"
#include "host_util.h"
#include "pointmap.cuh"

struct StaGraph {
  int max_nodes = 0, max_edges = 0, max_views = 0, H = 0, W = 0;
  float* pose = nullptr;        // [max_nodes][8]  tx ty tz | qx qy qz qw | s
  float* depth = nullptr;       // [max_nodes][H][W]
  float* conf = nullptr;        // [max_nodes][H][W]
  float* intri = nullptr;       // [max_nodes][3][3]
  float* cmean = nullptr;       // [max_nodes]
  int64_t* node_view = nullptr;   // [max_nodes]
  int64_t* node_cview = nullptr;  // [max_nodes]
  int64_t* best_node = nullptr;   // [max_views]
  float* best_mean = nullptr;     // [max_views]
  int64_t* edges = nullptr;       // [max_edges][2]
  float* meas = nullptr;          // [max_edges][8]
  float* weight = nullptr;        // [max_edges][7]
  double* partial = nullptr;      // [STA_GRAPH_MAX_KEYFRAME_EDGES * 2][kStatBlocks][kStatVals]
  int* flags_host = nullptr;      // mapped host word, written by the link kernel
  int* flags_dev = nullptr;       // its device alias
};

namespace sta {
namespace {

constexpr int kMaxKf = STA_GRAPH_MAX_KEYFRAME_EDGES;

struct KfArgs {
  int n, n_scale, node0, edge0, view;
  long long hw;
  int cand[kMaxKf];         // candidate row of edge k in pose / pose_conf
  long long js[kMaxKf];     // view j of edge k
  int first_j[kMaxKf];      // first node of view j when edge k is inserted, -1 if it has none
  const float* pose;        // [*][4][4]
  const float* pconf;       // [*]
  const float* confs;       // [2][n][H][W]
  const float* depths;      // [2][n][H][W]
  const float* intri;       // [n][3][3]
  const float* cmean;       // [2][n]
};

// Map of node `slot`: the keyframe's own nodes node0 + 2k + r are row r of edge k in the inputs, older ones are in
// the store.
__device__ __forceinline__ const float* map_of(const KfArgs& a, const float* store, const float* in, int slot) {
  if (slot >= a.node0) {
    const int d = slot - a.node0;
    return in + (static_cast<long long>(d & 1) * a.n + (d >> 1)) * a.hw;
  }
  return store + static_cast<long long>(slot) * a.hw;
}

// Scale edge s of the keyframe, in edge order: (new node, first node of its view).
__device__ void scale_edge(const KfArgs& a, int s, int* nnew, int* nother) {
  int c = 0;
  for (int k = 0; k < a.n; ++k) {
    if (k > 0) {
      if (c++ == s) { *nnew = a.node0 + 2 * k; *nother = a.node0; return; }
    }
    if (a.first_j[k] >= 0) {
      if (c++ == s) { *nnew = a.node0 + 2 * k + 1; *nother = a.first_j[k]; return; }
    }
  }
}

// grid (kStatBlocks, n_scale + 2n), 256 threads
__global__ void __launch_bounds__(256) graph_ingest_kernel(StaGraph g, KfArgs a) {
  const int y = blockIdx.y;
  if (y < a.n_scale) {
    int nn = 0, no = 0;
    scale_edge(a, y, &nn, &no);
    // estimate_scale_with_depth_and_confidence(depth, depth_other, conf, conf_other), slam.py:224
    scale_partial(map_of(a, g.depth, a.depths, nn), map_of(a, g.depth, a.depths, no), map_of(a, g.conf, a.confs, nn),
                  map_of(a, g.conf, a.confs, no), a.hw, blockIdx.x,
                  g.partial + (static_cast<long long>(y) * kStatBlocks + blockIdx.x) * kStatVals);
    return;
  }
  const int slot = a.node0 + (y - a.n_scale);
  const float* d = map_of(a, g.depth, a.depths, slot);
  const float* c = map_of(a, g.conf, a.confs, slot);
  float* dd = g.depth + static_cast<long long>(slot) * a.hw;
  float* cd = g.conf + static_cast<long long>(slot) * a.hw;
  for (long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x; i < a.hw; i += kStatBlocks * 256) {
    dd[i] = d[i];
    cd[i] = c[i];
  }
  if (blockIdx.x == 0 && threadIdx.x < 9)
    g.intri[slot * 9 + threadIdx.x] = a.intri[((slot - a.node0) >> 1) * 9 + threadIdx.x];
}

// Sim(3) a * b in the [t | q | s] layout; the quaternion is kept with w >= 0.
__device__ void sim3_mul(const float* a, const float* b, float* o) {
  const float ax = a[3], ay = a[4], az = a[5], aw = a[6];
  const float bx = b[3], by = b[4], bz = b[5], bw = b[6];
  // t = t_a + s_a R_a t_b, with R_a t_b = t_b + 2 w (u x t_b) + 2 u x (u x t_b)
  const float tx = b[0], ty = b[1], tz = b[2];
  const float cx = ay * tz - az * ty, cy = az * tx - ax * tz, cz = ax * ty - ay * tx;
  const float rx = tx + 2.f * (aw * cx + ay * cz - az * cy);
  const float ry = ty + 2.f * (aw * cy + az * cx - ax * cz);
  const float rz = tz + 2.f * (aw * cz + ax * cy - ay * cx);
  float q[4] = {aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz};
  const float sg = q[3] < 0.f ? -1.f : 1.f;
  o[0] = a[0] + a[7] * rx;
  o[1] = a[1] + a[7] * ry;
  o[2] = a[2] + a[7] * rz;
  for (int i = 0; i < 4; ++i) o[3 + i] = sg * q[i];
  o[7] = a[7] * b[7];
}

// Rotation (row-major 3x3 inside a 4x4) -> unit quaternion (x, y, z, w), w >= 0 (Shepperd's method, fp64).
// Returns false when R is not orthonormal with det +1 to 1e-3 (what pp.mat2SE3(atol=1e-3) refuses).
__device__ bool rot_to_quat(const float* M, float* q) {
  double R[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R[r][c] = M[r * 4 + c];
  bool ok = true;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      const double d = R[r][0] * R[c][0] + R[r][1] * R[c][1] + R[r][2] * R[c][2] - (r == c ? 1.0 : 0.0);
      ok = ok && fabs(d) <= 1e-3;
    }
  const double det = R[0][0] * (R[1][1] * R[2][2] - R[1][2] * R[2][1]) - R[0][1] * (R[1][0] * R[2][2] - R[1][2] * R[2][0]) +
                     R[0][2] * (R[1][0] * R[2][1] - R[1][1] * R[2][0]);
  ok = ok && fabs(det - 1.0) <= 1e-3;
  double x[4];
  const double t = R[0][0] + R[1][1] + R[2][2];
  if (t > 0) {
    const double s = sqrt(t + 1.0) * 2;
    x[0] = (R[2][1] - R[1][2]) / s; x[1] = (R[0][2] - R[2][0]) / s; x[2] = (R[1][0] - R[0][1]) / s; x[3] = 0.25 * s;
  } else {
    int i = 0;
    if (R[1][1] > R[i][i]) i = 1;
    if (R[2][2] > R[i][i]) i = 2;
    const int j = (i + 1) % 3, k = (i + 2) % 3;
    const double s = sqrt(1.0 + R[i][i] - R[j][j] - R[k][k]) * 2;
    x[i] = 0.25 * s;
    x[j] = (R[j][i] + R[i][j]) / s;
    x[k] = (R[k][i] + R[i][k]) / s;
    x[3] = (R[k][j] - R[j][k]) / s;
  }
  const double sg = x[3] < 0 ? -1.0 : 1.0;
  const double nrm = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2] + x[3] * x[3]);
  for (int e = 0; e < 4; ++e) q[e] = static_cast<float>(sg * x[e] / nrm);
  return ok;
}

__device__ void put_edge(const StaGraph& g, int e, long long ni, long long nj, const float* m8, const float* w7) {
  g.edges[2 * e] = ni;
  g.edges[2 * e + 1] = nj;
  for (int i = 0; i < 8; ++i) g.meas[e * 8 + i] = m8[i];
  for (int i = 0; i < 7; ++i) g.weight[e * 7 + i] = w7[i];
}

// one block of 64 threads
__global__ void graph_link_kernel(StaGraph g, KfArgs a) {
  __shared__ float sc[2 * kMaxKf][2];
  if (threadIdx.x < a.n_scale)
    scale_finalize(g.partial + static_cast<long long>(threadIdx.x) * kStatBlocks * kStatVals, a.hw, sc[threadIdx.x]);
  __syncthreads();
  if (threadIdx.x != 0) return;
  int e = a.edge0, s = 0;
  for (int k = 0; k < a.n; ++k) {
    for (int r = 0; r < 2; ++r) {  // add_node(i), its scale edge, add_node(j), its scale edge (slam.py:210-232)
      const int slot = a.node0 + 2 * k + r;
      const long long v = r ? a.js[k] : a.view;
      g.node_view[slot] = v;
      g.node_cview[slot] = r ? a.view : a.js[k];
      const float m = a.cmean[r * a.n + k];
      g.cmean[slot] = m;
      if (m > g.best_mean[v]) {  // pose_graph.py:42: strict, so the first node wins a tie
        g.best_mean[v] = m;
        g.best_node[v] = slot;
      }
      const int other = r ? a.first_j[k] : (k > 0 ? a.node0 : -1);
      if (other >= 0) {
        const float sim3[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 1.f, sc[s][0]};
        const float w[7] = {2.f, 2.f, 2.f, 2.f, 2.f, 2.f, sc[s][1]};  // PoseGraphEdges.id_pose_conf = 2.0
        ++s;
        put_edge(g, e++, slot, other, sim3, w);
        sim3_mul(g.pose + other * 8, sim3, g.pose + slot * 8);
      }
    }
    const float* M = a.pose + a.cand[k] * 16;
    float sim3[8] = {M[3], M[7], M[11], 0.f, 0.f, 0.f, 1.f, 1.f};
    if (!rot_to_quat(M, sim3 + 3)) *reinterpret_cast<volatile int*>(g.flags_dev) |= STA_GRAPH_FLAG_NOT_SO3;
    const int ni = a.node0 + 2 * k, nj = ni + 1;
    if (k == 0) sim3_mul(g.pose + nj * 8, sim3, g.pose + ni * 8);  // view i is new at its first node (slam.py:234-236)
    const float c = a.pconf[a.cand[k]];
    const float w[7] = {c, c, c, c, c, c, c};
    put_edge(g, e++, ni, nj, sim3, w);
  }
  __threadfence_system();
}

// Triples (node, parent, edge) of one replay launch: 256 x 12 bytes keeps the parameters under 4 KB.
constexpr int kReplayChunk = 256;
struct ReplayArgs {
  int count;
  int t[kReplayChunk][3];
};

// one thread: pose[node] = pose[parent] * meas[edge] for each triple in order, through graph_link_kernel's sim3_mul, so
// a node re-derived from the same parent pose and measurement gets the bits its insertion would have given it
__global__ void __launch_bounds__(32) graph_replay_kernel(float* pose, const float* meas, ReplayArgs a) {
  if (threadIdx.x != 0) return;
  for (int t = 0; t < a.count; ++t) {
    const int* r = a.t[t];
    sim3_mul(pose + static_cast<long long>(r[1]) * 8, meas + static_cast<long long>(r[2]) * 8,
             pose + static_cast<long long>(r[0]) * 8);
  }
}

// grid-stride over max(max_nodes, max_edges, max_views): the state of PoseGraphNodes/Edges.reset (pose_graph.py:19-54)
__global__ void graph_reset_kernel(StaGraph g) {
  const long long n = max(max(g.max_nodes, g.max_edges), g.max_views);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (i < g.max_nodes) {
      for (int c = 0; c < 8; ++c) g.pose[i * 8 + c] = (c == 6 || c == 7) ? 1.f : 0.f;
      g.node_view[i] = -1;
      g.node_cview[i] = -1;
      g.cmean[i] = 0.f;
    }
    if (i < g.max_edges) {
      for (int c = 0; c < 8; ++c) g.meas[i * 8 + c] = (c == 6 || c == 7) ? 1.f : 0.f;
      for (int c = 0; c < 7; ++c) g.weight[i * 7 + c] = 1.f;
      g.edges[2 * i] = -1;
      g.edges[2 * i + 1] = -1;
    }
    if (i < g.max_views) {
      g.best_node[i] = -1;
      g.best_mean[i] = -100.f;
    }
  }
}

// ---- export ----

// grid (H, V), 256 threads: view v = view0 + blockIdx.y through its best node; row blockIdx.y of depth / conf, the row's
// count of conf > thres, and (row 0) the 4x4 pose with the scale dropped, the scale and the intrinsics.
__global__ void __launch_bounds__(256)
export_gather_kernel(StaGraph g, int view0, float thres, float* pose_out, float* scale_out, float* depth_out, float* conf_out,
                     float* intri_out, int* counts) {
  const int v = blockIdx.y, row = blockIdx.x;
  const long long b = g.best_node[view0 + v];
  const int W = g.W;
  const long long hw = static_cast<long long>(g.H) * W;
  const float* dsrc = g.depth + b * hw + static_cast<long long>(row) * W;
  const float* csrc = g.conf + b * hw + static_cast<long long>(row) * W;
  int cnt = 0;
  for (int x = threadIdx.x; x < W; x += 256) {
    const float c = csrc[x];
    if (depth_out) depth_out[v * hw + static_cast<long long>(row) * W + x] = dsrc[x];
    if (conf_out) conf_out[v * hw + static_cast<long long>(row) * W + x] = c;
    cnt += c > thres;
  }
  if (counts) {
    const int t = block_count_256(cnt);
    if (threadIdx.x == 0) counts[static_cast<long long>(v) * g.H + row] = t;
  }
  if (row == 0 && threadIdx.x == 0) {
    const float* p = g.pose + b * 8;
    const float x = p[3], y = p[4], z = p[5], w = p[6];  // LieTensor.rotation().matrix()
    const float R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                        2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                        2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
    float* P = pose_out + v * 16;
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) P[r * 4 + c] = R[r * 3 + c];
      P[r * 4 + 3] = p[r];
    }
    P[12] = 0.f; P[13] = 0.f; P[14] = 0.f; P[15] = 1.f;
    scale_out[v] = p[7];
    for (int i = 0; i < 9; ++i) intri_out[v * 9 + i] = g.intri[b * 9 + i];
  }
}

// grid (H, V), 256 threads: the points of row blockIdx.x of view blockIdx.y with conf > thres, in column order, at the
// row's offset: world = R (K^-1 [x y 1]^T depth s) + t, colour = (img + 1) / 2.
__global__ void __launch_bounds__(256)
export_scatter_kernel(StaGraph g, float thres, const float* pose_out, const float* scale_out, const float* intri_out,
                      const float* depth_out, const float* conf_out, const float* imgs, const long long* offsets,
                      float* points, float* colors) {
  const int v = blockIdx.y, row = blockIdx.x, W = g.W;
  const long long hw = static_cast<long long>(g.H) * W;
  const float* P = pose_out + v * 16;
  float Ki[9];
  inv3_f32(intri_out + v * 9, Ki);
  const float s = scale_out[v];
  const float* crow = conf_out + v * hw + static_cast<long long>(row) * W;
  const float* drow = depth_out + v * hw + static_cast<long long>(row) * W;
  row_compact_256(W, offsets[static_cast<long long>(v) * g.H + row], [&](int x) { return crow[x] > thres; },
                  [&](int x, long long o) {
                    unproject_f32(Ki, P, static_cast<float>(x), static_cast<float>(row), drow[x] * s, points + o * 3);
                    for (int c = 0; c < 3; ++c)
                      colors[o * 3 + c] = (imgs[(static_cast<long long>(v) * 3 + c) * hw + static_cast<long long>(row) * W + x] + 1.f) / 2.f;
                  });
}

}  // namespace
}  // namespace sta

using namespace sta;

extern "C" {

int sta_graph_create(int max_nodes, int max_edges, int max_views, int H, int W, StaGraph** out) {
  STA_REQUIRE(out != nullptr, "null output pointer");
  *out = nullptr;
  STA_REQUIRE(max_nodes > 0 && max_edges > 0 && max_views > 0 && H > 0 && W > 0, "capacities and map size must be positive");
  STA_REQUIRE(static_cast<long long>(H) * W < (1ll << 30) && H <= 65535, "map too large");
  StaGraph* g = new StaGraph();
  g->max_nodes = max_nodes;
  g->max_edges = max_edges;
  g->max_views = max_views;
  g->H = H;
  g->W = W;
  const size_t hw = static_cast<size_t>(H) * W;
  cudaError_t e = cudaSuccess;
  auto take = [&](auto** p, size_t bytes) {
    if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(p), bytes);
  };
  take(&g->pose, sizeof(float) * 8 * max_nodes);
  take(&g->depth, sizeof(float) * hw * max_nodes);
  take(&g->conf, sizeof(float) * hw * max_nodes);
  take(&g->intri, sizeof(float) * 9 * max_nodes);
  take(&g->cmean, sizeof(float) * max_nodes);
  take(&g->node_view, sizeof(int64_t) * max_nodes);
  take(&g->node_cview, sizeof(int64_t) * max_nodes);
  take(&g->best_node, sizeof(int64_t) * max_views);
  take(&g->best_mean, sizeof(float) * max_views);
  take(&g->edges, sizeof(int64_t) * 2 * max_edges);
  take(&g->meas, sizeof(float) * 8 * max_edges);
  take(&g->weight, sizeof(float) * 7 * max_edges);
  take(&g->partial, sizeof(double) * 2 * kMaxKf * kStatBlocks * kStatVals);
  if (e == cudaSuccess) e = cudaHostAlloc(reinterpret_cast<void**>(&g->flags_host), sizeof(int), cudaHostAllocMapped);
  if (e == cudaSuccess) {
    *g->flags_host = 0;
    e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&g->flags_dev), g->flags_host, 0);
  }
  if (e == cudaSuccess) {
    graph_reset_kernel<<<256, 256>>>(*g);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    set_last_error(std::string("sta_graph_create: ") + cudaGetErrorString(e));
    sta_graph_destroy(g);
    return 1;
  }
  *out = g;
  return 0;
}

void sta_graph_destroy(StaGraph* g) {
  if (!g) return;
  cudaDeviceSynchronize();
  void* bufs[] = {g->pose, g->depth, g->conf, g->intri, g->cmean, g->node_view, g->node_cview, g->best_node, g->best_mean,
                  g->edges, g->meas, g->weight, g->partial};
  for (void* p : bufs)
    if (p) cudaFree(p);
  if (g->flags_host) cudaFreeHost(g->flags_host);
  delete g;
}

int sta_graph_tables(const StaGraph* g, void** out12) {
  STA_REQUIRE(g != nullptr && out12 != nullptr, "null argument");
  void* t[12] = {g->pose, g->depth, g->conf, g->intri, g->cmean, g->node_view, g->node_cview, g->best_node, g->best_mean,
                 g->edges, g->meas, g->weight};
  for (int i = 0; i < 12; ++i) out12[i] = t[i];
  return 0;
}

int sta_graph_reset(StaGraph* g, void* stream) {
  STA_REQUIRE(g != nullptr, "null graph");
  graph_reset_kernel<<<256, 256, 0, static_cast<cudaStream_t>(stream)>>>(*g);
  STA_CHECK_CUDA(cudaGetLastError());
  *g->flags_host = 0;
  return 0;
}

int sta_graph_flags(const StaGraph* g, int* flags_out) {
  STA_REQUIRE(g != nullptr && flags_out != nullptr, "null argument");
  *flags_out = *reinterpret_cast<volatile int*>(g->flags_host);
  return 0;
}

int sta_graph_add_keyframe(StaGraph* g, int view, int n, const int64_t* js_host, const int* cand_host,
                           const int* first_j_host, int node0, int edge0, int H, int W, const float* pose_dev,
                           const float* pose_conf_dev, const float* confs_dev, const float* depths_dev, const float* intri_dev,
                           const float* conf_mean_dev, void* stream) {
  STA_REQUIRE(g != nullptr && js_host && cand_host && first_j_host, "null argument");
  STA_REQUIRE(n >= 1 && n <= kMaxKf, "1 to STA_GRAPH_MAX_KEYFRAME_EDGES kept edges per keyframe");
  STA_REQUIRE(H == g->H && W == g->W, "map size differs from the graph's");
  STA_REQUIRE(pose_dev && pose_conf_dev && confs_dev && depths_dev && intri_dev && conf_mean_dev, "null device input");
  STA_REQUIRE(on_device(pose_dev) && on_device(pose_conf_dev) && on_device(confs_dev) && on_device(depths_dev) &&
                  on_device(intri_dev) && on_device(conf_mean_dev),
              "inputs must be device memory");
  STA_REQUIRE(view >= 0 && view < g->max_views, "view index out of range");
  KfArgs a = {};
  a.n = n;
  a.view = view;
  a.node0 = node0;
  a.edge0 = edge0;
  a.hw = static_cast<long long>(H) * W;
  int n_scale = 0;
  for (int k = 0; k < n; ++k) {
    STA_REQUIRE(js_host[k] >= 0 && js_host[k] < view, "j must be an earlier view");
    STA_REQUIRE(cand_host[k] >= 0, "negative candidate index");
    STA_REQUIRE(first_j_host[k] >= -1 && first_j_host[k] < node0 + 2 * k, "first node of view j is not in the graph");
    a.js[k] = js_host[k];
    a.cand[k] = cand_host[k];
    a.first_j[k] = first_j_host[k];
    n_scale += (k > 0) + (first_j_host[k] >= 0);
  }
  a.n_scale = n_scale;
  STA_REQUIRE(node0 >= 0 && static_cast<long long>(node0) + 2 * n <= g->max_nodes, "node capacity exceeded");
  STA_REQUIRE(edge0 >= 0 && static_cast<long long>(edge0) + n_scale + n <= g->max_edges, "edge capacity exceeded");
  a.pose = pose_dev;
  a.pconf = pose_conf_dev;
  a.confs = confs_dev;
  a.depths = depths_dev;
  a.intri = intri_dev;
  a.cmean = conf_mean_dev;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  graph_ingest_kernel<<<dim3(kStatBlocks, n_scale + 2 * n), 256, 0, st>>>(*g, a);
  STA_CHECK_CUDA(cudaGetLastError());
  graph_link_kernel<<<1, 64, 0, st>>>(*g, a);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int sta_graph_replay_nodes(StaGraph* g, int count, const int* triples_host, void* stream) {
  STA_REQUIRE(g != nullptr, "null graph");
  STA_REQUIRE(count >= 0, "negative triple count");
  STA_REQUIRE(count == 0 || triples_host != nullptr, "null triples");
  for (int t = 0; t < count; ++t) {
    const int node = triples_host[3 * t], parent = triples_host[3 * t + 1], edge = triples_host[3 * t + 2];
    STA_REQUIRE(node >= 0 && node < g->max_nodes, "replayed node out of range");
    STA_REQUIRE(parent >= 0 && parent < g->max_nodes && parent != node, "parent out of range or the node itself");
    STA_REQUIRE(edge >= 0 && edge < g->max_edges, "edge out of range");
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (int t0 = 0; t0 < count; t0 += kReplayChunk) {
    ReplayArgs a;
    a.count = count - t0 < kReplayChunk ? count - t0 : kReplayChunk;
    for (int t = 0; t < a.count; ++t)
      for (int c = 0; c < 3; ++c) a.t[t][c] = triples_host[3 * (t0 + t) + c];
    graph_replay_kernel<<<1, 32, 0, st>>>(g->pose, g->meas, a);
    STA_CHECK_CUDA(cudaGetLastError());
  }
  return 0;
}

size_t sta_graph_export_scratch_bytes(int num_views, int H) {
  const long long rows = static_cast<long long>(num_views > 0 ? num_views : 1) * H;
  return static_cast<size_t>(rows * sizeof(int) + (rows + 1) * sizeof(long long) + 16);
}

int sta_graph_export(StaGraph* g, int view0, int num_views, float conf_thres, const float* imgs_dev, float* pose_out,
                     float* scale_out, float* depth_out, float* conf_out, float* intri_out, float* points_out,
                     float* colors_out, int64_t* count_out, void* scratch, void* stream) {
  STA_REQUIRE(g != nullptr, "null graph");
  STA_REQUIRE(num_views >= 1 && view0 >= 0 && static_cast<long long>(view0) + num_views <= g->max_views,
              "view range out of the graph");
  STA_REQUIRE(num_views <= 65535, "at most 65535 views per export");
  STA_REQUIRE(pose_out && scale_out && intri_out, "null output");
  const bool cloud = points_out != nullptr;
  STA_REQUIRE(!cloud || (imgs_dev && colors_out && count_out && scratch && depth_out && conf_out),
              "the point cloud needs images, depth / conf outputs, colours, a count and scratch");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long rows = static_cast<long long>(num_views) * g->H;
  int* counts = nullptr;
  long long* offsets = nullptr;
  if (cloud) {
    STA_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 7) == 0, "scratch must be 8-byte aligned");
    offsets = static_cast<long long*>(scratch);
    counts = reinterpret_cast<int*>(offsets + rows + 1);
  }
  export_gather_kernel<<<dim3(g->H, num_views), 256, 0, st>>>(*g, view0, conf_thres, pose_out, scale_out, depth_out, conf_out,
                                                              intri_out, counts);
  STA_CHECK_CUDA(cudaGetLastError());
  if (!cloud) return 0;
  row_scan_kernel<<<1, 1024, 0, st>>>(counts, rows, offsets, count_out);
  STA_CHECK_CUDA(cudaGetLastError());
  export_scatter_kernel<<<dim3(g->H, num_views), 256, 0, st>>>(*g, conf_thres, pose_out, scale_out, intri_out, depth_out, conf_out,
                                                               imgs_dev, offsets, points_out, colors_out);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
