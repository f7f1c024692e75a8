// Device-resident pose graph of OnlineSLAM (vista_slam/slam.py:20-447 over vista_slam/pose_graph.py:5-54): the node
// and edge tables, the per-node depth / confidence / intrinsics store, the per-view best node, the graph update of one
// keyframe (connect_view_i_j, slam.py:191-241, for all its kept edges) and the per-view gather + world point cloud of
// save_data_all / get_view (slam.py:299-412).
//
// The reference keeps the maps on the host (pose_graph.py:37) and reads a confidence mean back per node (:41) and per
// scale edge (slam.py:227); here everything stays on the device and any number of keyframes, of one graph or of many
// (up to STA_GRAPH_MAX_GROUP_KEYFRAMES), cost two launches with no host synchronisation:
//   graph_ingest_kernel  copies the 2n maps of each keyframe's n kept edges into the node store and runs its up to
//                        2n - 1 scale-edge reductions (pointmap.cuh, the reduction of sta_depth_scale);
//   graph_link_kernel    one block per graph: for each of its keyframes in order, finishes the reductions, then one
//                        thread walks the edges in the reference's order: node tables, best node (strict > against
//                        -100), rotation -> quaternion, node poses and edge records.
// A scale reduction that reads a node inserted earlier in the same launch reads it from that keyframe's inputs, not
// from the store the copies are writing (map_of).
//
// Tracked frames (OnlineSLAM.track) read the graph and never write it: track_reduce_kernel runs each frame's scale
// reduction against its anchor node in the store, and track_link_kernel composes the frame's pose with the Sim(3)
// algebra of sim3.cuh in the order graph_link_kernel would use for a keyframe with that single edge.
// frame_poses_kernel recomposes stored frames on their anchors' current poses.
#include <string>

#include "../../include/sta_b200.h"
#include "cloud.cuh"
#include "host_util.h"
#include "pointmap.cuh"
#include "sim3.cuh"

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
  double* partial = nullptr;      // [STA_GRAPH_MAX_KEYFRAME_EDGES * 2][kStatBlocks][kStatVals]: one keyframe's records
  int* flags_host = nullptr;      // mapped host word, written by the link kernel
  int* flags_dev = nullptr;       // its device alias
};

namespace sta {
namespace {

constexpr int kMaxKf = STA_GRAPH_MAX_KEYFRAME_EDGES;
constexpr int kMaxGroup = STA_GRAPH_MAX_GROUP_KEYFRAMES;
constexpr long long kPartialDoubles = static_cast<long long>(kStatBlocks) * kStatVals;  // one scale edge's records

// One keyframe of a grouped insertion: its graph's tables, its inputs and its place in the launch.
struct KfDesc {
  float *pose, *depth, *conf, *intri, *cmean, *best_mean, *meas, *weight;
  long long *node_view, *node_cview, *best_node, *edges;
  int* flags;
  const float* in_pose;    // [*][4][4]
  const float* pconf;      // [*]
  const float* confs;      // [2][n][H][W]
  const float* depths;     // [2][n][H][W]
  const float* in_intri;   // [n][3][3]
  const float* in_cmean;   // [2][n]
  long long hw;
  int gid;                 // index of its graph among the launch's graphs
  int n, n_scale, node0, edge0, view;
  int row0;                // first ingest row (grid y) of the keyframe
  int s0;                  // first scale-edge record set of the keyframe in the scratch
  int cand[kMaxKf];        // candidate row of edge k in pose / pose_conf
  int js[kMaxKf];          // view j of edge k
  int first_j[kMaxKf];     // first node of view j when edge k is inserted, -1 if it has none
};

// The keyframes of one launch pair, in table order; the kernels are instantiated for groups of one and of up to
// kMaxGroup, so a single keyframe does not pass the large table.  Passed as a __grid_constant__ kernel parameter:
// no copy of the table precedes the launches.
template <int N>
struct KfGroup {
  int count, graphs;
  KfDesc k[N];
};
static_assert(sizeof(KfGroup<kMaxGroup>) + 64 <= 32764, "the keyframe table must fit the kernel-parameter space");

// Map of node `slot` of keyframe t's graph: a node inserted by keyframe t or by an earlier keyframe of the same graph in
// this launch is row r of edge k in that keyframe's inputs (slot = node0 + 2k + r); older ones are in the store.  So
// the scale reductions never read a store slot that this launch's copies write.
template <int N>
__device__ __forceinline__ const float* map_of(const KfGroup<N>& p, int t, bool depth, int slot) {
  const KfDesc& a = p.k[t];
  for (int u = t; u >= 0; --u) {
    const KfDesc& b = p.k[u];
    if (b.gid != a.gid || slot < b.node0 || slot >= b.node0 + 2 * b.n) continue;
    const int d = slot - b.node0;
    return (depth ? b.depths : b.confs) + (static_cast<long long>(d & 1) * b.n + (d >> 1)) * b.hw;
  }
  return (depth ? a.depth : a.conf) + static_cast<long long>(slot) * a.hw;
}

// Scale edge s of a keyframe, in edge order: (new node, first node of its view).
__device__ void scale_edge(const KfDesc& a, int s, int* nnew, int* nother) {
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

// grid (kStatBlocks, sum over keyframes of n_scale + 2n), 256 threads: row y of keyframe t is its scale edge y (y <
// n_scale, records into the scratch) or the copy of its node node0 + y - n_scale into the store
template <int N>
__global__ void __launch_bounds__(256) graph_ingest_kernel(const __grid_constant__ KfGroup<N> p, double* partial) {
  int t = 0;
  while (t + 1 < p.count && static_cast<int>(blockIdx.y) >= p.k[t + 1].row0) ++t;
  const KfDesc& a = p.k[t];
  const int y = blockIdx.y - a.row0;
  if (y < a.n_scale) {
    int nn = 0, no = 0;
    scale_edge(a, y, &nn, &no);
    // estimate_scale_with_depth_and_confidence(depth, depth_other, conf, conf_other), slam.py:224
    scale_partial(map_of(p, t, true, nn), map_of(p, t, true, no), map_of(p, t, false, nn), map_of(p, t, false, no), a.hw,
                  blockIdx.x, partial + (a.s0 + y) * kPartialDoubles + static_cast<long long>(blockIdx.x) * kStatVals);
    return;
  }
  const int slot = a.node0 + (y - a.n_scale);
  const int d = y - a.n_scale;
  const long long src = (static_cast<long long>(d & 1) * a.n + (d >> 1)) * a.hw;
  float* dd = a.depth + static_cast<long long>(slot) * a.hw;
  float* cd = a.conf + static_cast<long long>(slot) * a.hw;
  for (long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x; i < a.hw; i += kStatBlocks * 256) {
    dd[i] = a.depths[src + i];
    cd[i] = a.confs[src + i];
  }
  if (blockIdx.x == 0 && threadIdx.x < 9) a.intri[slot * 9 + threadIdx.x] = a.in_intri[(d >> 1) * 9 + threadIdx.x];
}

__device__ void put_edge(const KfDesc& g, int e, long long ni, long long nj, const float* m8, const float* w7) {
  g.edges[2 * e] = ni;
  g.edges[2 * e + 1] = nj;
  for (int i = 0; i < 8; ++i) g.meas[e * 8 + i] = m8[i];
  for (int i = 0; i < 7; ++i) g.weight[e * 7 + i] = w7[i];
}

// grid (graphs), 64 threads: block b walks the keyframes of graph b in table order -- each keyframe's reductions
// finished, then one thread walks its edges in the reference's order: node tables, best node (strict > against -100),
// rotation -> quaternion, node poses and edge records
template <int N>
__global__ void __launch_bounds__(64) graph_link_kernel(const __grid_constant__ KfGroup<N> p, const double* partial) {
  __shared__ float sc[2 * kMaxKf][2];
  for (int t = 0; t < p.count; ++t) {
    const KfDesc& a = p.k[t];
    if (a.gid != static_cast<int>(blockIdx.x)) continue;
    if (threadIdx.x < a.n_scale) scale_finalize(partial + (a.s0 + threadIdx.x) * kPartialDoubles, a.hw, sc[threadIdx.x]);
    __syncthreads();
    if (threadIdx.x == 0) {
      int e = a.edge0, s = 0;
      for (int k = 0; k < a.n; ++k) {
        for (int r = 0; r < 2; ++r) {  // add_node(i), its scale edge, add_node(j), its scale edge (slam.py:210-232)
          const int slot = a.node0 + 2 * k + r;
          const long long v = r ? a.js[k] : a.view;
          a.node_view[slot] = v;
          a.node_cview[slot] = r ? a.view : a.js[k];
          const float m = a.in_cmean[r * a.n + k];
          a.cmean[slot] = m;
          if (m > a.best_mean[v]) {  // pose_graph.py:42: strict, so the first node wins a tie
            a.best_mean[v] = m;
            a.best_node[v] = slot;
          }
          const int other = r ? a.first_j[k] : (k > 0 ? a.node0 : -1);
          if (other >= 0) {
            const float sim3[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 1.f, sc[s][0]};
            const float w[7] = {2.f, 2.f, 2.f, 2.f, 2.f, 2.f, sc[s][1]};  // PoseGraphEdges.id_pose_conf = 2.0
            ++s;
            put_edge(a, e++, slot, other, sim3, w);
            sim3_mul(a.pose + other * 8, sim3, a.pose + slot * 8);
          }
        }
        const float* M = a.in_pose + a.cand[k] * 16;
        float sim3[8] = {M[3], M[7], M[11], 0.f, 0.f, 0.f, 1.f, 1.f};
        if (!rot_to_quat(M, sim3 + 3)) *reinterpret_cast<volatile int*>(a.flags) |= STA_GRAPH_FLAG_NOT_SO3;
        const int ni = a.node0 + 2 * k, nj = ni + 1;
        if (k == 0) sim3_mul(a.pose + nj * 8, sim3, a.pose + ni * 8);  // view i is new at its first node (slam.py:234-236)
        const float c = a.pconf[a.cand[k]];
        const float w[7] = {c, c, c, c, c, c, c};
        put_edge(a, e++, ni, nj, sim3, w);
      }
    }
    __syncthreads();  // sc is reused by the graph's next keyframe
  }
  if (threadIdx.x == 0) __threadfence_system();
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
    scale_out[v] = sim3_to_pose44(g.pose + b * 8, pose_out + v * 16);
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

// ---- tracked frames ----

// Host anchors of a track or frame-pose launch, passed as a __grid_constant__ kernel parameter: one launch for up to
// STA_GRAPH_MAX_TRACK_FRAMES frames with no copy before it.  Instantiated for up to kTrackSmall frames and for the
// maximum, so that a few frames do not pass the large table.
constexpr int kTrackSmall = 64;
constexpr int kMaxTrack = STA_GRAPH_MAX_TRACK_FRAMES;
template <int N>
struct TrackArgs {
  int count;
  int anchor[N];
};
static_assert(sizeof(TrackArgs<kMaxTrack>) + 128 <= 32764, "the anchor table must fit the kernel-parameter space");

// grid (kStatBlocks, F), 256 threads: frame f's scale reduction against its anchor in the store, with the argument
// order of the scale edge a new node of the keyframe view gets (estimate_scale_with_depth_and_confidence(depth,
// depth_other, conf, conf_other), slam.py:224): the frame pair's keyframe-side maps first.
template <int N>
__global__ void __launch_bounds__(256) track_reduce_kernel(const __grid_constant__ TrackArgs<N> p, const float* gdepth,
                                                          const float* gconf, const float* depth, const float* conf,
                                                          long long hw, double* partial) {
  const int f = blockIdx.y;
  const long long a = p.anchor[f];
  scale_partial(depth + f * hw, gdepth + a * hw, conf + f * hw, gconf + a * hw, hw, blockIdx.x,
                partial + f * kPartialDoubles + static_cast<long long>(blockIdx.x) * kStatVals);
}

// pose[anchor] * Sim3(0, id, s) * Sim3(T): the product graph_link_kernel gives node i of a keyframe whose first kept
// edge is (i, k) -- the scale edge's node of k from the anchor, then the pose edge -- as [t | q | s].
__device__ void track_compose(const float* anchor_pose, float s, const float* T, float* out) {
  const float S[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 1.f, s};
  float j[8];
  sim3_mul(anchor_pose, S, j);
  sim3_mul(j, T, out);
}

// one thread per frame: the reduction finished, T_fk -> [t | q | 1] (a failed SO(3) check clears valid and raises no
// graph flag), the composed pose as 4x4 (scale dropped) and its scale
template <int N>
__global__ void __launch_bounds__(64) track_link_kernel(const __grid_constant__ TrackArgs<N> p, const float* gpose,
                                                        const double* partial, long long hw, const float* pose_in,
                                                        float* meas_out, float* s_out, unsigned char* valid_out,
                                                        float* pose_out, float* scale_out) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= p.count) return;
  float sc[2];
  scale_finalize(partial + f * kPartialDoubles, hw, sc);
  const float* M = pose_in + f * 16;
  float T[8] = {M[3], M[7], M[11], 0.f, 0.f, 0.f, 1.f, 1.f};
  const bool ok = rot_to_quat(M, T + 3);
  for (int i = 0; i < 8; ++i) meas_out[f * 8 + i] = T[i];
  s_out[f] = sc[0];
  valid_out[f] = ok ? 1 : 0;
  float P[8];
  track_compose(gpose + static_cast<long long>(p.anchor[f]) * 8, sc[0], T, P);
  scale_out[f] = sim3_to_pose44(P, pose_out + f * 16);
}

// one thread per frame: a stored frame recomposed on its anchor's current pose
template <int N>
__global__ void __launch_bounds__(64) frame_poses_kernel(const __grid_constant__ TrackArgs<N> p, const float* gpose,
                                                         const float* meas, const float* s, float* pose_out,
                                                         float* scale_out) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= p.count) return;
  float P[8];
  track_compose(gpose + static_cast<long long>(p.anchor[f]) * 8, s[f], meas + f * 8, P);
  scale_out[f] = sim3_to_pose44(P, pose_out + f * 16);
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

}  // extern "C"

namespace {

// The n_scale of a keyframe: a scale edge for every edge k > 0 (to view i's first node) and for every j with a node.
int scale_edges_of(const StaGraphKeyframe& f) {
  int c = 0;
  for (int k = 0; k < f.n; ++k) c += (k > 0) + (f.first_j[k] >= 0);
  return c;
}

// Every refusal of sta_graph_add_keyframes, before any launch; fills the table of the launch pair.
template <int N>
int fill_group(const StaGraphKeyframe* kfs, int count, KfGroup<N>* p, int* rows, int* records) {
  STA_REQUIRE(kfs != nullptr, "null keyframe table");
  STA_REQUIRE(count >= 1 && count <= N, "1 to STA_GRAPH_MAX_GROUP_KEYFRAMES keyframes per call");
  const StaGraph* graphs[kMaxGroup];
  int last[kMaxGroup];  // the graph's previous keyframe in the table
  p->count = count;
  p->graphs = 0;
  *rows = 0;
  *records = 0;
  for (int t = 0; t < count; ++t) {
    const StaGraphKeyframe& f = kfs[t];
    StaGraph* g = f.graph;
    const int n = f.n;
    STA_REQUIRE(g != nullptr && f.js && f.cand && f.first_j, "null argument");
    STA_REQUIRE(n >= 1 && n <= kMaxKf, "1 to STA_GRAPH_MAX_KEYFRAME_EDGES kept edges per keyframe");
    STA_REQUIRE(f.H == g->H && f.W == g->W, "map size differs from the graph's");
    STA_REQUIRE(f.pose && f.pose_conf && f.confs && f.depths && f.intri && f.conf_mean, "null device input");
    STA_REQUIRE(on_device(f.pose) && on_device(f.pose_conf) && on_device(f.confs) && on_device(f.depths) &&
                    on_device(f.intri) && on_device(f.conf_mean),
                "inputs must be device memory");
    STA_REQUIRE(f.view >= 0 && f.view < g->max_views, "view index out of range");
    for (int k = 0; k < n; ++k) {
      STA_REQUIRE(f.js[k] >= 0 && f.js[k] < f.view, "j must be an earlier view");
      STA_REQUIRE(f.cand[k] >= 0, "negative candidate index");
      STA_REQUIRE(f.first_j[k] >= -1 && f.first_j[k] < f.node0 + 2 * k, "first node of view j is not in the graph");
    }
    const int n_scale = scale_edges_of(f);
    STA_REQUIRE(f.node0 >= 0 && static_cast<long long>(f.node0) + 2 * n <= g->max_nodes, "node capacity exceeded");
    STA_REQUIRE(f.edge0 >= 0 && static_cast<long long>(f.edge0) + n_scale + n <= g->max_edges, "edge capacity exceeded");
    int gid = 0;
    while (gid < p->graphs && graphs[gid] != g) ++gid;
    if (gid == p->graphs) {
      graphs[p->graphs++] = g;
    } else {
      const StaGraphKeyframe& q = kfs[last[gid]];
      STA_REQUIRE(f.node0 == q.node0 + 2 * q.n && f.edge0 == q.edge0 + scale_edges_of(q) + q.n,
                  "a keyframe's node0 / edge0 do not continue its graph's previous keyframe in the call");
    }
    last[gid] = t;
    KfDesc& a = p->k[t];
    a = KfDesc{};
    a.pose = g->pose; a.depth = g->depth; a.conf = g->conf; a.intri = g->intri; a.cmean = g->cmean;
    a.best_mean = g->best_mean; a.meas = g->meas; a.weight = g->weight;
    a.node_view = reinterpret_cast<long long*>(g->node_view);
    a.node_cview = reinterpret_cast<long long*>(g->node_cview);
    a.best_node = reinterpret_cast<long long*>(g->best_node);
    a.edges = reinterpret_cast<long long*>(g->edges);
    a.flags = g->flags_dev;
    a.in_pose = f.pose; a.pconf = f.pose_conf; a.confs = f.confs; a.depths = f.depths; a.in_intri = f.intri;
    a.in_cmean = f.conf_mean;
    a.hw = static_cast<long long>(f.H) * f.W;
    a.gid = gid;
    a.n = n; a.n_scale = n_scale; a.node0 = f.node0; a.edge0 = f.edge0; a.view = f.view;
    a.row0 = *rows;
    a.s0 = *records;
    for (int k = 0; k < n; ++k) {
      a.cand[k] = f.cand[k];
      a.js[k] = static_cast<int>(f.js[k]);
      a.first_j[k] = f.first_j[k];
    }
    *rows += n_scale + 2 * n;
    *records += n_scale;
  }
  return 0;
}

template <int N>
int launch_group(const StaGraphKeyframe* kfs, int count, double* scratch, size_t scratch_bytes, bool own_partial,
                 cudaStream_t st) {
  KfGroup<N> p;
  int rows = 0, records = 0;
  if (int rc = fill_group(kfs, count, &p, &rows, &records)) return rc;
  if (own_partial) scratch = kfs[0].graph->partial;
  STA_REQUIRE(scratch != nullptr, "null scratch");
  STA_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 7) == 0, "scratch must be 8-byte aligned");
  STA_REQUIRE(own_partial || scratch_bytes >= sizeof(double) * kPartialDoubles * (records > 0 ? records : 1),
              "scratch smaller than sta_graph_add_keyframes_scratch_bytes");
  graph_ingest_kernel<N><<<dim3(kStatBlocks, rows), 256, 0, st>>>(p, scratch);
  STA_CHECK_CUDA(cudaGetLastError());
  graph_link_kernel<N><<<p.graphs, 64, 0, st>>>(p, scratch);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" {

int sta_graph_add_keyframe(StaGraph* g, int view, int n, const int64_t* js_host, const int* cand_host,
                           const int* first_j_host, int node0, int edge0, int H, int W, const float* pose_dev,
                           const float* pose_conf_dev, const float* confs_dev, const float* depths_dev, const float* intri_dev,
                           const float* conf_mean_dev, void* stream) {
  STA_REQUIRE(g != nullptr, "null argument");
  const StaGraphKeyframe f = {g, view, n, node0, edge0, H, W, js_host, cand_host, first_j_host,
                              pose_dev, pose_conf_dev, confs_dev, depths_dev, intri_dev, conf_mean_dev};
  return launch_group<1>(&f, 1, nullptr, 0, true, static_cast<cudaStream_t>(stream));
}

size_t sta_graph_add_keyframes_scratch_bytes(const StaGraphKeyframe* kfs, int count) {
  int rows = 0, records = 0, rc = 0;
  if (count == 1) {
    KfGroup<1> p;
    rc = fill_group(kfs, count, &p, &rows, &records);
  } else {
    KfGroup<kMaxGroup> p;
    rc = fill_group(kfs, count, &p, &rows, &records);
  }
  return rc ? 0 : sizeof(double) * kPartialDoubles * (records > 0 ? records : 1);
}

int sta_graph_add_keyframes(const StaGraphKeyframe* kfs, int count, void* scratch, size_t scratch_bytes, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  double* s = static_cast<double*>(scratch);
  if (count == 1) return launch_group<1>(kfs, count, s, scratch_bytes, false, st);
  return launch_group<kMaxGroup>(kfs, count, s, scratch_bytes, false, st);
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

namespace {

// The refusals shared by sta_graph_track_frames and sta_graph_frame_poses, before any launch.
int check_frames(const StaGraph* g, int F, const int* anchors_host) {
  STA_REQUIRE(F >= 1 && F <= kMaxTrack, "1 to STA_GRAPH_MAX_TRACK_FRAMES frames per call");
  STA_REQUIRE(g != nullptr && anchors_host != nullptr, "null argument");
  for (int f = 0; f < F; ++f)
    STA_REQUIRE(anchors_host[f] >= 0 && anchors_host[f] < g->max_nodes, "anchor node out of the graph's capacity");
  return 0;
}

template <int N>
TrackArgs<N> track_args(int F, const int* anchors_host) {
  TrackArgs<N> p;
  p.count = F;
  for (int f = 0; f < F; ++f) p.anchor[f] = anchors_host[f];
  return p;
}

template <int N>
int launch_track(StaGraph* g, int F, const int* anchors_host, const float* pose_dev, const float* depth_dev,
                 const float* conf_dev, float* meas_out, float* s_out, unsigned char* valid_out, float* pose_out,
                 float* scale_out, double* partial, cudaStream_t st) {
  const TrackArgs<N> p = track_args<N>(F, anchors_host);
  const long long hw = static_cast<long long>(g->H) * g->W;
  track_reduce_kernel<N><<<dim3(kStatBlocks, F), 256, 0, st>>>(p, g->depth, g->conf, depth_dev, conf_dev, hw, partial);
  STA_CHECK_CUDA(cudaGetLastError());
  track_link_kernel<N><<<(F + 63) / 64, 64, 0, st>>>(p, g->pose, partial, hw, pose_dev, meas_out, s_out, valid_out,
                                                    pose_out, scale_out);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

template <int N>
int launch_frame_poses(StaGraph* g, int F, const int* anchors_host, const float* meas_dev, const float* s_dev,
                       float* pose_out, float* scale_out, cudaStream_t st) {
  frame_poses_kernel<N><<<(F + 63) / 64, 64, 0, st>>>(track_args<N>(F, anchors_host), g->pose, meas_dev, s_dev, pose_out,
                                                      scale_out);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" {

size_t sta_graph_track_frames_scratch_bytes(int num_frames) {
  if (num_frames < 1 || num_frames > kMaxTrack) return 0;
  return sizeof(double) * kPartialDoubles * num_frames;
}

int sta_graph_track_frames(StaGraph* g, int num_frames, const int* anchors_host, const float* pose_dev,
                           const float* depth_dev, const float* conf_dev, float* meas_out, float* scale_edge_out,
                           unsigned char* valid_out, float* pose_out, float* scale_out, void* scratch,
                           size_t scratch_bytes, void* stream) {
  const int F = num_frames;
  if (int rc = check_frames(g, F, anchors_host)) return rc;
  STA_REQUIRE(pose_dev && depth_dev && conf_dev, "null device input");
  STA_REQUIRE(meas_out && scale_edge_out && valid_out && pose_out && scale_out, "null output");
  STA_REQUIRE(scratch != nullptr && (reinterpret_cast<uintptr_t>(scratch) & 7) == 0, "null or misaligned scratch");
  STA_REQUIRE(scratch_bytes >= sta_graph_track_frames_scratch_bytes(F), "scratch smaller than sta_graph_track_frames_scratch_bytes");
  STA_REQUIRE(on_device(pose_dev) && on_device(depth_dev) && on_device(conf_dev) && on_device(meas_out) &&
                  on_device(scale_edge_out) && on_device(valid_out) && on_device(pose_out) && on_device(scale_out) &&
                  on_device(scratch),
              "inputs and outputs must be device memory");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  double* partial = static_cast<double*>(scratch);
  if (F <= kTrackSmall)
    return launch_track<kTrackSmall>(g, F, anchors_host, pose_dev, depth_dev, conf_dev, meas_out, scale_edge_out,
                                     valid_out, pose_out, scale_out, partial, st);
  return launch_track<kMaxTrack>(g, F, anchors_host, pose_dev, depth_dev, conf_dev, meas_out, scale_edge_out, valid_out,
                                 pose_out, scale_out, partial, st);
}

int sta_graph_frame_poses(StaGraph* g, int num_frames, const int* anchors_host, const float* meas_dev,
                          const float* scale_edge_dev, float* pose_out, float* scale_out, void* stream) {
  const int F = num_frames;
  if (int rc = check_frames(g, F, anchors_host)) return rc;
  STA_REQUIRE(meas_dev && scale_edge_dev && pose_out && scale_out, "null device argument");
  STA_REQUIRE(on_device(meas_dev) && on_device(scale_edge_dev) && on_device(pose_out) && on_device(scale_out),
              "inputs and outputs must be device memory");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (F <= kTrackSmall) return launch_frame_poses<kTrackSmall>(g, F, anchors_host, meas_dev, scale_edge_dev, pose_out, scale_out, st);
  return launch_frame_poses<kMaxTrack>(g, F, anchors_host, meas_dev, scale_edge_dev, pose_out, scale_out, st);
}

}  // extern "C"
