// TSDF fusion of the SLAM map (fusion.fuse_views, OnlineSLAM.extract_mesh): a sparse volume of 8x8x8-sample bricks
// rebuilt from every view of the map, then a coloured triangle mesh by marching cubes.
//
//   bricks     grid (ceil(W / 256), H, V): each used pixel (conf > thres, d = depth * scale > 0) is the PLY's world
//              point p (cloud.cuh); the bricks floor((p -+ tau) / 8v) per axis that the cube [p - tau, p + tau] touches
//              (at most 2 per axis since tau <= 4v) are deduplicated in a shared-memory hash per 256-pixel tile, counted,
//              scanned over the tiles and written; then recon.cu's radix sort (sta_op_radix_sort) and a unique pass.
//              A key is the three brick coordinates biased by 2^20 in 21 bits each, z above y above x (brick.cuh).
//   integrate  brick_views_kernel: one bit per (brick, view) for the views whose frustum and depth range can reach
//              the brick, tested on the brick's box grown by one voxel (conservative: it never drops a view that
//              reaches a sample); integrate_kernel: one CTA per brick, one thread per sample, the brick's views in
//              increasing index, KinectFusion's unit-weight running averages in registers.  No atomics: the volume is
//              the same bit for bit on every call.
//   mesh       mc_classify_kernel: per cube (the sample and its +x, +y, +z neighbours, found by binary search over the
//              sorted keys) the case and triangle count, and one bit per lattice edge that an emitted face uses, at the
//              edge's lower sample (integer atomicOr: order-free); mc_count_kernel: vertices per brick; two scans over
//              the bricks; then mc_vertices_kernel and mc_faces_kernel write vertices in (brick, sample, axis) order
//              and faces in (brick, cube, triangle) order.  The table is mc_table.h, made by tools/make_mc_table.py.
#include <math.h>
#include <stdint.h>

#include "../../include/sta_b200.h"
#include "brick.cuh"
#include "cloud.cuh"
#include "host_util.h"
#define STA_MC_SPACE __constant__
#include "mc_table.h"

namespace sta {
namespace {

constexpr int kSamples = kBrickSamples;            // 512
constexpr int kTileSlots = 4096;                    // hash slots per 256-pixel tile: 8 keys per pixel at most
constexpr int kUniqueChunk = 2048;                  // sorted keys per unique block
constexpr unsigned long long kEmptyKey = ~0ull;     // above every 63-bit key

struct MapArgs {
  const float *depth, *conf, *pose, *scale, *intri, *imgs, *w2c;
  int V, H, W;
  float thres;
};

// ---------------------------------------------------------------------------------------------------------- bricks

__device__ __forceinline__ void hash_insert(unsigned long long* slots, unsigned long long key) {
  unsigned h = static_cast<unsigned>((key * 0x9E3779B97F4A7C15ull) >> 52);  // 12 bits
  while (true) {
    const unsigned long long old = atomicCAS(slots + h, kEmptyKey, key);
    if (old == kEmptyKey || old == key) return;
    h = (h + 1) & (kTileSlots - 1);
  }
}

// grid (ceil(W / 256), H, V), 256 threads.  Count pass (keys == nullptr): tile_counts[tile] = the tile's distinct
// bricks.  Fill pass: the tile's bricks to keys[tile_off[tile] ...], dropping any beyond cap.
__global__ void __launch_bounds__(256) brick_keys_kernel(const __grid_constant__ MapArgs m, float vox, float tau,
                                                          int* tile_counts, const long long* tile_off,
                                                          unsigned long long* keys, long long cap) {
  __shared__ unsigned long long slots[kTileSlots];
  for (int k = threadIdx.x; k < kTileSlots; k += 256) slots[k] = kEmptyKey;
  __syncthreads();
  const int v = blockIdx.z, row = blockIdx.y, x = blockIdx.x * 256 + threadIdx.x;
  const long long tile = (static_cast<long long>(v) * m.H + row) * gridDim.x + blockIdx.x;
  if (x < m.W) {
    const long long pix = (static_cast<long long>(v) * m.H + row) * m.W + x;
    const float d = m.depth[pix] * m.scale[v];
    if (m.conf[pix] > m.thres && d > 0.f) {
      float Ki[9], p[3];
      inv3_f32(m.intri + v * 9, Ki);
      unproject_f32(Ki, m.pose + v * 16, static_cast<float>(x), static_cast<float>(row), d, p);
      const float bs = vox * static_cast<float>(kBrick);
      float lo[3], hi[3];
      bool ok = true;
      for (int c = 0; c < 3; ++c) {
        lo[c] = floorf((p[c] - tau) / bs);
        hi[c] = floorf((p[c] + tau) / bs);
        // false for NaN and infinities too
        ok = ok && lo[c] >= -static_cast<float>(kBias) && hi[c] <= static_cast<float>(kBias - 1);
      }
      if (ok) {
        const int x0 = static_cast<int>(lo[0]), y0 = static_cast<int>(lo[1]), z0 = static_cast<int>(lo[2]);
        const int x1 = static_cast<int>(hi[0]), y1 = static_cast<int>(hi[1]), z1 = static_cast<int>(hi[2]);
        for (int bz = z0; bz <= z1; ++bz)
          for (int by = y0; by <= y1; ++by)
            for (int bx = x0; bx <= x1; ++bx) hash_insert(slots, brick_key(bx, by, bz));
      }
    }
  }
  __syncthreads();
  if (keys == nullptr) {
    int cnt = 0;
    for (int k = threadIdx.x; k < kTileSlots; k += 256) cnt += slots[k] != kEmptyKey;
    cnt = block_count_256(cnt);
    if (threadIdx.x == 0) tile_counts[tile] = cnt;
    return;
  }
  row_compact_256(kTileSlots, tile_off[tile], [&](int k) { return slots[k] != kEmptyKey; },
                  [&](int k, long long o) {
                    if (o < cap) keys[o] = slots[k];
                  });
}

// grid ceil(n / kUniqueChunk), 256 threads: counts[blk] = sorted keys of the chunk that differ from their predecessor
// (the empty padding excluded); with out, write them there from off[blk]
__global__ void __launch_bounds__(256) unique_kernel(const unsigned long long* sorted, long long n, int* counts,
                                                     const long long* off, int64_t* out) {
  const long long c0 = static_cast<long long>(blockIdx.x) * kUniqueChunk;
  const int len = static_cast<int>(min(static_cast<long long>(kUniqueChunk), n - c0));
  auto head = [&](int k) {
    const long long i = c0 + k;
    const unsigned long long key = sorted[i];
    return key != kEmptyKey && (i == 0 || sorted[i - 1] != key);
  };
  if (out == nullptr) {
    int cnt = 0;
    for (int k = threadIdx.x; k < len; k += 256) cnt += head(k);
    cnt = block_count_256(cnt);
    if (threadIdx.x == 0) counts[blockIdx.x] = cnt;
    return;
  }
  row_compact_256(len, off[blockIdx.x], head,
                  [&](int k, long long o) { out[o] = static_cast<int64_t>(sorted[c0 + k]); });
}

struct BrickScratch {
  int* tile_counts;
  long long* tile_off;
  unsigned long long* keys;
  uint32_t* idx;
  int* chunk_counts;
  long long* chunk_off;
  void* sort;
};

long long align16(long long b) { return (b + 15) / 16 * 16; }

long long num_tiles(int V, int H, int W) { return static_cast<long long>((W + 255) / 256) * H * V; }

// tile counts and offsets, the cap keys, their sort indices, chunk counts and offsets, the sort's own scratch
size_t brick_scratch(int V, int H, int W, long long cap, BrickScratch* s, void* base) {
  const long long tiles = num_tiles(V, H, W), chunks = (cap + kUniqueChunk - 1) / kUniqueChunk;
  char* p = static_cast<char*>(base);
  long long o = 0;
  auto take = [&](long long bytes) {
    char* q = p + o;
    o += align16(bytes);
    return q;
  };
  char* a = take(4 * tiles);
  char* b = take(8 * (tiles + 1));
  char* c = take(8 * cap);
  char* d = take(4 * cap);
  char* e = take(4 * (chunks + 1));
  char* f = take(8 * (chunks + 1));
  char* g = take(static_cast<long long>(sta_sort_scratch_bytes(cap)));
  if (s) *s = {reinterpret_cast<int*>(a), reinterpret_cast<long long*>(b), reinterpret_cast<unsigned long long*>(c),
               reinterpret_cast<uint32_t*>(d), reinterpret_cast<int*>(e), reinterpret_cast<long long*>(f), g};
  return static_cast<size_t>(o);
}

// ---------------------------------------------------------------------------------------------------------- integrate

// grid V, 256 threads: dmax[v] = the largest used depth of view v (0 without one).  Max is order-free.
__global__ void __launch_bounds__(256) view_depth_kernel(const __grid_constant__ MapArgs m, float* dmax) {
  const int v = blockIdx.x;
  const long long hw = static_cast<long long>(m.H) * m.W;
  const float s = m.scale[v];
  float best = 0.f;
  for (long long i = threadIdx.x; i < hw; i += 256) {
    const float d = m.depth[v * hw + i] * s;
    if (m.conf[v * hw + i] > m.thres && d > 0.f) best = fmaxf(best, d);
  }
  for (int o = 16; o; o >>= 1) best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, o));
  __shared__ float w[8];
  if ((threadIdx.x & 31) == 0) w[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k) best = fmaxf(best, w[k]);
    dmax[v] = best;
  }
}

// grid B, 128 threads: bit v of mask[b][.] is set unless brick b's box grown by one voxel lies wholly behind view v's
// camera, outside one side of its pixel frustum (grown by one pixel) or beyond its largest used depth plus tau.  Each
// test is a linear function of the point, so its maximum over the box is at a corner; fp64.
__global__ void __launch_bounds__(128) brick_views_kernel(const __grid_constant__ MapArgs m, const int64_t* keys,
                                                          double vox, double tau, const float* dmax, int words,
                                                          unsigned* mask) {
  const int b = blockIdx.x;
  int bx, by, bz;
  key_brick(static_cast<unsigned long long>(keys[b]), bx, by, bz);
  const double lo[3] = {(kBrick * bx - 1) * vox, (kBrick * by - 1) * vox, (kBrick * bz - 1) * vox};
  const double span = (kBrick + 1) * vox;
  for (int v0 = 0; v0 < m.V; v0 += 128) {
    const int v = v0 + threadIdx.x;
    bool keep = false;
    if (v < m.V) {
      const float* M = m.w2c + v * 16;
      const float* K = m.intri + v * 9;
      double zmax = -INFINITY, zmin = INFINITY, l0 = -INFINITY, l1 = -INFINITY, l2 = -INFINITY, l3 = -INFINITY;
      for (int c = 0; c < 8; ++c) {
        const double p[3] = {lo[0] + (c & 1) * span, lo[1] + (c >> 1 & 1) * span, lo[2] + (c >> 2 & 1) * span};
        double q[3];
        for (int r = 0; r < 3; ++r) q[r] = M[r * 4] * p[0] + M[r * 4 + 1] * p[1] + M[r * 4 + 2] * p[2] + M[r * 4 + 3];
        const double ku = K[0] * q[0] + K[1] * q[1] + K[2] * q[2], kv = K[3] * q[0] + K[4] * q[1] + K[5] * q[2];
        zmax = fmax(zmax, q[2]);
        zmin = fmin(zmin, q[2]);
        // pixel column u = ku / z within [-0.5 - 1, W - 0.5 + 1], rows alike, as halfspaces of z > 0
        l0 = fmax(l0, ku + 1.5 * q[2]);
        l1 = fmax(l1, (m.W + 0.5) * q[2] - ku);
        l2 = fmax(l2, kv + 1.5 * q[2]);
        l3 = fmax(l3, (m.H + 0.5) * q[2] - kv);
      }
      keep = zmax > 0.0 && l0 >= 0.0 && l1 >= 0.0 && l2 >= 0.0 && l3 >= 0.0 &&
             zmin <= (static_cast<double>(dmax[v]) + tau) * (1.0 + 1e-6) + vox;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    const int word = (v0 >> 5) + (threadIdx.x >> 5);
    if ((threadIdx.x & 31) == 0 && word < words) mask[static_cast<long long>(b) * words + word] = bal;
  }
}

// grid B, 512 threads: sample (x, y, z) = thread (t & 7, t >> 3 & 7, t >> 6) of brick b, at world (i v, j v, k v)
__global__ void __launch_bounds__(512) integrate_kernel(const __grid_constant__ MapArgs m, const int64_t* keys,
                                                        float vox, float tau, int words, const unsigned* mask,
                                                        float* tsdf, float* weight, float* color) {
  const int b = blockIdx.x, t = threadIdx.x;
  int bx, by, bz;
  key_brick(static_cast<unsigned long long>(keys[b]), bx, by, bz);
  const float px = static_cast<float>(kBrick * bx + (t & 7)) * vox, py = static_cast<float>(kBrick * by + (t >> 3 & 7)) * vox,
              pz = static_cast<float>(kBrick * bz + (t >> 6)) * vox;
  const long long hw = static_cast<long long>(m.H) * m.W;
  float T = 0.f, Wt = 0.f, C0 = 0.f, C1 = 0.f, C2 = 0.f;
  for (int w = 0; w < words; ++w) {
    unsigned bits = mask[static_cast<long long>(b) * words + w];
    while (bits) {
      const int v = w * 32 + __ffs(bits) - 1;
      bits &= bits - 1;
      const float* M = m.w2c + v * 16;
      const float cz = M[8] * px + M[9] * py + M[10] * pz + M[11];
      if (!(cz > 0.f)) continue;
      const float cx = M[0] * px + M[1] * py + M[2] * pz + M[3], cy = M[4] * px + M[5] * py + M[6] * pz + M[7];
      const float* K = m.intri + v * 9;
      const float u = (K[0] * cx + K[1] * cy + K[2] * cz) / cz, r = (K[3] * cx + K[4] * cy + K[5] * cz) / cz;
      const float fu = floorf(u + 0.5f), fr = floorf(r + 0.5f);
      if (!(fu >= 0.f && fu < static_cast<float>(m.W) && fr >= 0.f && fr < static_cast<float>(m.H))) continue;
      const long long pix = v * hw + static_cast<long long>(fr) * m.W + static_cast<long long>(fu);
      const float d = m.depth[pix] * m.scale[v];
      if (!(m.conf[pix] > m.thres && d > 0.f)) continue;
      const float sdf = d - cz;
      if (sdf < -tau) continue;
      const float tv = fminf(1.f, sdf / tau), n1 = Wt + 1.f;
      const float* img = m.imgs + static_cast<long long>(v) * 3 * hw + (pix - v * hw);
      T = (T * Wt + tv) / n1;
      C0 = (C0 * Wt + (img[0] + 1.f) / 2.f) / n1;
      C1 = (C1 * Wt + (img[hw] + 1.f) / 2.f) / n1;
      C2 = (C2 * Wt + (img[2 * hw] + 1.f) / 2.f) / n1;
      Wt = n1;
    }
  }
  const long long o = static_cast<long long>(b) * kSamples + t;
  tsdf[o] = T;
  weight[o] = Wt;
  color[o * 3] = C0;
  color[o * 3 + 1] = C1;
  color[o * 3 + 2] = C2;
}

// ---------------------------------------------------------------------------------------------------------- mesh

struct MeshArgs {
  const int64_t* keys;
  long long B;
  const float *tsdf, *weight, *color;
  float vox, min_weight;
};

// threads 0..7 of the block: nb[o] = the brick at offset (o & 1, o >> 1 & 1, o >> 2) from brick b, or -1
__device__ __forceinline__ void load_neighbours(const MeshArgs& a, int b, int* nb) {
  if (threadIdx.x < 8) {
    const int o = threadIdx.x;
    int bx, by, bz;
    key_brick(static_cast<unsigned long long>(a.keys[b]), bx, by, bz);
    bx += o & 1;
    by += o >> 1 & 1;
    bz += o >> 2;
    nb[o] = (bx < kBias && by < kBias && bz < kBias) ? find_brick(a.keys, a.B, static_cast<long long>(brick_key(bx, by, bz)))
                                                     : -1;
  }
  __syncthreads();
}

// global sample index of local (x, y, z) + (dx, dy, dz), each of x + dx etc. in [0, 16); -1 when its brick is missing
__device__ __forceinline__ long long sample_at(const int* nb, int x, int y, int z) {
  const int n = nb[(x >> 3) | ((y >> 3) << 1) | ((z >> 3) << 2)];
  return n < 0 ? -1 : static_cast<long long>(n) * kSamples + (((z & 7) << 6) | ((y & 7) << 3) | (x & 7));
}

// exclusive scan of one int per thread over a 512-thread block; total to *total
__device__ __forceinline__ int block_scan_512(int val, int* total) {
  __shared__ int wsum[16];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = val;
  for (int o = 1; o < 32; o <<= 1) {
    const int n = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += n;
  }
  if (lane == 31) wsum[warp] = inc;
  __syncthreads();
  int before = 0, all = 0;
  for (int w = 0; w < 16; ++w) {
    before += w < warp ? wsum[w] : 0;
    all += wsum[w];
  }
  *total = all;
  return before + inc - val;
}

// the cube at sample t of brick b: its case, or -1 when a corner is missing or below min_weight; corner samples to g
__device__ __forceinline__ int cube_case(const MeshArgs& a, const int* nb, int t, long long* g) {
  const int x = t & 7, y = t >> 3 & 7, z = t >> 6;
  int cs = 0;
  for (int c = 0; c < 8; ++c) {
    g[c] = sample_at(nb, x + (c & 1), y + (c >> 1 & 1), z + (c >> 2));
    if (g[c] < 0 || !(a.weight[g[c]] >= a.min_weight)) return -1;
    cs |= (a.tsdf[g[c]] < 0.f) << c;
  }
  return cs;
}

// lower corner of cube edge e (mc_table.h: e = 4 axis + the other two coordinates as bits)
__device__ __forceinline__ int edge_lower_corner(int e) {
  const int axis = e >> 2, o0 = e & 1, o1 = e >> 1 & 1;
  return axis == 0 ? (o0 << 1) | (o1 << 2) : axis == 1 ? o0 | (o1 << 2) : o0 | (o1 << 1);
}

// grid B, 512 threads: cube cases (0 for an unmeshed cube), faces per brick, and the axis bits of used edges at their
// lower samples
__global__ void __launch_bounds__(512) mc_classify_kernel(const __grid_constant__ MeshArgs a, unsigned char* cases,
                                                          unsigned* edge_bits, int* brick_faces) {
  __shared__ int nb[8];
  const int b = blockIdx.x, t = threadIdx.x;
  load_neighbours(a, b, nb);
  long long g[8];
  int cs = cube_case(a, nb, t, g);
  cs = cs < 0 ? 0 : cs;
  const int ntri = kMcNumTris[cs];
  cases[static_cast<long long>(b) * kSamples + t] = static_cast<unsigned char>(cs);
  if (ntri > 0) {
    // every crossing edge of a meshed cube is used by its triangles
    for (int e = 0; e < 12; ++e) {
      const int lc = edge_lower_corner(e), uc = lc | (1 << (e >> 2));
      if (((cs >> lc) ^ (cs >> uc)) & 1) atomicOr(edge_bits + g[lc], 1u << (e >> 2));
    }
  }
  int all;
  block_scan_512(ntri, &all);
  if (t == 0) brick_faces[b] = all;
}

// grid B, 512 threads: vertices per brick
__global__ void __launch_bounds__(512) mc_count_kernel(const unsigned* edge_bits, int* brick_verts) {
  const int b = blockIdx.x;
  int all;
  block_scan_512(__popc(edge_bits[static_cast<long long>(b) * kSamples + threadIdx.x]), &all);
  if (threadIdx.x == 0) brick_verts[b] = all;
}

// grid B, 512 threads: the vertices of sample t's used edges, axes in order, from voff[b]; vbase[sample] = its first
__global__ void __launch_bounds__(512) mc_vertices_kernel(const __grid_constant__ MeshArgs a, const unsigned* edge_bits,
                                                          const long long* voff, long long cap, unsigned* vbase,
                                                          float* verts, float* vcols) {
  __shared__ int nb[8];
  const int b = blockIdx.x, t = threadIdx.x;
  load_neighbours(a, b, nb);
  const long long s = static_cast<long long>(b) * kSamples + t;
  const unsigned bits = edge_bits[s];
  int all;
  long long o = voff[b] + block_scan_512(__popc(bits), &all);
  vbase[s] = static_cast<unsigned>(o);
  if (!bits) return;
  int bx, by, bz;
  key_brick(static_cast<unsigned long long>(a.keys[b]), bx, by, bz);
  const int x = t & 7, y = t >> 3 & 7, z = t >> 6;
  const int ii[3] = {kBrick * bx + x, kBrick * by + y, kBrick * bz + z};
  const float Ta = a.tsdf[s];
  for (int axis = 0; axis < 3; ++axis) {
    if (!(bits >> axis & 1)) continue;
    const long long n = sample_at(nb, x + (axis == 0), y + (axis == 1), z + (axis == 2));
    const float Tb = a.tsdf[n], f = Ta / (Ta - Tb);
    if (o < cap) {
      for (int c = 0; c < 3; ++c) {
        const float pa = static_cast<float>(ii[c]) * a.vox;
        verts[o * 3 + c] = c == axis ? pa + f * (static_cast<float>(ii[c] + 1) * a.vox - pa) : pa;
        const float ca = a.color[s * 3 + c];
        vcols[o * 3 + c] = ca + f * (a.color[n * 3 + c] - ca);
      }
    }
    ++o;
  }
}

// grid B, 512 threads: the triangles of cube t from foff[b], as vertex ids of their edges
__global__ void __launch_bounds__(512) mc_faces_kernel(const __grid_constant__ MeshArgs a, const unsigned char* cases,
                                                       const unsigned* edge_bits, const unsigned* vbase,
                                                       const long long* foff, long long cap, int32_t* faces) {
  __shared__ int nb[8];
  const int b = blockIdx.x, t = threadIdx.x;
  load_neighbours(a, b, nb);
  const int cs = cases[static_cast<long long>(b) * kSamples + t], ntri = kMcNumTris[cs];
  int all;
  const long long o = foff[b] + block_scan_512(ntri, &all);
  const int x = t & 7, y = t >> 3 & 7, z = t >> 6;
  for (int k = 0; k < ntri; ++k) {
    if (o + k >= cap) break;
    for (int j = 0; j < 3; ++j) {
      const int e = kMcTris[cs][3 * k + j], lc = edge_lower_corner(e), axis = e >> 2;
      const long long g = sample_at(nb, x + (lc & 1), y + (lc >> 1 & 1), z + (lc >> 2));
      faces[(o + k) * 3 + j] = static_cast<int32_t>(vbase[g] + __popc(edge_bits[g] & ((1u << axis) - 1u)));
    }
  }
}

struct MeshScratch {
  unsigned char* cases;
  unsigned* edge_bits;
  unsigned* vbase;
  int* brick_counts;  // [2][B]: vertices, faces
  long long* offs;    // [2][B + 1]
};

size_t mesh_scratch(long long B, MeshScratch* s, void* base) {
  char* p = static_cast<char*>(base);
  long long o = 0;
  auto take = [&](long long bytes) {
    char* q = p + o;
    o += align16(bytes);
    return q;
  };
  char* a = take(B * kSamples);
  char* b = take(4 * B * kSamples);
  char* c = take(4 * B * kSamples);
  char* d = take(8 * (B + 1));
  char* e = take(16 * (B + 1));
  if (s) *s = {reinterpret_cast<unsigned char*>(a), reinterpret_cast<unsigned*>(b), reinterpret_cast<unsigned*>(c),
               reinterpret_cast<int*>(d), reinterpret_cast<long long*>(e)};
  return static_cast<size_t>(o);
}

bool fusion_sizes_ok(int V, int H, int W) {
  return V >= 1 && V <= 65535 && H >= 1 && H <= 65535 && W >= 1 && W <= 65535;
}

bool voxel_ok(float vox, float tau) {
  return isfinite(vox) && vox > 0.f && tau > 0.f && tau <= 4.f * vox;
}

}  // namespace
}  // namespace sta

using namespace sta;

extern "C" {

size_t sta_fusion_bricks_scratch_bytes(int V, int H, int W, int64_t key_capacity) {
  if (!fusion_sizes_ok(V, H, W) || key_capacity < 0 || key_capacity >= (1ll << 31)) return 0;
  return brick_scratch(V, H, W, key_capacity, nullptr, nullptr);
}

int sta_fusion_bricks(const float* depth, const float* conf, const float* pose44, const float* scale, const float* intri,
                      int V, int H, int W, float conf_thres, float voxel, float trunc, int64_t key_capacity,
                      void* scratch, size_t scratch_bytes, int64_t* keys_out, int64_t* counts_out, void* stream) {
  STA_REQUIRE(fusion_sizes_ok(V, H, W), "V, H and W must lie in [1, 65535]");
  STA_REQUIRE(voxel_ok(voxel, trunc), "voxel size must be positive and finite, trunc in (0, 4 voxel]");
  STA_REQUIRE(key_capacity >= 0 && key_capacity < (1ll << 31), "key capacity outside [0, 2^31)");
  STA_REQUIRE(depth && conf && pose44 && scale && intri && counts_out, "null map input or counts");
  STA_REQUIRE(key_capacity == 0 || keys_out, "null keys_out with a nonzero key capacity");
  STA_REQUIRE(scratch != nullptr && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0, "null or misaligned scratch");
  STA_REQUIRE(scratch_bytes >= sta_fusion_bricks_scratch_bytes(V, H, W, key_capacity),
              "scratch smaller than sta_fusion_bricks_scratch_bytes");
  STA_REQUIRE(on_device(depth) && on_device(conf) && on_device(pose44) && on_device(scale) && on_device(intri) &&
                  on_device(counts_out) && on_device(scratch) && (key_capacity == 0 || on_device(keys_out)),
              "every array must be device memory");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  BrickScratch s;
  brick_scratch(V, H, W, key_capacity, &s, scratch);
  const MapArgs m{depth, conf, pose44, scale, intri, nullptr, nullptr, V, H, W, conf_thres};
  const dim3 grid((W + 255) / 256, H, V);
  const long long tiles = num_tiles(V, H, W);
  brick_keys_kernel<<<grid, 256, 0, st>>>(m, voxel, trunc, s.tile_counts, nullptr, nullptr, 0);
  STA_CHECK_CUDA(cudaGetLastError());
  row_scan_kernel<<<1, 1024, 0, st>>>(s.tile_counts, tiles, s.tile_off, counts_out);
  STA_CHECK_CUDA(cudaGetLastError());
  STA_CHECK_CUDA(cudaMemsetAsync(counts_out + 1, 0, sizeof(int64_t), st));
  if (key_capacity == 0) return 0;
  // keys beyond the count (a capacity larger than it) stay empty and sort last
  STA_CHECK_CUDA(cudaMemsetAsync(s.keys, 0xff, 8 * key_capacity, st));
  brick_keys_kernel<<<grid, 256, 0, st>>>(m, voxel, trunc, nullptr, s.tile_off, s.keys, key_capacity);
  STA_CHECK_CUDA(cudaGetLastError());
  const int rc = sta_op_radix_sort(reinterpret_cast<const uint64_t*>(s.keys), nullptr, key_capacity, 64,
                                   reinterpret_cast<uint64_t*>(s.keys), s.idx, s.sort, stream);
  if (rc != 0) return rc;
  const long long chunks = (key_capacity + kUniqueChunk - 1) / kUniqueChunk;
  unique_kernel<<<static_cast<unsigned>(chunks), 256, 0, st>>>(s.keys, key_capacity, s.chunk_counts, nullptr, nullptr);
  STA_CHECK_CUDA(cudaGetLastError());
  row_scan_kernel<<<1, 1024, 0, st>>>(s.chunk_counts, chunks, s.chunk_off, counts_out + 1);
  STA_CHECK_CUDA(cudaGetLastError());
  unique_kernel<<<static_cast<unsigned>(chunks), 256, 0, st>>>(s.keys, key_capacity, nullptr, s.chunk_off, keys_out);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

size_t sta_fusion_integrate_scratch_bytes(int64_t num_bricks, int V) {
  if (num_bricks < 0 || num_bricks > STA_FUSION_MAX_BRICKS || V < 1 || V > 65535) return 0;
  return static_cast<size_t>(align16(4ll * V) + 4ll * num_bricks * ((V + 31) / 32));
}

int sta_fusion_integrate(const float* depth, const float* conf, const float* scale, const float* intri, const float* imgs,
                         const float* w2c, int V, int H, int W, float conf_thres, const int64_t* keys, int64_t num_bricks,
                         float voxel, float trunc, void* scratch, size_t scratch_bytes, float* tsdf_out,
                         float* weight_out, float* color_out, void* stream) {
  STA_REQUIRE(fusion_sizes_ok(V, H, W), "V, H and W must lie in [1, 65535]");
  STA_REQUIRE(voxel_ok(voxel, trunc), "voxel size must be positive and finite, trunc in (0, 4 voxel]");
  STA_REQUIRE(num_bricks >= 0 && num_bricks <= STA_FUSION_MAX_BRICKS, "brick count outside [0, STA_FUSION_MAX_BRICKS]");
  if (num_bricks == 0) return 0;
  STA_REQUIRE(depth && conf && scale && intri && imgs && w2c && keys, "null input");
  STA_REQUIRE(tsdf_out && weight_out && color_out, "null output");
  STA_REQUIRE(scratch != nullptr && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0, "null or misaligned scratch");
  STA_REQUIRE(scratch_bytes >= sta_fusion_integrate_scratch_bytes(num_bricks, V),
              "scratch smaller than sta_fusion_integrate_scratch_bytes");
  STA_REQUIRE(on_device(depth) && on_device(conf) && on_device(scale) && on_device(intri) && on_device(imgs) &&
                  on_device(w2c) && on_device(keys) && on_device(scratch) && on_device(tsdf_out) &&
                  on_device(weight_out) && on_device(color_out),
              "every array must be device memory");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* dmax = static_cast<float*>(scratch);
  unsigned* mask = reinterpret_cast<unsigned*>(static_cast<char*>(scratch) + align16(4ll * V));
  const int words = (V + 31) / 32;
  const MapArgs m{depth, conf, nullptr, scale, intri, imgs, w2c, V, H, W, conf_thres};
  view_depth_kernel<<<V, 256, 0, st>>>(m, dmax);
  STA_CHECK_CUDA(cudaGetLastError());
  brick_views_kernel<<<static_cast<unsigned>(num_bricks), 128, 0, st>>>(m, keys, voxel, trunc, dmax, words, mask);
  STA_CHECK_CUDA(cudaGetLastError());
  integrate_kernel<<<static_cast<unsigned>(num_bricks), kSamples, 0, st>>>(m, keys, voxel, trunc, words, mask, tsdf_out,
                                                                           weight_out, color_out);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

size_t sta_fusion_mesh_scratch_bytes(int64_t num_bricks) {
  if (num_bricks < 0 || num_bricks > STA_FUSION_MAX_BRICKS) return 0;
  return mesh_scratch(num_bricks, nullptr, nullptr);
}

int sta_fusion_mesh(const int64_t* keys, int64_t num_bricks, const float* tsdf, const float* weight, const float* color,
                    float voxel, float min_weight, int64_t max_vertices, int64_t max_faces, void* scratch,
                    size_t scratch_bytes, float* vertices_out, float* vertex_colors_out, int32_t* faces_out,
                    int64_t* counts_out, void* stream) {
  STA_REQUIRE(num_bricks >= 0 && num_bricks <= STA_FUSION_MAX_BRICKS, "brick count outside [0, STA_FUSION_MAX_BRICKS]");
  STA_REQUIRE(isfinite(voxel) && voxel > 0.f, "voxel size must be positive and finite");
  STA_REQUIRE(min_weight >= 1.f, "min_weight must be at least 1");
  STA_REQUIRE(max_vertices >= 0 && max_faces >= 0, "negative capacity");
  STA_REQUIRE(counts_out != nullptr, "null counts");
  STA_REQUIRE(num_bricks == 0 || (keys && tsdf && weight && color), "null volume");
  STA_REQUIRE(max_vertices == 0 || (vertices_out && vertex_colors_out), "null vertex output with a nonzero capacity");
  STA_REQUIRE(max_faces == 0 || faces_out, "null face output with a nonzero capacity");
  STA_REQUIRE(scratch != nullptr && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0, "null or misaligned scratch");
  STA_REQUIRE(scratch_bytes >= sta_fusion_mesh_scratch_bytes(num_bricks), "scratch smaller than sta_fusion_mesh_scratch_bytes");
  STA_REQUIRE(on_device(counts_out) && on_device(scratch) &&
                  (num_bricks == 0 || (on_device(keys) && on_device(tsdf) && on_device(weight) && on_device(color))) &&
                  (max_vertices == 0 || (on_device(vertices_out) && on_device(vertex_colors_out))) &&
                  (max_faces == 0 || on_device(faces_out)),
              "every array must be device memory");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (num_bricks == 0) {
    STA_CHECK_CUDA(cudaMemsetAsync(counts_out, 0, 2 * sizeof(int64_t), st));
    return 0;
  }
  MeshScratch s;
  mesh_scratch(num_bricks, &s, scratch);
  const MeshArgs a{keys, num_bricks, tsdf, weight, color, voxel, min_weight};
  const unsigned B = static_cast<unsigned>(num_bricks);
  int* bverts = s.brick_counts;
  int* bfaces = s.brick_counts + num_bricks;
  long long* voff = s.offs;
  long long* foff = s.offs + num_bricks + 1;
  STA_CHECK_CUDA(cudaMemsetAsync(s.edge_bits, 0, 4 * num_bricks * kSamples, st));
  mc_classify_kernel<<<B, kSamples, 0, st>>>(a, s.cases, s.edge_bits, bfaces);
  STA_CHECK_CUDA(cudaGetLastError());
  mc_count_kernel<<<B, kSamples, 0, st>>>(s.edge_bits, bverts);
  STA_CHECK_CUDA(cudaGetLastError());
  row_scan_kernel<<<1, 1024, 0, st>>>(bverts, num_bricks, voff, counts_out);
  STA_CHECK_CUDA(cudaGetLastError());
  row_scan_kernel<<<1, 1024, 0, st>>>(bfaces, num_bricks, foff, counts_out + 1);
  STA_CHECK_CUDA(cudaGetLastError());
  if (max_vertices == 0 && max_faces == 0) return 0;
  mc_vertices_kernel<<<B, kSamples, 0, st>>>(a, s.edge_bits, voff, max_vertices, s.vbase, vertices_out, vertex_colors_out);
  STA_CHECK_CUDA(cudaGetLastError());
  if (max_faces > 0) {
    mc_faces_kernel<<<B, kSamples, 0, st>>>(a, s.cases, s.edge_bits, s.vbase, foff, max_faces, faces_out);
    STA_CHECK_CUDA(cudaGetLastError());
  }
  return 0;
}

}  // extern "C"
