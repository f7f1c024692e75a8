// Reconstruction evaluation (vista_slam/eval/eval_recon.py:108-206) on the device: the ground-truth and estimated world
// clouds, open3d's voxel_down_sample, the moments of open3d's point-to-point ICP, and the nearest-neighbour distances of
// the Chamfer metric.
//
//   radix sort     stable LSD sort of (u64 key, u32 index) pairs, 8 bits per pass over the significant bits only:
//                  per-block digit histograms, one exclusive scan over (digit, block), then a scatter that ranks equal
//                  digits inside a block with __match_any_sync, warp by warp, so the sort is stable.
//   voxels         key = floor((p - min_bound) / v) per axis in fp64, sorted by (kx, ky, kz); each voxel's point is the
//                  fp64 sum of its points in input order (the sort is stable) divided by their count.
//   nn index       points sorted by a 63-bit Morton code over the cloud's box; leaves of 32 consecutive points under an
//                  implicit complete binary tree of fp64 boxes, built bottom-up.  A query starts from best = r^2, prunes
//                  every node whose box is not nearer than best, and accepts a point only when d^2 < best.  Distances
//                  are (dx dx + dy dy) + dz dz, each operation rounded on its own (no FMA contraction): a box's distance
//                  is then never above that of a point inside it, so pruning never loses the exact minimum, whatever the
//                  tree's shape.  Queries run in the Morton order of the query cloud and are scattered back.
//   reductions     fixed order (contiguous ranges within a block, blocks in order), no floating-point atomics: repeated
//                  runs are bit-identical.
#include <float.h>
#include <limits.h>
#include <math.h>

#include <string>

#include "../../include/sta_b200.h"
#include "cloud.cuh"
#include "host_util.h"

struct StaNnIndex {
  long long n = 0;
  int leaves = 0, P = 0;     // leaves = ceil(n / 32); P = leaves rounded up to a power of two
  double* x = nullptr;       // [n] sorted coordinates (SoA)
  double* y = nullptr;
  double* z = nullptr;
  uint32_t* id = nullptr;    // [n] input index of each sorted point
  double* box = nullptr;     // [2P][6] lo xyz, hi xyz; node 1 is the root, leaves are P .. 2P - 1
  double* bb = nullptr;      // [6] the cloud's box
};

namespace sta {
namespace {

constexpr int kTile = 2048;       // keys per sort block: 256 threads x 8
constexpr int kScanTile = 4096;   // elements per scan block: 256 threads x 16
constexpr int kRedBlocks = 256;   // partial records per reduction
constexpr int kRedVals = 16;      // doubles per record
constexpr int kLeaf = 32;

__device__ __forceinline__ double dist2(double ax, double ay, double az, double bx, double by, double bz) {
  const double dx = __dsub_rn(ax, bx), dy = __dsub_rn(ay, by), dz = __dsub_rn(az, bz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// ---------------------------------------------------------------------------------------------------------- scan

// exclusive scan of m u32 values in place; bsum has room for ceil(m / kScanTile) + 1 values
__global__ void __launch_bounds__(256) scan_reduce_kernel(const unsigned* v, long long m, unsigned* bsum) {
  const long long base = static_cast<long long>(blockIdx.x) * kScanTile;
  unsigned t = 0;
  for (int k = threadIdx.x; k < kScanTile; k += 256)
    if (base + k < m) t += v[base + k];
  t = __reduce_add_sync(0xffffffffu, t);
  __shared__ unsigned ws[8];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned s = 0;
    for (int w = 0; w < 8; ++w) s += ws[w];
    bsum[blockIdx.x] = s;
  }
}

__global__ void __launch_bounds__(1024) scan_top_kernel(unsigned* bsum, long long nb) {
  __shared__ unsigned part[1024];
  const long long per = (nb + 1023) / 1024;
  const long long lo = threadIdx.x * per, hi = min(nb, lo + per);
  unsigned t = 0;
  for (long long i = lo; i < hi; ++i) t += bsum[i];
  part[threadIdx.x] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned run = 0;
    for (int i = 0; i < 1024; ++i) {
      const unsigned c = part[i];
      part[i] = run;
      run += c;
    }
    bsum[nb] = run;
  }
  __syncthreads();
  unsigned run = part[threadIdx.x];
  for (long long i = lo; i < hi; ++i) {
    const unsigned c = bsum[i];
    bsum[i] = run;
    run += c;
  }
}

__global__ void __launch_bounds__(256) scan_down_kernel(unsigned* v, long long m, const unsigned* bsum) {
  const long long base = static_cast<long long>(blockIdx.x) * kScanTile + threadIdx.x * 16;
  unsigned loc[16], t = 0;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    loc[k] = base + k < m ? v[base + k] : 0u;
    t += loc[k];
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned inc = t;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  __shared__ unsigned ws[8];
  if (lane == 31) ws[warp] = inc;
  __syncthreads();
  unsigned run = bsum[blockIdx.x] + inc - t;
  for (int w = 0; w < warp; ++w) run += ws[w];
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    if (base + k < m) v[base + k] = run;
    run += loc[k];
  }
}

long long scan_blocks(long long m) { return (m + kScanTile - 1) / kScanTile; }

// in-place exclusive scan; the total lands in bsum[scan_blocks(m)]
cudaError_t scan_u32(unsigned* v, long long m, unsigned* bsum, cudaStream_t st) {
  const long long nb = scan_blocks(m);
  if (nb == 0) return cudaMemsetAsync(bsum, 0, sizeof(unsigned), st);
  scan_reduce_kernel<<<static_cast<unsigned>(nb), 256, 0, st>>>(v, m, bsum);
  scan_top_kernel<<<1, 1024, 0, st>>>(bsum, nb);
  scan_down_kernel<<<static_cast<unsigned>(nb), 256, 0, st>>>(v, m, bsum);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------- sort

__device__ __forceinline__ unsigned digit_of(uint64_t k, int shift, int bits) {
  return static_cast<unsigned>(k >> shift) & ((1u << bits) - 1u);
}

// hist[d * nb + block] = number of keys of the block with digit d
__global__ void __launch_bounds__(256) sort_hist_kernel(const uint64_t* keys, long long n, int shift, int bits, unsigned* hist,
                                                        long long nb) {
  __shared__ unsigned h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const long long base = static_cast<long long>(blockIdx.x) * kTile;
  for (int k = 0; k < kTile / 256; ++k) {
    const long long i = base + k * 256 + threadIdx.x;
    if (i < n) atomicAdd(&h[digit_of(keys[i], shift, bits)], 1u);
  }
  __syncthreads();
  hist[threadIdx.x * nb + blockIdx.x] = h[threadIdx.x];
}

// Stable scatter: keys of a block are ranked in index order, 256 at a time; within 256, by warp then lane.
__global__ void __launch_bounds__(256) sort_scatter_kernel(const uint64_t* kin, const uint32_t* iin, long long n, int shift,
                                                           int bits, const unsigned* offs, long long nb, uint64_t* kout,
                                                           uint32_t* iout) {
  __shared__ unsigned base[256];
  __shared__ unsigned wc[8][256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  base[threadIdx.x] = offs[threadIdx.x * nb + blockIdx.x];
  const long long tile = static_cast<long long>(blockIdx.x) * kTile;
  for (int k = 0; k < kTile / 256; ++k) {
    for (int w = 0; w < 8; ++w) wc[w][threadIdx.x] = 0;
    __syncthreads();
    const long long i = tile + k * 256 + threadIdx.x;
    const bool valid = i < n;
    uint64_t key = 0;
    unsigned d = 256u + lane;  // never equal to a digit, nor to another invalid lane's value
    if (valid) {
      key = kin[i];
      d = digit_of(key, shift, bits);
    }
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const unsigned rank = __popc(peers & ((1u << lane) - 1u));
    if (valid && rank == 0) wc[warp][d] = __popc(peers);
    __syncthreads();
    if (valid) {
      unsigned pos = base[d] + rank;
      for (int w = 0; w < warp; ++w) pos += wc[w][d];
      kout[pos] = key;
      iout[pos] = iin ? iin[i] : static_cast<uint32_t>(i);
    }
    __syncthreads();
    unsigned t = 0;
    for (int w = 0; w < 8; ++w) t += wc[w][threadIdx.x];
    base[threadIdx.x] += t;
  }
}

struct SortScratch {
  uint64_t* keys;
  uint32_t* idx;
  unsigned* hist;
  unsigned* bsum;
};

size_t sort_scratch_bytes(long long n) {
  const long long nb = (n + kTile - 1) / kTile, m = 256 * nb;
  return static_cast<size_t>(8 * n + 4 * n + 4 * m + 4 * (scan_blocks(m) + 2) + 64);
}

SortScratch carve_sort(void* scratch, long long n) {
  const long long nb = (n + kTile - 1) / kTile;
  char* p = static_cast<char*>(scratch);
  SortScratch s;
  s.keys = reinterpret_cast<uint64_t*>(p);
  p += 8 * n;
  s.idx = reinterpret_cast<uint32_t*>(p);
  p += ((4 * n + 15) / 16) * 16;
  s.hist = reinterpret_cast<unsigned*>(p);
  p += 4 * 256 * nb;
  s.bsum = reinterpret_cast<unsigned*>(p);
  return s;
}

__global__ void iota_kernel(uint32_t* idx, long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x)
    idx[i] = static_cast<uint32_t>(i);
}

unsigned grid_for(long long n, int threads = 256) {
  const long long b = (n + threads - 1) / threads;
  return static_cast<unsigned>(b < 1 ? 1 : (b > 65535 * 8 ? 65535 * 8 : b));
}

// keys / idx (idx may be null: 0 .. n-1) -> kout / iout sorted stably by the low nbits of the keys; the outputs may be
// the inputs
cudaError_t radix_sort(const uint64_t* keys, const uint32_t* idx, long long n, int nbits, uint64_t* kout, uint32_t* iout,
                       void* scratch, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  const int passes = (nbits + 7) / 8;
  if (passes == 0) {
    cudaError_t e = kout == keys ? cudaSuccess : cudaMemcpyAsync(kout, keys, 8 * n, cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) return e;
    if (idx) return iout == idx ? cudaSuccess : cudaMemcpyAsync(iout, idx, 4 * n, cudaMemcpyDeviceToDevice, st);
    iota_kernel<<<grid_for(n), 256, 0, st>>>(iout, n);
    return cudaGetLastError();
  }
  SortScratch s = carve_sort(scratch, n);
  const long long nb = (n + kTile - 1) / kTile;
  const uint64_t* ksrc = keys;
  const uint32_t* isrc = idx;
  if ((passes & 1) && (keys == kout || (idx && idx == iout))) {  // the first pass writes the outputs: read a copy
    cudaError_t e = cudaMemcpyAsync(s.keys, keys, 8 * n, cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess && idx) e = cudaMemcpyAsync(s.idx, idx, 4 * n, cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) return e;
    ksrc = s.keys;
    isrc = idx ? s.idx : nullptr;
  }
  for (int p = 0; p < passes; ++p) {
    const int shift = 8 * p, bits = min(8, nbits - shift);
    const bool to_out = ((passes - 1 - p) & 1) == 0;  // the last pass writes the outputs
    uint64_t* kd = to_out ? kout : s.keys;
    uint32_t* id = to_out ? iout : s.idx;
    sort_hist_kernel<<<static_cast<unsigned>(nb), 256, 0, st>>>(ksrc, n, shift, bits, s.hist, nb);
    cudaError_t e = scan_u32(s.hist, 256 * nb, s.bsum, st);
    if (e != cudaSuccess) return e;
    sort_scatter_kernel<<<static_cast<unsigned>(nb), 256, 0, st>>>(ksrc, isrc, n, shift, bits, s.hist, nb, kd, id);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    ksrc = kd;
    isrc = id;
  }
  return cudaSuccess;
}

// ---------------------------------------------------------------------------------------------------------- reductions

// record[b] of kRedBlocks: thread t sums a contiguous range of block b's contiguous range, thread 0 sums the threads in
// order.  F::vals values per element.
template <class F>
__global__ void __launch_bounds__(256) reduce_partial_kernel(long long n, F f, double* partial) {
  constexpr int K = F::vals;
  __shared__ double red[256][K];
  const long long per_block = (n + kRedBlocks - 1) / kRedBlocks;
  const long long b0 = blockIdx.x * per_block, b1 = min(n, b0 + per_block);
  const long long per_thread = (per_block + 255) / 256;
  const long long t0 = b0 + threadIdx.x * per_thread, t1 = min(b1, t0 + per_thread);
  double s[K];
  for (int k = 0; k < K; ++k) s[k] = 0.0;
  for (long long i = t0; i < t1; ++i) f(i, s);
  for (int k = 0; k < K; ++k) red[threadIdx.x][k] = s[k];
  __syncthreads();
  if (threadIdx.x < K) {
    double t = 0.0;
    for (int w = 0; w < 256; ++w) t = __dadd_rn(t, red[w][threadIdx.x]);
    partial[blockIdx.x * kRedVals + threadIdx.x] = t;
  }
}

// out[k] = sum of the records in block order, times scale[k] when scale is given
__global__ void reduce_final_kernel(const double* partial, int K, double* out) {
  const int k = threadIdx.x;
  if (k >= K) return;
  double t = 0.0;
  for (int b = 0; b < kRedBlocks; ++b) t = __dadd_rn(t, partial[b * kRedVals + k]);
  out[k] = t;
}

// count, sum d^2, sum src, sum dst over the points with a correspondence
struct MomentsA {
  static constexpr int vals = 8;
  const double* src;
  const double* dst;
  const int64_t* corr;
  __device__ void operator()(long long i, double* s) const {
    const int64_t j = corr[i];
    if (j < 0) return;
    const double* a = src + 3 * i;
    const double* b = dst + 3 * j;
    s[0] += 1.0;
    s[1] = __dadd_rn(s[1], dist2(a[0], a[1], a[2], b[0], b[1], b[2]));
    for (int c = 0; c < 3; ++c) {
      s[2 + c] = __dadd_rn(s[2 + c], a[c]);
      s[5 + c] = __dadd_rn(s[5 + c], b[c]);
    }
  }
};

// centred cross-covariance sum (dst - mean_dst)(src - mean_src)^T, row-major; means = sums / count from pass A
struct MomentsB {
  static constexpr int vals = 9;
  const double* src;
  const double* dst;
  const int64_t* corr;
  const double* a;  // the 8 sums of pass A
  __device__ void operator()(long long i, double* s) const {
    const int64_t j = corr[i];
    if (j < 0) return;
    const double n = a[0];
    double xs[3], ys[3];
    for (int c = 0; c < 3; ++c) {
      xs[c] = __dsub_rn(src[3 * i + c], __ddiv_rn(a[2 + c], n));
      ys[c] = __dsub_rn(dst[3 * j + c], __ddiv_rn(a[5 + c], n));
    }
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) s[r * 3 + c] = __dadd_rn(s[r * 3 + c], __dmul_rn(ys[r], xs[c]));
  }
};

struct SumSqClipped {
  static constexpr int vals = 1;
  const double* d;
  double clip;
  __device__ void operator()(long long i, double* s) const {
    const double v = fmin(fmax(d[i], 0.0), clip);
    s[0] = __dadd_rn(s[0], __dmul_rn(v, v));
  }
};

template <class F>
cudaError_t reduce(long long n, F f, double* partial, double* out, cudaStream_t st) {
  reduce_partial_kernel<F><<<kRedBlocks, 256, 0, st>>>(n, f, partial);
  reduce_final_kernel<<<1, 32, 0, st>>>(partial, F::vals, out);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------- boxes

// partial boxes per block, then one thread combines (min / max are exact in any order)
__global__ void __launch_bounds__(256) bbox_partial_kernel(const double* p, long long n, double* part) {
  double lo[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, hi[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX};
  for (long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * 256)
    for (int c = 0; c < 3; ++c) {
      lo[c] = fmin(lo[c], p[3 * i + c]);
      hi[c] = fmax(hi[c], p[3 * i + c]);
    }
  __shared__ double s[256][6];
  for (int c = 0; c < 3; ++c) {
    s[threadIdx.x][c] = lo[c];
    s[threadIdx.x][3 + c] = hi[c];
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    double v = s[0][threadIdx.x];
    for (int t = 1; t < 256; ++t) v = threadIdx.x < 3 ? fmin(v, s[t][threadIdx.x]) : fmax(v, s[t][threadIdx.x]);
    part[blockIdx.x * 6 + threadIdx.x] = v;
  }
}

__global__ void bbox_final_kernel(const double* part, int nb, double* bb) {
  const int c = threadIdx.x;
  if (c >= 6) return;
  double v = part[c];
  for (int b = 1; b < nb; ++b) v = c < 3 ? fmin(v, part[b * 6 + c]) : fmax(v, part[b * 6 + c]);
  bb[c] = v;
}

constexpr int kBoxBlocks = 264;

cudaError_t bbox(const double* p, long long n, double* part, double* bb, cudaStream_t st) {
  bbox_partial_kernel<<<kBoxBlocks, 256, 0, st>>>(p, n, part);
  bbox_final_kernel<<<1, 32, 0, st>>>(part, kBoxBlocks, bb);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------- voxels

struct VoxelGrid {
  double mn[3], v;
  int shift[3];  // packed key = kx << shift[0] | ky << shift[1] | kz << shift[2]; shift < 0: the axis is left out
};

__device__ __forceinline__ long long voxel_coord(double p, double mn, double v) {
  return static_cast<long long>(floor(__ddiv_rn(__dsub_rn(p, mn), v)));
}

// key of point idx[i] (idx null: i)
__global__ void voxel_key_kernel(const double* p, const uint32_t* idx, long long n, VoxelGrid g, uint64_t* key) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long j = idx ? idx[i] : i;
    uint64_t k = 0;
    for (int c = 0; c < 3; ++c)
      if (g.shift[c] >= 0) k |= static_cast<uint64_t>(voxel_coord(p[3 * j + c], g.mn[c], g.v)) << g.shift[c];
    key[i] = k;
  }
}

// head[i] = 1 where sorted point i starts a voxel
__global__ void voxel_head_kernel(const double* p, const uint32_t* idx, long long n, VoxelGrid g, unsigned* head) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    bool h = i == 0;
    if (!h) {
      const long long a = idx[i], b = idx[i - 1];
      for (int c = 0; c < 3; ++c) h = h || voxel_coord(p[3 * a + c], g.mn[c], g.v) != voxel_coord(p[3 * b + c], g.mn[c], g.v);
    }
    head[i] = h;
  }
}

// start[s] = first sorted position of voxel s, start[nv] = n (head_scan: exclusive scan of the head flags)
__global__ void voxel_start_kernel(const unsigned* head_scan, long long n, const unsigned* total, unsigned* start) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const unsigned s = head_scan[i];
    if ((i + 1 < n ? head_scan[i + 1] : *total) != s) start[s] = static_cast<unsigned>(i);  // i is a head
    if (i == 0) start[*total] = static_cast<unsigned>(n);
  }
}

// voxel j: sorted points start[j] .. start[j + 1] - 1, summed in input order (the sort is stable)
__global__ void voxel_sum_kernel(const double* p, const uint32_t* idx, const unsigned* start, long long nv, double* out) {
  for (long long j = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; j < nv; j += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = start[j], e = start[j + 1];
    double s[3] = {0.0, 0.0, 0.0};
    for (long long i = b; i < e; ++i)
      for (int c = 0; c < 3; ++c) s[c] = __dadd_rn(s[c], p[3 * static_cast<long long>(idx[i]) + c]);
    const double cnt = static_cast<double>(e - b);
    for (int c = 0; c < 3; ++c) out[3 * j + c] = __ddiv_rn(s[c], cnt);
  }
}

int bit_width(long long v) {
  int b = 0;
  while (v > 0) {
    ++b;
    v >>= 1;
  }
  return b;
}

// ---------------------------------------------------------------------------------------------------------- nn index

__device__ __forceinline__ uint64_t spread3(uint64_t v) {  // 21 bits -> every third bit
  v &= 0x1fffffull;
  v = (v | v << 32) & 0x1f00000000ffffull;
  v = (v | v << 16) & 0x1f0000ff0000ffull;
  v = (v | v << 8) & 0x100f00f00f00f00full;
  v = (v | v << 4) & 0x10c30c30c30c30c3ull;
  v = (v | v << 2) & 0x1249249249249249ull;
  return v;
}

__device__ __forceinline__ uint64_t morton63(const double* p, const double* bb) {
  uint64_t code = 0;
  for (int c = 0; c < 3; ++c) {
    const double ext = bb[3 + c] - bb[c];
    double t = ext > 0.0 ? (p[c] - bb[c]) / ext * 2097152.0 : 0.0;
    t = fmin(fmax(t, 0.0), 2097151.0);  // also maps NaN to 0
    code |= spread3(static_cast<uint64_t>(t)) << (2 - c);
  }
  return code;
}

__global__ void morton_kernel(const double* p, long long n, const double* bb, int shift, uint64_t* code) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x)
    code[i] = morton63(p + 3 * i, bb) >> shift;
}

__global__ void nn_gather_kernel(const double* p, const uint32_t* order, long long n, double* x, double* y, double* z) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long j = order[i];
    x[i] = p[3 * j];
    y[i] = p[3 * j + 1];
    z[i] = p[3 * j + 2];
  }
}

__global__ void nn_leaf_kernel(StaNnIndex ix) {
  for (long long l = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; l < ix.P; l += static_cast<long long>(gridDim.x) * blockDim.x) {
    double b[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};  // empty: farther than anything
    const long long i0 = l * kLeaf, i1 = min(ix.n, i0 + kLeaf);
    for (long long i = i0; i < i1; ++i) {
      const double q[3] = {ix.x[i], ix.y[i], ix.z[i]};
      for (int c = 0; c < 3; ++c) {
        b[c] = fmin(b[c], q[c]);
        b[3 + c] = fmax(b[3 + c], q[c]);
      }
    }
    for (int c = 0; c < 6; ++c) ix.box[(ix.P + l) * 6 + c] = b[c];
  }
}

// nodes lvl .. 2 lvl - 1 from their children
__global__ void nn_level_kernel(double* box, long long lvl) {
  for (long long k = lvl + static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; k < 2 * lvl; k += static_cast<long long>(gridDim.x) * blockDim.x)
    for (int c = 0; c < 6; ++c) {
      const double a = box[2 * k * 6 + c], b = box[(2 * k + 1) * 6 + c];
      box[k * 6 + c] = c < 3 ? fmin(a, b) : fmax(a, b);
    }
}

__device__ __forceinline__ double box_dist2(const double* b, double qx, double qy, double qz) {
  const double dx = fmax(fmax(__dsub_rn(b[0], qx), __dsub_rn(qx, b[3])), 0.0);
  const double dy = fmax(fmax(__dsub_rn(b[1], qy), __dsub_rn(qy, b[4])), 0.0);
  const double dz = fmax(fmax(__dsub_rn(b[2], qz), __dsub_rn(qz, b[5])), 0.0);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// query order[i] (Morton order of the queries); results scattered back to the query's own position
__global__ void __launch_bounds__(128) nn_query_kernel(StaNnIndex ix, const double* q, const uint32_t* order, long long nq,
                                                       double r, double* dist, int64_t* idx) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= nq) return;
  const long long j = order[i];
  const double qx = q[3 * j], qy = q[3 * j + 1], qz = q[3 * j + 2];
  double best = __dmul_rn(r, r);
  long long bi = -1;
  if (ix.n > 0) {
    int stack[64];
    int sp = 0;
    stack[sp++] = 1;
    while (sp > 0) {
      const int node = stack[--sp];
      if (!(box_dist2(ix.box + node * 6, qx, qy, qz) < best)) continue;
      if (node >= ix.P) {
        const long long i0 = static_cast<long long>(node - ix.P) * kLeaf, i1 = min(ix.n, i0 + kLeaf);
        for (long long k = i0; k < i1; ++k) {
          const double d = dist2(ix.x[k], ix.y[k], ix.z[k], qx, qy, qz);
          if (d < best) {
            best = d;
            bi = k;
          }
        }
      } else {
        const int a = 2 * node, b = a + 1;
        const double da = box_dist2(ix.box + a * 6, qx, qy, qz), db = box_dist2(ix.box + b * 6, qx, qy, qz);
        const bool a_near = da <= db;
        const int near = a_near ? a : b, far = a_near ? b : a;
        const double dn = a_near ? da : db, df = a_near ? db : da;
        if (df < best) stack[sp++] = far;
        if (dn < best) stack[sp++] = near;
      }
    }
  }
  dist[j] = bi >= 0 ? sqrt(best) : r;
  idx[j] = bi >= 0 ? static_cast<int64_t>(ix.id[bi]) : -1;
}

// ---------------------------------------------------------------------------------------------------------- transform

struct Affine {
  double m[12];
};

// p <- M[:, :3] p + M[:, 3], each operation rounded on its own
__global__ void transform_kernel(double* p, long long n, Affine a) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const double x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
    for (int r = 0; r < 3; ++r) {
      const double* m = a.m + 4 * r;
      p[3 * i + r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[0], x), __dmul_rn(m[1], y)), __dmul_rn(m[2], z)), m[3]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------- clouds

struct CloudArgs {
  int N, H, W;
  float thres;
  const float* gt_depth;  // [N][H][W]
  const float* gt_pose;   // [N][4][4]
  const float* gt_intri;  // [3][3], shared
  const float* depth;     // [N][H][W]
  const float* scale;     // [N] or null
  const float* pose;      // [N][4][4]
  const float* intri;     // [N][3][3]
  const float* conf;      // [N][H][W]
};

// cloud 0: gt_depth > 0; cloud 1: conf > thres and gt_depth > 0
__device__ __forceinline__ bool cloud_keep(const CloudArgs& a, int z, long long i) {
  return a.gt_depth[i] > 0.f && (z == 0 || a.conf[i] > a.thres);
}

// grid (H, N, 2), 256 threads
__global__ void __launch_bounds__(256) cloud_count_kernel(CloudArgs a, int* counts) {
  const int row = blockIdx.x, v = blockIdx.y, z = blockIdx.z;
  const long long r0 = (static_cast<long long>(v) * a.H + row) * a.W;
  int cnt = 0;
  for (int x = threadIdx.x; x < a.W; x += 256) cnt += cloud_keep(a, z, r0 + x);
  const int t = block_count_256(cnt);
  if (threadIdx.x == 0) counts[(static_cast<long long>(z) * a.N + v) * a.H + row] = t;
}

// grid (H, N, 2), 256 threads: world points of row blockIdx.x of view blockIdx.y as fp64 [n][3]
__global__ void __launch_bounds__(256) cloud_scatter_kernel(CloudArgs a, const long long* offsets0, const long long* offsets1,
                                                            double* out0, double* out1) {
  const int row = blockIdx.x, v = blockIdx.y, z = blockIdx.z;
  const long long r0 = (static_cast<long long>(v) * a.H + row) * a.W;
  const float* P = (z == 0 ? a.gt_pose : a.pose) + v * 16;
  float Ki[9];
  inv3_f32(z == 0 ? a.gt_intri : a.intri + v * 9, Ki);
  const float s = (z == 1 && a.scale) ? a.scale[v] : 1.f;
  const float* D = z == 0 ? a.gt_depth : a.depth;
  double* out = z == 0 ? out0 : out1;
  const long long base = (z == 0 ? offsets0 : offsets1)[static_cast<long long>(v) * a.H + row];
  row_compact_256(a.W, base, [&](int x) { return cloud_keep(a, z, r0 + x); }, [&](int x, long long o) {
    float w[3];
    const float d = z == 1 && a.scale ? D[r0 + x] * s : D[r0 + x];
    unproject_f32(Ki, P, static_cast<float>(x), static_cast<float>(row), d, w);
    for (int c = 0; c < 3; ++c) out[3 * o + c] = w[c];
  });
}

bool dev_or_null(const void* p) { return p == nullptr || on_device(p); }

}  // namespace
}  // namespace sta

using namespace sta;

extern "C" {

size_t sta_sort_scratch_bytes(int64_t n) { return sort_scratch_bytes(n > 0 ? n : 0); }

int sta_op_radix_sort(const uint64_t* keys, const uint32_t* idx, int64_t n, int nbits, uint64_t* keys_out, uint32_t* idx_out,
                      void* scratch, void* stream) {
  STA_REQUIRE(n >= 0 && n < (1ll << 31), "0 <= n < 2^31");
  STA_REQUIRE(nbits >= 0 && nbits <= 64, "nbits in [0, 64]");
  if (n == 0) return 0;
  STA_REQUIRE(keys && keys_out && idx_out && scratch, "null argument");
  STA_REQUIRE(on_device(keys) && dev_or_null(idx) && on_device(keys_out) && on_device(idx_out) && on_device(scratch),
              "arguments must be device memory");
  STA_CHECK_CUDA(radix_sort(keys, idx, n, nbits, keys_out, idx_out, scratch, static_cast<cudaStream_t>(stream)));
  return 0;
}

size_t sta_eval_clouds_scratch_bytes(int N, int H) {
  const long long rows = static_cast<long long>(N > 0 ? N : 1) * H;
  return static_cast<size_t>(2 * rows * sizeof(int) + 2 * (rows + 1) * sizeof(long long) + 16);
}

int sta_eval_clouds(int N, int H, int W, const float* gt_depth, const float* gt_pose, const float* gt_intri, const float* depth,
                    const float* scale, const float* pose, const float* intri, const float* conf, float thres, double* gt_out,
                    double* est_out, int64_t* count_out, void* scratch, void* stream) {
  STA_REQUIRE(N >= 1 && N <= 65535 && H >= 1 && H <= 65535 && W >= 1, "1 <= N, H <= 65535 and W >= 1");
  STA_REQUIRE(static_cast<long long>(N) * H * W < (1ll << 40), "clouds too large");
  STA_REQUIRE(gt_depth && gt_pose && gt_intri && depth && pose && intri && conf && gt_out && est_out && count_out && scratch,
              "null argument");
  STA_REQUIRE(on_device(gt_depth) && on_device(gt_pose) && on_device(gt_intri) && on_device(depth) && dev_or_null(scale) &&
                  on_device(pose) && on_device(intri) && on_device(conf) && on_device(gt_out) && on_device(est_out) &&
                  on_device(count_out) && on_device(scratch),
              "arguments must be device memory");
  STA_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 7) == 0, "scratch must be 8-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CloudArgs a = {N, H, W, thres, gt_depth, gt_pose, gt_intri, depth, scale, pose, intri, conf};
  const long long rows = static_cast<long long>(N) * H;
  long long* off0 = static_cast<long long*>(scratch);
  long long* off1 = off0 + rows + 1;
  int* counts = reinterpret_cast<int*>(off1 + rows + 1);
  cloud_count_kernel<<<dim3(H, N, 2), 256, 0, st>>>(a, counts);
  STA_CHECK_CUDA(cudaGetLastError());
  row_scan_kernel<<<1, 1024, 0, st>>>(counts, rows, off0, count_out);
  row_scan_kernel<<<1, 1024, 0, st>>>(counts + rows, rows, off1, count_out + 1);
  STA_CHECK_CUDA(cudaGetLastError());
  cloud_scatter_kernel<<<dim3(H, N, 2), 256, 0, st>>>(a, off0, off1, gt_out, est_out);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

size_t sta_voxel_scratch_bytes(int64_t n) {
  n = n > 0 ? n : 0;
  return sort_scratch_bytes(n) + static_cast<size_t>(8 * n + 4 * n + 4 * n + 4 * (scan_blocks(n) + 2) + 8 * 6 * kBoxBlocks +
                                                     8 * 8 + 256);
}

int sta_voxel_down(const double* pts, int64_t n, double voxel, double* out, int64_t* count_host, void* scratch, void* stream) {
  STA_REQUIRE(count_host != nullptr, "null count");
  *count_host = 0;
  STA_REQUIRE(voxel > 0.0, "voxel_size <= 0");
  STA_REQUIRE(n >= 0 && n < (1ll << 31), "0 <= n < 2^31");
  if (n == 0) return 0;
  STA_REQUIRE(pts && out && scratch, "null argument");
  STA_REQUIRE(on_device(pts) && on_device(out) && on_device(scratch), "arguments must be device memory");
  STA_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 15) == 0, "scratch must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  char* p = static_cast<char*>(scratch);
  void* sort_s = p;
  p += (sort_scratch_bytes(n) + 15) / 16 * 16;
  uint64_t* key = reinterpret_cast<uint64_t*>(p);
  p += 8 * n;
  uint32_t* idx = reinterpret_cast<uint32_t*>(p);
  p += (4 * n + 15) / 16 * 16;
  unsigned* head = reinterpret_cast<unsigned*>(p);
  p += (4 * n + 15) / 16 * 16;
  unsigned* bsum = reinterpret_cast<unsigned*>(p);
  p += (4 * (scan_blocks(n) + 2) + 15) / 16 * 16;
  double* part = reinterpret_cast<double*>(p);
  p += 8 * 6 * kBoxBlocks;
  double* bb = reinterpret_cast<double*>(p);
  // the box decides the key widths and open3d's refusal: one read-back
  STA_CHECK_CUDA(bbox(pts, n, part, bb, st));
  double hb[6];
  STA_CHECK_CUDA(cudaMemcpyAsync(hb, bb, sizeof(hb), cudaMemcpyDeviceToHost, st));
  STA_CHECK_CUDA(cudaStreamSynchronize(st));
  VoxelGrid g;
  g.v = voxel;
  double extent = 0.0;
  long long kmax[3];
  for (int c = 0; c < 3; ++c) {
    g.mn[c] = hb[c] - voxel * 0.5;
    extent = fmax(extent, (hb[3 + c] + voxel * 0.5) - g.mn[c]);
  }
  STA_REQUIRE(!(voxel * static_cast<double>(INT_MAX) < extent), "voxel_size is too small");
  STA_REQUIRE(std::isfinite(extent), "points must be finite");
  int bits[3];
  for (int c = 0; c < 3; ++c) {
    kmax[c] = static_cast<long long>(floor((hb[3 + c] - g.mn[c]) / voxel));
    bits[c] = bit_width(kmax[c]);
  }
  if (bits[0] + bits[1] + bits[2] <= 64) {
    g.shift[0] = bits[1] + bits[2];
    g.shift[1] = bits[2];
    g.shift[2] = 0;
    voxel_key_kernel<<<grid_for(n), 256, 0, st>>>(pts, nullptr, n, g, key);
    STA_CHECK_CUDA(cudaGetLastError());
    STA_CHECK_CUDA(radix_sort(key, nullptr, n, bits[0] + bits[1] + bits[2], key, idx, sort_s, st));
  } else {  // (ky, kz) first, then kx: LSD over the axes
    VoxelGrid lo = g, hi = g;
    lo.shift[0] = -1;
    lo.shift[1] = bits[2];
    lo.shift[2] = 0;
    hi.shift[0] = 0;
    hi.shift[1] = hi.shift[2] = -1;
    voxel_key_kernel<<<grid_for(n), 256, 0, st>>>(pts, nullptr, n, lo, key);
    STA_CHECK_CUDA(cudaGetLastError());
    STA_CHECK_CUDA(radix_sort(key, nullptr, n, bits[1] + bits[2], key, idx, sort_s, st));
    voxel_key_kernel<<<grid_for(n), 256, 0, st>>>(pts, idx, n, hi, key);
    STA_CHECK_CUDA(cudaGetLastError());
    STA_CHECK_CUDA(radix_sort(key, idx, n, bits[0], key, idx, sort_s, st));
  }
  voxel_head_kernel<<<grid_for(n), 256, 0, st>>>(pts, idx, n, g, head);
  STA_CHECK_CUDA(cudaGetLastError());
  STA_CHECK_CUDA(scan_u32(head, n, bsum, st));
  unsigned nv = 0;
  STA_CHECK_CUDA(cudaMemcpyAsync(&nv, bsum + scan_blocks(n), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
  STA_CHECK_CUDA(cudaStreamSynchronize(st));
  unsigned* start = reinterpret_cast<unsigned*>(key);  // [nv + 1] <= [n + 1]: the keys are no longer needed
  voxel_start_kernel<<<grid_for(n), 256, 0, st>>>(head, n, bsum + scan_blocks(n), start);
  voxel_sum_kernel<<<grid_for(nv), 256, 0, st>>>(pts, idx, start, nv, out);
  STA_CHECK_CUDA(cudaGetLastError());
  *count_host = nv;
  return 0;
}

int sta_nn_create(const double* pts, int64_t n, StaNnIndex** out, void* stream) {
  STA_REQUIRE(out != nullptr, "null output pointer");
  *out = nullptr;
  STA_REQUIRE(n >= 0 && n < (1ll << 31), "0 <= n < 2^31");
  STA_REQUIRE(n == 0 || (pts && on_device(pts)), "points must be device memory");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  StaNnIndex* ix = new StaNnIndex();
  ix->n = n;
  ix->leaves = static_cast<int>((n + kLeaf - 1) / kLeaf);
  ix->P = 1;
  while (ix->P < ix->leaves) ix->P <<= 1;
  cudaError_t e = cudaSuccess;
  auto take = [&](auto** p, size_t bytes) {
    if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(p), bytes > 0 ? bytes : 8);
  };
  take(&ix->x, 8 * n);
  take(&ix->y, 8 * n);
  take(&ix->z, 8 * n);
  take(&ix->id, 4 * n);
  take(&ix->box, 8 * 6 * 2 * static_cast<size_t>(ix->P));
  take(&ix->bb, 8 * 6);
  void* tmp = nullptr;
  const size_t tmp_bytes = sort_scratch_bytes(n) + 8 * n + 8 * 6 * kBoxBlocks + 64;
  if (n > 0) take(&tmp, tmp_bytes);
  if (e == cudaSuccess && n > 0) {
    char* p = static_cast<char*>(tmp);
    void* sort_s = p;
    p += (sort_scratch_bytes(n) + 15) / 16 * 16;
    uint64_t* code = reinterpret_cast<uint64_t*>(p);
    p += 8 * n;
    double* part = reinterpret_cast<double*>(p);
    e = bbox(pts, n, part, ix->bb, st);
    if (e == cudaSuccess) {
      morton_kernel<<<grid_for(n), 256, 0, st>>>(pts, n, ix->bb, 0, code);
      e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = radix_sort(code, nullptr, n, 63, code, ix->id, sort_s, st);
    if (e == cudaSuccess) {
      nn_gather_kernel<<<grid_for(n), 256, 0, st>>>(pts, ix->id, n, ix->x, ix->y, ix->z);
      nn_leaf_kernel<<<grid_for(ix->P), 256, 0, st>>>(*ix);
      for (long long lvl = ix->P / 2; lvl >= 1; lvl /= 2) nn_level_kernel<<<grid_for(lvl), 256, 0, st>>>(ix->box, lvl);
      e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);  // before the sort's scratch goes
  }
  if (tmp) cudaFree(tmp);
  if (e != cudaSuccess) {
    set_last_error(std::string("sta_nn_create: ") + cudaGetErrorString(e));
    sta_nn_destroy(ix);
    return 1;
  }
  *out = ix;
  return 0;
}

void sta_nn_destroy(StaNnIndex* ix) {
  if (!ix) return;
  cudaDeviceSynchronize();
  void* bufs[] = {ix->x, ix->y, ix->z, ix->id, ix->box, ix->bb};
  for (void* p : bufs)
    if (p) cudaFree(p);
  delete ix;
}

size_t sta_nn_query_scratch_bytes(int64_t nq) {
  nq = nq > 0 ? nq : 0;
  return sort_scratch_bytes(nq) + static_cast<size_t>(8 * nq + 4 * nq + 64);
}

int sta_nn_query(const StaNnIndex* ix, const double* q, int64_t nq, double radius, double* dist_out, int64_t* idx_out,
                 void* scratch, void* stream) {
  STA_REQUIRE(ix != nullptr, "null index");
  STA_REQUIRE(nq >= 0 && nq < (1ll << 31), "0 <= nq < 2^31");
  STA_REQUIRE(radius >= 0.0, "radius must be >= 0");
  if (nq == 0) return 0;
  STA_REQUIRE(q && dist_out && idx_out && scratch, "null argument");
  STA_REQUIRE(on_device(q) && on_device(dist_out) && on_device(idx_out) && on_device(scratch), "arguments must be device memory");
  STA_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 15) == 0, "scratch must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  char* p = static_cast<char*>(scratch);
  void* sort_s = p;
  p += (sort_scratch_bytes(nq) + 15) / 16 * 16;
  uint64_t* code = reinterpret_cast<uint64_t*>(p);
  p += 8 * nq;
  uint32_t* order = reinterpret_cast<uint32_t*>(p);
  if (ix->n > 0) {
    // 30 bits of the queries' Morton codes in the index's box are enough for coherent warps
    morton_kernel<<<grid_for(nq), 256, 0, st>>>(q, nq, ix->bb, 33, code);
    STA_CHECK_CUDA(cudaGetLastError());
    STA_CHECK_CUDA(radix_sort(code, nullptr, nq, 30, code, order, sort_s, st));
  } else {
    iota_kernel<<<grid_for(nq), 256, 0, st>>>(order, nq);
  }
  nn_query_kernel<<<static_cast<unsigned>((nq + 127) / 128), 128, 0, st>>>(*ix, q, order, nq, radius, dist_out, idx_out);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

size_t sta_reduce_scratch_bytes(void) { return sizeof(double) * (kRedBlocks * kRedVals + 16); }

int sta_op_moments(const double* src, const double* dst, const int64_t* corr, int64_t n, double* out17, void* scratch,
                   void* stream) {
  STA_REQUIRE(n >= 0, "n >= 0");
  STA_REQUIRE(src && dst && corr && out17 && scratch, "null argument");
  STA_REQUIRE(on_device(src) && on_device(dst) && on_device(corr) && on_device(out17) && on_device(scratch),
              "arguments must be device memory");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  double* partial = static_cast<double*>(scratch);
  STA_CHECK_CUDA(reduce(n, MomentsA{src, dst, corr}, partial, out17, st));
  STA_CHECK_CUDA(reduce(n, MomentsB{src, dst, corr, out17}, partial, out17 + 8, st));
  return 0;
}

size_t sta_icp_scratch_bytes(int64_t n) {
  n = n > 0 ? n : 0;
  return sta_nn_query_scratch_bytes(n) + static_cast<size_t>(16 * n) + sta_reduce_scratch_bytes() + 64;
}

int sta_icp_moments(const StaNnIndex* target, const double* target_pts, const double* src, int64_t n, double radius,
                    double* out17, void* scratch, void* stream) {
  STA_REQUIRE(target != nullptr && out17 && scratch, "null argument");
  STA_REQUIRE(target->n == 0 || (target_pts && on_device(target_pts)), "target points must be device memory");
  STA_REQUIRE(n >= 0 && (n == 0 || (src && on_device(src))), "source points must be device memory");
  STA_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 15) == 0, "scratch must be 16-byte aligned");
  char* p = static_cast<char*>(scratch);
  void* q_s = p;
  p += (sta_nn_query_scratch_bytes(n) + 15) / 16 * 16;
  double* dist = reinterpret_cast<double*>(p);
  p += 8 * n;
  int64_t* corr = reinterpret_cast<int64_t*>(p);
  p += 8 * n;
  if (n > 0) {
    const int rc = sta_nn_query(target, src, n, radius, dist, corr, q_s, stream);
    if (rc) return rc;
  }
  return sta_op_moments(n ? src : out17, target->n ? target_pts : out17, corr, n, out17, p, stream);
}

int sta_transform_points(double* pts, int64_t n, const double* m12_host, void* stream) {
  STA_REQUIRE(m12_host != nullptr, "null matrix");
  STA_REQUIRE(n >= 0, "n >= 0");
  if (n == 0) return 0;
  STA_REQUIRE(pts && on_device(pts), "points must be device memory");
  Affine a;
  for (int i = 0; i < 12; ++i) a.m[i] = m12_host[i];
  transform_kernel<<<grid_for(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(pts, n, a);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int sta_sum_sq_clipped(const double* d, int64_t n, double clip, double* out_dev, void* scratch, void* stream) {
  STA_REQUIRE(n >= 0 && out_dev && scratch, "null argument");
  STA_REQUIRE((n == 0 || (d && on_device(d))) && on_device(out_dev) && on_device(scratch), "arguments must be device memory");
  STA_CHECK_CUDA(reduce(n, SumSqClipped{n ? d : out_dev, clip}, static_cast<double*>(scratch), out_dev,
                        static_cast<cudaStream_t>(stream)));
  return 0;
}

}  // extern "C"
