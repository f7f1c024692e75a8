// DBoW3 bag-of-words loop detection on the device: what vista_slam/loop_detector.py::LoopDetector does on the host with
// DBoW3Py (Vocabulary::load / transform / score, L1 scoring) around cv2 ORB.
//
// The vocabulary is parsed on the host (text format of Vocabulary::load_fromtxt, or the binary stream of
// Vocabulary::fromStream, plain or QuickLZ-compressed) and uploaded once: node descriptors as 8 x u32, the children of
// each node as a range of a child table in file order, weights (fp64) and word ids.  A detector owns the ORB scratch of
// one frame size and a device-resident database (CSR) of every view's normalised bag-of-words vector.
//
// Bit-exact with the numpy restatement under oracle/ (tests/test_loop_gpu.py): the descent takes the first child of minimal
// Hamming distance; a word's value is its weight added once per descriptor in fp64 (addWeight; all addends of a word
// are equal, so the order of descriptors does not matter) or set once (addIfNotExist); the L1 norm, the division and the
// score s += |v - w| - |v| - |w| are sequential fp64 in ascending word id; detect_loop runs in one thread per row.
//
// One path serves F >= 1 frames of one size, of one detector or of several that share one vocabulary, frame f belonging
// to dets[f] (sta_loop_add_frames_group / sta_loop_detect_group; one detector's frame is a group of one): ORB with a
// frame grid dimension and one transform over F x 4096 descriptor slots in dets[0]'s workspace, one CTA per frame
// building its vector into a staging slot, then the append, score and detect launches, each reading per row a GroupRow
// (mapped pinned memory) that names the row's database, view and loop parameters, and one host synchronisation: the
// read-back of the candidate lists.  Every per-frame result is independent of F and of the other detectors.
#include "../../include/sta_b200.h"
#include "common.cuh"
#include "host_util.h"
#include "loop.h"

#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <fstream>
#include <sstream>
#include <string>
#include <vector>

namespace sta {
namespace {

constexpr uint64_t kMagic = 88877711233ull;
constexpr int kBuildThreads = 1024;
enum { kTfIdf = 0, kTf = 1, kIdf = 2, kBinary = 3 };

struct HostVocab {
  int k = 0, L = 0, scoring = 0, weighting = 0;
  std::vector<uint32_t> desc;    // [n][8]
  std::vector<int> parent;       // -1 for the root
  std::vector<double> weight;
  std::vector<int> word;         // -1: not a word
  int n_words = 0;
};

bool fail(std::string* err, const std::string& msg) {
  *err = msg;
  return false;
}

bool validate_header(const HostVocab& v, std::string* err) {
  if (v.scoring != 0) {
    static const char* names[] = {"L1_NORM", "L2_NORM", "CHI_SQUARE", "KL", "BHATTACHARYYA", "DOT_PRODUCT"};
    return fail(err, std::string("only L1 scoring is supported; the vocabulary uses ") +
                         (v.scoring >= 0 && v.scoring < 6 ? names[v.scoring] : "an unknown scoring"));
  }
  if (v.weighting < 0 || v.weighting > 3) return fail(err, "unknown weighting type");
  return true;
}

// Vocabulary::load_fromtxt
bool load_text(const std::string& path, HostVocab* v, std::string* err) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return fail(err, "cannot open " + path);
  std::string data;
  {
    char buf[1 << 16];
    size_t n;
    while ((n = fread(buf, 1, sizeof(buf), f)) > 0) data.append(buf, n);
    fclose(f);
  }
  const char* p = data.c_str();
  const char* end = p + data.size();
  const char* eol = static_cast<const char*>(memchr(p, '\n', end - p));
  if (!eol) eol = end;
  int n1, n2;
  if (sscanf(std::string(p, eol).c_str(), "%d %d %d %d", &v->k, &v->L, &n1, &n2) != 4 || v->k < 0 || v->k > 20 ||
      v->L < 1 || v->L > 10 || n1 < 0 || n1 > 5 || n2 < 0 || n2 > 3)
    return fail(err, "not a DBoW3 text vocabulary: " + path);
  v->scoring = n1;
  v->weighting = n2;
  if (!validate_header(*v, err)) return false;
  v->desc.assign(8, 0u);
  v->parent.assign(1, -1);
  v->weight.assign(1, 0.0);
  v->word.assign(1, -1);
  p = eol < end ? eol + 1 : end;
  float vals[64];
  while (p < end) {
    eol = static_cast<const char*>(memchr(p, '\n', end - p));
    if (!eol) eol = end;
    if (eol == p) break;  // an empty line ends the node list
    const std::string line(p, eol);
    p = eol < end ? eol + 1 : end;
    const char* s = line.c_str();
    char* q;
    const long pid = strtol(s, &q, 10);
    if (q == s) break;
    s = q;
    const long leaf = strtol(s, &q, 10);
    if (q == s) return fail(err, "malformed node line in " + path);
    s = q;
    int nv = 0;
    for (;;) {
      const float d = strtof(s, &q);
      if (q == s) break;
      if (nv == 64) return fail(err, "only binary (32-byte) descriptors are supported: a node has too many values");
      vals[nv++] = d;
      s = q;
    }
    if (nv != 33) return fail(err, "only binary 32-byte descriptors are supported (a node line has " + std::to_string(nv - 1) +
                                       " descriptor values)");
    const int nid = static_cast<int>(v->parent.size());
    if (pid < 0 || pid >= nid) return fail(err, "node " + std::to_string(nid) + " names a parent that does not precede it");
    v->parent.push_back(static_cast<int>(pid));
    v->weight.push_back(static_cast<double>(vals[32]));
    uint8_t bytes[32];
    for (int i = 0; i < 32; ++i) bytes[i] = static_cast<uint8_t>(vals[i]);
    uint32_t w8[8];
    memcpy(w8, bytes, 32);
    v->desc.insert(v->desc.end(), w8, w8 + 8);
    v->word.push_back(leaf > 0 ? v->n_words++ : -1);
  }
  return true;
}

template <typename T>
bool rd(const std::string& b, size_t& pos, T* out) {
  if (pos + sizeof(T) > b.size()) return false;
  memcpy(out, b.data() + pos, sizeof(T));
  pos += sizeof(T);
  return true;
}

// One QuickLZ 1.5 chunk as DBoW3's toStream writes them (compression level 1, streaming buffer 0), written from the
// format: a header (flag byte: bit 0 compressed, bit 1 sizes as u32 rather than u8; then compressed and decompressed
// sizes), then 32-bit control words whose bits, least significant first, select a match (1) or a literal byte (0); a
// control word is spent when only its sentinel bit is left.  A match token names a 12-bit hash of the 3 bytes it
// repeats and a length (low nibble + 2, or the next byte when the nibble is 0); the decoder keeps the table of the last
// output position of each hash, updated for every position up to the start of a match and up to 3 bytes behind the
// last literal (positions inside a match are not hashed).  The last UNCONDITIONAL_MATCHLEN + UNCOMPRESSED_END = 10
// bytes are literals whatever the control bits say.  *used receives the chunk's compressed size.
bool qlz1_chunk(const uint8_t* in, size_t avail, std::string* out, size_t* used, std::string* err) {
  if (avail < 3) return fail(err, "truncated QuickLZ chunk");
  const bool wide = (in[0] & 2) != 0;
  const size_t hdr = wide ? 9 : 3;
  if (avail < hdr) return fail(err, "truncated QuickLZ chunk");
  uint32_t csize = 0, dsize = 0;
  if (wide) {
    memcpy(&csize, in + 1, 4);
    memcpy(&dsize, in + 5, 4);
  } else {
    csize = in[1];
    dsize = in[2];
  }
  if (csize < hdr || csize > avail) return fail(err, "truncated QuickLZ chunk");
  *used = csize;
  if (!(in[0] & 1)) {
    if (csize - hdr < dsize) return fail(err, "corrupt QuickLZ chunk");
    out->append(reinterpret_cast<const char*>(in + hdr), dsize);
    return true;
  }
  std::vector<uint8_t> dst(dsize);
  std::vector<uint32_t> table(4096, 0);
  auto hash_at = [&](size_t p) {
    const uint32_t v = dst[p] | (dst[p + 1] << 8) | (static_cast<uint32_t>(dst[p + 2]) << 16);
    return ((v >> 12) ^ v) & 0xfffu;
  };
  const uint8_t* src = in + hdr;
  const uint8_t* end = in + csize;
  size_t d = 0;
  long long last_hashed = -1;
  const long long last_matchstart = static_cast<long long>(dsize) - 1 - 6 - 4;
  auto hash_upto = [&](long long upto) {
    while (last_hashed < upto) {
      ++last_hashed;
      table[hash_at(static_cast<size_t>(last_hashed))] = static_cast<uint32_t>(last_hashed);
    }
  };
  uint32_t cword = 1;
  while (d < dsize) {
    if (cword == 1) {
      if (end - src < 4) return fail(err, "corrupt QuickLZ chunk");
      memcpy(&cword, src, 4);
      src += 4;
    }
    if (cword & 1) {
      cword >>= 1;
      if (end - src < 3) return fail(err, "corrupt QuickLZ chunk");
      const uint32_t fetch = src[0] | (src[1] << 8) | (static_cast<uint32_t>(src[2]) << 16);
      const uint32_t from = table[(fetch >> 4) & 0xfff];
      uint32_t len;
      if (fetch & 0xf) {
        len = (fetch & 0xf) + 2;
        src += 2;
      } else {
        len = src[2];
        src += 3;
      }
      if (from >= d || len > dsize - d) return fail(err, "corrupt QuickLZ chunk");
      for (uint32_t k = 0; k < len; ++k) dst[d + k] = dst[from + k];
      hash_upto(static_cast<long long>(d));
      d += len;
      last_hashed = static_cast<long long>(d) - 1;
    } else if (static_cast<long long>(d) < last_matchstart) {
      if (src >= end) return fail(err, "corrupt QuickLZ chunk");
      dst[d++] = *src++;
      cword >>= 1;
      hash_upto(static_cast<long long>(d) - 3);
    } else {
      while (d < dsize) {
        if (cword == 1) {
          src += 4;
          cword = 1u << 31;
        }
        if (src >= end) return fail(err, "corrupt QuickLZ chunk");
        dst[d++] = *src++;
        cword >>= 1;
      }
    }
  }
  out->append(reinterpret_cast<const char*>(dst.data()), dsize);
  return true;
}

// Vocabulary::fromStream: a plain stream, or chunks of 10 000 bytes compressed with QuickLZ level 1
bool load_binary(const std::string& file, HostVocab* v, std::string* err, std::vector<int>* order) {
  size_t pos = 8;
  uint32_t nnodes = 0;
  uint8_t cflag;
  if (!rd(file, pos, &cflag) || !rd(file, pos, &nnodes)) return fail(err, "truncated DBoW3 binary vocabulary");
  if (nnodes == 0) return fail(err, "empty vocabulary");
  std::string inflated;
  if (cflag) {
    uint32_t nchunks;
    if (!rd(file, pos, &nchunks)) return fail(err, "truncated DBoW3 binary vocabulary");
    for (uint32_t c = 0; c < nchunks; ++c) {
      size_t used = 0;
      if (pos >= file.size() ||
          !qlz1_chunk(reinterpret_cast<const uint8_t*>(file.data()) + pos, file.size() - pos, &inflated, &used, err))
        return fail(err, "DBoW3 vocabulary: " + (err->empty() ? std::string("truncated chunk") : *err));
      pos += used;
    }
    pos = 0;
  }
  const std::string& data = cflag ? inflated : file;
  if (!rd(data, pos, &v->k) || !rd(data, pos, &v->L) || !rd(data, pos, &v->scoring) || !rd(data, pos, &v->weighting))
    return fail(err, "truncated DBoW3 binary vocabulary");
  if (!validate_header(*v, err)) return false;
  v->desc.assign(static_cast<size_t>(nnodes) * 8, 0u);
  v->parent.assign(nnodes, -1);
  v->weight.assign(nnodes, 0.0);
  v->word.assign(nnodes, -1);
  for (uint32_t i = 1; i < nnodes; ++i) {
    uint32_t nid, pid;
    double w;
    int cols, rows, type;
    if (!rd(data, pos, &nid) || !rd(data, pos, &pid) || !rd(data, pos, &w) || !rd(data, pos, &cols) ||
        !rd(data, pos, &rows) || !rd(data, pos, &type))
      return fail(err, "truncated DBoW3 binary vocabulary");
    if (type != 0 || rows != 1 || cols != 32)
      return fail(err, "only binary 32-byte (CV_8U) descriptors are supported");
    if (nid == 0 || nid >= nnodes || pid >= nnodes) return fail(err, "node id out of range in the vocabulary");
    if (pos + 32 > data.size()) return fail(err, "truncated DBoW3 binary vocabulary");
    memcpy(&v->desc[static_cast<size_t>(nid) * 8], data.data() + pos, 32);
    pos += 32;
    v->parent[nid] = static_cast<int>(pid);
    v->weight[nid] = w;
    order->push_back(static_cast<int>(nid));
  }
  uint32_t nw;
  if (!rd(data, pos, &nw)) return fail(err, "truncated DBoW3 binary vocabulary");
  for (uint32_t i = 0; i < nw; ++i) {
    uint32_t wid, nid;
    if (!rd(data, pos, &wid) || !rd(data, pos, &nid)) return fail(err, "truncated DBoW3 binary vocabulary");
    if (nid >= nnodes) return fail(err, "word names a node out of range");
    v->word[nid] = static_cast<int>(wid);
  }
  v->n_words = static_cast<int>(nw);
  return true;
}

}  // namespace
}  // namespace sta

struct StaVocab {
  int k, L, scoring, weighting, n_nodes, n_words, device;
  uint32_t* desc;     // [n][8]
  int* child_start;   // [n + 1] into child
  int* child;         // [n - 1], file order
  double* weight;
  int* word;
};

namespace sta {
namespace {

int upload_vocab(const HostVocab& v, const std::vector<int>& order, StaVocab** out) {
  const int n = static_cast<int>(v.parent.size());
  std::vector<int> count(n + 1, 0), start(n + 1, 0), child(n > 1 ? n - 1 : 1, 0);
  for (int nid : order) count[v.parent[nid]]++;
  for (int i = 0; i < n; ++i) start[i + 1] = start[i] + count[i];
  std::vector<int> fill(start.begin(), start.end() - 1);
  for (int nid : order) child[fill[v.parent[nid]]++] = nid;
  StaVocab* h = new StaVocab();
  h->k = v.k;
  h->L = v.L;
  h->scoring = v.scoring;
  h->weighting = v.weighting;
  h->n_nodes = n;
  h->n_words = v.n_words;
  cudaGetDevice(&h->device);
  h->desc = nullptr;
  h->child_start = h->child = h->word = nullptr;
  h->weight = nullptr;
  cudaError_t e = cudaMalloc(&h->desc, sizeof(uint32_t) * 8 * n);
  if (e == cudaSuccess) e = cudaMalloc(&h->child_start, sizeof(int) * (n + 1));
  if (e == cudaSuccess) e = cudaMalloc(&h->child, sizeof(int) * child.size());
  if (e == cudaSuccess) e = cudaMalloc(&h->weight, sizeof(double) * n);
  if (e == cudaSuccess) e = cudaMalloc(&h->word, sizeof(int) * n);
  if (e == cudaSuccess) e = cudaMemcpy(h->desc, v.desc.data(), sizeof(uint32_t) * 8 * n, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(h->child_start, start.data(), sizeof(int) * (n + 1), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(h->child, child.data(), sizeof(int) * child.size(), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(h->weight, v.weight.data(), sizeof(double) * n, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(h->word, v.word.data(), sizeof(int) * n, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(h->desc);
    cudaFree(h->child_start);
    cudaFree(h->child);
    cudaFree(h->weight);
    cudaFree(h->word);
    delete h;
    set_last_error(std::string("vocabulary upload failed: ") + cudaGetErrorString(e));
    return 1;
  }
  *out = h;
  return 0;
}

// Row f of a group: the database of frame f's detector, the view the frame becomes there, the batch index of that
// detector's first frame, and its detect_loop parameters.
struct GroupRow {
  int* db_word;
  double* db_val;
  long long* db_start;
  int* db_len;
  int view, first, dist_min, nms, thresh_neighbor;
};

// Vocabulary::transform(feature, word_id, weight): one thread per descriptor
// blockIdx.y = frame of a batch: its descriptors and outputs are kOrbMaxKeypoints slots after the previous frame's,
// its count n_dev[f].
__global__ void transform_kernel(const uint8_t* desc, const int* n_dev, int n_host, StaVocab v, int* word_out,
                                 double* weight_out) {
  const long long f = blockIdx.y, m = f * kOrbMaxKeypoints;
  desc += 32 * m;
  word_out += m;
  weight_out += m;
  if (n_dev) n_dev += f;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = n_dev ? *n_dev : n_host;
  if (i >= n) return;
  uint32_t d[8];
  for (int k = 0; k < 8; ++k) d[k] = *reinterpret_cast<const uint32_t*>(desc + 32 * i + 4 * k);
  int node = 0;
  while (v.child_start[node + 1] > v.child_start[node]) {
    unsigned best = 0xffffffffu;
    int next = node;
    for (int c = v.child_start[node]; c < v.child_start[node + 1]; ++c) {
      const int id = v.child[c];
      const uint32_t* nd = v.desc + 8 * static_cast<long long>(id);
      unsigned dist = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) dist += __popc(d[k] ^ nd[k]);
      if (dist < best) {
        best = dist;
        next = id;
      }
    }
    node = next;
  }
  word_out[i] = v.word[node];
  weight_out[i] = v.weight[node];
}

// BowVector of n descriptors: accumulate (addWeight / addIfNotExist), then normalize(L1), into out_word / out_val
// (words ascending).  Run by a whole CTA; returns the length in thread 0.
__device__ int build_vector(const int* word, const double* weight, int n, int weighting, int* out_word, double* out_val) {
  __shared__ int s_first[kOrbMaxKeypoints];  // rank -> descriptor of the sorted (word, index) list
  __shared__ int s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  // rank sort of the descriptors with weight > 0 by (word, index)
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    if (!(weight[i] > 0.0)) continue;
    const int wi = word[i];
    int rank = 0;
    for (int j = 0; j < n; ++j) {
      if (!(weight[j] > 0.0)) continue;
      const int wj = word[j];
      rank += (wj < wi || (wj == wi && j < i)) ? 1 : 0;
    }
    s_first[rank] = i;
    atomicAdd(&s_cnt, 1);
  }
  __syncthreads();
  int len = 0;
  if (threadIdx.x == 0) {
    const int m = s_cnt;
    for (int r = 0; r < m;) {
      const int wv = word[s_first[r]];
      const double x = weight[s_first[r]];
      double acc = x;
      int e = r + 1;
      for (; e < m && word[s_first[e]] == wv; ++e)
        if (weighting == kTf || weighting == kTfIdf) acc = __dadd_rn(acc, x);
      out_word[len] = wv;
      out_val[len] = acc;
      ++len;
      r = e;
    }
    double norm = 0.0;
    for (int i = 0; i < len; ++i) norm = __dadd_rn(norm, fabs(out_val[i]));
    if (norm > 0.0)
      for (int i = 0; i < len; ++i) out_val[i] = __ddiv_rn(out_val[i], norm);
  }
  return len;
}

// One CTA per frame f: the vector of the descriptors at slot f (kOrbMaxKeypoints apart; count n_dev[f], or n_host
// without n_dev) into out_word / out_val at slot f, its length (-1: None) into out_len[f].
__global__ void __launch_bounds__(kBuildThreads) build_kernel(const int* word, const double* weight, const int* n_dev,
                                                              int n_host, int weighting, int* out_word, double* out_val,
                                                              int* out_len) {
  const long long f = blockIdx.x, m = f * kOrbMaxKeypoints;
  const int n = n_dev ? n_dev[f] : n_host;
  const int len = build_vector(word + m, weight + m, n, weighting, out_word + m, out_val + m);
  if (threadIdx.x == 0) out_len[f] = n > 0 ? len : -1;
}

// Database entries in use after view v: a None view (length -1) starts where the next one does.
__device__ long long db_end(const long long* db_start, const int* db_len, int v) {
  return db_start[v] + (db_len[v] > 0 ? db_len[v] : 0);
}

// Appends the F staged vectors, one CTA per frame: frame f goes to rows[f]'s database as view rows[f].view, after the
// frames of its detector that precede it in the batch.  The CTA reads its row once into shared memory.
__global__ void append_kernel(const int* stage_word, const double* stage_val, const int* stage_len, const GroupRow* rows) {
  const int f = blockIdx.x;
  __shared__ GroupRow r;
  if (threadIdx.x == 0) r = rows[f];
  __syncthreads();
  const int view0 = r.view - (f - r.first);  // the view of the detector's first frame in the batch
  long long base = view0 > 0 ? db_end(r.db_start, r.db_len, view0 - 1) : 0;
  for (int g = r.first; g < f; ++g) base += stage_len[g] > 0 ? stage_len[g] : 0;
  const int len = stage_len[f];
  for (int k = threadIdx.x; k < len; k += blockDim.x) {
    r.db_word[base + k] = stage_word[static_cast<long long>(f) * kOrbMaxKeypoints + k];
    r.db_val[base + k] = stage_val[static_cast<long long>(f) * kOrbMaxKeypoints + k];
  }
  if (threadIdx.x == 0) {
    r.db_start[r.view] = base;
    r.db_len[r.view] = len;
  }
}

// L1Scoring::score of vector a against vector b, a merge over ascending word ids; NaN when either is None (length -1).
__device__ double l1_score(const int* aw, const double* av, int na, const int* bw, const double* bv, int nb) {
  if (na < 0 || nb < 0) return __longlong_as_double(0x7ff8000000000000ll);
  double s = 0.0;
  int a = 0, b = 0;
  while (a < na && b < nb) {
    if (aw[a] == bw[b]) {
      const double vi = av[a], wi = bv[b];
      s = __dadd_rn(s, __dsub_rn(__dsub_rn(fabs(__dsub_rn(vi, wi)), fabs(vi)), fabs(wi)));
      ++a;
      ++b;
    } else if (aw[a] < bw[b]) {
      ++a;
    } else {
      ++b;
    }
  }
  return __ddiv_rn(-s, 2.0);
}

// One thread per view j.  Row y = blockIdx.y of a group detect: view rows[y].view of rows[y]'s database against its
// earlier views, into sims + y stride.  Without rows (sta_op_bow_score): the query (qw, qv, length *q_len) against views
// [0, nviews) of the database db_*, into sims.
__global__ void score_kernel(const int* qw, const double* qv, const int* q_len, const int* db_word, const double* db_val,
                             const long long* db_start, const int* db_len, int nviews, double* sims, long long stride,
                             const GroupRow* rows) {
  const int y = blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (!rows) {
    if (j < nviews) sims[j] = l1_score(qw, qv, *q_len, db_word + db_start[j], db_val + db_start[j], db_len[j]);
    return;
  }
  __shared__ GroupRow row;
  if (threadIdx.x == 0) row = rows[y];
  __syncthreads();
  const int i = row.view;
  if (j >= i) return;
  const long long* st = row.db_start;
  const int* ln = row.db_len;
  sims[y * stride + j] = l1_score(row.db_word + st[i], row.db_val + st[i], ln[i], row.db_word + st[j],
                                  row.db_val + st[j], ln[j]);
}

// loop_detector.py:23-50 over the precomputed similarities of view i; out: [0] = count, [1] = length of view i, then
// (j, sim) pairs as {int64 j, double sim}, sorted by descending similarity, ties keeping the scan's descending-j order.
__device__ void detect_row(const double* sims, const int* db_len, int i, int farthest, int dist_min, int nms,
                           int thresh_neighbor, long long* out) {
  const bool none_i = db_len[i] < 0;
  const int lo = i - thresh_neighbor > 0 ? i - thresh_neighbor : 0;
  double th = 1.0;
  bool any = false;
  for (int j = lo; j < i; ++j) {
    if (none_i || db_len[j] < 0) continue;
    th = any ? fmin(th, sims[j]) : sims[j];
    any = true;
  }
  long long n = 0;
  long long* c = out + 2;
  int last = farthest;
  for (int j = farthest - 1; j >= 0; --j) {
    if (last - j > nms && i - j > dist_min) {
      if (none_i || db_len[j] < 0) continue;
      const double s = sims[j];
      if (s > th) {
        // stable insertion by descending similarity
        long long k = n;
        while (k > 0 && __longlong_as_double(c[2 * (k - 1) + 1]) < s) {
          c[2 * k] = c[2 * (k - 1)];
          c[2 * k + 1] = c[2 * (k - 1) + 1];
          --k;
        }
        c[2 * k] = j;
        c[2 * k + 1] = __double_as_longlong(s);
        ++n;
        last = j;
      }
    }
  }
  out[0] = n;
  out[1] = db_len[i];
}

// One thread per row f: view rows[f].view of rows[f]'s database with that row's parameters.  Out row f = {ORB overflow
// flag of frame f, then detect_row's count, length and pairs}, `out_stride` entries apart; after the gridDim.x rows,
// entry gridDim.x out_stride + f holds the entries in use of row f's database.
__global__ void detect_kernel(const double* sims, long long sims_stride, const int* farthest, long long* out,
                              long long out_stride, const unsigned* overflow, size_t overflow_stride,
                              const GroupRow* rows) {
  const int f = blockIdx.x;
  const GroupRow r = rows[f];
  out[gridDim.x * out_stride + f] = db_end(r.db_start, r.db_len, r.view);
  long long* row = out + f * out_stride;
  row[0] = *reinterpret_cast<const unsigned*>(reinterpret_cast<const char*>(overflow) + f * overflow_stride);
  detect_row(sims + f * sims_stride, r.db_len, r.view, farthest[f], r.dist_min, r.nms, r.thresh_neighbor, row + 1);
}

}  // namespace
}  // namespace sta

using namespace sta;

struct StaLoopDetector {
  StaVocab* vocab;
  int dist_min, nms, thresh_neighbor;
  int H = 0, W = 0;
  OrbLayout lay = {};
  void* scratch = nullptr;        // ORB scratch: frame_cap slices of lay.total bytes
  void* kp = nullptr;             // ORB outputs + transform outputs: frame_cap slices of kKpSlice bytes
  int frame_cap = 0, stage_cap = 0;
  int* stage_word = nullptr;      // [stage_cap][kOrbMaxKeypoints] vectors of a batch before the append
  double* stage_val = nullptr;
  int* stage_len = nullptr;       // [stage_cap]
  int* farthest_pinned = nullptr; // [stage_cap], read by the detect kernel in place (mapped host memory)
  double* sims = nullptr;         // [rows][views] of the last detect
  long long* result = nullptr;    // its rows and the database entries in use
  long long* pinned = nullptr;    // host copy of result
  long long out_cap = 0;          // entries of sims / result / pinned
  long long last_row = 0;         // offset in sims of the last row of this detector's last detect of its own rows
  int last_row_len = 0;           // its length (the view index of that row)
  int views = 0, view_cap = 0;
  // Upper bound on the database entries in use, kept on the host: each appended view may add up to kOrbMaxKeypoints
  // words, and the exact count is only read back at the synchronisation of a detect.
  long long entries_bound = 0, entry_cap = 0;
  cudaStream_t last_stream = nullptr;  // the stream of the last call, synchronised before destruction
  int* db_word = nullptr;
  double* db_val = nullptr;
  long long* db_start = nullptr;
  int* db_len = nullptr;
  // Calls of which this detector is dets[0]: the row table of the last add (mapped host memory, read by its append,
  // score and detect launches), that add's detectors per frame and each one's view count after it.
  GroupRow* rows_pinned = nullptr;
  int rows_cap = 0;
  std::vector<StaLoopDetector*> group_dets;
  std::vector<int> group_views;
  bool group_pending = false;   // the last add's append may still read rows_pinned (no detect since)
  bool group_detected = false;  // this detector's last detect had other detectors' rows: sta_loop_similarities is refused
};

namespace {

struct KpBufs {
  int2* xy;
  int* level;
  float2* pts;
  float* angle;
  float* resp;
  uint8_t* desc;
  int* count;
  int* word;
  double* weight;
};

// Field-major buffers of `frames` frames: frame f's entries of each field start at slot f kOrbMaxKeypoints, its count
// at count[f] (the output layout of orb_run).
KpBufs kp_bufs(void* base, int frames) {
  char* p = static_cast<char*>(base);
  KpBufs b;
  const size_t M = static_cast<size_t>(kOrbMaxKeypoints) * frames;
  b.xy = reinterpret_cast<int2*>(p);          p += sizeof(int2) * M;
  b.pts = reinterpret_cast<float2*>(p);       p += sizeof(float2) * M;
  b.weight = reinterpret_cast<double*>(p);    p += sizeof(double) * M;
  b.level = reinterpret_cast<int*>(p);        p += sizeof(int) * M;
  b.angle = reinterpret_cast<float*>(p);      p += sizeof(float) * M;
  b.resp = reinterpret_cast<float*>(p);       p += sizeof(float) * M;
  b.word = reinterpret_cast<int*>(p);         p += sizeof(int) * M;
  b.desc = reinterpret_cast<uint8_t*>(p);     p += 32 * M;
  b.count = reinterpret_cast<int*>(p);
  return b;
}
size_t kp_bytes(int frames) { return ((8 + 8 + 8 + 4 + 4 + 4 + 4 + 32) * kOrbMaxKeypoints + 16) * static_cast<size_t>(frames); }

template <typename T>
int grow(T** p, long long old_n, long long new_n, cudaStream_t st) {
  T* q = nullptr;
  STA_CHECK_CUDA(cudaMallocAsync(&q, sizeof(T) * new_n, st));
  if (*p && old_n) STA_CHECK_CUDA(cudaMemcpyAsync(q, *p, sizeof(T) * old_n, cudaMemcpyDeviceToDevice, st));
  if (*p) STA_CHECK_CUDA(cudaFreeAsync(*p, st));
  *p = q;
  return 0;
}

// room for F more views of up to kOrbMaxKeypoints words each
int reserve(StaLoopDetector* d, cudaStream_t st, int F) {
  if (d->views + F > d->view_cap) {
    int cap = d->view_cap ? 2 * d->view_cap : 256;
    while (cap < d->views + F) cap *= 2;
    if (grow(&d->db_start, d->view_cap, cap, st) || grow(&d->db_len, d->view_cap, cap, st)) return 1;
    d->view_cap = cap;
  }
  const long long need = d->entries_bound + static_cast<long long>(F) * kOrbMaxKeypoints;
  if (need > d->entry_cap) {
    long long cap = d->entry_cap ? 2 * d->entry_cap : 64LL * kOrbMaxKeypoints;
    while (cap < need) cap *= 2;
    if (grow(&d->db_word, d->entry_cap, cap, st) || grow(&d->db_val, d->entry_cap, cap, st)) return 1;
    d->entry_cap = cap;
  }
  return 0;
}

// F frames (with n_dev): kOrbMaxKeypoints descriptor slots per frame, counts n_dev[0..F)
int bow_of_descriptors(StaVocab* v, const uint8_t* desc, const int* n_dev, int n_host, int* word, double* weight,
                       cudaStream_t st, int F = 1) {
  const int cap = n_dev ? kOrbMaxKeypoints : n_host;
  if (cap > 0) transform_kernel<<<dim3((cap + 127) / 128, F), 128, 0, st>>>(desc, n_dev, n_host, *v, word, weight);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ORB scratch and keypoint buffers for F frames of H x W (the frame size may change between calls)
int prepare_frames(StaLoopDetector* d, int F, int H, int W, cudaStream_t st) {
  if (H != d->H || W != d->W || F > d->frame_cap) {
    const OrbLayout lay = orb_layout(H, W);
    const int cap = F > d->frame_cap ? F : d->frame_cap;
    if (d->scratch) STA_CHECK_CUDA(cudaFreeAsync(d->scratch, st));
    d->scratch = nullptr;
    STA_CHECK_CUDA(cudaMallocAsync(&d->scratch, lay.total * cap, st));
    if (cap > d->frame_cap) {
      if (d->kp) STA_CHECK_CUDA(cudaFreeAsync(d->kp, st));
      d->kp = nullptr;
      STA_CHECK_CUDA(cudaMallocAsync(&d->kp, kp_bytes(cap), st));
    }
    d->lay = lay;
    d->H = H;
    d->W = W;
    d->frame_cap = cap;
  }
  return 0;
}

int grow_batch(StaLoopDetector* d, int F, cudaStream_t st) {
  if (F <= d->stage_cap) return 0;
  const long long M = kOrbMaxKeypoints;
  if (grow(&d->stage_word, 0, M * F, st) || grow(&d->stage_val, 0, M * F, st) || grow(&d->stage_len, 0, F, st)) return 1;
  if (d->farthest_pinned) cudaFreeHost(d->farthest_pinned);
  d->farthest_pinned = nullptr;
  STA_CHECK_CUDA(cudaMallocHost(&d->farthest_pinned, sizeof(int) * F));
  d->stage_cap = F;
  return 0;
}

// sims / result / pinned of at least `need` entries
int grow_results(StaLoopDetector* d, long long need, cudaStream_t st) {
  if (need <= d->out_cap) return 0;
  long long cap = d->out_cap ? 2 * d->out_cap : 1LL << 14;
  while (cap < need) cap *= 2;
  if (grow(&d->sims, 0, cap, st) || grow(&d->result, 0, cap, st)) return 1;
  if (d->pinned) cudaFreeHost(d->pinned);
  d->pinned = nullptr;
  STA_CHECK_CUDA(cudaMallocHost(&d->pinned, sizeof(long long) * cap));
  d->out_cap = cap;
  return 0;
}

// The ORB overflow of a batch's frames as the error of its first such frame (after the read-back of a detect)
int report_overflow(const long long* pinned, int F, long long out_stride) {
  for (int f = 0; f < F; ++f) {
    if (pinned[f * out_stride]) {
      set_last_error((F == 1 ? std::string("the frame") : "frame " + std::to_string(f) + " of the batch") +
                     " has more ORB candidates or keypoints than the detector holds");
      return 1;
    }
  }
  return 0;
}

// One detect row's results from the pinned read-back into n_out / js_out / sims_out (host)
void copy_row(const long long* row, int f, int* n_out, int64_t* js_out, double* sims_out, int cap_per_view) {
  const int n = static_cast<int>(row[1]);
  n_out[2 * f] = n;
  n_out[2 * f + 1] = static_cast<int>(row[2]);
  for (int k = 0; k < n && k < cap_per_view; ++k) {
    js_out[static_cast<long long>(f) * cap_per_view + k] = row[3 + 2 * k];
    memcpy(&sims_out[static_cast<long long>(f) * cap_per_view + k], &row[4 + 2 * k], sizeof(double));
  }
}

}  // namespace

extern "C" {

int sta_vocab_load(const char* path, StaVocab** out) {
  STA_REQUIRE(path && out, "null argument");
  std::string p(path), err;
  HostVocab v;
  std::vector<int> order;
  uint64_t sig = 0;
  {
    std::ifstream f(p, std::ios::binary);
    STA_REQUIRE(f.good(), (std::string("cannot open vocabulary ") + p).c_str());
    f.read(reinterpret_cast<char*>(&sig), sizeof(sig));
  }
  bool ok;
  if (sig == kMagic) {
    std::ifstream f(p, std::ios::binary);
    const std::string data((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    ok = load_binary(data, &v, &err, &order);
  } else if (p.find(".txt") != std::string::npos) {
    ok = load_text(p, &v, &err);
    for (int i = 1; ok && i < static_cast<int>(v.parent.size()); ++i) order.push_back(i);
  } else {
    ok = fail(&err, "unsupported vocabulary format (expected a DBoW3 .txt or binary file): " + p);
  }
  if (!ok) {
    set_last_error("sta_vocab_load: " + err);
    return 2;
  }
  return upload_vocab(v, order, out);
}

int sta_vocab_info(const StaVocab* v, int64_t* out6) {
  STA_REQUIRE(v && out6, "null argument");
  out6[0] = v->k;
  out6[1] = v->L;
  out6[2] = v->scoring;
  out6[3] = v->weighting;
  out6[4] = v->n_nodes;
  out6[5] = v->n_words;
  return 0;
}

void sta_vocab_destroy(StaVocab* v) {
  if (!v) return;
  cudaFree(v->desc);
  cudaFree(v->child_start);
  cudaFree(v->child);
  cudaFree(v->weight);
  cudaFree(v->word);
  delete v;
}

int sta_op_bow_transform(const StaVocab* v, const uint8_t* desc_dev, int n, int32_t* word_out, double* weight_out,
                         void* stream) {
  STA_REQUIRE(v && n >= 0, "bad argument");
  return bow_of_descriptors(const_cast<StaVocab*>(v), desc_dev, nullptr, n, word_out, weight_out,
                            static_cast<cudaStream_t>(stream));
}

int sta_op_bow_vector(const StaVocab* v, const int32_t* word, const double* weight, int n, int32_t* words_out,
                      double* vals_out, int32_t* len_out, void* stream) {
  STA_REQUIRE(v && n >= 0 && n <= kOrbMaxKeypoints, "descriptor count must be in [0, 4096]");
  build_kernel<<<1, kBuildThreads, 0, static_cast<cudaStream_t>(stream)>>>(word, weight, nullptr, n, v->weighting,
                                                                           words_out, vals_out, len_out);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int sta_op_bow_score(const int32_t* qw, const double* qv, const int32_t* q_len_dev, const int32_t* db_word,
                     const double* db_val, const int64_t* db_start, const int32_t* db_len, int nviews, double* sims_out,
                     void* stream) {
  STA_REQUIRE(nviews >= 0, "bad view count");
  if (nviews)
    score_kernel<<<(nviews + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(
        qw, qv, q_len_dev, db_word, db_val, reinterpret_cast<const long long*>(db_start), db_len, nviews, sims_out, 0,
        nullptr);
  STA_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int sta_loop_create(StaVocab* v, int loop_dist_min, int loop_nms, int loop_cand_thresh_neighbor, StaLoopDetector** out) {
  STA_REQUIRE(v && out, "null argument");
  StaLoopDetector* d = new StaLoopDetector();
  d->vocab = v;
  d->dist_min = loop_dist_min;
  d->nms = loop_nms;
  d->thresh_neighbor = loop_cand_thresh_neighbor;
  *out = d;
  return 0;
}

void sta_loop_destroy(StaLoopDetector* d) {
  if (!d) return;
  if (d->last_stream) cudaStreamSynchronize(d->last_stream);
  cudaFree(d->scratch);
  cudaFree(d->kp);
  cudaFree(d->db_word);
  cudaFree(d->db_val);
  cudaFree(d->db_start);
  cudaFree(d->db_len);
  cudaFree(d->sims);
  cudaFree(d->result);
  cudaFree(d->stage_word);
  cudaFree(d->stage_val);
  cudaFree(d->stage_len);
  if (d->pinned) cudaFreeHost(d->pinned);
  if (d->farthest_pinned) cudaFreeHost(d->farthest_pinned);
  if (d->rows_pinned) cudaFreeHost(d->rows_pinned);
  delete d;
}

int sta_loop_views(const StaLoopDetector* d) { return d ? d->views : -1; }

// compute_bow_feat for F frames [F][H][W] of one size: frame f belongs to dets[f], each detector's frames are
// consecutive, and all share one vocabulary (refused before any launch otherwise).  ORB, transform and build run over
// all F frames in dets[0]'s workspace; one append launch writes each frame into its own detector's database, in frame
// order, through dets[0]'s row table.  Asynchronous, unless dets[0]'s previous add has had no detect yet: its append
// may still read the row table, so the stream is synchronised before the table is rewritten.
int sta_loop_add_frames_group(StaLoopDetector* const* dets, int F, const void* frames_dev, int frames_is_f32, int H,
                              int W, void* stream) {
  STA_REQUIRE(dets && frames_dev, "null argument");
  STA_REQUIRE(F >= 1, "the frame count must be at least 1");
  STA_REQUIRE(orb_size_ok(H, W), "ORB frame sides must be in [32, 4096]");
  for (int f = 0; f < F; ++f) {
    STA_REQUIRE(dets[f], "null detector");
    STA_REQUIRE(dets[f]->vocab == dets[0]->vocab, "all detectors of a group must share one vocabulary");
    if (f > 0 && dets[f] != dets[f - 1])
      for (int g = 0; g < f - 1; ++g) STA_REQUIRE(dets[g] != dets[f], "a detector's frames must be consecutive");
  }
  StaLoopDetector* d0 = dets[0];
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (d0->group_pending && d0->last_stream) STA_CHECK_CUDA(cudaStreamSynchronize(d0->last_stream));
  d0->group_pending = false;
  if (prepare_frames(d0, F, H, W, st) || grow_batch(d0, F, st)) return 1;
  if (F > d0->rows_cap) {
    if (d0->rows_pinned) cudaFreeHost(d0->rows_pinned);
    d0->rows_pinned = nullptr;
    d0->rows_cap = 0;
    STA_CHECK_CUDA(cudaMallocHost(&d0->rows_pinned, sizeof(GroupRow) * F));
    d0->rows_cap = F;
  }
  for (int f = 0, e; f < F; f = e) {
    for (e = f + 1; e < F && dets[e] == dets[f];) ++e;
    if (reserve(dets[f], st, e - f)) return 1;
  }
  // the row table after every reserve, which may move a database
  for (int f = 0, first = 0; f < F; ++f) {
    if (f > 0 && dets[f] != dets[f - 1]) first = f;
    StaLoopDetector* d = dets[f];
    d0->rows_pinned[f] = {d->db_word, d->db_val, d->db_start, d->db_len, d->views + f - first, first,
                          d->dist_min, d->nms, d->thresh_neighbor};
  }
  KpBufs b = kp_bufs(d0->kp, d0->frame_cap);
  OrbOut o = {b.xy, b.level, b.pts, b.angle, b.resp, b.desc, b.count};
  if (orb_run(d0->lay, d0->scratch, frames_dev, frames_is_f32, o, st, F)) return 1;
  if (bow_of_descriptors(d0->vocab, b.desc, b.count, 0, b.word, b.weight, st, F)) return 1;
  build_kernel<<<F, kBuildThreads, 0, st>>>(b.word, b.weight, b.count, 0, d0->vocab->weighting, d0->stage_word,
                                            d0->stage_val, d0->stage_len);
  append_kernel<<<F, 256, 0, st>>>(d0->stage_word, d0->stage_val, d0->stage_len, d0->rows_pinned);
  STA_CHECK_CUDA(cudaGetLastError());
  d0->group_pending = true;
  for (int f = 0; f < F; ++f) {
    StaLoopDetector* d = dets[f];
    d->views++;
    d->entries_bound += kOrbMaxKeypoints;
    d->last_stream = st;
  }
  d0->group_dets.assign(dets, dets + F);
  d0->group_views.resize(F);
  for (int f = 0; f < F; ++f) d0->group_views[f] = dets[f]->views;
  return 0;
}

// detect_loop for the rows of the last sta_loop_add_frames_group of dets[0], with the same dets and F and no view added
// to any of them since: one score launch and one detect launch over all rows, each against its own database with its
// own detector's parameters, then one read-back, which also brings every detector's entry count.  n_out [2F] =
// {candidates, length (-1: None)} per row; row f's first cap_per_view candidates go to js_out / sims_out + f
// cap_per_view (host).  Afterwards sta_loop_similarities returns the last row when every row was dets[0]'s, and is
// refused on the detectors until their own next detect otherwise.
int sta_loop_detect_group(StaLoopDetector* const* dets, int F, const int* farthest_host, int* n_out, int64_t* js_out,
                          double* sims_out, int cap_per_view, void* stream) {
  STA_REQUIRE(dets && dets[0] && farthest_host && n_out && (cap_per_view == 0 || (js_out && sims_out)), "null argument");
  STA_REQUIRE(cap_per_view >= 0, "bad capacity");
  StaLoopDetector* d0 = dets[0];
  STA_REQUIRE(F >= 1 && F == static_cast<int>(d0->group_dets.size()),
              "F must be the frame count of the last group add of dets[0]");
  int max_view = 0;
  for (int f = 0; f < F; ++f) {
    STA_REQUIRE(dets[f] == d0->group_dets[f] && dets[f]->views == d0->group_views[f],
                "the detectors must be those of the last group add of dets[0], with no view added since");
    const int i = d0->rows_pinned[f].view;
    STA_REQUIRE(farthest_host[f] >= 0 && farthest_host[f] <= i, "farthest_neighbor must be in [0, view index]");
    max_view = i > max_view ? i : max_view;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long sims_stride = max_view + 1, out_stride = 3 + 2LL * (max_view + 1);  // out_stride > sims_stride
  const long long need = F * out_stride + F;
  if (grow_results(d0, need, st)) return 1;
  memcpy(d0->farthest_pinned, farthest_host, sizeof(int) * F);  // every earlier detect has synchronised
  if (max_view > 0)
    score_kernel<<<dim3((max_view + 127) / 128, F), 128, 0, st>>>(nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                                                                   nullptr, 0, d0->sims, sims_stride, d0->rows_pinned);
  detect_kernel<<<F, 1, 0, st>>>(d0->sims, sims_stride, d0->farthest_pinned, d0->result, out_stride,
                                 reinterpret_cast<const unsigned*>(static_cast<char*>(d0->scratch) + d0->lay.counters +
                                                                   3 * sizeof(unsigned)),
                                 d0->lay.total, d0->rows_pinned);
  STA_CHECK_CUDA(cudaGetLastError());
  STA_CHECK_CUDA(cudaMemcpyAsync(d0->pinned, d0->result, sizeof(long long) * need, cudaMemcpyDeviceToHost, st));
  STA_CHECK_CUDA(cudaStreamSynchronize(st));
  d0->group_pending = false;
  const bool own = dets[F - 1] == d0;  // every row is d0's: a detector's frames are consecutive
  if (own) {
    d0->last_row = (F - 1) * sims_stride;
    d0->last_row_len = max_view;
  }
  for (int f = 0; f < F; ++f) {
    dets[f]->group_detected = !own;
    dets[f]->last_stream = st;
    if (f == F - 1 || dets[f + 1] != dets[f]) dets[f]->entries_bound = d0->pinned[F * out_stride + f];
  }
  if (report_overflow(d0->pinned, F, out_stride)) return 1;
  for (int f = 0; f < F; ++f) copy_row(d0->pinned + f * out_stride, f, n_out, js_out, sims_out, cap_per_view);
  return 0;
}

// Host copy of view `view`'s vector (synchronises): *len_out = -1 for None; up to cap entries are written.
int sta_loop_view(StaLoopDetector* d, int view, int32_t* words_out, double* vals_out, int cap, int* len_out, void* stream) {
  STA_REQUIRE(d && view >= 0 && view < d->views, "view out of range");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int len;
  long long start;
  STA_CHECK_CUDA(cudaMemcpyAsync(&len, d->db_len + view, sizeof(int), cudaMemcpyDeviceToHost, st));
  STA_CHECK_CUDA(cudaMemcpyAsync(&start, d->db_start + view, sizeof(long long), cudaMemcpyDeviceToHost, st));
  STA_CHECK_CUDA(cudaStreamSynchronize(st));
  *len_out = len;
  const int m = len < cap ? len : cap;
  if (m > 0) {
    STA_CHECK_CUDA(cudaMemcpyAsync(words_out, d->db_word + start, sizeof(int) * m, cudaMemcpyDeviceToHost, st));
    STA_CHECK_CUDA(cudaMemcpyAsync(vals_out, d->db_val + start, sizeof(double) * m, cudaMemcpyDeviceToHost, st));
    STA_CHECK_CUDA(cudaStreamSynchronize(st));
  }
  return 0;
}

// Host copy of the last row of the last detect (NaN where a vector is None); n = that row's view index.
int sta_loop_similarities(StaLoopDetector* d, double* sims_out, int n, void* stream) {
  STA_REQUIRE(d, "null argument");
  STA_REQUIRE(!d->group_detected,
              "the detector's last detect was a group detect over several detectors, whose rows it does not keep");
  STA_REQUIRE(n >= 0 && n <= d->last_row_len, "bad count: n must be at most the view index of the last detect");
  if (n == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  STA_CHECK_CUDA(cudaMemcpyAsync(sims_out, d->sims + d->last_row, sizeof(double) * n, cudaMemcpyDeviceToHost, st));
  STA_CHECK_CUDA(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"
