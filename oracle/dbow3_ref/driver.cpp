// C entry points over the unmodified DBoW3 sources (compiled by oracle/dbow3_ref/build.py into oracle/_ref/), used by
// tools/make_golden_loop.py and tools/loop_stream.py as the reference bag-of-words implementation.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "Vocabulary.h"

namespace {

struct Peek : DBoW3::Vocabulary {
  static const std::vector<Node>& nodes(const DBoW3::Vocabulary& v) { return static_cast<const Peek&>(v).m_nodes; }
  static const std::vector<Node*>& words(const DBoW3::Vocabulary& v) { return static_cast<const Peek&>(v).m_words; }
};

cv::Mat rows_of(const uint8_t* desc, int n) {
  cv::Mat m(n, 32, CV_8U);
  if (n) memcpy(m.ptr<uchar>(), desc, static_cast<size_t>(n) * 32);
  return m;
}

void set_err(char* err, int len, const char* msg) {
  if (err && len > 0) {
    strncpy(err, msg, len - 1);
    err[len - 1] = 0;
  }
}

}  // namespace

extern "C" {

// Vocabulary(k, L, weighting, scoring).create(features): counts[i] descriptors of image i, rows of 32 bytes.
void* dbow_create(const uint8_t* desc, const int* counts, int nimg, int k, int L, int weighting, int scoring,
                  unsigned seed) {
  srand(seed);
  std::vector<std::vector<cv::Mat>> feats(nimg);
  const uint8_t* p = desc;
  for (int i = 0; i < nimg; ++i) {
    for (int r = 0; r < counts[i]; ++r, p += 32) feats[i].push_back(rows_of(p, 1));
  }
  auto* v = new DBoW3::Vocabulary(k, L, static_cast<DBoW3::WeightingType>(weighting),
                                  static_cast<DBoW3::ScoringType>(scoring));
  v->create(feats);
  return v;
}

void* dbow_load(const char* path, char* err, int errlen) {
  auto* v = new DBoW3::Vocabulary();
  try {
    v->load(path);
  } catch (const std::exception& e) {
    set_err(err, errlen, e.what());
    delete v;
    return nullptr;
  }
  return v;
}

int dbow_save(void* h, const char* path, int compressed) {
  static_cast<DBoW3::Vocabulary*>(h)->save(path, compressed != 0);
  return 0;
}

void dbow_free(void* h) { delete static_cast<DBoW3::Vocabulary*>(h); }

int dbow_nodes(void* h) { return static_cast<int>(Peek::nodes(*static_cast<DBoW3::Vocabulary*>(h)).size()); }

// info4 = {k, L, scoring, weighting}; per node: parent, weight, 32 descriptor bytes, word id (-1 when not a word);
// children: (parent, child) pairs in each node's child order, parents ascending.
int dbow_dump(void* h, int* info4, int* parent, double* weight, uint8_t* desc, int* word, int* children) {
  auto* v = static_cast<DBoW3::Vocabulary*>(h);
  const auto& nodes = Peek::nodes(*v);
  info4[0] = v->getBranchingFactor();
  info4[1] = v->getDepthLevels();
  info4[2] = v->getScoringType();
  info4[3] = v->getWeightingType();
  int c = 0;
  for (size_t i = 0; i < nodes.size(); ++i) {
    const auto& n = nodes[i];
    parent[i] = i == 0 ? -1 : static_cast<int>(n.parent);
    weight[i] = n.weight;
    memset(desc + 32 * i, 0, 32);
    if (!n.descriptor.empty()) memcpy(desc + 32 * i, n.descriptor.ptr<uchar>(), 32);
    word[i] = -1;
    for (int ch : n.children) {
      children[2 * c] = static_cast<int>(i);
      children[2 * c + 1] = ch;
      ++c;
    }
  }
  const auto& words = Peek::words(*v);
  for (size_t w = 0; w < words.size(); ++w)
    if (words[w]) word[words[w]->id] = static_cast<int>(w);
  return c;
}

// Vocabulary::transform(features, BowVector): returns the vector's length, writes up to cap (word, value) pairs
int dbow_transform(void* h, const uint8_t* desc, int n, int* words, double* vals, int cap) {
  DBoW3::BowVector bv;
  static_cast<DBoW3::Vocabulary*>(h)->transform(rows_of(desc, n), bv);
  int i = 0;
  for (const auto& kv : bv) {
    if (i < cap) {
      words[i] = static_cast<int>(kv.first);
      vals[i] = kv.second;
    }
    ++i;
  }
  return i;
}

double dbow_score(void* h, const int* wa, const double* va, int na, const int* wb, const double* vb, int nb) {
  DBoW3::BowVector a, b;
  for (int i = 0; i < na; ++i) a.addWeight(wa[i], va[i]);
  for (int i = 0; i < nb; ++i) b.addWeight(wb[i], vb[i]);
  return static_cast<DBoW3::Vocabulary*>(h)->score(a, b);
}

}  // extern "C"
