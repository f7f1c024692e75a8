// Minimal stand-in for the slice of OpenCV's core module that DBoW3 (Vocabulary.cpp, DescManip.cpp, ...) uses, so the
// unmodified DBoW3 sources compile without OpenCV.  Mat is a dense row-major matrix that owns its bytes (copies are
// deep: DBoW3 never relies on shared headers).  FileStorage / FileNode exist only so the YAML paths compile; using them
// throws.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <assert.h>
#include <limits.h>

#include <cmath>
#include <stdexcept>
#include <string>
#include <vector>

typedef unsigned char uchar;
#define CV_8U 0
#define CV_8UC1 0
#define CV_32F 5

namespace cv {

struct Scalar {
  double v;
  static Scalar all(double x) { return Scalar{x}; }
};

class Mat {
 public:
  int rows = 0, cols = 0;
  Mat() {}
  Mat(int r, int c, int t) { create(r, c, t); }
  int type() const { return type_; }
  size_t elemSize() const { return type_ == CV_32F ? 4 : 1; }
  bool empty() const { return buf_.empty(); }
  bool isContinuous() const { return true; }
  void create(int r, int c, int t) {
    rows = r;
    cols = c;
    type_ = t;
    buf_.assign(static_cast<size_t>(r) * c * elemSize(), 0);
  }
  template <typename T = uchar>
  T* ptr(int i = 0) { return reinterpret_cast<T*>(buf_.data() + static_cast<size_t>(i) * cols * elemSize()); }
  template <typename T = uchar>
  const T* ptr(int i = 0) const {
    return reinterpret_cast<const T*>(buf_.data() + static_cast<size_t>(i) * cols * elemSize());
  }
  Mat row(int r) const {
    Mat m(1, cols, type_);
    memcpy(m.buf_.data(), ptr<uchar>(r), cols * elemSize());
    return m;
  }
  Mat rowRange(int a, int b) const {
    Mat m(b - a, cols, type_);
    memcpy(m.buf_.data(), ptr<uchar>(a), static_cast<size_t>(b - a) * cols * elemSize());
    return m;
  }
  Mat clone() const { return *this; }
  void release() { *this = Mat(); }
  // the float-descriptor mean of DescManip::meanValue; binary vocabularies never reach it
  Mat operator*(float s) const {
    Mat m = *this;
    float* p = m.ptr<float>();
    for (int i = 0; i < rows * cols; ++i) p[i] *= s;
    return m;
  }
  Mat& operator+=(const Mat& o) {
    float* p = ptr<float>();
    const float* q = o.ptr<float>();
    for (int i = 0; i < rows * cols; ++i) p[i] += q[i];
    return *this;
  }
  void setTo(const Scalar& s) {
    if (type_ == CV_32F) {
      float* p = ptr<float>();
      for (int i = 0; i < rows * cols; ++i) p[i] = static_cast<float>(s.v);
    } else {
      memset(buf_.data(), static_cast<int>(s.v), buf_.size());
    }
  }
  static Mat zeros(int r, int c, int t) { return Mat(r, c, t); }

 private:
  int type_ = 0;
  std::vector<uchar> buf_;
};

[[noreturn]] inline void no_filestorage() { throw std::runtime_error("YAML vocabularies need OpenCV's FileStorage"); }

class FileNode;
class FileNodeIterator {};
class FileNode {
 public:
  FileNode operator[](const std::string&) const { no_filestorage(); }
  FileNode operator[](const char*) const { no_filestorage(); }
  FileNode operator[](int) const { no_filestorage(); }
  size_t size() const { no_filestorage(); }
  bool empty() const { no_filestorage(); }
  explicit operator int() const { no_filestorage(); }
  explicit operator double() const { no_filestorage(); }
  explicit operator float() const { no_filestorage(); }
  explicit operator std::string() const { no_filestorage(); }
  FileNodeIterator begin() const { no_filestorage(); }
  FileNodeIterator end() const { no_filestorage(); }
};

class FileStorage {
 public:
  enum { READ = 0, WRITE = 1 };
  FileStorage() {}
  FileStorage(const std::string&, int) { no_filestorage(); }
  bool isOpened() const { return false; }
  FileNode operator[](const std::string&) const { no_filestorage(); }
  FileNode operator[](const char*) const { no_filestorage(); }
  template <typename T>
  FileStorage& operator<<(const T&) { no_filestorage(); }
};

}  // namespace cv
