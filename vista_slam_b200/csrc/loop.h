// Internal interface between the ORB kernels (orb.cu) and the loop detector (bow.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace sta {

constexpr int kOrbLevels = 8;
constexpr int kOrbMaxKeypoints = 4096;  // kept keypoints per frame, ties of retainBest included
constexpr int kOrbMaxCandidates = 1 << 16;  // FAST corners past the border filter, all levels

// Scratch layout of one frame size (byte offsets into one device buffer).
struct OrbLayout {
  int H, W;
  int h[kOrbLevels], w[kOrbLevels];
  long long lvl[kOrbLevels];  // offset of level l in the pyramid / blurred / score images
  long long pix;              // pixels of all levels
  int quota[kOrbLevels];      // features per level
  size_t pyr, blur, score, cand, resp, hist, counters, alive, kept, total;
};

bool orb_size_ok(int H, int W);
OrbLayout orb_layout(int H, int W);

// Device outputs in canonical (level, y, x) order; count [1] receives the number of keypoints and the counters inside
// the scratch (OrbLayout::counters) flag an overflow in counters[3].
struct OrbOut {
  int2* xy;         // level coordinates
  int* level;
  float2* pts;      // level-0 coordinates
  float* angle;
  float* response;
  uint8_t* desc;    // [kOrbMaxKeypoints][32]
  int* count;
};

// F frames of one size (frame-major [F][H][W] input, F scratch slices of s.total bytes, F output slots of
// kOrbMaxKeypoints and F counts); each frame's result is the one of a call with F = 1.
int orb_run(const OrbLayout& s, void* scratch, const void* frame, int is_f32, const OrbOut& out, cudaStream_t st,
            int F = 1);

}  // namespace sta
