// letterbox_launch.h -- launchers of letterbox.cu: the per-frame statistics of the reference's LetterboxTracker
// (core/render_depth.py:273-392), cv2.Canny with L2 gradients, and the depth re-pad of process_video2 (1919-1933).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vd3d {

// numpy's pairwise float32 summation splits a node above this size; the frame-wide luma sum is evaluated as a
// top tree over "cut" nodes of at most this many elements, one warp per node
constexpr int kLbCutNode = 4096;

// (start, length) of the cut nodes of numpy's pairwise tree over n elements, in left-to-right order
void lb_cut_nodes(int64_t n, int64_t* starts, int* lens, int* count, int cap);

struct LbRowArgs {
  const uint8_t* frames;     // [n, h, w, 3] BGR
  const uint8_t* prev_gray;  // [h, w] gray before frame 0, or null
  int n, h, w;
  uint8_t* gray;        // [n, h, w] cv2 BGR2GRAY of every frame
  float* y_mean;        // [n, h]
  float* y_var;         // [n, h]
  float* s_mean;        // [n, h]
  uint32_t* hist;       // [n, 64], zeroed by the caller
  unsigned long long* absdiff;  // [n], zeroed by the caller
};
void launch_lb_rows(const LbRowArgs& a, cudaStream_t s);

// float32 mean of the Rec.709 luma of each whole frame, numpy's pairwise order: node sums, then the top tree
void launch_lb_frame_mean(const uint8_t* frames, int n, int64_t npix, const int64_t* node_start, const int* node_len,
                          int nodes, float* node_sum, float* y_mean, cudaStream_t s);

// cv2.Canny(gray, low, high, 3, L2gradient=True) of n planes; low2/high2 are the squared integer thresholds.
// Scratch: mag and label [n*h*w] int32, strong flags [n*h*w] u8.  edges (optional) gets 0/255, row_count (optional,
// zeroed by the caller) the edge pixels per row [n*h].
void launch_canny(const uint8_t* gray, int n, int h, int w, int low2, int high2, int32_t* mag, int32_t* label,
                  uint8_t* flag, uint8_t* edges, int32_t* row_count, cudaStream_t s);

// fill the bar rows of dst [h, w] with the median of the core rows [top, top + core_h); hist is 256 words of scratch
void launch_lb_pad(uint8_t* dst, int h, int w, int top, int core_h, uint32_t* hist, cudaStream_t s);

}  // namespace vd3d
