// tiled_launch.h -- launchers of tiled_depth.cu: the reference's tiled depth inference (core/render_depth.py:102-170)
// and its percentile front end _normalize_to_u8 (173-194).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vd3d {

// one tile of one frame.  Core rect [y0, y0 + ch) x [x0, x0 + cw) of the frame; padded crop [yp0, yp0 + pch) x
// [xp0, xp0 + pcw); the engine sees the crop INTER_CUBIC-resized to [rh, rw] (multiples of 14) and predicts at that size
struct TileJob {
  const uint8_t* frame;  // BGR [h, w, 3]
  uint8_t* crop;         // BGR [rh, rw, 3]
  const float* pred;     // [rh, rw]
  const float* wgt;      // [ch, cw]: the tile's Hann weights
  int y0, x0, ch, cw;
  int yp0, xp0, pch, pcw;
  int rh, rw;
};

// every job's crop in one launch (frame width fw)
void launch_tile_gather(const TileJob* jobs, int njobs, int max_rh, int max_rw, int fw, cudaStream_t s);

// n frames [h, w] of out = sum(center * w) / max(sum(w), 1e-8) over the tiles covering each pixel, in plan order.
// jobs: n x (ny * nx) in row-major tile order, tiles start every `step` rows / columns and are `tile` long.
// mm_keys [2n] (min, max per frame) receives order keys of the frame's NaN-free extremes.
void launch_tile_blend(const TileJob* jobs, int n, int h, int w, int step, int tile, int nx, int ny, float* out,
                       uint32_t* mm_keys, cudaStream_t s);

// decode order keys to floats
void launch_keys_to_float(const uint32_t* keys, int count, float* out, cudaStream_t s);

// the order statistics _normalize_to_u8 needs: ranks of the two neighbours of each percentile, then the minimum and
// the maximum of the plane
constexpr int kSelTargets = 6;
struct NormArgs {
  uint32_t rank[kSelTargets];
  float gamma_lo, gamma_hi;  // numpy's interpolation weights of the two percentiles
  int invert;
};
// device words of scratch per frame that launch_normalize_u8 needs
size_t normalize_scratch_words();
// n planes d [n, h*w] -> u8 [n, h*w]: nan_to_num, exact selection, numpy's linear interpolation and branches, truncation,
// inversion.  stats (optional, device) receives (lo, hi, min, max) per frame.
void launch_normalize_u8(const float* d, int n, int64_t npix, const NormArgs& a, uint32_t* scratch, uint8_t* u8,
                         float* stats, cudaStream_t s);

}  // namespace vd3d
