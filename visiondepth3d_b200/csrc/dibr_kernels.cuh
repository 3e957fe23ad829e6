// dibr_kernels.cuh -- sm_90a kernels of the DIBR (depth-image-based rendering) stage.
//
// Reference behaviour restated from core/render_3d.py (file:line cited per kernel);
// arithmetic follows oracle/dibr.py one rounding at a time: this TU is compiled with
// -fmad=false and uses __fmaf_rn exactly where torch / cv2 fuse (grid_sample and
// bilinear accumulation, Gaussian conv and filter2D chains, linspace).
//
// Memory-bound design (H100: 132 SMs, 3.35 TB/s HBM3, 50 MB L2):
//   * u8 frames are consumed as they arrive (BGR interleaved) -- no f32 RGB planes
//     are materialised on the identity-resize path (4K Full-SBS);
//   * every intermediate (depth planes, shift map, edge masks, eyes) is written once
//     and re-read from L2; order statistics use a 3-pass radix select on the fp32
//     bit pattern (12+12+6 bits) instead of torch.quantile's full sort;
//   * all per-frame scalars (EMAs, trackers, quantiles) live in device memory and are
//     advanced by single-thread kernels, so a frame is a fixed kernel sequence with no
//     host synchronisation and replays from a CUDA graph.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vd3d {

// ---------------------------------------------------------------------------
// device-resident state
// ---------------------------------------------------------------------------
struct DevState {  // persists across frames
  // module singletons (core/render_3d.py:284-285,500,511)
  float pct_lo, pct_hi;
  int pct_init;
  double conv_val;
  int conv_init;
  double fw_prev;
  int fw_count;
  int bar_prev;
  // per-render objects (core/render_3d.py:1174-1182)
  int tdf_init;
  double sm_fg, sm_mg, sm_bg;
  int sm_init;
  double focal, focal_alpha;
  int focal_init;
  int have_prev_depth;
  int dn_cur;  // which of the two normalised-depth planes holds this frame
};

struct FrameScalars {  // recomputed every frame
  // DepthPercentileEMA.normalize
  float q_lo, q_hi;
  int pct_flat;
  float n_lo, n_den;  // normalise with (d - n_lo) / n_den
  // centre-crop statistics / motion
  double sum, sumsq, mad_sum;
  double dyn, fg, mg, bg;
  double motion, focal;
  float subj_norm;
  double stable_zero;
  int bar_width, bar_side;
  // pixel_shift_cuda
  float subj_raw, st_lo, st_hi, st_den, st_subj;
  int st_flat;
  float subj;
  double zpo;
  // coefficients of the shift map (all already rounded like the reference rounds them)
  float c_fg, c_fgm, c_mg, c_bg, c_bgm, c_pb, c_half, c_mid, c_gamma;
  float c_zpo, c_max, c_conv, c_m1, c_m2;
  int use_zpo, use_conv;
  // auto_crop_black_bars (k_black_bars): max(H - y) and max(y + 1) over the bright rows y of the frame; 0 = none
  uint32_t bars[2];
};

struct SelTarget {
  uint32_t rank;   // 0-based rank within the selected set
  uint32_t p1, p2; // chosen bins of pass 1 / 2
  uint32_t r1, r2; // residual rank inside the chosen bin
  int alias;       // >=0: shares (p1[,p2]) histogram with an earlier target
  int alias2;
  uint32_t bits;   // result: fp32 bit pattern of the selected element
};

struct SelJob {
  const float* data;
  int W;               // row pitch in elements
  int x0, x1, y0, y1;  // region [y0,y1) x [x0,x1)
  int masked;          // keep 0.05 < v < 0.95 only (estimate_subject_depth)
  int ntargets;        // <= 4
  int rank_from_count; // target 0 rank = (n-1)/2 (torch.median lower middle)
  uint32_t* hist1;     // [4096]
  uint32_t* hist2;     // [4][4096]
  uint32_t* hist3;     // [4][64]
  uint32_t* hist64;    // [64] histc bins (or null)
  SelTarget* tg;       // [4]
  uint32_t* count;     // number of selected elements
};

}  // namespace vd3d
