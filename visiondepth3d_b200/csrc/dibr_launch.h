// dibr_launch.h -- argument blocks and launch prototypes shared by dibr_kernels.cu
// (device code) and vd3d_api.cu (host orchestration).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/vd3d.h"
#include "dibr_kernels.cuh"

namespace vd3d {

struct IngestArgs {
  const uint8_t* frame;  // BGR u8 [src_h, src_w, 3]
  const uint8_t* depth;  // u8 [src_h, src_w, depth_ch]
  int depth_ch;
  int src_w, src_h;
  int cx0, cy0, cw, ch;  // aspect crop (core/render_3d.py:1236-1248)
  int tw, th;            // target_eye size
  float* tdf;            // TemporalDepthFilter state [th, tw]
  float* rgb_s;          // resized RGB planes [3, th, tw] or null on the identity path
  float alpha, one_minus_alpha;
  const DevState* st;
  // auto_crop_black_bars: the crop of this frame is derived on the device from the two words k_black_bars left in
  // bars (FrameScalars::bars) and the aspect ratio; cx0 .. ch above are then unused.  null: the fixed crop above.
  const uint32_t* bars;
  double aspect;
  int32_t* crop_out;  // (top, bottom) of the frame, written once (may be null)
};

// centre crop of a w x h frame to `ratio` (core/render_3d.py:1236-1248), fp64 like the reference's Python floats;
// rect = {x0, y0, w, h}
__host__ __device__ inline void aspect_crop(int w, int h, double ratio, int* rect) {
  rect[0] = 0;
  rect[1] = 0;
  rect[2] = w;
  rect[3] = h;
  const double cur = (double)w / (double)h;
  if (fabs(cur - ratio) > 0.01) {
    if (cur > ratio) {
      rect[2] = (int)(h * ratio);
      rect[0] = (w - rect[2]) / 2;
    } else {
      rect[3] = (int)(w / ratio);
      rect[1] = (h - rect[3]) / 2;
    }
  }
}
// (top, bottom) of detect_black_bars from the two words of k_black_bars (0: no bright row)
__host__ __device__ inline void bar_rows(int h, uint32_t first, uint32_t last, int* top, int* bottom) {
  *top = first ? h - (int)first : 0;
  *bottom = last ? h - (int)last : 0;
}
// The source rectangle of one auto-cropped frame: the rows of the black bars off (crop_black_bars_torch, which keeps the
// frame when top + bottom >= H), then the aspect crop on what is left (1238-1248).  first / last: the words of
// k_black_bars.
__host__ __device__ inline void black_bar_crop(int src_w, int src_h, uint32_t first, uint32_t last, double ratio,
                                               int* rect, int* top, int* bottom) {
  bar_rows(src_h, first, last, top, bottom);
  int y0 = *top, rows = src_h - *top - *bottom;
  if (*top + *bottom >= src_h) {
    y0 = 0;
    rows = src_h;
  }
  aspect_crop(src_w, rows, ratio, rect);
  rect[1] += y0;
}

struct LoopArgs {
  double fg, mg, bg;  // render_sbs_3d arguments
  double ipd;
  int resized_width;
  int use_floating_window, use_subject_tracking;
  long long crop_count;  // elements of the centre crop
  long long npix;        // th*tw
  float dyn_min, dyn_span;
};

struct ShiftArgs {
  vd3d_shift_params p;
  int W, H;
};

struct ComposeArgs {
  const uint8_t* src_u8;  // identity path: BGR u8 source frame (else null)
  int src_pitch, cx0, cy0;
  const float* src_f32;  // RGB planes [3,H,W]
  const float* shift;
  const float2* e2;
  const float* xs;
  const float* ys;
  int H, W;
  int k, feather;
  int grade;
  float sat, con, bri;
  uint8_t* left;
  uint8_t* right;
};

struct DofArgs {
  const uint8_t* src_l;
  const uint8_t* src_r;
  uint8_t* dst_l;
  uint8_t* dst_r;
  int H, W;
  const float* depth;
  int dh, dw;
  float focal, focus_w, idx_max;
  const FrameScalars* fs;  // non-null: focal = FocalDepthTracker state of this frame
  int nlevels;
  int ksize[8];
  int koff[8];
  const float* kern;
  int halo;
  float sat, con, bri;
};

struct PostArgs {
  const uint8_t* left;
  const uint8_t* right;
  int H, W;
  const FrameScalars* fs;  // bar width / side (may be null)
  int sharpen;
  float kc, ke;
  int fmt;
  int per_eye_w, per_eye_h;
  int fit_x0, fit_y0, fit_w, fit_h;  // placement of the resized eye inside the per-eye canvas
  int sx, sy;                        // integer INTER_AREA factors
  float inv_area;
  // general (non-integer) INTER_AREA shrink = cv2's ResizeArea_ tables (xal == null: integer / identity path).
  // Per fitted column / row: first source index, tap count, fp32 weights [index * area_t + k].
  const int* xofs;
  const int* xcnt;
  const float* xal;
  const int* yofs;
  const int* ycnt;
  const float* yal;
  int area_t;
  // lin != 0: cv2's INTER_AREA emulation when an axis is enlarged (fixed-point bilinear): xofs/yofs = first source
  // index, xal/yal = the two 11-bit weights per index stored as floats (exact integers), area_t == 2
  int lin;
  uint8_t* out;
  int out_w, out_h;
};

void launch_ingest(const IngestArgs& a, cudaStream_t s);
// detect_black_bars (core/render_3d.py:293-316) on a u8 BGR frame [h, w, 3]: integer row sums of cv2 gray, row y bright
// when sum > threshold * w; atomicMax(words[0], h - y) and atomicMax(words[1], y + 1) over the bright rows (the caller
// zeroes words).  One warp per row.
void launch_black_bars(const uint8_t* frame, int h, int w, int threshold, uint32_t* words, cudaStream_t s);
void launch_resize_planar(const float* src, int C, int sh, int sw, float* dst, int oh, int ow, cudaStream_t s);
// 3 histogram passes + 3 bin searches; b may be null.  b's region must lie inside a's
// and share a.data.  nblocks = grid of the pass kernels.
constexpr int kSelectLaunches = 6;
void launch_select(const SelJob& a, const SelJob* b, int nblocks, cudaStream_t s);
void launch_fin_pct(const SelJob& j, float w_lo, float w_hi, float alpha, float oma, DevState* st, FrameScalars* fs,
                    cudaStream_t s);
void launch_normalize(const float* tdf, float* dn, const float* dn_prev, int th, int tw, const DevState* st,
                      FrameScalars* fs, cudaStream_t s);
void launch_fin_norm(const SelJob& j, const LoopArgs& la, DevState* st, FrameScalars* fs, cudaStream_t s);
void launch_set_ranks(SelTarget* tg, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3, cudaStream_t s);
void launch_set_shifts(FrameScalars* fs, double fg, double mg, double bg, cudaStream_t s);
void launch_d0(const float* src, int sh, int sw, float* d0, int H, int W, const float* xs, const float* ys,
               float strength, cudaStream_t s);
void launch_fin_d0(const SelJob& q, const SelJob& sj, float w_lo, float w_hi, FrameScalars* fs, cudaStream_t s);
void launch_shape(float* d, int n, const FrameScalars* fs, float mid, float gamma, cudaStream_t s);
void launch_fin_shape(const SelJob& sj, const ShiftArgs& sa, DevState* st, FrameScalars* fs, cudaStream_t s);
void launch_shift(const float* d, float* shift, int H, int W, const FrameScalars* fs, int edge_mask, float feather,
                  cudaStream_t s);
void launch_warp_edges(const float* d, const float* shift, float2* e2, int H, int W, const float* xs,
                       const float* ys, float feather, cudaStream_t s);
int compose_smem_bytes(int k);
cudaError_t init_kernel_attributes();
void launch_compose(const ComposeArgs& a, cudaStream_t s);
void launch_dof(const DofArgs& a, int eyes, cudaStream_t s);
void launch_post(const PostArgs& a, cudaStream_t s);
void launch_grade_f32(const float* src, float* dst, int n, float sat, float con, float bri, cudaStream_t s);
void launch_resize_cubic_u8(const uint8_t* src, int h, int w, int ch, uint8_t* dst, int oh, int ow, cudaStream_t s);
void launch_add_weighted(const uint8_t* a, float alpha, const uint8_t* b, float beta, uint8_t* dst, size_t n,
                         cudaStream_t s);
// sr_kernels.cu: the x4 output of the SR network (last conv f32 NHWC [h*w, 48] + network input BGR u8 [h,w,3]) resampled
// with INTER_CUBIC straight to [oh, ow, 3] without materialising the 4h x 4w image
// postprocess_esr of an RRDBNet output: f32 RGB rows of ld floats -> clip [0,1], x255, truncate, BGR u8 [npix, 3]
void launch_rrdb_out(const float* rgb, int ld, uint8_t* bgr, size_t npix, cudaStream_t s);
void launch_sr_tail_cubic(const float* conv, const uint8_t* bgr, int h, int w, uint8_t* dst, int oh, int ow,
                          cudaStream_t s);
void launch_heal(const float* warped, const float* orig, const float* edge, float* out, int H, int W, float hs,
                 cudaStream_t s);

// ---- fast path (dibr_fast.cu) ------------------------------------------------------------------------------------
struct JobMem {  // device memory of one selection job
  uint32_t* hist1;   // [4096]
  uint32_t* hist2;   // [4][4096]
  uint32_t* hist3;   // [4][64]
  uint32_t* hist64;  // [64]
  uint32_t* count;
  SelTarget* tg;     // [4] (exact path only)
};

struct StatsArgs {
  int loop;          // 1: one render_sbs_3d loop iteration (from ingest); 0: pixel_shift_cuda entry (from d0)
  IngestArgs ia;     // loop only; ia.rgb_s unused
  float4* rgbx_s;    // [th, tw] RGBx of the frame resized to target_eye (null on the identity path)
  float4* rgbx;      // [H, W] RGBx upsampled to the warp resolution (null when not needed)
  float* dn;         // normalised depth of this frame [th, tw]
  const float* dn_prev;
  const float* core_depth;  // source of d0 [sh, sw] (== dn in loop mode)
  int sh, sw;
  float* d;          // [H, W] d0 -> shaped depth (in place)
  int H, W;
  const float* xs;
  const float* ys;
  LoopArgs la;
  ShiftArgs sa;
  uint32_t pct_rank[4];
  float pct_wlo, pct_whi;
  uint32_t q_rank[4];
  float q_wlo, q_whi;
  JobMem jm[5];
  DevState* st;
  FrameScalars* fs;  // zeroed by the host before the launch (the centre / motion sums accumulate into it)
  unsigned* bar;     // grid barrier counter, zeroed by the host before the launch
};

struct RenderArgs {
  ComposeArgs c;           // c.e2 unused; c.left / c.right only when fuse == 0
  const float4* src_rgbx;  // [H, W] RGBx source (resize paths); else c.src_u8 or c.src_f32
  const float* d;          // shaped depth [H, W]
  float feather_strength;
  int fuse;                // 0: write eyes; 1: bars + sharpen + 1:1 fit + SBS pack; 2: same with the 2:1 Half-SBS fit
  const FrameScalars* fs;  // bars (fuse != 0; may be null)
  int sharpen;
  float kc, ke;
  uint8_t* out;
  int out_w, per_eye_w;    // packed row length in pixels; width of one eye in the packed frame
};

bool render_supports(int feather, int k);
// inst: set to the (K, SRC, FUSE) of the k_render instance launched
cudaError_t launch_render(const RenderArgs& a, cudaStream_t s, int inst[3]);
cudaError_t stats_grid(int device, int* blocks);
cudaError_t launch_stats(const StatsArgs& a, int blocks, cudaStream_t s);
void launch_shift_fast(const float* d, float* shift, int H, int W, const FrameScalars* fs, int edge_mask, float feather,
                       cudaStream_t s);

}  // namespace vd3d
