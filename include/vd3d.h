/* vd3d.h -- C ABI of libvd3d.so, the H100 (sm_90a) depth->stereo engine.
 *
 * The reference (VisionDepth3D) has no FFI: its boundary is the Python function
 * surface of core/render_3d.py and the `pipe` callable of core/render_depth.py
 * (SURVEY.md section 8(b)).  Each entry point below names the reference function it
 * replaces; visiondepth3d_b200/render_3d.py and render_depth.py bind them with
 * ctypes and re-expose the reference's names and signatures (INTEGRATION.md).
 *
 * Conventions: every function returns 0 on success or a negative vd3d_status;
 * nothing throws; a ctx is not re-entrant, distinct ctxs are independent.
 * Image pointers may be host or device memory as stated by `mem`
 * (VD3D_MEM_HOST / VD3D_MEM_DEVICE); outputs are caller-owned buffers.
 * There is no CPU fallback: without a CUDA device vd3d_create fails.
 */
#ifndef VD3D_H
#define VD3D_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vd3d_ctx vd3d_ctx;
typedef struct vd3d_depth vd3d_depth; /* depth-forward engine, see the end of this header */

typedef enum {
  VD3D_OK = 0,
  VD3D_ERR_CUDA = -1,        /* CUDA runtime error; see vd3d_last_error */
  VD3D_ERR_ARG = -2,         /* bad argument */
  VD3D_ERR_UNSUPPORTED = -3, /* valid in the reference, not implemented here */
  VD3D_ERR_NOMEM = -4,
  VD3D_ERR_STATE = -5        /* call sequence error (e.g. weights not loaded) */
} vd3d_status;

enum { VD3D_MEM_HOST = 0, VD3D_MEM_DEVICE = 1 };

/* output_format of render_sbs_3d / format_3d_output (core/render_3d.py:837-860) */
enum {
  VD3D_FMT_HALF_SBS = 0,
  VD3D_FMT_FULL_SBS = 1,
  VD3D_FMT_ANAGLYPH = 2,   /* "Red-Cyan Anaglyph" */
  VD3D_FMT_INTERLACED = 3, /* "Passive Interlaced" */
  VD3D_FMT_VR = 4          /* 2 x 1440x1600: eyes fitted by pad_to_aspect_ratio (INTER_AREA shrink only) */
};

/* which temporal state vd3d_reset_state clears */
enum {
  VD3D_STATE_GLOBAL = 1, /* module singletons: depth_ema_norm, conv_ema,
                            floating_window_tracker, bar_easer
                            (core/render_3d.py:284-285,500,511) */
  VD3D_STATE_CLIP = 2    /* per-render objects created at core/render_3d.py:1174-1182 */
};

/* kwargs of pixel_shift_cuda (core/render_3d.py:561-590).  Shifts are Python
 * floats (double) in the reference and are rounded to fp32 where a tensor op
 * consumes them, which the kernels reproduce. */
typedef struct {
  double fg_shift, mg_shift, bg_shift;
  int32_t blur_ksize;
  double feather_strength;
  double max_pixel_shift_percent;
  double parallax_balance;
  double zero_parallax_strength;
  int32_t use_subject_tracking;
  int32_t enable_floating_window;
  int32_t enable_feathering;
  int32_t enable_edge_masking;
  double convergence_strength;
  int32_t enable_dynamic_convergence;
  double depth_pop_gamma, depth_pop_mid;
  double depth_stretch_lo, depth_stretch_hi;
  double fg_pop_multiplier, bg_push_multiplier;
  double subject_lock_strength;
} vd3d_shift_params;

/* arguments of render_sbs_3d (core/render_3d.py:933-985) that reach the frame loop */
typedef struct {
  int32_t output_width, output_height;
  double fg_shift, mg_shift, bg_shift;
  double sharpness_factor;
  int32_t output_format;      /* VD3D_FMT_* */
  double aspect_ratio;        /* aspect_ratios[selected_aspect_ratio.get()] */
  double dof_strength;
  double feather_strength;
  int32_t blur_ksize;
  int32_t use_subject_tracking, use_floating_window;
  double max_pixel_shift_percent;
  int32_t preserve_original_aspect;
  double zero_parallax_strength;
  int32_t enable_edge_masking, enable_feathering;
  int32_t original_video_width, original_video_height; /* 0 = None */
  double convergence_strength;
  int32_t enable_dynamic_convergence;
  double ipd_factor;
  double color_saturation, color_contrast, color_brightness;
  /* detect_black_bars + crop_black_bars_torch on every frame (core/render_3d.py:293-326,1238-1242): the rows of the
   * top / bottom black bars found on the colour frame are cut from the frame and the depth map before the aspect crop.
   * Sizes do not change per frame.  The reference sizes a preserve_original_aspect output with original_video_* = None
   * from the cropped first frame; here 0 means the uncropped source size, so callers pass that size explicitly
   * (vd3d_detect_black_bars on the first frame). */
  int32_t auto_crop_black_bars;
} vd3d_render_params;

/* sizes derived at core/render_3d.py:1074-1138,1250-1259 */
typedef struct {
  int32_t crop_x0, crop_y0, crop_w, crop_h;
  int32_t target_eye_w, target_eye_h;
  int32_t resized_width, resized_height;
  int32_t per_eye_w, per_eye_h;
  int32_t out_width, out_height;
} vd3d_size_plan;

/* per-frame scalars, for parity tests and progress reporting */
typedef struct {
  float pct_lo, pct_hi;       /* DepthPercentileEMA state after this frame */
  float subj_raw, stretch_lo, stretch_hi, subj_shaped;
  float subj_norm;            /* estimate_subject_depth(depth_tensor) (1334/1390) */
  double dyn_scale, fg, mg, bg;
  double zero_parallax_offset;
  double focal_depth, motion_metric;
  double stable_zero;
  int32_t bar_width, bar_side; /* side: 0 none, 1 right, 2 left */
  int32_t crop_top, crop_bottom; /* black-bar rows detected on the frame (0 without auto_crop_black_bars) */
} vd3d_frame_info;

/* sizeof() of the ABI structs, so bindings can verify their layout:
 * 0 vd3d_shift_params, 1 vd3d_render_params, 2 vd3d_size_plan, 3 vd3d_frame_info, 4 vd3d_upscale_params,
 * 5 vd3d_tile */
int vd3d_struct_size(int which);

/* ---- lifecycle ------------------------------------------------------- */
int vd3d_create(int device, vd3d_ctx** out);
void vd3d_destroy(vd3d_ctx* ctx);
const char* vd3d_last_error(vd3d_ctx* ctx); /* ctx may be NULL: last create error */
int vd3d_reset_state(vd3d_ctx* ctx, uint32_t which);
/* pinned host memory for the end-to-end path */
void* vd3d_host_alloc(size_t bytes);
void vd3d_host_free(void* p);
/* the stream all work of this ctx is enqueued on (cudaStream_t) */
void* vd3d_stream(vd3d_ctx* ctx);
int vd3d_sync(vd3d_ctx* ctx);
/* number of kernels this ctx has launched since creation (bench: gpu_launches) */
uint64_t vd3d_launch_count(vd3d_ctx* ctx);
/* device-side stage timing for the roofline report (CUDA events on the ctx stream):
 * stage 0 = whole DIBR frame (ingest..pack), 1 = compose kernel, 2 = depth forward.
 * vd3d_profile_collect synchronises, returns the summed time and sample count since the
 * last collect, and resets. */
int vd3d_profile(vd3d_ctx* ctx, int enable);
int vd3d_profile_collect(vd3d_ctx* ctx, int stage, double* total_ms, int* count);
/* replay the per-frame kernel sequence from a captured CUDA graph (default 1) */
int vd3d_set_graphs(vd3d_ctx* ctx, int enable);
/* DIBR arithmetic mode.  0 (default): persistent statistics kernel + fused warp/feather/compose/pack kernel, fp32
 * hardware pow/exp, separable box sums -- inside the 1e-3 / 1-LSB tolerances of the reference's outputs.
 * 1: one kernel per reference op, correctly rounded transcendentals, the reference's row-major summation order
 * (bit-for-bit with oracle/dibr.py; what the exactness tests drive).  Env VD3D_EXACT=1 makes 1 the default. */
int vd3d_set_exact(vd3d_ctx* ctx, int enable);
int vd3d_get_exact(vd3d_ctx* ctx);
/* 1 while CUDA-graph replay is on; 0 after vd3d_set_graphs(ctx, 0) or after a failed capture fell back to eager launches */
int vd3d_graphs_active(vd3d_ctx* ctx);

/* ---- DIBR ------------------------------------------------------------ */
/* pixel_shift_cuda (core/render_3d.py:561-712).
 * rgb: f32 planar RGB [3,in_h,in_w] in 0..1; depth: f32 [in_h,in_w];
 * left/right: u8 BGR interleaved [height,width,3]; shift: f32 [height,width] or NULL.
 * Mutates the floating-window tracker held by ctx (the module singleton). */
int vd3d_pixel_shift(vd3d_ctx* ctx, const float* rgb, const float* depth, int in_h, int in_w,
                     int width, int height, const vd3d_shift_params* p, uint8_t* left_bgr,
                     uint8_t* right_bgr, float* shift, int mem, vd3d_frame_info* info);

/* sizing rules of render_sbs_3d (core/render_3d.py:1074-1138,1236-1259) */
int vd3d_plan_sizes(int src_w, int src_h, const vd3d_render_params* rp, vd3d_size_plan* out);

/* one iteration of the render_sbs_3d frame loop (core/render_3d.py:1227-1419):
 * frame_to_tensor/depth_to_tensor, aspect crop, resize, TemporalDepthFilter,
 * DepthPercentileEMA, ShiftSmoother, dynamic parallax scale, pixel_shift_cuda,
 * FocalDepthTracker, DOF, colour grade, floating-window bars, sharpen, eye fit,
 * format_3d_output.  frame/depth: u8 BGR [src_h,src_w,3] (depth may also be one
 * channel: depth_channels = 1); out: u8 BGR [out_height,out_width,3]. */
int vd3d_render_frame(vd3d_ctx* ctx, const uint8_t* frame_bgr, const uint8_t* depth, int depth_channels,
                      int src_h, int src_w, const vd3d_render_params* rp, uint8_t* out_bgr, int mem,
                      vd3d_frame_info* info);

/* Throughput form of the same loop: n frames, host or device arrays of
 * frame pointers; H2D of frame i+1 and D2H of frame i-1 overlap the kernels of
 * frame i on separate streams.  State carries across calls exactly as across
 * loop iterations.  infos may be NULL. */
int vd3d_render_clip(vd3d_ctx* ctx, int n, const uint8_t* const* frames, const uint8_t* const* depths,
                     int depth_channels, int src_h, int src_w, const vd3d_render_params* rp,
                     uint8_t* const* outs, int mem, vd3d_frame_info* infos);

/* depth + stereo in one pipelined loop: depth of frame i is inferred on the GPU by `depth`
 * (vd3d_depth_infer_device) and handed to the DIBR loop in HBM as a 1-channel u8 map -- the
 * in-memory replacement of the reference's XVID depth-video round trip (SURVEY 0.5). */
int vd3d_render_clip_depth(vd3d_ctx* ctx, vd3d_depth* depth, int n, const uint8_t* const* frames, int src_h,
                           int src_w, const vd3d_render_params* rp, uint8_t* const* outs, int mem);

/* (top, bottom) of each of the n frames of the last vd3d_render_clip / vd3d_render_clip_depth call, as int32 pairs.
 * The per-frame values are copied behind the output frames on the device-to-host stream (no synchronisation inside the
 * clip).  VD3D_ERR_STATE when that call had auto_crop_black_bars off or rendered fewer than n frames. */
int vd3d_last_crops(vd3d_ctx* ctx, int32_t* top_bottom, int n);

/* detect_black_bars (core/render_3d.py:293-316) on one u8 BGR frame [h,w,3]: top = first row whose cv2 gray mean is
 * above 10, bottom = h-1-last such row, both 0 when there is none.  The kernel the frame loop runs for
 * auto_crop_black_bars; synchronises. */
int vd3d_detect_black_bars(vd3d_ctx* ctx, const uint8_t* frame_bgr, int h, int w, int mem, int* top, int* bottom);

/* ---- letterbox tracker of the depth-video pass (core/render_depth.py:273-573, 1919-1933) ---------------------------
 * Per-frame statistics of n u8 BGR frames [n,h,w,3] (contiguous; host or device memory per `mem`, w <= 8192), from
 * which the host-side tracker decides the bar rows:
 *   row_y_mean / row_y_var [n,h]: float32 mean and variance of the Rec.709 luma 0.2126 r + 0.7152 g + 0.0722 b, equal
 *     to numpy's float32 y.mean(axis=1) / y.var(axis=1) bit for bit (pairwise summation order);
 *   row_s_mean [n,h]: float32 mean of cv2 BGR2HSV's S; row_edges [n,h]: edge pixels of cv2.Canny(gray, 30, 90,
 *     apertureSize=3, L2gradient=True) per row;
 *   frame_y_mean [n]: float32 y.mean() of the whole frame; frame_hist [n,64]: 64-bin histogram of cv2 BGR2GRAY
 *     (bin = gray >> 2); frame_absdiff [n]: sum |gray - previous gray|, the previous gray being frame i-1, and for
 *     frame 0 prev_gray [h,w] (0 when prev_gray is null).
 * The records are host memory.  last_gray (optional, `mem` space) receives the gray plane of frame n-1.  Synchronises. */
int vd3d_letterbox_stats(vd3d_ctx* ctx, int n, const uint8_t* frames, int h, int w, const uint8_t* prev_gray, int mem,
                         float* row_y_mean, float* row_y_var, float* row_s_mean, int32_t* row_edges,
                         float* frame_y_mean, uint32_t* frame_hist, uint64_t* frame_absdiff, uint8_t* last_gray);
/* cv2.Canny(gray [h,w], low, high, apertureSize=3, L2gradient=True) -> dst [h,w] of 0/255, bit for bit */
int vd3d_canny_u8(vd3d_ctx* ctx, const uint8_t* gray, int h, int w, double low, double high, uint8_t* dst, int mem);
/* process_video2's depth re-pad: u8 depth [h,w] -> dst [h,w] with the INTER_CUBIC resize of the depth to
 * (w, h - top - bottom) at rows [top, h - bottom) and the bar rows filled with int(np.median(core)).  No bars, or
 * h - top - bottom <= 0 (the reference then drops the bars), copies the depth.  src and dst must not alias. */
int vd3d_letterbox_repad(vd3d_ctx* ctx, const uint8_t* src, int h, int w, int top, int bottom, uint8_t* dst, int mem);

/* ---- tiled depth inference (core/render_depth.py:46-51, 62-194) ----------------------------------------------------
 * The plan of an [h,w] image for (tile, pad) is infer_depth_tile's loop: core = max(1, tile - 2*pad), tiles start every
 * core rows / columns, row-major; each is a core rect of up to `tile` pixels, padded by `pad` and clipped to the image,
 * and the padded crop is INTER_CUBIC-resized to the next multiples of 14 (copied when it is one already).  Every entry
 * point checks that `tiles` is exactly that plan. */
typedef struct {
  int32_t y0, y1, x0, x1;     /* core rect [y0, y1) x [x0, x1) */
  int32_t yp0, yp1, xp0, xp1; /* padded crop */
  int32_t rh, rw;             /* crop size rounded up to multiples of 14: the engine's input and prediction size */
  int32_t cls;                /* index of the engine serving this tile (vd3d_depth_tiled); tiles of a class share rh, rw */
} vd3d_tile;
/* the crops the engine sees, of one u8 BGR frame [h,w,3], concatenated in plan order: out [sum(rh*rw*3)] */
int vd3d_tile_crops(vd3d_ctx* ctx, const uint8_t* frame, int h, int w, int tile, int pad, const vd3d_tile* tiles,
                    int n_tiles, uint8_t* out, int mem);
/* infer_depth_tile's blend: preds[t] f32 [rh,rw] (the prediction of tile t), weights[t] f32 [y1-y0, x1-x0] (its Hann
 * weights) -> out f32 [h,w] = sum(center * w) / max(sum(w), 1e-8f) with center = pred[y0-yp0 :, x0-xp0 :], accumulated
 * in plan order with float32 rounding.  minmax (optional, host) receives np.nanmin / np.nanmax of out. */
int vd3d_tile_blend(vd3d_ctx* ctx, int h, int w, int tile, int pad, const vd3d_tile* tiles, int n_tiles,
                    const float* const* preds, const float* const* weights, float* out, float* minmax, int mem);
/* _normalize_to_u8(d, (ow, oh), invert, (p_lo, p_hi)) on d f32 [h,w]: nan_to_num, np.percentile (linear, float32) at
 * p_lo and p_hi by exact selection, clip to [lo, hi] (min-max when hi - lo < 1e-6, flat 128 when that is flat too),
 * x255 truncated to u8, 255 - u8 when inverted, INTER_CUBIC to [oh,ow] -> out.  stats_out (optional, host): lo, hi,
 * min, max. */
int vd3d_normalize_u8(vd3d_ctx* ctx, const float* d, int h, int w, double p_lo, double p_hi, int invert, uint8_t* out,
                      int oh, int ow, float* stats_out, int mem);
/* The tiled depth-video step on n u8 BGR frames [h,w,3]: every tile crop of every frame in one launch, forwards of up
 * to 8 tiles per class through vd3d_depth_infer_batch_device on engines[cls] (created on vd3d_stream(ctx)), the blend
 * and _normalize_to_u8(p1, p99) of each frame to out_u8[i] [oh,ow].  weights[t]: device memory (uploaded once per
 * plan).  out_f32[i] (optional) receives the blended depth [h,w], minmax (optional, host) [n,2] its extremes.  Host
 * memory: one upload and one download per frame; device memory: nothing crosses PCIe.  Synchronises. */
int vd3d_depth_tiled(vd3d_ctx* ctx, vd3d_depth* const* engines, int n_classes, int n, const uint8_t* const* frames,
                     int h, int w, int tile, int pad, const vd3d_tile* tiles, int n_tiles, const float* const* weights,
                     int invert, int oh, int ow, uint8_t* const* out_u8, float* const* out_f32, float* minmax, int mem);

/* ---- exact frame sharding (SURVEY 8(e)) --------------------------------------------------
 * The loop is stateful (7 EMAs / trackers + the temporal depth plane).  A rank that renders frames
 * [a, b) exactly needs the state after frame a-1: vd3d_advance_state runs one loop iteration
 * WITHOUT rendering (all state updates, ~1/3 of the DIBR cost), vd3d_export_state /
 * vd3d_import_state move the state (struct + two f32 planes of target_eye size) between contexts
 * or GPUs (NCCL send/recv of the blob). */
int vd3d_advance_state(vd3d_ctx* ctx, const uint8_t* frame_bgr, const uint8_t* depth, int depth_channels,
                       int src_h, int src_w, const vd3d_render_params* rp, int mem);
size_t vd3d_state_bytes(vd3d_ctx* ctx);
int vd3d_export_state(vd3d_ctx* ctx, void* dst, size_t capacity, int mem);
int vd3d_import_state(vd3d_ctx* ctx, const void* src, size_t bytes, int mem);

/* drop the per-ctx clones / graphs built for `depth`; call before vd3d_depth_destroy(depth) */
int vd3d_release_depth(vd3d_ctx* ctx, vd3d_depth* depth);

/* Validate a render configuration without launching anything (sizes, eye-fit mode, DOF kernel bank): what
 * render_sbs_3d (core/render_3d.py:1086-1138) decides before it opens its writer.  0 or a negative error + message. */
int vd3d_check_config(vd3d_ctx* ctx, int src_h, int src_w, const vd3d_render_params* rp);

/* stage entry points (same kernels, exposed for stage-isolated parity tests) */
/* apply_color_grade (core/render_3d.py:734-767): f32 RGB planes [3,h,w] in 0..1 -> same (saturation around Rec.709
 * luma, contrast around 0.5, additive brightness, clamp) */
int vd3d_color_grade(vd3d_ctx* ctx, const float* rgb, int h, int w, double saturation, double contrast,
                     double brightness, float* out, int mem);
/* cv2.resize(u8 plane [h,w], (ow,oh), interpolation=cv2.INTER_CUBIC): the resize the depth writer applies to the u8
 * depth (core/render_depth.py:1917, 193): float32 bicubic (A = -0.75), round half to even */
int vd3d_resize_cubic_u8(vd3d_ctx* ctx, const uint8_t* src, int h, int w, uint8_t* dst, int oh, int ow, int mem);
/* the same on interleaved u8 [h,w,ch] (ch <= 4): run_esrgan's INTER_CUBIC chain on BGR frames
 * (core/merged_pipeline.py:262-266) */
int vd3d_resize_cubic(vd3d_ctx* ctx, const uint8_t* src, int h, int w, int ch, uint8_t* dst, int oh, int ow, int mem);
/* cv2.addWeighted(a, alpha, b, beta, 0) on n u8 values: blend_images (core/merged_pipeline.py:233-238) */
int vd3d_add_weighted(vd3d_ctx* ctx, const uint8_t* a, double alpha, const uint8_t* b, double beta, size_t n, uint8_t* dst,
                      int mem);
/* apply_sharpening (717-732) on u8 BGR [h,w,3] */
int vd3d_sharpen(vd3d_ctx* ctx, const uint8_t* src, int h, int w, double factor, uint8_t* dst, int mem);
/* heal_missing_pixels (431-459; the reference's "gradient-blend occlusion fill", defined but not called by
 * its render loop): f32 RGB planes [3,h,w] warped + original, optional edge mask [h,w] -> f32 [3,h,w] */
int vd3d_heal(vd3d_ctx* ctx, const float* warped, const float* original, const float* edge_mask_or_null, int h, int w,
              double heal_strength, float* out, int mem);
/* eye fit on one u8 BGR image [h,w,3] -> [target_h,target_w,3]: keep_aspect != 0 = pad_to_aspect_ratio (101-131, black
 * canvas), 0 = cv2.resize(..., INTER_AREA) as in the Half-SBS branch (1413-1414).  Shrinking only: identity, integer
 * factors, or cv2's general (fractional) area tables; enlarging returns VD3D_ERR_UNSUPPORTED */
int vd3d_fit_eye(vd3d_ctx* ctx, const uint8_t* src, int h, int w, int target_w, int target_h, int keep_aspect,
                 uint8_t* dst, int mem);
/* host-only test hook (no GPU needed): the cv2 area-resize tables vd3d_fit_eye / the frame path build for a
 * ssize -> dsize shrink; ofs/cnt [dsize], alpha [dsize*cap]; returns the largest tap count or a negative error */
int vd3d_area_table(int ssize, int dsize, int* ofs, int* cnt, float* alpha, int cap);
/* same for the enlarging case (cv2 emulates INTER_AREA with fixed-point bilinear weights): ofs [dsize], a01 [2*dsize] */
int vd3d_area_linear_table(int ssize, int dsize, int* ofs, int* a01);
/* format_3d_output / generate_anaglyph_3d (837-883) on two same-size u8 BGR eyes [h,w,3]:
 * SBS -> [h,2w,3]; anaglyph / interlaced -> [h,w,3] */
int vd3d_pack(vd3d_ctx* ctx, const uint8_t* left, const uint8_t* right, int h, int w, int fmt, uint8_t* dst, int mem);
/* apply_dof_cuda (769-834) + apply_color_grade (734-767) + tensor_to_frame on a u8 BGR eye;
 * depth01: f32 [dh,dw] resized bilinearly to [h,w] as at 1347-1350; max_sigma<=0 skips DOF */
int vd3d_dof_grade(vd3d_ctx* ctx, const uint8_t* eye_bgr, int h, int w, const float* depth01, int dh, int dw,
                   double focal, double max_sigma, double sat, double con, double bri, uint8_t* dst, int mem);

/* ---- depth forward (Depth-Anything-V2: DINOv2 ViT + DPT neck/head) ----------
 * Replaces model.forward inside transformers' depth-estimation pipeline as called by
 * hf_batch_safe_pipe (core/render_depth.py:1106-1119).  GEMMs / 3x3 convs run on wgmma
 * tensor cores (f16 operands, fp32 accumulation) fed by TMA. */
typedef struct {
  int32_t hidden, layers, heads; /* 384/12/6, 768/12/12, 1024/24/16 */
  int32_t taps[4];               /* out_indices of the backbone (1-based layer numbers) */
  int32_t neck[4];               /* neck_hidden_sizes */
  int32_t fusion;                /* fusion_hidden_size */
  int32_t image_h, image_w;      /* processed size, multiples of 14 (518 x 924 for 16:9) */
} vd3d_depth_config;
int vd3d_depth_create(const vd3d_depth_config* cfg, void* cuda_stream, vd3d_depth** out);
void vd3d_depth_destroy(vd3d_depth* e);
/* CUDA-event timing of the fc1 GEMM launches (k_umma_gemm<128,4>; M = tokens, N = 4*hidden, K = hidden) */
int vd3d_depth_profile(vd3d_depth* e, int enable);
int vd3d_depth_profile_collect(vd3d_depth* e, double* total_ms, int* count, double* gflop_per_launch);
/* tuning aid: after vd3d_depth_profile(e, 2), every launch class of an eager forward is bracketed by CUDA events; this
   returns "tag total_ms spans" lines (NUL-terminated, truncated to cap) and clears the record */
int vd3d_depth_profile_spans(vd3d_depth* e, char* out, size_t cap);
/* another instance on `cuda_stream` sharing e's weights (own activations); destroy it before e */
int vd3d_depth_clone(vd3d_depth* e, void* cuda_stream, vd3d_depth** out);
const char* vd3d_depth_last_error(vd3d_depth* e);
uint64_t vd3d_depth_launch_count(vd3d_depth* e);
void vd3d_depth_add_launches(vd3d_depth* e, uint64_t n); /* bookkeeping for CUDA-graph replays */
/* upload one prepared weight tensor (names / layouts: visiondepth3d_b200/depth_weights.py) */
int vd3d_depth_set_tensor(vd3d_depth* e, const char* name, const void* host_data, size_t bytes);
/* pixel_values f32 [3,image_h,image_w] -> predicted_depth f32 [image_h,image_w] */
int vd3d_depth_forward(vd3d_depth* e, const float* pixel_values, float* depth_out, int mem);
/* the whole depth stage of the reference for one frame: DPT image processor (antialiased
 * bicubic to image_h x image_w, /255, mean/std) -> forward -> post_process_depth_estimation
 * (bicubic back to h x w) -> convert_depth_to_grayscale min-max u8 (core/render_depth.py:
 * 1113-1119, 605-611).  _device: all pointers on the GPU, enqueued without synchronising
 * (this is what vd3d_render_clip uses for the in-memory depth -> stereo handoff). */
int vd3d_depth_infer(vd3d_depth* e, const uint8_t* frame_bgr, int h, int w, float* depth_f32, uint8_t* depth_u8,
                     int invert);
int vd3d_depth_infer_device(vd3d_depth* e, const uint8_t* frame_bgr_dev, int h, int w, uint8_t* depth_u8_dev,
                            float* depth_f32_dev_or_null, int invert);
/* The same for B (1..8) frames of one size with ONE batched forward: the token-wise GEMMs see the stacked token
 * matrix of all frames (the reference hands the whole list to the HF pipeline too, core/render_depth.py:1113-1119).
 * Arrays of B pointers; depth_f32 / depth_u8 (or single entries) may be NULL. */
int vd3d_depth_infer_batch(vd3d_depth* e, int B, const uint8_t* const* frames_bgr, int h, int w, float* const* depth_f32,
                           uint8_t* const* depth_u8, int invert);
int vd3d_depth_infer_batch_device(vd3d_depth* e, int B, const uint8_t* const* frames_bgr_dev, int h, int w,
                                  uint8_t* const* depth_u8_dev, float* const* depth_f32_dev, int invert);
/* ---- still images (process_image / process_images_in_folder, core/render_depth.py:1229-1477) ----------------------
 * Image.resize((ow, oh), Image.BICUBIC) of one u8 RGB image [h,w,3] -> [oh,ow,3], bit for bit with Pillow's 8-bit
 * resampling: width pass then height pass (a pass is skipped when its axis keeps its size), fixed-point weights with 22
 * fractional bits from tables built on the host once per (in, out) size pair and cached by the engine, integer sums.
 * Host memory synchronises; device memory is enqueued on the engine stream. */
int vd3d_depth_resize_pil(vd3d_depth* e, const uint8_t* src, int h, int w, uint8_t* dst, int oh, int ow, int mem);
/* host-only test hook (no GPU needed): the table of one axis, in_size -> out_size: bounds [2*out_size] = (first input,
 * tap count) per output index, kk [out_size*cap] fixed-point weights.  Returns the taps per output (ksize); with bounds or
 * kk NULL only that; VD3D_ERR_ARG when cap < ksize. */
int vd3d_pil_bicubic_table(int in_size, int out_size, int32_t* bounds, int32_t* kk, int cap);
/* B (1..8) u8 RGB images, each of its own size, through ONE batched forward.  sizes [B][4] = src_h, src_w, in_h, in_w:
 * the image's size and its input size (the inference size, or the source size again).  Every input size must map to the
 * engine's processed size (the DPT processor's keep-aspect multiple-of-14 size), else VD3D_ERR_ARG.  Per image: the
 * Pillow resize to the input size when it differs, the DPT processor into the image's slot of the batch; then the
 * forward on the stacked token matrix (as vd3d_depth_infer_batch); then per image bicubic back to the input size, min-max
 * u8 (255 - u8 when invert) and cv2 INTER_CUBIC to the source size when it differs -> depth_u8[b] [src_h,src_w].
 * depth_f32 (optional; the array or single entries may be NULL): the predicted depth at the input size [in_h,in_w].
 * Host memory: one upload per image and one download per output, synchronises; device memory: enqueued on the engine
 * stream. */
int vd3d_depth_infer_images(vd3d_depth* e, int B, const uint8_t* const* images_rgb, const int32_t* sizes,
                            uint8_t* const* depth_u8, float* const* depth_f32, int invert, int mem);
/* frames per depth forward inside vd3d_render_clip_depth (1..8, default 4; env VD3D_DEPTH_BATCH) */
int vd3d_set_depth_batch(vd3d_ctx* ctx, int frames);
int vd3d_get_depth_batch(vd3d_ctx* ctx);
/* ---- Real-ESRGAN upscale stage (SURVEY 8(f) rank 3; core/merged_pipeline.py:221-267) --------------------------------
 * The reference runs an ONNX export of xinntao/Real-ESRGAN's SRVGGNetCompact (realesr-general-x4v3: 32 body convs;
 * realesr-animevideov3: 16) through ONNXRuntime.  vd3d_sr_create returns an engine container (weights by name through
 * vd3d_depth_set_tensor: "sr.c{i}.w" f16 [Cout, 9*64], "sr.c{i}.b" f32, "sr.a{i}" f32 PReLU slopes; destroy with
 * vd3d_depth_destroy).  vd3d_sr_forward: BGR u8 [h,w,3] -> BGR u8 [4h,4w,3] = preprocess_esr -> network (wgmma
 * implicit-GEMM convs, f16 activations, fp32 accumulate, fp32 last layer) -> PixelShuffle + input -> postprocess_esr. */
int vd3d_sr_create(void* cuda_stream, vd3d_depth** out);
int vd3d_sr_forward(vd3d_depth* e, const uint8_t* frame_bgr, int h, int w, int num_conv, uint8_t* out_bgr, int mem);
/* Make an SR engine an RRDBNet (the generator of ESRGAN / Real-ESRGAN RealESRGAN_x4plus / BSRGAN: num_feat 64, growth
 * 32, nb RRDB blocks of three dense blocks, net_scale 4 = two nearest-x2 up-convs or 2 = one), or SRVGGNetCompact
 * again with nb = 0.  Weights (vd3d_depth_set_tensor, ".w" f16 [Cout, 9 * Cin_padded] tap-major, ".b" f32 [Cout]):
 * "rr.first" (Cin 3 padded to 64), "rr.{i}.{j}.{k}" for block i, dense block j = 0..2 and conv k = 1..5 (input
 * channels laid out as 64 + 64 per 32-channel growth slice, zero columns in the padding: Cin_padded = 64 k), "rr.body",
 * "rr.up1" / "rr.up2" (nearest x2 + conv as four phase convs: [4 * 64, 9 * 64], rows (py * 2 + px) * 64 + co),
 * "rr.hr", "rr.last" ([32, 9 * 64], rows 3..31 zero).  vd3d_sr_forward then returns BGR u8 [net_scale h,
 * net_scale w, 3] and vd3d_sr_upscale runs the reference's resize chain on it (scale stays the model-name quirk);
 * num_conv is ignored.  VD3D_ERR_ARG for nb outside 0..64 or another net_scale. */
int vd3d_sr_set_rrdb(vd3d_depth* e, int nb, int net_scale);
/* arguments of run_esrgan (core/merged_pipeline.py:240-267) without tiling.  input_res_pct and blend_alpha are Python
 * floats there (double here, rounded where the reference's cv2 calls round them). */
typedef struct {
  double input_res_pct;       /* < 100 INTER_AREA, > 100 INTER_CUBIC, 100 none (247-249) */
  int32_t scale;              /* 4, or 2 when the reference's model_name contains "x2" (262) */
  int32_t target_w, target_h; /* 0, 0 = no target_size (265-266) */
  double blend_alpha;         /* < 0: mode "OFF" (no addWeighted); else the alpha of blend_images (233-238) */
} vd3d_upscale_params;
/* run_esrgan's whole untiled chain for n frames BGR u8 [h,w,3] -> outs [target or h,w,3], every step on the device:
 * input resize (the INTER_AREA kernels of vd3d_fit_eye / INTER_CUBIC), the network of vd3d_sr_forward, the x4 image
 * resampled with INTER_CUBIC straight from the last conv to the original size (to 2x the network input for scale 2,
 * then INTER_CUBIC to the original size) without materialising it, INTER_CUBIC to the target, addWeighted.  Same-size
 * resizes are skipped (cv2 copies).  A blend of two different sizes is VD3D_ERR_ARG (cv2.addWeighted raises).  sr must
 * have been created on vd3d_stream(ctx).  Host memory: one upload and one download per frame, overlapping the compute
 * of the neighbouring frames (page-locked buffers for full overlap); device memory: no PCIe traffic.  Synchronises. */
int vd3d_sr_upscale(vd3d_ctx* ctx, vd3d_depth* sr, int n, const uint8_t* const* frames, int h, int w, int num_conv,
                    const vd3d_upscale_params* p, uint8_t* const* outs, int mem);
/* copy an internal activation buffer to the host (parity triage: "x", "tap0.0".., "f0".., "fused3") */
int vd3d_depth_get_buffer(vd3d_depth* e, const char* name, void* host_out, size_t bytes);
/* unit-test hooks for the tensor-core kernels */
int vd3d_gemm_f16(vd3d_depth* e, const void* A_f16, const void* B_f16, int M, int N, int K, float* C_host, int bn);
/* tuning hook: average launch time (ms) of one M x N x K GEMM on device-resident operands, on the 128 x 128 tile
   kernel with an operand ring of 4 (variant 0, the default), 3 (variant 1) or 2 (variant 2) stages; other variants
   return VD3D_ERR_ARG.  dbg (low 3 bits): 0 normal, 2 no TMA loads (MMA rate), 3 prologue + teardown only, 4 no
   epilogue (the epilogue warpgroup only releases the staging tile), other values VD3D_ERR_ARG; bit 3: poll barriers with test_wait.  act: 0 none, 1 GELU; 0x100 selects the
   residual (proj / fc2) epilogue */
int vd3d_gemm_bench(vd3d_depth* e, int M, int N, int K, int variant, int dbg, int act, int iters, float* ms_out);
int vd3d_conv_f16(vd3d_depth* e, const void* in_nhwc_f16, int H, int W, int cin, const void* w_f16, int cout,
                  int k3, const float* bias, int relu, float* out_host);

#ifdef __cplusplus
}
#endif
#endif /* VD3D_H */
