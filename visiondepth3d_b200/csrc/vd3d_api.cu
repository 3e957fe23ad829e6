// vd3d_api.cu -- host side of libvd3d.so: context, workspaces, the per-frame kernel
// sequence of render_sbs_3d / pixel_shift_cuda (core/render_3d.py:561-712,1227-1419),
// and the C ABI declared in include/vd3d.h.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "dibr_launch.h"
#include "letterbox_launch.h"
#include "sr_engine.h"
#include "tiled_launch.h"

using namespace vd3d;

namespace {

std::string g_create_error;

struct Buf {
  void* p = nullptr;
  size_t cap = 0;
};

constexpr int kSlots = 16;   // staging slots: two depth batches of up to kMaxDepthBatch frames in flight
constexpr int kClones = 2;   // depth engine instances (own activation buffers / stream), alternating per batch
constexpr int kMaxDepthBatch = 8;
constexpr int kSrSlots = 3;  // vd3d_sr_upscale: upload of frame i+1 | compute of frame i | download of frame i-1
constexpr int kJobs = 5;  // pct, subj(norm), quantile(d0), subj(d0), subj(shaped)
constexpr size_t kJobWords = 4096 + 4 * 4096 + 4 * 64 + 64 + 64;  // + count (padded)
constexpr size_t kBarWords = 64;

}  // namespace

struct vd3d_ctx {
  int device = 0;
  cudaStream_t stream = nullptr, s_h2d = nullptr, s_d2h = nullptr;
  std::string err;
  uint64_t launches = 0;
  int use_graphs = 1;
  int stats_only = 0;  // advance temporal state only (exact multi-GPU sharding: SURVEY 8(e))
  int exact = 0;       // 1: one-kernel-per-op path with correctly rounded transcendentals (dibr_kernels.cu);
                       // 0: persistent stats kernel + fused render kernel (dibr_fast.cu)
  int stats_blocks = 0;
  // bumped whenever a device resource that captured graphs bake in moves or changes content (ensure() reallocations,
  // linspace axes, INTER_AREA tables, DOF kernel bank); run_frame_slot drops stale graphs
  uint64_t res_epoch = 0, fg_epoch = 0;
  int prof_depth_frames = 0;  // frames covered by the stage-2 (depth) samples since the last collect
  uint64_t dclone_wver = 0;
  unsigned* bar = nullptr;  // grid barrier counter of k_stats (inside jobwords: zeroed by begin_frame)
  // auto_crop_black_bars: (top, bottom) written by the ingest of each staging slot [kSlots][2], their copies for the
  // frames of the last clip call (pinned, crops_n frames), and the two words of vd3d_detect_black_bars
  int32_t* crops_dev = nullptr;
  int32_t* crops_host = nullptr;
  int crops_cap = 0, crops_n = 0;
  uint32_t* detect_words = nullptr;
  // letterbox tracker statistics, Canny and depth re-pad (letterbox.cu): inputs, planes, per-row/per-frame records
  // and the cut nodes of the frame-wide pairwise luma sum (cached per pixel count)
  Buf lb_in, lb_prev, lb_gray, lb_mag, lb_label, lb_flag, lb_rec, lb_nodes, lb_node_sum, lb_out, lb_hist;
  int64_t lb_nodes_npix = -1;
  int lb_nodes_n = 0;
  // tiled depth (tiled_depth.cu): frames, tile crops, per-tile predictions and weights, tile jobs, blended depth, u8
  // planes before the output resize, selection scratch, extremes, outputs staged for host memory
  Buf td_frames, td_crops, td_preds, td_wgt, td_jobs, td_depth, td_u8, td_sel, td_mm, td_stats, td_out, td_outf;

  DevState* st = nullptr;
  FrameScalars* fs = nullptr;
  vd3d_frame_info* info_pinned = nullptr;
  FrameScalars* fs_pinned = nullptr;
  DevState* st_pinned = nullptr;
  uint32_t* jobwords = nullptr;  // kJobs * kJobWords, zeroed every frame
  SelTarget* tgs = nullptr;      // kJobs * 4
  JobMem jm[kJobs];

  // linspace tables
  Buf xs, ys;
  int xs_n = 0, ys_n = 0;
  // planes
  Buf tdf, dn0, dn1, rgb_s, frameB, d, shift, e2, eyeL, eyeR, eyeL2, eyeR2;
  Buf in_frame[kSlots], in_depth[kSlots], out_dev[kSlots], in_rgbf, in_depthf;
  Buf dof_kern;
  // host-memory staging of vd3d_sr_upscale (frame in, result out), apart from the frame path's slots
  Buf sr_in[kSrSlots], sr_out[kSrSlots];
  // cv2 ResizeArea_ tables of the current non-integer eye fit (device) + the sizes they were built for
  // ([0]: the frame path, whose CUDA graphs bake the pointers in; [1]: the stage entry points vd3d_fit_eye ...)
  Buf area_tab[2];
  int at_key[2][4] = {};
  int at_t[2] = {0, 0};
  int tdf_w = 0, tdf_h = 0;
  int frame_parity = 0;
  cudaEvent_t ev_h2d[kSlots] = {}, ev_done[kSlots] = {}, ev_d2h[kSlots] = {};
  // optional per-stage device timing (bench.py roofline): event pairs on ctx->stream
  int prof = 0;
  std::vector<cudaEvent_t> prof_ev[4];  // stage -> [start, stop, start, stop, ...]
  std::vector<cudaEvent_t> prof_pool;
  // CUDA graphs of the per-frame kernel sequence, keyed by (staging slot, depth ping-pong parity)
  struct FrameGraph {
    cudaGraphExec_t exec = nullptr;
    uint64_t n_ctx = 0;
  } fg[kSlots][2];
  vd3d_render_params fg_rp;
  int fg_h = 0, fg_w = 0, fg_dch = 0, fg_warm = 0;
  // depth stage of the depth+stereo clip: two engine clones (shared weights) on two streams so the
  // depth forwards of consecutive frames overlap each other and the DIBR kernels of the previous frame
  vd3d_depth* dclone[kClones] = {};
  vd3d_depth* dclone_parent = nullptr;
  cudaStream_t s_depth[kClones] = {};
  cudaEvent_t ev_depth[kClones] = {};
  struct DepthGraph {  // one graph per (engine instance, frames in the batch)
    cudaGraphExec_t exec = nullptr;
    uint64_t n = 0;
  } dg[kClones][kMaxDepthBatch + 1];
  int dg_warm = 0, dg_h = 0, dg_w = 0;
  int depth_batch = 4;  // frames per depth forward in vd3d_render_clip_depth (env VD3D_DEPTH_BATCH, 1..8)
  // dof kernel cache
  double dof_sigma_cached = -1.0;
  int dof_nlevels = 0, dof_ksize[8] = {0}, dof_koff[8] = {0}, dof_halo = 0;
};

extern "C" {
uint64_t vd3d_depth_weights_version(vd3d_depth* e);
static void drop_graphs(vd3d_ctx* ctx);
static void drop_depth_graphs(vd3d_ctx* ctx);
int vd3d_depth_clone(vd3d_depth* e, void* cuda_stream, vd3d_depth** out);
void vd3d_depth_destroy(vd3d_depth* e);
}

namespace {

#define CK(call)                                                                    \
  do {                                                                              \
    cudaError_t _e = (call);                                                        \
    if (_e != cudaSuccess) {                                                        \
      char _b[512];                                                                 \
      snprintf(_b, sizeof _b, "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
      ctx->err = _b;                                                                \
      return VD3D_ERR_CUDA;                                                         \
    }                                                                               \
  } while (0)

cudaEvent_t prof_event(vd3d_ctx* ctx) {
  cudaEvent_t e;
  if (!ctx->prof_pool.empty()) {
    e = ctx->prof_pool.back();
    ctx->prof_pool.pop_back();
  } else {
    cudaEventCreate(&e);
  }
  return e;
}
struct ProfScope {  // records start now, stop at destruction
  vd3d_ctx* c;
  int stage;
  ProfScope(vd3d_ctx* ctx, int st) : c(ctx), stage(st) {
    if (c->prof) {
      cudaEvent_t e = prof_event(c);
      cudaEventRecord(e, c->stream);
      c->prof_ev[stage].push_back(e);
    }
  }
  ~ProfScope() {
    if (c->prof) {
      cudaEvent_t e = prof_event(c);
      cudaEventRecord(e, c->stream);
      c->prof_ev[stage].push_back(e);
    }
  }
};

int fail(vd3d_ctx* ctx, int code, const char* msg) {
  if (ctx) ctx->err = msg;
  return code;
}

int ensure(vd3d_ctx* ctx, Buf& b, size_t bytes) {
  if (b.cap >= bytes) return VD3D_OK;
  if (b.p) {
    CK(cudaDeviceSynchronize());  // frames still in flight (other streams, graph replays) may read the old block
    CK(cudaFree(b.p));
  }
  b.p = nullptr;
  b.cap = 0;
  ctx->res_epoch++;
  CK(cudaMalloc(&b.p, bytes));
  b.cap = bytes;
  return VD3D_OK;
}

// torch.linspace(-1, 1, n) fp32: step=(end-start)/(n-1); i<n/2: fma(step,i,start) else fma(-step,n-1-i,end)
void linspace32(float start, float end, int n, std::vector<float>& out) {
  out.resize(n);
  if (n == 1) {
    out[0] = start;
    return;
  }
  float step = (end - start) / (float)(n - 1);
  for (int i = 0; i < n; ++i)
    out[i] = (i < n / 2) ? fmaf(step, (float)i, start) : fmaf(-step, (float)(n - 1 - i), end);
}

int ensure_axes(vd3d_ctx* ctx, int W, int H) {
  std::vector<float> v;
  if (ctx->xs_n != W || ctx->ys_n != H) CK(cudaDeviceSynchronize());  // queued frames may still read the old axes
  if (ctx->xs_n != W) {
    int r = ensure(ctx, ctx->xs, sizeof(float) * W);
    if (r) return r;
    linspace32(-1.f, 1.f, W, v);
    CK(cudaMemcpyAsync(ctx->xs.p, v.data(), sizeof(float) * W, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->xs_n = W;
    ctx->res_epoch++;
  }
  if (ctx->ys_n != H) {
    int r = ensure(ctx, ctx->ys, sizeof(float) * H);
    if (r) return r;
    linspace32(-1.f, 1.f, H, v);
    CK(cudaMemcpyAsync(ctx->ys.p, v.data(), sizeof(float) * H, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->ys_n = H;
    ctx->res_epoch++;
  }
  return VD3D_OK;
}

// torch.quantile rank arithmetic: rank = fp32(q) * (n-1) in fp32
void quantile_rank(double q, long long n, uint32_t& lo, uint32_t& hi, float& w) {
  float rank = (float)q * (float)(n - 1);
  float fl = floorf(rank), ce = ceilf(rank);
  lo = (uint32_t)fl;
  hi = (uint32_t)ce;
  w = rank - fl;
}

SelJob make_job(const JobMem& m, const float* data, int W, int x0, int x1, int y0, int y1, int masked, int nt,
                int rank_from_count, bool hist64) {
  SelJob j;
  j.data = data;
  j.W = W;
  j.x0 = x0;
  j.x1 = x1;
  j.y0 = y0;
  j.y1 = y1;
  j.masked = masked;
  j.ntargets = nt;
  j.rank_from_count = rank_from_count;
  j.hist1 = m.hist1;
  j.hist2 = m.hist2;
  j.hist3 = m.hist3;
  j.hist64 = hist64 ? m.hist64 : nullptr;
  j.tg = m.tg;
  j.count = m.count;
  return j;
}

int sel_blocks(int rows) {
  int b = 132 * 4;  // four CTAs per SM of an H100
  return rows < b ? rows : b;
}

// ---------------------------------------------------------------------------
// pixel_shift core: from a depth plane [sh,sw] (already normalised) and an RGB source
// to the two u8 eyes.  Shared by vd3d_pixel_shift and vd3d_render_frame.
// ---------------------------------------------------------------------------
struct CoreIn {
  const float* depth;  // f32 [sh, sw]
  int sh, sw;
  const uint8_t* src_u8;  // identity path
  int src_pitch, cx0, cy0;
  const float* src_f32;  // RGB planes [3,H,W]
  int W, H;
  vd3d_shift_params p;
  int grade;
  float sat, con, bri;
  uint8_t* left;
  uint8_t* right;
};

// the feathering box sizes the compose kernels support
int check_blur_ksize(vd3d_ctx* ctx, int feather, int k) {
  if (feather && (k < 1 || k > 63)) return fail(ctx, VD3D_ERR_UNSUPPORTED, "blur_ksize must be in [1,63]");
  return VD3D_OK;
}

// compose inputs of a core whose shift map is in ctx->shift (e2: left to the caller)
ComposeArgs compose_args(vd3d_ctx* ctx, const CoreIn& in) {
  ComposeArgs ca;
  memset(&ca, 0, sizeof ca);
  ca.src_u8 = in.src_u8;
  ca.src_pitch = in.src_pitch;
  ca.cx0 = in.cx0;
  ca.cy0 = in.cy0;
  ca.src_f32 = in.src_f32;
  ca.shift = (const float*)ctx->shift.p;
  ca.xs = (const float*)ctx->xs.p;
  ca.ys = (const float*)ctx->ys.p;
  ca.H = in.H;
  ca.W = in.W;
  ca.k = in.p.blur_ksize;
  ca.feather = in.p.enable_feathering ? 1 : 0;
  ca.grade = in.grade;
  ca.sat = in.sat;
  ca.con = in.con;
  ca.bri = in.bri;
  ca.left = in.left;
  ca.right = in.right;
  return ca;
}

// generic tail of both cores, any box size: [k_warp_edges ->] k_compose into in.left / in.right
int compose_generic(vd3d_ctx* ctx, const CoreIn& in) {
  cudaStream_t s = ctx->stream;
  ComposeArgs ca = compose_args(ctx, in);
  if (ca.feather) {
    int r;
    if ((r = ensure(ctx, ctx->e2, sizeof(float2) * (size_t)ca.W * ca.H))) return r;
    launch_warp_edges((const float*)ctx->d.p, ca.shift, (float2*)ctx->e2.p, ca.H, ca.W, ca.xs, ca.ys,
                      (float)in.p.feather_strength, s);
    ctx->launches += 1;
  }
  ca.e2 = (const float2*)ctx->e2.p;
  {
    ProfScope ps(ctx, 1);
    launch_compose(ca, s);
  }
  ctx->launches += 1;
  CK(cudaGetLastError());
  return VD3D_OK;
}

int run_core(vd3d_ctx* ctx, const CoreIn& in) {
  cudaStream_t s = ctx->stream;
  const int W = in.W, H = in.H;
  int r;
  if ((r = ensure_axes(ctx, W, H))) return r;
  if ((r = ensure(ctx, ctx->d, sizeof(float) * (size_t)W * H))) return r;
  if ((r = ensure(ctx, ctx->shift, sizeof(float) * (size_t)W * H))) return r;
  const float* xs = (const float*)ctx->xs.p;
  const float* ys = (const float*)ctx->ys.p;
  float* d = (float*)ctx->d.p;
  float* shift = (float*)ctx->shift.p;

  launch_d0(in.depth, in.sh, in.sw, d, H, W, xs, ys, 0.08f, s);
  ctx->launches += 1;
  // quantiles (depth_stretch_lo/hi) over the full map + subject estimate on the centre crop
  uint32_t l0, l1, h0, h1;
  float wlo, whi;
  quantile_rank(in.p.depth_stretch_lo, (long long)W * H, l0, l1, wlo);
  quantile_rank(in.p.depth_stretch_hi, (long long)W * H, h0, h1, whi);
  launch_set_ranks(ctx->jm[2].tg, l0, l1, h0, h1, s);
  ctx->launches += 1;
  SelJob qj = make_job(ctx->jm[2], d, W, 0, W, 0, H, 0, 4, 0, false);
  SelJob s0 = make_job(ctx->jm[3], d, W, W / 5, W * 4 / 5, H / 5, H * 4 / 5, 1, 1, 1, true);
  launch_select(qj, &s0, sel_blocks(H), s);
  ctx->launches += kSelectLaunches;
  launch_fin_d0(qj, s0, wlo, whi, ctx->fs, s);
  ctx->launches += 1;
  launch_shape(d, W * H, ctx->fs, (float)in.p.depth_pop_mid, (float)in.p.depth_pop_gamma, s);
  ctx->launches += 1;
  SelJob s1 = make_job(ctx->jm[4], d, W, W / 5, W * 4 / 5, H / 5, H * 4 / 5, 1, 1, 1, true);
  launch_select(s1, nullptr, sel_blocks(H * 4 / 5 - H / 5), s);
  ctx->launches += kSelectLaunches;
  ShiftArgs sa;
  sa.p = in.p;
  sa.W = W;
  sa.H = H;
  launch_fin_shape(s1, sa, ctx->st, ctx->fs, s);
  ctx->launches += 1;
  if (ctx->stats_only) {  // every temporal state update of the frame has happened by now
    CK(cudaGetLastError());
    return VD3D_OK;
  }
  launch_shift(d, shift, H, W, ctx->fs, in.p.enable_edge_masking ? 1 : 0, (float)in.p.feather_strength, s);
  ctx->launches += 1;
  if ((r = check_blur_ksize(ctx, in.p.enable_feathering, in.p.blur_ksize))) return r;
  return compose_generic(ctx, in);
}

// ---------------------------------------------------------------------------
// fast path (dibr_fast.cu): k_stats -> k_shift<fast> -> k_render
// ---------------------------------------------------------------------------
struct FastLoop {  // loop-level inputs of k_stats (null for the pixel_shift_cuda entry)
  const IngestArgs* ia;
  float4* rgbx_s;
  float4* rgbx;
  float* dn;
  const float* dn_prev;
  const LoopArgs* la;
};
struct FastPost {  // fused bars + sharpen + fit + pack (fuse == 0: write the eyes)
  int fuse = 0;
  int sharpen = 0;
  float kc = 0.f, ke = 0.f;
  uint8_t* out = nullptr;
  int out_w = 0, per_eye_w = 0;
  const float4* src_rgbx = nullptr;
};

// Box sizes k_render does not support (render_supports) take run_core instead.
int run_core_fast(vd3d_ctx* ctx, const CoreIn& in, const FastLoop* lp, const FastPost& post) {
  cudaStream_t s = ctx->stream;
  const int W = in.W, H = in.H;
  int r;
  if ((r = ensure_axes(ctx, W, H))) return r;
  if ((r = ensure(ctx, ctx->d, sizeof(float) * (size_t)W * H))) return r;
  if ((r = ensure(ctx, ctx->shift, sizeof(float) * (size_t)W * H))) return r;
  const float* xs = (const float*)ctx->xs.p;
  const float* ys = (const float*)ctx->ys.p;
  float* d = (float*)ctx->d.p;
  float* shift = (float*)ctx->shift.p;

  StatsArgs sa;
  memset(&sa, 0, sizeof sa);
  sa.loop = lp ? 1 : 0;
  if (lp) {
    sa.ia = *lp->ia;
    sa.rgbx_s = lp->rgbx_s;
    sa.rgbx = lp->rgbx;
    sa.dn = lp->dn;
    sa.dn_prev = lp->dn_prev;
    sa.la = *lp->la;
    quantile_rank(0.02, (long long)lp->ia->tw * lp->ia->th, sa.pct_rank[0], sa.pct_rank[1], sa.pct_wlo);
    quantile_rank(0.98, (long long)lp->ia->tw * lp->ia->th, sa.pct_rank[2], sa.pct_rank[3], sa.pct_whi);
  }
  sa.core_depth = in.depth;
  sa.sh = in.sh;
  sa.sw = in.sw;
  sa.d = d;
  sa.H = H;
  sa.W = W;
  sa.xs = xs;
  sa.ys = ys;
  sa.sa.p = in.p;
  sa.sa.W = W;
  sa.sa.H = H;
  quantile_rank(in.p.depth_stretch_lo, (long long)W * H, sa.q_rank[0], sa.q_rank[1], sa.q_wlo);
  quantile_rank(in.p.depth_stretch_hi, (long long)W * H, sa.q_rank[2], sa.q_rank[3], sa.q_whi);
  for (int j = 0; j < kJobs; ++j) sa.jm[j] = ctx->jm[j];
  sa.st = ctx->st;
  sa.fs = ctx->fs;
  sa.bar = ctx->bar;
  CK(launch_stats(sa, ctx->stats_blocks, s));
  ctx->launches += 1;
  if (ctx->stats_only) return VD3D_OK;
  launch_shift_fast(d, shift, H, W, ctx->fs, in.p.enable_edge_masking ? 1 : 0, (float)in.p.feather_strength, s);
  ctx->launches += 1;

  RenderArgs ra;
  memset(&ra, 0, sizeof ra);
  ra.c = compose_args(ctx, in);
  ra.src_rgbx = post.src_rgbx;
  ra.d = d;
  ra.feather_strength = (float)in.p.feather_strength;
  ra.fuse = post.fuse;
  ra.fs = ctx->fs;
  ra.sharpen = post.sharpen;
  ra.kc = post.kc;
  ra.ke = post.ke;
  ra.out = post.out;
  ra.out_w = post.out_w;
  ra.per_eye_w = post.per_eye_w;
  {
    ProfScope ps(ctx, 1);
    CK(launch_render(ra, s));
  }
  ctx->launches += 1;
  CK(cudaGetLastError());
  return VD3D_OK;
}

int begin_frame(vd3d_ctx* ctx) {
  CK(cudaMemsetAsync(ctx->jobwords, 0, sizeof(uint32_t) * (kJobs * kJobWords + kBarWords), ctx->stream));
  CK(cudaMemsetAsync(ctx->fs, 0, sizeof(FrameScalars), ctx->stream));
  ctx->launches += 2;
  return VD3D_OK;
}

// crop_slot >= 0: the frame was auto-cropped, its (top, bottom) sits in crops_dev[crop_slot]
int fetch_info(vd3d_ctx* ctx, vd3d_frame_info* info, int crop_slot = -1) {
  int32_t tb[2] = {0, 0};
  CK(cudaMemcpyAsync(ctx->fs_pinned, ctx->fs, sizeof(FrameScalars), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(ctx->st_pinned, ctx->st, sizeof(DevState), cudaMemcpyDeviceToHost, ctx->stream));
  if (crop_slot >= 0)
    CK(cudaMemcpyAsync(tb, ctx->crops_dev + 2 * crop_slot, sizeof tb, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  info->crop_top = tb[0];
  info->crop_bottom = tb[1];
  const FrameScalars& f = *ctx->fs_pinned;
  const DevState& t = *ctx->st_pinned;
  info->pct_lo = t.pct_lo;
  info->pct_hi = t.pct_hi;
  info->subj_raw = f.subj_raw;
  info->stretch_lo = f.st_lo;
  info->stretch_hi = f.st_hi;
  info->subj_shaped = f.subj;
  info->subj_norm = f.subj_norm;
  info->dyn_scale = f.dyn;
  info->fg = f.fg;
  info->mg = f.mg;
  info->bg = f.bg;
  info->zero_parallax_offset = f.zpo;
  info->focal_depth = f.focal;
  info->motion_metric = f.motion;
  info->stable_zero = f.stable_zero;
  info->bar_width = f.bar_width;
  info->bar_side = f.bar_side;
  return VD3D_OK;
}

// torchvision _get_gaussian_kernel2d for the DOF levels (core/render_3d.py:798-806)
int ensure_dof_kernels(vd3d_ctx* ctx, double max_sigma, int num_levels) {
  if (ctx->dof_sigma_cached == max_sigma && ctx->dof_nlevels == num_levels) return VD3D_OK;
  std::vector<float> sig;
  linspace32(0.f, (float)max_sigma, num_levels, sig);
  std::vector<float> all;
  int halo = 0;
  for (int l = 0; l < num_levels; ++l) {
    float s = sig[l];
    int ks = 1;
    if ((double)s != 0.0) ks = (int)(2 * ceil(2 * (double)s) + 1);
    if (ks > 17) return fail(ctx, VD3D_ERR_UNSUPPORTED, "dof_strength too large (Gaussian ksize > 17)");
    ctx->dof_ksize[l] = ks;
    ctx->dof_koff[l] = (int)all.size();
    if (ks > 1) {
      std::vector<float> x, pdf(ks);
      float half = (float)((ks - 1) * 0.5);
      linspace32(-half, half, ks, x);
      float sum = 0.f;
      for (int i = 0; i < ks; ++i) {
        float q = x[i] / (float)(double)s;
        float e = -0.5f * (q * q);
        pdf[i] = (float)exp((double)e);
      }
      for (int i = 0; i < ks; ++i) sum += pdf[i];
      for (int i = 0; i < ks; ++i) pdf[i] = pdf[i] / sum;
      for (int y = 0; y < ks; ++y)
        for (int xx = 0; xx < ks; ++xx) all.push_back(pdf[y] * pdf[xx]);
      if (ks / 2 > halo) halo = ks / 2;
    }
  }
  if (all.empty()) all.push_back(1.f);
  CK(cudaDeviceSynchronize());
  int r = ensure(ctx, ctx->dof_kern, sizeof(float) * all.size());
  if (r) return r;
  CK(cudaMemcpyAsync(ctx->dof_kern.p, all.data(), sizeof(float) * all.size(), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->res_epoch++;
  ctx->dof_sigma_cached = max_sigma;
  ctx->dof_nlevels = num_levels;
  ctx->dof_halo = halo;
  return VD3D_OK;
}

void sharpen_coeffs(double factor, float& kc, float& ke) {
  // apply_sharpening: fp32 kernel [[0,-1,0],[-1,5+f,-1],[0,-1,0]] / sum (core/render_3d.py:719-728)
  float c = (float)(5.0 + factor);
  float ks = c - 4.0f;
  kc = c;
  ke = -1.0f;
  if (ks != 0.f) {
    kc = c / ks;
    ke = -1.0f / ks;
  }
}

struct FitPlan {
  int fit_x0, fit_y0, fit_w, fit_h, sx, sy;
  // non-integer INTER_AREA shrink: device tables (null otherwise), see PostArgs
  const int *xofs = nullptr, *xcnt = nullptr, *yofs = nullptr, *ycnt = nullptr;
  const float *xal = nullptr, *yal = nullptr;
  int area_t = 0;
  int lin = 0;  // enlarged axis: cv2's fixed-point bilinear emulation of INTER_AREA (see plan_fit)
};

// cv2's computeResizeAreaTab (imgproc/src/resize.cpp, opencv 4.13 as installed with the reference): geometry in double,
// one fp32 weight per (destination, source) pair; the sources of one destination index are consecutive.
void area_axis_tab(int ssize, int dsize, std::vector<int>& ofs, std::vector<int>& cnt, std::vector<std::vector<float>>& al) {
  const double scale = 1.0 / ((double)dsize / (double)ssize);
  ofs.assign(dsize, 0);
  cnt.assign(dsize, 0);
  al.assign(dsize, {});
  for (int dx = 0; dx < dsize; ++dx) {
    const double fsx1 = dx * scale, fsx2 = fsx1 + scale;
    const double cell = fmin(scale, (double)ssize - fsx1);
    int sx1 = (int)ceil(fsx1), sx2 = (int)floor(fsx2);
    if (sx2 > ssize - 1) sx2 = ssize - 1;
    if (sx1 > sx2) sx1 = sx2;
    int first = -1;
    auto push = [&](int si, float a) {
      if (first < 0) first = si;
      al[dx].push_back(a);
    };
    if (sx1 - fsx1 > 1e-3) push(sx1 - 1, (float)((sx1 - fsx1) / cell));
    for (int sx = sx1; sx < sx2; ++sx) push(sx, (float)(1.0 / cell));
    if (fsx2 - sx2 > 1e-3) push(sx2, (float)(fmin(fmin(fsx2 - sx2, 1.0), cell) / cell));
    ofs[dx] = first < 0 ? 0 : first;
    cnt[dx] = (int)al[dx].size();
  }
}

// cv2 resize(): the "area_mode" coefficients of the bilinear scheme INTER_AREA falls back to when an axis grows
// (generic path of imgproc/src/resize.cpp): source index + two weights, saturate_cast<short>(c * 2048)
void area_linear_tab(int ssize, int dsize, std::vector<int>& ofs, std::vector<int>& a01) {
  const double inv = (double)dsize / (double)ssize, scale = 1.0 / inv;
  ofs.assign(dsize, 0);
  a01.assign((size_t)2 * dsize, 0);
  for (int dx = 0; dx < dsize; ++dx) {
    int sx = (int)floor(dx * scale);
    float fx = (float)((dx + 1) - (sx + 1) * inv);
    fx = fx <= 0 ? 0.f : fx - floorf(fx);
    if (sx < 0) {
      fx = 0.f;
      sx = 0;
    }
    if (sx >= ssize - 1) {
      fx = 0.f;
      sx = ssize - 1;
    }
    const float c0 = 1.f - fx;
    ofs[dx] = sx;
    a01[2 * dx] = (int)lrintf(c0 * 2048.f);
    a01[2 * dx + 1] = (int)lrintf(fx * 2048.f);
  }
}

// build (or reuse) the device tables for a W x H -> nw x nh non-integer INTER_AREA shrink
int ensure_area_tabs(vd3d_ctx* ctx, int which, int W, int H, int nw, int nh, FitPlan& f, bool lin = false) {
  Buf& tab = ctx->area_tab[which];
  int* key = ctx->at_key[which];
  const bool have = key[0] == W && key[1] == H && key[2] == nw && key[3] == nh && tab.p;
  if (!have) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(ctx->stream, &cs);
    if (cs != cudaStreamCaptureStatusNone) return fail(ctx, VD3D_ERR_STATE, "INTER_AREA tables missing during capture");
    std::vector<int> xo, xc, yo, yc;
    std::vector<std::vector<float>> xa, ya;
    if (lin) {
      std::vector<int> ax, ay;
      area_linear_tab(W, nw, xo, ax);
      area_linear_tab(H, nh, yo, ay);
      xc.assign(nw, 2);
      yc.assign(nh, 2);
      xa.resize(nw);
      ya.resize(nh);
      for (int i = 0; i < nw; ++i) xa[i] = {(float)ax[2 * i], (float)ax[2 * i + 1]};
      for (int i = 0; i < nh; ++i) ya[i] = {(float)ay[2 * i], (float)ay[2 * i + 1]};
    } else {
      area_axis_tab(W, nw, xo, xc, xa);
      area_axis_tab(H, nh, yo, yc, ya);
    }
    int T = lin ? 2 : 1;
    for (int c : xc) T = c > T ? c : T;
    for (int c : yc) T = c > T ? c : T;
    if (T > 64) return fail(ctx, VD3D_ERR_UNSUPPORTED, "INTER_AREA shrink factor too large");
    const size_t nint = (size_t)2 * nw + (size_t)2 * nh, nflt = ((size_t)nw + nh) * T;
    std::vector<unsigned char> host(nint * 4 + nflt * 4);
    int* ip = (int*)host.data();
    float* fp = (float*)(host.data() + nint * 4);
    memcpy(ip, xo.data(), (size_t)nw * 4);
    memcpy(ip + nw, xc.data(), (size_t)nw * 4);
    memcpy(ip + 2 * nw, yo.data(), (size_t)nh * 4);
    memcpy(ip + 2 * nw + nh, yc.data(), (size_t)nh * 4);
    for (int i = 0; i < nw; ++i)
      for (int k = 0; k < T; ++k) fp[(size_t)i * T + k] = k < xc[i] ? xa[i][k] : 0.f;
    for (int i = 0; i < nh; ++i)
      for (int k = 0; k < T; ++k) fp[((size_t)nw + i) * T + k] = k < yc[i] ? ya[i][k] : 0.f;
    // frames already queued may still read the previous tables
    CK(cudaStreamSynchronize(ctx->stream));
    int r = ensure(ctx, tab, host.size());
    if (r) return r;
    CK(cudaMemcpy(tab.p, host.data(), host.size(), cudaMemcpyHostToDevice));
    key[0] = W;
    key[1] = H;
    key[2] = nw;
    key[3] = nh;
    ctx->at_t[which] = T;
    ctx->res_epoch++;
  }
  const int* ip = (const int*)tab.p;
  f.xofs = ip;
  f.xcnt = ip + nw;
  f.yofs = ip + 2 * nw;
  f.ycnt = ip + 2 * nw + nh;
  f.xal = (const float*)(ip + 2 * nw + 2 * nh);
  f.yal = f.xal + (size_t)nw * ctx->at_t[which];
  f.area_t = ctx->at_t[which];
  f.lin = lin ? 1 : 0;
  return VD3D_OK;
}

// eye fit: cv2.resize INTER_AREA (Half-SBS) or pad_to_aspect_ratio (core/render_3d.py:101-131,1409-1417)
int plan_fit(vd3d_ctx* ctx, int fmt, int W, int H, int pw, int ph, FitPlan& f, int tab_slot = 0) {
  int nw, nh;
  if (fmt == VD3D_FMT_HALF_SBS) {
    nw = pw;
    nh = ph;
    f.fit_x0 = f.fit_y0 = 0;
  } else {
    double ta = (double)pw / (double)ph;
    double ca = (double)W / (double)H;
    if (ca > ta) {
      nw = pw;
      nh = (int)(pw / ca);
    } else {
      nh = ph;
      nw = (int)(ca * ph);
    }
    f.fit_x0 = (pw - nw) / 2;
    f.fit_y0 = (ph - nh) / 2;
  }
  if (nw <= 0 || nh <= 0) return fail(ctx, VD3D_ERR_ARG, "degenerate eye size");
  f.fit_w = nw;
  f.fit_h = nh;
  if (W % nw == 0 && H % nh == 0) {  // identity or cv2's integer "area fast" path
    f.sx = W / nw;
    f.sy = H / nh;
    return VD3D_OK;
  }
  if (nw > W || nh > H) {
    // cv2 switches INTER_AREA to a fixed-point bilinear scheme as soon as one axis grows (e.g. the hard-coded
    // 1920x1080 Full-SBS eyes for sources below 1080p, core/render_3d.py:1121).
    f.sx = f.sy = 0;
    // the key of the cached tables does not encode the mode: W x H -> nw x nh is either a shrink or an enlargement
    return ensure_area_tabs(ctx, tab_slot, W, H, nw, nh, f, true);
  }
  f.sx = f.sy = 0;
  return ensure_area_tabs(ctx, tab_slot, W, H, nw, nh, f);
}

void set_fit(PostArgs& pa, const FitPlan& fp) {
  pa.fit_x0 = fp.fit_x0;
  pa.fit_y0 = fp.fit_y0;
  pa.fit_w = fp.fit_w;
  pa.fit_h = fp.fit_h;
  pa.sx = fp.sx;
  pa.sy = fp.sy;
  pa.inv_area = fp.sx > 0 ? (float)(1.0 / (double)(fp.sx * fp.sy)) : 1.f;
  pa.xofs = fp.xofs;
  pa.xcnt = fp.xcnt;
  pa.xal = fp.xal;
  pa.yofs = fp.yofs;
  pa.ycnt = fp.ycnt;
  pa.yal = fp.yal;
  pa.area_t = fp.area_t;
  pa.lin = fp.lin;
}

int copy_in(vd3d_ctx* ctx, Buf& b, const void* src, size_t bytes, int mem, cudaStream_t s, const void** dev) {
  if (mem == VD3D_MEM_DEVICE) {
    *dev = src;
    return VD3D_OK;
  }
  int r = ensure(ctx, b, bytes);
  if (r) return r;
  CK(cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, s));
  *dev = b.p;
  return VD3D_OK;
}

// where a stage entry point writes its output: dst itself, or the staging buffer b when dst is host memory
int stage_out(vd3d_ctx* ctx, Buf& b, void* dst, size_t bytes, int mem, void** dev) {
  *dev = dst;
  if (mem != VD3D_MEM_HOST) return VD3D_OK;
  int r = ensure(ctx, b, bytes);
  if (r) return r;
  *dev = b.p;
  return VD3D_OK;
}

// after the launch: check it, copy a staged output back to dst and wait for the result
int stage_finish(vd3d_ctx* ctx, void* dst, const void* dev, size_t bytes, int mem) {
  CK(cudaGetLastError());
  if (mem == VD3D_MEM_HOST) CK(cudaMemcpyAsync(dst, dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return VD3D_OK;
}

// DOF blur + colour grade of an eye pair [H, W] from a depth map [dh, dw] with the cached five-level Gaussian bank
// (levels == 1: grade only); sources, destinations and the focal depth are the caller's
DofArgs dof_args(const vd3d_ctx* ctx, int levels, int H, int W, const float* depth, int dh, int dw, double sat,
                 double con, double bri) {
  DofArgs da;
  memset(&da, 0, sizeof da);
  da.H = H;
  da.W = W;
  da.depth = depth;
  da.dh = dh;
  da.dw = dw;
  da.focus_w = (float)(0.35 + 1e-6);
  da.idx_max = (float)(5 - 1 - 1e-6);
  da.nlevels = levels;
  if (levels > 1) {
    for (int i = 0; i < 8; ++i) {
      da.ksize[i] = ctx->dof_ksize[i];
      da.koff[i] = ctx->dof_koff[i];
    }
    da.kern = (const float*)ctx->dof_kern.p;
    da.halo = ctx->dof_halo;
  }
  da.sat = (float)sat;
  da.con = (float)con;
  da.bri = (float)bri;
  return da;
}

// k_post on one image [h, w] in the single-eye pass-through layout: identity fit onto an ow x oh output, no bars
PostArgs single_eye_post(const void* src, int h, int w, uint8_t* out, int ow, int oh) {
  PostArgs pa;
  memset(&pa, 0, sizeof pa);
  pa.left = (const uint8_t*)src;
  pa.right = (const uint8_t*)src;
  pa.H = h;
  pa.W = w;
  pa.fmt = VD3D_FMT_INTERLACED;
  pa.per_eye_w = ow;
  pa.per_eye_h = oh;
  pa.fit_w = ow;
  pa.fit_h = oh;
  pa.sx = pa.sy = 1;
  pa.inv_area = 1.f;
  pa.out = out;
  pa.out_w = ow;
  pa.out_h = oh;
  return pa;
}

// Capture what enqueue() launches on stream s into *exec.  When capture is unavailable or fails, this context
// switches to eager launches for good (with a message on stderr) and false is returned: the caller then undoes its
// bookkeeping of the captured enqueue and launches eagerly.
template <class Enqueue>
bool capture(vd3d_ctx* ctx, cudaStream_t s, cudaGraphExec_t* exec, Enqueue enqueue) {
  if (cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
    fprintf(stderr, "vd3d: CUDA graph capture unavailable (%s); continuing with eager launches\n",
            cudaGetErrorString(cudaGetLastError()));
    ctx->use_graphs = 0;
    return false;
  }
  const int r = enqueue();
  cudaGraph_t graph = nullptr;
  const cudaError_t ce = cudaStreamEndCapture(s, &graph);
  if (r != VD3D_OK || ce != cudaSuccess || !graph || cudaGraphInstantiate(exec, graph, 0) != cudaSuccess) {
    fprintf(stderr, "vd3d: CUDA graph capture failed (r=%d, %s); continuing with eager launches\n", r,
            cudaGetErrorString(cudaGetLastError()));
    if (graph) cudaGraphDestroy(graph);
    *exec = nullptr;
    ctx->use_graphs = 0;
    return false;
  }
  cudaGraphDestroy(graph);
  return true;
}

}  // namespace

// ===========================================================================
// C ABI
// ===========================================================================
extern "C" {

int vd3d_struct_size(int which) {
  switch (which) {
    case 0: return (int)sizeof(vd3d_shift_params);
    case 1: return (int)sizeof(vd3d_render_params);
    case 2: return (int)sizeof(vd3d_size_plan);
    case 3: return (int)sizeof(vd3d_frame_info);
    case 4: return (int)sizeof(vd3d_upscale_params);
    case 5: return (int)sizeof(vd3d_tile);
    case 6: return (int)sizeof(vd3d_depth_config_ex);
    default: return -1;
  }
}

int vd3d_create(int device, vd3d_ctx** out) {
  if (!out) return VD3D_ERR_ARG;
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    g_create_error = std::string("no CUDA device: ") + cudaGetErrorString(e) +
                     " (libvd3d has no CPU fallback)";
    return VD3D_ERR_CUDA;
  }
  if (device < 0 || device >= n) {
    g_create_error = "bad device index";
    return VD3D_ERR_ARG;
  }
  vd3d_ctx* ctx = new vd3d_ctx();
  ctx->device = device;
  auto bail = [&](const char* what, cudaError_t er) {
    g_create_error = std::string(what) + ": " + cudaGetErrorString(er);
    delete ctx;
    return VD3D_ERR_CUDA;
  };
  if ((e = cudaSetDevice(device)) != cudaSuccess) return bail("cudaSetDevice", e);
  if ((e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)) != cudaSuccess) return bail("stream", e);
  if ((e = cudaStreamCreateWithFlags(&ctx->s_h2d, cudaStreamNonBlocking)) != cudaSuccess) return bail("stream", e);
  if ((e = cudaStreamCreateWithFlags(&ctx->s_d2h, cudaStreamNonBlocking)) != cudaSuccess) return bail("stream", e);
  for (int i = 0; i < kSlots; ++i) {
    cudaEventCreateWithFlags(&ctx->ev_h2d[i], cudaEventDisableTiming);
    cudaEventCreateWithFlags(&ctx->ev_done[i], cudaEventDisableTiming);
    cudaEventCreateWithFlags(&ctx->ev_d2h[i], cudaEventDisableTiming);
  }
  if ((e = cudaMalloc(&ctx->st, sizeof(DevState))) != cudaSuccess) return bail("cudaMalloc", e);
  if ((e = cudaMalloc(&ctx->fs, sizeof(FrameScalars))) != cudaSuccess) return bail("cudaMalloc", e);
  if ((e = cudaMalloc(&ctx->jobwords, sizeof(uint32_t) * (kJobs * kJobWords + kBarWords))) != cudaSuccess)
    return bail("cudaMalloc", e);
  ctx->bar = ctx->jobwords + kJobs * kJobWords;
  if ((e = cudaMalloc(&ctx->tgs, sizeof(SelTarget) * kJobs * 4)) != cudaSuccess) return bail("cudaMalloc", e);
  if ((e = cudaMalloc(&ctx->crops_dev, sizeof(int32_t) * 2 * kSlots)) != cudaSuccess) return bail("cudaMalloc", e);
  if ((e = cudaMalloc(&ctx->detect_words, sizeof(uint32_t) * 2)) != cudaSuccess) return bail("cudaMalloc", e);
  cudaMemset(ctx->crops_dev, 0, sizeof(int32_t) * 2 * kSlots);
  cudaMemset(ctx->st, 0, sizeof(DevState));
  cudaMemset(ctx->fs, 0, sizeof(FrameScalars));
  cudaMemset(ctx->jobwords, 0, sizeof(uint32_t) * (kJobs * kJobWords + kBarWords));
  cudaMemset(ctx->tgs, 0, sizeof(SelTarget) * kJobs * 4);
  for (int j = 0; j < kJobs; ++j) {
    uint32_t* b = ctx->jobwords + (size_t)j * kJobWords;
    ctx->jm[j].hist1 = b;
    ctx->jm[j].hist2 = b + 4096;
    ctx->jm[j].hist3 = b + 4096 + 4 * 4096;
    ctx->jm[j].hist64 = b + 4096 + 4 * 4096 + 4 * 64;
    ctx->jm[j].count = b + 4096 + 4 * 4096 + 4 * 64 + 64;
    ctx->jm[j].tg = ctx->tgs + j * 4;
  }
  if ((e = cudaMallocHost(&ctx->fs_pinned, sizeof(FrameScalars))) != cudaSuccess) return bail("cudaMallocHost", e);
  if ((e = cudaMallocHost(&ctx->st_pinned, sizeof(DevState))) != cudaSuccess) return bail("cudaMallocHost", e);
  if ((e = init_kernel_attributes()) != cudaSuccess) return bail("cudaFuncSetAttribute", e);
  if ((e = stats_grid(device, &ctx->stats_blocks)) != cudaSuccess) return bail("k_stats occupancy", e);
  {
    const char* v = getenv("VD3D_EXACT");
    ctx->exact = (v && atoi(v)) ? 1 : 0;
    if ((v = getenv("VD3D_DEPTH_BATCH"))) ctx->depth_batch = atoi(v);
    if (ctx->depth_batch < 1) ctx->depth_batch = 1;
    if (ctx->depth_batch > kMaxDepthBatch) ctx->depth_batch = kMaxDepthBatch;
  }
  *out = ctx;
  return VD3D_OK;
}

void vd3d_destroy(vd3d_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  Buf* bufs[] = {&ctx->xs,    &ctx->ys,    &ctx->tdf,   &ctx->dn0,   &ctx->dn1,      &ctx->rgb_s,
                 &ctx->frameB, &ctx->d,     &ctx->shift, &ctx->e2,    &ctx->eyeL,     &ctx->eyeR,
                 &ctx->eyeL2, &ctx->eyeR2, &ctx->in_rgbf, &ctx->in_depthf, &ctx->dof_kern,
                 &ctx->area_tab[0], &ctx->area_tab[1], &ctx->lb_in, &ctx->lb_prev, &ctx->lb_gray, &ctx->lb_mag,
                 &ctx->lb_label, &ctx->lb_flag, &ctx->lb_rec, &ctx->lb_nodes, &ctx->lb_node_sum, &ctx->lb_out,
                 &ctx->lb_hist, &ctx->td_frames, &ctx->td_crops, &ctx->td_preds, &ctx->td_wgt, &ctx->td_jobs,
                 &ctx->td_depth, &ctx->td_u8, &ctx->td_sel, &ctx->td_mm, &ctx->td_stats, &ctx->td_out, &ctx->td_outf};
  for (Buf* b : bufs)
    if (b->p) cudaFree(b->p);
  for (int i = 0; i < kSlots; ++i) {
    if (ctx->in_frame[i].p) cudaFree(ctx->in_frame[i].p);
    if (ctx->in_depth[i].p) cudaFree(ctx->in_depth[i].p);
    if (ctx->out_dev[i].p) cudaFree(ctx->out_dev[i].p);
  }
  for (int i = 0; i < kSrSlots; ++i) {
    if (ctx->sr_in[i].p) cudaFree(ctx->sr_in[i].p);
    if (ctx->sr_out[i].p) cudaFree(ctx->sr_out[i].p);
  }
  drop_graphs(ctx);
  drop_depth_graphs(ctx);
  for (int i = 0; i < kClones; ++i) {
    if (ctx->dclone[i]) vd3d_depth_destroy(ctx->dclone[i]);
    if (ctx->s_depth[i]) cudaStreamDestroy(ctx->s_depth[i]);
    if (ctx->ev_depth[i]) cudaEventDestroy(ctx->ev_depth[i]);
  }
  cudaFree(ctx->st);
  cudaFree(ctx->fs);
  cudaFree(ctx->jobwords);
  cudaFree(ctx->tgs);
  cudaFree(ctx->crops_dev);
  cudaFree(ctx->detect_words);
  if (ctx->crops_host) cudaFreeHost(ctx->crops_host);
  cudaFreeHost(ctx->fs_pinned);
  cudaFreeHost(ctx->st_pinned);
  for (int i = 0; i < kSlots; ++i) {
    cudaEventDestroy(ctx->ev_h2d[i]);
    cudaEventDestroy(ctx->ev_done[i]);
    cudaEventDestroy(ctx->ev_d2h[i]);
  }
  cudaStreamDestroy(ctx->stream);
  cudaStreamDestroy(ctx->s_h2d);
  cudaStreamDestroy(ctx->s_d2h);
  delete ctx;
}

const char* vd3d_last_error(vd3d_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int vd3d_reset_state(vd3d_ctx* ctx, uint32_t which) {
  if (!ctx) return VD3D_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));
  DevState h;
  CK(cudaMemcpy(&h, ctx->st, sizeof h, cudaMemcpyDeviceToHost));
  if (which & VD3D_STATE_GLOBAL) {
    h.pct_lo = h.pct_hi = 0.f;
    h.pct_init = 0;
    h.conv_val = 0.0;
    h.conv_init = 0;
    h.fw_prev = 0.0;
    h.fw_count = 0;
    h.bar_prev = 0;
  }
  if (which & VD3D_STATE_CLIP) {
    h.tdf_init = 0;
    h.sm_fg = h.sm_mg = h.sm_bg = 0.0;
    h.sm_init = 0;
    h.focal = 0.0;
    h.focal_alpha = 0.15;
    h.focal_init = 0;
    h.have_prev_depth = 0;
    ctx->frame_parity = 0;
  }
  CK(cudaMemcpy(ctx->st, &h, sizeof h, cudaMemcpyHostToDevice));
  return VD3D_OK;
}

void* vd3d_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMallocHost(&p, bytes) != cudaSuccess) return nullptr;
  return p;
}
void vd3d_host_free(void* p) {
  if (p) cudaFreeHost(p);
}
void* vd3d_stream(vd3d_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
int vd3d_sync(vd3d_ctx* ctx) {
  if (!ctx) return VD3D_ERR_ARG;
  CK(cudaStreamSynchronize(ctx->stream));
  CK(cudaStreamSynchronize(ctx->s_d2h));
  return VD3D_OK;
}
uint64_t vd3d_launch_count(vd3d_ctx* ctx) { return ctx ? ctx->launches : 0; }
int vd3d_profile(vd3d_ctx* ctx, int enable) {
  if (!ctx) return VD3D_ERR_ARG;
  ctx->prof = enable;
  return VD3D_OK;
}
int vd3d_profile_collect(vd3d_ctx* ctx, int stage, double* total_ms, int* count) {
  if (!ctx || stage < 0 || stage >= 4 || !total_ms || !count) return VD3D_ERR_ARG;
  CK(cudaStreamSynchronize(ctx->stream));
  double t = 0;
  int n = 0;
  auto& v = ctx->prof_ev[stage];
  for (size_t i = 0; i + 1 < v.size(); i += 2) {
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, v[i], v[i + 1]));
    t += ms;
    ++n;
  }
  for (cudaEvent_t e : v) ctx->prof_pool.push_back(e);
  v.clear();
  *total_ms = t;
  *count = n;
  if (stage == 2) {  // depth samples cover whole batches: report frames so that total / count is per frame
    if (ctx->prof_depth_frames > 0) *count = ctx->prof_depth_frames;
    ctx->prof_depth_frames = 0;
  }
  return VD3D_OK;
}
// 1: the one-kernel-per-op path with correctly rounded transcendentals (bit-for-bit with oracle/dibr.py);
// 0 (default; env VD3D_EXACT=1 flips the default): persistent stats kernel + fused render kernel
int vd3d_set_exact(vd3d_ctx* ctx, int enable) {
  if (!ctx) return VD3D_ERR_ARG;
  if (ctx->exact != (enable ? 1 : 0)) {
    cudaStreamSynchronize(ctx->stream);
    drop_graphs(ctx);
    ctx->exact = enable ? 1 : 0;
  }
  return VD3D_OK;
}
int vd3d_get_exact(vd3d_ctx* ctx) { return ctx ? ctx->exact : -1; }
// 1 while frame graphs are enabled (0 after vd3d_set_graphs(0) or after a failed capture fell back to eager launches)
int vd3d_graphs_active(vd3d_ctx* ctx) { return ctx ? ctx->use_graphs : -1; }
int vd3d_set_graphs(vd3d_ctx* ctx, int enable) {
  if (!ctx) return VD3D_ERR_ARG;
  ctx->use_graphs = enable;
  if (!enable) drop_graphs(ctx);
  return VD3D_OK;
}

// ---------------------------------------------------------------------------
int vd3d_pixel_shift(vd3d_ctx* ctx, const float* rgb, const float* depth, int in_h, int in_w, int width,
                     int height, const vd3d_shift_params* p, uint8_t* left_bgr, uint8_t* right_bgr, float* shift,
                     int mem, vd3d_frame_info* info) {
  if (!ctx || !rgb || !depth || !p || !left_bgr || !right_bgr) return fail(ctx, VD3D_ERR_ARG, "null argument");
  if (in_h < 2 || in_w < 2 || width < 2 || height < 2) return fail(ctx, VD3D_ERR_ARG, "image too small");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const int W = width, H = height;
  int r;
  const bool fastp = !ctx->exact && render_supports(p->enable_feathering ? 1 : 0, p->blur_ksize);
  if ((r = begin_frame(ctx))) return r;
  if (!fastp) {  // k_stats does it itself
    launch_set_shifts(ctx->fs, p->fg_shift, p->mg_shift, p->bg_shift, s);
    ctx->launches += 1;
  }
  const void *rgb_d, *depth_d;
  if ((r = copy_in(ctx, ctx->in_rgbf, rgb, sizeof(float) * 3 * (size_t)in_h * in_w, mem, s, &rgb_d))) return r;
  if ((r = copy_in(ctx, ctx->in_depthf, depth, sizeof(float) * (size_t)in_h * in_w, mem, s, &depth_d))) return r;
  const float* src_f32 = (const float*)rgb_d;
  if (in_h != H || in_w != W) {
    if ((r = ensure(ctx, ctx->frameB, sizeof(float) * 3 * (size_t)W * H))) return r;
    launch_resize_planar((const float*)rgb_d, 3, in_h, in_w, (float*)ctx->frameB.p, H, W, s);
    ctx->launches += 1;
    src_f32 = (const float*)ctx->frameB.p;
  }
  void *l_d, *r_d;
  size_t eye_bytes = (size_t)W * H * 3;
  if ((r = stage_out(ctx, ctx->eyeL, left_bgr, eye_bytes, mem, &l_d))) return r;
  if ((r = stage_out(ctx, ctx->eyeR, right_bgr, eye_bytes, mem, &r_d))) return r;
  CoreIn ci;
  ci.depth = (const float*)depth_d;
  ci.sh = in_h;
  ci.sw = in_w;
  ci.src_u8 = nullptr;
  ci.src_pitch = 0;
  ci.cx0 = ci.cy0 = 0;
  ci.src_f32 = src_f32;
  ci.W = W;
  ci.H = H;
  ci.p = *p;
  ci.grade = 0;
  ci.sat = 1.f;
  ci.con = 1.f;
  ci.bri = 0.f;
  ci.left = (uint8_t*)l_d;
  ci.right = (uint8_t*)r_d;
  if (fastp) {
    FastPost post;
    if ((r = run_core_fast(ctx, ci, nullptr, post))) return r;
  } else {
    if ((r = run_core(ctx, ci))) return r;
  }
  if (mem == VD3D_MEM_HOST) {
    CK(cudaMemcpyAsync(left_bgr, l_d, eye_bytes, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(right_bgr, r_d, eye_bytes, cudaMemcpyDeviceToHost, s));
  }
  if (shift)
    CK(cudaMemcpyAsync(shift, ctx->shift.p, sizeof(float) * (size_t)W * H,
                       mem == VD3D_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, s));
  if (info) {
    if ((r = fetch_info(ctx, info))) return r;
  } else {
    CK(cudaStreamSynchronize(s));
  }
  return VD3D_OK;
}

int vd3d_plan_sizes(int src_w, int src_h, const vd3d_render_params* rp, vd3d_size_plan* o) {
  if (!rp || !o || src_w < 2 || src_h < 2) return VD3D_ERR_ARG;
  double target_ratio = rp->aspect_ratio;
  int crop[4];
  aspect_crop(src_w, src_h, target_ratio, crop);
  int rw, rh, pw, ph, outw, outh, tew, teh;
  int fmt = rp->output_format;
  if (rp->preserve_original_aspect) {
    // original_video_* default to the FIRST frame tensor's size (pre-crop) (core/render_3d.py:1087-1092)
    int ow = src_w, oh = src_h;
    if (rp->original_video_width > 0 && rp->original_video_height > 0) {
      ow = rp->original_video_width;
      oh = rp->original_video_height;
    }
    rw = ow;
    rh = oh;
    if (fmt == VD3D_FMT_FULL_SBS) {
      pw = rw; ph = rh; outw = rw * 2; outh = rh;
    } else if (fmt == VD3D_FMT_HALF_SBS) {
      pw = rw / 2; ph = rh; outw = rw; outh = rh;
    } else if (fmt == VD3D_FMT_VR) {  // core/render_3d.py:1104-1108
      pw = 1440; ph = 1600; outw = 2880; outh = 1600;
    } else {
      pw = rw; ph = rh; outw = rw * 2; outh = rh;
    }
    tew = pw;
    teh = ph;
  } else {
    rh = rp->output_height;
    rw = (int)(rh * target_ratio);
    if (rw % 2 != 0) rw += 1;
    if (fmt == VD3D_FMT_FULL_SBS) {
      pw = 1920; ph = 1080; outw = 3840; outh = 1080;
    } else if (fmt == VD3D_FMT_HALF_SBS) {
      pw = rw / 2; ph = rh; outw = rw; outh = rh;
    } else if (fmt == VD3D_FMT_VR) {  // core/render_3d.py:1129-1133
      pw = 1440; ph = 1600; outw = 2880; outh = 1600;
    } else {
      pw = rw; ph = rh; outw = rw * 2; outh = rh;
    }
    tew = pw;
    teh = (int)(pw / target_ratio);
    if (teh % 2 != 0) teh += 1;
  }
  o->crop_x0 = crop[0];
  o->crop_y0 = crop[1];
  o->crop_w = crop[2];
  o->crop_h = crop[3];
  o->target_eye_w = tew;
  o->target_eye_h = teh;
  o->resized_width = rw;
  o->resized_height = rh;
  o->per_eye_w = pw;
  o->per_eye_h = ph;
  o->out_width = outw;
  o->out_height = outh;
  return VD3D_OK;
}

// the vd3d_shift_params render_sbs_3d hands to pixel_shift_cuda (core/render_3d.py:1284-1331)
static vd3d_shift_params loop_shift_params(const vd3d_render_params* rp) {
  vd3d_shift_params sp;
  memset(&sp, 0, sizeof sp);
  sp.fg_shift = sp.mg_shift = sp.bg_shift = 0.0;  // taken from FrameScalars (set by k_fin_norm)
  sp.blur_ksize = rp->blur_ksize;
  sp.feather_strength = rp->feather_strength;
  sp.max_pixel_shift_percent = rp->max_pixel_shift_percent;
  sp.parallax_balance = 0.8;  // never forwarded by render_sbs_3d (core/render_3d.py:1284-1331)
  sp.zero_parallax_strength = rp->zero_parallax_strength;
  sp.use_subject_tracking = rp->use_subject_tracking;
  sp.enable_floating_window = rp->use_floating_window;
  sp.enable_feathering = rp->enable_feathering;
  sp.enable_edge_masking = rp->enable_edge_masking;
  sp.convergence_strength = rp->convergence_strength;
  sp.enable_dynamic_convergence = rp->enable_dynamic_convergence;
  sp.depth_pop_gamma = 0.85;  // hard-coded at the call site (1299-1305)
  sp.depth_pop_mid = 0.50;
  sp.depth_stretch_lo = 0.05;
  sp.depth_stretch_hi = 0.95;
  sp.fg_pop_multiplier = 1.20;
  sp.bg_push_multiplier = 1.10;
  sp.subject_lock_strength = 1.00;
  return sp;
}

// fast-path core of one loop iteration: k_stats (ingest .. scalar trackers) -> k_shift -> k_render.  *fused tells the
// caller that bars + sharpen + eye fit + pack already happened inside k_render (out_d is complete).
static int enqueue_core_fast(vd3d_ctx* ctx, const IngestArgs& ia, const LoopArgs& la, float* dn, const float* dn_prev,
                             CoreIn ci, const vd3d_render_params* rp, const vd3d_size_plan& pl, uint8_t* out_d,
                             bool ident, bool* fused) {
  int r;
  const int tw = ia.tw, th = ia.th, W = ci.W, H = ci.H;
  FastLoop lp;
  memset(&lp, 0, sizeof lp);
  lp.ia = &ia;
  lp.dn = dn;
  lp.dn_prev = dn_prev;
  lp.la = &la;
  FastPost post;
  if (!ident) {
    if ((r = ensure(ctx, ctx->rgb_s, sizeof(float4) * (size_t)tw * th))) return r;
    lp.rgbx_s = (float4*)ctx->rgb_s.p;
    post.src_rgbx = lp.rgbx_s;
    if (W != tw || H != th) {
      if ((r = ensure(ctx, ctx->frameB, sizeof(float4) * (size_t)W * H))) return r;
      lp.rgbx = (float4*)ctx->frameB.p;
      post.src_rgbx = lp.rgbx;
    }
  }

  // can k_render finish the frame?  SBS formats whose eye fit is the identity or cv2's integer 2:1 horizontal INTER_AREA
  *fused = false;
  const bool dof = rp->dof_strength > 0.0;
  if (!ctx->stats_only && !dof && (rp->output_format == VD3D_FMT_HALF_SBS || rp->output_format == VD3D_FMT_FULL_SBS)) {
    FitPlan fp;
    if ((r = plan_fit(ctx, rp->output_format, W, H, pl.per_eye_w, pl.per_eye_h, fp))) return r;
    const bool plain = !fp.xal && !fp.lin && fp.fit_x0 == 0 && fp.fit_y0 == 0 && fp.fit_w == pl.per_eye_w &&
                       fp.fit_h == pl.per_eye_h && fp.sy == 1 && pl.per_eye_h == H;
    if (plain && fp.sx == 1 && pl.per_eye_w == W) post.fuse = 1;
    if (plain && fp.sx == 2 && pl.per_eye_w * 2 == W) post.fuse = 2;
  }
  if (post.fuse) {
    post.sharpen = 1;
    sharpen_coeffs(rp->sharpness_factor, post.kc, post.ke);
    post.out = out_d;
    post.out_w = 2 * pl.per_eye_w;
    post.per_eye_w = pl.per_eye_w;
    *fused = true;
  } else if (!ctx->stats_only) {
    const size_t eye_bytes = (size_t)W * H * 3;
    if ((r = ensure(ctx, ctx->eyeL, eye_bytes))) return r;
    if ((r = ensure(ctx, ctx->eyeR, eye_bytes))) return r;
    ci.left = (uint8_t*)ctx->eyeL.p;
    ci.right = (uint8_t*)ctx->eyeR.p;
  }
  return run_core_fast(ctx, ci, &lp, post);
}

// exact-path core of one loop iteration, one kernel per reference op: ingest + TemporalDepthFilter,
// DepthPercentileEMA, normalisation + subject estimate, then pixel_shift_cuda into eyeL / eyeR
static int enqueue_core_exact(vd3d_ctx* ctx, IngestArgs ia, const LoopArgs& la, float* dn, const float* dn_prev,
                              CoreIn ci, bool ident) {
  cudaStream_t s = ctx->stream;
  int r;
  const int tw = ia.tw, th = ia.th, W = ci.W, H = ci.H;
  const size_t tpx = (size_t)tw * th;
  if (!ident) {
    if ((r = ensure(ctx, ctx->rgb_s, sizeof(float) * 3 * tpx))) return r;
    ia.rgb_s = (float*)ctx->rgb_s.p;
  }
  launch_ingest(ia, s);
  ctx->launches += 1;
  // ---- DepthPercentileEMA(p_lo=.02, p_hi=.98, alpha=.92)
  uint32_t l0, l1, h0, h1;
  float wlo, whi;
  quantile_rank(0.02, (long long)tpx, l0, l1, wlo);
  quantile_rank(0.98, (long long)tpx, h0, h1, whi);
  launch_set_ranks(ctx->jm[0].tg, l0, l1, h0, h1, s);
  ctx->launches += 1;
  SelJob pj = make_job(ctx->jm[0], ia.tdf, tw, 0, tw, 0, th, 0, 4, 0, false);
  launch_select(pj, nullptr, sel_blocks(th), s);
  ctx->launches += kSelectLaunches;
  launch_fin_pct(pj, wlo, whi, 0.92f, (float)(1 - 0.92), ctx->st, ctx->fs, s);
  ctx->launches += 1;
  launch_normalize(ia.tdf, dn, dn_prev, th, tw, ctx->st, ctx->fs, s);
  ctx->launches += 1;
  SelJob sn = make_job(ctx->jm[1], dn, tw, tw / 5, tw * 4 / 5, th / 5, th * 4 / 5, 1, 1, 1, true);
  launch_select(sn, nullptr, sel_blocks(th * 4 / 5 - th / 5), s);
  ctx->launches += kSelectLaunches;
  launch_fin_norm(sn, la, ctx->st, ctx->fs, s);
  ctx->launches += 1;

  // ---- pixel_shift_cuda
  const size_t eye_bytes = (size_t)W * H * 3;
  if ((r = ensure(ctx, ctx->eyeL, eye_bytes))) return r;
  if ((r = ensure(ctx, ctx->eyeR, eye_bytes))) return r;
  if (!ident) {
    ci.src_f32 = ia.rgb_s;
    if (W != tw || H != th) {
      if ((r = ensure(ctx, ctx->frameB, sizeof(float) * 3 * (size_t)W * H))) return r;
      launch_resize_planar(ia.rgb_s, 3, th, tw, (float*)ctx->frameB.p, H, W, s);
      ctx->launches += 1;
      ci.src_f32 = (const float*)ctx->frameB.p;
    }
  }
  ci.left = (uint8_t*)ctx->eyeL.p;
  ci.right = (uint8_t*)ctx->eyeR.p;
  return run_core(ctx, ci);
}

// DOF (when on), then bars + sharpen + eye fit + pack of the eyes in eyeL / eyeR into out_d
static int enqueue_dof_post(vd3d_ctx* ctx, const vd3d_render_params* rp, const vd3d_size_plan& pl, const float* dn,
                            uint8_t* out_d) {
  cudaStream_t s = ctx->stream;
  int r;
  const int W = pl.resized_width, H = pl.resized_height;
  const uint8_t* eye_l = (const uint8_t*)ctx->eyeL.p;
  const uint8_t* eye_r = (const uint8_t*)ctx->eyeR.p;
  if (rp->dof_strength > 0.0) {
    const size_t eye_bytes = (size_t)W * H * 3;
    if ((r = ensure_dof_kernels(ctx, rp->dof_strength, 5))) return r;
    if ((r = ensure(ctx, ctx->eyeL2, eye_bytes))) return r;
    if ((r = ensure(ctx, ctx->eyeR2, eye_bytes))) return r;
    DofArgs da = dof_args(ctx, 5, H, W, dn, pl.target_eye_h, pl.target_eye_w, rp->color_saturation,
                          rp->color_contrast, rp->color_brightness);
    da.src_l = eye_l;
    da.src_r = eye_r;
    da.dst_l = (uint8_t*)ctx->eyeL2.p;
    da.dst_r = (uint8_t*)ctx->eyeR2.p;
    da.fs = ctx->fs;  // focal comes from the FocalDepthTracker state on the device
    launch_dof(da, 2, s);
    ctx->launches += 1;
    eye_l = da.dst_l;
    eye_r = da.dst_r;
  }
  FitPlan fp;
  if ((r = plan_fit(ctx, rp->output_format, W, H, pl.per_eye_w, pl.per_eye_h, fp))) return r;
  PostArgs pa;
  pa.left = eye_l;
  pa.right = eye_r;
  pa.H = H;
  pa.W = W;
  pa.fs = ctx->fs;
  pa.sharpen = 1;
  sharpen_coeffs(rp->sharpness_factor, pa.kc, pa.ke);
  pa.fmt = rp->output_format;
  pa.per_eye_w = pl.per_eye_w;
  pa.per_eye_h = pl.per_eye_h;
  set_fit(pa, fp);
  pa.out = out_d;
  if (rp->output_format == VD3D_FMT_ANAGLYPH || rp->output_format == VD3D_FMT_INTERLACED) {
    pa.out_w = pl.per_eye_w;
    pa.out_h = pl.per_eye_h;
  } else {
    pa.out_w = 2 * pl.per_eye_w;  // hstack of the fitted eyes
    pa.out_h = pl.per_eye_h;
  }
  launch_post(pa, s);
  ctx->launches += 1;
  CK(cudaGetLastError());
  return VD3D_OK;
}

// enqueue one loop iteration on ctx->stream; inputs/outputs are DEVICE pointers.  slot: the staging slot whose
// crops_dev entry receives the frame's (top, bottom) under auto_crop_black_bars.
static int enqueue_frame(vd3d_ctx* ctx, const uint8_t* frame_d, const uint8_t* depth_d, int depth_channels,
                         int src_h, int src_w, const vd3d_render_params* rp, const vd3d_size_plan& pl,
                         uint8_t* out_d, int slot) {
  int r;
  ProfScope frame_scope(ctx, 0);
  const int tw = pl.target_eye_w, th = pl.target_eye_h;
  const int W = pl.resized_width, H = pl.resized_height;
  if (tw < 8 || th < 8 || W < 8 || H < 8) return fail(ctx, VD3D_ERR_ARG, "frame too small");
  const size_t tpx = (size_t)tw * th;
  if (ctx->tdf_w != tw || ctx->tdf_h != th) {
    if ((r = ensure(ctx, ctx->tdf, sizeof(float) * tpx))) return r;
    if ((r = ensure(ctx, ctx->dn0, sizeof(float) * tpx))) return r;
    if ((r = ensure(ctx, ctx->dn1, sizeof(float) * tpx))) return r;
    ctx->tdf_w = tw;
    ctx->tdf_h = th;
    if ((r = vd3d_reset_state(ctx, VD3D_STATE_CLIP))) return r;
  }
  if ((r = begin_frame(ctx))) return r;
  const bool autocrop = rp->auto_crop_black_bars != 0;
  if (autocrop) {  // detect_black_bars on the frame; the ingest derives the crop from the two words on the device
    launch_black_bars(frame_d, src_h, src_w, 10, ctx->fs->bars, ctx->stream);
    ctx->launches += 1;
  }

  // ---- loop-level inputs: ingest + TemporalDepthFilter, trackers, normalised-depth ping-pong, pixel_shift_cuda
  IngestArgs ia;
  memset(&ia, 0, sizeof ia);
  ia.frame = frame_d;
  ia.depth = depth_d;
  ia.depth_ch = depth_channels;
  ia.src_w = src_w;
  ia.src_h = src_h;
  ia.cx0 = pl.crop_x0;
  ia.cy0 = pl.crop_y0;
  ia.cw = pl.crop_w;
  ia.ch = pl.crop_h;
  ia.tw = tw;
  ia.th = th;
  ia.tdf = (float*)ctx->tdf.p;
  ia.alpha = 0.5f;
  ia.one_minus_alpha = (float)(1 - 0.5);
  ia.st = ctx->st;
  if (autocrop) {
    ia.bars = ctx->fs->bars;
    ia.aspect = rp->aspect_ratio;
    ia.crop_out = ctx->crops_dev + 2 * slot;
  }
  LoopArgs la;
  la.fg = rp->fg_shift;
  la.mg = rp->mg_shift;
  la.bg = rp->bg_shift;
  la.ipd = rp->ipd_factor;
  la.resized_width = W;
  la.use_floating_window = rp->use_floating_window;
  la.use_subject_tracking = rp->use_subject_tracking;
  la.crop_count = (long long)(th * 3 / 4 - th / 4) * (long long)(tw * 3 / 4 - tw / 4);
  la.npix = (long long)tpx;
  la.dyn_min = (float)0.90;
  la.dyn_span = (float)(1.15 - 0.90);
  float* dn = (float*)(ctx->frame_parity ? ctx->dn1.p : ctx->dn0.p);
  const float* dn_prev = (const float*)(ctx->frame_parity ? ctx->dn0.p : ctx->dn1.p);
  // identity (the eyes sample the u8 frame directly): not under auto-crop, whose crop is only known on the device; its
  // bilinear resize at scale 1 is an exact identity too, like F.interpolate
  const bool ident = !autocrop && (tw == pl.crop_w && th == pl.crop_h && W == tw && H == th);
  CoreIn ci;
  memset(&ci, 0, sizeof ci);
  ci.depth = dn;
  ci.sh = th;
  ci.sw = tw;
  ci.src_u8 = ident ? frame_d : nullptr;
  ci.src_pitch = src_w;
  ci.cx0 = pl.crop_x0;
  ci.cy0 = pl.crop_y0;
  ci.W = W;
  ci.H = H;
  ci.p = loop_shift_params(rp);
  ci.grade = rp->dof_strength > 0.0 ? 0 : 1;
  ci.sat = (float)rp->color_saturation;
  ci.con = (float)rp->color_contrast;
  ci.bri = (float)rp->color_brightness;

  bool fused = false;
  if (!ctx->exact && render_supports(rp->enable_feathering ? 1 : 0, rp->blur_ksize))
    r = enqueue_core_fast(ctx, ia, la, dn, dn_prev, ci, rp, pl, out_d, ident, &fused);
  else
    r = enqueue_core_exact(ctx, ia, la, dn, dn_prev, ci, ident);
  if (r) return r;
  if (!ctx->stats_only && !fused && (r = enqueue_dof_post(ctx, rp, pl, dn, out_d))) return r;
  ctx->frame_parity ^= 1;
  return VD3D_OK;
}

extern "C" uint64_t vd3d_depth_launch_count(vd3d_depth* e);
extern "C" void vd3d_depth_add_launches(vd3d_depth* e, uint64_t n);

extern "C" int vd3d_depth_infer_batch_device(vd3d_depth* e, int B, const uint8_t* const* frames_bgr_dev, int h, int w,
                                             uint8_t* const* depth_u8_dev, float* const* depth_f32_dev, int invert);

static void drop_depth_graphs(vd3d_ctx* ctx) {
  for (int i = 0; i < kClones; ++i)
    for (int j = 0; j <= kMaxDepthBatch; ++j)
      if (ctx->dg[i][j].exec) {
        cudaGraphExecDestroy(ctx->dg[i][j].exec);
        ctx->dg[i][j].exec = nullptr;
      }
  ctx->dg_warm = 0;
}

static int ensure_depth_clones(vd3d_ctx* ctx, vd3d_depth* parent) {
  if (ctx->dclone_parent == parent && ctx->dclone[0] && ctx->dclone_wver == vd3d_depth_weights_version(parent))
    return VD3D_OK;
  CK(cudaDeviceSynchronize());
  drop_depth_graphs(ctx);
  drop_graphs(ctx);
  ctx->dclone_wver = vd3d_depth_weights_version(parent);
  for (int i = 0; i < kClones; ++i) {
    if (ctx->dclone[i]) vd3d_depth_destroy(ctx->dclone[i]);
    ctx->dclone[i] = nullptr;
    if (!ctx->s_depth[i]) CK(cudaStreamCreateWithFlags(&ctx->s_depth[i], cudaStreamNonBlocking));
    if (!ctx->ev_depth[i]) CK(cudaEventCreateWithFlags(&ctx->ev_depth[i], cudaEventDisableTiming));
    if (vd3d_depth_clone(parent, ctx->s_depth[i], &ctx->dclone[i]) != VD3D_OK)
      return fail(ctx, VD3D_ERR_ARG, "vd3d_depth_clone failed");
  }
  ctx->dclone_parent = parent;
  return VD3D_OK;
}

// depth inference of one batch (staging slots slot0 .. slot0+nb-1) on engine instance c and its stream; one batched
// forward for the nb frames, graph-replayed once the configuration has been seen a few times
static int run_depth_group(vd3d_ctx* ctx, vd3d_depth* parent, int c, int slot0, int nb, int src_h, int src_w) {
  vd3d_depth* e = ctx->dclone[c];
  const uint8_t* f_d[kMaxDepthBatch];
  uint8_t* d_d[kMaxDepthBatch];
  for (int j = 0; j < nb; ++j) {
    f_d[j] = (const uint8_t*)ctx->in_frame[slot0 + j].p;
    d_d[j] = (uint8_t*)ctx->in_depth[slot0 + j].p;
  }
  if (ctx->dg_h != src_h || ctx->dg_w != src_w) {
    drop_depth_graphs(ctx);
    ctx->dg_h = src_h;
    ctx->dg_w = src_w;
  }
  auto eager = [&]() -> int {
    uint64_t l0 = vd3d_depth_launch_count(e);
    int r = vd3d_depth_infer_batch_device(e, nb, f_d, src_h, src_w, d_d, nullptr, 0);
    if (r) ctx->err = std::string("depth engine: ") + vd3d_depth_last_error(e);
    vd3d_depth_add_launches(parent, vd3d_depth_launch_count(e) - l0);
    return r;
  };
  if (!ctx->use_graphs || ctx->dg_warm < 2 * kClones) {  // workspaces of both instances are allocated eagerly first
    ctx->dg_warm++;
    return eager();
  }
  vd3d_ctx::DepthGraph& g = ctx->dg[c][nb];
  if (!g.exec) {
    const uint64_t l0 = vd3d_depth_launch_count(e);
    if (!capture(ctx, ctx->s_depth[c], &g.exec,
                 [&] { return vd3d_depth_infer_batch_device(e, nb, f_d, src_h, src_w, d_d, nullptr, 0); }))
      return eager();
    g.n = vd3d_depth_launch_count(e) - l0;
  }
  CK(cudaGraphLaunch(g.exec, ctx->s_depth[c]));
  vd3d_depth_add_launches(parent, g.n);
  return VD3D_OK;
}

static void drop_graphs(vd3d_ctx* ctx) {
  for (int i = 0; i < kSlots; ++i)
    for (int j = 0; j < 2; ++j)
      if (ctx->fg[i][j].exec) {
        cudaGraphExecDestroy(ctx->fg[i][j].exec);
        ctx->fg[i][j].exec = nullptr;
      }
  ctx->fg_warm = 0;
}

// One frame on the staging buffers of slot b: the render_sbs_3d loop body.
// After two eager frames of an unchanged configuration the launch sequence (~200 kernels) is captured
// once per (slot, parity) into a CUDA graph and replayed; all scalars it depends on live on the device.
static int run_frame_slot(vd3d_ctx* ctx, int b, int depth_channels, int src_h, int src_w,
                          const vd3d_render_params* rp, const vd3d_size_plan& pl) {
  const uint8_t* f_d = (const uint8_t*)ctx->in_frame[b].p;
  uint8_t* d_d = (uint8_t*)ctx->in_depth[b].p;
  uint8_t* o_d = (uint8_t*)ctx->out_dev[b].p;
  auto eager = [&]() { return enqueue_frame(ctx, f_d, d_d, depth_channels, src_h, src_w, rp, pl, o_d, b); };
  bool same = ctx->fg_h == src_h && ctx->fg_w == src_w && ctx->fg_dch == depth_channels &&
              memcmp(&ctx->fg_rp, rp, sizeof *rp) == 0;
  if (ctx->fg_epoch != ctx->res_epoch) {  // another entry point moved / rewrote something the graphs bake in
    drop_graphs(ctx);
    ctx->fg_epoch = ctx->res_epoch;
  }
  if (!same) {
    drop_graphs(ctx);
    ctx->fg_h = src_h;
    ctx->fg_w = src_w;
    ctx->fg_dch = depth_channels;
    ctx->fg_rp = *rp;
  }
  if (!ctx->use_graphs || ctx->prof || ctx->fg_warm < 3) {
    ctx->fg_warm++;
    return eager();
  }
  const int par = ctx->frame_parity;
  vd3d_ctx::FrameGraph& g = ctx->fg[b][par];
  if (!g.exec) {
    const uint64_t l0 = ctx->launches;
    const bool ok = capture(ctx, ctx->stream, &g.exec, eager);
    ctx->frame_parity = par;  // capture does not execute
    g.n_ctx = ctx->launches - l0;
    ctx->launches = l0;
    if (!ok) return eager();
  }
  CK(cudaGraphLaunch(g.exec, ctx->stream));
  ctx->launches += g.n_ctx;
  ctx->frame_parity ^= 1;
  return VD3D_OK;
}

// the packed frame format_3d_output produces (core/render_3d.py:837-860): SBS / VR = hstack of the two fitted eyes,
// i.e. 2 * per_eye_w wide -- for an odd preserve-aspect Half-SBS width that is one less than `out_width`, the size the
// reference opens its writer with (1099-1103)
static int packed_w(const vd3d_render_params* rp, const vd3d_size_plan& pl) {
  if (rp->output_format == VD3D_FMT_ANAGLYPH || rp->output_format == VD3D_FMT_INTERLACED) return pl.per_eye_w;
  return 2 * pl.per_eye_w;
}
static size_t out_bytes(const vd3d_render_params* rp, const vd3d_size_plan& pl) {
  return (size_t)packed_w(rp, pl) * pl.per_eye_h * 3;
}

// vd3d_last_crops bookkeeping of a clip call: room for n (top, bottom) pairs in pinned memory (auto-crop only)
static int begin_crops(vd3d_ctx* ctx, const vd3d_render_params* rp, int n) {
  ctx->crops_n = 0;
  if (!rp->auto_crop_black_bars) return VD3D_OK;
  if (n > ctx->crops_cap) {
    CK(cudaStreamSynchronize(ctx->s_d2h));  // copies of an earlier call may still target the old block
    if (ctx->crops_host) CK(cudaFreeHost(ctx->crops_host));
    ctx->crops_host = nullptr;
    ctx->crops_cap = 0;
    CK(cudaMallocHost(&ctx->crops_host, sizeof(int32_t) * 2 * (size_t)n));
    ctx->crops_cap = n;
  }
  ctx->crops_n = n;
  return VD3D_OK;
}

// behind the output frame of clip frame i (staging slot b) on the D2H stream: its (top, bottom)
static int copy_crop(vd3d_ctx* ctx, const vd3d_render_params* rp, int i, int b) {
  if (!rp->auto_crop_black_bars) return VD3D_OK;
  CK(cudaMemcpyAsync(ctx->crops_host + 2 * (size_t)i, ctx->crops_dev + 2 * b, 2 * sizeof(int32_t),
                     cudaMemcpyDeviceToHost, ctx->s_d2h));
  return VD3D_OK;
}

int vd3d_last_crops(vd3d_ctx* ctx, int32_t* top_bottom, int n) {
  if (!ctx || !top_bottom || n < 0) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  if (n > ctx->crops_n) return fail(ctx, VD3D_ERR_STATE, "the last clip call did not auto-crop that many frames");
  memcpy(top_bottom, ctx->crops_host, sizeof(int32_t) * 2 * (size_t)n);  // the clip call synchronised its D2H stream
  return VD3D_OK;
}

int vd3d_detect_black_bars(vd3d_ctx* ctx, const uint8_t* frame_bgr, int h, int w, int mem, int* top, int* bottom) {
  if (!ctx || !frame_bgr || !top || !bottom || h < 1 || w < 1) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const void* f_d;
  int r;
  if ((r = copy_in(ctx, ctx->in_frame[0], frame_bgr, (size_t)h * w * 3, mem, s, &f_d))) return r;
  CK(cudaMemsetAsync(ctx->detect_words, 0, 2 * sizeof(uint32_t), s));
  launch_black_bars((const uint8_t*)f_d, h, w, 10, ctx->detect_words, s);
  ctx->launches += 2;
  CK(cudaGetLastError());
  uint32_t words[2];
  CK(cudaMemcpyAsync(words, ctx->detect_words, sizeof words, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  bar_rows(h, words[0], words[1], top, bottom);
  return VD3D_OK;
}

int vd3d_render_frame(vd3d_ctx* ctx, const uint8_t* frame_bgr, const uint8_t* depth, int depth_channels,
                      int src_h, int src_w, const vd3d_render_params* rp, uint8_t* out_bgr, int mem,
                      vd3d_frame_info* info) {
  if (!ctx || !frame_bgr || !depth || !rp || !out_bgr) return fail(ctx, VD3D_ERR_ARG, "null argument");
  if (depth_channels != 1 && depth_channels != 3) return fail(ctx, VD3D_ERR_ARG, "depth_channels must be 1 or 3");
  CK(cudaSetDevice(ctx->device));
  vd3d_size_plan pl;
  int r = vd3d_plan_sizes(src_w, src_h, rp, &pl);
  if (r) return fail(ctx, r, "unsupported output format / sizes");
  cudaStream_t s = ctx->stream;
  const void *f_d, *d_d;
  size_t fb = (size_t)src_w * src_h * 3, db = (size_t)src_w * src_h * depth_channels;
  if ((r = copy_in(ctx, ctx->in_frame[0], frame_bgr, fb, mem, s, &f_d))) return r;
  if ((r = copy_in(ctx, ctx->in_depth[0], depth, db, mem, s, &d_d))) return r;
  size_t ob = out_bytes(rp, pl);
  void* o_d;
  if ((r = stage_out(ctx, ctx->out_dev[0], out_bgr, ob, mem, &o_d))) return r;
  if ((r = enqueue_frame(ctx, (const uint8_t*)f_d, (const uint8_t*)d_d, depth_channels, src_h, src_w, rp, pl,
                         (uint8_t*)o_d, 0)))
    return r;
  if (mem == VD3D_MEM_HOST) CK(cudaMemcpyAsync(out_bgr, o_d, ob, cudaMemcpyDeviceToHost, s));
  if (info) return fetch_info(ctx, info, rp->auto_crop_black_bars ? 0 : -1);
  CK(cudaStreamSynchronize(s));
  return VD3D_OK;
}

int vd3d_render_clip(vd3d_ctx* ctx, int n, const uint8_t* const* frames, const uint8_t* const* depths,
                     int depth_channels, int src_h, int src_w, const vd3d_render_params* rp,
                     uint8_t* const* outs, int mem, vd3d_frame_info* infos) {
  if (!ctx || !frames || !depths || !rp || !outs || n < 0) return fail(ctx, VD3D_ERR_ARG, "null argument");
  if (depth_channels != 1 && depth_channels != 3) return fail(ctx, VD3D_ERR_ARG, "depth_channels must be 1 or 3");
  CK(cudaSetDevice(ctx->device));
  vd3d_size_plan pl;
  int r = vd3d_plan_sizes(src_w, src_h, rp, &pl);
  if (r) return fail(ctx, r, "unsupported output format / sizes");
  size_t fb = (size_t)src_w * src_h * 3, db = (size_t)src_w * src_h * depth_channels;
  size_t ob = out_bytes(rp, pl);
  for (int b = 0; b < kSlots; ++b) {
    if ((r = ensure(ctx, ctx->in_frame[b], fb))) return r;
    if ((r = ensure(ctx, ctx->in_depth[b], db))) return r;
    if ((r = ensure(ctx, ctx->out_dev[b], ob))) return r;
  }
  if ((r = begin_crops(ctx, rp, n))) return r;
  for (int i = 0; i < n; ++i) {
    int b = i % kSlots;
    if (mem == VD3D_MEM_DEVICE) {
      // fixed staging addresses keep the frame graph replayable; D2D copies are ~1 % of a frame
      if (i >= kSlots) CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_d2h[b], 0));
      CK(cudaMemcpyAsync(ctx->in_frame[b].p, frames[i], fb, cudaMemcpyDeviceToDevice, ctx->stream));
      CK(cudaMemcpyAsync(ctx->in_depth[b].p, depths[i], db, cudaMemcpyDeviceToDevice, ctx->stream));
    } else {
      // software pipeline over three streams: H2D(i+1) | kernels(i) | D2H(i-1)
      if (i >= kSlots) CK(cudaStreamWaitEvent(ctx->s_h2d, ctx->ev_done[b], 0));
      CK(cudaMemcpyAsync(ctx->in_frame[b].p, frames[i], fb, cudaMemcpyHostToDevice, ctx->s_h2d));
      CK(cudaMemcpyAsync(ctx->in_depth[b].p, depths[i], db, cudaMemcpyHostToDevice, ctx->s_h2d));
      CK(cudaEventRecord(ctx->ev_h2d[b], ctx->s_h2d));
      CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_h2d[b], 0));
      if (i >= kSlots) CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_d2h[b], 0));
    }
    if ((r = run_frame_slot(ctx, b, depth_channels, src_h, src_w, rp, pl))) return r;
    if (infos && (r = fetch_info(ctx, &infos[i], rp->auto_crop_black_bars ? b : -1))) return r;
    CK(cudaEventRecord(ctx->ev_done[b], ctx->stream));
    CK(cudaStreamWaitEvent(ctx->s_d2h, ctx->ev_done[b], 0));
    CK(cudaMemcpyAsync(outs[i], ctx->out_dev[b].p, ob,
                       mem == VD3D_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, ctx->s_d2h));
    if ((r = copy_crop(ctx, rp, i, b))) return r;
    CK(cudaEventRecord(ctx->ev_d2h[b], ctx->s_d2h));
  }
  CK(cudaStreamSynchronize(ctx->stream));
  CK(cudaStreamSynchronize(ctx->s_d2h));
  return VD3D_OK;
}

int vd3d_render_clip_depth(vd3d_ctx* ctx, vd3d_depth* depth, int n, const uint8_t* const* frames, int src_h,
                           int src_w, const vd3d_render_params* rp, uint8_t* const* outs, int mem) {
  if (!ctx || !depth || !frames || !rp || !outs || n < 0) return fail(ctx, VD3D_ERR_ARG, "null argument");
  if (depth_family(depth) != VD3D_DEPTH_DA_V2)
    return fail(ctx, VD3D_ERR_UNSUPPORTED, "the joined depth -> stereo path serves Depth-Anything-V2 engines only");
  CK(cudaSetDevice(ctx->device));
  vd3d_size_plan pl;
  int r = vd3d_plan_sizes(src_w, src_h, rp, &pl);
  if (r) return fail(ctx, r, "unsupported output format / sizes");
  size_t fb = (size_t)src_w * src_h * 3, db = (size_t)src_w * src_h;
  size_t ob = out_bytes(rp, pl);
  for (int b = 0; b < kSlots; ++b) {
    if ((r = ensure(ctx, ctx->in_frame[b], fb))) return r;
    if ((r = ensure(ctx, ctx->in_depth[b], db))) return r;
    if ((r = ensure(ctx, ctx->out_dev[b], ob))) return r;
  }
  if ((r = begin_crops(ctx, rp, n))) return r;
  // Frames travel in groups of `depth_batch`: one batched depth forward per group on one of two engine instances
  // (group g+1's forward overlaps the neck / head tail of group g and the DIBR kernels of group g's frames), then the
  // DIBR loop body frame by frame on the main stream (sequential temporal state), D2H behind it.
  const bool serial = ctx->prof != 0;  // stage timing wants everything on one stream
  const int B = ctx->depth_batch;
  if (!serial && (r = ensure_depth_clones(ctx, depth))) return r;
  const cudaMemcpyKind kin = mem == VD3D_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  const cudaMemcpyKind kout = mem == VD3D_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  int group = 0;
  for (int i0 = 0; i0 < n; i0 += B, ++group) {
    const int nb = (n - i0) < B ? (n - i0) : B;
    const int c = group % kClones;
    const int slot0 = c * kMaxDepthBatch;
    const bool reuse = group >= kClones;  // these slots have been used before in this call
    // ---- stage the frames of the group (a slot is free once the DIBR pass that read it has finished) ----
    for (int j = 0; j < nb; ++j) {
      const int sl = slot0 + j;
      if (reuse) CK(cudaStreamWaitEvent(ctx->s_h2d, ctx->ev_done[sl], 0));
      CK(cudaMemcpyAsync(ctx->in_frame[sl].p, frames[i0 + j], fb, kin, ctx->s_h2d));
      CK(cudaEventRecord(ctx->ev_h2d[sl], ctx->s_h2d));
    }
    if (serial) {
      for (int j = 0; j < nb; ++j) CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_h2d[slot0 + j], 0));
      {
        ProfScope ps(ctx, 2);  // one sample per batch: vd3d_profile_collect divides by the frames it covered
        const uint8_t* f_d[kMaxDepthBatch];
        uint8_t* d_d[kMaxDepthBatch];
        for (int j = 0; j < nb; ++j) {
          f_d[j] = (const uint8_t*)ctx->in_frame[slot0 + j].p;
          d_d[j] = (uint8_t*)ctx->in_depth[slot0 + j].p;
        }
        if ((r = vd3d_depth_infer_batch_device(depth, nb, f_d, src_h, src_w, d_d, nullptr, 0))) {
          ctx->err = std::string("depth engine: ") + vd3d_depth_last_error(depth);
          return r;
        }
        ctx->prof_depth_frames += nb;
      }
    } else {
      cudaStream_t sd = ctx->s_depth[c];
      for (int j = 0; j < nb; ++j) {
        CK(cudaStreamWaitEvent(sd, ctx->ev_h2d[slot0 + j], 0));
        if (reuse) CK(cudaStreamWaitEvent(sd, ctx->ev_done[slot0 + j], 0));  // in_depth[slot] consumed
      }
      if ((r = run_depth_group(ctx, depth, c, slot0, nb, src_h, src_w))) return r;
      CK(cudaEventRecord(ctx->ev_depth[c], sd));
      CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_depth[c], 0));
    }
    // ---- DIBR loop body of the group's frames on the main stream ----
    for (int j = 0; j < nb; ++j) {
      const int sl = slot0 + j;
      if (reuse) CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_d2h[sl], 0));  // out_dev[slot] drained
      if ((r = run_frame_slot(ctx, sl, 1, src_h, src_w, rp, pl))) return r;
      CK(cudaEventRecord(ctx->ev_done[sl], ctx->stream));
      CK(cudaStreamWaitEvent(ctx->s_d2h, ctx->ev_done[sl], 0));
      CK(cudaMemcpyAsync(outs[i0 + j], ctx->out_dev[sl].p, ob, kout, ctx->s_d2h));
      if ((r = copy_crop(ctx, rp, i0 + j, sl))) return r;
      CK(cudaEventRecord(ctx->ev_d2h[sl], ctx->s_d2h));
    }
  }
  CK(cudaStreamSynchronize(ctx->stream));
  CK(cudaStreamSynchronize(ctx->s_d2h));
  if (!serial)
    for (int b = 0; b < kClones; ++b) CK(cudaStreamSynchronize(ctx->s_depth[b]));
  return VD3D_OK;
}

int vd3d_set_depth_batch(vd3d_ctx* ctx, int frames) {
  if (!ctx || frames < 1 || frames > kMaxDepthBatch) return fail(ctx, VD3D_ERR_ARG, "depth batch must be in [1, 8]");
  if (frames != ctx->depth_batch) {
    CK(cudaDeviceSynchronize());
    ctx->depth_batch = frames;
  }
  return VD3D_OK;
}
int vd3d_get_depth_batch(vd3d_ctx* ctx) { return ctx ? ctx->depth_batch : -1; }

// ---- exact frame sharding (SURVEY 8(e)): advance / export / import the temporal state ----------
// One loop iteration without rendering: updates TemporalDepthFilter, DepthPercentileEMA, ShiftSmoother,
// FocalDepthTracker, ConvergenceEMA, FloatingBarEaser and FloatingWindowTracker exactly as
// vd3d_render_frame would (same kernels up to the shift map), at ~1/3 of a frame's DIBR cost.
int vd3d_advance_state(vd3d_ctx* ctx, const uint8_t* frame_bgr, const uint8_t* depth, int depth_channels, int src_h,
                       int src_w, const vd3d_render_params* rp, int mem) {
  if (!ctx || !frame_bgr || !depth || !rp) return fail(ctx, VD3D_ERR_ARG, "null argument");
  if (depth_channels != 1 && depth_channels != 3) return fail(ctx, VD3D_ERR_ARG, "depth_channels must be 1 or 3");
  CK(cudaSetDevice(ctx->device));
  vd3d_size_plan pl;
  int r = vd3d_plan_sizes(src_w, src_h, rp, &pl);
  if (r) return fail(ctx, r, "unsupported output format / sizes");
  cudaStream_t s = ctx->stream;
  const void *f_d, *d_d;
  size_t fb = (size_t)src_w * src_h * 3, db = (size_t)src_w * src_h * depth_channels;
  if ((r = copy_in(ctx, ctx->in_frame[0], frame_bgr, fb, mem, s, &f_d))) return r;
  if ((r = copy_in(ctx, ctx->in_depth[0], depth, db, mem, s, &d_d))) return r;
  ctx->stats_only = 1;
  r = enqueue_frame(ctx, (const uint8_t*)f_d, (const uint8_t*)d_d, depth_channels, src_h, src_w, rp, pl, nullptr, 0);
  ctx->stats_only = 0;
  if (r) return r;
  CK(cudaStreamSynchronize(s));
  return VD3D_OK;
}

struct StateHeader {
  uint32_t magic, tw, th, reserved;
};
size_t vd3d_state_bytes(vd3d_ctx* ctx) {
  if (!ctx) return 0;
  return sizeof(StateHeader) + sizeof(DevState) + 2 * sizeof(float) * (size_t)ctx->tdf_w * ctx->tdf_h;
}
// blob = header | DevState | tdf plane | previous normalised-depth plane   (host or device memory)
int vd3d_export_state(vd3d_ctx* ctx, void* dst, size_t cap, int mem) {
  if (!ctx || !dst) return VD3D_ERR_ARG;
  size_t need = vd3d_state_bytes(ctx);
  if (cap < need) return fail(ctx, VD3D_ERR_ARG, "state buffer too small");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  cudaMemcpyKind kd = mem == VD3D_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  cudaMemcpyKind kh = mem == VD3D_MEM_HOST ? cudaMemcpyHostToHost : cudaMemcpyHostToDevice;
  StateHeader h = {0x56443344u, (uint32_t)ctx->tdf_w, (uint32_t)ctx->tdf_h, 0};
  uint8_t* p = (uint8_t*)dst;
  CK(cudaMemcpyAsync(p, &h, sizeof h, kh, s));
  CK(cudaStreamSynchronize(s));  // h is a stack object
  p += sizeof h;
  CK(cudaMemcpyAsync(p, ctx->st, sizeof(DevState), kd, s));
  p += sizeof(DevState);
  size_t plane = sizeof(float) * (size_t)ctx->tdf_w * ctx->tdf_h;
  if (plane) {
    CK(cudaMemcpyAsync(p, ctx->tdf.p, plane, kd, s));
    p += plane;
    const void* prev = ctx->frame_parity ? ctx->dn0.p : ctx->dn1.p;  // what the next frame reads as prev_depth
    CK(cudaMemcpyAsync(p, prev, plane, kd, s));
  }
  CK(cudaStreamSynchronize(s));
  return VD3D_OK;
}
int vd3d_import_state(vd3d_ctx* ctx, const void* src, size_t bytes, int mem) {
  if (!ctx || !src || bytes < sizeof(StateHeader) + sizeof(DevState)) return fail(ctx, VD3D_ERR_ARG, "bad state blob");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  cudaMemcpyKind kd = mem == VD3D_MEM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
  cudaMemcpyKind kh = mem == VD3D_MEM_HOST ? cudaMemcpyHostToHost : cudaMemcpyDeviceToHost;
  StateHeader h;
  CK(cudaMemcpyAsync(&h, src, sizeof h, kh, s));
  CK(cudaStreamSynchronize(s));
  if (h.magic != 0x56443344u) return fail(ctx, VD3D_ERR_ARG, "bad state blob magic");
  size_t plane = sizeof(float) * (size_t)h.tw * h.th;
  if (bytes < sizeof h + sizeof(DevState) + 2 * plane) return fail(ctx, VD3D_ERR_ARG, "state blob truncated");
  int r;
  if (plane) {
    if ((r = ensure(ctx, ctx->tdf, plane)) || (r = ensure(ctx, ctx->dn0, plane)) || (r = ensure(ctx, ctx->dn1, plane)))
      return r;
  }
  ctx->tdf_w = (int)h.tw;
  ctx->tdf_h = (int)h.th;
  const uint8_t* p = (const uint8_t*)src + sizeof h;
  CK(cudaMemcpyAsync(ctx->st, p, sizeof(DevState), kd, s));
  p += sizeof(DevState);
  if (plane) {
    CK(cudaMemcpyAsync(ctx->tdf.p, p, plane, kd, s));
    p += plane;
    ctx->frame_parity = 0;  // next frame writes dn0 and reads dn1 as prev_depth
    CK(cudaMemcpyAsync(ctx->dn1.p, p, plane, kd, s));
  }
  CK(cudaStreamSynchronize(s));
  drop_graphs(ctx);
  return VD3D_OK;
}

// forget the engine clones made for `depth` (call before destroying that engine)
int vd3d_release_depth(vd3d_ctx* ctx, vd3d_depth* depth) {
  if (!ctx) return VD3D_ERR_ARG;
  if (ctx->dclone_parent == depth || !depth) {
    cudaStreamSynchronize(ctx->stream);
    drop_depth_graphs(ctx);
    drop_graphs(ctx);
    for (int i = 0; i < kClones; ++i) {
      if (ctx->s_depth[i]) cudaStreamSynchronize(ctx->s_depth[i]);
      if (ctx->dclone[i]) vd3d_depth_destroy(ctx->dclone[i]);
      ctx->dclone[i] = nullptr;
    }
    ctx->dclone_parent = nullptr;
  }
  return VD3D_OK;
}

// Validate a render configuration without launching anything: sizes, eye-fit mode (builds the INTER_AREA tables it
// will need), DOF kernel bank.  render_sbs_3d calls it before it creates the output file, so that an unsupported
// configuration fails with a message instead of leaving an empty video behind.
int vd3d_check_config(vd3d_ctx* ctx, int src_h, int src_w, const vd3d_render_params* rp) {
  if (!ctx || !rp) return fail(ctx, VD3D_ERR_ARG, "null argument");
  CK(cudaSetDevice(ctx->device));
  vd3d_size_plan pl;
  int r = vd3d_plan_sizes(src_w, src_h, rp, &pl);
  if (r) return fail(ctx, r, "unsupported output format / sizes");
  if (pl.target_eye_w < 8 || pl.target_eye_h < 8 || pl.resized_width < 8 || pl.resized_height < 8)
    return fail(ctx, VD3D_ERR_ARG, "frame too small");
  if ((r = check_blur_ksize(ctx, rp->enable_feathering, rp->blur_ksize))) return r;
  FitPlan fp;
  if ((r = plan_fit(ctx, rp->output_format, pl.resized_width, pl.resized_height, pl.per_eye_w, pl.per_eye_h, fp)))
    return r;
  if (rp->dof_strength > 0.0 && (r = ensure_dof_kernels(ctx, rp->dof_strength, 5))) return r;
  return VD3D_OK;
}

// cv2.resize(u8 [h,w,ch], (ow,oh), INTER_CUBIC): the resize of the depth writer (core/render_depth.py:1917, 193; ch = 1)
// and of run_esrgan's resize chain (core/merged_pipeline.py:262-266; ch = 3)
int vd3d_resize_cubic(vd3d_ctx* ctx, const uint8_t* src, int h, int w, int ch, uint8_t* dst, int oh, int ow, int mem) {
  if (!ctx || !src || !dst || h < 1 || w < 1 || oh < 1 || ow < 1 || ch < 1 || ch > 4) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const void* s_d;
  int r;
  if ((r = copy_in(ctx, ctx->eyeL, src, (size_t)h * w * ch, mem, s, &s_d))) return r;
  void* o_d;
  if ((r = stage_out(ctx, ctx->out_dev[0], dst, (size_t)oh * ow * ch, mem, &o_d))) return r;
  if (h == oh && w == ow)
    CK(cudaMemcpyAsync(o_d, s_d, (size_t)h * w * ch, cudaMemcpyDeviceToDevice, s));  // cv2.resize copies on equal sizes
  else
    launch_resize_cubic_u8((const uint8_t*)s_d, h, w, ch, (uint8_t*)o_d, oh, ow, s);
  ctx->launches += 1;
  return stage_finish(ctx, dst, o_d, (size_t)oh * ow * ch, mem);
}

// cv2.addWeighted(a, alpha, b, 1 - alpha... any beta, 0) on n bytes (blend_images, core/merged_pipeline.py:233-238)
int vd3d_add_weighted(vd3d_ctx* ctx, const uint8_t* a, double alpha, const uint8_t* b, double beta, size_t n, uint8_t* dst,
                      int mem) {
  if (!ctx || !a || !b || !dst || !n) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const void *a_d, *b_d;
  int r;
  if ((r = copy_in(ctx, ctx->eyeL, a, n, mem, s, &a_d)) || (r = copy_in(ctx, ctx->eyeR, b, n, mem, s, &b_d))) return r;
  void* o_d;
  if ((r = stage_out(ctx, ctx->out_dev[0], dst, n, mem, &o_d))) return r;
  launch_add_weighted((const uint8_t*)a_d, (float)alpha, (const uint8_t*)b_d, (float)beta, (uint8_t*)o_d, n, s);
  ctx->launches += 1;
  return stage_finish(ctx, dst, o_d, n, mem);
}

// run_esrgan (core/merged_pipeline.py:240-267) without tiling on n frames.  Per frame, on ctx->stream: the input resize
// (247-249), the network, k_sr_tail_cubic from the last conv straight to the size of the first non-identity INTER_CUBIC
// resize of 263-264, the remaining INTER_CUBIC resizes (264-266) and addWeighted (233-238).  The chain never needs the
// 4h x 4w image: the reference's 4x resize is the identity for scale 4, and its next resize reads each of those pixels
// through 16 taps that k_sr_tail_cubic computes from the conv output.
int vd3d_sr_upscale(vd3d_ctx* ctx, vd3d_depth* sr, int n, const uint8_t* const* frames, int h, int w, int num_conv,
                    const vd3d_upscale_params* p, uint8_t* const* outs, int mem) {
  if (!ctx || !sr || !frames || !p || !outs || n < 0 || h < 1 || w < 1) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  if (sr_stream(sr) != ctx->stream) return fail(ctx, VD3D_ERR_ARG, "the SR engine must be created on vd3d_stream(ctx)");
  if (p->scale != 4 && p->scale != 2) return fail(ctx, VD3D_ERR_ARG, "scale must be 4 or 2");
  if (p->target_w < 0 || p->target_h < 0 || (p->target_w == 0) != (p->target_h == 0))
    return fail(ctx, VD3D_ERR_ARG, "target size: both positive, or both 0 for none");
  const double pct = p->input_res_pct;
  int rw = w, rh = h;  // network input: int(w * input_res_pct / 100) in double, as the reference computes it
  if (pct != 100.0) {
    rw = (int)((double)w * pct / 100.0);
    rh = (int)((double)h * pct / 100.0);
  }
  if (rw < 8 || rh < 8) return fail(ctx, VD3D_ERR_ARG, "network input below 8 x 8 pixels");
  const int t1w = p->scale == 4 ? w : 2 * rw, t1h = p->scale == 4 ? h : 2 * rh;  // k_sr_tail_cubic output
  const bool to_orig = t1w != w || t1h != h;                                     // scale 2: then to the original size
  const int fw = p->target_w ? p->target_w : w, fh = p->target_h ? p->target_h : h;
  const bool to_target = fw != w || fh != h;
  const bool blend = p->blend_alpha >= 0.0;
  if (blend && to_target) return fail(ctx, VD3D_ERR_ARG, "blend of two different sizes (cv2.addWeighted raises)");
  int nst = 1 + (int)to_orig + (int)to_target + (int)blend;  // kernels after the network
  size_t tb = (size_t)(t1w * t1h > w * h ? t1w * t1h : w * h) * 3;
  // RRDBNet engine: postprocess_esr of the network output [ns rh, ns rw], then the reference's INTER_CUBIC resizes to
  // (scale rw, scale rh), to (w, h) and to the target one by one, same-size ones skipped (cv2 copies)
  const int ns = sr_net_scale(sr);
  int chain_h[3], chain_w[3], nres = 0;
  if (ns) {
    int ch = ns * rh, cw = ns * rw;
    tb = (size_t)ch * cw * 3;
    const int want_h[3] = {p->scale * rh, h, fh}, want_w[3] = {p->scale * rw, w, fw};
    for (int q = 0; q < 3; ++q) {
      if (want_h[q] == ch && want_w[q] == cw) continue;
      ch = chain_h[nres] = want_h[q];
      cw = chain_w[nres++] = want_w[q];
      if ((size_t)ch * cw * 3 > tb) tb = (size_t)ch * cw * 3;
    }
    nst = 1 + nres + (int)blend;
  }
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  int r;
  FitPlan fp;
  if (pct < 100.0 && (r = plan_fit(ctx, VD3D_FMT_HALF_SBS, w, h, rw, rh, fp, 1))) return r;
  const size_t fb = (size_t)h * w * 3, ob = (size_t)fh * fw * 3;
  void *rs = nullptr, *tmp[2] = {nullptr, nullptr};
  if (pct != 100.0 && (r = sr_buffer(sr, "up.in", (size_t)rw * rh * 3, &rs))) return r;
  if (nst > 1 && (r = sr_buffer(sr, "up.0", tb, &tmp[0]))) return r;
  if (nst > 2 && (r = sr_buffer(sr, "up.1", tb, &tmp[1]))) return r;
  if (mem == VD3D_MEM_HOST)
    for (int b = 0; b < kSrSlots; ++b)
      if ((r = ensure(ctx, ctx->sr_in[b], fb)) || (r = ensure(ctx, ctx->sr_out[b], ob))) return r;
  for (int i = 0; i < n; ++i) {
    const int b = i % kSrSlots;
    const uint8_t* f_d = frames[i];
    uint8_t* o_d = outs[i];
    if (mem == VD3D_MEM_HOST) {  // three streams: H2D(i+1) | kernels(i) | D2H(i-1)
      if (i >= kSrSlots) CK(cudaStreamWaitEvent(ctx->s_h2d, ctx->ev_done[b], 0));
      CK(cudaMemcpyAsync(ctx->sr_in[b].p, frames[i], fb, cudaMemcpyHostToDevice, ctx->s_h2d));
      CK(cudaEventRecord(ctx->ev_h2d[b], ctx->s_h2d));
      CK(cudaStreamWaitEvent(s, ctx->ev_h2d[b], 0));
      if (i >= kSrSlots) CK(cudaStreamWaitEvent(s, ctx->ev_d2h[b], 0));
      f_d = (const uint8_t*)ctx->sr_in[b].p;
      o_d = (uint8_t*)ctx->sr_out[b].p;
    }
    const uint8_t* x = f_d;
    if (pct < 100.0) {
      PostArgs pa = single_eye_post(f_d, h, w, (uint8_t*)rs, rw, rh);
      set_fit(pa, fp);
      launch_post(pa, s);
      ctx->launches += 1;
      x = (const uint8_t*)rs;
    } else if (pct > 100.0) {
      launch_resize_cubic_u8(f_d, h, w, 3, (uint8_t*)rs, rh, rw, s);
      ctx->launches += 1;
      x = (const uint8_t*)rs;
    }
    const float* cv;
    if ((r = ns ? rrdb_network(sr, x, rh, rw, &cv) : sr_network(sr, x, rh, rw, num_conv, &cv))) {
      ctx->err = std::string("SR engine: ") + vd3d_depth_last_error(sr);
      return r;
    }
    int k = 0;
    auto next = [&]() { return ++k == nst ? o_d : (uint8_t*)tmp[(k - 1) & 1]; };
    uint8_t* cur = next();
    if (ns) {
      launch_rrdb_out(cv, 32, cur, (size_t)ns * rh * ns * rw, s);
      int ch = ns * rh, cw = ns * rw;
      for (int q = 0; q < nres; ++q) {
        uint8_t* d = next();
        launch_resize_cubic_u8(cur, ch, cw, 3, d, chain_h[q], chain_w[q], s);
        cur = d;
        ch = chain_h[q];
        cw = chain_w[q];
      }
    } else {
      launch_sr_tail_cubic(cv, x, rh, rw, cur, t1h, t1w, s);
    }
    if (!ns && to_orig) {
      uint8_t* d = next();
      launch_resize_cubic_u8(cur, t1h, t1w, 3, d, h, w, s);
      cur = d;
    }
    if (!ns && to_target) {
      uint8_t* d = next();
      launch_resize_cubic_u8(cur, h, w, 3, d, fh, fw, s);
      cur = d;
    }
    if (blend)
      launch_add_weighted(cur, (float)p->blend_alpha, f_d, (float)(1.0 - p->blend_alpha), next(), fb, s);
    ctx->launches += nst;
    if (mem == VD3D_MEM_HOST) {
      CK(cudaEventRecord(ctx->ev_done[b], s));
      CK(cudaStreamWaitEvent(ctx->s_d2h, ctx->ev_done[b], 0));
      CK(cudaMemcpyAsync(outs[i], o_d, ob, cudaMemcpyDeviceToHost, ctx->s_d2h));
      CK(cudaEventRecord(ctx->ev_d2h[b], ctx->s_d2h));
    }
  }
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(s));
  CK(cudaStreamSynchronize(ctx->s_d2h));
  return VD3D_OK;
}

// apply_color_grade (core/render_3d.py:734-767) on f32 RGB planes [3,h,w] in 0..1
int vd3d_color_grade(vd3d_ctx* ctx, const float* rgb, int h, int w, double sat, double con, double bri, float* out,
                     int mem) {
  if (!ctx || !rgb || !out || h < 1 || w < 1) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  size_t bytes = sizeof(float) * 3 * (size_t)h * w;
  const void* r_d;
  int r;
  if ((r = copy_in(ctx, ctx->in_rgbf, rgb, bytes, mem, s, &r_d))) return r;
  void* o_d;
  if ((r = stage_out(ctx, ctx->frameB, out, bytes, mem, &o_d))) return r;
  launch_grade_f32((const float*)r_d, (float*)o_d, h * w, (float)sat, (float)con, (float)bri, s);
  ctx->launches += 1;
  return stage_finish(ctx, out, o_d, bytes, mem);
}

int vd3d_sharpen(vd3d_ctx* ctx, const uint8_t* src, int h, int w, double factor, uint8_t* dst, int mem) {
  if (!ctx || !src || !dst || h < 2 || w < 2) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  size_t bytes = (size_t)h * w * 3;
  const void* s_d;
  int r;
  if ((r = copy_in(ctx, ctx->eyeL, src, bytes, mem, s, &s_d))) return r;
  void* o_d;
  if ((r = stage_out(ctx, ctx->out_dev[0], dst, bytes, mem, &o_d))) return r;
  PostArgs pa = single_eye_post(s_d, h, w, (uint8_t*)o_d, w, h);
  pa.sharpen = 1;
  sharpen_coeffs(factor, pa.kc, pa.ke);
  launch_post(pa, s);
  ctx->launches += 1;
  return stage_finish(ctx, dst, o_d, bytes, mem);
}

// heal_missing_pixels (core/render_3d.py:431-459) on f32 RGB planes [3,h,w]; edge_mask [h,w] or null
int vd3d_heal(vd3d_ctx* ctx, const float* warped, const float* original, const float* edge_mask, int h, int w,
              double heal_strength, float* out, int mem) {
  if (!ctx || !warped || !original || !out || h < 1 || w < 1) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  size_t bytes = sizeof(float) * 3 * (size_t)h * w;
  const void *w_d, *o_d, *e_d = nullptr;
  int r;
  if ((r = copy_in(ctx, ctx->in_rgbf, warped, bytes, mem, s, &w_d))) return r;
  if ((r = copy_in(ctx, ctx->frameB, original, bytes, mem, s, &o_d))) return r;
  if (edge_mask && (r = copy_in(ctx, ctx->in_depthf, edge_mask, bytes / 3, mem, s, &e_d))) return r;
  void* out_d;
  if ((r = stage_out(ctx, ctx->rgb_s, out, bytes, mem, &out_d))) return r;
  launch_heal((const float*)w_d, (const float*)o_d, (const float*)e_d, (float*)out_d, h, w, (float)heal_strength, s);
  ctx->launches += 1;
  return stage_finish(ctx, out, out_d, bytes, mem);
}

// format_3d_output / generate_anaglyph_3d (core/render_3d.py:837-883) on two same-size u8 BGR eyes
int vd3d_pack(vd3d_ctx* ctx, const uint8_t* left, const uint8_t* right, int h, int w, int fmt, uint8_t* dst, int mem) {
  if (!ctx || !left || !right || !dst || h < 1 || w < 1) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  if (fmt < VD3D_FMT_HALF_SBS || fmt > VD3D_FMT_VR) return fail(ctx, VD3D_ERR_UNSUPPORTED, "format");
  // VR: format_3d_output resizes each eye to 1440x1600 (846-849); the render loop hands it eyes that already have that
  // size (pad_to_aspect_ratio, 1415-1417), where cv2.resize is the identity.  Other sizes (INTER_LINEAR) are off-path.
  if (fmt == VD3D_FMT_VR && (w != 1440 || h != 1600))
    return fail(ctx, VD3D_ERR_UNSUPPORTED, "VR pack expects 1440x1600 eyes (pad_to_aspect_ratio output)");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  size_t bytes = (size_t)h * w * 3;
  bool sbs = (fmt == VD3D_FMT_HALF_SBS || fmt == VD3D_FMT_FULL_SBS || fmt == VD3D_FMT_VR);
  size_t obytes = sbs ? bytes * 2 : bytes;
  const void *l_d, *r_d;
  int r;
  if ((r = copy_in(ctx, ctx->eyeL, left, bytes, mem, s, &l_d))) return r;
  if ((r = copy_in(ctx, ctx->eyeR, right, bytes, mem, s, &r_d))) return r;
  void* o_d;
  if ((r = stage_out(ctx, ctx->out_dev[0], dst, obytes, mem, &o_d))) return r;
  PostArgs pa;
  memset(&pa, 0, sizeof pa);
  pa.left = (const uint8_t*)l_d;
  pa.right = (const uint8_t*)r_d;
  pa.H = h;
  pa.W = w;
  pa.fmt = fmt;
  pa.per_eye_w = w;
  pa.per_eye_h = h;
  pa.fit_w = w;
  pa.fit_h = h;
  pa.sx = pa.sy = 1;
  pa.inv_area = 1.f;
  pa.out = (uint8_t*)o_d;
  pa.out_w = sbs ? 2 * w : w;
  pa.out_h = h;
  launch_post(pa, s);
  ctx->launches += 1;
  return stage_finish(ctx, dst, o_d, obytes, mem);
}

// eye fit on one u8 BGR image: keep_aspect != 0 -> pad_to_aspect_ratio(image, target_w, target_h) with a black canvas
// (core/render_3d.py:101-131); 0 -> cv2.resize(image, (target_w, target_h), interpolation=cv2.INTER_AREA) (1413-1414).
// INTER_AREA shrinking only (identity, integer "area fast", or cv2's general ResizeArea_ tables).
int vd3d_fit_eye(vd3d_ctx* ctx, const uint8_t* src, int h, int w, int target_w, int target_h, int keep_aspect,
                 uint8_t* dst, int mem) {
  if (!ctx || !src || !dst || h < 1 || w < 1 || target_w < 1 || target_h < 1) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const size_t bytes = (size_t)h * w * 3, obytes = (size_t)target_h * target_w * 3;
  const void* s_d;
  int r;
  if ((r = copy_in(ctx, ctx->eyeL, src, bytes, mem, s, &s_d))) return r;
  void* o_d;
  if ((r = stage_out(ctx, ctx->out_dev[0], dst, obytes, mem, &o_d))) return r;
  FitPlan fp;
  if ((r = plan_fit(ctx, keep_aspect ? VD3D_FMT_FULL_SBS : VD3D_FMT_HALF_SBS, w, h, target_w, target_h, fp, 1))) return r;
  PostArgs pa = single_eye_post(s_d, h, w, (uint8_t*)o_d, target_w, target_h);
  set_fit(pa, fp);
  launch_post(pa, s);
  ctx->launches += 1;
  return stage_finish(ctx, dst, o_d, obytes, mem);
}

// host-only test hook: the cv2 computeResizeAreaTab restatement used by the fractional INTER_AREA fit.
// ofs/cnt [dsize], alpha [dsize * cap] (zero padded); returns the largest tap count, or a negative error.
int vd3d_area_table(int ssize, int dsize, int* ofs, int* cnt, float* alpha, int cap) {
  if (ssize < 1 || dsize < 1 || dsize > ssize || !ofs || !cnt || !alpha || cap < 1) return VD3D_ERR_ARG;
  std::vector<int> o, c;
  std::vector<std::vector<float>> a;
  area_axis_tab(ssize, dsize, o, c, a);
  int T = 0;
  for (int i = 0; i < dsize; ++i) {
    if (c[i] > cap) return VD3D_ERR_ARG;
    T = c[i] > T ? c[i] : T;
    ofs[i] = o[i];
    cnt[i] = c[i];
    for (int k = 0; k < cap; ++k) alpha[(size_t)i * cap + k] = k < c[i] ? a[i][k] : 0.f;
  }
  return T;
}

// host-only test hook: the fixed-point bilinear tables of cv2's INTER_AREA emulation for an enlarged axis
int vd3d_area_linear_table(int ssize, int dsize, int* ofs, int* a01) {
  if (ssize < 1 || dsize < 1 || !ofs || !a01) return VD3D_ERR_ARG;
  std::vector<int> o, a;
  area_linear_tab(ssize, dsize, o, a);
  memcpy(ofs, o.data(), (size_t)dsize * sizeof(int));
  memcpy(a01, a.data(), (size_t)2 * dsize * sizeof(int));
  return VD3D_OK;
}

int vd3d_dof_grade(vd3d_ctx* ctx, const uint8_t* eye_bgr, int h, int w, const float* depth01, int dh, int dw,
                   double focal, double max_sigma, double sat, double con, double bri, uint8_t* dst, int mem) {
  if (!ctx || !eye_bgr || !dst || h < 2 || w < 2) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  size_t bytes = (size_t)h * w * 3;
  const void *s_d, *dp_d = nullptr;
  int r;
  if ((r = copy_in(ctx, ctx->eyeL, eye_bgr, bytes, mem, s, &s_d))) return r;
  bool dof = max_sigma > 0.0;
  if (dof) {
    if (!depth01) return fail(ctx, VD3D_ERR_ARG, "depth required for DOF");
    if ((r = copy_in(ctx, ctx->in_depthf, depth01, sizeof(float) * (size_t)dh * dw, mem, s, &dp_d))) return r;
    if ((r = ensure_dof_kernels(ctx, max_sigma, 5))) return r;
  }
  void* o_d;
  if ((r = stage_out(ctx, ctx->out_dev[0], dst, bytes, mem, &o_d))) return r;
  DofArgs da = dof_args(ctx, dof ? 5 : 1, h, w, (const float*)dp_d, dh, dw, sat, con, bri);
  da.src_l = da.src_r = (const uint8_t*)s_d;
  da.dst_l = da.dst_r = (uint8_t*)o_d;
  da.focal = (float)focal;
  launch_dof(da, 1, s);
  ctx->launches += 1;
  return stage_finish(ctx, dst, o_d, bytes, mem);
}

// ---- letterbox tracker (core/render_depth.py:273-573) and depth re-pad (1919-1933); kernels in letterbox.cu ----

// cv2.Canny's integer thresholds with L2gradient: clamp to 32767, square, floor; low > high is swapped
static void canny_thresholds(double low, double high, int* low2, int* high2) {
  if (low > high) {
    const double t = low;
    low = high;
    high = t;
  }
  low = fmin(32767.0, low);
  high = fmin(32767.0, high);
  if (low > 0) low *= low;
  if (high > 0) high *= high;
  *low2 = (int)floor(low);
  *high2 = (int)floor(high);
}

static int lb_canny_scratch(vd3d_ctx* ctx, size_t npx) {
  int r;
  if ((r = ensure(ctx, ctx->lb_mag, npx * 4)) || (r = ensure(ctx, ctx->lb_label, npx * 4)) ||
      (r = ensure(ctx, ctx->lb_flag, npx * 2)))
    return r;
  return VD3D_OK;
}

int vd3d_canny_u8(vd3d_ctx* ctx, const uint8_t* gray, int h, int w, double low, double high, uint8_t* dst, int mem) {
  if (!ctx || !gray || !dst || h < 1 || w < 1 || (size_t)h * w >= (1u << 31)) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const size_t npx = (size_t)h * w;
  const void* g_d;
  void* o_d;
  int r;
  if ((r = copy_in(ctx, ctx->lb_prev, gray, npx, mem, s, &g_d))) return r;
  if ((r = stage_out(ctx, ctx->lb_out, dst, npx, mem, &o_d))) return r;
  if ((r = lb_canny_scratch(ctx, npx))) return r;
  int low2, high2;
  canny_thresholds(low, high, &low2, &high2);
  launch_canny((const uint8_t*)g_d, 1, h, w, low2, high2, (int32_t*)ctx->lb_mag.p, (int32_t*)ctx->lb_label.p,
               (uint8_t*)ctx->lb_flag.p, (uint8_t*)o_d, nullptr, s);
  ctx->launches += 5;
  return stage_finish(ctx, dst, o_d, npx, mem);
}

int vd3d_letterbox_stats(vd3d_ctx* ctx, int n, const uint8_t* frames, int h, int w, const uint8_t* prev_gray, int mem,
                         float* row_y_mean, float* row_y_var, float* row_s_mean, int32_t* row_edges,
                         float* frame_y_mean, uint32_t* frame_hist, uint64_t* frame_absdiff, uint8_t* last_gray) {
  if (!ctx || !frames || n < 1 || h < 1 || w < 1 || w > 8192 || !row_y_mean || !row_y_var || !row_s_mean ||
      !row_edges || !frame_y_mean || !frame_hist || !frame_absdiff)
    return fail(ctx, VD3D_ERR_ARG, "bad argument (frames of 1..8192 columns, every record pointer set)");
  const size_t npix = (size_t)h * w, npx = npix * n, rows = (size_t)h * n;
  if (npx >= (1u << 31)) return fail(ctx, VD3D_ERR_ARG, "n * h * w must stay below 2^31");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const void *f_d, *p_d = nullptr;
  int r;
  if ((r = copy_in(ctx, ctx->lb_in, frames, npx * 3, mem, s, &f_d))) return r;
  if (prev_gray && (r = copy_in(ctx, ctx->lb_prev, prev_gray, npix, mem, s, &p_d))) return r;
  if ((r = ensure(ctx, ctx->lb_gray, npx)) || (r = lb_canny_scratch(ctx, npx))) return r;
  if (ctx->lb_nodes_npix != (int64_t)npix) {
    int cnt = 0;
    lb_cut_nodes((int64_t)npix, nullptr, nullptr, &cnt, 0);
    std::vector<int64_t> st(cnt);
    std::vector<int> ln(cnt);
    lb_cut_nodes((int64_t)npix, st.data(), ln.data(), &cnt, cnt);
    if ((r = ensure(ctx, ctx->lb_nodes, (size_t)cnt * 12))) return r;
    CK(cudaMemcpyAsync(ctx->lb_nodes.p, st.data(), (size_t)cnt * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync((char*)ctx->lb_nodes.p + (size_t)cnt * 8, ln.data(), (size_t)cnt * 4, cudaMemcpyHostToDevice, s));
    CK(cudaStreamSynchronize(s));
    ctx->lb_nodes_npix = (int64_t)npix;
    ctx->lb_nodes_n = cnt;
  }
  const int nodes = ctx->lb_nodes_n;
  if ((r = ensure(ctx, ctx->lb_node_sum, (size_t)nodes * n * 4))) return r;
  // one record block, one D2H: absdiff u64 [n] | y_mean, y_var, s_mean f32 [rows] | edges i32 [rows] | hist u32 [n,64]
  // | frame y_mean f32 [n]
  const size_t o_mean = 8 * (size_t)n, o_var = o_mean + 4 * rows, o_sat = o_var + 4 * rows, o_edge = o_sat + 4 * rows,
               o_hist = o_edge + 4 * rows, o_fmean = o_hist + 256 * (size_t)n, rec = o_fmean + 4 * (size_t)n;
  if ((r = ensure(ctx, ctx->lb_rec, rec))) return r;
  char* R = (char*)ctx->lb_rec.p;
  CK(cudaMemsetAsync(R, 0, rec, s));
  LbRowArgs a;
  a.frames = (const uint8_t*)f_d;
  a.prev_gray = (const uint8_t*)p_d;
  a.n = n;
  a.h = h;
  a.w = w;
  a.gray = (uint8_t*)ctx->lb_gray.p;
  a.y_mean = (float*)(R + o_mean);
  a.y_var = (float*)(R + o_var);
  a.s_mean = (float*)(R + o_sat);
  a.hist = (uint32_t*)(R + o_hist);
  a.absdiff = (unsigned long long*)R;
  launch_lb_rows(a, s);
  launch_lb_frame_mean(a.frames, n, (int64_t)npix, (const int64_t*)ctx->lb_nodes.p,
                       (const int*)((char*)ctx->lb_nodes.p + (size_t)nodes * 8), nodes, (float*)ctx->lb_node_sum.p,
                       (float*)(R + o_fmean), s);
  launch_canny(a.gray, n, h, w, 900, 8100, (int32_t*)ctx->lb_mag.p, (int32_t*)ctx->lb_label.p,
               (uint8_t*)ctx->lb_flag.p, nullptr, (int32_t*)(R + o_edge), s);
  ctx->launches += 8;
  CK(cudaGetLastError());
  std::vector<char> host(rec);
  CK(cudaMemcpyAsync(host.data(), R, rec, cudaMemcpyDeviceToHost, s));
  if (last_gray)
    CK(cudaMemcpyAsync(last_gray, a.gray + npix * (n - 1), npix,
                       mem == VD3D_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, s));
  CK(cudaStreamSynchronize(s));
  memcpy(frame_absdiff, host.data(), 8 * (size_t)n);
  memcpy(row_y_mean, host.data() + o_mean, 4 * rows);
  memcpy(row_y_var, host.data() + o_var, 4 * rows);
  memcpy(row_s_mean, host.data() + o_sat, 4 * rows);
  memcpy(row_edges, host.data() + o_edge, 4 * rows);
  memcpy(frame_hist, host.data() + o_hist, 256 * (size_t)n);
  memcpy(frame_y_mean, host.data() + o_fmean, 4 * (size_t)n);
  return VD3D_OK;
}

int vd3d_letterbox_repad(vd3d_ctx* ctx, const uint8_t* src, int h, int w, int top, int bottom, uint8_t* dst, int mem) {
  if (!ctx || !src || !dst || h < 1 || w < 1 || top < 0 || bottom < 0) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  if (mem == VD3D_MEM_DEVICE && src == dst) return fail(ctx, VD3D_ERR_ARG, "src and dst must not alias");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const size_t npx = (size_t)h * w;
  const void* s_d;
  void* o_d;
  int r;
  if ((r = copy_in(ctx, ctx->lb_prev, src, npx, mem, s, &s_d))) return r;
  if ((r = stage_out(ctx, ctx->lb_out, dst, npx, mem, &o_d))) return r;
  const int core_h = h - top - bottom;
  if ((top == 0 && bottom == 0) || core_h <= 0) {
    // no bars, or the reference's fallback (bars dropped, core = the whole frame): cv2.resize to the same size copies
    CK(cudaMemcpyAsync(o_d, s_d, npx, cudaMemcpyDeviceToDevice, s));
    ctx->launches += 1;
  } else {
    if ((r = ensure(ctx, ctx->lb_hist, 256 * 4))) return r;
    CK(cudaMemsetAsync(ctx->lb_hist.p, 0, 256 * 4, s));
    launch_resize_cubic_u8((const uint8_t*)s_d, h, w, 1, (uint8_t*)o_d + (size_t)top * w, core_h, w, s);
    launch_lb_pad((uint8_t*)o_d, h, w, top, core_h, (uint32_t*)ctx->lb_hist.p, s);
    ctx->launches += 4;
  }
  return stage_finish(ctx, dst, o_d, npx, mem);
}

}  // extern "C"

// ===========================================================================
// tiled depth inference (core/render_depth.py:102-194)
// ===========================================================================
namespace {

int r14(int v) { return (v + 13) / 14 * 14; }

// the plan infer_depth_tile walks for an [h,w] image: tiles must be exactly it.  n_classes > 0 also checks that every
// tile names a class and that the tiles of one class share their rounded size.
int check_plan(vd3d_ctx* ctx, int h, int w, int tile, int pad, const vd3d_tile* tiles, int n_tiles, int n_classes,
               int* step, int* nx, int* ny) {
  if (h < 1 || w < 1 || tile < 1 || pad < 0 || !tiles) return fail(ctx, VD3D_ERR_ARG, "bad tile plan argument");
  const int core = tile - 2 * pad > 1 ? tile - 2 * pad : 1;
  *step = core;
  *nx = (w + core - 1) / core;
  *ny = (h + core - 1) / core;
  if (n_tiles != *nx * *ny) return fail(ctx, VD3D_ERR_ARG, "tile count does not match the plan");
  std::vector<int> cls_h(n_classes > 0 ? n_classes : 0, -1), cls_w(cls_h.size(), -1);
  for (int i = 0; i < *ny; ++i)
    for (int j = 0; j < *nx; ++j) {
      const vd3d_tile& t = tiles[i * *nx + j];
      const int y0 = i * core, x0 = j * core, y1 = std::min(y0 + tile, h), x1 = std::min(x0 + tile, w);
      const int yp0 = std::max(0, y0 - pad), xp0 = std::max(0, x0 - pad);
      const int yp1 = std::min(h, y1 + pad), xp1 = std::min(w, x1 + pad);
      if (t.y0 != y0 || t.y1 != y1 || t.x0 != x0 || t.x1 != x1 || t.yp0 != yp0 || t.yp1 != yp1 || t.xp0 != xp0 ||
          t.xp1 != xp1 || t.rh != r14(yp1 - yp0) || t.rw != r14(xp1 - xp0))
        return fail(ctx, VD3D_ERR_ARG, "tile does not match the plan");
      if (n_classes > 0) {
        if (t.cls < 0 || t.cls >= n_classes) return fail(ctx, VD3D_ERR_ARG, "tile class out of range");
        if (cls_h[t.cls] < 0) {
          cls_h[t.cls] = t.rh;
          cls_w[t.cls] = t.rw;
        } else if (cls_h[t.cls] != t.rh || cls_w[t.cls] != t.rw) {
          return fail(ctx, VD3D_ERR_ARG, "tiles of one class differ in size");
        }
      }
    }
  return VD3D_OK;
}

// jobs of n frames (frame-major, plan order); crops and predictions are packed per frame at the offsets of the plan
void tile_jobs(const uint8_t* const* frames, int n, const vd3d_tile* tiles, int n_tiles, uint8_t* crops,
               float* preds, const float* const* weights, std::vector<TileJob>& jobs, size_t* crop_bytes,
               size_t* pred_count) {
  size_t cb = 0, pc = 0;
  for (int t = 0; t < n_tiles; ++t) {
    cb += (size_t)tiles[t].rh * tiles[t].rw * 3;
    pc += (size_t)tiles[t].rh * tiles[t].rw;
  }
  *crop_bytes = cb;
  *pred_count = pc;
  jobs.resize((size_t)n * n_tiles);
  for (int f = 0; f < n; ++f) {
    size_t co = cb * f, po = pc * f;
    for (int t = 0; t < n_tiles; ++t) {
      const vd3d_tile& s = tiles[t];
      TileJob& j = jobs[(size_t)f * n_tiles + t];
      j.frame = frames ? frames[f] : nullptr;
      j.crop = crops ? crops + co : nullptr;
      j.pred = preds ? preds + po : nullptr;
      j.wgt = weights ? weights[t] : nullptr;
      j.y0 = s.y0;
      j.x0 = s.x0;
      j.ch = s.y1 - s.y0;
      j.cw = s.x1 - s.x0;
      j.yp0 = s.yp0;
      j.xp0 = s.xp0;
      j.pch = s.yp1 - s.yp0;
      j.pcw = s.xp1 - s.xp0;
      j.rh = s.rh;
      j.rw = s.rw;
      co += (size_t)s.rh * s.rw * 3;
      po += (size_t)s.rh * s.rw;
    }
  }
}

int upload_jobs(vd3d_ctx* ctx, const std::vector<TileJob>& jobs, const TileJob** dev) {
  int r;
  if ((r = ensure(ctx, ctx->td_jobs, jobs.size() * sizeof(TileJob)))) return r;
  // pageable source: the copy is staged before cudaMemcpyAsync returns, so `jobs` may go out of scope afterwards
  CK(cudaMemcpyAsync(ctx->td_jobs.p, jobs.data(), jobs.size() * sizeof(TileJob), cudaMemcpyHostToDevice, ctx->stream));
  *dev = (const TileJob*)ctx->td_jobs.p;
  return VD3D_OK;
}

void gather(vd3d_ctx* ctx, const TileJob* jobs_dev, const vd3d_tile* tiles, int n_tiles, int njobs, int w) {
  int mh = 0, mw = 0;
  for (int t = 0; t < n_tiles; ++t) {
    mh = std::max(mh, tiles[t].rh);
    mw = std::max(mw, tiles[t].rw);
  }
  launch_tile_gather(jobs_dev, njobs, mh, mw, w, ctx->stream);
  ctx->launches += 1;
}

// numpy's percentile bookkeeping for a plane of npix values (numpy 2.x, float32 data): q = float32(p) / float32(100),
// virtual index float32(npix - 1) * q in float32, neighbours floor(v) and floor(v) + 1 (both the last element when
// v >= npix - 1), gamma = v - floor(v) in float32
void pct_targets(int64_t npix, double p, uint32_t* k0, uint32_t* k1, float* gamma) {
  const float q = (float)p / 100.0f;
  const float nm1 = (float)(npix - 1);
  const float v = nm1 * q;
  if (v >= nm1) {
    *k0 = *k1 = (uint32_t)(npix - 1);
    *gamma = (float)((double)v + 1.0);  // gamma against the index -1 numpy substitutes; b - a is 0 there
    return;
  }
  const float fl = floorf(v);
  *k0 = (uint32_t)fl;
  *k1 = (uint32_t)std::min<int64_t>((int64_t)fl + 1, npix - 1);
  *gamma = v - fl;
}

// _normalize_to_u8 of n planes at d_dev [n, h*w] -> outs[f] [oh, ow] (device); stats_host (optional) [n, 4]
int normalize_planes(vd3d_ctx* ctx, const float* d_dev, int n, int h, int w, double p_lo, double p_hi, int invert,
                     uint8_t* const* outs, int oh, int ow, float* stats_host) {
  cudaStream_t s = ctx->stream;
  const int64_t npix = (int64_t)h * w;
  if (npix > 0xffffffffLL) return fail(ctx, VD3D_ERR_ARG, "plane too large");
  NormArgs a;
  pct_targets(npix, p_lo, &a.rank[0], &a.rank[1], &a.gamma_lo);
  pct_targets(npix, p_hi, &a.rank[2], &a.rank[3], &a.gamma_hi);
  a.rank[4] = 0;
  a.rank[5] = (uint32_t)(npix - 1);
  a.invert = invert ? 1 : 0;
  int r;
  if ((r = ensure(ctx, ctx->td_sel, (size_t)n * normalize_scratch_words() * 4)) ||
      (r = ensure(ctx, ctx->td_u8, (size_t)n * npix)) || (r = ensure(ctx, ctx->td_stats, (size_t)n * 16)))
    return r;
  launch_normalize_u8(d_dev, n, npix, a, (uint32_t*)ctx->td_sel.p, (uint8_t*)ctx->td_u8.p,
                      stats_host ? (float*)ctx->td_stats.p : nullptr, s);
  ctx->launches += 10;  // four histogram + pick passes, the scalars, the u8 write
  for (int f = 0; f < n; ++f) {
    const uint8_t* u = (const uint8_t*)ctx->td_u8.p + (size_t)f * npix;
    if (oh == h && ow == w)
      CK(cudaMemcpyAsync(outs[f], u, npix, cudaMemcpyDeviceToDevice, s));  // cv2.resize copies on equal sizes
    else
      launch_resize_cubic_u8(u, h, w, 1, outs[f], oh, ow, s);
    ctx->launches += 1;
  }
  if (stats_host) CK(cudaMemcpyAsync(stats_host, ctx->td_stats.p, (size_t)n * 16, cudaMemcpyDeviceToHost, s));
  return VD3D_OK;
}

// blend of n frames from the jobs at jobs_dev into ctx->td_depth [n, h, w]; minmax_host (optional) [n, 2]
int blend_frames(vd3d_ctx* ctx, const TileJob* jobs_dev, int n, int h, int w, int tile, int step, int nx, int ny,
                 float* minmax_host) {
  cudaStream_t s = ctx->stream;
  int r;
  if ((r = ensure(ctx, ctx->td_depth, (size_t)n * h * w * 4)) || (r = ensure(ctx, ctx->td_mm, (size_t)n * 16)))
    return r;
  uint32_t* keys = (uint32_t*)ctx->td_mm.p;
  launch_tile_blend(jobs_dev, n, h, w, step, tile, nx, ny, (float*)ctx->td_depth.p, keys, s);
  ctx->launches += 2;
  if (minmax_host) {
    float* mmf = (float*)(keys + 2 * n);
    launch_keys_to_float(keys, 2 * n, mmf, s);
    ctx->launches += 1;
    CK(cudaMemcpyAsync(minmax_host, mmf, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
  }
  return VD3D_OK;
}

}  // namespace

extern "C" {

int vd3d_tile_crops(vd3d_ctx* ctx, const uint8_t* frame, int h, int w, int tile, int pad, const vd3d_tile* tiles,
                    int n_tiles, uint8_t* out, int mem) {
  if (!ctx || !frame || !out) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  int step, nx, ny, r;
  if ((r = check_plan(ctx, h, w, tile, pad, tiles, n_tiles, 0, &step, &nx, &ny))) return r;
  CK(cudaSetDevice(ctx->device));
  const void* f_d;
  if ((r = copy_in(ctx, ctx->td_frames, frame, (size_t)h * w * 3, mem, ctx->stream, &f_d))) return r;
  std::vector<TileJob> jobs;
  size_t cb, pc;
  tile_jobs(nullptr, 1, tiles, n_tiles, nullptr, nullptr, nullptr, jobs, &cb, &pc);
  void* o_d;
  if ((r = stage_out(ctx, ctx->td_out, out, cb, mem, &o_d))) return r;
  const uint8_t* fp = (const uint8_t*)f_d;
  tile_jobs(&fp, 1, tiles, n_tiles, (uint8_t*)o_d, nullptr, nullptr, jobs, &cb, &pc);
  const TileJob* jd;
  if ((r = upload_jobs(ctx, jobs, &jd))) return r;
  gather(ctx, jd, tiles, n_tiles, n_tiles, w);
  return stage_finish(ctx, out, o_d, cb, mem);
}

int vd3d_tile_blend(vd3d_ctx* ctx, int h, int w, int tile, int pad, const vd3d_tile* tiles, int n_tiles,
                    const float* const* preds, const float* const* weights, float* out, float* minmax, int mem) {
  if (!ctx || !preds || !weights || !out) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  int step, nx, ny, r;
  if ((r = check_plan(ctx, h, w, tile, pad, tiles, n_tiles, 0, &step, &nx, &ny))) return r;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  std::vector<TileJob> jobs;
  size_t cb, pc;
  tile_jobs(nullptr, 1, tiles, n_tiles, nullptr, nullptr, nullptr, jobs, &cb, &pc);
  std::vector<const float*> wd(weights, weights + n_tiles);
  float* pred_base = nullptr;
  if (mem == VD3D_MEM_HOST) {  // pack the predictions and the weights into device buffers
    size_t wc = 0;
    for (int t = 0; t < n_tiles; ++t) wc += (size_t)(tiles[t].y1 - tiles[t].y0) * (tiles[t].x1 - tiles[t].x0);
    if ((r = ensure(ctx, ctx->td_preds, pc * 4)) || (r = ensure(ctx, ctx->td_wgt, wc * 4))) return r;
    pred_base = (float*)ctx->td_preds.p;
    size_t po = 0, wo = 0;
    for (int t = 0; t < n_tiles; ++t) {
      const size_t np = (size_t)tiles[t].rh * tiles[t].rw;
      const size_t nw = (size_t)(tiles[t].y1 - tiles[t].y0) * (tiles[t].x1 - tiles[t].x0);
      CK(cudaMemcpyAsync(pred_base + po, preds[t], np * 4, cudaMemcpyHostToDevice, s));
      CK(cudaMemcpyAsync((float*)ctx->td_wgt.p + wo, weights[t], nw * 4, cudaMemcpyHostToDevice, s));
      wd[t] = (const float*)ctx->td_wgt.p + wo;
      po += np;
      wo += nw;
    }
  }
  tile_jobs(nullptr, 1, tiles, n_tiles, nullptr, pred_base, wd.data(), jobs, &cb, &pc);
  if (mem != VD3D_MEM_HOST)
    for (int t = 0; t < n_tiles; ++t) jobs[t].pred = preds[t];
  const TileJob* jd;
  if ((r = upload_jobs(ctx, jobs, &jd))) return r;
  if ((r = blend_frames(ctx, jd, 1, h, w, tile, step, nx, ny, minmax))) return r;
  const size_t bytes = (size_t)h * w * 4;
  CK(cudaMemcpyAsync(out, ctx->td_depth.p, bytes,
                     mem == VD3D_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, s));
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(s));
  return VD3D_OK;
}

int vd3d_normalize_u8(vd3d_ctx* ctx, const float* d, int h, int w, double p_lo, double p_hi, int invert, uint8_t* out,
                      int oh, int ow, float* stats_out, int mem) {
  if (!ctx || !d || !out || h < 1 || w < 1 || oh < 1 || ow < 1) return fail(ctx, VD3D_ERR_ARG, "bad argument");
  CK(cudaSetDevice(ctx->device));
  const void* d_d;
  void* o_d;
  int r;
  if ((r = copy_in(ctx, ctx->td_depth, d, (size_t)h * w * 4, mem, ctx->stream, &d_d))) return r;
  if ((r = stage_out(ctx, ctx->td_out, out, (size_t)oh * ow, mem, &o_d))) return r;
  uint8_t* outs[1] = {(uint8_t*)o_d};
  if ((r = normalize_planes(ctx, (const float*)d_d, 1, h, w, p_lo, p_hi, invert, outs, oh, ow, stats_out))) return r;
  return stage_finish(ctx, out, o_d, (size_t)oh * ow, mem);
}

int vd3d_depth_tiled(vd3d_ctx* ctx, vd3d_depth* const* engines, int n_classes, int n, const uint8_t* const* frames,
                     int h, int w, int tile, int pad, const vd3d_tile* tiles, int n_tiles, const float* const* weights,
                     int invert, int oh, int ow, uint8_t* const* out_u8, float* const* out_f32, float* minmax,
                     int mem) {
  if (!ctx || !engines || n_classes < 1 || n < 1 || !frames || !weights || !out_u8 || oh < 1 || ow < 1)
    return fail(ctx, VD3D_ERR_ARG, "bad argument");
  for (int c = 0; c < n_classes; ++c) {
    if (!engines[c]) return fail(ctx, VD3D_ERR_ARG, "missing engine");
    if (depth_family(engines[c]) != VD3D_DEPTH_DA_V2)
      return fail(ctx, VD3D_ERR_UNSUPPORTED, "tiled depth serves Depth-Anything-V2 engines only");
    // the gather and the blend run on ctx->stream: an engine on another stream would race them
    if (sr_stream(engines[c]) != ctx->stream)
      return fail(ctx, VD3D_ERR_ARG, "the depth engines must be created on vd3d_stream(ctx)");
  }
  int step, nx, ny, r;
  if ((r = check_plan(ctx, h, w, tile, pad, tiles, n_tiles, n_classes, &step, &nx, &ny))) return r;
  for (int t = 0; t < n_tiles; ++t)
    if (tiles[t].rh < 16 || tiles[t].rw < 16)
      return fail(ctx, VD3D_ERR_ARG, "a tile crop is below the depth engine's 16 x 16 minimum");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const size_t fbytes = (size_t)h * w * 3, npix = (size_t)h * w, obytes = (size_t)oh * ow;
  std::vector<const uint8_t*> fd(frames, frames + n);
  if (mem == VD3D_MEM_HOST) {
    if ((r = ensure(ctx, ctx->td_frames, fbytes * n))) return r;
    for (int f = 0; f < n; ++f) {
      fd[f] = (const uint8_t*)ctx->td_frames.p + fbytes * f;
      CK(cudaMemcpyAsync((void*)fd[f], frames[f], fbytes, cudaMemcpyHostToDevice, s));
    }
  }
  std::vector<TileJob> jobs;
  size_t cb, pc;
  tile_jobs(nullptr, 1, tiles, n_tiles, nullptr, nullptr, nullptr, jobs, &cb, &pc);
  if ((r = ensure(ctx, ctx->td_crops, cb * n)) || (r = ensure(ctx, ctx->td_preds, pc * 4 * n))) return r;
  tile_jobs(fd.data(), n, tiles, n_tiles, (uint8_t*)ctx->td_crops.p, (float*)ctx->td_preds.p, weights, jobs, &cb, &pc);
  const TileJob* jd;
  if ((r = upload_jobs(ctx, jobs, &jd))) return r;
  gather(ctx, jd, tiles, n_tiles, n * n_tiles, w);
  // forwards: the tiles of each class, frame-major in plan order, up to 8 per batch
  for (int c = 0; c < n_classes; ++c) {
    const uint8_t* cin[8];
    float* cout_[8];
    int b = 0, rh = 0, rw = 0;
    for (size_t k = 0; k <= jobs.size(); ++k) {
      const bool take = k < jobs.size() && tiles[k % n_tiles].cls == c;
      if (take) {
        cin[b] = jobs[k].crop;
        cout_[b] = (float*)jobs[k].pred;
        rh = jobs[k].rh;
        rw = jobs[k].rw;
        ++b;
      }
      if (b == 8 || (k == jobs.size() && b > 0)) {
        if ((r = vd3d_depth_infer_batch_device(engines[c], b, cin, rh, rw, nullptr, cout_, 0))) {
          ctx->err = std::string("tile forward: ") + vd3d_depth_last_error(engines[c]);
          return r;
        }
        b = 0;
      }
    }
  }
  if ((r = blend_frames(ctx, jd, n, h, w, tile, step, nx, ny, minmax))) return r;
  std::vector<uint8_t*> od(out_u8, out_u8 + n);
  if (mem == VD3D_MEM_HOST) {
    if ((r = ensure(ctx, ctx->td_out, obytes * n))) return r;
    for (int f = 0; f < n; ++f) od[f] = (uint8_t*)ctx->td_out.p + obytes * f;
  }
  if ((r = normalize_planes(ctx, (const float*)ctx->td_depth.p, n, h, w, 1.0, 99.0, invert, od.data(), oh, ow,
                            nullptr)))
    return r;
  for (int f = 0; f < n; ++f) {
    const cudaMemcpyKind k = mem == VD3D_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    if (mem == VD3D_MEM_HOST) CK(cudaMemcpyAsync(out_u8[f], od[f], obytes, k, s));
    if (out_f32 && out_f32[f])
      CK(cudaMemcpyAsync(out_f32[f], (const float*)ctx->td_depth.p + npix * f, npix * 4, k, s));
  }
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(s));
  return VD3D_OK;
}

}  // extern "C"
