// depth_engine.cu -- Depth-Anything-V2 (DINOv2 ViT + DPT neck/head) forward as a fixed
// launch sequence of wgmma GEMMs and small fused kernels.  Host side: named device
// tensors (pushed by the Python loader in HF state_dict terms), TMA tensor maps, buffers.
//
// Reference call path: core/render_depth.py:1106-1119 -> transformers pipeline
// ("depth-estimation") -> DepthAnythingForDepthEstimation.forward (transformers 5.5.0,
// models/depth_anything/modeling_depth_anything.py; backbone models/dinov2/modeling_dinov2.py).
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "../../include/vd3d.h"
#include "depth_launch.h"
#include "dibr_launch.h"  // launch_resize_cubic_u8 (cv2 INTER_CUBIC) for the image path
#include "sr_engine.h"
#include "umma_gemm.cuh"

using namespace vd3d;

namespace {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

bool load_encode() {
  if (g_encode) return true;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qr;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) != cudaSuccess || !fn) return false;
  g_encode = (EncodeTiledFn)fn;
  return true;
}

struct DTensor {
  void* p = nullptr;
  size_t bytes = 0;
};

// What a model family changes in the forward and in the drivers (family_traits).
struct FamilyTraits {
  bool bit_front_end;    // DPT-Hybrid: a BiT backbone replaces the patch embedding; its stages 1 and 2 feed neck
                         // inputs 0 and 1
  bool readout;          // DPT: raw taps through the project readout (else Depth-Anything's final-LayerNorm taps)
  bool rel_pos_bias;     // BEiT: a relative position bias table per layer in the attention
  bool zoe_head;         // ZoeDepth: the metric-bins head, the reflect-pad pre-process and the cropped post-process
  bool square_grid;      // the tokens are reshaped as a square grid (DPT-Large, DPT-Hybrid)
  bool keep_aspect_fit;  // the processor may keep the aspect ratio (vd3d_depth_set_fit)
};

// the traits of a VD3D_DEPTH_* code; false for an unknown code
bool family_traits(int family, FamilyTraits* t) {
  switch (family) {
    case VD3D_DEPTH_DA_V2: *t = {false, false, false, false, false, false}; return true;
    case VD3D_DEPTH_DPT: *t = {false, true, false, false, true, false}; return true;
    case VD3D_DEPTH_DPT_HYBRID: *t = {true, true, false, false, true, false}; return true;
    case VD3D_DEPTH_DPT_BEIT: *t = {false, true, true, false, false, true}; return true;
    // ZoeDepth's trunk, neck and fusion are dpt-beit-large-512's
    case VD3D_DEPTH_ZOEDEPTH: *t = {false, true, true, true, false, true}; return true;
  }
  return false;
}

// The model an engine serves: everything vd3d_depth_clone hands to a clone besides the weights.
struct DepthSettings {
  vd3d_depth_config cfg;
  // model family, patch, LayerNorm epsilon and image processor (vd3d_depth_create_ex; DA-V2 defaults otherwise)
  int family = VD3D_DEPTH_DA_V2, patch = 14;
  FamilyTraits traits = {};
  float ln_eps = 1e-6f;
  PreprocParams pre = kImagenetBicubic;
  // the keep-aspect processor of vd3d_depth_infer_images: target and multiple; fit_multiple 0: a fixed size.
  // Depth-Anything's is 518 x 518 and 14; BEiT's is set by vd3d_depth_set_fit
  int fit_h = 0, fit_w = 0, fit_multiple = 0;
  // ZoeDepth's metric head (vd3d_depth_set_zoe): bin configurations (0: not set), attractors per layer, temperature
  // range, whether the relative depth is the log-binomial's 33rd input
  int zoe_nc = 0, zoe_na[4] = {}, zoe_cat = 0;
  float zoe_tmin = 0.f, zoe_tmax = 0.f;
  // the head's last activation (VD3D_HEAD_RELATIVE / _METRIC) and the metric head's scale; every EPI_HEAD reads them
  int head = VD3D_HEAD_RELATIVE;
  float max_depth = 1.f;
  int ph = 0, pw = 0, ntok = 0, npad = 0;  // token grid, tokens with CLS, tokens rounded up to the 128-row tile
};

}  // namespace

struct vd3d_depth : DepthSettings {
  cudaStream_t stream = nullptr;
  std::string err;
  std::map<std::string, DTensor> w;    // weights by name
  std::map<std::string, DTensor> buf;  // activations by name
  uint64_t launches = 0;
  // the per-image neck / head tails of a batch run on side streams (forked after the transformer, joined at the end)
  cudaStream_t cur = nullptr;          // stream the helpers launch on (null: `stream`; set by StreamScope only)
  cudaStream_t aux[8] = {};
  cudaEvent_t ev_fork = nullptr, ev_join[8] = {};
  bool owns_weights = true;  // clones share the weight tensors of their parent
  uint64_t weights_version = 0;  // bumped whenever a weight tensor moves (clones / captured graphs hold raw pointers)
  // optional device timing of one GEMM class (the fc1 launches) for the roofline report
  bool prof = false;
  std::vector<cudaEvent_t> prof_ev;
  long long prof_rows = 0;  // rows (tokens of all images of the batch) summed over the timed fc1 launches
  // tuning aid (vd3d_depth_profile(e, 2)): device time of every launch class of the forward, eager mode only
  struct Span {
    const char* tag;
    cudaEvent_t e0, e1;
  };
  std::vector<Span> spans;
  int span_begin(const char* tag, cudaStream_t s) {
    if (!prof_spans) return -1;
    Span sp{tag, nullptr, nullptr};
    cudaEventCreate(&sp.e0);
    cudaEventCreate(&sp.e1);
    cudaEventRecord(sp.e0, s);
    spans.push_back(sp);
    return (int)spans.size() - 1;
  }
  void span_end(int i, cudaStream_t s) {
    if (i >= 0) cudaEventRecord(spans[i].e1, s);
  }
  bool prof_spans = false;
  // SR engines: RRDBNet with rr_nb blocks and network scale rr_scale (vd3d_sr_set_rrdb); 0: SRVGGNetCompact
  int rr_nb = 0, rr_scale = 0;
};

namespace {

#define DCK(call)                                                                   \
  do {                                                                              \
    cudaError_t _e = (call);                                                        \
    if (_e != cudaSuccess) {                                                        \
      char _b[512];                                                                 \
      snprintf(_b, sizeof _b, "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
      e->err = _b;                                                                  \
      return VD3D_ERR_CUDA;                                                         \
    }                                                                               \
  } while (0)

int dfail(vd3d_depth* e, int code, const std::string& msg) {
  e->err = msg;
  return code;
}

// the stream gemm, conv and get_buf's zeroing enqueue on
cudaStream_t launch_stream(const vd3d_depth* e) { return e->cur ? e->cur : e->stream; }

// Makes the helpers launch on `s` until it goes out of scope, on every return path (a per-image tail of forward_core)
struct StreamScope {
  vd3d_depth* e;
  cudaStream_t prev;
  StreamScope(vd3d_depth* e_, cudaStream_t s) : e(e_), prev(e_->cur) { e->cur = s; }
  ~StreamScope() { e->cur = prev; }
};

template <typename T>
int get_buf(vd3d_depth* e, const std::string& name, size_t bytes, T** out, bool zero = false) {
  DTensor& t = e->buf[name];
  if (t.bytes < bytes) {
    if (t.p) DCK(cudaFree(t.p));
    DCK(cudaMalloc(&t.p, bytes));
    t.bytes = bytes;
    zero = true;
  }
  if (zero) DCK(cudaMemsetAsync(t.p, 0, t.bytes, launch_stream(e)));
  *out = (T*)t.p;
  return VD3D_OK;
}

template <typename T>
int W(vd3d_depth* e, const std::string& name, const T** out, size_t min_count = 0) {
  auto it = e->w.find(name);
  if (it == e->w.end()) return dfail(e, VD3D_ERR_STATE, "missing weight tensor: " + name);
  if (min_count && it->second.bytes < min_count * sizeof(T))
    return dfail(e, VD3D_ERR_STATE, "weight tensor too small: " + name);
  *out = (const T*)it->second.p;
  return VD3D_OK;
}

// the f16 weight "<base>.w" (at least nw elements) and f32 bias "<base>.b" (nb) of a layer
int layer(vd3d_depth* e, const std::string& base, const __half** w, size_t nw, const float** b, size_t nb) {
  const int r = W(e, base + ".w", w, nw);
  return r ? r : W(e, base + ".b", b, nb);
}

// a tensor or buffer name from a printf format with integer arguments, e.g. fmt("r%d.proj", i)
std::string fmt(const char* f, int a, int b = 0) {
  char nm[64];
  snprintf(nm, sizeof nm, f, a, b);
  return nm;
}

// f16 3-D tensor map: dims (d0 inner, d1, d2), strides in ELEMENTS for d1 and d2, box (64, b1, b2)
int make_map(vd3d_depth* e, CUtensorMap* m, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t s1,
             uint64_t s2, uint32_t b1, uint32_t b2) {
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {s1 * 2, s2 * 2};
  cuuint32_t box[3] = {64, b1, b2};
  cuuint32_t es[3] = {1, 1, 1};
  if ((strides[0] % 16) || (strides[1] % 16) || ((uintptr_t)ptr % 16))
    return dfail(e, VD3D_ERR_ARG, "tensor map: pointer / strides must be 16-byte aligned");
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char b[256];
    snprintf(b, sizeof b, "cuTensorMapEncodeTiled failed (%d) dims=(%llu,%llu,%llu) strides=(%llu,%llu) box=(64,%u,%u)",
             (int)r, (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2,
             (unsigned long long)strides[0], (unsigned long long)strides[1], b1, b2);
    return dfail(e, VD3D_ERR_CUDA, b);
  }
  return VD3D_OK;
}

GemmArgs base_args(int M, int N, int K, int epi) {
  GemmArgs g;
  memset(&g, 0, sizeof g);
  g.M = M;
  g.N = N;
  g.K = K;
  g.epi = epi;
  g.ldc = N;
  return g;
}

// Tile width of a GEMM / conv: one 128 x bn kernel for every shape.  The choice depends on N only, never on the
// batch size, so a frame's depth is the same inferred alone or in a batch
// (tests/test_depth_gpu.py::test_infer_batch_equals_single_frames; exact sharding == one GPU).
int pick_bn(int N) { return N >= 128 ? 128 : (N >= 64 ? 64 : 32); }

// plain GEMM: A [M, K] (lda), B [N, K] (ldb)
int gemm(vd3d_depth* e, const __half* A, int lda, const __half* B, int ldb, GemmArgs g, int bn = 0) {
  if (!bn) bn = pick_bn(g.N);
  CUtensorMap ma, mb;
  int r;
  if ((r = make_map(e, &ma, A, g.K, g.M, 1, lda, (uint64_t)lda * g.M, 128, 1))) return r;
  if ((r = make_map(e, &mb, B, g.K, g.N, 1, ldb, (uint64_t)ldb * g.N, bn, 1))) return r;
  cudaError_t ce = launch_gemm(bn, ma, mb, g, (g.M + 127) / 128, 1, launch_stream(e));
  if (ce != cudaSuccess) return dfail(e, VD3D_ERR_CUDA, std::string("gemm launch: ") + cudaGetErrorString(ce));
  e->launches++;
  return VD3D_OK;
}

void pick_tile(int W, int H, int& tw, int& th) {
  const int cand[4][2] = {{128, 1}, {64, 2}, {32, 4}, {16, 8}};
  long best = -1;
  for (auto& c : cand) {
    long cover = (long)((W + c[0] - 1) / c[0]) * c[0] * (long)((H + c[1] - 1) / c[1]) * c[1];
    if (best < 0 || cover < best) {
      best = cover;
      tw = c[0];
      th = c[1];
    }
  }
}

// conv over an NHWC f16 map [H, W, cin] (3x3 pad 1 when k3, else 1x1); weights [N, taps*cin].  pitch: channels per
// pixel of the map when it holds more than the cin read (0: cin); sr: the RRDBNet epilogue (EPI_SR)
int conv(vd3d_depth* e, const __half* in, int H, int W, int cin, const __half* wt, bool k3, GemmArgs g, int bn = 0,
         int pitch = 0, bool sr = false) {
  if (cin % 64) return dfail(e, VD3D_ERR_ARG, "conv: cin must be a multiple of 64");
  if (!bn) bn = pick_bn(g.N);
  int tw, th;
  pick_tile(W, H, tw, th);
  g.conv = k3 ? 1 : 2;
  g.cin = cin;
  g.imgW = W;
  g.imgH = H;
  g.tw = tw;
  g.th = th;
  g.M = H * W;
  g.K = (k3 ? 9 : 1) * cin;
  CUtensorMap ma, mb;
  int r;
  if (!pitch) pitch = cin;
  if ((r = make_map(e, &ma, in, cin, W, H, pitch, (uint64_t)pitch * W, tw, th))) return r;
  if ((r = make_map(e, &mb, wt, g.K, g.N, 1, g.K, (uint64_t)g.K * g.N, bn, 1))) return r;
  int m_tiles = ((W + tw - 1) / tw) * ((H + th - 1) / th);
  cudaStream_t s = launch_stream(e);
  cudaError_t ce = sr ? launch_gemm_sr(bn, ma, mb, g, m_tiles, s) : launch_gemm(bn, ma, mb, g, m_tiles, 1, s);
  if (ce != cudaSuccess) return dfail(e, VD3D_ERR_CUDA, std::string("conv launch: ") + cudaGetErrorString(ce));
  e->launches++;
  return VD3D_OK;
}

int round_up(int v, int m) { return (v + m - 1) / m * m; }

// One conv of the BiT backbone (bit_backbone; vd3d_bit_kernel op 4) on k_umma_gemm, no bias: f16 NHWC in [H, W, cin]
// -> f32 out [Ho * Wo, cout].  BIT_1X1: a GEMM on the map's pixel rows, w [cout, cin].  BIT_3X3: stride 1, pad 1, on
// the implicit-GEMM conv, w [cout, 9 cin] tap-major.  BIT_3X3_S2: stride 2 with TF-SAME pads (0 before, 1 after), a
// GEMM on k_im2col_same's rows written to col.  BIT_1X1_S2: stride 2, a GEMM on the even pixels gathered into col.
// Ho = H / 2 and Wo = W / 2 at stride 2; col holds round_up(Ho * Wo, 128) rows of the GEMM's K columns.
enum { BIT_1X1 = 0, BIT_3X3 = 1, BIT_3X3_S2 = 2, BIT_1X1_S2 = 3 };
int bit_conv(vd3d_depth* e, int kind, const __half* in, int H, int Wd, int cin, const __half* w, int cout, float* out,
             __half* col) {
  cudaStream_t s = e->stream;
  const bool s2 = kind == BIT_3X3_S2 || kind == BIT_1X1_S2;
  const int k = (kind == BIT_3X3 || kind == BIT_3X3_S2) ? 3 : 1, K = k * k * cin;
  GemmArgs g = base_args(s2 ? (H / 2) * (Wd / 2) : H * Wd, cout, K, EPI_F32);
  g.out_f32 = out;
  const __half* a = in;
  if (s2) {
    const int sp = e->span_begin("bit.im2col", s);
    launch_im2col_same(in, H, Wd, cin, k, 0, col, s);
    e->span_end(sp, s);
    e->launches++;
    a = col;
  }
  const int sp = e->span_begin("bit.conv", s);
  const int r = kind == BIT_3X3 ? conv(e, in, H, Wd, cin, w, true, g) : gemm(e, a, K, w, K, g);
  e->span_end(sp, s);
  return r;
}

// ZoeDepthImageProcessor's reflect padding of an h-row (or w-column) image: int(sqrt(h / 2) * 3), the same value
// post_process_depth_estimation crops off
int zoe_pad(int n) { return (int)(sqrt(n / 2.0) * 3.0); }

}  // namespace

extern "C" {

int vd3d_depth_create_ex(const vd3d_depth_config_ex* x, void* stream, vd3d_depth** out) {
  if (!x || !out) return VD3D_ERR_ARG;
  *out = nullptr;
  if (!load_encode()) return VD3D_ERR_CUDA;
  const vd3d_depth_config* cfg = &x->base;
  FamilyTraits t;
  if (!family_traits(x->family, &t) || (x->patch != 14 && x->patch != 16) || (x->resample != 2 && x->resample != 3) ||
      !(x->ln_eps > 0.f) || cfg->heads < 1)
    return VD3D_ERR_ARG;
  if ((x->head != VD3D_HEAD_RELATIVE && x->head != VD3D_HEAD_METRIC) || !(x->max_depth > 0.f) ||
      !isfinite(x->max_depth) || (t.readout && x->head == VD3D_HEAD_METRIC))
    return VD3D_ERR_ARG;
  if (cfg->hidden % 128 || cfg->hidden > 1024 || cfg->hidden / cfg->heads != 64 || cfg->fusion % 64 ||
      cfg->image_h % x->patch || cfg->image_w % x->patch)
    return VD3D_ERR_ARG;
  // every fusion x2 must land on the next map: sides that are multiples of 32.  DPT-Large and the hybrid reshape the
  // tokens as a square grid; BEiT takes the grid of the input (patch_height x patch_width), rectangular included
  if (t.readout && (cfg->image_h % 32 || cfg->image_w % 32)) return VD3D_ERR_ARG;
  if (t.square_grid && cfg->image_h != cfg->image_w) return VD3D_ERR_ARG;
  // the hybrid's fixed BiT front end: patch 16 (stage 3 is the S/16 token grid), stage maps of 256 / 512 channels
  if (t.bit_front_end && (x->patch != 16 || cfg->neck[0] != 256 || cfg->neck[1] != 512)) return VD3D_ERR_ARG;
  // BEiT: the relative position bias table of the grid is staged in the attention's shared memory
  if (t.rel_pos_bias &&
      (x->patch != 16 || attention_bias_smem(cfg->image_h / 16, cfg->image_w / 16) > (size_t)kAttnSmemMax))
    return VD3D_ERR_ARG;
  for (int c = 0; c < 3; ++c)
    if (!(x->std[c] != 0.f)) return VD3D_ERR_ARG;
  vd3d_depth* e = new vd3d_depth();
  e->cfg = *cfg;
  e->family = x->family;
  e->traits = t;
  e->patch = x->patch;
  e->ln_eps = x->ln_eps;
  e->head = x->head;
  e->max_depth = x->max_depth;
  e->pre.bilinear = x->resample == 2;
  for (int c = 0; c < 3; ++c) {
    e->pre.mean[c] = x->mean[c];
    e->pre.std[c] = x->std[c];
  }
  if (!t.readout) {  // Depth-Anything's processor (depth_engine.py processed_size); DPT's resizes to a fixed size
    e->fit_h = e->fit_w = 518;
    e->fit_multiple = 14;
  }
  e->stream = (cudaStream_t)stream;
  e->ph = cfg->image_h / x->patch;
  e->pw = cfg->image_w / x->patch;
  e->ntok = e->ph * e->pw + 1;
  e->npad = round_up(e->ntok, 128);
  if (e->ntok > 3072) {
    delete e;
    return VD3D_ERR_UNSUPPORTED;
  }
  *out = e;
  return VD3D_OK;
}

int vd3d_depth_set_fit(vd3d_depth* e, int fit_h, int fit_w, int multiple) {
  if (!e || !e->traits.keep_aspect_fit || (multiple != 0 && multiple != 32) || (multiple && (fit_h < 32 || fit_w < 32)))
    return VD3D_ERR_ARG;
  e->fit_h = multiple ? fit_h : 0;
  e->fit_w = multiple ? fit_w : 0;
  e->fit_multiple = multiple;
  return VD3D_OK;
}

int vd3d_depth_set_zoe(vd3d_depth* e, int n_conf, int n_bins, const float* min_depth, const float* max_depth,
                       float min_temp, float max_temp, const int32_t* attractors, int cat_relative) {
  if (!e || !e->traits.zoe_head || (n_conf != 1 && n_conf != 2) || n_bins != kZoeBins || !min_depth ||
      !max_depth || !attractors || !(min_temp > 0.f) || !(max_temp > min_temp) || !isfinite(max_temp) ||
      (cat_relative != 0 && cat_relative != 1))
    return VD3D_ERR_ARG;
  for (int i = 0; i < n_conf; ++i)
    if (!(min_depth[i] >= 0.f) || !(max_depth[i] > min_depth[i]) || !isfinite(max_depth[i])) return VD3D_ERR_ARG;
  for (int j = 0; j < 4; ++j)
    if (attractors[j] < 1 || attractors[j] > kZoeMaxAttr) return VD3D_ERR_ARG;
  e->zoe_nc = n_conf;
  e->zoe_cat = cat_relative;
  e->zoe_tmin = min_temp;
  e->zoe_tmax = max_temp;
  for (int j = 0; j < 4; ++j) e->zoe_na[j] = attractors[j];
  return VD3D_OK;
}

int vd3d_depth_create(const vd3d_depth_config* cfg, void* stream, vd3d_depth** out) {
  if (!cfg || !out) return VD3D_ERR_ARG;
  vd3d_depth_config_ex x;
  memset(&x, 0, sizeof x);
  x.base = *cfg;
  x.family = VD3D_DEPTH_DA_V2;
  x.patch = 14;
  x.ln_eps = 1e-6f;
  x.resample = 3;
  x.head = VD3D_HEAD_RELATIVE;
  x.max_depth = 1.f;
  for (int c = 0; c < 3; ++c) {
    x.mean[c] = kImagenetBicubic.mean[c];
    x.std[c] = kImagenetBicubic.std[c];
  }
  return vd3d_depth_create_ex(&x, stream, out);
}

// device timing of the fc1 GEMM launches (k_umma_gemm<128,4>, M=tokens, N=4D, K=D): bench.py roofline
int vd3d_depth_profile(vd3d_depth* e, int enable) {
  if (!e) return VD3D_ERR_ARG;
  e->prof = enable == 1;
  e->prof_spans = enable == 2;
  return VD3D_OK;
}
// "tag total_ms launches" lines of the spans recorded since the last call (vd3d_depth_profile(e, 2))
int vd3d_depth_profile_spans(vd3d_depth* e, char* out, size_t cap) {
  if (!e || !out || !cap) return VD3D_ERR_ARG;
  DCK(cudaDeviceSynchronize());
  std::vector<std::pair<std::string, std::pair<double, int>>> acc;
  for (auto& sp : e->spans) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, sp.e0, sp.e1) != cudaSuccess) ms = 0.f;
    cudaEventDestroy(sp.e0);
    cudaEventDestroy(sp.e1);
    size_t i = 0;
    for (; i < acc.size(); ++i)
      if (acc[i].first == sp.tag) break;
    if (i == acc.size()) acc.push_back({sp.tag, {0.0, 0}});
    acc[i].second.first += ms;
    acc[i].second.second++;
  }
  e->spans.clear();
  std::string txt;
  char line[128];
  for (auto& a : acc) {
    snprintf(line, sizeof line, "%s %.4f %d\n", a.first.c_str(), a.second.first, a.second.second);
    txt += line;
  }
  snprintf(out, cap, "%s", txt.c_str());
  return VD3D_OK;
}
int vd3d_depth_profile_collect(vd3d_depth* e, double* total_ms, int* count, double* gflop_per_launch) {
  if (!e || !total_ms || !count) return VD3D_ERR_ARG;
  DCK(cudaStreamSynchronize(e->stream));
  double t = 0;
  int n = 0;
  for (size_t i = 0; i + 1 < e->prof_ev.size(); i += 2) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, e->prof_ev[i], e->prof_ev[i + 1]) == cudaSuccess) {
      t += ms;
      ++n;
    }
  }
  for (cudaEvent_t ev : e->prof_ev) cudaEventDestroy(ev);
  e->prof_ev.clear();
  *total_ms = t;
  *count = n;
  if (gflop_per_launch)  // average over the timed launches (batches of different sizes have different row counts)
    *gflop_per_launch = 2.0 * (n ? (double)e->prof_rows / n : (double)e->ntok) * (4.0 * e->cfg.hidden) * e->cfg.hidden / 1e9;
  e->prof_rows = 0;
  return VD3D_OK;
}

// A second engine instance on another stream that shares the parent's weights (own activation
// buffers): lets two frames' depth forwards overlap on the GPU (vd3d_render_clip_depth).
int vd3d_depth_clone(vd3d_depth* src, void* stream, vd3d_depth** out) {
  if (!src || !out) return VD3D_ERR_ARG;
  vd3d_depth* e = new vd3d_depth();
  static_cast<DepthSettings&>(*e) = *src;
  e->stream = (cudaStream_t)stream;
  e->w = src->w;
  e->owns_weights = false;
  *out = e;
  return VD3D_OK;
}

void vd3d_depth_destroy(vd3d_depth* e) {
  if (!e) return;
  cudaStreamSynchronize(e->stream);
  for (int i = 0; i < 8; ++i) {
    if (e->aux[i]) {
      cudaStreamSynchronize(e->aux[i]);
      cudaStreamDestroy(e->aux[i]);
    }
    if (e->ev_join[i]) cudaEventDestroy(e->ev_join[i]);
  }
  if (e->ev_fork) cudaEventDestroy(e->ev_fork);
  for (auto& kv : e->w)
    if (e->owns_weights && kv.second.p) cudaFree(kv.second.p);
  for (auto& kv : e->buf)
    if (kv.second.p) cudaFree(kv.second.p);
  delete e;
}

const char* vd3d_depth_last_error(vd3d_depth* e) { return e ? e->err.c_str() : "null depth engine"; }
uint64_t vd3d_depth_launch_count(vd3d_depth* e) { return e ? e->launches : 0; }
void vd3d_depth_add_launches(vd3d_depth* e, uint64_t n) {
  if (e) e->launches += n;  // graph replays account for the launches they contain
}

int vd3d_depth_set_tensor(vd3d_depth* e, const char* name, const void* host_data, size_t bytes) {
  if (!e || !name || !host_data || !bytes) return VD3D_ERR_ARG;
  if (!e->owns_weights) return dfail(e, VD3D_ERR_STATE, "weights of an engine clone belong to its parent");
  DTensor& t = e->w[name];
  const size_t cap = (bytes + 255) / 256 * 256;
  if (t.p && (t.bytes + 255) / 256 * 256 == cap) {
    // same footprint: overwrite in place so that clones and captured graphs (raw pointers) stay valid; work already
    // enqueued on any stream finishes first
    DCK(cudaDeviceSynchronize());
    t.bytes = bytes;
    DCK(cudaMemcpy(t.p, host_data, bytes, cudaMemcpyHostToDevice));
    return VD3D_OK;
  }
  if (t.p) {
    DCK(cudaDeviceSynchronize());
    cudaFree(t.p);
  }
  t.p = nullptr;
  e->weights_version++;  // the tensor moves: vd3d_ctx rebuilds its clones and drops its graphs (vd3d_api.cu)
  DCK(cudaMalloc(&t.p, cap));
  t.bytes = bytes;
  DCK(cudaMemcpy(t.p, host_data, bytes, cudaMemcpyHostToDevice));
  return VD3D_OK;
}
uint64_t vd3d_depth_weights_version(vd3d_depth* e) { return e ? e->weights_version : 0; }

int vd3d_depth_get_buffer(vd3d_depth* e, const char* name, void* host_out, size_t bytes) {
  if (!e || !name || !host_out) return VD3D_ERR_ARG;
  auto it = e->buf.find(name);
  if (it == e->buf.end()) return dfail(e, VD3D_ERR_ARG, std::string("no such buffer: ") + name);
  if (bytes > it->second.bytes) return dfail(e, VD3D_ERR_ARG, "buffer smaller than requested");
  DCK(cudaStreamSynchronize(e->stream));
  DCK(cudaMemcpy(host_out, it->second.p, bytes, cudaMemcpyDeviceToHost));
  return VD3D_OK;
}

// unit-test hook: C[M,N] f32 = A[M,K] f16 x B[N,K]^T f16 through the wgmma kernel
int vd3d_gemm_f16(vd3d_depth* e, const void* A, const void* B, int M, int N, int K, float* C_host, int bn) {
  if (!e || !A || !B || !C_host || (K % 8)) return VD3D_ERR_ARG;
  void *da, *db, *dc;
  int r;
  if ((r = get_buf(e, "t.a", (size_t)M * K * 2, &da))) return r;
  if ((r = get_buf(e, "t.b", (size_t)N * K * 2, &db))) return r;
  if ((r = get_buf(e, "t.c", (size_t)M * N * 4, &dc, true))) return r;
  DCK(cudaMemcpyAsync(da, A, (size_t)M * K * 2, cudaMemcpyHostToDevice, e->stream));
  DCK(cudaMemcpyAsync(db, B, (size_t)N * K * 2, cudaMemcpyHostToDevice, e->stream));
  GemmArgs g = base_args(M, N, K, EPI_F32);
  g.out_f32 = (float*)dc;
  if ((r = gemm(e, (const __half*)da, K, (const __half*)db, K, g, bn))) return r;
  DCK(cudaMemcpyAsync(C_host, dc, (size_t)M * N * 4, cudaMemcpyDeviceToHost, e->stream));
  DCK(cudaStreamSynchronize(e->stream));
  return VD3D_OK;
}

// unit-test hook: 3x3 (or 1x1) conv on an NHWC f16 map through the implicit-GEMM path
int vd3d_conv_f16(vd3d_depth* e, const void* in_nhwc, int H, int W, int cin, const void* wt, int cout, int k3,
                  const float* bias, int relu, float* out_host) {
  if (!e || !in_nhwc || !wt || !out_host) return VD3D_ERR_ARG;
  int taps = k3 ? 9 : 1;
  void *di, *dw, *dob, *dbias = nullptr;
  int r;
  if ((r = get_buf(e, "t.ci", (size_t)H * W * cin * 2, &di))) return r;
  if ((r = get_buf(e, "t.cw", (size_t)cout * taps * cin * 2, &dw))) return r;
  if ((r = get_buf(e, "t.co", (size_t)H * W * cout * 2, &dob, true))) return r;
  DCK(cudaMemcpyAsync(di, in_nhwc, (size_t)H * W * cin * 2, cudaMemcpyHostToDevice, e->stream));
  DCK(cudaMemcpyAsync(dw, wt, (size_t)cout * taps * cin * 2, cudaMemcpyHostToDevice, e->stream));
  if (bias) {
    if ((r = get_buf(e, "t.cb", (size_t)cout * 4, &dbias))) return r;
    DCK(cudaMemcpyAsync(dbias, bias, (size_t)cout * 4, cudaMemcpyHostToDevice, e->stream));
  }
  GemmArgs g = base_args(H * W, cout, taps * cin, EPI_F16);
  g.out_f16 = (__half*)dob;
  g.bias = (const float*)dbias;
  g.act = relu ? 2 : 0;
  if ((r = conv(e, (const __half*)di, H, W, cin, (const __half*)dw, k3 != 0, g))) return r;
  std::vector<__half> tmp((size_t)H * W * cout);
  DCK(cudaMemcpyAsync(tmp.data(), dob, tmp.size() * 2, cudaMemcpyDeviceToHost, e->stream));
  DCK(cudaStreamSynchronize(e->stream));
  for (size_t i = 0; i < tmp.size(); ++i) out_host[i] = __half2float(tmp[i]);
  return VD3D_OK;
}

int vd3d_bit_kernel(vd3d_depth* e, int op, const int32_t* d) {
  if (!e || !d || op < 0 || op > 4) return VD3D_ERR_ARG;
  cudaStream_t s = e->stream;
  int r;
  void* out;
  if (op == 4) {
    const int H = d[0], Wd = d[1], cin = d[2], cout = d[3], kind = d[4];
    const bool s2 = kind == BIT_3X3_S2 || kind == BIT_1X1_S2;
    const int taps = (kind == BIT_3X3 || kind == BIT_3X3_S2) ? 9 : 1;
    if (kind < BIT_1X1 || kind > BIT_1X1_S2 || H < 2 || Wd < 2 || (s2 && (H | Wd) & 1) || cin < 64 || cin % 64 ||
        cout < 64 || cout % 64)
      return VD3D_ERR_ARG;
    const int rows = s2 ? (H / 2) * (Wd / 2) : H * Wd;
    const __half *in, *w;
    void* col = nullptr;
    if ((r = W(e, "t.in", &in, (size_t)H * Wd * cin)) || (r = W(e, "t.w", &w, (size_t)cout * taps * cin)) ||
        (r = get_buf(e, "t.out", (size_t)rows * cout * 4, &out)) ||
        (s2 && (r = get_buf(e, "t.col", (size_t)round_up(rows, 128) * taps * cin * 2, &col))))
      return r;
    if ((r = bit_conv(e, kind, in, H, Wd, cin, w, cout, (float*)out, (__half*)col))) return r;
  } else if (op == 0) {
    const int H = d[0], Wd = d[1];
    if (H < 2 || Wd < 2 || (H | Wd) & 1) return VD3D_ERR_ARG;
    const float *in, *w;
    if ((r = W(e, "t.in", &in, (size_t)3 * H * Wd)) || (r = W(e, "t.w", &w, 64 * 147))) return r;
    if ((r = get_buf(e, "t.out", (size_t)(H / 2) * (Wd / 2) * 64 * 4, &out))) return r;
    launch_bit_stem(in, H, Wd, w, (float*)out, s);
  } else if (op == 1) {
    const int rows = d[0], C = d[1], flags = d[2];
    if (rows < 1 || C < 64 || C > 1024 || (C & (C - 1))) return VD3D_ERR_ARG;
    GnInput a, b;
    memset(&b, 0, sizeof b);
    const __half* res = nullptr;
    void *p0, *p1;
    if ((r = W(e, "t.in", &a.y, (size_t)rows * C)) || (r = W(e, "t.g", &a.gamma, C)) || (r = W(e, "t.b", &a.beta, C)))
      return r;
    if ((flags & 2) && ((r = W(e, "t.in2", &b.y, (size_t)rows * C)) || (r = W(e, "t.g2", &b.gamma, C)) ||
                        (r = W(e, "t.b2", &b.beta, C))))
      return r;
    if ((flags & 4) && (r = W(e, "t.res", &res, (size_t)rows * C))) return r;
    if ((r = get_buf(e, "t.out", (size_t)rows * C * 2, &out)) ||
        (r = get_buf(e, "t.part", (size_t)kGnMaxChunks * 32 * sizeof(float2), &p0)) ||
        (r = get_buf(e, "t.part2", (size_t)kGnMaxChunks * 32 * sizeof(float2), &p1)))
      return r;
    a.part = (const float2*)p0;
    b.part = (const float2*)p1;
    launch_gn_stats(a.y, rows, C, (float2*)p0, s);
    if (b.y) launch_gn_stats(b.y, rows, C, (float2*)p1, s);
    launch_gn_apply(a, b, res, flags & 1, rows, C, (__half*)out, s);
  } else {
    const int H = d[0], Wd = d[1], C = d[2], k = op == 3 ? d[3] : 3, pb = op == 3 ? d[4] : 0;
    if (H < 2 || Wd < 2 || (H | Wd) & 1 || C < 8 || C % 8 || (k != 1 && k != 3) || pb < 0 || pb >= k) return VD3D_ERR_ARG;
    const __half* in;
    if ((r = W(e, "t.in", &in, (size_t)H * Wd * C))) return r;
    if ((r = get_buf(e, "t.out", (size_t)(H / 2) * (Wd / 2) * (op == 3 ? k * k : 1) * C * 2, &out))) return r;
    if (op == 2)
      launch_maxpool_same(in, H, Wd, C, (__half*)out, s);
    else
      launch_im2col_same(in, H, Wd, C, k, pb, (__half*)out, s);
  }
  DCK(cudaGetLastError());
  DCK(cudaStreamSynchronize(s));
  return VD3D_OK;
}

// unit-test hook: one ZoeDepth kernel on uploaded "t.*" tensors (vd3d.h vd3d_zoe_kernel), output in "t.out"
int vd3d_zoe_kernel(vd3d_depth* e, int op, const int32_t* d) {
  if (!e || !d || op < 0 || op > 3) return VD3D_ERR_ARG;
  cudaStream_t s = e->stream;
  int r;
  void *out, *route;
  if ((r = get_buf(e, "t.route", 16, &route))) return r;
  if (op == 0) {
    const int h = d[0], w = d[1], OH = d[2], OW = d[3];
    const uint8_t* img;
    if (h < 2 || w < 2 || OH < 1 || OW < 1) return VD3D_ERR_ARG;
    if ((r = W(e, "t.img", &img, (size_t)h * w * 3)) || (r = get_buf(e, "t.out", (size_t)3 * OH * OW * 4, &out))) return r;
    launch_zoe_preprocess(img, h, w, d[4] != 0, zoe_pad(h), zoe_pad(w), (float*)out, OH, OW, e->pre, s);
  } else if (op == 1) {
    const int n = d[0], F = d[1];
    const float *x, *wt, *pe;
    if (n < 1 || F < 64 || F % 64) return VD3D_ERR_ARG;
    if ((r = W(e, "t.x", &x, (size_t)n * F)) || (r = W(e, "t.w", &wt, zoe_router_floats(F))) ||
        (r = W(e, "t.pe", &pe, (size_t)(n + 1) * kZoeE)))
      return r;
    void* scratch;
    if ((r = get_buf(e, "t.scratch", zoe_router_scratch(n) * 4, &scratch)) || (r = get_buf(e, "t.out", 8, &out))) return r;
    launch_zoe_router(x, n, F, wt, pe, (float*)scratch, (float*)out, (int*)route, s);
  } else {
    const int H = d[0], Wd = d[1], Hp = d[2], Wp = d[3], nc = d[4], rt = d[5];
    if (H < 1 || Wd < 1 || Hp < 1 || Wp < 1 || (nc != 1 && nc != 2) || rt < 0 || rt >= nc) return VD3D_ERR_ARG;
    DCK(cudaMemcpyAsync(route, &rt, 4, cudaMemcpyHostToDevice, s));
    if (op == 2) {  // d[6] attractors, d[7] 1: prev is the seed regressor's raw conv2 of every configuration
      const int na = d[6], seed = d[7] != 0, ldp = seed ? nc * kZoeBins : kZoeBins;
      const __half* hid;
      const float *w2, *b2, *prev;
      if (na < 1 || na > kZoeMaxAttr) return VD3D_ERR_ARG;
      if ((r = W(e, "t.hid", &hid, (size_t)H * Wd * nc * kZoeE)) || (r = W(e, "t.w2", &w2, (size_t)nc * na * kZoeE)) ||
          (r = W(e, "t.b2", &b2, (size_t)nc * na)) || (r = W(e, "t.prev", &prev, (size_t)Hp * Wp * ldp)) ||
          (r = get_buf(e, "t.out", (size_t)H * Wd * kZoeBins * 4, &out)))
        return r;
      launch_zoe_attractor(hid, nc * kZoeE, kZoeE, w2, b2, na, prev, ldp, seed ? kZoeBins : 0, seed, Hp, Wp, (float*)out,
                           H, Wd, (const int*)route, s);
    } else {  // d[6] 1: the relative depth is the 33rd input; d[7] hidden units; t.temp f32 {min_temp, max_temp}
      const int cat = d[6] != 0, hid = d[7], cin = 32 + cat + kZoeE;
      const __half *act, *emb;
      const float *w3 = nullptr, *b3 = nullptr, *bins, *lb, *temp;
      if (hid != 40 && hid != 80) return VD3D_ERR_ARG;
      if ((r = W(e, "t.act", &act, (size_t)H * Wd * 32)) || (r = W(e, "t.emb", &emb, (size_t)Hp * Wp * kZoeE)) ||
          (r = W(e, "t.bins", &bins, (size_t)Hp * Wp * kZoeBins)) ||
          (r = W(e, "t.lb", &lb, (size_t)nc * zoe_logbinom_floats(cin, hid))) || (r = W(e, "t.temp", &temp, 2)) ||
          (cat && ((r = W(e, "t.w3", &w3, 32)) || (r = W(e, "t.b3", &b3, 1)))) ||
          (r = get_buf(e, "t.out", (size_t)H * Wd * 4, &out)))
        return r;
      float tt[2];
      DCK(cudaMemcpy(tt, temp, 8, cudaMemcpyDeviceToHost));
      DCK(launch_zoe_logbinom(act, w3, b3, emb, bins, Hp, Wp, kZoeE, lb, cin, hid, tt[0], tt[1], (float*)out, H, Wd,
                              (const int*)route, s));
    }
  }
  DCK(cudaGetLastError());
  DCK(cudaStreamSynchronize(s));
  return VD3D_OK;
}

}  // extern "C"

namespace {

constexpr int kMaxBatch = 8;

// ---- DPT-Hybrid (MiDaS 3.0): the BiT ResNet-50 front end, stem + stages 1-3 (depths 3 / 4 / 9, widths 256 / 512 /
// 1024, bottleneck mids a quarter of that, 32 groups), on one image of side S = IH = IW (a multiple of 32).
// transformers 5.5 BitEmbeddings / BitBottleneckLayer / BitDownsampleConv with global_padding "SAME":
//   stem  = maxpool3x3s2_SAME(relu(GN(conv7x7s2_SAME(px))))                                        -> [S/4]^2 x 64
//   block = relu(GN3(conv1x1(relu(GN2(conv3x3_s(relu(GN1(conv1x1(x)))))))) + shortcut)
//   shortcut = GN(conv1x1_s(x)) on the first block of a stage (stride 1, 2, 2), x on the others.
// Every conv is weight-standardised at load time (depth_weights.prepare_dpt_hybrid) and has no bias.  The stem conv runs
// in f32 on the CUDA cores; the others on k_umma_gemm (f16 operands, f32 output for the GroupNorm): 1x1 convs as plain
// GEMMs on the NHWC row matrix, stride-1 3x3 convs on the implicit-GEMM conv, and the stride-2 3x3 conv (SAME: 0 before,
// 1 after) and stride-2 1x1 shortcut on k_im2col_same's rows.  Block outputs are f16 NHWC.
// Weights: "bit.stem.w" f32 [64, 147], "bit.s{st}.b{k}.c{1,2,3}.w" f16 ([mid, cin], [mid, 9 mid] tap-major, [out, mid]),
// ".n{1,2,3}.g/.b" f32, first blocks ".ds.w" f16 [out, cin] and ".ds.g/.b"; "bit.stem.g/.b".
// Outputs: maps[0] = stage1 f16 [(S/4)^2, 256] and maps[1] = stage2 f16 [(S/8)^2, 512] in the per-image buffers
// "bit.stage1.{b}" / "bit.stage2.{b}" (neck inputs 0 and 1), maps[2] = stage3 f16 [(S/16)^2, 1024] in a scratch
// buffer (the patch projection's input).  The image's launches run in order on the engine stream with shared scratch
// buffers: "bit.y" / "bit.y2" (f32 conv outputs), "bit.t1" / "bit.t2" (f16 mids), "bit.xa" / "bit.xb" (f16 block
// outputs), "bit.col" (im2col), "bit.gn0" / "bit.gn1" (GroupNorm partials).
constexpr int kBitDepths[3] = {3, 4, 9}, kBitWidths[3] = {256, 512, 1024};

int bit_backbone(vd3d_depth* e, int b, const float* px, const __half** maps) {
  cudaStream_t s = e->stream;
  const int S = e->cfg.image_h, S2 = S / 2, S4 = S / 4;
  const size_t big = (size_t)S2 * S2 * 64;  // the largest map: stem output = stage-1 output = stage-2 block 0's conv1
  int r;
  void *y, *y2, *t1, *t2, *xa, *xb, *col, *p0, *p1, *st1, *st2;
  // im2col rows of the stride-2 3x3 convs (stages 2 and 3), rounded up to the GEMM's 128-row tiles
  const size_t col_el = std::max((size_t)round_up((S / 8) * (S / 8), 128) * 9 * 128,
                                 (size_t)round_up((S / 16) * (S / 16), 128) * 9 * 256);
  if ((r = get_buf(e, "bit.y", big * 4, &y)) || (r = get_buf(e, "bit.y2", big * 4, &y2)) ||
      (r = get_buf(e, "bit.t1", big * 2, &t1)) || (r = get_buf(e, "bit.t2", big * 2, &t2)) ||
      (r = get_buf(e, "bit.xa", big * 2, &xa)) || (r = get_buf(e, "bit.xb", big * 2, &xb)) ||
      (r = get_buf(e, "bit.col", col_el * 2, &col)) ||
      (r = get_buf(e, "bit.gn0", (size_t)kGnMaxChunks * 32 * sizeof(float2), &p0)) ||
      (r = get_buf(e, "bit.gn1", (size_t)kGnMaxChunks * 32 * sizeof(float2), &p1)))
    return r;
  if ((r = get_buf(e, fmt("bit.stage1.%d", b), (size_t)S4 * S4 * 256 * 2, &st1)) ||
      (r = get_buf(e, fmt("bit.stage2.%d", b), (size_t)(S / 8) * (S / 8) * 512 * 2, &st2)))
    return r;
  auto gn_in = [&](const char* base, const float* map, const void* part, GnInput* out) -> int {
    int rr;
    if ((rr = W(e, std::string(base) + ".g", &out->gamma)) || (rr = W(e, std::string(base) + ".b", &out->beta)))
      return rr;
    out->y = map;
    out->part = (const float2*)part;
    return VD3D_OK;
  };
  // GroupNorm of one f32 map (and optionally of a second, added) + residual / ReLU -> f16
  auto groupnorm = [&](const char* na, const float* ya, const char* nb, const float* yb, const __half* res, int relu,
                       int rows, int C, __half* out) -> int {
    GnInput ga, gb;
    memset(&gb, 0, sizeof gb);
    int rr;
    if ((rr = gn_in(na, ya, p0, &ga))) return rr;
    if (nb && (rr = gn_in(nb, yb, p1, &gb))) return rr;
    const int sp = e->span_begin("bit.gn", s);
    launch_gn_stats(ya, rows, C, (float2*)p0, s);
    if (nb) launch_gn_stats(yb, rows, C, (float2*)p1, s);
    launch_gn_apply(ga, gb, res, relu, rows, C, out, s);
    e->span_end(sp, s);
    e->launches += nb ? 3 : 2;
    return VD3D_OK;
  };
  // one conv (bit_conv) of an Hin x Hin map with the weight tensor wname
  auto bconv = [&](const std::string& wname, int kind, const __half* in, int Hin, int cin, int cout, float* out) -> int {
    const __half* w;
    int rr;
    const size_t taps = (kind == BIT_3X3 || kind == BIT_3X3_S2) ? 9 : 1;
    if ((rr = W(e, wname, &w, (size_t)cout * taps * cin))) return rr;
    return bit_conv(e, kind, in, Hin, Hin, cin, w, cout, out, (__half*)col);
  };

  // ---- stem ----
  {
    const float* w;
    if ((r = W(e, "bit.stem.w", &w, 64 * 147))) return r;
    int sp = e->span_begin("bit.stem", s);
    launch_bit_stem(px, S, S, w, (float*)y, s);
    e->span_end(sp, s);
    e->launches++;
    if ((r = groupnorm("bit.stem", (const float*)y, nullptr, nullptr, nullptr, 1, S2 * S2, 64, (__half*)t1))) return r;
    sp = e->span_begin("bit.pool", s);
    launch_maxpool_same((const __half*)t1, S2, S2, 64, (__half*)xa, s);
    e->span_end(sp, s);
    e->launches++;
  }
  // ---- stages ----
  const __half* x = (const __half*)xa;
  int H = S4, cin = 64;
  for (int st = 0; st < 3; ++st) {
    const int out_c = kBitWidths[st], mid = out_c / 4;
    for (int k = 0; k < kBitDepths[st]; ++k) {
      const bool first = k == 0, s2 = first && st > 0;
      const int Ho = s2 ? H / 2 : H, rows_in = H * H, rows = Ho * Ho;
      const std::string pfx = fmt("bit.s%d.b%d.", st, k);
      auto wn = [&](const char* suffix) { return pfx + suffix; };
      // conv1 (1x1) + GN1 + ReLU at the input resolution
      if ((r = bconv(wn("c1.w"), BIT_1X1, x, H, cin, mid, (float*)y))) return r;
      if ((r = groupnorm(wn("n1").c_str(), (const float*)y, nullptr, nullptr, nullptr, 1, rows_in, mid, (__half*)t1)))
        return r;
      // conv2 (3x3, stride 1 or 2) + GN2 + ReLU
      if ((r = bconv(wn("c2.w"), s2 ? BIT_3X3_S2 : BIT_3X3, (const __half*)t1, H, mid, mid, (float*)y))) return r;
      if ((r = groupnorm(wn("n2").c_str(), (const float*)y, nullptr, nullptr, nullptr, 1, rows, mid, (__half*)t2)))
        return r;
      // conv3 (1x1) -> y; the first block's shortcut conv -> y2
      if ((r = bconv(wn("c3.w"), BIT_1X1, (const __half*)t2, Ho, mid, out_c, (float*)y))) return r;
      __half* out = (k == kBitDepths[st] - 1 && st < 2) ? (__half*)(st == 0 ? st1 : st2)
                                                        : (__half*)(x == (const __half*)xa ? xb : xa);
      if (first) {
        if ((r = bconv(wn("ds.w"), s2 ? BIT_1X1_S2 : BIT_1X1, x, H, cin, out_c, (float*)y2))) return r;
        if ((r = groupnorm(wn("n3").c_str(), (const float*)y, wn("ds").c_str(), (const float*)y2, nullptr, 1, rows,
                           out_c, out)))
          return r;
      } else {
        if ((r = groupnorm(wn("n3").c_str(), (const float*)y, nullptr, nullptr, x, 1, rows, out_c, out))) return r;
      }
      x = out;
      H = Ho;
      cin = out_c;
    }
  }
  maps[0] = (const __half*)st1;
  maps[1] = (const __half*)st2;
  maps[2] = x;
  return VD3D_OK;
}

// an activation map of one image: NHWC f16 [h, w, C]
struct Map {
  const __half* p;
  int h, w;
};

// the per-image tail of a batch (neck, fusion, head): the stream of its launches and the suffix of its activation
// buffers ("#b" for image b when the tails of a batch run concurrently, else none)
struct Tail {
  cudaStream_t s;
  std::string sfx;
  std::string name(const std::string& base) const { return base + sfx; }
};

// ---- ZoeDepth's metric head (transformers 5.5 ZoeDepthMultipleMetricDepthEstimationHeads / ...MetricDepthEstimationHead)
// on one image, on the stream of its tail.  bott: neck.convs[3]'s output f16 [bh bw, F]; fused[j]: the fusion outputs
// (coarse to fine); act: the relative head's conv2 + ReLU f16 [IH IW, 32]; depth f32 [IH, IW].  The route is a device int
// (the router's argmax, or 0 for a single configuration) that the configuration-specific kernels read: no host
// synchronisation.  The config-independent 1x1 layers run on k_umma_gemm; the seed regressor's and the attractors' conv1,
// whose inputs do not depend on the route, run every configuration in one GEMM (weights concatenated along N; the seed
// conv2 block-diagonal) and the consumer reads the route's columns.
// Weights ("z.*", depth_weights.prepare_zoedepth): z.bt (bottleneck conv2), z.s1 / z.s2 (seed regressor), z.sp1 / z.sp2
// (seed projector), z.p{j}.1 / .2 (projectors), z.a{j}.1 (attractor conv1, f16) and z.a{j}.2.w / .b (attractor conv2,
// f32 [nc][na][E] / [nc][na]), z.lb (log-binomial MLPs, f32 [nc][zoe_logbinom_floats]), z.router and z.r.pe (router).
size_t wlen(vd3d_depth* e, const char* name) {
  auto it = e->w.find(name);
  return it == e->w.end() ? 0 : it->second.bytes / 4;
}
int zoe_head(vd3d_depth* e, const Tail& t, Map bott, const Map* fused, const __half* act, float* depth) {
  cudaStream_t s = t.s;
  const int F = e->cfg.fusion, NC = e->zoe_nc, E = kZoeE, NB = kZoeBins, IH = e->cfg.image_h, IW = e->cfg.image_w;
  const int bh = bott.h, bw = bott.w, nb3 = bh * bw;
  const int ms = (int)(wlen(e, "z.s1.b") / NC), mp = (int)wlen(e, "z.sp1.b");
  const int cin = 32 + e->zoe_cat + E;
  const int hid = (int)((wlen(e, "z.lb") / NC - 4) / (cin + 5));
  if (ms % 64 || mp % 64 || !ms || !mp || (hid != 40 && hid != 80) ||
      wlen(e, "z.lb") != (size_t)NC * zoe_logbinom_floats(cin, hid))
    return dfail(e, VD3D_ERR_STATE, "ZoeDepth: metric head tensors missing or of unserved sizes");
  int r;
  auto buf = [&](const char* base, size_t bytes, void** p) { return get_buf(e, t.name(base), bytes, p); };
  // 1x1 layer on k_umma_gemm: out = act(A W^T + b) [+ res], f16 (or f32 when out32)
  auto lin = [&](const __half* A, int M, int K, const __half* w, const float* bias, int N, int relu, void* out,
                 bool out32, const __half* res) {
    GemmArgs g = base_args(M, N, K, out32 ? EPI_F32 : EPI_F16);
    if (out32)
      g.out_f32 = (float*)out;
    else
      g.out_f16 = (__half*)out;
    g.bias = bias;
    g.act = relu ? 2 : 0;
    g.res_f16 = res;
    return gemm(e, A, K, w, K, g);
  };
  const size_t R3 = round_up(nb3, 128);
  void *zb16, *zb32, *route, *logits, *sh, *seed, *t1, *emb[2], *bins[2], *up, *x, *hb;
  const size_t Mmax = (size_t)round_up(fused[3].h * fused[3].w, 128);
  if ((r = buf("z.zb16", R3 * F * 2, &zb16)) || (r = buf("z.zb32", R3 * F * 4, &zb32)) ||
      (r = buf("z.route", 16, &route)) || (r = buf("z.logits", 16, &logits)) ||
      (r = buf("z.sh", R3 * NC * ms * 2, &sh)) || (r = buf("z.seed", R3 * NC * NB * 4, &seed)) ||
      (r = buf("z.t1", Mmax * std::max(mp, ms) * 2, &t1)) || (r = buf("z.emb0", Mmax * E * 2, &emb[0])) ||
      (r = buf("z.emb1", Mmax * E * 2, &emb[1])) || (r = buf("z.bins0", Mmax * NB * 4, &bins[0])) ||
      (r = buf("z.bins1", Mmax * NB * 4, &bins[1])) || (r = buf("z.up", Mmax * E * 2, &up)) ||
      (r = buf("z.x", Mmax * E * 2, &x)) || (r = buf("z.hid", Mmax * NC * E * 2, &hb)))
    return r;
  const __half* w16;
  const float* b32;
  // ---- bottleneck conv2 (f16 for the GEMMs, f32 for the router), router, seed regressor, seed projector ----
  int sp = e->span_begin("zoe.bottleneck", s);
  if ((r = layer(e, "z.bt", &w16, (size_t)F * F, &b32, F)) ||
      (r = lin(bott.p, nb3, F, w16, b32, F, 0, zb16, false, nullptr)) ||
      (r = lin(bott.p, nb3, F, w16, b32, F, 0, zb32, true, nullptr)))
    return r;
  e->span_end(sp, s);
  sp = e->span_begin("zoe.router", s);
  if (NC == 2) {
    const float *rw, *pe;
    if ((r = W(e, "z.router", &rw, zoe_router_floats(F))) || (r = W(e, "z.r.pe", &pe, (size_t)(nb3 + 1) * E))) return r;
    void* scratch;
    if ((r = buf("z.rscratch", zoe_router_scratch(nb3) * 4, &scratch))) return r;
    launch_zoe_router((const float*)zb32, nb3, F, rw, pe, (float*)scratch, (float*)logits, (int*)route, s);
    e->launches++;
  } else {
    DCK(cudaMemsetAsync(route, 0, 16, s));
  }
  e->span_end(sp, s);
  sp = e->span_begin("zoe.seed", s);
  if ((r = layer(e, "z.s1", &w16, (size_t)NC * ms * F, &b32, NC * ms)) ||
      (r = lin((const __half*)zb16, nb3, F, w16, b32, NC * ms, 1, sh, false, nullptr)) ||
      (r = layer(e, "z.s2", &w16, (size_t)NC * NB * NC * ms, &b32, NC * NB)) ||
      (r = lin((const __half*)sh, nb3, NC * ms, w16, b32, NC * NB, 0, seed, true, nullptr)) ||
      (r = layer(e, "z.sp1", &w16, (size_t)mp * F, &b32, mp)) ||
      (r = lin((const __half*)zb16, nb3, F, w16, b32, mp, 1, t1, false, nullptr)) ||
      (r = layer(e, "z.sp2", &w16, (size_t)E * mp, &b32, E)) ||
      (r = lin((const __half*)t1, nb3, mp, w16, b32, E, 0, emb[1], false, nullptr)))
    return r;
  e->span_end(sp, s);
  // ---- four attractor layers, coarse to fine ----
  int ph_ = bh, pw_ = bw;
  for (int j = 0; j < 4; ++j) {
    const int H = fused[j].h, Wd = fused[j].w, M = H * Wd;
    void *cur = emb[j & 1], *prev = emb[(j + 1) & 1];
    sp = e->span_begin("zoe.proj", s);
    if ((r = layer(e, fmt("z.p%d.1", j), &w16, (size_t)mp * F, &b32, mp)) ||
        (r = lin(fused[j].p, M, F, w16, b32, mp, 1, t1, false, nullptr)))
      return r;
    launch_upsample_ac((const __half*)prev, ph_, pw_, E, (__half*)up, H, Wd, s);
    e->launches++;
    if ((r = layer(e, fmt("z.p%d.2", j), &w16, (size_t)E * mp, &b32, E)) ||
        (r = lin((const __half*)t1, M, mp, w16, b32, E, 0, x, false, (const __half*)up)) ||
        (r = lin((const __half*)t1, M, mp, w16, b32, E, 0, cur, false, nullptr)))
      return r;
    e->span_end(sp, s);
    sp = e->span_begin("zoe.attractor", s);
    if ((r = layer(e, fmt("z.a%d.1", j), &w16, (size_t)NC * E * E, &b32, NC * E)) ||
        (r = lin((const __half*)x, M, E, w16, b32, NC * E, 1, hb, false, nullptr)))
      return r;
    const float *w2, *b2;
    const int na = e->zoe_na[j];
    if ((r = W(e, fmt("z.a%d.2.w", j), &w2, (size_t)NC * na * E)) ||
        (r = W(e, fmt("z.a%d.2.b", j), &b2, (size_t)NC * na)))
      return r;
    if (j == 0)
      launch_zoe_attractor((const __half*)hb, NC * E, E, w2, b2, na, (const float*)seed, NC * NB, NB, 1, bh, bw,
                           (float*)bins[0], H, Wd, (const int*)route, s);
    else
      launch_zoe_attractor((const __half*)hb, NC * E, E, w2, b2, na, (const float*)bins[(j + 1) & 1], NB, 0, 0, ph_, pw_,
                           (float*)bins[j & 1], H, Wd, (const int*)route, s);
    e->launches++;
    e->span_end(sp, s);
    ph_ = H;
    pw_ = Wd;
  }
  // ---- conditional log-binomial + expectation at the processed size ----
  const float *lb, *w3 = nullptr, *b3 = nullptr;
  if ((r = W(e, "z.lb", &lb)) || (e->zoe_cat && ((r = W(e, "h.c3.w", &w3, 32)) || (r = W(e, "h.c3.b", &b3, 1)))))
    return r;
  sp = e->span_begin("zoe.logbinom", s);
  cudaError_t ce = launch_zoe_logbinom(act, w3, b3, (const __half*)emb[1], (const float*)bins[1], ph_, pw_, E, lb, cin,
                                       hid, e->zoe_tmin, e->zoe_tmax, depth, IH, IW, (const int*)route, s);
  if (ce != cudaSuccess) return dfail(e, VD3D_ERR_CUDA, std::string("zoe log-binomial launch: ") + cudaGetErrorString(ce));
  e->launches++;
  e->span_end(sp, s);
  return VD3D_OK;
}

// One forward of B images (forward_core).  The token-wise stages (LayerNorm, QKV / proj / fc1 / fc2 GEMMs) see one
// matrix of MT = (B-1)*NP + NT rows -- image b owns rows [b*NP, b*NP + NT), NP = NT rounded up to the 128-row tile --
// so the GEMMs run at 3-4x the rows of one frame (the reference batches too: core/render_depth.py:1113-1119);
// attention runs with grid.y = B * heads; patch embedding, taps, neck and head stay per image (their maps are
// per-image 2-D tensors).
struct Fwd {
  int B, MT;
  float* x;                            // residual stream f32 [B*NP, D]
  __half *xn, *q, *k, *vt, *attn, *h;  // LayerNorm output, per-head q / k / v^T, attention output, fc1 output
};

// Patch embedding + CLS + position embeddings of every image into its rows of x.  DPT-Hybrid: the BiT stage-3 map
// [NPATCH, 1024] takes the place of the patch matrix (a 1x1 projection with bias), and the stage-1 / stage-2 maps are
// the image's neck inputs 0 and 1 (in[b][0..1]).
int embed(vd3d_depth* e, const Fwd& f, const float* const* px_dev, const __half* (*in)[4]) {
  cudaStream_t s = e->stream;
  const bool bit = e->traits.bit_front_end;
  const int D = e->cfg.hidden, P = e->patch, NT = e->ntok, NP = e->npad, NPATCH = e->ph * e->pw;
  const int KPE = round_up(3 * P * P, 16);  // 592 for patch 14 (588 + zero columns), 768 for 16
  const int KE = bit ? 1024 : KPE;
  __half* ape = nullptr;
  int r;
  if (!bit && (r = get_buf(e, "ape", (size_t)NPATCH * KPE * 2, &ape))) return r;
  const int sp_embed = bit ? -1 : e->span_begin("embed", s);  // the hybrid's backbone has spans of its own
  const __half* pe_w;
  const float *pe_b, *cls, *pos;
  if ((r = layer(e, "pe", &pe_w, (size_t)D * KE, &pe_b, D)) || (r = W(e, "cls", &cls, D)) ||
      (r = W(e, "pos", &pos, (size_t)NT * D)))
    return r;
  for (int b = 0; b < f.B; ++b) {
    float* xb = f.x + (size_t)b * NP * D;
    const __half* a = ape;
    if (bit) {
      const __half* maps[3];
      if ((r = bit_backbone(e, b, px_dev[b], maps))) return r;
      in[b][0] = maps[0];
      in[b][1] = maps[1];
      a = maps[2];
    } else {
      launch_patch_im2col(px_dev[b], e->cfg.image_h, e->cfg.image_w, e->ph, e->pw, ape, KPE, P, s);
      e->launches++;
    }
    const int sp_proj = bit ? e->span_begin("bit.proj", s) : -1;
    GemmArgs g = base_args(NPATCH, D, KE, EPI_PATCH);
    g.out_f32 = xb;
    g.bias = pe_b;
    g.pos = pos;
    g.ldc = D;
    if ((r = gemm(e, a, KE, pe_w, KE, g))) return r;
    launch_set_cls(xb, cls, pos, D, s);
    e->launches++;
    e->span_end(sp_proj, s);
    // rows [NT, NP) of every image but the last take part in the stacked GEMMs: keep them at zero so that they stay
    // finite from frame to frame (they are never read as keys / values: the attention tensor maps end at NT)
    if (b + 1 < f.B) DCK(cudaMemsetAsync(xb + (size_t)NT * D, 0, (size_t)(NP - NT) * D * 4, s));
  }
  e->span_end(sp_embed, s);
  return VD3D_OK;
}

// Encoder layer l on the stacked token matrix: x += ls1 * proj(attn(LN1(x))); x += ls2 * fc2(GELU(fc1(LN2(x)))).
// BEiT adds the layer's relative position bias to the attention scores.
int encoder_layer(vd3d_depth* e, const Fwd& f, int l) {
  cudaStream_t s = e->stream;
  const int D = e->cfg.hidden, Hh = e->cfg.heads, MT = f.MT, NT = e->ntok, NP = e->npad;
  const float *g1, *b1, *g2, *b2, *bqkv, *bo, *ls1, *bf1, *bf2, *ls2;
  const __half *wqkv, *wo, *wf1, *wf2;
  auto nmf = [&](const char* suffix) { return fmt("l%d.", l) + suffix; };
  int r;
  if ((r = W(e, nmf("ln1.g"), &g1, D)) || (r = W(e, nmf("ln1.b"), &b1, D)) || (r = W(e, nmf("ln2.g"), &g2, D)) ||
      (r = W(e, nmf("ln2.b"), &b2, D)) || (r = layer(e, nmf("qkv"), &wqkv, (size_t)3 * D * D, &bqkv, 3 * D)) ||
      (r = layer(e, nmf("proj"), &wo, (size_t)D * D, &bo, D)) || (r = W(e, nmf("ls1"), &ls1, D)) ||
      (r = layer(e, nmf("fc1"), &wf1, (size_t)4 * D * D, &bf1, 4 * D)) ||
      (r = layer(e, nmf("fc2"), &wf2, (size_t)4 * D * D, &bf2, D)) || (r = W(e, nmf("ls2"), &ls2, D)))
    return r;
  // BEiT: the layer's relative position bias, one table per head for this grid
  const float* rpb = nullptr;
  if (e->traits.rel_pos_bias &&
      (r = W(e, nmf("rpb"), &rpb, (size_t)Hh * ((2 * e->ph - 1) * (2 * e->pw - 1) + 3))))
    return r;
  int sp = e->span_begin("ln", s);
  launch_layernorm(f.x, MT, D, g1, b1, f.xn, 0, e->ln_eps, s);
  e->launches++;
  e->span_end(sp, s);
  sp = e->span_begin("qkv", s);
  GemmArgs g = base_args(MT, 3 * D, D, EPI_QKV);
  g.bias = bqkv;
  g.q = f.q;
  g.k = f.k;
  g.vt = f.vt;
  g.heads = Hh;
  g.npad = NP;
  g.dmodel = D;
  g.qscale = 0.125f;  // 1/sqrt(64), exact in f16
  if ((r = gemm(e, f.xn, D, wqkv, D, g))) return r;
  e->span_end(sp, s);
  // fused wgmma attention: scores and probabilities stay in registers
  sp = e->span_begin("attn", s);
  CUtensorMap mq, mk, mv;
  if ((r = make_map(e, &mq, f.q, 64, NT, f.B * Hh, 64, (uint64_t)NP * 64, kAttnRows, 1)) ||
      (r = make_map(e, &mk, f.k, 64, NT, f.B * Hh, 64, (uint64_t)NP * 64, 128, 1)) ||
      (r = make_map(e, &mv, f.vt, NT, 64, f.B * Hh, NP, (uint64_t)64 * NP, 64, 1)))
    return r;
  cudaError_t ce = launch_attention(mq, mk, mv, NT, D, f.attn, Hh, f.B, NP, s, rpb, e->pw);
  if (ce != cudaSuccess) return dfail(e, VD3D_ERR_CUDA, std::string("attention launch: ") + cudaGetErrorString(ce));
  e->launches++;
  e->span_end(sp, s);
  sp = e->span_begin("proj", s);
  g = base_args(MT, D, D, EPI_RESID_LS);
  g.out_f32 = f.x;
  g.bias = bo;
  g.ls = ls1;
  g.ldc = D;
  if ((r = gemm(e, f.attn, D, wo, D, g))) return r;
  e->span_end(sp, s);
  sp = e->span_begin("ln", s);
  launch_layernorm(f.x, MT, D, g2, b2, f.xn, 0, e->ln_eps, s);
  e->launches++;
  e->span_end(sp, s);
  sp = e->span_begin("fc1", s);
  g = base_args(MT, 4 * D, D, EPI_F16);
  g.out_f16 = f.h;
  g.bias = bf1;
  g.act = 1;
  g.ldc = 4 * D;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (e->prof) {
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    cudaEventRecord(e0, s);
    e->prof_rows += MT;
  }
  if ((r = gemm(e, f.xn, D, wf1, D, g))) return r;
  if (e->prof) {
    cudaEventRecord(e1, s);
    e->prof_ev.push_back(e0);
    e->prof_ev.push_back(e1);
  }
  e->span_end(sp, s);
  sp = e->span_begin("fc2", s);
  g = base_args(MT, D, 4 * D, EPI_RESID_LS);
  g.out_f32 = f.x;
  g.bias = bf2;
  g.ls = ls2;
  g.ldc = D;
  if ((r = gemm(e, f.h, 4 * D, wf2, 4 * D, g))) return r;
  e->span_end(sp, s);
  return VD3D_OK;
}

// Neck input i of every image (in[b][i]), taken after its encoder layer.  DPT (readout): the raw residual stream
// (hidden_states[l + 1]), then the project readout over the patch rows of all images in one GEMM,
// GELU(W_t tok + (W_c cls_b + bias)), the CLS term computed once per image; image b's rows start at b * NPATCH.
// Depth-Anything: the backbone output, final LayerNorm applied (apply_layernorm=True) per image, CLS dropped.
int take_tap(vd3d_depth* e, const Fwd& f, int i, const __half* (*in)[4]) {
  cudaStream_t s = e->stream;
  const int D = e->cfg.hidden, NP = e->npad, NPATCH = e->ph * e->pw;
  int r;
  if (e->traits.readout) {
    __half *tp, *ro;
    float* cb;
    const __half *wt, *wc;
    const float* rb;
    const int MR = f.B * NPATCH;
    if ((r = W(e, fmt("ro%d.wt", i), &wt, (size_t)D * D)) || (r = W(e, fmt("ro%d.wc", i), &wc, (size_t)D * D)) ||
        (r = W(e, fmt("ro%d.b", i), &rb, D)) ||
        (r = get_buf(e, fmt("tap%d", i), (size_t)round_up(MR, 128) * D * 2, &tp)) ||
        (r = get_buf(e, fmt("ro%d.c", i), (size_t)f.B * D * 4, &cb)) ||
        (r = get_buf(e, fmt("ro%d", i), (size_t)round_up(MR, 128) * D * 2, &ro)))
      return r;
    launch_tap_f16(f.x, NP, NPATCH, D, f.B, tp, s);
    e->launches++;
    launch_readout_cls(f.x, NP, D, f.B, wc, rb, D, cb, s);
    e->launches++;
    GemmArgs g = base_args(MR, D, D, EPI_READOUT);
    g.out_f16 = ro;
    g.img_bias = cb;
    g.npad = NPATCH;
    g.ldc = D;
    if ((r = gemm(e, tp, D, wt, D, g))) return r;
    for (int b = 0; b < f.B; ++b) in[b][i] = ro + (size_t)b * NPATCH * D;
    return VD3D_OK;
  }
  const float *ng, *nb;
  if ((r = W(e, "norm.g", &ng, D)) || (r = W(e, "norm.b", &nb, D))) return r;
  for (int b = 0; b < f.B; ++b) {
    __half* tp;
    if ((r = get_buf(e, fmt("tap%d.%d", i, b), (size_t)round_up(NPATCH, 128) * D * 2, &tp))) return r;
    launch_layernorm(f.x + (size_t)b * NP * D, NPATCH, D, ng, nb, tp, 1, e->ln_eps, s);
    e->launches++;
    in[b][i] = tp;
  }
  return VD3D_OK;
}

// Reassemble stage i of one image: the 1x1 projection of its token rows tok [NPATCH, D] to CP channels, then the
// resample to the stage's scale: ConvTranspose2d (kernel = stride = 4 / 2), none, or Conv2d (3x3, stride 2, pad 1)
int reassemble(vd3d_depth* e, const Tail& t, int i, const __half* tok, Map* out) {
  const int D = e->cfg.hidden, ph = e->ph, pw = e->pw, NPATCH = ph * pw, CP = round_up(e->cfg.neck[i], 64);
  const __half* wp;
  const float* bp;
  __half *rp, *rs;
  int r;
  if ((r = layer(e, fmt("r%d.proj", i), &wp, (size_t)CP * D, &bp, CP)) ||
      (r = get_buf(e, t.name(fmt("r%d.p", i)), (size_t)round_up(NPATCH, 128) * CP * 2, &rp)))
    return r;
  GemmArgs g = base_args(NPATCH, CP, D, EPI_F16);
  g.out_f16 = rp;
  g.bias = bp;
  g.ldc = CP;
  if ((r = gemm(e, tok, D, wp, D, g))) return r;
  if (i == 2) {
    *out = {rp, ph, pw};
    return VD3D_OK;
  }
  if (i < 2) {
    const int kk = (i == 0) ? 4 : 2;
    const __half* uw;
    const float* ub;
    if ((r = layer(e, fmt("r%d.up", i), &uw, (size_t)kk * kk * CP * CP, &ub, (size_t)kk * kk * CP)) ||
        (r = get_buf(e, t.name(fmt("r%d.s", i)), (size_t)ph * kk * pw * kk * CP * 2, &rs)))
      return r;
    g = base_args(NPATCH, kk * kk * CP, CP, EPI_CONVT);
    g.out_f16 = rs;
    g.bias = ub;
    g.ct_k = kk;
    g.ct_cout = CP;
    g.ct_w = pw;
    if ((r = gemm(e, rp, CP, uw, CP, g))) return r;
    *out = {rs, ph * kk, pw * kk};
    return VD3D_OK;
  }
  const __half* dw;
  const float* db;
  const int oh = (ph - 1) / 2 + 1, ow = (pw - 1) / 2 + 1;
  __half* col;
  if ((r = layer(e, "r3.down", &dw, (size_t)CP * 9 * CP, &db, CP)) ||
      (r = get_buf(e, t.name("r3.col"), (size_t)round_up(oh * ow, 128) * 9 * CP * 2, &col)))
    return r;
  launch_im2col_s2(rp, ph, pw, CP, CP, col, oh, ow, t.s);
  e->launches++;
  if ((r = get_buf(e, t.name("r3.s"), (size_t)round_up(oh * ow, 128) * CP * 2, &rs))) return r;
  g = base_args(oh * ow, CP, 9 * CP, EPI_F16);
  g.out_f16 = rs;
  g.bias = db;
  g.ldc = CP;
  if ((r = gemm(e, col, 9 * CP, dw, 9 * CP, g))) return r;
  *out = {rs, oh, ow};
  return VD3D_OK;
}

// The neck of one image: each input reassembled to its scale (DPT-Hybrid's BiT stage maps, inputs 0 and 1, are at
// theirs already), then the 3x3 conv to the fusion width -> feat[i] ("f{i}")
int neck(vd3d_depth* e, const Tail& t, const __half* const* in, Map* feat) {
  const int F = e->cfg.fusion;
  int r;
  for (int i = 0; i < 4; ++i) {
    const int CP = round_up(e->cfg.neck[i], 64);
    Map m;
    if (e->traits.bit_front_end && i < 2)
      m = {in[i], e->ph * (4 >> i), e->pw * (4 >> i)};
    else if ((r = reassemble(e, t, i, in[i], &m)))
      return r;
    const __half* cw;
    __half* out;
    if ((r = W(e, fmt("n%d.conv.w", i), &cw, (size_t)F * 9 * CP)) ||
        (r = get_buf(e, t.name(fmt("f%d", i)), (size_t)m.h * m.w * F * 2, &out)))
      return r;
    GemmArgs g = base_args(0, F, 0, EPI_F16);
    g.out_f16 = out;
    g.ldc = F;
    if ((r = conv(e, m.p, m.h, m.w, CP, cw, true, g))) return r;
    feat[i] = {out, m.h, m.w};
  }
  return VD3D_OK;
}

// One ResidualConvUnit ("rl1" / "rl2") of fusion block j on an H x Wd map: out = conv2(relu(conv1(x_relu))) + res,
// x_relu = relu(x) computed by the caller; mid receives conv1's output
int residual_unit(vd3d_depth* e, int j, const char* unit, const __half* x_relu, const __half* res, int H, int Wd,
                  __half* mid, __half* out) {
  const int F = e->cfg.fusion;
  const __half *w1, *w2;
  const float *b1, *b2;
  const std::string base = fmt("f%d.", j) + unit;
  int r;
  if ((r = layer(e, base + ".c1", &w1, (size_t)F * 9 * F, &b1, F)) ||
      (r = layer(e, base + ".c2", &w2, (size_t)F * 9 * F, &b2, F)))
    return r;
  GemmArgs g1 = base_args(0, F, 0, EPI_F16);
  g1.out_f16 = mid;
  g1.bias = b1;
  g1.act = 2;
  g1.ldc = F;
  if ((r = conv(e, x_relu, H, Wd, F, w1, true, g1))) return r;
  GemmArgs g2 = base_args(0, F, 0, EPI_F16);
  g2.out_f16 = out;
  g2.bias = b2;
  g2.res_f16 = res;
  g2.ldc = F;
  return conv(e, mid, H, Wd, F, w2, true, g2);
}

// The fusion stage of one image, coarsest first: block j takes feat[3 - j] (plus, after the first block, the previous
// block's output), upsamples to the next map's size (x2 after the last block) and projects (1x1) -> fused[j]
int fusion(vd3d_depth* e, const Tail& t, const Map* feat, Map* fused) {
  cudaStream_t s = t.s;
  const int F = e->cfg.fusion;
  int r;
  for (int j = 0; j < 4; ++j) {
    const Map& in = feat[3 - j];
    const int Hc = in.h, Wc = in.w;
    const size_t n = (size_t)Hc * Wc * F;
    __half *t_relu, *t_mid, *hraw, *hrelu, *yraw, *up, *prj;
    if ((r = get_buf(e, t.name("fu.relu"), n * 2, &t_relu)) || (r = get_buf(e, t.name("fu.mid"), n * 2, &t_mid)) ||
        (r = get_buf(e, t.name("fu.h"), n * 2, &hraw)) || (r = get_buf(e, t.name("fu.hrelu"), n * 2, &hrelu)) ||
        (r = get_buf(e, t.name("fu.y"), n * 2, &yraw)))
      return r;
    const __half* h = in.p;  // residual_layer2's input; hrelu: its ReLU
    if (j == 0) {
      launch_relu_f16(in.p, hrelu, n, s);
      e->launches++;
    } else {  // h = fused + residual_layer1(feat)
      launch_relu_f16(in.p, t_relu, n, s);
      e->launches++;
      if ((r = residual_unit(e, j, "rl1", t_relu, in.p, Hc, Wc, t_mid, yraw))) return r;
      launch_add_relu_f16(fused[j - 1].p, yraw, hraw, hrelu, n, s);
      e->launches++;
      h = hraw;
    }
    if ((r = residual_unit(e, j, "rl2", hrelu, h, Hc, Wc, t_mid, yraw))) return r;
    const int OH = (j < 3) ? feat[2 - j].h : Hc * 2, OW = (j < 3) ? feat[2 - j].w : Wc * 2;
    if ((r = get_buf(e, t.name(fmt("fu.up%d", j)), (size_t)OH * OW * F * 2, &up))) return r;
    launch_upsample_ac(yraw, Hc, Wc, F, up, OH, OW, s);
    e->launches++;
    const __half* pwt;
    const float* pbs;
    if ((r = layer(e, fmt("f%d.proj", j), &pwt, (size_t)F * F, &pbs, F)) ||
        (r = get_buf(e, t.name(fmt("fused%d", j)), (size_t)round_up(OH * OW, 128) * F * 2, &prj)))
      return r;
    GemmArgs g = base_args(OH * OW, F, F, EPI_F16);
    g.out_f16 = prj;
    g.bias = pbs;
    g.ldc = F;
    if ((r = gemm(e, up, F, pwt, F, g))) return r;
    fused[j] = {prj, OH, OW};
  }
  return VD3D_OK;
}

// The head of one image on the last fusion output: conv1 (3x3), bilinear (align corners) to the processed size, then
// conv2 (3x3) + ReLU with conv3 (1x1) and the last activation in the EPI_HEAD epilogue -> depth f32 [IH, IW].
// ZoeDepth: conv2 + ReLU ("z.act") feeds the metric head, with the bottleneck feat[3] and every fusion output.
int head(vd3d_depth* e, const Tail& t, const Map* feat, const Map* fused, float* depth) {
  const int F = e->cfg.fusion, F2 = round_up(F / 2, 64), IH = e->cfg.image_h, IW = e->cfg.image_w;
  const int ch = fused[3].h, cw = fused[3].w;
  const __half *w1, *w2;
  const float *b1, *b2, *w3, *b3;
  __half *h1, *h1u;
  int r;
  if ((r = layer(e, "h.c1", &w1, (size_t)F2 * 9 * F, &b1, F2)) ||
      (r = layer(e, "h.c2", &w2, (size_t)32 * 9 * F2, &b2, 32)) || (r = W(e, "h.c3.w", &w3, 32)) ||
      (r = W(e, "h.c3.b", &b3, 1)) ||
      (r = get_buf(e, t.name("h1"), (size_t)ch * cw * F2 * 2, &h1)) ||
      (r = get_buf(e, t.name("h1u"), (size_t)IH * IW * F2 * 2, &h1u)))
    return r;
  GemmArgs g1 = base_args(0, F2, 0, EPI_F16);
  g1.out_f16 = h1;
  g1.bias = b1;
  g1.ldc = F2;
  if ((r = conv(e, fused[3].p, ch, cw, F, w1, true, g1))) return r;
  launch_upsample_ac(h1, ch, cw, F2, h1u, IH, IW, t.s);
  e->launches++;
  if (e->traits.zoe_head) {
    __half* act;
    if ((r = get_buf(e, t.name("z.act"), (size_t)IH * IW * 32 * 2, &act))) return r;
    GemmArgs g2 = base_args(0, 32, 0, EPI_F16);
    g2.out_f16 = act;
    g2.bias = b2;
    g2.act = 2;
    g2.ldc = 32;
    if ((r = conv(e, h1u, IH, IW, F2, w2, true, g2, 32))) return r;
    return zoe_head(e, t, feat[3], fused, act, depth);
  }
  GemmArgs g2 = base_args(0, 32, 0, EPI_HEAD);
  g2.out_f32 = depth;
  g2.bias = b2;
  g2.w3 = w3;
  g2.b3p = b3;
  g2.head_max = e->head == VD3D_HEAD_METRIC ? e->max_depth : 0.f;
  return conv(e, h1u, IH, IW, F2, w2, true, g2, 32);
}

// neck, fusion and head of one image, every launch on t.s; in: its four neck inputs
int tail(vd3d_depth* e, const Tail& t, const __half* const* in, float* depth) {
  StreamScope on(e, t.s);
  Map feat[4], fused[4];
  int r;
  if ((r = neck(e, t, in, feat)) || (r = fusion(e, t, feat, fused))) return r;
  return head(e, t, feat, fused, depth);
}

// B images through the network in one pass.  px_dev / depth_dev: DEVICE pointers, f32 [3, image_h, image_w] in, f32
// [image_h, image_w] out.
int forward_core(vd3d_depth* e, int B, const float* const* px_dev, float* const* depth_dev) {
  if (B < 1 || B > kMaxBatch) return dfail(e, VD3D_ERR_ARG, "batch must be in [1, 8]");
  if (e->traits.zoe_head && !e->zoe_nc)
    return dfail(e, VD3D_ERR_STATE, "ZoeDepth: the metric head's settings are not set (vd3d_depth_set_zoe)");
  Fwd f{B, (B - 1) * e->npad + e->ntok};
  const size_t D = e->cfg.hidden, Hh = e->cfg.heads, NP = e->npad;
  const __half* in[kMaxBatch][4];  // the neck inputs of every image
  int r;
  if ((r = get_buf(e, "x", B * NP * D * 4, &f.x)) || (r = get_buf(e, "xn", B * NP * D * 2, &f.xn)) ||
      (r = get_buf(e, "q", B * Hh * NP * 64 * 2, &f.q)) || (r = get_buf(e, "k", B * Hh * NP * 64 * 2, &f.k)) ||
      (r = get_buf(e, "vt", B * Hh * 64 * NP * 2, &f.vt)) || (r = get_buf(e, "attn", B * NP * D * 2, &f.attn)) ||
      (r = get_buf(e, "h", B * NP * 4 * D * 2, &f.h)) || (r = embed(e, f, px_dev, in)))
    return r;
  int tap = e->traits.bit_front_end ? 2 : 0;  // the hybrid's neck inputs 0 and 1 are BiT stages, not taps
  for (int l = 0; l < e->cfg.layers; ++l) {
    if ((r = encoder_layer(e, f, l))) return r;
    if (tap < 4 && e->cfg.taps[tap] == l + 1) {
      if ((r = take_tap(e, f, tap, in))) return r;
      ++tap;
    }
  }
  if (tap != 4) return dfail(e, VD3D_ERR_ARG, "taps must be increasing layer indices <= layers");

  // neck + head: independent per image.  With more than one image each tail runs on its own side stream (forked here,
  // joined below) with its own activation buffers, so that the many small launches of the tails (grids of 5..77 CTAs on
  // the coarse maps) overlap each other instead of leaving most SMs idle; captured into the same CUDA graph.
  const bool fork = B > 1;
  const int sp_tail = e->span_begin("tail(all images, forked)", e->stream);
  if (fork) {
    if (!e->ev_fork) DCK(cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming));
    DCK(cudaEventRecord(e->ev_fork, e->stream));
  }
  for (int b = 0; b < B; ++b) {
    Tail t{e->stream, ""};
    if (fork) {
      if (!e->aux[b]) DCK(cudaStreamCreateWithFlags(&e->aux[b], cudaStreamNonBlocking));
      if (!e->ev_join[b]) DCK(cudaEventCreateWithFlags(&e->ev_join[b], cudaEventDisableTiming));
      t = Tail{e->aux[b], "#" + std::to_string(b)};
      DCK(cudaStreamWaitEvent(t.s, e->ev_fork, 0));
    }
    if ((r = tail(e, t, in[b], depth_dev[b]))) return r;
    if (fork) DCK(cudaEventRecord(e->ev_join[b], t.s));
  }
  if (fork)
    for (int b = 0; b < B; ++b) DCK(cudaStreamWaitEvent(e->stream, e->ev_join[b], 0));
  e->span_end(sp_tail, e->stream);
  DCK(cudaGetLastError());
  return VD3D_OK;
}

// Pillow's precompute_coeffs + normalize_coeffs_8bpc for the bicubic filter (a = -0.5, support 2 widened by the scale
// when shrinking), in double as Pillow computes them: tab = (first input, tap count) per output index, then ksize
// weights per output index in fixed point with 22 fractional bits, rounded away from zero.  Returns ksize.
double pil_bicubic(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}
int pil_bicubic_table(int in_size, int out_size, std::vector<int>& tab) {
  const double scale = (double)in_size / out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = 2.0 * filterscale, ss = 1.0 / filterscale;
  const int ksize = (int)ceil(support) * 2 + 1;
  tab.assign((size_t)out_size * (2 + ksize), 0);
  std::vector<double> w(ksize);
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = (xx + 0.5) * scale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      w[x] = pil_bicubic((x + xmin - center + 0.5) * ss);
      ww += w[x];
    }
    int* k = &tab[(size_t)2 * out_size + (size_t)xx * ksize];
    for (int x = 0; x < xmax; ++x) {
      const double v = ww != 0.0 ? w[x] / ww : w[x];
      k[x] = v < 0 ? (int)(-0.5 + v * (1 << 22)) : (int)(0.5 + v * (1 << 22));
    }
    tab[2 * xx] = xmin;
    tab[2 * xx + 1] = xmax;
  }
  return ksize;
}

// the device table of one (in, out) axis, built and uploaded on first use, then cached by the engine
int pil_table(vd3d_depth* e, int in_size, int out_size, const int** out, int* ksize) {
  const std::string nm = fmt("pil.%d.%d", in_size, out_size);
  const double scale = (double)in_size / out_size;
  *ksize = (int)ceil(2.0 * (scale < 1.0 ? 1.0 : scale)) * 2 + 1;
  const size_t bytes = (size_t)out_size * (2 + *ksize) * sizeof(int);
  void* d;
  int r;
  if (e->buf.find(nm) == e->buf.end()) {
    std::vector<int> tab;
    pil_bicubic_table(in_size, out_size, tab);
    if ((r = get_buf(e, nm, bytes, &d))) return r;
    // pageable source: the copy returns once the table is staged, so `tab` may go out of scope
    DCK(cudaMemcpyAsync(d, tab.data(), bytes, cudaMemcpyHostToDevice, e->stream));
  } else if ((r = get_buf(e, nm, bytes, &d))) {
    return r;
  }
  *out = (const int*)d;
  return VD3D_OK;
}

// Pillow's resize of u8 [h,w,3] -> [oh,ow,3]: width pass into tmp (>= h*ow*3 bytes), then height pass; a pass whose
// axis keeps its size is skipped.  src != dst.
int pil_resize(vd3d_depth* e, const uint8_t* src, int h, int w, uint8_t* tmp, uint8_t* dst, int oh, int ow) {
  const int *tx = nullptr, *ty = nullptr;
  int kx = 0, ky = 0, r;
  if (ow != w && (r = pil_table(e, w, ow, &tx, &kx))) return r;
  if (oh != h && (r = pil_table(e, h, oh, &ty, &ky))) return r;
  cudaStream_t s = e->stream;
  if (ow == w && oh == h) {
    DCK(cudaMemcpyAsync(dst, src, (size_t)h * w * 3, cudaMemcpyDeviceToDevice, s));
    return VD3D_OK;
  }
  if (ow != w) {
    launch_resize_pil_u8(src, h, w, oh == h ? dst : tmp, h, ow, tx, kx, 0, s);
    e->launches++;
    src = tmp;
  }
  if (oh != h) {
    launch_resize_pil_u8(src, h, ow, dst, oh, ow, ty, ky, 1, s);
    e->launches++;
  }
  DCK(cudaGetLastError());
  return VD3D_OK;
}

// (h, w) DPTImageProcessor resizes an image to with keep_aspect_ratio (depth_engine.py processed_size): scale the side
// whose scale to the target (th, tw) is closer to 1 for both, round each to a multiple of `mult` (Python's round: half to
// even), at least `mult`.  Depth-Anything: 518 x 518 and 14; BEiT: the processor's target and 32.
void processed_size(int h, int w, int th, int tw, int mult, int* ph, int* pw) {
  double sh = (double)th / h, sw = (double)tw / w;
  if (fabs(1 - sw) < fabs(1 - sh))
    sh = sw;
  else
    sw = sh;
  auto rnd = [mult](double v) { int r = (int)nearbyint(v / mult) * mult; return r < mult ? mult : r; };
  *ph = rnd(sh * h);
  *pw = rnd(sw * w);
}

// the f32 pixel and depth slots of image b of a forward: "px" / "depth" for the first, "px.{b}" / "depth.{b}" after
int batch_slots(vd3d_depth* e, int b, float** px, float** depth) {
  const size_t n = (size_t)e->cfg.image_h * e->cfg.image_w;
  const int r = get_buf(e, fmt(b ? "px.%d" : "px", b), 3 * n * 4, px);
  return r ? r : get_buf(e, fmt(b ? "depth.%d" : "depth", b), n * 4, depth);
}

// The model's image processor on one u8 image [h, w, 3] (BGR when swap_rb) into its pixel slot px: ZoeDepth's reflect
// padding and resize, or the resize (width pass into tmp, height pass into rgb) and normalisation.  timed: the
// ZoeDepth kernel is a "zoe.preprocess" span
void preprocess(vd3d_depth* e, const uint8_t* img, int h, int w, int swap_rb, void* tmp, void* rgb, float* px,
                bool timed) {
  cudaStream_t s = e->stream;
  const int IH = e->cfg.image_h, IW = e->cfg.image_w;
  if (e->traits.zoe_head) {
    const int sp = timed ? e->span_begin("zoe.preprocess", s) : -1;
    launch_zoe_preprocess(img, h, w, swap_rb, zoe_pad(h), zoe_pad(w), px, IH, IW, e->pre, s);
    e->span_end(sp, s);
    e->launches++;
  } else {
    launch_preprocess(img, h, w, (uint8_t*)tmp, (uint8_t*)rgb, px, IH, IW, s, swap_rb, e->pre);
    e->launches += 3;
  }
}

// The processed-size depth of one image back to its (h, w) input size: the bicubic resize into up f32 [h, w]
// (ZoeDepth: of the reflect-padded size, cropped) with its min / max in mm, and the min-max u8 [h, w] when u8 is set
void postprocess(vd3d_depth* e, const float* depth, int h, int w, float* up, unsigned* mm, uint8_t* u8, int invert) {
  const int pad_h = e->traits.zoe_head ? zoe_pad(h) : 0, pad_w = e->traits.zoe_head ? zoe_pad(w) : 0;
  launch_depth_post_crop(depth, e->cfg.image_h, e->cfg.image_w, up, h, w, pad_h, pad_w, mm, u8, invert, e->stream);
  e->launches += u8 ? 3 : 2;
}

}  // namespace

extern "C" {

// pixel_values: f32 [3, image_h, image_w] (already resized + normalised); depth_out f32 [image_h, image_w]
int vd3d_depth_forward(vd3d_depth* e, const float* pixel_values, float* depth_out, int mem) {
  if (!e || !pixel_values || !depth_out) return VD3D_ERR_ARG;
  const int IH = e->cfg.image_h, IW = e->cfg.image_w;
  cudaStream_t s = e->stream;
  int r;
  float *px_d = (float*)pixel_values, *depth_d = depth_out;
  if (mem == VD3D_MEM_HOST) {
    if ((r = batch_slots(e, 0, &px_d, &depth_d))) return r;
    DCK(cudaMemcpyAsync(px_d, pixel_values, (size_t)3 * IH * IW * 4, cudaMemcpyHostToDevice, s));
  }
  if ((r = forward_core(e, 1, &px_d, &depth_d))) return r;
  if (mem == VD3D_MEM_HOST) {
    DCK(cudaMemcpyAsync(depth_out, depth_d, (size_t)IH * IW * 4, cudaMemcpyDeviceToHost, s));
    DCK(cudaStreamSynchronize(s));
  }
  return VD3D_OK;
}

// B frames (BGR u8 [h,w,3], DEVICE) -> DPT processor each -> ONE batched forward -> bicubic back + min-max u8 each.
// depth_u8_dev[b] / depth_f32_dev[b] (either array may be null) receive the results; enqueues on the engine stream.
int vd3d_depth_infer_batch_device(vd3d_depth* e, int B, const uint8_t* const* frames_bgr_dev, int h, int w,
                                  uint8_t* const* depth_u8_dev, float* const* depth_f32_dev, int invert) {
  if (!e || !frames_bgr_dev || B < 1 || B > kMaxBatch || h < 16 || w < 16) return VD3D_ERR_ARG;
  const int IH = e->cfg.image_h, IW = e->cfg.image_w;
  void *tmp, *rgb, *mm, *up;
  int r;
  float *pxs[kMaxBatch], *dds[kMaxBatch];
  if ((r = get_buf(e, "pp.tmp", (size_t)h * IW * 3, &tmp)) || (r = get_buf(e, "pp.rgb", (size_t)IH * IW * 3, &rgb)) ||
      (r = get_buf(e, "post.up", (size_t)h * w * 4, &up)) || (r = get_buf(e, "post.mm", 64, &mm)))
    return r;
  for (int b = 0; b < B; ++b) {
    if ((r = batch_slots(e, b, &pxs[b], &dds[b]))) return r;
    preprocess(e, frames_bgr_dev[b], h, w, 1, tmp, rgb, pxs[b], true);
  }
  if ((r = forward_core(e, B, pxs, dds))) return r;
  for (int b = 0; b < B; ++b) {
    float* upt = (depth_f32_dev && depth_f32_dev[b]) ? depth_f32_dev[b] : (float*)up;
    postprocess(e, dds[b], h, w, upt, (unsigned*)mm, depth_u8_dev ? depth_u8_dev[b] : nullptr, invert);
  }
  DCK(cudaGetLastError());
  return VD3D_OK;
}

// host-buffer form of the batch (pipe protocol: the reference hands the whole list to the HF pipeline)
int vd3d_depth_infer_batch(vd3d_depth* e, int B, const uint8_t* const* frames_bgr, int h, int w, float* const* depth_f32,
                           uint8_t* const* depth_u8, int invert) {
  if (!e || !frames_bgr || B < 1 || B > kMaxBatch) return VD3D_ERR_ARG;
  int r;
  uint8_t *fd[kMaxBatch], *u8d[kMaxBatch];
  float* f32d[kMaxBatch];
  for (int b = 0; b < B; ++b) {
    if ((r = get_buf(e, fmt("io.frame.%d", b), (size_t)h * w * 3, &fd[b])) ||
        (r = get_buf(e, fmt("io.u8.%d", b), (size_t)h * w, &u8d[b])) ||
        (r = get_buf(e, fmt("io.f32.%d", b), (size_t)h * w * 4, &f32d[b])))
      return r;
    DCK(cudaMemcpyAsync(fd[b], frames_bgr[b], (size_t)h * w * 3, cudaMemcpyHostToDevice, e->stream));
  }
  if ((r = vd3d_depth_infer_batch_device(e, B, fd, h, w, u8d, f32d, invert))) return r;
  for (int b = 0; b < B; ++b) {
    if (depth_f32 && depth_f32[b])
      DCK(cudaMemcpyAsync(depth_f32[b], f32d[b], (size_t)h * w * 4, cudaMemcpyDeviceToHost, e->stream));
    if (depth_u8 && depth_u8[b])
      DCK(cudaMemcpyAsync(depth_u8[b], u8d[b], (size_t)h * w, cudaMemcpyDeviceToHost, e->stream));
  }
  DCK(cudaStreamSynchronize(e->stream));
  return VD3D_OK;
}

// host-only: the table pil_resize builds for one axis (tests pin it to Pillow)
int vd3d_pil_bicubic_table(int in_size, int out_size, int32_t* bounds, int32_t* kk, int cap) {
  if (in_size < 1 || out_size < 1) return VD3D_ERR_ARG;
  std::vector<int> tab;
  const int ksize = pil_bicubic_table(in_size, out_size, tab);
  if (!bounds || !kk) return ksize;
  if (cap < ksize) return VD3D_ERR_ARG;
  for (int o = 0; o < out_size; ++o) {
    bounds[2 * o] = tab[2 * o];
    bounds[2 * o + 1] = tab[2 * o + 1];
    for (int j = 0; j < cap; ++j) kk[(size_t)o * cap + j] = j < ksize ? tab[(size_t)2 * out_size + (size_t)o * ksize + j] : 0;
  }
  return ksize;
}

// Image.resize((ow, oh), Image.BICUBIC) of one u8 RGB image [h,w,3] -> [oh,ow,3]
int vd3d_depth_resize_pil(vd3d_depth* e, const uint8_t* src, int h, int w, uint8_t* dst, int oh, int ow, int mem) {
  if (!e || !src || !dst || h < 1 || w < 1 || oh < 1 || ow < 1) return VD3D_ERR_ARG;
  const size_t nin = (size_t)h * w * 3, nout = (size_t)oh * ow * 3;
  void *s_d = (void*)src, *d_d = dst, *tmp;
  int r;
  if ((r = get_buf(e, "pil.tmp", (size_t)h * ow * 3, &tmp))) return r;
  if (mem == VD3D_MEM_HOST) {
    if ((r = get_buf(e, "pil.src", nin, &s_d)) || (r = get_buf(e, "pil.dst", nout, &d_d))) return r;
    DCK(cudaMemcpyAsync(s_d, src, nin, cudaMemcpyHostToDevice, e->stream));
  }
  if ((r = pil_resize(e, (const uint8_t*)s_d, h, w, (uint8_t*)tmp, (uint8_t*)d_d, oh, ow))) return r;
  if (mem == VD3D_MEM_HOST) {
    DCK(cudaMemcpyAsync(dst, d_d, nout, cudaMemcpyDeviceToHost, e->stream));
    DCK(cudaStreamSynchronize(e->stream));
  }
  return VD3D_OK;
}

// Still images of their own sizes through ONE batched forward: per image the Pillow resize to its input size, the DPT
// processor into its slot of the batch; the forward; per image bicubic back to the input size + min-max u8, and
// cv2 INTER_CUBIC to the source size when that differs.  sizes: [B][4] = src_h, src_w, in_h, in_w.
int vd3d_depth_infer_images(vd3d_depth* e, int B, const uint8_t* const* images_rgb, const int32_t* sizes,
                            uint8_t* const* depth_u8, float* const* depth_f32, int invert, int mem) {
  if (!e || !images_rgb || !sizes || !depth_u8 || B < 1 || B > kMaxBatch) return VD3D_ERR_ARG;
  const int IH = e->cfg.image_h, IW = e->cfg.image_w;
  cudaStream_t s = e->stream;
  const bool host = mem == VD3D_MEM_HOST;
  size_t src_max = 0, rs_max = 0, tmp_max = 0, pp_max = 0, in_max = 0;
  for (int b = 0; b < B; ++b) {
    const int sh = sizes[4 * b], sw = sizes[4 * b + 1], ih = sizes[4 * b + 2], iw = sizes[4 * b + 3];
    if (!images_rgb[b] || !depth_u8[b] || sh < 1 || sw < 1 || ih < 16 || iw < 16) return VD3D_ERR_ARG;
    int ph = IH, pw = IW;  // a processor without keep-aspect fit resizes every input to its fixed size
    // ZoeDepth's processor sizes the reflect-padded image
    const bool zoe = e->traits.zoe_head;
    const int fh = zoe ? ih + 2 * zoe_pad(ih) : ih, fw = zoe ? iw + 2 * zoe_pad(iw) : iw;
    if (e->fit_multiple) processed_size(fh, fw, e->fit_h, e->fit_w, e->fit_multiple, &ph, &pw);
    if (ph != IH || pw != IW) {
      char m[160];
      snprintf(m, sizeof m, "image %d: a %dx%d input maps to processed size %dx%d, the engine serves %dx%d", b, iw, ih,
               pw, ph, IW, IH);
      return dfail(e, VD3D_ERR_ARG, m);
    }
    src_max = std::max(src_max, (size_t)sh * sw * 3);
    if (ih != sh || iw != sw) {
      rs_max = std::max(rs_max, (size_t)ih * iw * 3);
      tmp_max = std::max(tmp_max, (size_t)sh * iw * 3);
    }
    pp_max = std::max(pp_max, (size_t)ih * IW * 3);
    in_max = std::max(in_max, (size_t)ih * iw);
  }
  // every buffer first, so that no reallocation lands between enqueued launches
  void *src_d = nullptr, *rs = nullptr, *ptmp = nullptr, *tmp, *rgb, *mm, *up, *u8in;
  int r;
  if ((host && (r = get_buf(e, "im.src", src_max, &src_d))) || (rs_max && (r = get_buf(e, "im.rs", rs_max, &rs))) ||
      (tmp_max && (r = get_buf(e, "pil.tmp", tmp_max, &ptmp))) || (r = get_buf(e, "pp.tmp", pp_max, &tmp)) ||
      (r = get_buf(e, "pp.rgb", (size_t)IH * IW * 3, &rgb)) || (r = get_buf(e, "post.mm", 64, &mm)) ||
      (r = get_buf(e, "im.up", in_max * 4, &up)) || (r = get_buf(e, "im.u8in", in_max, &u8in)))
    return r;
  float *pxs[kMaxBatch], *dds[kMaxBatch], *o32[kMaxBatch];
  uint8_t* o8[kMaxBatch];
  for (int b = 0; b < B; ++b) {
    const int sh = sizes[4 * b], sw = sizes[4 * b + 1], ih = sizes[4 * b + 2], iw = sizes[4 * b + 3];
    o8[b] = depth_u8[b];
    o32[b] = depth_f32 ? depth_f32[b] : nullptr;
    if ((r = batch_slots(e, b, &pxs[b], &dds[b])) ||
        (host && (r = get_buf(e, fmt("im.u8.%d", b), (size_t)sh * sw, &o8[b]))) ||
        (host && o32[b] && (r = get_buf(e, fmt("im.f32.%d", b), (size_t)ih * iw * 4, &o32[b]))))
      return r;
    // the Pillow tables of this image, so that a first use uploads before anything of this call is enqueued
    const int* t;
    int k;
    if ((iw != sw && (r = pil_table(e, sw, iw, &t, &k))) || (ih != sh && (r = pil_table(e, sh, ih, &t, &k)))) return r;
  }
  for (int b = 0; b < B; ++b) {
    const int sh = sizes[4 * b], sw = sizes[4 * b + 1], ih = sizes[4 * b + 2], iw = sizes[4 * b + 3];
    const uint8_t* img = images_rgb[b];
    if (host) {
      DCK(cudaMemcpyAsync(src_d, img, (size_t)sh * sw * 3, cudaMemcpyHostToDevice, s));
      img = (const uint8_t*)src_d;
    }
    if (ih != sh || iw != sw) {
      if ((r = pil_resize(e, img, sh, sw, (uint8_t*)ptmp, (uint8_t*)rs, ih, iw))) return r;
      img = (const uint8_t*)rs;
    }
    preprocess(e, img, ih, iw, 0, tmp, rgb, pxs[b], false);
  }
  if ((r = forward_core(e, B, pxs, dds))) return r;
  for (int b = 0; b < B; ++b) {
    const int sh = sizes[4 * b], sw = sizes[4 * b + 1], ih = sizes[4 * b + 2], iw = sizes[4 * b + 3];
    const bool back = ih != sh || iw != sw;
    postprocess(e, dds[b], ih, iw, o32[b] ? o32[b] : (float*)up, (unsigned*)mm, back ? (uint8_t*)u8in : o8[b], invert);
    if (back) {
      launch_resize_cubic_u8((const uint8_t*)u8in, ih, iw, 1, o8[b], sh, sw, s);
      e->launches++;
    }
  }
  DCK(cudaGetLastError());
  if (host) {
    for (int b = 0; b < B; ++b) {
      const int sh = sizes[4 * b], sw = sizes[4 * b + 1], ih = sizes[4 * b + 2], iw = sizes[4 * b + 3];
      DCK(cudaMemcpyAsync(depth_u8[b], o8[b], (size_t)sh * sw, cudaMemcpyDeviceToHost, s));
      if (o32[b]) DCK(cudaMemcpyAsync(depth_f32[b], o32[b], (size_t)ih * iw * 4, cudaMemcpyDeviceToHost, s));
    }
    DCK(cudaStreamSynchronize(s));
  }
  return VD3D_OK;
}

// ---------------------------------------------------------------------------
// Real-ESRGAN upscale stage (core/merged_pipeline.py:240-267; the network is the ONNX export of xinntao/Real-ESRGAN's
// SRVGGNetCompact: conv3x3(3->64)+PReLU, num_conv x [conv3x3(64->64)+PReLU], conv3x3(64->48), PixelShuffle(4), + nearest
// x4 of the input).  Every conv is the wgmma implicit GEMM of the depth neck (f16 NHWC activations, fp32 accumulate);
// the last one keeps fp32.  The engine object is the depth engine's container (named weights + buffers).
int vd3d_sr_create(void* stream, vd3d_depth** out) {
  if (!out) return VD3D_ERR_ARG;
  *out = nullptr;
  if (!load_encode()) return VD3D_ERR_CUDA;
  vd3d_depth* e = new vd3d_depth();
  memset(&e->cfg, 0, sizeof e->cfg);
  e->stream = (cudaStream_t)stream;
  *out = e;
  return VD3D_OK;
}

// Make an SR engine an RRDBNet (ESRGAN / Real-ESRGAN / BSRGAN: num_feat 64, growth 32) with nb RRDB blocks and
// network scale 2 or 4; nb = 0 makes it an SRVGGNetCompact again.
int vd3d_sr_set_rrdb(vd3d_depth* e, int nb, int net_scale) {
  if (!e || nb < 0 || nb > 64 || (nb && net_scale != 2 && net_scale != 4)) return VD3D_ERR_ARG;
  e->rr_nb = nb;
  e->rr_scale = nb ? net_scale : 0;
  return VD3D_OK;
}

}  // extern "C"

namespace vd3d {

cudaStream_t sr_stream(vd3d_depth* e) { return e->stream; }

int sr_net_scale(vd3d_depth* e) { return e->rr_scale; }

int depth_family(vd3d_depth* e) { return e->family; }

int sr_buffer(vd3d_depth* e, const char* name, size_t bytes, void** out) { return get_buf(e, name, bytes, out); }

// Weights: "sr.c{i}.w" f16 [Cout, 9*64] (tap-major, input channels padded to 64), "sr.c{i}.b" f32 [Cout], "sr.a{i}" f32
// [64] (PReLU slopes), i = 0 .. num_conv+1.
int sr_network(vd3d_depth* e, const uint8_t* fd, int h, int w, int num_conv, const float** conv_out) {
  if (!e || !fd || !conv_out || h < 8 || w < 8 || num_conv < 1 || num_conv > 64) return VD3D_ERR_ARG;
  cudaStream_t s = e->stream;
  const size_t npix = (size_t)h * w;
  void *x0, *x1, *cvo;
  int r;
  char nm[32];
  if ((r = get_buf(e, "sr.x0", npix * 64 * 2, &x0)) || (r = get_buf(e, "sr.x1", npix * 64 * 2, &x1)) ||
      (r = get_buf(e, "sr.cv", npix * 48 * 4, &cvo)))
    return r;
  launch_sr_in(fd, (__half*)x0, (int)npix, s);
  e->launches++;
  __half *cur = (__half*)x0, *nxt = (__half*)x1;
  for (int i = 0; i <= num_conv + 1; ++i) {
    const bool last = (i == num_conv + 1);
    const int cout = last ? 48 : 64;
    const __half* wt;
    const float *bias, *slope = nullptr;
    snprintf(nm, sizeof nm, "sr.c%d.w", i);
    if ((r = W(e, nm, &wt, (size_t)cout * 9 * 64))) return r;
    snprintf(nm, sizeof nm, "sr.c%d.b", i);
    if ((r = W(e, nm, &bias, cout))) return r;
    if (!last) {
      snprintf(nm, sizeof nm, "sr.a%d", i);
      if ((r = W(e, nm, &slope, 64))) return r;
    }
    GemmArgs g = base_args(0, cout, 0, last ? EPI_F32 : EPI_F16);
    g.bias = bias;
    if (last) {
      g.out_f32 = (float*)cvo;
      g.ldc = 48;
    } else {
      g.out_f16 = nxt;
      g.ldc = 64;
      g.act = 3;
      g.ls = slope;
    }
    if ((r = conv(e, cur, h, w, 64, wt, true, g, last ? 32 : 64))) return r;
    if (!last) {
      __half* t = cur;
      cur = nxt;
      nxt = t;
    }
  }
  *conv_out = (const float*)cvo;
  return VD3D_OK;
}

// RRDBNet (ESRGAN, Wang et al. 2018; Real-ESRGAN and BSRGAN use the same generator), every 3x3 conv on the wgmma
// implicit GEMM with the EPI_SR epilogue, f16 NHWC activations, fp32 accumulate:
//   feat = conv_first(x);  nb x RRDB;  feat = feat + conv_body(trunk);  (scale / 2) x [lrelu(conv_up(nearest x2))];
//   out = conv_last(lrelu(conv_hr(.)))  (f32).
// Dense blocks without copies: each RDB owns one [h*w, 320] buffer, x in channels 0..63 and growth slice k (32
// channels) at 64 k, padded to 64 (the padding channels are zero from allocation and never written; the packed
// weights have zero columns there), so conv k reads the channel prefix 64 k through its tensor map and writes only its
// own slice.  The RDB output x + 0.2 x5 goes to channels 0..63 of the next RDB's buffer; the third RDB of an RRDB adds
// the RRDB residual in the same epilogue (x_rrdb + 0.2 (x + 0.2 x5)) in place over x_rrdb, which no conv of that
// launch reads.  Three buffers rotate: RDB j reads d[j] and writes d[(j + 1) % 3].  nearest x2 + conv is four phase
// convs on the low-resolution map, one 3x3 GEMM with N = 4 x 64 (combined weights) and the pixel-shuffle scatter.
// Weights "rr.first", "rr.{i}.{j}.{k}" (block i, RDB j = 0..2, conv k = 1..5: f16 [32 or 64, 9 * 64 k]), "rr.body",
// "rr.up1", "rr.up2" (f16 [256, 576]), "rr.hr", "rr.last" (f16 [32, 576], rows 3.. zero) with ".w" / ".b" (f32 [N]).
// *rgb: f32 [scale h * scale w, 32], RGB in columns 0..2.
int rrdb_network(vd3d_depth* e, const uint8_t* fd, int h, int w, const float** rgb) {
  if (!e || !fd || !rgb || h < 8 || w < 8 || !e->rr_nb) return VD3D_ERR_ARG;
  constexpr int P = 320;  // channels per pixel of a dense buffer
  cudaStream_t s = e->stream;
  const int ns = e->rr_scale, nb = e->rr_nb;
  const size_t npix = (size_t)h * w, nhr = npix * ns * ns;
  void *x0, *feat, *body, *d[3], *u[2];
  int r;
  if ((r = get_buf(e, "rr.x0", npix * 64 * 2, &x0)) || (r = get_buf(e, "rr.feat", npix * 64 * 2, &feat)) ||
      (r = get_buf(e, "rr.body", npix * 64 * 2, &body)) || (r = get_buf(e, "rr.d0", npix * P * 2, &d[0])) ||
      (r = get_buf(e, "rr.d1", npix * P * 2, &d[1])) || (r = get_buf(e, "rr.d2", npix * P * 2, &d[2])) ||
      (r = get_buf(e, "rr.u0", nhr * 64 * 2, &u[0])) || (r = get_buf(e, "rr.u1", nhr * 64 * 2, &u[1])))
    return r;
  __half* D[3] = {(__half*)d[0], (__half*)d[1], (__half*)d[2]};
  __half* U[2] = {(__half*)u[0], (__half*)u[1]};
  auto run = [&](const char* nm, const __half* in, int H, int Wd, int cin, int pitch, GemmArgs g) {
    const __half* wt;
    const float* b;
    int rr;
    if ((rr = W(e, std::string(nm) + ".w", &wt, (size_t)g.N * 9 * cin)) || (rr = W(e, std::string(nm) + ".b", &b, g.N)))
      return rr;
    g.bias = b;
    return conv(e, in, H, Wd, cin, wt, true, g, 0, pitch, true);
  };
  launch_sr_in(fd, (__half*)x0, (int)npix, s);
  e->launches++;
  GemmArgs g = base_args(0, 64, 0, EPI_SR);
  g.out_f16 = (__half*)feat;
  if ((r = run("rr.first", (const __half*)x0, h, w, 64, 64, g))) return r;
  DCK(cudaMemcpy2DAsync(D[0], P * 2, feat, 64 * 2, 64 * 2, npix, cudaMemcpyDeviceToDevice, s));
  char nm[48];
  for (int i = 0; i < nb; ++i)
    for (int j = 0; j < 3; ++j) {
      __half *X = D[j], *Y = D[(j + 1) % 3];
      for (int k = 1; k <= 5; ++k) {
        snprintf(nm, sizeof nm, "rr.%d.%d.%d", i, j, k);
        g = base_args(0, k < 5 ? 32 : 64, 0, EPI_SR);
        g.ldc = P;
        if (k < 5) {
          g.out_f16 = X + 64 * k;
          g.act = 4;
        } else {
          g.out_f16 = Y;
          g.res_f16 = X;
          g.rs = 0.2f;
          if (j == 2) {  // Y is the RRDB's input
            g.res2_f16 = Y;
            g.rs2 = 0.2f;
          }
        }
        if ((r = run(nm, X, h, w, 64 * k, P, g))) return r;
      }
    }
  g = base_args(0, 64, 0, EPI_SR);
  g.out_f16 = (__half*)body;
  g.res_f16 = (const __half*)feat;
  g.rs = 1.f;
  if ((r = run("rr.body", D[0], h, w, 64, P, g))) return r;
  const __half* src = (const __half*)body;
  int H = h, Wd = w, ui = 1;
  for (int k = 1; 1 << k <= ns; ++k) {
    snprintf(nm, sizeof nm, "rr.up%d", k);
    g = base_args(0, 256, 0, EPI_SR);
    g.out_f16 = U[ui];
    g.act = 4;
    g.ct_k = 2;
    g.ct_cout = 64;
    g.ct_w = Wd;
    if ((r = run(nm, src, H, Wd, 64, 64, g))) return r;
    src = U[ui];
    ui ^= 1;
    H *= 2;
    Wd *= 2;
  }
  g = base_args(0, 64, 0, EPI_SR);
  g.out_f16 = U[ui];
  g.act = 4;
  if ((r = run("rr.hr", src, H, Wd, 64, 64, g))) return r;
  g = base_args(0, 32, 0, EPI_SR);
  g.out_f32 = (float*)src;  // the last up-conv's output is no longer read: its buffer holds [H * Wd, 32] floats
  if ((r = run("rr.last", U[ui], H, Wd, 64, 64, g))) return r;
  *rgb = (const float*)src;
  return VD3D_OK;
}

}  // namespace vd3d

extern "C" {

// frame BGR u8 [h,w,3] -> BGR u8 [4h,4w,3] (preprocess_esr -> network -> postprocess_esr)
int vd3d_sr_forward(vd3d_depth* e, const uint8_t* frame_bgr, int h, int w, int num_conv, uint8_t* out_bgr, int mem) {
  if (!e || !frame_bgr || !out_bgr || h < 8 || w < 8 || (!e->rr_nb && (num_conv < 1 || num_conv > 64)))
    return VD3D_ERR_ARG;
  cudaStream_t s = e->stream;
  const size_t npix = (size_t)h * w;
  void *fd = (void*)frame_bgr, *od = out_bgr;
  const float* cvo;
  int r;
  if (e->rr_nb) {  // RRDBNet: BGR u8 [scale h, scale w, 3]
    const size_t nout = npix * e->rr_scale * e->rr_scale;
    if (mem == VD3D_MEM_HOST) {
      if ((r = get_buf(e, "sr.in", npix * 3, &fd)) || (r = get_buf(e, "sr.outu8", nout * 3, &od))) return r;
      DCK(cudaMemcpyAsync(fd, frame_bgr, npix * 3, cudaMemcpyHostToDevice, s));
    }
    if ((r = rrdb_network(e, (const uint8_t*)fd, h, w, &cvo))) return r;
    launch_rrdb_out(cvo, 32, (uint8_t*)od, nout, s);
    e->launches++;
    DCK(cudaGetLastError());
    if (mem == VD3D_MEM_HOST) {
      DCK(cudaMemcpyAsync(out_bgr, od, nout * 3, cudaMemcpyDeviceToHost, s));
      DCK(cudaStreamSynchronize(s));
    }
    return VD3D_OK;
  }
  if (mem == VD3D_MEM_HOST) {
    if ((r = get_buf(e, "sr.in", npix * 3, &fd)) || (r = get_buf(e, "sr.outu8", npix * 48, &od))) return r;
    DCK(cudaMemcpyAsync(fd, frame_bgr, npix * 3, cudaMemcpyHostToDevice, s));
  }
  if ((r = sr_network(e, (const uint8_t*)fd, h, w, num_conv, &cvo))) return r;
  launch_sr_out(cvo, 48, (const uint8_t*)fd, (uint8_t*)od, h, w, s);
  e->launches++;
  DCK(cudaGetLastError());
  if (mem == VD3D_MEM_HOST) {
    DCK(cudaMemcpyAsync(out_bgr, od, npix * 48, cudaMemcpyDeviceToHost, s));
    DCK(cudaStreamSynchronize(s));
  }
  return VD3D_OK;
}

}  // extern "C"
