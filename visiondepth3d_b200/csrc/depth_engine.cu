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

}  // namespace

struct vd3d_depth {
  vd3d_depth_config cfg;
  cudaStream_t stream = nullptr;
  std::string err;
  std::map<std::string, DTensor> w;    // weights by name
  std::map<std::string, DTensor> buf;  // activations by name
  uint64_t launches = 0;
  int ph = 0, pw = 0, ntok = 0, npad = 0;
  bool planned = false;
  // the per-image neck / head tails of a batch run on side streams (forked after the transformer, joined at the end)
  cudaStream_t cur = nullptr;          // stream the helpers launch on (null: `stream`)
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

int get_buf(vd3d_depth* e, const std::string& name, size_t bytes, void** out, bool zero = false) {
  DTensor& t = e->buf[name];
  if (t.bytes < bytes) {
    if (t.p) DCK(cudaFree(t.p));
    DCK(cudaMalloc(&t.p, bytes));
    t.bytes = bytes;
    zero = true;
  }
  if (zero) DCK(cudaMemsetAsync(t.p, 0, t.bytes, e->cur ? e->cur : e->stream));
  *out = t.p;
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
  cudaError_t ce = launch_gemm(bn, ma, mb, g, (g.M + 127) / 128, 1, e->cur ? e->cur : e->stream);
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
  cudaStream_t s = e->cur ? e->cur : e->stream;
  cudaError_t ce = sr ? launch_gemm_sr(bn, ma, mb, g, m_tiles, s) : launch_gemm(bn, ma, mb, g, m_tiles, 1, s);
  if (ce != cudaSuccess) return dfail(e, VD3D_ERR_CUDA, std::string("conv launch: ") + cudaGetErrorString(ce));
  e->launches++;
  return VD3D_OK;
}

int round_up(int v, int m) { return (v + m - 1) / m * m; }

}  // namespace

extern "C" {

int vd3d_depth_create(const vd3d_depth_config* cfg, void* stream, vd3d_depth** out) {
  if (!cfg || !out) return VD3D_ERR_ARG;
  *out = nullptr;
  if (!load_encode()) return VD3D_ERR_CUDA;
  if (cfg->hidden % 128 || cfg->hidden > 1024 || cfg->hidden / cfg->heads != 64 || cfg->fusion % 64 ||
      cfg->image_h % 14 || cfg->image_w % 14)
    return VD3D_ERR_ARG;
  vd3d_depth* e = new vd3d_depth();
  e->cfg = *cfg;
  e->stream = (cudaStream_t)stream;
  e->ph = cfg->image_h / 14;
  e->pw = cfg->image_w / 14;
  e->ntok = e->ph * e->pw + 1;
  e->npad = round_up(e->ntok, 128);
  if (e->ntok > 3072) {
    delete e;
    return VD3D_ERR_UNSUPPORTED;
  }
  *out = e;
  return VD3D_OK;
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
  e->cfg = src->cfg;
  e->stream = (cudaStream_t)stream;
  e->w = src->w;
  e->owns_weights = false;
  e->ph = src->ph;
  e->pw = src->pw;
  e->ntok = src->ntok;
  e->npad = src->npad;
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

// tuning hook: time one GEMM shape (EPI_F16 epilogue, optional GELU) on device-resident operands with an explicit
// kernel variant (launch_gemm_variant) and debug mode (GemmArgs::dbg); returns the average launch time in ms
int vd3d_gemm_bench(vd3d_depth* e, int M, int N, int K, int variant, int dbg, int act, int iters, float* ms_out) {
  if (!e || !ms_out || (K % 8) || iters < 1) return VD3D_ERR_ARG;
  if (variant < 0 || variant > 2 || (dbg & 7) == 1 || (dbg & 7) > 4) return VD3D_ERR_ARG;
  void *da, *db, *dc;
  int r;
  if ((r = get_buf(e, "t.ba", (size_t)M * K * 2, &da))) return r;
  if ((r = get_buf(e, "t.bb", (size_t)N * K * 2, &db))) return r;
  if ((r = get_buf(e, "t.bc", (size_t)M * N * 2, &dc))) return r;
  DCK(cudaMemsetAsync(da, 0x2c, (size_t)M * K * 2, e->stream));  // 0x2c2c = 0.0652 in f16
  DCK(cudaMemsetAsync(db, 0x2c, (size_t)N * K * 2, e->stream));
  GemmArgs g = base_args(M, N, K, EPI_F16);
  g.out_f16 = (__half*)dc;
  g.act = act & 0xff;
  g.dbg = dbg;
  if (act & 0x100) {  // the proj / fc2 epilogue: fp32 residual stream read-modify-write with bias and LayerScale
    void *dx, *dv;
    if ((r = get_buf(e, "t.bx", (size_t)M * N * 4, &dx))) return r;
    if ((r = get_buf(e, "t.bv", (size_t)N * 4, &dv))) return r;  // zeros: bias = ls = 0 keeps x finite over the iterations
    g.epi = EPI_RESID_LS;
    g.act = 0;
    g.out_f32 = (float*)dx;
    g.bias = (const float*)dv;
    g.ls = (const float*)dv;
    g.ldc = N;
  }
  CUtensorMap ma, mb;
  if ((r = make_map(e, &ma, da, K, M, 1, K, (uint64_t)K * M, 128, 1))) return r;
  if ((r = make_map(e, &mb, db, K, N, 1, K, (uint64_t)K * N, 128, 1))) return r;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  auto done = [&](int rc) {
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    return rc;
  };
  if (cudaEventCreate(&e0) != cudaSuccess || cudaEventCreate(&e1) != cudaSuccess)
    return done(dfail(e, VD3D_ERR_CUDA, "gemm bench: event creation failed"));
  cudaError_t ce = cudaSuccess;
  for (int i = 0; i < 3 + iters && ce == cudaSuccess; ++i) {
    if (i == 3) ce = cudaEventRecord(e0, e->stream);
    if (ce == cudaSuccess) ce = launch_gemm_variant(variant, ma, mb, g, (M + 127) / 128, 1, e->stream);
  }
  if (ce == cudaSuccess) ce = cudaEventRecord(e1, e->stream);
  if (ce == cudaSuccess) ce = cudaEventSynchronize(e1);
  float ms = 0.f;
  if (ce == cudaSuccess) ce = cudaEventElapsedTime(&ms, e0, e1);
  if (ce != cudaSuccess) return done(dfail(e, VD3D_ERR_CUDA, std::string("gemm bench: ") + cudaGetErrorString(ce)));
  done(0);
  *ms_out = ms / iters;
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

}  // extern "C"

namespace {

constexpr int kMaxBatch = 8;

// B images through the network in one pass.  The token-wise stages (LayerNorm, QKV / proj / fc1 / fc2 GEMMs) see one
// matrix of (B-1)*NP + NT rows -- image b owns rows [b*NP, b*NP + NT), NP = NT rounded up to the 128-row tile -- so the
// GEMMs run at 3-4x the rows of one frame (the reference batches too: core/render_depth.py:1113-1119); attention runs
// with grid.y = B * heads; patch embedding, taps, neck and head stay per image (their maps are per-image 2-D tensors).
// px_dev / depth_dev: DEVICE pointers, f32 [3, image_h, image_w] in, f32 [image_h, image_w] out.
int forward_core(vd3d_depth* e, int B, const float* const* px_dev, float* const* depth_dev) {
  if (B < 1 || B > kMaxBatch) return dfail(e, VD3D_ERR_ARG, "batch must be in [1, 8]");
  e->cur = nullptr;  // (an earlier call may have failed inside its forked section)
  const vd3d_depth_config& c = e->cfg;
  cudaStream_t s = e->stream;
  const int D = c.hidden, L = c.layers, Hh = c.heads, F = c.fusion;
  const int ph = e->ph, pw = e->pw, NT = e->ntok, NP = e->npad, NPATCH = ph * pw;
  const int IH = c.image_h, IW = c.image_w;
  const int KPE = 592;
  int r;
  char nm[96];
  // ---- buffers ----
  void *x, *xn, *q, *k, *vt, *attn, *hb, *ape;
  const int MT = (B - 1) * NP + NT;  // rows of the stacked token matrix
  if ((r = get_buf(e, "x", (size_t)B * NP * D * 4, &x))) return r;
  if ((r = get_buf(e, "xn", (size_t)B * NP * D * 2, &xn))) return r;
  if ((r = get_buf(e, "q", (size_t)B * Hh * NP * 64 * 2, &q))) return r;
  if ((r = get_buf(e, "k", (size_t)B * Hh * NP * 64 * 2, &k))) return r;
  if ((r = get_buf(e, "vt", (size_t)B * Hh * 64 * NP * 2, &vt))) return r;
  if ((r = get_buf(e, "attn", (size_t)B * NP * D * 2, &attn))) return r;
  if ((r = get_buf(e, "h", (size_t)B * NP * 4 * D * 2, &hb))) return r;
  if ((r = get_buf(e, "ape", (size_t)NPATCH * KPE * 2, &ape))) return r;

  // ---- patch embedding + CLS + position embeddings ----
  const int sp_embed = e->span_begin("embed", s);
  const __half* pe_w;
  const float *pe_b, *cls, *pos;
  if ((r = W(e, "pe.w", &pe_w, (size_t)D * KPE)) || (r = W(e, "pe.b", &pe_b, D)) || (r = W(e, "cls", &cls, D)) ||
      (r = W(e, "pos", &pos, (size_t)NT * D)))
    return r;
  for (int b = 0; b < B; ++b) {
    float* xb = (float*)x + (size_t)b * NP * D;
    launch_patch_im2col(px_dev[b], IH, IW, ph, pw, (__half*)ape, KPE, s);
    GemmArgs g = base_args(NPATCH, D, KPE, EPI_PATCH);
    g.out_f32 = xb;
    g.bias = pe_b;
    g.pos = pos;
    g.ldc = D;
    if ((r = gemm(e, (const __half*)ape, KPE, pe_w, KPE, g))) return r;
    launch_set_cls(xb, cls, pos, D, s);
    e->launches += 2;
    // rows [NT, NP) of every image but the last take part in the stacked GEMMs: keep them at zero so that they stay
    // finite from frame to frame (they are never read as keys / values: the attention tensor maps end at NT)
    if (b + 1 < B) DCK(cudaMemsetAsync(xb + (size_t)NT * D, 0, (size_t)(NP - NT) * D * 4, s));
  }

  e->span_end(sp_embed, s);
  // ---- transformer blocks ----
  int tap_idx = 0;
  for (int l = 0; l < L; ++l) {
    const float *g1, *b1, *g2, *b2, *bqkv, *bo, *ls1, *bf1, *bf2, *ls2;
    const __half *wqkv, *wo, *wf1, *wf2;
    auto nmf = [&](const char* suffix) {
      snprintf(nm, sizeof nm, "l%d.%s", l, suffix);
      return std::string(nm);
    };
    if ((r = W(e, nmf("ln1.g"), &g1, D)) || (r = W(e, nmf("ln1.b"), &b1, D)) || (r = W(e, nmf("ln2.g"), &g2, D)) ||
        (r = W(e, nmf("ln2.b"), &b2, D)) || (r = W(e, nmf("qkv.w"), &wqkv, (size_t)3 * D * D)) ||
        (r = W(e, nmf("qkv.b"), &bqkv, 3 * D)) || (r = W(e, nmf("proj.w"), &wo, (size_t)D * D)) ||
        (r = W(e, nmf("proj.b"), &bo, D)) || (r = W(e, nmf("ls1"), &ls1, D)) ||
        (r = W(e, nmf("fc1.w"), &wf1, (size_t)4 * D * D)) || (r = W(e, nmf("fc1.b"), &bf1, 4 * D)) ||
        (r = W(e, nmf("fc2.w"), &wf2, (size_t)4 * D * D)) || (r = W(e, nmf("fc2.b"), &bf2, D)) ||
        (r = W(e, nmf("ls2"), &ls2, D)))
      return r;
    int sp_ = e->span_begin("ln", s);
    launch_layernorm((const float*)x, MT, D, g1, b1, (__half*)xn, 0, s);
    e->span_end(sp_, s);
    sp_ = e->span_begin("qkv", s);
    {
      GemmArgs g = base_args(MT, 3 * D, D, EPI_QKV);
      g.bias = bqkv;
      g.q = (__half*)q;
      g.k = (__half*)k;
      g.vt = (__half*)vt;
      g.heads = Hh;
      g.npad = NP;
      g.dmodel = D;
      g.qscale = 0.125f;  // 1/sqrt(64), exact in f16
      if ((r = gemm(e, (const __half*)xn, D, wqkv, D, g))) return r;
    }
    e->span_end(sp_, s);
    sp_ = e->span_begin("attn", s);
    {  // fused wgmma attention: scores and probabilities stay in registers
      CUtensorMap mq, mk, mv;
      if ((r = make_map(e, &mq, q, 64, NT, B * Hh, 64, (uint64_t)NP * 64, 128, 1))) return r;
      if ((r = make_map(e, &mk, k, 64, NT, B * Hh, 64, (uint64_t)NP * 64, 128, 1))) return r;
      if ((r = make_map(e, &mv, vt, NT, 64, B * Hh, NP, (uint64_t)64 * NP, 64, 1))) return r;
      cudaError_t ce = launch_attention(mq, mk, mv, NT, D, (__half*)attn, Hh, B, NP, s);
      if (ce != cudaSuccess) return dfail(e, VD3D_ERR_CUDA, std::string("attention launch: ") + cudaGetErrorString(ce));
      e->launches++;
    }
    e->span_end(sp_, s);
    sp_ = e->span_begin("proj", s);
    {
      GemmArgs g = base_args(MT, D, D, EPI_RESID_LS);
      g.out_f32 = (float*)x;
      g.bias = bo;
      g.ls = ls1;
      g.ldc = D;
      if ((r = gemm(e, (const __half*)attn, D, wo, D, g))) return r;
    }
    e->span_end(sp_, s);
    sp_ = e->span_begin("ln", s);
    launch_layernorm((const float*)x, MT, D, g2, b2, (__half*)xn, 0, s);
    e->span_end(sp_, s);
    sp_ = e->span_begin("fc1", s);
    {
      GemmArgs g = base_args(MT, 4 * D, D, EPI_F16);
      g.out_f16 = (__half*)hb;
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
      if ((r = gemm(e, (const __half*)xn, D, wf1, D, g))) return r;
      if (e->prof) {
        cudaEventRecord(e1, s);
        e->prof_ev.push_back(e0);
        e->prof_ev.push_back(e1);
      }
    }
    e->span_end(sp_, s);
    sp_ = e->span_begin("fc2", s);
    {
      GemmArgs g = base_args(MT, D, 4 * D, EPI_RESID_LS);
      g.out_f32 = (float*)x;
      g.bias = bf2;
      g.ls = ls2;
      g.ldc = D;
      if ((r = gemm(e, (const __half*)hb, 4 * D, wf2, 4 * D, g))) return r;
    }
    e->span_end(sp_, s);
    e->launches += 2;
    if (tap_idx < 4 && c.taps[tap_idx] == l + 1) {
      // backbone output: final LayerNorm applied (apply_layernorm=True), CLS dropped by the neck
      const float *ng, *nb;
      if ((r = W(e, "norm.g", &ng, D)) || (r = W(e, "norm.b", &nb, D))) return r;
      for (int b = 0; b < B; ++b) {
        void* tp;
        snprintf(nm, sizeof nm, "tap%d.%d", tap_idx, b);
        if ((r = get_buf(e, nm, (size_t)round_up(NPATCH, 128) * D * 2, &tp))) return r;
        launch_layernorm((const float*)x + (size_t)b * NP * D, NPATCH, D, ng, nb, (__half*)tp, 1, s);
        e->launches++;
      }
      ++tap_idx;
    }
  }
  if (tap_idx != 4) return dfail(e, VD3D_ERR_ARG, "taps must be increasing layer indices <= layers");

  // neck + head: independent per image.  With more than one image each tail runs on its own side stream (forked here,
  // joined below) with its own activation buffers, so that the many small launches of the tails (grids of 5..77 CTAs on
  // the coarse maps) overlap each other instead of leaving most SMs idle; captured into the same CUDA graph.
  const bool fork = B > 1;
  cudaStream_t s_main = s;
  const int sp_tail = e->span_begin("tail(all images, forked)", s_main);
  if (fork) {
    if (!e->ev_fork) DCK(cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming));
    DCK(cudaEventRecord(e->ev_fork, s_main));
  }
  for (int b = 0; b < B; ++b) {
  if (fork) {
    if (!e->aux[b]) DCK(cudaStreamCreateWithFlags(&e->aux[b], cudaStreamNonBlocking));
    if (!e->ev_join[b]) DCK(cudaEventCreateWithFlags(&e->ev_join[b], cudaEventDisableTiming));
    s = e->aux[b];
    e->cur = s;
    DCK(cudaStreamWaitEvent(s, e->ev_fork, 0));
  }
  auto bname = [&](const char* base) {  // per-image activation buffers when the tails run concurrently
    std::string n(base);
    if (fork) n += "#" + std::to_string(b);
    return n;
  };
  void* depth_d = depth_dev[b];
  // ---- neck: reassemble + 3x3 conv to the fusion width ----
  int fh[4], fw[4];
  void* feat[4];
  for (int i = 0; i < 4; ++i) {
    const int C = c.neck[i], CP = round_up(C, 64);
    const __half *pw_, *cw;
    const float* pb;
    snprintf(nm, sizeof nm, "r%d.proj.w", i);
    if ((r = W(e, nm, &pw_, (size_t)CP * D))) return r;
    snprintf(nm, sizeof nm, "r%d.proj.b", i);
    if ((r = W(e, nm, &pb, CP))) return r;
    snprintf(nm, sizeof nm, "tap%d.%d", i, b);
    void *tp = e->buf[nm].p, *rp, *rs = nullptr;
    snprintf(nm, sizeof nm, "r%d.p", i);
    if ((r = get_buf(e, bname(nm), (size_t)round_up(NPATCH, 128) * CP * 2, &rp))) return r;
    {
      GemmArgs g = base_args(NPATCH, CP, D, EPI_F16);
      g.out_f16 = (__half*)rp;
      g.bias = pb;
      g.ldc = CP;
      if ((r = gemm(e, (const __half*)tp, D, pw_, D, g))) return r;
    }
    if (i < 2) {  // ConvTranspose2d(kernel=stride=4 / 2)
      const int kk = (i == 0) ? 4 : 2;
      const __half* uw;
      const float* ub;
      snprintf(nm, sizeof nm, "r%d.up.w", i);
      if ((r = W(e, nm, &uw, (size_t)kk * kk * CP * CP))) return r;
      snprintf(nm, sizeof nm, "r%d.up.b", i);
      if ((r = W(e, nm, &ub, (size_t)kk * kk * CP))) return r;
      fh[i] = ph * kk;
      fw[i] = pw * kk;
      snprintf(nm, sizeof nm, "r%d.s", i);
      if ((r = get_buf(e, bname(nm), (size_t)fh[i] * fw[i] * CP * 2, &rs))) return r;
      GemmArgs g = base_args(NPATCH, kk * kk * CP, CP, EPI_CONVT);
      g.out_f16 = (__half*)rs;
      g.bias = ub;
      g.ct_k = kk;
      g.ct_cout = CP;
      g.ct_w = pw;
      if ((r = gemm(e, (const __half*)rp, CP, uw, CP, g))) return r;
    } else if (i == 2) {
      fh[i] = ph;
      fw[i] = pw;
      rs = rp;
    } else {  // Conv2d(3x3, stride 2, pad 1)
      const __half* dw;
      const float* db;
      if ((r = W(e, "r3.down.w", &dw, (size_t)CP * 9 * CP)) || (r = W(e, "r3.down.b", &db, CP))) return r;
      fh[i] = (ph - 1) / 2 + 1;
      fw[i] = (pw - 1) / 2 + 1;
      void* col;
      if ((r = get_buf(e, bname("r3.col"), (size_t)round_up(fh[i] * fw[i], 128) * 9 * CP * 2, &col))) return r;
      launch_im2col_s2((const __half*)rp, ph, pw, CP, CP, (__half*)col, fh[i], fw[i], s);
      e->launches++;
      if ((r = get_buf(e, bname("r3.s"), (size_t)round_up(fh[i] * fw[i], 128) * CP * 2, &rs))) return r;
      GemmArgs g = base_args(fh[i] * fw[i], CP, 9 * CP, EPI_F16);
      g.out_f16 = (__half*)rs;
      g.bias = db;
      g.ldc = CP;
      if ((r = gemm(e, (const __half*)col, 9 * CP, dw, 9 * CP, g))) return r;
    }
    snprintf(nm, sizeof nm, "n%d.conv.w", i);
    if ((r = W(e, nm, &cw, (size_t)F * 9 * CP))) return r;
    snprintf(nm, sizeof nm, "f%d", i);
    if ((r = get_buf(e, bname(nm), (size_t)fh[i] * fw[i] * F * 2, &feat[i]))) return r;
    GemmArgs g = base_args(0, F, 0, EPI_F16);
    g.out_f16 = (__half*)feat[i];
    g.ldc = F;
    if ((r = conv(e, (const __half*)rs, fh[i], fw[i], CP, cw, true, g))) return r;
  }

  // ---- fusion stage (coarsest first) ----
  void* fused = nullptr;
  int ch = 0, cw_ = 0;
  for (int j = 0; j < 4; ++j) {
    const int fi = 3 - j;
    const int Hc = fh[fi], Wc = fw[fi];
    const size_t n = (size_t)Hc * Wc * F;
    void *t_relu, *t_mid, *hraw, *hrelu, *yraw, *up, *prj;
    if ((r = get_buf(e, bname("fu.relu"), n * 2, &t_relu)) || (r = get_buf(e, bname("fu.mid"), n * 2, &t_mid)) ||
        (r = get_buf(e, bname("fu.h"), n * 2, &hraw)) || (r = get_buf(e, bname("fu.hrelu"), n * 2, &hrelu)) ||
        (r = get_buf(e, bname("fu.y"), n * 2, &yraw)))
      return r;
    auto cv = [&](const char* unit, const char* which, const __half** wv, const float** bv) -> int {
      snprintf(nm, sizeof nm, "f%d.%s.%s.w", j, unit, which);
      int rr = W(e, nm, wv, (size_t)F * 9 * F);
      if (rr) return rr;
      snprintf(nm, sizeof nm, "f%d.%s.%s.b", j, unit, which);
      return W(e, nm, bv, F);
    };
    const __half *w1, *w2;
    const float *bb1, *bb2;
    const __half* hin_raw;
    if (j == 0) {
      hin_raw = (const __half*)feat[fi];
      launch_relu_f16(hin_raw, (__half*)hrelu, n, s);
      e->launches++;
    } else {
      // h = fused + residual_layer1(feat)
      if ((r = cv("rl1", "c1", &w1, &bb1)) || (r = cv("rl1", "c2", &w2, &bb2))) return r;
      launch_relu_f16((const __half*)feat[fi], (__half*)t_relu, n, s);
      e->launches++;
      GemmArgs g1 = base_args(0, F, 0, EPI_F16);
      g1.out_f16 = (__half*)t_mid;
      g1.bias = bb1;
      g1.act = 2;
      g1.ldc = F;
      if ((r = conv(e, (const __half*)t_relu, Hc, Wc, F, w1, true, g1))) return r;
      // y = conv2(mid) + b2 + feat ; h = y + fused  (two residual adds: second via res on a 1x1-free pass)
      GemmArgs g2 = base_args(0, F, 0, EPI_F16);
      g2.out_f16 = (__half*)yraw;
      g2.bias = bb2;
      g2.res_f16 = (const __half*)feat[fi];
      g2.ldc = F;
      if ((r = conv(e, (const __half*)t_mid, Hc, Wc, F, w2, true, g2))) return r;
      // h = fused + y ; relu(h) feeds residual_layer2's first conv
      launch_add_relu_f16((const __half*)fused, (const __half*)yraw, (__half*)hraw, (__half*)hrelu, n, s);
      e->launches++;
      hin_raw = (const __half*)hraw;
    }
    // residual_layer2
    if ((r = cv("rl2", "c1", &w1, &bb1)) || (r = cv("rl2", "c2", &w2, &bb2))) return r;
    {
      GemmArgs g1 = base_args(0, F, 0, EPI_F16);
      g1.out_f16 = (__half*)t_mid;
      g1.bias = bb1;
      g1.act = 2;
      g1.ldc = F;
      if ((r = conv(e, (const __half*)hrelu, Hc, Wc, F, w1, true, g1))) return r;
      GemmArgs g2 = base_args(0, F, 0, EPI_F16);
      g2.out_f16 = (__half*)yraw;
      g2.bias = bb2;
      g2.res_f16 = hin_raw;
      g2.ldc = F;
      if ((r = conv(e, (const __half*)t_mid, Hc, Wc, F, w2, true, g2))) return r;
    }
    // upsample (to the next feature's size, or x2 at the end), then 1x1 projection
    int OH = (j < 3) ? fh[fi - 1] : Hc * 2, OW = (j < 3) ? fw[fi - 1] : Wc * 2;
    snprintf(nm, sizeof nm, "fu.up%d", j);
    if ((r = get_buf(e, bname(nm), (size_t)OH * OW * F * 2, &up))) return r;
    launch_upsample_ac((const __half*)yraw, Hc, Wc, F, (__half*)up, OH, OW, s);
    e->launches++;
    const __half* pwt;
    const float* pbs;
    snprintf(nm, sizeof nm, "f%d.proj.w", j);
    if ((r = W(e, nm, &pwt, (size_t)F * F))) return r;
    snprintf(nm, sizeof nm, "f%d.proj.b", j);
    if ((r = W(e, nm, &pbs, F))) return r;
    snprintf(nm, sizeof nm, "fused%d", j);
    if ((r = get_buf(e, bname(nm), (size_t)round_up(OH * OW, 128) * F * 2, &prj))) return r;
    GemmArgs g = base_args(OH * OW, F, F, EPI_F16);
    g.out_f16 = (__half*)prj;
    g.bias = pbs;
    g.ldc = F;
    if ((r = gemm(e, (const __half*)up, F, pwt, F, g))) return r;
    fused = prj;
    ch = OH;
    cw_ = OW;
  }

  // ---- head ----
  {
    const int F2 = round_up(F / 2, 64);
    const __half *w1, *w2;
    const float *b1h, *b2h, *w3, *b3;
    if ((r = W(e, "h.c1.w", &w1, (size_t)F2 * 9 * F)) || (r = W(e, "h.c1.b", &b1h, F2)) ||
        (r = W(e, "h.c2.w", &w2, (size_t)32 * 9 * F2)) || (r = W(e, "h.c2.b", &b2h, 32)) ||
        (r = W(e, "h.c3.w", &w3, 32)) || (r = W(e, "h.c3.b", &b3, 1)))
      return r;
    void *h1, *h1u;
    if ((r = get_buf(e, bname("h1"), (size_t)ch * cw_ * F2 * 2, &h1)) || (r = get_buf(e, bname("h1u"), (size_t)IH * IW * F2 * 2, &h1u)))
      return r;
    GemmArgs g1 = base_args(0, F2, 0, EPI_F16);
    g1.out_f16 = (__half*)h1;
    g1.bias = b1h;
    g1.ldc = F2;
    if ((r = conv(e, (const __half*)fused, ch, cw_, F, w1, true, g1))) return r;
    launch_upsample_ac((const __half*)h1, ch, cw_, F2, (__half*)h1u, IH, IW, s);
    e->launches++;
    GemmArgs g2 = base_args(0, 32, 0, EPI_HEAD);
    g2.out_f32 = (float*)depth_d;
    g2.bias = b2h;
    g2.w3 = w3;
    g2.b3p = b3;
    if ((r = conv(e, (const __half*)h1u, IH, IW, F2, w2, true, g2, 32))) return r;
  }
  if (fork) DCK(cudaEventRecord(e->ev_join[b], s));
  }  // images
  e->cur = nullptr;
  if (fork)
    for (int b = 0; b < B; ++b) DCK(cudaStreamWaitEvent(s_main, e->ev_join[b], 0));
  e->span_end(sp_tail, s_main);
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
  char nm[48];
  snprintf(nm, sizeof nm, "pil.%d.%d", in_size, out_size);
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

// (h, w) the DPT image processor resizes an image to (depth_engine.py processed_size): keep the aspect ratio, scale the
// side closer to 518, round to multiples of 14 (Python's round: half to even)
void processed_size(int h, int w, int* ph, int* pw) {
  double sh = 518.0 / h, sw = 518.0 / w;
  if (fabs(1 - sw) < fabs(1 - sh))
    sh = sw;
  else
    sw = sh;
  auto rnd = [](double v) { int r = (int)nearbyint(v / 14) * 14; return r < 14 ? 14 : r; };
  *ph = rnd(sh * h);
  *pw = rnd(sw * w);
}

}  // namespace

extern "C" {

// pixel_values: f32 [3, image_h, image_w] (already resized + normalised); depth_out f32 [image_h, image_w]
int vd3d_depth_forward(vd3d_depth* e, const float* pixel_values, float* depth_out, int mem) {
  if (!e || !pixel_values || !depth_out) return VD3D_ERR_ARG;
  const int IH = e->cfg.image_h, IW = e->cfg.image_w;
  cudaStream_t s = e->stream;
  int r;
  void *px_d = (void*)pixel_values, *depth_d = depth_out;
  if (mem == VD3D_MEM_HOST) {
    if ((r = get_buf(e, "px", (size_t)3 * IH * IW * 4, &px_d))) return r;
    if ((r = get_buf(e, "depth", (size_t)IH * IW * 4, &depth_d))) return r;
    DCK(cudaMemcpyAsync(px_d, pixel_values, (size_t)3 * IH * IW * 4, cudaMemcpyHostToDevice, s));
  }
  const float* pxs[1] = {(const float*)px_d};
  float* ds[1] = {(float*)depth_d};
  if ((r = forward_core(e, 1, pxs, ds))) return r;
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
  cudaStream_t s = e->stream;
  void *tmp, *rgb, *mm, *up;
  int r;
  char nm[32];
  const float* pxs[kMaxBatch];
  float* dds[kMaxBatch];
  if ((r = get_buf(e, "pp.tmp", (size_t)h * IW * 3, &tmp)) || (r = get_buf(e, "pp.rgb", (size_t)IH * IW * 3, &rgb)) ||
      (r = get_buf(e, "post.up", (size_t)h * w * 4, &up)) || (r = get_buf(e, "post.mm", 64, &mm)))
    return r;
  for (int b = 0; b < B; ++b) {
    void *px, *dd;
    snprintf(nm, sizeof nm, b ? "px.%d" : "px", b);
    if ((r = get_buf(e, nm, (size_t)3 * IH * IW * 4, &px))) return r;
    snprintf(nm, sizeof nm, b ? "depth.%d" : "depth", b);
    if ((r = get_buf(e, nm, (size_t)IH * IW * 4, &dd))) return r;
    launch_preprocess(frames_bgr_dev[b], h, w, (uint8_t*)tmp, (uint8_t*)rgb, (float*)px, IH, IW, s);
    e->launches += 3;
    pxs[b] = (const float*)px;
    dds[b] = (float*)dd;
  }
  if ((r = forward_core(e, B, pxs, dds))) return r;
  for (int b = 0; b < B; ++b) {
    float* upt = (depth_f32_dev && depth_f32_dev[b]) ? depth_f32_dev[b] : (float*)up;
    uint8_t* u8 = depth_u8_dev ? depth_u8_dev[b] : nullptr;
    launch_depth_post(dds[b], IH, IW, upt, h, w, (unsigned*)mm, u8, invert, s);
    e->launches += u8 ? 3 : 2;
  }
  DCK(cudaGetLastError());
  return VD3D_OK;
}

// host-buffer form of the batch (pipe protocol: the reference hands the whole list to the HF pipeline)
int vd3d_depth_infer_batch(vd3d_depth* e, int B, const uint8_t* const* frames_bgr, int h, int w, float* const* depth_f32,
                           uint8_t* const* depth_u8, int invert) {
  if (!e || !frames_bgr || B < 1 || B > kMaxBatch) return VD3D_ERR_ARG;
  int r;
  char nm[32];
  const uint8_t* fd[kMaxBatch];
  uint8_t* u8d[kMaxBatch];
  float* f32d[kMaxBatch];
  for (int b = 0; b < B; ++b) {
    void *a, *c, *d;
    snprintf(nm, sizeof nm, "io.frame.%d", b);
    if ((r = get_buf(e, nm, (size_t)h * w * 3, &a))) return r;
    snprintf(nm, sizeof nm, "io.u8.%d", b);
    if ((r = get_buf(e, nm, (size_t)h * w, &c))) return r;
    snprintf(nm, sizeof nm, "io.f32.%d", b);
    if ((r = get_buf(e, nm, (size_t)h * w * 4, &d))) return r;
    DCK(cudaMemcpyAsync(a, frames_bgr[b], (size_t)h * w * 3, cudaMemcpyHostToDevice, e->stream));
    fd[b] = (const uint8_t*)a;
    u8d[b] = (uint8_t*)c;
    f32d[b] = (float*)d;
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
    int ph, pw;
    processed_size(ih, iw, &ph, &pw);
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
  char nm[32];
  if ((host && (r = get_buf(e, "im.src", src_max, &src_d))) || (rs_max && (r = get_buf(e, "im.rs", rs_max, &rs))) ||
      (tmp_max && (r = get_buf(e, "pil.tmp", tmp_max, &ptmp))) || (r = get_buf(e, "pp.tmp", pp_max, &tmp)) ||
      (r = get_buf(e, "pp.rgb", (size_t)IH * IW * 3, &rgb)) || (r = get_buf(e, "post.mm", 64, &mm)) ||
      (r = get_buf(e, "im.up", in_max * 4, &up)) || (r = get_buf(e, "im.u8in", in_max, &u8in)))
    return r;
  const float* pxs[kMaxBatch];
  float* dds[kMaxBatch];
  uint8_t* o8[kMaxBatch];
  float* o32[kMaxBatch];
  for (int b = 0; b < B; ++b) {
    const int sh = sizes[4 * b], sw = sizes[4 * b + 1], ih = sizes[4 * b + 2], iw = sizes[4 * b + 3];
    void *px, *dd;
    snprintf(nm, sizeof nm, b ? "px.%d" : "px", b);
    if ((r = get_buf(e, nm, (size_t)3 * IH * IW * 4, &px))) return r;
    snprintf(nm, sizeof nm, b ? "depth.%d" : "depth", b);
    if ((r = get_buf(e, nm, (size_t)IH * IW * 4, &dd))) return r;
    pxs[b] = (const float*)px;
    dds[b] = (float*)dd;
    o8[b] = depth_u8[b];
    o32[b] = depth_f32 ? depth_f32[b] : nullptr;
    if (host) {
      void* p;
      snprintf(nm, sizeof nm, "im.u8.%d", b);
      if ((r = get_buf(e, nm, (size_t)sh * sw, &p))) return r;
      o8[b] = (uint8_t*)p;
      if (o32[b]) {
        snprintf(nm, sizeof nm, "im.f32.%d", b);
        if ((r = get_buf(e, nm, (size_t)ih * iw * 4, &p))) return r;
        o32[b] = (float*)p;
      }
    }
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
    launch_preprocess(img, ih, iw, (uint8_t*)tmp, (uint8_t*)rgb, (float*)pxs[b], IH, IW, s, 0);
    e->launches += 3;
  }
  if ((r = forward_core(e, B, pxs, dds))) return r;
  for (int b = 0; b < B; ++b) {
    const int sh = sizes[4 * b], sw = sizes[4 * b + 1], ih = sizes[4 * b + 2], iw = sizes[4 * b + 3];
    const bool back = ih != sh || iw != sw;
    launch_depth_post(dds[b], IH, IW, o32[b] ? o32[b] : (float*)up, ih, iw, (unsigned*)mm,
                      back ? (uint8_t*)u8in : o8[b], invert, s);
    e->launches += 3;
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

// frame (BGR u8 [h,w,3], DEVICE) -> processor -> forward -> bicubic back to (h,w) -> min-max u8 [h,w]
// (hf pipeline + convert_depth_to_grayscale, core/render_depth.py:1113-1119,605-611,1907-1917).
// Enqueues on the engine stream without synchronising; depth_f32_or_null receives the resized
// float depth ("predicted_depth" of the pipe protocol).
int vd3d_depth_infer_device(vd3d_depth* e, const uint8_t* frame_bgr_dev, int h, int w, uint8_t* depth_u8_dev,
                            float* depth_f32_or_null, int invert) {
  if (!e || !frame_bgr_dev || h < 16 || w < 16) return VD3D_ERR_ARG;
  const int IH = e->cfg.image_h, IW = e->cfg.image_w;
  cudaStream_t s = e->stream;
  void *tmp, *rgb, *px, *up, *mm, *dd;
  int r;
  if ((r = get_buf(e, "pp.tmp", (size_t)h * IW * 3, &tmp)) || (r = get_buf(e, "pp.rgb", (size_t)IH * IW * 3, &rgb)) ||
      (r = get_buf(e, "px", (size_t)3 * IH * IW * 4, &px)) || (r = get_buf(e, "depth", (size_t)IH * IW * 4, &dd)) ||
      (r = get_buf(e, "post.up", (size_t)h * w * 4, &up)) || (r = get_buf(e, "post.mm", 64, &mm)))
    return r;
  launch_preprocess(frame_bgr_dev, h, w, (uint8_t*)tmp, (uint8_t*)rgb, (float*)px, IH, IW, s);
  e->launches += 3;
  if ((r = vd3d_depth_forward(e, (const float*)px, (float*)dd, VD3D_MEM_DEVICE))) return r;
  float* upt = depth_f32_or_null ? depth_f32_or_null : (float*)up;
  launch_depth_post((const float*)dd, IH, IW, upt, h, w, (unsigned*)mm, depth_u8_dev, invert, s);
  e->launches += depth_u8_dev ? 3 : 2;
  DCK(cudaGetLastError());
  return VD3D_OK;
}

// host-buffer form (pipe protocol / tests): frame BGR u8 [h,w,3] -> depth f32 [h,w] and/or u8 [h,w]
int vd3d_depth_infer(vd3d_depth* e, const uint8_t* frame_bgr, int h, int w, float* depth_f32, uint8_t* depth_u8,
                     int invert) {
  if (!e || !frame_bgr) return VD3D_ERR_ARG;
  void *fd, *u8d, *f32d;
  int r;
  if ((r = get_buf(e, "io.frame", (size_t)h * w * 3, &fd)) || (r = get_buf(e, "io.u8", (size_t)h * w, &u8d)) ||
      (r = get_buf(e, "io.f32", (size_t)h * w * 4, &f32d)))
    return r;
  DCK(cudaMemcpyAsync(fd, frame_bgr, (size_t)h * w * 3, cudaMemcpyHostToDevice, e->stream));
  if ((r = vd3d_depth_infer_device(e, (const uint8_t*)fd, h, w, (uint8_t*)u8d, (float*)f32d, invert))) return r;
  if (depth_f32) DCK(cudaMemcpyAsync(depth_f32, f32d, (size_t)h * w * 4, cudaMemcpyDeviceToHost, e->stream));
  if (depth_u8) DCK(cudaMemcpyAsync(depth_u8, u8d, (size_t)h * w, cudaMemcpyDeviceToHost, e->stream));
  DCK(cudaStreamSynchronize(e->stream));
  return VD3D_OK;
}

}  // extern "C"
