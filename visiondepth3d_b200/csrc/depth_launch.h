// depth_launch.h -- launch prototypes of depth_kernels.cu
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vd3d {
struct GemmArgs;
// the image processor's filter and normalisation (Depth-Anything-V2: bicubic, ImageNet mean / std)
struct PreprocParams {
  int bilinear;  // 0: bicubic (PIL resample 3), 1: bilinear (2)
  float mean[3], std[3];
};
constexpr PreprocParams kImagenetBicubic = {0, {0.485f, 0.456f, 0.406f}, {0.229f, 0.224f, 0.225f}};
void launch_layernorm(const float* x, int rows, int D, const float* g, const float* b, __half* out, int row_off,
                      float eps, cudaStream_t s);
// patch embedding im2col for patch x patch patches: A f16 [ph*pw, kpad], K = 3*patch*patch
void launch_patch_im2col(const float* px, int IH, int IW, int ph, int pw, __half* A, int kpad, int patch,
                         cudaStream_t s);
// DPT: the patch rows of B images' fp32 residual stream -> f16 [B*npatch, D] (saturating), and the per-image CLS half
// of the project readout c [B, N] = Wc . cls_b + bias
void launch_tap_f16(const float* x, int npad, int npatch, int D, int images, __half* out, cudaStream_t s);
void launch_readout_cls(const float* x, int npad, int D, int images, const __half* wc, const float* bias, int N,
                        float* c, cudaStream_t s);
void launch_set_cls(float* x, const float* cls, const float* pos, int D, cudaStream_t s);
void launch_im2col_s2(const __half* in, int H, int W, int C, int ldc, __half* out, int OH, int OW, cudaStream_t s);
void launch_upsample_ac(const __half* in, int H, int W, int C, __half* out, int OH, int OW, cudaStream_t s);
// DPT image processor: BGR u8 [H,W,3] -> pixel_values f32 [3,OH,OW] (3 launches); swap_rb = 0 takes RGB input
void launch_preprocess(const uint8_t* frame_bgr, int H, int W, uint8_t* tmp_u8, uint8_t* rgb_u8, float* px, int OH,
                       int OW, cudaStream_t s, int swap_rb = 1, const PreprocParams& pp = kImagenetBicubic);
// one pass of Pillow's 8-bit bicubic resize on u8 [IH,IW,3] (axis_y = 0: width, 1: height) with a host-built table
void launch_resize_pil_u8(const uint8_t* src, int IH, int IW, uint8_t* dst, int OH, int OW, const int* tab, int ksize,
                          int axis_y, cudaStream_t s);
// bicubic to (OH,OW) + min/max (+ u8 quantisation when out_u8 != null) (2-3 launches).  pad_h / pad_w > 0 (ZoeDepth's
// post-process): only the (OH, OW) window at (pad_h, pad_w) of the bicubic resize to (OH + 2 pad_h, OW + 2 pad_w) is
// evaluated, i.e. the resize to the padded size, then the crop
void launch_depth_post_crop(const float* depth, int IH, int IW, float* up, int OH, int OW, int pad_h, int pad_w,
                            unsigned* mm, uint8_t* out_u8, int invert, cudaStream_t s);
// ---- ZoeDepth metric head (see depth_kernels.cu) ----
// the patch transformer of the router: width 128, 4 heads, FFN 1024, 4 post-norm layers; 64 bins; at most 16 attractors
constexpr int kZoeE = 128, kZoeHeads = 4, kZoeFF = 1024, kZoeLayers = 4, kZoeBins = 64, kZoeMaxAttr = 16;
// u8 [h, w, 3] (BGR when swap_rb) -> reflect pad -> bilinear align_corners to OH x OW -> f32 [3, OH, OW] normalised
void launch_zoe_preprocess(const uint8_t* img, int h, int w, int swap_rb, int pad_h, int pad_w, float* px, int OH,
                           int OW, const PreprocParams& pp, cudaStream_t s);
// floats of the packed router weights for a bottleneck of F channels, and of the scratch of a router over n tokens
size_t zoe_router_floats(int F);
size_t zoe_router_scratch(int n);
// one image: x f32 [n, F] (the bottleneck conv2) -> logits f32 [2] and route (device int)
void launch_zoe_router(const float* x, int n, int F, const float* wts, const float* pe, float* scratch, float* logits,
                       int* route, cudaStream_t s);
void launch_zoe_attractor(const __half* hid, int ldh, int E, const float* w2, const float* b2, int na, const float* prev,
                          int ldp, int prev_cfg_stride, int prev_softplus, int Hp, int Wp, float* out, int H, int W,
                          const int* route, cudaStream_t s);
// floats of one configuration's packed log-binomial MLP (cin inputs, hid hidden units: 40 or 80)
size_t zoe_logbinom_floats(int cin, int hid);
cudaError_t launch_zoe_logbinom(const __half* act, const float* w3, const float* b3, const __half* emb,
                                const float* bins, int He, int We, int E, const float* mlp, int cin, int hid,
                                float min_t, float max_t, float* depth, int H, int W, const int* route, cudaStream_t s);
void launch_add_relu_f16(const __half* a, const __half* b, __half* sum, __half* sum_relu, size_t n, cudaStream_t s);
void launch_relu_f16(const __half* in, __half* out, size_t n, cudaStream_t s);
// Real-ESRGAN stage: BGR u8 -> 64-channel f16 NHWC (RGB/255 in channels 0..2); pixel-shuffle + base + clip + u8 BGR
void launch_sr_in(const uint8_t* bgr, __half* x, int npix, cudaStream_t s);
void launch_sr_out(const float* conv, int ldc, const uint8_t* bgr, uint8_t* out, int h, int w, cudaStream_t s);
// fused attention: q,k [image][h][npad][64] (q pre-scaled), vT [image][h][64][npad] -> out [images * npad, dmodel].
// One CTA per kAttnRows queries of one head; the q map's box is 64 x kAttnRows (the k map's 64 x 128, v's 64 x 64).
// rpb (BEiT): the layer's relative position bias tables f32 [heads][(2 ph - 1)(2 pw - 1) + 3] of the ph x gw token grid
// (ntok = ph * gw + 1), added to the scores in k_umma_attention<true>; null: the bias-free kernel.
constexpr int kAttnRows = 192;
cudaError_t launch_attention(const CUtensorMap& q, const CUtensorMap& k, const CUtensorMap& v, int ntok, int dmodel,
                             __half* out, int heads, int images, int npad, cudaStream_t s, const float* rpb = nullptr,
                             int gw = 0);
// dynamic shared memory of k_umma_attention<true> on a ph x pw grid: the bias-free kernel's, one head's table (rounded to
// 16 bytes) and one int per key column of its 128-key tiles.  It must stay within kAttnSmemMax, the opt-in limit of an
// sm_90 block (227 KB).
constexpr int kAttnSmemMax = 227 * 1024;
size_t attention_bias_smem(int ph, int pw);
// bn in {32, 64, 128}; grid = (ceil(N/bn), m_tiles, batch)
cudaError_t launch_gemm(int bn, const CUtensorMap& a, const CUtensorMap& b, const GemmArgs& g, int m_tiles,
                        int batch, cudaStream_t s);
// ---- BiT front end of DPT-Hybrid (even H, W; the output of every stride-2 op is H/2 x W/2) ----
// 7x7 stride-2 stem conv 3 -> 64 in f32 (SAME: pad 2 before, 3 after): px [3, H, W], w f32 [64, 147] -> y f32 NHWC
void launch_bit_stem(const float* px, int H, int W, const float* w, float* y, cudaStream_t s);
// GroupNorm(32, eps 1e-5) on NHWC f32 [rows, C], C a power of two in 64..1024.  Statistics: chunk partials (mean, M2)
// float2 [ceil(rows / gn_chunk(rows))][32] (at most kGnMaxChunks chunks), merged in a fixed order by the apply kernel.
constexpr int kGnMaxChunks = 128;
constexpr float kGnEps = 1e-5f;
int gn_chunk(int rows);
void launch_gn_stats(const float* y, int rows, int C, float2* part, cudaStream_t s);
// one GroupNorm'd input: the map, its partials and its affine (f32 [C])
struct GnInput {
  const float* y;
  const float2* part;
  const float *gamma, *beta;
};
// out f16 [rows, C] = [relu](GN_a(a.y) [+ GN_b(b.y) when b.y] [+ res f16 [rows, C]])
void launch_gn_apply(const GnInput& a, const GnInput& b, const __half* res, int relu, int rows, int C, __half* out,
                     cudaStream_t s);
// 3x3 stride-2 max-pool, SAME padding 0 before / 1 after with pad value 0: f16 NHWC [H, W, C] -> [H/2, W/2, C]
void launch_maxpool_same(const __half* in, int H, int W, int C, __half* out, cudaStream_t s);
// stride-2 im2col of a k x k conv (k 1 or 3) with `pb` zero pixels before and the rest after: f16 NHWC [H, W, C] ->
// [(H/2) * (W/2), k * k * C] (tap-major); k = 1, pb = 0: the even pixels.  C a multiple of 8.
void launch_im2col_same(const __half* in, int H, int W, int C, int k, int pb, __half* out, cudaStream_t s);
// launch_gemm for the RRDBNet convs (epilogue EPI_SR), batch 1
cudaError_t launch_gemm_sr(int bn, const CUtensorMap& a, const CUtensorMap& b, const GemmArgs& g, int m_tiles,
                           cudaStream_t s);
}  // namespace vd3d
