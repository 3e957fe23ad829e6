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
// bicubic to (OH,OW) + min/max (+ u8 quantisation when out_u8 != null) (2-3 launches)
void launch_depth_post(const float* depth, int IH, int IW, float* up, int OH, int OW, unsigned* mm, uint8_t* out_u8,
                       int invert, cudaStream_t s);
void launch_add_relu_f16(const __half* a, const __half* b, __half* sum, __half* sum_relu, size_t n, cudaStream_t s);
void launch_relu_f16(const __half* in, __half* out, size_t n, cudaStream_t s);
// Real-ESRGAN stage: BGR u8 -> 64-channel f16 NHWC (RGB/255 in channels 0..2); pixel-shuffle + base + clip + u8 BGR
void launch_sr_in(const uint8_t* bgr, __half* x, int npix, cudaStream_t s);
void launch_sr_out(const float* conv, int ldc, const uint8_t* bgr, uint8_t* out, int h, int w, cudaStream_t s);
// fused attention: q,k [image][h][npad][64] (q pre-scaled), vT [image][h][64][npad] -> out [images * npad, dmodel].
// One CTA per kAttnRows queries of one head; the q map's box is 64 x kAttnRows (the k map's 64 x 128, v's 64 x 64).
constexpr int kAttnRows = 192;
cudaError_t launch_attention(const CUtensorMap& q, const CUtensorMap& k, const CUtensorMap& v, int ntok, int dmodel,
                             __half* out, int heads, int images, int npad, cudaStream_t s);
// bn in {32, 64, 128}; grid = (ceil(N/bn), m_tiles, batch)
cudaError_t launch_gemm(int bn, const CUtensorMap& a, const CUtensorMap& b, const GemmArgs& g, int m_tiles,
                        int batch, cudaStream_t s);
// launch_gemm for the RRDBNet convs (epilogue EPI_SR), batch 1
cudaError_t launch_gemm_sr(int bn, const CUtensorMap& a, const CUtensorMap& b, const GemmArgs& g, int m_tiles,
                           cudaStream_t s);
}  // namespace vd3d
