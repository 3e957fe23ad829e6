// depth_kernels.cu -- non-GEMM kernels of the Depth-Anything-V2 forward and the
// instantiations / launchers of the wgmma GEMM and attention kernels (umma_gemm.cuh, umma_attention.cuh).
// Reference: transformers 5.5.0 models/dinov2/modeling_dinov2.py and
// models/depth_anything/modeling_depth_anything.py as called by
// core/render_depth.py:1106-1119 (hf_batch_safe_pipe).
#include <stdlib.h>

#include "depth_launch.h"
#include "umma_gemm.cuh"
#include "umma_attention.cuh"

namespace vd3d {

// ---------------------------------------------------------------------------
// LayerNorm (eps 1e-6 for DINOv2, 1e-12 for DPT's ViT) over the fp32 residual stream -> f16 GEMM operand.  One warp per row.
// row_off / out_off: skip the CLS row when producing the backbone feature maps.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_layernorm(const float* __restrict__ x, int rows, int D,
                                                   const float* __restrict__ gamma, const float* __restrict__ beta,
                                                   __half* __restrict__ out, int row_off, float eps) {
  int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float4* xr = (const float4*)(x + (size_t)(row + row_off) * D);
  float4 v[8];  // D <= 1024, D % 128 == 0: lane owns float4 #(lane + 32 i)
  const int n = D / 128;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if (i < n) {
      v[i] = xr[lane + 32 * i];
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if (i < n) {
      float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += (a * a + b * b) + (c * c + d * d);
    }
  for (int o = 16; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / (float)D + eps);
  uint2* orow = (uint2*)(out + (size_t)row * D);
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if (i < n) {
      const int c4 = lane + 32 * i;
      float4 g4 = ((const float4*)gamma)[c4], b4 = ((const float4*)beta)[c4];
      __half2 h0 = __floats2half2_rn((v[i].x - mean) * rstd * g4.x + b4.x, (v[i].y - mean) * rstd * g4.y + b4.y);
      __half2 h1 = __floats2half2_rn((v[i].z - mean) * rstd * g4.z + b4.z, (v[i].w - mean) * rstd * g4.w + b4.w);
      uint2 u;
      u.x = *(uint32_t*)&h0;
      u.y = *(uint32_t*)&h1;
      orow[c4] = u;
    }
}

// patch embedding im2col: pixel_values f32 [3, IH, IW] -> A f16 [ph*pw, kpad], k = c*P*P + dy*P + dx (P = patch)
__global__ void __launch_bounds__(256) k_patch_im2col(const float* __restrict__ px, int IH, int IW, int ph, int pw,
                                                      __half* __restrict__ A, int kpad, int P) {
  int idx = blockIdx.x * 256 + threadIdx.x;
  const int kk = 3 * P * P;
  int total = ph * pw * kk;
  if (idx >= total) return;
  int k = idx % kk, t = idx / kk;
  int c = k / (P * P), rr = k % (P * P), dy = rr / P, dx = rr % P;
  int py = t / pw, pxx = t % pw;
  float v = px[((size_t)c * IH + (py * P + dy)) * IW + (pxx * P + dx)];
  A[(size_t)t * kpad + k] = __float2half_rn(v);
}

// the un-normalised taps of DPT's ViT: patch rows of the fp32 residual stream of B images ([B * npad, D], CLS at row
// 0 of each image) -> f16 [B * npatch, D], image after image.  Without LayerScale the residual stream of a ViT-L
// carries channels in the hundreds; values beyond the f16 range saturate to +-65504 instead of becoming inf.
__global__ void __launch_bounds__(256) k_tap_f16(const float* __restrict__ x, int npad, int npatch, int D, int images,
                                                 __half* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;  // one thread per 4 channels
  const int d4 = D / 4;
  if (i >= (size_t)images * npatch * d4) return;
  const int c4 = (int)(i % d4);
  const size_t row = i / d4;
  const int b = (int)(row / npatch), t = (int)(row % npatch);
  const float4 v = ((const float4*)(x + ((size_t)b * npad + 1 + t) * D))[c4];
  const float L = 65504.f;
  __half2 h0 = __floats2half2_rn(fminf(fmaxf(v.x, -L), L), fminf(fmaxf(v.y, -L), L));
  __half2 h1 = __floats2half2_rn(fminf(fmaxf(v.z, -L), L), fminf(fmaxf(v.w, -L), L));
  uint2 u;
  u.x = *(uint32_t*)&h0;
  u.y = *(uint32_t*)&h1;
  ((uint2*)(out + row * D))[c4] = u;
}

// the CLS half of DPT's project readout: c[b, n] = bias[n] + sum_k Wc[n, k] * x[b * npad, k] for every image b, with
// the fp32 CLS row of the residual stream and Wc f16 [N, D].  One warp per output column n, all images at once.
__global__ void __launch_bounds__(256) k_readout_cls(const float* __restrict__ x, int npad, int D, int images,
                                                     const __half* __restrict__ wc, const float* __restrict__ bias,
                                                     int N, float* __restrict__ c) {
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (n >= N) return;
  float acc[8];
#pragma unroll
  for (int b = 0; b < 8; ++b) acc[b] = 0.f;
  const __half* w = wc + (size_t)n * D;
  for (int k = lane * 2; k < D; k += 64) {
    const float2 wf = __half22float2(*(const __half2*)(w + k));
#pragma unroll
    for (int b = 0; b < 8; ++b)
      if (b < images) {
        const float2 xv = *(const float2*)(x + (size_t)b * npad * D + k);
        acc[b] = fmaf(wf.x, xv.x, fmaf(wf.y, xv.y, acc[b]));
      }
  }
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    float v = acc[b];
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0 && b < images) c[(size_t)b * N + n] = v + bias[n];
  }
}

// x[0, :] = cls + pos[0, :]
__global__ void k_set_cls(float* __restrict__ x, const float* __restrict__ cls, const float* __restrict__ pos, int D) {
  int i = blockIdx.x * 256 + threadIdx.x;
  if (i < D) x[i] = cls[i] + pos[i];
}

// 3x3 stride-2 pad-1 im2col on NHWC f16 (reassemble factor 0.5): out [(OH*OW), 9*C]
__global__ void __launch_bounds__(256) k_im2col_s2(const __half* __restrict__ in, int H, int W, int C, int ldc,
                                                   __half* __restrict__ out, int OH, int OW) {
  size_t idx = (size_t)blockIdx.x * 256 + threadIdx.x;
  size_t total = (size_t)OH * OW * 9 * C;
  if (idx >= total) return;
  int c = idx % C;
  size_t r = idx / C;
  int tap = r % 9;
  size_t o = r / 9;
  int ox = o % OW, oy = o / OW;
  int iy = oy * 2 - 1 + tap / 3, ix = ox * 2 - 1 + tap % 3;
  __half v = __float2half_rn(0.f);
  if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = in[((size_t)iy * W + ix) * ldc + c];
  out[idx] = v;
}

// bilinear upsample, align_corners=True, NHWC f16 (fusion stages and the head)
__global__ void __launch_bounds__(256) k_upsample_ac(const __half* __restrict__ in, int H, int W, int C,
                                                     __half* __restrict__ out, int OH, int OW) {
  size_t idx = (size_t)blockIdx.x * 256 + threadIdx.x;  // one thread per (pixel, 8 channels)
  int c8 = C / 8;
  size_t total = (size_t)OH * OW * c8;
  if (idx >= total) return;
  int cg = idx % c8;
  size_t o = idx / c8;
  int ox = o % OW, oy = o / OW;
  float sy = (OH > 1) ? (float)(H - 1) / (float)(OH - 1) : 0.f;
  float sx = (OW > 1) ? (float)(W - 1) / (float)(OW - 1) : 0.f;
  float fy = sy * oy, fx = sx * ox;
  int y0 = (int)fy, x0 = (int)fx;
  int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
  float ly = fy - y0, lx = fx - x0;
  const uint4* p00 = (const uint4*)(in + ((size_t)y0 * W + x0) * C) + cg;
  const uint4* p01 = (const uint4*)(in + ((size_t)y0 * W + x1) * C) + cg;
  const uint4* p10 = (const uint4*)(in + ((size_t)y1 * W + x0) * C) + cg;
  const uint4* p11 = (const uint4*)(in + ((size_t)y1 * W + x1) * C) + cg;
  uint4 a = *p00, b = *p01, c = *p10, d = *p11, r;
  const __half2* ha = (const __half2*)&a;
  const __half2* hb = (const __half2*)&b;
  const __half2* hc = (const __half2*)&c;
  const __half2* hd = (const __half2*)&d;
  __half2* hr = (__half2*)&r;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float2 fa = __half22float2(ha[j]), fb = __half22float2(hb[j]), fc = __half22float2(hc[j]),
           fd = __half22float2(hd[j]);
    float t0x = fa.x + lx * (fb.x - fa.x), t0y = fa.y + lx * (fb.y - fa.y);
    float t1x = fc.x + lx * (fd.x - fc.x), t1y = fc.y + lx * (fd.y - fc.y);
    hr[j] = __floats2half2_rn(t0x + ly * (t1x - t0x), t0y + ly * (t1y - t0y));
  }
  ((uint4*)(out + o * C))[cg] = r;
}

// elementwise relu copy (f16)
__global__ void __launch_bounds__(256) k_relu_f16(const __half* __restrict__ in, __half* __restrict__ out, size_t n8) {
  size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (i >= n8) return;
  uint4 a = ((const uint4*)in)[i];
  __half2* h = (__half2*)&a;
  const __half2 z = __floats2half2_rn(0.f, 0.f);
#pragma unroll
  for (int j = 0; j < 4; ++j) h[j] = __hmax2(h[j], z);
  ((uint4*)out)[i] = a;
}

// ---------------------------------------------------------------------------
// DPT image processor (transformers 5.5 image_processing_dpt.py): antialiased bicubic (or, for a
// checkpoint whose processor names resample 2, bilinear) resize of the uint8 frame (separable, width
// first, uint8 intermediate, like ATen's _upsample_{bicubic,bilinear}2d_aa on uint8), then rescale 1/255
// and mean/std (ImageNet for Depth-Anything, 0.5 for DPT).
// ---------------------------------------------------------------------------
__device__ __forceinline__ float cubic_aa(float x) {  // a = -0.5 (PIL / ATen antialias filter)
  const float a = -0.5f;
  x = fabsf(x);
  if (x < 1.0f) return ((a + 2.0f) * x - (a + 3.0f)) * x * x + 1.0f;
  if (x < 2.0f) return (((x - 5.0f) * x + 8.0f) * x - 4.0f) * a;
  return 0.0f;
}

// one axis of the antialiased resize on interleaved u8 [rows, in, 3] -> [rows, out, 3] (axis = x)
// or [in, cols, 3] -> [out, cols, 3] (axis = y); bilinear: the triangle filter (support 1) instead of the cubic
__global__ void __launch_bounds__(256) k_resize_aa_u8(const uint8_t* __restrict__ src, int IH, int IW,
                                                      uint8_t* __restrict__ dst, int OH, int OW, int axis_y,
                                                      int bgr_to_rgb, int bilinear) {
  int ox = blockIdx.x * 32 + (threadIdx.x & 31);
  int oy = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (ox >= OW || oy >= OH) return;
  const int in_sz = axis_y ? IH : IW, out_sz = axis_y ? OH : OW, o = axis_y ? oy : ox;
  float scale = (float)in_sz / (float)out_sz;
  const float base = bilinear ? 1.0f : 2.0f;
  float support = (scale >= 1.0f) ? base * scale : base;
  float invscale = (scale >= 1.0f) ? 1.0f / scale : 1.0f;
  float center = scale * ((float)o + 0.5f);
  int xmin = max(0, (int)(center - support + 0.5f));
  int xmax = min(in_sz, (int)(center + support + 0.5f));
  float wsum = 0.f, acc[3] = {0.f, 0.f, 0.f};
  for (int j = xmin; j < xmax; ++j) {
    const float t = ((float)j - center + 0.5f) * invscale;
    float w = bilinear ? fmaxf(0.f, 1.0f - fabsf(t)) : cubic_aa(t);
    wsum += w;
    const uint8_t* q = axis_y ? src + ((size_t)j * IW + ox) * 3 : src + ((size_t)oy * IW + j) * 3;
    acc[0] += w * (float)q[0];
    acc[1] += w * (float)q[1];
    acc[2] += w * (float)q[2];
  }
  uint8_t* d = dst + ((size_t)oy * OW + ox) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v = acc[c] / wsum;
    int iv = __float2int_rn(v);
    iv = iv < 0 ? 0 : (iv > 255 ? 255 : iv);
    d[bgr_to_rgb ? 2 - c : c] = (uint8_t)iv;
  }
}

// one pass of Pillow's 8-bit bicubic resize (ImagingResample{Horizontal,Vertical}_8bpc) on interleaved u8 [IH, IW, 3]
// -> [OH, OW, 3] along x (axis_y = 0) or y.  tab: the host-built table of the axis (vd3d_pil_bicubic_table): (first
// input, tap count) per output index, then ksize fixed-point weights per output index.  Integer arithmetic only: sums
// start at 1 << 21, then >> 22 and clip to 0..255.
__global__ void __launch_bounds__(256) k_resize_pil_u8(const uint8_t* __restrict__ src, int IH, int IW,
                                                       uint8_t* __restrict__ dst, int OH, int OW,
                                                       const int* __restrict__ tab, int ksize, int axis_y) {
  int ox = blockIdx.x * 32 + (threadIdx.x & 31);
  int oy = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (ox >= OW || oy >= OH) return;
  const int o = axis_y ? oy : ox, out_sz = axis_y ? OH : OW;
  const int x0 = tab[2 * o], cnt = tab[2 * o + 1];
  const int* k = tab + 2 * out_sz + (size_t)o * ksize;
  const size_t step = axis_y ? (size_t)IW * 3 : 3;
  const uint8_t* q = axis_y ? src + ((size_t)x0 * IW + ox) * 3 : src + ((size_t)oy * IW + x0) * 3;
  int s0 = 1 << 21, s1 = 1 << 21, s2 = 1 << 21;
  for (int j = 0; j < cnt; ++j, q += step) {
    const int w = k[j];
    s0 += (int)q[0] * w;
    s1 += (int)q[1] * w;
    s2 += (int)q[2] * w;
  }
  uint8_t* d = dst + ((size_t)oy * OW + ox) * 3;
  d[0] = (uint8_t)min(max(s0 >> 22, 0), 255);
  d[1] = (uint8_t)min(max(s1 >> 22, 0), 255);
  d[2] = (uint8_t)min(max(s2 >> 22, 0), 255);
}

// u8 RGB interleaved [H, W, 3] -> f32 CHW normalised pixel_values
__global__ void __launch_bounds__(256) k_normalize_px(const uint8_t* __restrict__ rgb, int H, int W,
                                                      float* __restrict__ px, PreprocParams pp) {
  int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= H * W) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v = (float)rgb[(size_t)i * 3 + c] * (1.0f / 255.0f);
    px[(size_t)c * H * W + i] = (v - pp.mean[c]) / pp.std[c];
  }
}

// post_process_depth_estimation: F.interpolate(bicubic, align_corners=False) (a = -0.75, clamped taps)
__device__ __forceinline__ void cubic_coeffs(float t, float* c) {
  const float A = -0.75f;
  float x;
  x = t + 1.0f;
  c[0] = ((A * x - 5.0f * A) * x + 8.0f * A) * x - 4.0f * A;
  x = t;
  c[1] = ((A + 2.0f) * x - (A + 3.0f)) * x * x + 1.0f;
  x = 1.0f - t;
  c[2] = ((A + 2.0f) * x - (A + 3.0f)) * x * x + 1.0f;
  x = 2.0f - t;
  c[3] = ((A * x - 5.0f * A) * x + 8.0f * A) * x - 4.0f * A;
}
__device__ __forceinline__ unsigned f2ord(float f) {  // order-preserving float -> uint
  unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u);
}
__global__ void __launch_bounds__(256) k_depth_upsample_minmax(const float* __restrict__ d, int IH, int IW,
                                                               float* __restrict__ out, int OH, int OW,
                                                               unsigned* __restrict__ mm) {
  int ox = blockIdx.x * 32 + (threadIdx.x & 31);
  int oy = blockIdx.y * 8 + (threadIdx.x >> 5);
  float v = 0.f;
  bool ok = ox < OW && oy < OH;
  if (ok) {
    if (IH == OH && IW == OW) {
      v = d[(size_t)oy * IW + ox];
    } else {
      float sy = (float)IH / (float)OH, sx = (float)IW / (float)OW;
      float fy = sy * ((float)oy + 0.5f) - 0.5f, fx = sx * ((float)ox + 0.5f) - 0.5f;
      int iy = (int)floorf(fy), ix = (int)floorf(fx);
      float cy[4], cx[4];
      cubic_coeffs(fy - (float)iy, cy);
      cubic_coeffs(fx - (float)ix, cx);
      v = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int yy = min(max(iy - 1 + j, 0), IH - 1);
        float r = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          int xx = min(max(ix - 1 + i, 0), IW - 1);
          r += cx[i] * d[(size_t)yy * IW + xx];
        }
        v += cy[j] * r;
      }
    }
    out[(size_t)oy * OW + ox] = v;
  }
  __shared__ float slo[8], shi[8];
  float lo = ok ? v : INFINITY, hi = ok ? v : -INFINITY;
  for (int o = 16; o; o >>= 1) {
    lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((threadIdx.x & 31) == 0) {
    slo[threadIdx.x >> 5] = lo;
    shi[threadIdx.x >> 5] = hi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {  // one pair of atomics per block (was per warp: 130 K serialised atomics at 1080p)
    for (int i = 1; i < 8; ++i) {
      lo = fminf(lo, slo[i]);
      hi = fmaxf(hi, shi[i]);
    }
    if (lo <= hi) {
      atomicMin(&mm[0], f2ord(lo));
      atomicMax(&mm[1], f2ord(hi));
    }
  }
}
__global__ void k_minmax_reset(unsigned* mm) {
  mm[0] = 0xFFFFFFFFu;
  mm[1] = 0u;
}
// convert_depth_to_grayscale tensor path (core/render_depth.py:605-611): (d-min)/(max-min+1e-6)*255, truncate
__global__ void __launch_bounds__(256) k_depth_to_u8(const float* __restrict__ d, int n, const unsigned* __restrict__ mm,
                                                     uint8_t* __restrict__ out, int invert) {
  int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  float lo = ord2f(mm[0]), hi = ord2f(mm[1]);
  float v = ((d[i] - lo) / (hi - lo + 1e-6f)) * 255.0f;
  int iv = (int)v;
  iv = iv < 0 ? 0 : (iv > 255 ? 255 : iv);
  out[i] = (uint8_t)(invert ? 255 - iv : iv);
}

// sum = a + b ; sum_relu = relu(sum)   (fusion: hidden_state + residual_layer1(residual))
__global__ void __launch_bounds__(256) k_add_relu_f16(const __half* __restrict__ a, const __half* __restrict__ b,
                                                      __half* __restrict__ sum, __half* __restrict__ sum_relu,
                                                      size_t n8) {
  size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (i >= n8) return;
  uint4 ua = ((const uint4*)a)[i], ub = ((const uint4*)b)[i], us, ur;
  const __half2* ha = (const __half2*)&ua;
  const __half2* hb = (const __half2*)&ub;
  __half2* hs = (__half2*)&us;
  __half2* hr = (__half2*)&ur;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float2 fa = __half22float2(ha[j]), fb = __half22float2(hb[j]);
    float sx = fa.x + fb.x, sy = fa.y + fb.y;
    hs[j] = __floats2half2_rn(sx, sy);
    hr[j] = __floats2half2_rn(fmaxf(sx, 0.f), fmaxf(sy, 0.f));
  }
  ((uint4*)sum)[i] = us;
  ((uint4*)sum_relu)[i] = ur;
}

// ---------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------
void launch_preprocess(const uint8_t* frame_bgr, int H, int W, uint8_t* tmp_u8, uint8_t* rgb_u8, float* px, int OH,
                       int OW, cudaStream_t s, int swap_rb, const PreprocParams& pp) {
  dim3 g1((OW + 31) / 32, (H + 7) / 8), g2((OW + 31) / 32, (OH + 7) / 8);
  k_resize_aa_u8<<<g1, 256, 0, s>>>(frame_bgr, H, W, tmp_u8, H, OW, 0, 0, pp.bilinear);       // width pass
  k_resize_aa_u8<<<g2, 256, 0, s>>>(tmp_u8, H, OW, rgb_u8, OH, OW, 1, swap_rb, pp.bilinear);  // height pass (+BGR->RGB)
  k_normalize_px<<<(OH * OW + 255) / 256, 256, 0, s>>>(rgb_u8, OH, OW, px, pp);
}
void launch_resize_pil_u8(const uint8_t* src, int IH, int IW, uint8_t* dst, int OH, int OW, const int* tab, int ksize,
                          int axis_y, cudaStream_t s) {
  dim3 g((OW + 31) / 32, (OH + 7) / 8);
  k_resize_pil_u8<<<g, 256, 0, s>>>(src, IH, IW, dst, OH, OW, tab, ksize, axis_y);
}
void launch_depth_post(const float* depth, int IH, int IW, float* up, int OH, int OW, unsigned* mm, uint8_t* out_u8,
                       int invert, cudaStream_t s) {
  k_minmax_reset<<<1, 1, 0, s>>>(mm);
  dim3 g((OW + 31) / 32, (OH + 7) / 8);
  k_depth_upsample_minmax<<<g, 256, 0, s>>>(depth, IH, IW, up, OH, OW, mm);
  if (out_u8) k_depth_to_u8<<<(OH * OW + 255) / 256, 256, 0, s>>>(up, OH * OW, mm, out_u8, invert);
}
void launch_add_relu_f16(const __half* a, const __half* b, __half* sum, __half* sum_relu, size_t n, cudaStream_t s) {
  size_t n8 = n / 8;
  k_add_relu_f16<<<(unsigned)((n8 + 255) / 256), 256, 0, s>>>(a, b, sum, sum_relu, n8);
}
void launch_layernorm(const float* x, int rows, int D, const float* g, const float* b, __half* out, int row_off,
                      float eps, cudaStream_t s) {
  k_layernorm<<<(rows + 7) / 8, 256, 0, s>>>(x, rows, D, g, b, out, row_off, eps);
}
void launch_patch_im2col(const float* px, int IH, int IW, int ph, int pw, __half* A, int kpad, int patch,
                         cudaStream_t s) {
  int total = ph * pw * 3 * patch * patch;
  k_patch_im2col<<<(total + 255) / 256, 256, 0, s>>>(px, IH, IW, ph, pw, A, kpad, patch);
}
void launch_tap_f16(const float* x, int npad, int npatch, int D, int images, __half* out, cudaStream_t s) {
  const size_t total = (size_t)images * npatch * (D / 4);
  k_tap_f16<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(x, npad, npatch, D, images, out);
}
void launch_readout_cls(const float* x, int npad, int D, int images, const __half* wc, const float* bias, int N,
                        float* c, cudaStream_t s) {
  k_readout_cls<<<(N + 7) / 8, 256, 0, s>>>(x, npad, D, images, wc, bias, N, c);
}
void launch_set_cls(float* x, const float* cls, const float* pos, int D, cudaStream_t s) {
  k_set_cls<<<(D + 255) / 256, 256, 0, s>>>(x, cls, pos, D);
}
void launch_im2col_s2(const __half* in, int H, int W, int C, int ldc, __half* out, int OH, int OW, cudaStream_t s) {
  size_t total = (size_t)OH * OW * 9 * C;
  k_im2col_s2<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(in, H, W, C, ldc, out, OH, OW);
}
void launch_upsample_ac(const __half* in, int H, int W, int C, __half* out, int OH, int OW, cudaStream_t s) {
  size_t total = (size_t)OH * OW * (C / 8);
  k_upsample_ac<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(in, H, W, C, out, OH, OW);
}
// ---------------------------------------------------------------------------
// Real-ESRGAN stage (SRVGGNetCompact): input / output ends of the conv stack
// preprocess_esr (core/merged_pipeline.py:221-225): BGR u8 -> RGB / 255, here as the first 3 of 64 f16 channels (NHWC)
__global__ void __launch_bounds__(256) k_sr_in(const uint8_t* __restrict__ bgr, __half* __restrict__ x, int npix) {
  int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= npix) return;
  const uint8_t* q = bgr + (size_t)i * 3;
  uint4 z = make_uint4(0, 0, 0, 0);
  uint4* dst = (uint4*)(x + (size_t)i * 64);
  __align__(16) __half h4[8];
  h4[0] = __float2half_rn((float)q[2] / 255.0f);
  h4[1] = __float2half_rn((float)q[1] / 255.0f);
  h4[2] = __float2half_rn((float)q[0] / 255.0f);
#pragma unroll
  for (int k = 3; k < 8; ++k) h4[k] = __float2half_rn(0.f);
  dst[0] = *(uint4*)h4;
#pragma unroll
  for (int k = 1; k < 8; ++k) dst[k] = z;
}
// PixelShuffle(4) + nearest x4 of the input + postprocess_esr (227-231): out[c, 4y+i, 4x+j] = conv[c*16 + i*4 + j, y, x] +
// in[c, y, x]; clip to [0,1], x255, truncate, RGB -> BGR.  One thread per output pixel.
__global__ void __launch_bounds__(256) k_sr_out(const float* __restrict__ conv, int ldc, const uint8_t* __restrict__ bgr,
                                                uint8_t* __restrict__ out, int h, int w) {
  int X = blockIdx.x * 32 + (threadIdx.x & 31);
  int Y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (X >= 4 * w || Y >= 4 * h) return;
  const int y = Y >> 2, x = X >> 2, sub = (Y & 3) * 4 + (X & 3);
  const float* cv = conv + ((size_t)y * w + x) * ldc + sub;
  const uint8_t* q = bgr + ((size_t)y * w + x) * 3;
  uint8_t* o = out + ((size_t)Y * 4 * w + X) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {  // c: 0 = R, 1 = G, 2 = B
    float v = cv[c * 16] + ((float)q[2 - c] / 255.0f);
    v = fminf(fmaxf(v, 0.f), 1.f) * 255.0f;
    o[2 - c] = (uint8_t)(int)v;
  }
}
void launch_sr_in(const uint8_t* bgr, __half* x, int npix, cudaStream_t s) {
  k_sr_in<<<(npix + 255) / 256, 256, 0, s>>>(bgr, x, npix);
}
void launch_sr_out(const float* conv, int ldc, const uint8_t* bgr, uint8_t* out, int h, int w, cudaStream_t s) {
  dim3 g((4 * w + 31) / 32, (4 * h + 7) / 8);
  k_sr_out<<<g, 256, 0, s>>>(conv, ldc, bgr, out, h, w);
}

void launch_relu_f16(const __half* in, __half* out, size_t n, cudaStream_t s) {
  size_t n8 = n / 8;
  k_relu_f16<<<(unsigned)((n8 + 255) / 256), 256, 0, s>>>(in, out, n8);
}

template <int BN, int STAGES, bool kSr = false>
static cudaError_t launch_gemm_t(const CUtensorMap& a, const CUtensorMap& b, const GemmArgs& g, dim3 grid,
                                 cudaStream_t s) {
  static bool attr_set = false;
  constexpr int smem = GemmSmem<BN, STAGES>::kTotal;
  if (!attr_set) {
    cudaError_t e =
        cudaFuncSetAttribute(k_umma_gemm<BN, STAGES, kSr>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  k_umma_gemm<BN, STAGES, kSr><<<grid, kGemmThreads, smem, s>>>(a, b, g);
  return cudaGetLastError();
}

cudaError_t launch_attention(const CUtensorMap& q, const CUtensorMap& k, const CUtensorMap& v, int ntok, int dmodel,
                             __half* out, int heads, int images, int npad, cudaStream_t s) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k_umma_attention, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmem);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  AttnArgs a;
  a.ntok = ntok;
  a.dmodel = dmodel;
  a.out = out;
  a.heads = heads;
  a.npad = npad;
  dim3 grid((ntok + kAttnRows - 1) / kAttnRows, heads * images);
  k_umma_attention<<<grid, kAttnThreads, kAttnSmem, s>>>(q, k, v, a);
  return cudaGetLastError();
}

static int sm_count() {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}

// bn: 32 / 64 / 128 = 128 x bn tiles; the B tensor map's box has bn rows
cudaError_t launch_gemm(int bn, const CUtensorMap& a, const CUtensorMap& b, const GemmArgs& g_in, int m_tiles,
                        int batch, cudaStream_t s) {
  GemmArgs g = g_in;
  g.nt = (g.N + bn - 1) / bn;
  g.mt = m_tiles;
  g.nz = batch;
  // persistent grid: one CTA per SM (producer, epilogue and two consumer warpgroups, up to 144 KB of operand ring),
  // each walks its tiles
  const int total = g.nt * g.mt * g.nz, sms = sm_count();
  dim3 grid(total < sms ? total : sms, 1, 1);
  switch (bn) {
    case 128: return launch_gemm_t<128, 4>(a, b, g, grid, s);
    case 64: return launch_gemm_t<64, 6>(a, b, g, grid, s);
    case 32: return launch_gemm_t<32, 6>(a, b, g, grid, s);
    default: return cudaErrorInvalidValue;
  }
}

// the RRDBNet convs: launch_gemm's tiles and grid with the EPI_SR epilogue (k_umma_gemm<BN, STAGES, true>)
cudaError_t launch_gemm_sr(int bn, const CUtensorMap& a, const CUtensorMap& b, const GemmArgs& g_in, int m_tiles,
                           cudaStream_t s) {
  GemmArgs g = g_in;
  g.nt = (g.N + bn - 1) / bn;
  g.mt = m_tiles;
  g.nz = 1;
  const int total = g.nt * g.mt, sms = sm_count();
  dim3 grid(total < sms ? total : sms, 1, 1);
  switch (bn) {
    case 128: return launch_gemm_t<128, 4, true>(a, b, g, grid, s);
    case 64: return launch_gemm_t<64, 6, true>(a, b, g, grid, s);
    case 32: return launch_gemm_t<32, 6, true>(a, b, g, grid, s);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace vd3d
