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
// BiT ResNet front end of DPT-Hybrid (transformers 5.5 models/bit/modeling_bit.py: BitEmbeddings and
// BitBottleneckLayer with global_padding "SAME").  The convolutions run on k_umma_gemm; these are the stem conv, the
// GroupNorm, the max-pool and the stride-2 im2col with TF SAME (asymmetric) padding.
// ---------------------------------------------------------------------------

// 7x7 stride-2 conv 3 -> 64 without bias, TF SAME padding (2 before, 3 after), in f32 on the CUDA cores: pixel_values
// [3, H, W] -> y NHWC f32 [OH * OW, 64].  w: the weight-standardised kernel f32 [64, 3 * 49] (c, ky, kx order).  Each
// output sums its taps in (c, ky, kx) order with fmaf, skipping the padding.  A warp owns 32 pixels and 16 channels,
// so every weight read is a shared-memory broadcast.
__global__ void __launch_bounds__(256) k_bit_stem(const float* __restrict__ px, int H, int W,
                                                  const float* __restrict__ w, float* __restrict__ y, int OH, int OW) {
  __shared__ float ws[64 * 147];
  for (int i = threadIdx.x; i < 64 * 147; i += 256) ws[i] = w[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cg = warp & 3, sub = warp >> 2;
  const int npix = OH * OW;
  for (int p0 = blockIdx.x * 64; p0 < npix; p0 += gridDim.x * 64) {
    const int p = p0 + sub * 32 + lane;
    if (p >= npix) continue;
    const int oy = p / OW, ox = p % OW;
    const int iy0 = 2 * oy - 2, ix0 = 2 * ox - 2;
    float acc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = 0.f;
    for (int c = 0; c < 3; ++c)
      for (int ky = 0; ky < 7; ++ky) {
        const int iy = iy0 + ky;
        if (iy < 0 || iy >= H) continue;
        const float* row = px + ((size_t)c * H + iy) * W;
        const float* wr = ws + (cg * 16) * 147 + c * 49 + ky * 7;
#pragma unroll
        for (int kx = 0; kx < 7; ++kx) {
          const int ix = ix0 + kx;
          if (ix < 0 || ix >= W) continue;
          const float v = __ldg(row + ix);
#pragma unroll
          for (int j = 0; j < 16; ++j) acc[j] = fmaf(wr[j * 147 + kx], v, acc[j]);
        }
      }
    float4* dst = (float4*)(y + (size_t)p * 64 + cg * 16);
#pragma unroll
    for (int j = 0; j < 4; ++j) dst[j] = make_float4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]);
  }
}

// GroupNorm(32) statistics of an NHWC f32 map [rows, C] (C a power of two, 64 .. 1024), one CTA per chunk of `chunk`
// rows (gn_chunk): the chunk's mean of every group, then the sum of squared deviations from it (two passes; no E[x^2]
// - E[x]^2), both summed in a fixed order -> part [chunk index][32] = (mean, M2).  A thread owns 4 channels of every
// (256 / (C / 4))-th row; each group then gathers exactly 32 thread values, one per lane of a warp.
__global__ void __launch_bounds__(256) k_gn_stats(const float* __restrict__ y, int rows, int C, int chunk,
                                                  float2* __restrict__ part) {
  __shared__ float red[256 * 4];
  __shared__ float gmean[32];
  const int t = threadIdx.x, c4n = C >> 2, R = 256 / c4n, cpg = C >> 5;
  const int c4 = t % c4n, rl = t / c4n;
  const int r0 = blockIdx.x * chunk, r1 = min(rows, r0 + chunk);
  const int warp = t >> 5, lane = t & 31;
  const float n = (float)((r1 - r0) * cpg);
  auto group_sum = [&](int g) {  // the 32 values of group g: row lane lane / cpg, channel g * cpg + lane % cpg
    const int ch = g * cpg + lane % cpg;
    float v = red[((lane / cpg) * c4n + (ch >> 2)) * 4 + (ch & 3)];
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
  };
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r = r0 + rl; r < r1; r += R) {
    const float4 v = __ldg((const float4*)(y + (size_t)r * C) + c4);
    s.x += v.x;
    s.y += v.y;
    s.z += v.z;
    s.w += v.w;
  }
  *(float4*)(red + 4 * t) = s;
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float v = group_sum(warp + 8 * i);
    if (lane == 0) gmean[warp + 8 * i] = v / n;
  }
  __syncthreads();
  const float m0 = gmean[(4 * c4) / cpg], m1 = gmean[(4 * c4 + 1) / cpg], m2 = gmean[(4 * c4 + 2) / cpg],
              m3 = gmean[(4 * c4 + 3) / cpg];
  float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r = r0 + rl; r < r1; r += R) {
    const float4 v = __ldg((const float4*)(y + (size_t)r * C) + c4);
    const float a = v.x - m0, b = v.y - m1, c = v.z - m2, d = v.w - m3;
    q.x = fmaf(a, a, q.x);
    q.y = fmaf(b, b, q.y);
    q.z = fmaf(c, c, q.z);
    q.w = fmaf(d, d, q.w);
  }
  *(float4*)(red + 4 * t) = q;
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int g = warp + 8 * i;
    const float v = group_sum(g);
    if (lane == 0) part[(size_t)blockIdx.x * 32 + g] = make_float2(gmean[g], v);
  }
}

// Chan et al.'s pairwise update: (n, mean, M2) of the union of two disjoint sets
__device__ __forceinline__ void chan_merge(float& n, float& m, float& M2, float nb, float mb, float Mb) {
  if (nb == 0.f) return;
  if (n == 0.f) {
    n = nb;
    m = mb;
    M2 = Mb;
    return;
  }
  const float nn = n + nb, d = mb - m;
  m = fmaf(d, nb / nn, m);
  M2 = M2 + Mb + d * d * (n * nb / nn);
  n = nn;
}

// mean and 1 / sqrt(var + eps) of group g from the chunk partials of k_gn_stats, by one warp: lane l merges chunks l,
// l + 32, ... in order, then lanes merge down a fixed tree into lane 0, which stores them to st[0][g] / st[1][g].  The
// same order in every CTA and every launch.
__device__ __forceinline__ void gn_group_stats(const float2* __restrict__ part, int rows, int chunk, int cpg, int g,
                                               float eps, int lane, float (*st)[32]) {
  const int nch = (rows + chunk - 1) / chunk;
  float n = 0.f, m = 0.f, M2 = 0.f;
  for (int k = lane; k < nch; k += 32) {
    const float2 p = part[(size_t)k * 32 + g];
    chan_merge(n, m, M2, (float)((min(rows, (k + 1) * chunk) - k * chunk) * cpg), p.x, p.y);
  }
  for (int o = 16; o; o >>= 1) {
    const float nb = __shfl_down_sync(0xffffffffu, n, o), mb = __shfl_down_sync(0xffffffffu, m, o),
                Mb = __shfl_down_sync(0xffffffffu, M2, o);
    if (lane < o) chan_merge(n, m, M2, nb, mb, Mb);
  }
  if (lane == 0) {
    st[0][g] = m;
    st[1][g] = rsqrtf(M2 / n + eps);
  }
}

// v[j] (+)= (y - mean) rstd gamma + beta for the 8 channels c0 .. c0 + 7 of the f32 element offset o
__device__ __forceinline__ void gn_norm8(const GnInput& in, const float (*st)[32], size_t o, int c0, int cpg, bool add,
                                         float* v) {
  float y[8], gm[8], bt[8];
  *(float4*)y = __ldg((const float4*)(in.y + o));
  *(float4*)(y + 4) = __ldg((const float4*)(in.y + o) + 1);
  *(float4*)gm = __ldg((const float4*)(in.gamma + c0));
  *(float4*)(gm + 4) = __ldg((const float4*)(in.gamma + c0) + 1);
  *(float4*)bt = __ldg((const float4*)(in.beta + c0));
  *(float4*)(bt + 4) = __ldg((const float4*)(in.beta + c0) + 1);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int grp = (c0 + j) / cpg;
    const float r = (y[j] - st[0][grp]) * st[1][grp] * gm[j] + bt[j];
    v[j] = add ? v[j] + r : r;
  }
}

// GroupNorm apply on NHWC f32 [rows, C] -> f16: out = [relu]( (y - mean) rstd gamma + beta  [+ the same of y2 with its
// own statistics and affine]  [+ res] ).  8 channels per thread: two 16-byte loads per f32 input, one 16-byte store.
__global__ void __launch_bounds__(256) k_gn_apply(GnInput a, GnInput b, const __half* __restrict__ res, int relu,
                                                  int rows, int C, int chunk, float eps, __half* __restrict__ out) {
  __shared__ float st[2][2][32];  // [input][mean, rstd][group]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, cpg = C >> 5;
#pragma unroll 1
  for (int i = 0; i < 4; ++i) {
    gn_group_stats(a.part, rows, chunk, cpg, warp + 8 * i, eps, lane, st[0]);
    if (b.y) gn_group_stats(b.part, rows, chunk, cpg, warp + 8 * i, eps, lane, st[1]);
  }
  __syncthreads();
  const size_t idx = (size_t)blockIdx.x * 256 + threadIdx.x;
  const int c8n = C >> 3;
  if (idx >= (size_t)rows * c8n) return;
  const int c0 = (int)(idx % c8n) * 8;
  const size_t o = idx * 8;
  __align__(16) float v[8];
  gn_norm8(a, st[0], o, c0, cpg, false, v);
  if (b.y) gn_norm8(b, st[1], o, c0, cpg, true, v);
  if (res) {
    const uint4 rv = __ldg((const uint4*)(res + o));
    const __half2* h = (const __half2*)&rv;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      v[2 * j] += f.x;
      v[2 * j + 1] += f.y;
    }
  }
  uint4 u;
  __half2* hu = (__half2*)&u;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float x0 = v[2 * j], x1 = v[2 * j + 1];
    if (relu) {
      x0 = fmaxf(x0, 0.f);
      x1 = fmaxf(x1, 0.f);
    }
    hu[j] = __floats2half2_rn(x0, x1);
  }
  *(uint4*)(out + o) = u;
}

// 3x3 stride-2 max-pool with TF SAME padding (0 before, 1 after, pad value 0: BitMaxPool2d with dynamic padding) on
// NHWC f16 [H, W, C] -> [OH, OW, C], 8 channels per thread
__global__ void __launch_bounds__(256) k_maxpool_same(const __half* __restrict__ in, int H, int W, int C,
                                                      __half* __restrict__ out, int OH, int OW) {
  const size_t idx = (size_t)blockIdx.x * 256 + threadIdx.x;
  const int c8n = C >> 3;
  if (idx >= (size_t)OH * OW * c8n) return;
  const int c8 = (int)(idx % c8n);
  const size_t o = idx / c8n;
  const int ox = (int)(o % OW), oy = (int)(o / OW);
  const bool padded = 2 * oy + 2 >= H || 2 * ox + 2 >= W;
  const __half2 init = padded ? __floats2half2_rn(0.f, 0.f) : __half2half2(__ushort_as_half(0xFC00u));  // 0 or -inf
  __half2 m[4] = {init, init, init, init};
  for (int dy = 0; dy < 3; ++dy) {
    const int iy = 2 * oy + dy;
    if (iy >= H) break;
    for (int dx = 0; dx < 3; ++dx) {
      const int ix = 2 * ox + dx;
      if (ix >= W) break;
      const uint4 v = __ldg((const uint4*)(in + ((size_t)iy * W + ix) * C) + c8);
      const __half2* h = (const __half2*)&v;
#pragma unroll
      for (int j = 0; j < 4; ++j) m[j] = __hmax2(m[j], h[j]);
    }
  }
  ((uint4*)(out + o * C))[c8] = *(const uint4*)m;
}

// stride-2 im2col of a k x k conv (k = 1 or 3) with TF SAME padding: `pb` zero rows / columns before, the rest after,
// on NHWC f16 [H, W, C] -> [OH * OW, k * k * C], column tap * C + c.  k = 1, pb = 0 is the subsample of the even pixels.
// 8 channels per thread.
__global__ void __launch_bounds__(256) k_im2col_same(const __half* __restrict__ in, int H, int W, int C, int k, int pb,
                                                     __half* __restrict__ out, int OH, int OW) {
  const size_t idx = (size_t)blockIdx.x * 256 + threadIdx.x;
  const int c8n = C >> 3, kk = k * k;
  if (idx >= (size_t)OH * OW * kk * c8n) return;
  const int c8 = (int)(idx % c8n);
  const size_t r = idx / c8n;
  const int tap = (int)(r % kk);
  const size_t o = r / kk;
  const int ox = (int)(o % OW), oy = (int)(o / OW);
  const int iy = 2 * oy - pb + tap / k, ix = 2 * ox - pb + tap % k;
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = __ldg((const uint4*)(in + ((size_t)iy * W + ix) * C) + c8);
  ((uint4*)out)[idx] = v;
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

size_t attention_bias_smem(int ph, int pw) {
  const size_t num = (size_t)(2 * ph - 1) * (2 * pw - 1) + 3;
  return kAttnSmem + (num + 3) / 4 * 16 + (size_t)((ph * pw + 1 + 127) / 128) * 128 * 4;
}

cudaError_t launch_attention(const CUtensorMap& q, const CUtensorMap& k, const CUtensorMap& v, int ntok, int dmodel,
                             __half* out, int heads, int images, int npad, cudaStream_t s, const float* rpb, int gw) {
  static bool attr_set = false, attr_bias_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k_umma_attention<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmem);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  AttnArgs a;
  a.ntok = ntok;
  a.dmodel = dmodel;
  a.out = out;
  a.heads = heads;
  a.npad = npad;
  a.rpb = rpb;
  a.gw = gw;
  dim3 grid((ntok + kAttnRows - 1) / kAttnRows, heads * images);
  if (!rpb) {
    k_umma_attention<false><<<grid, kAttnThreads, kAttnSmem, s>>>(q, k, v, a);
    return cudaGetLastError();
  }
  if (gw < 1 || (ntok - 1) % gw) return cudaErrorInvalidValue;
  const size_t smem = attention_bias_smem((ntok - 1) / gw, gw);
  if (smem > (size_t)kAttnSmemMax) return cudaErrorInvalidValue;
  if (!attr_bias_set) {
    cudaError_t e = cudaFuncSetAttribute(k_umma_attention<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmemMax);
    if (e != cudaSuccess) return e;
    attr_bias_set = true;
  }
  k_umma_attention<true><<<grid, kAttnThreads, smem, s>>>(q, k, v, a);
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

// BiT front end of DPT-Hybrid
void launch_bit_stem(const float* px, int H, int W, const float* w, float* y, cudaStream_t s) {
  const int OH = H / 2, OW = W / 2;
  const int blocks = (OH * OW + 63) / 64, cap = 4 * sm_count();  // 37.6 KB of weights per CTA: a few CTAs per SM
  k_bit_stem<<<blocks < cap ? blocks : cap, 256, 0, s>>>(px, H, W, w, y, OH, OW);
}
int gn_chunk(int rows) { return (rows + kGnMaxChunks - 1) / kGnMaxChunks; }
void launch_gn_stats(const float* y, int rows, int C, float2* part, cudaStream_t s) {
  const int chunk = gn_chunk(rows);
  k_gn_stats<<<(rows + chunk - 1) / chunk, 256, 0, s>>>(y, rows, C, chunk, part);
}
void launch_gn_apply(const GnInput& a, const GnInput& b, const __half* res, int relu, int rows, int C, __half* out,
                     cudaStream_t s) {
  const size_t total = (size_t)rows * (C / 8);
  k_gn_apply<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(a, b, res, relu, rows, C, gn_chunk(rows), kGnEps, out);
}
void launch_maxpool_same(const __half* in, int H, int W, int C, __half* out, cudaStream_t s) {
  const int OH = H / 2, OW = W / 2;
  const size_t total = (size_t)OH * OW * (C / 8);
  k_maxpool_same<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(in, H, W, C, out, OH, OW);
}
void launch_im2col_same(const __half* in, int H, int W, int C, int k, int pb, __half* out, cudaStream_t s) {
  const int OH = H / 2, OW = W / 2;
  const size_t total = (size_t)OH * OW * k * k * (C / 8);
  k_im2col_same<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(in, H, W, C, k, pb, out, OH, OW);
}

}  // namespace vd3d
