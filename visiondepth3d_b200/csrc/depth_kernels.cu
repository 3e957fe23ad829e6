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
// The output is the window [oy0, oy0 + OH) x [ox0, ox0 + OW) of a VH x VW resize (ZoeDepth: the padded size, cropped);
// VH = OH, VW = OW and zero offsets for every other model.
__global__ void __launch_bounds__(256) k_depth_upsample_minmax(const float* __restrict__ d, int IH, int IW,
                                                               float* __restrict__ out, int OH, int OW, int VH, int VW,
                                                               int oy0, int ox0, unsigned* __restrict__ mm) {
  int ox = blockIdx.x * 32 + (threadIdx.x & 31);
  int oy = blockIdx.y * 8 + (threadIdx.x >> 5);
  float v = 0.f;
  bool ok = ox < OW && oy < OH;
  if (ok) {
    if (IH == VH && IW == VW) {
      v = d[(size_t)(oy + oy0) * IW + ox + ox0];
    } else {
      float sy = (float)IH / (float)VH, sx = (float)IW / (float)VW;
      float fy = sy * ((float)(oy + oy0) + 0.5f) - 0.5f, fx = sx * ((float)(ox + ox0) + 0.5f) - 0.5f;
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
// ZoeDepth (transformers 5.5 models/zoedepth): image processor, domain router, attractor update and the conditional
// log-binomial head.  Every f32 step writes its products and sums with explicit _rn intrinsics where the order matters,
// so that the compiler does not contract them into FMAs the CPU reference does not use.
// ---------------------------------------------------------------------------

// torch upsample_bilinear2d(align_corners=True) index and weight of one axis, in f32 as ATen's CPU kernel computes them
__device__ __forceinline__ void ac_axis(int o, int in, int out, int& i0, int& i1, float& l0, float& l1) {
  const float scale = out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f;
  const float real = scale * (float)o;
  i0 = min((int)floorf(real), in - 1);
  l1 = fminf(fmaxf(real - (float)i0, 0.f), 1.f);
  l0 = 1.f - l1;
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
}
// ((x00 w0 + x01 w1) h0) + ((x10 w0 + x11 w1) h1): ATen's Interpolate<2> order
__device__ __forceinline__ float bilerp(float x00, float x01, float x10, float x11, float h0, float h1, float w0,
                                        float w1) {
  const float t0 = __fadd_rn(__fmul_rn(x00, w0), __fmul_rn(x01, w1));
  const float t1 = __fadd_rn(__fmul_rn(x10, w0), __fmul_rn(x11, w1));
  return __fadd_rn(__fmul_rn(t0, h0), __fmul_rn(t1, h1));
}
__device__ __forceinline__ float softplus_t(float x) { return x > 20.f ? x : log1pf(expf(x)); }  // torch beta 1, 20

// ZoeDepthImageProcessor: rescale (x * (1/255) in f32), reflect-pad pad_h rows / pad_w columns, bilinear
// align_corners=True to OH x OW, (v - mean) / std.  The padding is folded into the sampler: padded index p maps to
// source row |p - pad| reflected at the far edge.  u8 [h, w, 3] (BGR when swap_rb) -> f32 [3, OH, OW].
__device__ __forceinline__ int reflect_idx(int p, int pad, int n) {
  int r = p - pad;
  if (r < 0) r = -r;
  if (r >= n) r = 2 * (n - 1) - r;
  return r;
}
__global__ void __launch_bounds__(256) k_zoe_preprocess(const uint8_t* __restrict__ img, int h, int w, int swap_rb,
                                                        int pad_h, int pad_w, float* __restrict__ px, int OH, int OW,
                                                        PreprocParams pp) {
  const int ox = blockIdx.x * 32 + (threadIdx.x & 31), oy = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (ox >= OW || oy >= OH) return;
  int y0, y1, x0, x1;
  float h0, h1, w0, w1;
  ac_axis(oy, h + 2 * pad_h, OH, y0, y1, h0, h1);
  ac_axis(ox, w + 2 * pad_w, OW, x0, x1, w0, w1);
  y0 = reflect_idx(y0, pad_h, h);
  y1 = reflect_idx(y1, pad_h, h);
  x0 = reflect_idx(x0, pad_w, w);
  x1 = reflect_idx(x1, pad_w, w);
  const float rs = 1.0f / 255.0f;
  const uint8_t *p00 = img + ((size_t)y0 * w + x0) * 3, *p01 = img + ((size_t)y0 * w + x1) * 3,
                *p10 = img + ((size_t)y1 * w + x0) * 3, *p11 = img + ((size_t)y1 * w + x1) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int sc = swap_rb ? 2 - c : c;
    const float v = bilerp(__fmul_rn((float)p00[sc], rs), __fmul_rn((float)p01[sc], rs), __fmul_rn((float)p10[sc], rs),
                           __fmul_rn((float)p11[sc], rs), h0, h1, w0, w1);
    px[((size_t)c * OH + oy) * OW + ox] = __fdiv_rn(__fsub_rn(v, pp.mean[c]), pp.std[c]);
  }
}

// ---- router: ZoeDepthPatchTransformerEncoder + ZoeDepthMLPClassifier on one image, one CTA, f32 throughout ----
// Y[r, n] (= or +=) act(sum_k X[r, k] W[n, k] (/ div) + b[n]) for r < R, n < N; W element (n, k) at W[n wsn + k wsk].
// 32 x 32 output tiles, K staged 32 at a time in shared memory; each of the 256 threads owns 4 rows of one column.
// mode 0: store, 1: ReLU then store, 2: add to Y (the post-norm residual).  Ends with a barrier.
__device__ __forceinline__ void zr_linear(const float* __restrict__ X, int ldx, int R, int K, const float* __restrict__ Wt, int wsn,
                          int wsk, const float* __restrict__ b, int N, float* Y, int ldy, int mode, float div) {
  __shared__ float xs[32][33], ws[32][33];
  const int tid = threadIdx.x, col = tid & 31, rg = tid >> 5;
  for (int r0 = 0; r0 < R; r0 += 32)
    for (int n0 = 0; n0 < N; n0 += 32) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int k0 = 0; k0 < K; k0 += 32) {
        for (int i = tid; i < 32 * 32; i += 256) {
          const int rr = i >> 5, kk = i & 31;
          xs[rr][kk] = (r0 + rr < R && k0 + kk < K) ? X[(size_t)(r0 + rr) * ldx + k0 + kk] : 0.f;
          ws[rr][kk] = (n0 + rr < N && k0 + kk < K) ? Wt[(size_t)(n0 + rr) * wsn + (size_t)(k0 + kk) * wsk] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int kk = 0; kk < 32; ++kk) {
          const float wv = ws[col][kk];
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[i] = fmaf(xs[rg * 4 + i][kk], wv, acc[i]);
        }
        __syncthreads();
      }
      const int n = n0 + col;
      if (n < N)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int r = r0 + rg * 4 + i;
          float v = div != 1.f ? acc[i] / div : acc[i];
          if (b) v += b[n];
          if (mode == 1) v = fmaxf(v, 0.f);
          if (r < R) {
            float* y = Y + (size_t)r * ldy + n;
            *y = mode == 2 ? *y + v : v;
          }
        }
    }
  __syncthreads();
}
// LayerNorm(eps 1e-5) of rows [0, R) of X [., 128] in place, one warp per row
__device__ __forceinline__ void zr_layernorm(float* X, int R, const float* __restrict__ g, const float* __restrict__ b) {
  const int lane = threadIdx.x & 31;
  for (int r = threadIdx.x >> 5; r < R; r += blockDim.x >> 5) {
    float* x = X + (size_t)r * kZoeE;
    float v[4], s = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) s += v[i] = x[lane + 32 * i];
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)kZoeE;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) q += (v[i] - mean) * (v[i] - mean);
    for (int o = 16; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = 1.f / sqrtf(q / (float)kZoeE + 1e-5f);
#pragma unroll
    for (int i = 0; i < 4; ++i) x[lane + 32 * i] = (v[i] - mean) * rstd * g[lane + 32 * i] + b[lane + 32 * i];
  }
  __syncthreads();
}
// softmax of rows [0, R) of P [., S] in place, one warp per row
__device__ __forceinline__ void zr_softmax(float* P, int R, int S) {
  const int lane = threadIdx.x & 31;
  for (int r = threadIdx.x >> 5; r < R; r += blockDim.x >> 5) {
    float* p = P + (size_t)r * S;
    float m = -INFINITY;
    for (int j = lane; j < S; j += 32) m = fmaxf(m, p[j]);
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int j = lane; j < S; j += 32) s += p[j] = expf(p[j] - m);
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    for (int j = lane; j < S; j += 32) p[j] = p[j] / s;
  }
  __syncthreads();
}
// x: the bottleneck conv2 output f32 [n, F]; wts: the packed router (zoe_router_floats); pe f32 [n + 1, 128];
// scratch: zoe_router_scratch(n) floats.  Writes logits[2] and route (1 when logits[1] > logits[0], torch.argmax's
// first index on a tie).  The last encoder layer computes the CLS row only: nothing else of it is read.
__global__ void __launch_bounds__(256, 1) k_zoe_router(const float* __restrict__ x, int n, int F,
                                                    const float* __restrict__ wts, const float* __restrict__ pe,
                                                    float* __restrict__ scratch, float* __restrict__ logits,
                                                    int* __restrict__ route) {
  constexpr int E = kZoeE, FF = kZoeFF, HD = E / kZoeHeads;
  const int S = n + 1;
  float *X = scratch, *QKV = X + (size_t)S * E, *A = QKV + (size_t)S * 3 * E, *Hb = A + (size_t)S * E,
        *P = Hb + (size_t)S * FF;
  const float* w = wts;
  const float *ew = w, *eb = ew + E * F;
  w = eb + E;
  for (int i = threadIdx.x; i < E; i += blockDim.x) X[i] = 0.f;  // the zero CLS token
  zr_linear(x, F, n, F, ew, F, 1, eb, E, X + E, E, 0, 1.f);
  for (int i = threadIdx.x; i < S * E; i += blockDim.x) X[i] = X[i] + pe[i];
  __syncthreads();
  for (int l = 0; l < kZoeLayers; ++l) {
    const int Rq = l == kZoeLayers - 1 ? 1 : S;
    const float *qw = w, *qb = qw + 3 * E * E, *ow = qb + 3 * E, *ob = ow + E * E, *n1g = ob + E, *n1b = n1g + E,
                *l1w = n1b + E, *l1b = l1w + FF * E, *l2w = l1b + FF, *l2b = l2w + E * FF, *n2g = l2b + E,
                *n2b = n2g + E;
    w = n2b + E;
    zr_linear(X, E, S, E, qw, E, 1, qb, 3 * E, QKV, 3 * E, 0, 1.f);
    for (int h = 0; h < kZoeHeads; ++h) {
      zr_linear(QKV + h * HD, 3 * E, Rq, HD, QKV + E + h * HD, 3 * E, 1, nullptr, S, P, S, 0, sqrtf((float)HD));
      zr_softmax(P, Rq, S);
      zr_linear(P, S, Rq, S, QKV + 2 * E + h * HD, 1, 3 * E, nullptr, HD, A + h * HD, E, 0, 1.f);
    }
    zr_linear(A, E, Rq, E, ow, E, 1, ob, E, X, E, 2, 1.f);
    zr_layernorm(X, Rq, n1g, n1b);
    zr_linear(X, E, Rq, E, l1w, E, 1, l1b, FF, Hb, FF, 1, 1.f);
    zr_linear(Hb, FF, Rq, FF, l2w, FF, 1, l2b, E, X, E, 2, 1.f);
    zr_layernorm(X, Rq, n2g, n2b);
  }
  const float *c1w = w, *c1b = c1w + E * E, *c2w = c1b + E, *c2b = c2w + 2 * E;
  zr_linear(X, E, 1, E, c1w, E, 1, c1b, E, Hb, E, 1, 1.f);
  zr_linear(Hb, E, 1, E, c2w, E, 1, c2b, 2, A, 2, 0, 1.f);
  if (threadIdx.x == 0) {
    logits[0] = A[0];
    logits[1] = A[1];
    *route = A[1] > A[0] ? 1 : 0;
  }
}

// ZoeDepthAttractorLayerUnnormed on an H x W map, one thread per pixel: attractors a = Softplus(conv2(hid)) with the
// route's conv2 (staged in shared memory; hid f16 [H W, ldh] holds ReLU(conv1) of every configuration, the route's at
// column route * E), bins c = bilinear_ac(prev) (prev f32 [Hp Wp, ldp] at column route * prev_cfg_stride, Softplus
// applied first when prev_softplus: the seed regressor's raw conv2), then c += (sum_i dx / (1 + 300 dx^2)) / na with
// dx = a_i - c, summed attractor by attractor -> out f32 [H W, kZoeBins].
__global__ void __launch_bounds__(128) k_zoe_attractor(const __half* __restrict__ hid, int ldh, int E,
                                                       const float* __restrict__ w2, const float* __restrict__ b2,
                                                       int na, const float* __restrict__ prev, int ldp,
                                                       int prev_cfg_stride, int prev_softplus, int Hp, int Wp,
                                                       float* __restrict__ out, int H, int W,
                                                       const int* __restrict__ route) {
  __shared__ float sw[kZoeMaxAttr * kZoeE + kZoeMaxAttr];
  const int rt = *route;
  for (int i = threadIdx.x; i < na * E; i += blockDim.x) sw[i] = w2[(size_t)rt * na * E + i];
  for (int i = threadIdx.x; i < na; i += blockDim.x) sw[na * E + i] = b2[rt * na + i];
  __syncthreads();
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= H * W) return;
  const int oy = pix / W, ox = pix % W;
  float a[kZoeMaxAttr];
#pragma unroll
  for (int i = 0; i < kZoeMaxAttr; ++i) a[i] = 0.f;
  const __half* hp = hid + (size_t)pix * ldh + (size_t)rt * E;
  for (int e0 = 0; e0 < E; e0 += 8) {
    const uint4 u = *(const uint4*)(hp + e0);
    const __half2* h2 = (const __half2*)&u;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h2[j]);
#pragma unroll
      for (int i = 0; i < kZoeMaxAttr; ++i)
        if (i < na) a[i] = fmaf(sw[i * E + e0 + 2 * j + 1], f.y, fmaf(sw[i * E + e0 + 2 * j], f.x, a[i]));
    }
  }
#pragma unroll
  for (int i = 0; i < kZoeMaxAttr; ++i)
    if (i < na) a[i] = softplus_t(a[i] + sw[na * E + i]);
  int y0, y1, x0, x1;
  float h0, h1, w0, w1;
  ac_axis(oy, Hp, H, y0, y1, h0, h1);
  ac_axis(ox, Wp, W, x0, x1, w0, w1);
  const float *q00 = prev + ((size_t)y0 * Wp + x0) * ldp + (size_t)rt * prev_cfg_stride,
              *q01 = prev + ((size_t)y0 * Wp + x1) * ldp + (size_t)rt * prev_cfg_stride,
              *q10 = prev + ((size_t)y1 * Wp + x0) * ldp + (size_t)rt * prev_cfg_stride,
              *q11 = prev + ((size_t)y1 * Wp + x1) * ldp + (size_t)rt * prev_cfg_stride;
  const float nf = (float)na;
  float* o = out + (size_t)pix * kZoeBins;
  for (int j0 = 0; j0 < kZoeBins; j0 += 16) {
    float c[16], dc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      float v00 = q00[j0 + j], v01 = q01[j0 + j], v10 = q10[j0 + j], v11 = q11[j0 + j];
      if (prev_softplus) {
        v00 = softplus_t(v00);
        v01 = softplus_t(v01);
        v10 = softplus_t(v10);
        v11 = softplus_t(v11);
      }
      c[j] = bilerp(v00, v01, v10, v11, h0, h1, w0, w1);
      dc[j] = 0.f;
    }
#pragma unroll
    for (int i = 0; i < kZoeMaxAttr; ++i)
      if (i < na)
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float dx = __fsub_rn(a[i], c[j]);
          dc[j] = __fadd_rn(dc[j], __fdiv_rn(dx, __fadd_rn(1.f, __fmul_rn(300.f, __fmul_rn(dx, dx)))));
        }
#pragma unroll
    for (int j = 0; j < 16; ++j) o[j0 + j] = __fadd_rn(c[j], __fdiv_rn(dc[j], nf));
  }
}

// ZoeDepthConditionalLogBinomialSoftmax and the expectation, one thread per pixel of the H x W processed size:
// the input is cat(act (32 channels f16 [H W, 32]) [, relu(w3 . act + b3) when w3], bilinear_ac(emb) (f16 [He We, E]));
// MLP conv -> GELU -> conv(4) -> Softplus with the route's weights (staged in shared memory: w1 [cin][HID], b1 [HID],
// w2 [4][HID], b2 [4]); p and t from the normalised pairs (+1e-4); y_k = log_binom(K - 1, k) + k log p + (K - 1 - k)
// log(1 - p) with p clamped to [1e-4, 1]; depth = sum_k softmax(y / t)_k * bilinear_ac(bins)_k (bins f32 [He We, K]).
template <int HID>
__global__ void __launch_bounds__(128) k_zoe_logbinom(const __half* __restrict__ act, const float* __restrict__ w3,
                                                      const float* __restrict__ b3, const __half* __restrict__ emb,
                                                      const float* __restrict__ bins, int He, int We, int E,
                                                      const float* __restrict__ mlp, int cin, float min_t, float max_t,
                                                      float* __restrict__ depth, int H, int W,
                                                      const int* __restrict__ route) {
  extern __shared__ float sm[];
  const int per = cin * HID + HID + 4 * HID + 4;
  const float* src = mlp + (size_t)(*route) * per;
  for (int i = threadIdx.x; i < per; i += blockDim.x) sm[i] = src[i];
  __syncthreads();
  const float *w1 = sm, *b1 = w1 + cin * HID, *w2 = b1 + HID, *b2 = w2 + 4 * HID;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= H * W) return;
  const int oy = pix / W, ox = pix % W;
  float hacc[HID];
#pragma unroll
  for (int j = 0; j < HID; ++j) hacc[j] = b1[j];
  int k = 0;
  auto feed = [&](float v) {
#pragma unroll
    for (int j = 0; j < HID; ++j) hacc[j] = fmaf(w1[k * HID + j], v, hacc[j]);
    ++k;
  };
  const __half* ap = act + (size_t)pix * 32;
  float rel = b3 ? b3[0] : 0.f;
  for (int c0 = 0; c0 < 32; c0 += 8) {
    const uint4 u = *(const uint4*)(ap + c0);
    const __half2* h2 = (const __half2*)&u;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h2[j]);
      feed(f.x);
      feed(f.y);
      if (b3) rel = fmaf(w3[c0 + 2 * j + 1], f.y, fmaf(w3[c0 + 2 * j], f.x, rel));
    }
  }
  if (b3) feed(fmaxf(rel, 0.f));
  int y0, y1, x0, x1;
  float h0, h1, wx0, wx1;
  ac_axis(oy, He, H, y0, y1, h0, h1);
  ac_axis(ox, We, W, x0, x1, wx0, wx1);
  const size_t i00 = (size_t)y0 * We + x0, i01 = (size_t)y0 * We + x1, i10 = (size_t)y1 * We + x0,
               i11 = (size_t)y1 * We + x1;
  for (int e = 0; e < E; ++e)
    feed(bilerp(__half2float(emb[i00 * E + e]), __half2float(emb[i01 * E + e]), __half2float(emb[i10 * E + e]),
                __half2float(emb[i11 * E + e]), h0, h1, wx0, wx1));
  float o4[4];
#pragma unroll
  for (int m = 0; m < 4; ++m) o4[m] = b2[m];
#pragma unroll
  for (int j = 0; j < HID; ++j) {
    const float g = 0.5f * hacc[j] * (1.f + erff(hacc[j] * 0.70710678118654752f));
#pragma unroll
    for (int m = 0; m < 4; ++m) o4[m] = fmaf(w2[m * HID + j], g, o4[m]);
  }
#pragma unroll
  for (int m = 0; m < 4; ++m) o4[m] = softplus_t(o4[m]);
  const float pe = 1e-4f;
  const float pa = __fadd_rn(o4[0], pe), pb = __fadd_rn(o4[1], pe);
  float p = __fdiv_rn(pa, __fadd_rn(pa, pb));
  const float ta = __fadd_rn(o4[2], pe), tb = __fadd_rn(o4[3], pe);
  const float t = __fadd_rn(__fmul_rn(max_t - min_t, __fdiv_rn(ta, __fadd_rn(ta, tb))), min_t);
  const float q = fminf(fmaxf(__fsub_rn(1.f, p), pe), 1.f);
  p = fminf(fmaxf(p, pe), 1.f);
  const float lp = logf(p), lq = logf(q);
  constexpr int K = kZoeBins;
  const float n = __fadd_rn((float)(K - 1), 1e-7f), nl = __fmul_rn(n, logf(n));
  auto logit = [&](int kk) {
    const float kf = __fadd_rn((float)kk, 1e-7f), nk = __fsub_rn(n, kf);
    const float lb = __fsub_rn(__fsub_rn(nl, __fmul_rn(kf, logf(kf))), __fmul_rn(nk, logf(__fadd_rn(nk, 1e-7f))));
    const float y = __fadd_rn(__fadd_rn(lb, __fmul_rn((float)kk, lp)), __fmul_rn((float)(K - 1 - kk), lq));
    return __fdiv_rn(y, t);
  };
  float mx = -INFINITY;
  for (int kk = 0; kk < K; ++kk) mx = fmaxf(mx, logit(kk));
  float s = 0.f;
  for (int kk = 0; kk < K; ++kk) s = __fadd_rn(s, expf(__fsub_rn(logit(kk), mx)));
  float d = 0.f;
  for (int kk = 0; kk < K; ++kk) {
    const float c = bilerp(bins[i00 * K + kk], bins[i01 * K + kk], bins[i10 * K + kk], bins[i11 * K + kk], h0, h1, wx0,
                           wx1);
    d = __fadd_rn(d, __fmul_rn(__fdiv_rn(expf(__fsub_rn(logit(kk), mx)), s), c));
  }
  depth[pix] = d;
}

// ---------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------
size_t zoe_router_floats(int F) {
  constexpr size_t E = kZoeE, FF = kZoeFF;
  const size_t layer = 3 * E * E + 3 * E + E * E + E + 2 * E + FF * E + FF + E * FF + E + 2 * E;
  return E * F + E + kZoeLayers * layer + E * E + E + 2 * E + 2;
}
size_t zoe_router_scratch(int n) {
  const size_t S = n + 1;
  return S * kZoeE * 5 + S * kZoeFF + S * S;
}
void launch_zoe_preprocess(const uint8_t* img, int h, int w, int swap_rb, int pad_h, int pad_w, float* px, int OH,
                           int OW, const PreprocParams& pp, cudaStream_t s) {
  dim3 g((OW + 31) / 32, (OH + 7) / 8);
  k_zoe_preprocess<<<g, 256, 0, s>>>(img, h, w, swap_rb, pad_h, pad_w, px, OH, OW, pp);
}
void launch_zoe_router(const float* x, int n, int F, const float* wts, const float* pe, float* scratch, float* logits,
                       int* route, cudaStream_t s) {
  k_zoe_router<<<1, 256, 0, s>>>(x, n, F, wts, pe, scratch, logits, route);
}
void launch_zoe_attractor(const __half* hid, int ldh, int E, const float* w2, const float* b2, int na, const float* prev,
                          int ldp, int prev_cfg_stride, int prev_softplus, int Hp, int Wp, float* out, int H, int W,
                          const int* route, cudaStream_t s) {
  k_zoe_attractor<<<(H * W + 127) / 128, 128, 0, s>>>(hid, ldh, E, w2, b2, na, prev, ldp, prev_cfg_stride,
                                                      prev_softplus, Hp, Wp, out, H, W, route);
}
size_t zoe_logbinom_floats(int cin, int hid) { return (size_t)cin * hid + hid + 4 * hid + 4; }
template <int HID>
static cudaError_t launch_logbinom_t(const __half* act, const float* w3, const float* b3, const __half* emb,
                                     const float* bins, int He, int We, int E, const float* mlp, int cin, float min_t,
                                     float max_t, float* depth, int H, int W, const int* route, cudaStream_t s) {
  const size_t smem = zoe_logbinom_floats(cin, HID) * sizeof(float);
  cudaError_t e = cudaFuncSetAttribute(k_zoe_logbinom<HID>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k_zoe_logbinom<HID><<<(H * W + 127) / 128, 128, smem, s>>>(act, w3, b3, emb, bins, He, We, E, mlp, cin, min_t, max_t,
                                                            depth, H, W, route);
  return cudaGetLastError();
}
cudaError_t launch_zoe_logbinom(const __half* act, const float* w3, const float* b3, const __half* emb,
                                const float* bins, int He, int We, int E, const float* mlp, int cin, int hid,
                                float min_t, float max_t, float* depth, int H, int W, const int* route, cudaStream_t s) {
  if (hid == 40)
    return launch_logbinom_t<40>(act, w3, b3, emb, bins, He, We, E, mlp, cin, min_t, max_t, depth, H, W, route, s);
  if (hid == 80)
    return launch_logbinom_t<80>(act, w3, b3, emb, bins, He, We, E, mlp, cin, min_t, max_t, depth, H, W, route, s);
  return cudaErrorInvalidValue;
}
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
void launch_depth_post_crop(const float* depth, int IH, int IW, float* up, int OH, int OW, int pad_h, int pad_w,
                            unsigned* mm, uint8_t* out_u8, int invert, cudaStream_t s) {
  k_minmax_reset<<<1, 1, 0, s>>>(mm);
  dim3 g((OW + 31) / 32, (OH + 7) / 8);
  k_depth_upsample_minmax<<<g, 256, 0, s>>>(depth, IH, IW, up, OH, OW, OH + 2 * pad_h, OW + 2 * pad_w, pad_h, pad_w, mm);
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
