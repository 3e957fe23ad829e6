// sr_kernels.cu -- the output end of the Real-ESRGAN stage fused into run_esrgan's first INTER_CUBIC resize
// (core/merged_pipeline.py:256-264).  Compiled with -fmad=false like dibr_kernels.cu: k_resize_cubic_u8's `v + src * c`
// chain is not contracted there, and this kernel must round exactly like k_sr_out followed by k_resize_cubic_u8.
#include "dibr_device.cuh"
#include "dibr_launch.h"

namespace vd3d {

// One byte of the virtual 4h x 4w BGR image of k_sr_out (depth_kernels.cu): PixelShuffle(4) of the last conv + the
// network input / 255, clipped to [0,1], x255, truncated.  cv = conv[y, x, (2 - b) * 16 + (Y & 3) * 4 + (X & 3)],
// base = bgr[y, x, b] / 255 (b: 0 = B).
__device__ __forceinline__ float sr_byte(float cv, float base) {
  float v = cv + base;
  v = fminf(fmaxf(v, 0.f), 1.f) * 255.0f;
  return (float)(uint8_t)(int)v;
}

// cv2.resize(virtual [4h, 4w, 3], (ow, oh), INTER_CUBIC): taps and summation order of k_resize_cubic_u8, each tap
// computed from the conv output on the fly.  kBlock (ow == w, oh == h, the 4:1 ratio of input_res_pct = 100): every
// output pixel's 4 x 4 taps are its own PixelShuffle block (fraction 0.5, no border clamping), one contiguous row of
// 48 floats.
template <bool kBlock>
__global__ void __launch_bounds__(256) k_sr_tail_cubic(const float* __restrict__ conv, const uint8_t* __restrict__ bgr,
                                                       int h, int w, uint8_t* __restrict__ dst, int oh, int ow) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= ow || y >= oh) return;
  const CubicTap tx = cubic_tap(x, 4 * w, ow), ty = cubic_tap(y, 4 * h, oh);
  uint8_t* o = dst + ((size_t)y * ow + x) * 3;
  if constexpr (kBlock) {
    const float4* row = reinterpret_cast<const float4*>(conv + ((size_t)y * w + x) * 48);
    const uint8_t* q = bgr + ((size_t)y * w + x) * 3;
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      const float base = (float)q[b] / 255.0f;
      float s[4][4];  // [tap row][tap column]
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float4 v = __ldg(row + (2 - b) * 4 + k);
        s[k][0] = sr_byte(v.x, base);
        s[k][1] = sr_byte(v.y, base);
        s[k][2] = sr_byte(v.z, base);
        s[k][3] = sr_byte(v.w, base);
      }
      float col[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float v = s[0][k] * ty.c[0];
        v = v + (s[1][k] * ty.c[1]);
        v = v + (s[2][k] * ty.c[2]);
        v = v + (s[3][k] * ty.c[3]);
        col[k] = v;
      }
      float r = (((col[0] * tx.c[0]) + (col[1] * tx.c[1])) + (col[2] * tx.c[2])) + (col[3] * tx.c[3]);
      o[b] = rhe_u8(r);
    }
  } else {
    for (int b = 0; b < 3; ++b) {
      float col[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {  // rows first: the value of column tx.o[k] at output row y
        const int X = tx.o[k];
        float s[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int Y = ty.o[j];
          const size_t px = (size_t)(Y >> 2) * w + (X >> 2);
          s[j] = sr_byte(__ldg(conv + px * 48 + (2 - b) * 16 + (Y & 3) * 4 + (X & 3)), (float)bgr[px * 3 + b] / 255.0f);
        }
        float v = s[0] * ty.c[0];
        v = v + (s[1] * ty.c[1]);
        v = v + (s[2] * ty.c[2]);
        v = v + (s[3] * ty.c[3]);
        col[k] = v;
      }
      float r = (((col[0] * tx.c[0]) + (col[1] * tx.c[1])) + (col[2] * tx.c[2])) + (col[3] * tx.c[3]);
      o[b] = rhe_u8(r);
    }
  }
}

// postprocess_esr (core/merged_pipeline.py:227-231) of the RRDBNet output, whose network output has no base add:
// one thread per pixel.
__global__ void __launch_bounds__(256) k_rrdb_out(const float* __restrict__ rgb, int ld, uint8_t* __restrict__ bgr,
                                                  size_t npix) {
  const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (i >= npix) return;
  const float* p = rgb + i * ld;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = fminf(fmaxf(__ldg(p + c), 0.f), 1.f) * 255.0f;
    bgr[i * 3 + 2 - c] = (uint8_t)(int)v;
  }
}

void launch_rrdb_out(const float* rgb, int ld, uint8_t* bgr, size_t npix, cudaStream_t s) {
  k_rrdb_out<<<(unsigned)((npix + 255) / 256), 256, 0, s>>>(rgb, ld, bgr, npix);
}

void launch_sr_tail_cubic(const float* conv, const uint8_t* bgr, int h, int w, uint8_t* dst, int oh, int ow,
                          cudaStream_t s) {
  dim3 g((ow + 31) / 32, (oh + 7) / 8);
  if (ow == w && oh == h)
    k_sr_tail_cubic<true><<<g, 256, 0, s>>>(conv, bgr, h, w, dst, oh, ow);
  else
    k_sr_tail_cubic<false><<<g, 256, 0, s>>>(conv, bgr, h, w, dst, oh, ow);
}

}  // namespace vd3d
