// dibr_device.cuh -- device helpers shared by dibr_kernels.cu (exact path) and dibr_fast.cu (fast path).
// Every function restates one rounding sequence of the reference (file:line cited in place); both
// translation units are compiled with -fmad=false and spell the fused ops (__fmaf_rn) explicitly.
#pragma once
#include <math.h>
#include <stdint.h>

#include "dibr_launch.h"

namespace vd3d {

// ---------------------------------------------------------------------------
// helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

// cv2.cvtColor(BGR2GRAY) on u8: (B*3735 + G*19235 + R*9798 + 2^14) >> 15
__device__ __forceinline__ float depth_src01(const uint8_t* __restrict__ p, int ch, int pitch_px, int y, int x) {
  const uint8_t* q = p + ((size_t)y * pitch_px + x) * ch;
  int g;
  if (ch == 1) {
    g = q[0];
  } else {
    g = (q[0] * 3735 + q[1] * 19235 + q[2] * 9798 + (1 << 14)) >> 15;
  }
  return (float)g / 255.0f;
}

// F.interpolate(bilinear, align_corners=False) axis set-up (torch 2.11 rounding:
// src = fma(scale, dst+0.5, -0.5), clamped at 0)
struct RsAxis {
  int i0, i1;
  float l0, l1;
};
__device__ __forceinline__ RsAxis rs_axis(int d, int insz, int outsz) {
  RsAxis a;
  float scale = (float)insz / (float)outsz;
  float s = __fmaf_rn(scale, (float)d + 0.5f, -0.5f);
  s = fmaxf(s, 0.f);
  a.i0 = (int)s;
  if (a.i0 > insz - 1) a.i0 = insz - 1;
  a.i1 = a.i0 + (a.i0 < insz - 1 ? 1 : 0);
  a.l1 = s - (float)a.i0;
  a.l0 = 1.f - a.l1;
  return a;
}
// value = fma(row(y0), ly0, row(y1)*ly1), row = fma(a, lx0, b*lx1)
__device__ __forceinline__ float rs_combine(float v00, float v01, float v10, float v11, const RsAxis& ax,
                                            const RsAxis& ay) {
  float r0 = __fmaf_rn(v00, ax.l0, v01 * ax.l1);
  float r1 = __fmaf_rn(v10, ax.l0, v11 * ax.l1);
  return __fmaf_rn(r0, ay.l0, r1 * ay.l1);
}

__device__ __forceinline__ float bilinear_f32(const float* __restrict__ src, int sh, int sw, int oh, int ow, int y,
                                              int x) {
  if (sh == oh && sw == ow) return src[(size_t)y * sw + x];
  RsAxis ax = rs_axis(x, sw, ow), ay = rs_axis(y, sh, oh);
  const float* r0 = src + (size_t)ay.i0 * sw;
  const float* r1 = src + (size_t)ay.i1 * sw;
  return rs_combine(r0[ax.i0], r0[ax.i1], r1[ax.i0], r1[ax.i1], ax, ay);
}

__device__ __forceinline__ uint8_t trunc_u8(float v01) {
  // tensor_to_frame (core/render_3d.py:289-291): (v*255).astype(uint8), v in [0,1]
  float t = v01 * 255.0f;
  int i = (int)t;
  return (uint8_t)(i < 0 ? 0 : (i > 255 ? 255 : i));
}

__device__ __forceinline__ uint8_t rhe_u8(float v) {  // cvRound + saturate_cast<uchar>
  int i = __float2int_rn(v);
  return (uint8_t)(i < 0 ? 0 : (i > 255 ? 255 : i));
}

// cv2 INTER_CUBIC taps of destination index d (ssize -> dsize): source indices clamped to the border and the float32
// coefficients (A = -0.75), as k_resize_cubic_u8 (dibr_kernels.cu) and k_sr_tail_cubic (sr_kernels.cu) apply them
struct CubicTap {
  int o[4];
  float c[4];
};
__device__ __forceinline__ CubicTap cubic_tap(int d, int ssize, int dsize) {
  CubicTap t;
  const double scale = (double)ssize / (double)dsize;
  float fx = (float)(((double)d + 0.5) * scale - 0.5);
  float fl = floorf(fx);
  int sx = (int)fl;
  float x = fx - fl;
  const float A = -0.75f;
  float x1 = x + 1.0f, xm = 1.0f - x;
  t.c[0] = ((((A * x1) - (5.0f * A)) * x1) + (8.0f * A)) * x1 - (4.0f * A);
  t.c[1] = ((((A + 2.0f) * x) - (A + 3.0f)) * x) * x + 1.0f;
  t.c[2] = ((((A + 2.0f) * xm) - (A + 3.0f)) * xm) * xm + 1.0f;
  t.c[3] = ((1.0f - t.c[0]) - t.c[1]) - t.c[2];
#pragma unroll
  for (int k = 0; k < 4; ++k) t.o[k] = min(max(sx - 1 + k, 0), ssize - 1);
  return t;
}

// output pixel (x, y) of cv2.resize(u8 [h, w, ch] -> [oh, ow, ch], INTER_CUBIC): float32 bicubic, rows then columns,
// round half to even.  src rows are `pitch` bytes apart, so a crop of a larger image is resized in place.
__device__ __forceinline__ void resize_cubic_u8_px(const uint8_t* __restrict__ src, size_t pitch, int h, int w, int ch,
                                                   uint8_t* __restrict__ dst, int oh, int ow, int x, int y) {
  CubicTap tx = cubic_tap(x, w, ow), ty = cubic_tap(y, h, oh);
  for (int c = 0; c < ch; ++c) {
    float col[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {  // rows first: the value of column tx.o[k] at output row y
      const size_t xc = (size_t)tx.o[k] * ch + c;
      float v = (float)src[(size_t)ty.o[0] * pitch + xc] * ty.c[0];
      v = v + ((float)src[(size_t)ty.o[1] * pitch + xc] * ty.c[1]);
      v = v + ((float)src[(size_t)ty.o[2] * pitch + xc] * ty.c[2]);
      v = v + ((float)src[(size_t)ty.o[3] * pitch + xc] * ty.c[3]);
      col[k] = v;
    }
    float r = (((col[0] * tx.c[0]) + (col[1] * tx.c[1])) + (col[2] * tx.c[2])) + (col[3] * tx.c[3]);
    dst[((size_t)y * ow + x) * ch + c] = rhe_u8(r);
  }
}

__device__ __forceinline__ int reflect101(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * n - 2 - i;
  return i;
}

// apply_color_grade (core/render_3d.py:734-767) on one pixel
__device__ __forceinline__ void grade_px(float& r, float& g, float& b, float sat, float con, float bri) {
  float luma = ((0.2126f * r) + (0.7152f * g)) + (0.0722f * b);
  float c[3] = {r, g, b};
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    float s = luma + ((c[i] - luma) * sat);
    s = 0.5f + ((s - 0.5f) * con);
    s = s + bri;
    c[i] = clamp01(s);
  }
  r = c[0];
  g = c[1];
  b = c[2];
}

__device__ __forceinline__ float torch_lerp(float a, float b, float w) {
  float diff = b - a;
  return (fabsf(w) < 0.5f) ? (a + (w * diff)) : (b - (diff * (1.0f - w)));
}

// ---------------------------------------------------------------------------
// horizontal-parallax sampling set-up (F.grid_sample bilinear/border/align_corners=True)
// ---------------------------------------------------------------------------
struct Tap {
  int x0, x1, y0, y1;
  float nw, ne, sw, se;
};
__device__ __forceinline__ Tap make_tap(float gx, float gy, int H, int W) {
  Tap t;
  float ix = (gx + 1.0f) * ((float)(W - 1) / 2.0f);
  float iy = (gy + 1.0f) * ((float)(H - 1) / 2.0f);
  ix = fminf((float)(W - 1), fmaxf(ix, 0.f));
  iy = fminf((float)(H - 1), fmaxf(iy, 0.f));
  float fx = floorf(ix), fy = floorf(iy);
  float wx = ix - fx, ex = 1.0f - wx;
  float ny = iy - fy, sy = 1.0f - ny;
  t.x0 = (int)fx;
  t.y0 = (int)fy;
  t.x1 = min(t.x0 + 1, W - 1);
  t.y1 = min(t.y0 + 1, H - 1);
  t.nw = sy * ex;
  t.ne = sy * wx;
  t.sw = ny * ex;
  t.se = ny * wx;
  return t;
}
__device__ __forceinline__ float tap_apply(const Tap& t, float v00, float v01, float v10, float v11) {
  float o = v00 * t.nw;
  o = __fmaf_rn(v01, t.ne, o);
  o = __fmaf_rn(v10, t.sw, o);
  o = __fmaf_rn(v11, t.se, o);
  return o;
}
__device__ __forceinline__ float sample_plane(const float* __restrict__ p, int W, const Tap& t) {
  const float* r0 = p + (size_t)t.y0 * W;
  const float* r1 = p + (size_t)t.y1 * W;
  return tap_apply(t, r0[t.x0], r0[t.x1], r1[t.x0], r1[t.x1]);
}

// estimate_subject_depth (core/render_3d.py:145-172) from the histc bins + lower median of the kept pixels
__device__ __forceinline__ float subject_core(uint32_t n, const uint32_t* hist64, float med) {
  if (n < 20) return 0.5f;
  uint32_t best = 0;
  int peak = 0;
  for (int i = 0; i < 64; ++i) {
    uint32_t c = hist64[i];
    if (c > best) {
      best = c;
      peak = i;
    }
  }
  float subj = ((float)peak + 0.5f) * (1.0f / 64.0f);
  float v = (0.7f * subj) + (0.3f * med);
  return clamp01(v);
}

// DepthPercentileEMA.normalize state update (core/render_3d.py:249-262); v0..v3 = the order statistics
// floor/ceil(rank_lo), floor/ceil(rank_hi)
__device__ __forceinline__ void fin_pct_core(float v0, float v1, float v2, float v3, float w_lo, float w_hi, float alpha,
                                             float one_minus_alpha, DevState* st, FrameScalars* fs) {
  float lo = torch_lerp(v0, v1, w_lo);
  float hi = torch_lerp(v2, v3, w_hi);
  fs->q_lo = lo;
  fs->q_hi = hi;
  if ((hi - lo) < 1e-5f) {
    fs->pct_flat = 1;
    fs->n_lo = 0.f;
    fs->n_den = 1.f;
    return;
  }
  fs->pct_flat = 0;
  if (!st->pct_init) {
    st->pct_lo = lo;
    st->pct_hi = hi;
    st->pct_init = 1;
  } else {
    st->pct_lo = (alpha * st->pct_lo) + (one_minus_alpha * lo);
    st->pct_hi = (alpha * st->pct_hi) + (one_minus_alpha * hi);
  }
  fs->n_lo = st->pct_lo;
  fs->n_den = (st->pct_hi - st->pct_lo) + 1e-6f;
}

// ShiftSmoother, compute_dynamic_parallax_scale, FocalDepthTracker, motion metric, ConvergenceEMA,
// FloatingBarEaser (core/render_3d.py:412-427,463-511,895-929,1269-1276,1334-1403); sd = subject depth of the
// normalised plane; fs->sum / sumsq / mad_sum hold the centre-crop and motion sums
__device__ __forceinline__ void fin_norm_core(float sd, const LoopArgs& la, DevState* st, FrameScalars* fs) {
  st->tdf_init = 1;
  // dynamic parallax scale
  double n = (double)la.crop_count;
  double mean64 = fs->sum / n;
  float mean = (float)mean64;
  float var = (float)((fs->sumsq - fs->sum * mean64) / (n - 1.0));
  float nv = var / (mean + 1e-5f);
  nv = clamp01(nv);
  float scale = la.dyn_min + (nv * la.dyn_span);
  double dyn = (double)scale;
  fs->dyn = dyn;
  // ShiftSmoother(alpha=0.15)
  if (!st->sm_init) {
    st->sm_fg = la.fg;
    st->sm_mg = la.mg;
    st->sm_bg = la.bg;
    st->sm_init = 1;
  } else {
    st->sm_fg = 0.15 * la.fg + (1 - 0.15) * st->sm_fg;
    st->sm_mg = 0.15 * la.mg + (1 - 0.15) * st->sm_mg;
    st->sm_bg = 0.15 * la.bg + (1 - 0.15) * st->sm_bg;
  }
  double fg = st->sm_fg * dyn, mg = st->sm_mg * dyn, bg = st->sm_bg * dyn;
  if (la.ipd != 0.0) {
    fg *= la.ipd;
    mg *= la.ipd;
    bg *= la.ipd;
  }
  fs->fg = fg;
  fs->mg = mg;
  fs->bg = bg;
  // candidate focal / floating-window subject
  fs->subj_norm = sd;
  // motion metric
  double motion = 0.0;
  if (st->have_prev_depth) {
    float mad = (float)(fs->mad_sum / (double)la.npix);
    motion = fmax(0.0, fmin(1.0, (double)mad * 4.0));
  }
  fs->motion = motion;
  st->have_prev_depth = 1;
  // FocalDepthTracker
  st->focal_alpha = 0.10 + 0.20 * fmax(0.0, fmin(1.0, motion));
  double c = (double)sd;
  if (!st->focal_init) {
    st->focal = c;
    st->focal_init = 1;
  } else {
    if (fabs(c - st->focal) < 0.03) c = st->focal;
    double nf = (1.0 - st->focal_alpha) * st->focal + st->focal_alpha * c;
    double delta = nf - st->focal;
    if (delta > 0.02)
      nf = st->focal + 0.02;
    else if (delta < -0.02)
      nf = st->focal - 0.02;
    st->focal = fmax(0.0, fmin(1.0, nf));
  }
  fs->focal = st->focal;
  // floating-window bars
  float half = (float)((double)la.resized_width / 2 + 1e-6);
  float rz = (((-sd) * (float)fg) + ((-sd) * (float)mg)) + (sd * (float)bg);
  double raw_zero = (double)(rz / half);
  if (!st->conv_init) {
    st->conv_val = raw_zero;
    st->conv_init = 1;
  } else {
    st->conv_val = 0.97 * st->conv_val + (1 - 0.97) * raw_zero;
  }
  double stable = st->conv_val;
  fs->stable_zero = stable;
  int bar = 0, side = 0;
  if (la.use_floating_window && la.use_subject_tracking) {
    int raw_bar = (int)(fabs(stable) * la.resized_width * 0.75);
    st->bar_prev = (int)(0.85 * st->bar_prev + (1 - 0.85) * raw_bar);
    bar = max(min(st->bar_prev, 80), 0);
    if (stable > 0.005)
      side = 1;
    else if (stable < -0.005)
      side = 2;
  }
  fs->bar_width = bar;
  fs->bar_side = side;
}

// shape_depth_for_pop scalars (core/render_3d.py:534-553)
__device__ __forceinline__ void fin_d0_core(float subj, float v0, float v1, float v2, float v3, float w_lo, float w_hi,
                                            FrameScalars* fs) {
  fs->subj_raw = subj;
  float lo = torch_lerp(v0, v1, w_lo);
  float hi = torch_lerp(v2, v3, w_hi);
  fs->st_lo = lo;
  fs->st_hi = hi;
  subj = clamp01(subj);
  if ((hi - lo) < 1e-5f) {
    fs->st_flat = 1;
    fs->st_den = 1.f;
    fs->st_subj = subj;
  } else {
    fs->st_flat = 0;
    float den = (hi - lo) + 1e-6f;
    fs->st_den = den;
    fs->st_subj = clamp01((subj - lo) / den);
  }
}

// zero-parallax offset, FloatingWindowTracker, clamp, convergence, mask strength (core/render_3d.py:633-678)
__device__ __forceinline__ void fin_shape_core(float subj, const ShiftArgs& sa, DevState* st, FrameScalars* fs) {
  fs->subj = subj;
  const vd3d_shift_params& p = sa.p;
  float fg = (float)fs->fg, mg = (float)fs->mg, bg = (float)fs->bg;
  float fgm = (float)p.fg_pop_multiplier, bgm = (float)p.bg_push_multiplier;
  float pb = (float)p.parallax_balance;
  double half = (double)sa.W / 2.0;
  fs->c_fg = fg;
  fs->c_mg = mg;
  fs->c_bg = bg;
  fs->c_fgm = fgm;
  fs->c_bgm = bgm;
  fs->c_pb = pb;
  fs->c_half = (float)half;
  fs->c_mid = (float)p.depth_pop_mid;
  fs->c_gamma = (float)p.depth_pop_gamma;
  double zpo = 0.0;
  fs->use_zpo = p.use_subject_tracking ? 1 : 0;
  if (p.use_subject_tracking) {
    float a = subj * pb;
    float t1 = ((-a) * fg) * fgm;
    float t2 = (-a) * mg;
    float t3 = (a * bg) * bgm;
    float z = ((t1 + t2) + t3) / (float)half;
    z = z * (float)p.subject_lock_strength;
    z = z - (float)p.zero_parallax_strength;
    if (p.enable_floating_window) {
      float sw = fminf(fmaxf(1.0f - (subj * 2.0f), 0.5f), 1.0f);
      z = z * sw;
      z = fminf(fmaxf(z, -0.35f), 0.35f);
      double cur = (double)z;
      // FloatingWindowTracker.smooth_offset(threshold=0.0015), alpha=0.97
      if (fabs(cur - st->fw_prev) < 0.0015) {
        zpo = st->fw_prev;
      } else {
        st->fw_prev = 0.97 * st->fw_prev + (1 - 0.97) * cur;
        st->fw_count += 1;
        if (st->fw_count >= 100) {
          st->fw_prev = fmax(fmin(st->fw_prev, 1.0), -1.0);
          st->fw_count = 0;
        }
        zpo = st->fw_prev;
      }
    } else {
      zpo = (double)z;
    }
  }
  fs->zpo = zpo;
  fs->c_zpo = (float)zpo;
  fs->c_max = (float)(((double)sa.W * p.max_pixel_shift_percent) / half);
  fs->use_conv = (p.convergence_strength != 0.0) ? 1 : 0;
  fs->c_conv = 0.f;
  if (fs->use_conv) {
    double conv = p.enable_dynamic_convergence ? (double)(subj * (float)p.convergence_strength)
                                               : p.convergence_strength;
    fs->c_conv = (float)(conv / half);
  }
  double ms = fmin(fmax(p.feather_strength / 10.0, 0.05), 0.3);
  fs->c_m1 = (float)(1.0 - ms);
  fs->c_m2 = (float)ms;
}

}  // namespace vd3d
