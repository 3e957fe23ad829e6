// dibr_kernels.cu -- see dibr_kernels.cuh.  Compiled with -fmad=false.
#include "dibr_device.cuh"
#include "dibr_launch.h"

#include <math.h>

namespace vd3d {


// ---------------------------------------------------------------------------
// K1 ingest: depth_to_tensor + aspect crop + resize + TemporalDepthFilter (alpha .5)
//            (+ frame_to_tensor + resize of RGB when a resize is needed)
// core/render_3d.py:135-143, 220-229, 1236-1266
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_ingest(IngestArgs a) {
  int x = blockIdx.x * 32 + (threadIdx.x & 31);
  int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.tw || y >= a.th) return;
  int cx0 = a.cx0, cy0 = a.cy0, cw = a.cw, ch = a.ch;
  if (a.bars) {  // auto_crop_black_bars: this frame's rectangle from the words of k_black_bars
    int rect[4], top, bottom;
    black_bar_crop(a.src_w, a.src_h, a.bars[0], a.bars[1], a.aspect, rect, &top, &bottom);
    cx0 = rect[0];
    cy0 = rect[1];
    cw = rect[2];
    ch = rect[3];
    if (x == 0 && y == 0 && a.crop_out) {
      a.crop_out[0] = top;
      a.crop_out[1] = bottom;
    }
  }
  float cur;
  RsAxis ax, ay;
  bool fast = (a.tw == cw && a.th == ch) && !a.rgb_s;
  if (fast) {
    cur = depth_src01(a.depth, a.depth_ch, a.src_w, cy0 + y, cx0 + x);
  } else {  // same-size axes degenerate to i0 = d, l1 = 0: an exact identity
    ax = rs_axis(x, cw, a.tw);
    ay = rs_axis(y, ch, a.th);
    float v00 = depth_src01(a.depth, a.depth_ch, a.src_w, cy0 + ay.i0, cx0 + ax.i0);
    float v01 = depth_src01(a.depth, a.depth_ch, a.src_w, cy0 + ay.i0, cx0 + ax.i1);
    float v10 = depth_src01(a.depth, a.depth_ch, a.src_w, cy0 + ay.i1, cx0 + ax.i0);
    float v11 = depth_src01(a.depth, a.depth_ch, a.src_w, cy0 + ay.i1, cx0 + ax.i1);
    cur = rs_combine(v00, v01, v10, v11, ax, ay);
  }
  size_t o = (size_t)y * a.tw + x;
  float prev = a.st->tdf_init ? a.tdf[o] : cur;
  float nv = (a.alpha * prev) + (a.one_minus_alpha * cur);
  a.tdf[o] = nv;
  if (a.rgb_s) {  // resized RGB planes
    size_t plane = (size_t)a.th * a.tw;
#pragma unroll
    for (int c = 0; c < 3; ++c) {  // c: 0=R 1=G 2=B ; source is BGR
      int sc = 2 - c;
      const uint8_t* f = a.frame + sc;
      float v00 = (float)f[((size_t)(cy0 + ay.i0) * a.src_w + cx0 + ax.i0) * 3] / 255.0f;
      float v01 = (float)f[((size_t)(cy0 + ay.i0) * a.src_w + cx0 + ax.i1) * 3] / 255.0f;
      float v10 = (float)f[((size_t)(cy0 + ay.i1) * a.src_w + cx0 + ax.i0) * 3] / 255.0f;
      float v11 = (float)f[((size_t)(cy0 + ay.i1) * a.src_w + cx0 + ax.i1) * 3] / 255.0f;
      a.rgb_s[c * plane + o] = rs_combine(v00, v01, v10, v11, ax, ay);
    }
  }
}

// ---------------------------------------------------------------------------
// detect_black_bars (core/render_3d.py:293-316): one warp per row of the u8 BGR frame.  The row sum of cv2 BGR2GRAY is
// an exact integer, and np.mean(gray[y]) > threshold  <=>  sum > threshold * w.  Rows whose start is 16-byte aligned
// (w % 16 == 0 on an aligned frame) are read 48 bytes = 16 pixels per lane and step; others one pixel at a time.
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t gray_u8(uint32_t b, uint32_t g, uint32_t r) {
  return (b * 3735u + g * 19235u + r * 9798u + (1u << 14)) >> 15;
}

__global__ void __launch_bounds__(256) k_black_bars(const uint8_t* __restrict__ frame, int h, int w, int threshold,
                                                    uint32_t* __restrict__ words) {
  __shared__ uint32_t s_first, s_last;
  const int lane = threadIdx.x & 31;
  const int y = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (threadIdx.x == 0) s_first = s_last = 0u;
  __syncthreads();
  if (y < h) {
    const uint8_t* row = frame + (size_t)y * w * 3;
    uint32_t sum = 0;
    int x0 = 0;
    if (((uintptr_t)row & 15) == 0) {
      const int chunks = w / 16;
      const uint4* v = reinterpret_cast<const uint4*>(row);
      for (int c = lane; c < chunks; c += 32) {
        uint4 q[3];
        q[0] = __ldg(v + 3 * c);
        q[1] = __ldg(v + 3 * c + 1);
        q[2] = __ldg(v + 3 * c + 2);
        const uint8_t* p = reinterpret_cast<const uint8_t*>(q);
#pragma unroll
        for (int k = 0; k < 16; ++k) sum += gray_u8(p[3 * k], p[3 * k + 1], p[3 * k + 2]);
      }
      x0 = chunks * 16;
    }
    for (int x = x0 + lane; x < w; x += 32) sum += gray_u8(row[3 * x], row[3 * x + 1], row[3 * x + 2]);
    sum = __reduce_add_sync(0xffffffffu, sum);
    if (lane == 0 && sum > (uint32_t)threshold * (uint32_t)w) {
      atomicMax(&s_first, (uint32_t)(h - y));
      atomicMax(&s_last, (uint32_t)(y + 1));
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_first) {
    atomicMax(words, s_first);
    atomicMax(words + 1, s_last);
  }
}

// generic planar f32 resize [C,sh,sw] -> [C,oh,ow] (pixel_shift_cuda:595-596)
__global__ void __launch_bounds__(256) k_resize_planar(const float* __restrict__ src, int C, int sh, int sw,
                                                       float* __restrict__ dst, int oh, int ow) {
  int x = blockIdx.x * 32 + (threadIdx.x & 31);
  int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= ow || y >= oh) return;
  for (int c = 0; c < C; ++c)
    dst[((size_t)c * oh + y) * ow + x] = bilinear_f32(src + (size_t)c * sh * sw, sh, sw, oh, ow, y, x);
}

// ---------------------------------------------------------------------------
// radix select: exact k-th order statistics on fp32 in [0,1] (bit pattern is
// monotone for non-negative floats).  pass 1: bits[29:18], pass 2: bits[17:6],
// pass 3: bits[5:0].  Replaces torch.quantile's sort (core/render_3d.py:249-250,
// 536-537) and torch.median / torch.histc (157-170).
// ---------------------------------------------------------------------------
__device__ __forceinline__ void warp_hist_add(uint32_t* hist, bool on, uint32_t bin, bool shared) {
  unsigned act = __activemask();
  if (!__any_sync(act, on)) return;
  unsigned key = on ? bin : 0xFFFFFFFFu;
  unsigned m = __match_any_sync(act, key);
  if (on && (int)(threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(&hist[bin], (uint32_t)__popc(m));
  (void)shared;
}

__device__ __forceinline__ bool in_job(const SelJob& j, int y, int x, float v) {
  if (y < j.y0 || y >= j.y1 || x < j.x0 || x >= j.x1) return false;
  if (j.masked) return (v > 0.05f) && (v < 0.95f);
  return true;
}

template <int PASS>
__global__ void __launch_bounds__(256) k_sel_pass(SelJob a, SelJob b, int nb) {
  __shared__ uint32_t sh[2][4096];
  __shared__ uint32_t sh64[2][64];
  if (PASS == 1) {
    for (int i = threadIdx.x; i < 4096; i += 256) {
      sh[0][i] = 0;
      sh[1][i] = 0;
    }
    if (threadIdx.x < 64) {
      sh64[0][threadIdx.x] = 0;
      sh64[1][threadIdx.x] = 0;
    }
    __syncthreads();
  }
  const int rw = a.x1 - a.x0;
  const int rw_pad = (rw + 31) & ~31;
  for (int y = a.y0 + blockIdx.x; y < a.y1; y += gridDim.x) {
    const float* row = a.data + (size_t)y * a.W;
    for (int xi = threadIdx.x; xi < rw_pad; xi += 256) {
      int x = a.x0 + xi;
      bool inb = xi < rw;
      float v = inb ? clamp01(row[x]) : 0.f;
      uint32_t key = __float_as_uint(v) & 0x7FFFFFFFu;
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        if (jj == 1 && !nb) break;
        const SelJob& j = jj ? b : a;
        bool on = inb && in_job(j, y, x, v);
        if (PASS == 1) {
          warp_hist_add(sh[jj], on, key >> 18, true);
          if (j.hist64) {
            int b64 = (int)(v * 64.0f);
            b64 = b64 > 63 ? 63 : b64;
            warp_hist_add(sh64[jj], on, (uint32_t)b64, true);
          }
        } else {
          for (int t = 0; t < j.ntargets; ++t) {
            const SelTarget& tg = j.tg[t];
            if (PASS == 2) {
              if (tg.alias >= 0) continue;
              bool m = on && ((key >> 18) == tg.p1);
              warp_hist_add(j.hist2 + t * 4096, m, (key >> 6) & 4095u, false);
            } else {
              if (tg.alias2 >= 0) continue;
              bool m = on && ((key >> 18) == tg.p1) && (((key >> 6) & 4095u) == tg.p2);
              warp_hist_add(j.hist3 + t * 64, m, key & 63u, false);
            }
          }
        }
      }
    }
  }
  if (PASS == 1) {
    __syncthreads();
    for (int i = threadIdx.x; i < 4096; i += 256) {
      if (sh[0][i]) atomicAdd(&a.hist1[i], sh[0][i]);
      if (nb && sh[1][i]) atomicAdd(&b.hist1[i], sh[1][i]);
    }
    if (threadIdx.x < 64) {
      if (a.hist64 && sh64[0][threadIdx.x]) atomicAdd(&a.hist64[threadIdx.x], sh64[0][threadIdx.x]);
      if (nb && b.hist64 && sh64[1][threadIdx.x]) atomicAdd(&b.hist64[threadIdx.x], sh64[1][threadIdx.x]);
    }
  }
}

// one block per job: find, for every target, the bin holding its rank
template <int PASS>
__global__ void __launch_bounds__(1024) k_sel_find(SelJob a, SelJob b) {
  const SelJob& j = blockIdx.x ? b : a;
  constexpr int NB = (PASS == 3) ? 64 : 4096;
  __shared__ uint32_t cum[4096];
  __shared__ uint32_t part[1024];
  const int tid = threadIdx.x;
  for (int t = 0; t < j.ntargets; ++t) {
    SelTarget& tg = j.tg[t];
    const uint32_t* hist;
    uint32_t rank;
    if (PASS == 1) {
      if (t > 0) break;  // pass-1 histogram is shared: handled below for all targets at once
      hist = j.hist1;
      rank = 0;
    } else if (PASS == 2) {
      if (tg.alias >= 0) continue;
      hist = j.hist2 + t * 4096;
      rank = tg.r1;
    } else {
      if (tg.alias2 >= 0) continue;
      hist = j.hist3 + t * 64;
      rank = tg.r2;
    }
    // inclusive scan of hist into cum
    constexpr int PER = NB / 1024 > 0 ? NB / 1024 : 1;
    uint32_t loc[PER];
    uint32_t s = 0;
    for (int k = 0; k < PER; ++k) {
      int i = tid * PER + k;
      uint32_t v = (i < NB) ? hist[i] : 0u;
      s += v;
      loc[k] = s;
    }
    part[tid] = s;
    __syncthreads();
    for (int off = 1; off < 1024; off <<= 1) {
      uint32_t v = (tid >= off) ? part[tid - off] : 0u;
      __syncthreads();
      part[tid] += v;
      __syncthreads();
    }
    uint32_t base = tid ? part[tid - 1] : 0u;
    for (int k = 0; k < PER; ++k) {
      int i = tid * PER + k;
      if (i < NB) cum[i] = base + loc[k];
    }
    __syncthreads();
    if (PASS == 1) {
      uint32_t n = cum[NB - 1];
      if (tid == 0) *j.count = n;
      // all targets search the shared histogram
      for (int tt = 0; tt < j.ntargets; ++tt) {
        uint32_t r = j.tg[tt].rank;
        if (j.rank_from_count && tt == 0) r = n ? (n - 1) / 2 : 0;
        for (int k = 0; k < PER; ++k) {
          int i = tid * PER + k;
          uint32_t lo = i ? cum[i - 1] : 0u;
          if (r >= lo && r < cum[i]) {
            j.tg[tt].p1 = i;
            j.tg[tt].r1 = r - lo;
            if (j.rank_from_count && tt == 0) j.tg[tt].rank = r;
          }
        }
      }
      __syncthreads();
      if (tid == 0) {
        for (int tt = 0; tt < j.ntargets; ++tt) {
          j.tg[tt].alias = -1;
          for (int u = 0; u < tt; ++u)
            if (j.tg[u].p1 == j.tg[tt].p1 && j.tg[u].alias < 0) {
              j.tg[tt].alias = u;
              break;
            }
        }
      }
    } else {
      // this histogram may serve several aliased targets
      for (int tt = t; tt < j.ntargets; ++tt) {
        SelTarget& g = j.tg[tt];
        bool mine = (tt == t) || (PASS == 2 ? g.alias == t : g.alias2 == t);
        if (!mine) continue;
        uint32_t r = (PASS == 2) ? g.r1 : g.r2;
        for (int k = 0; k < PER; ++k) {
          int i = tid * PER + k;
          if (i >= NB) continue;
          uint32_t lo = i ? cum[i - 1] : 0u;
          if (r >= lo && r < cum[i]) {
            if (PASS == 2) {
              g.p2 = i;
              g.r2 = r - lo;
            } else {
              g.bits = (g.p1 << 18) | (g.p2 << 6) | (uint32_t)i;
            }
          }
        }
      }
      __syncthreads();
    }
    (void)rank;
  }
  if (PASS == 2) {
    __syncthreads();
    if (tid == 0) {
      for (int tt = 0; tt < j.ntargets; ++tt) {
        j.tg[tt].alias2 = -1;
        for (int u = 0; u < tt; ++u)
          if (j.tg[u].p1 == j.tg[tt].p1 && j.tg[u].p2 == j.tg[tt].p2 && j.tg[u].alias2 < 0) {
            j.tg[tt].alias2 = u;
            break;
          }
      }
    }
  }
}


__device__ float subject_from_job(const SelJob& j) {
  return subject_core(*j.count, j.hist64, __uint_as_float(j.tg[0].bits));
}

// ---------------------------------------------------------------------------
// scalar kernels (one thread): the reference's Python-side control flow
// ---------------------------------------------------------------------------
// DepthPercentileEMA.normalize state update (core/render_3d.py:249-262)
__global__ void k_fin_pct(SelJob j, float w_lo, float w_hi, float alpha, float one_minus_alpha, DevState* st,
                          FrameScalars* fs) {
  fin_pct_core(__uint_as_float(j.tg[0].bits), __uint_as_float(j.tg[1].bits), __uint_as_float(j.tg[2].bits),
               __uint_as_float(j.tg[3].bits), w_lo, w_hi, alpha, one_minus_alpha, st, fs);
}

// ShiftSmoother, compute_dynamic_parallax_scale, FocalDepthTracker, motion metric,
// ConvergenceEMA, FloatingBarEaser (core/render_3d.py:412-427,463-511,895-929,1269-1276,1334-1403)
__global__ void k_fin_norm(SelJob subj_job, LoopArgs la, DevState* st, FrameScalars* fs) {
  fin_norm_core(subject_from_job(subj_job), la, st, fs);
}

__global__ void k_set_ranks(SelTarget* tg, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  tg[0].rank = r0;
  tg[1].rank = r1;
  tg[2].rank = r2;
  tg[3].rank = r3;
}

__global__ void k_set_shifts(FrameScalars* fs, double fg, double mg, double bg) {
  fs->fg = fg;
  fs->mg = mg;
  fs->bg = bg;
}

// shape_depth_for_pop scalars (core/render_3d.py:534-553)
__global__ void k_fin_d0(SelJob qjob, SelJob sjob, float w_lo, float w_hi, FrameScalars* fs) {
  fin_d0_core(subject_from_job(sjob), __uint_as_float(qjob.tg[0].bits), __uint_as_float(qjob.tg[1].bits),
              __uint_as_float(qjob.tg[2].bits), __uint_as_float(qjob.tg[3].bits), w_lo, w_hi, fs);
}

// zero-parallax offset, FloatingWindowTracker, clamp, convergence, mask strength
// (core/render_3d.py:633-678)
__global__ void k_fin_shape(SelJob sjob, ShiftArgs sa, DevState* st, FrameScalars* fs) {
  fin_shape_core(subject_from_job(sjob), sa, st, fs);
}

// ---------------------------------------------------------------------------
// K2 normalise + centre statistics + motion (core/render_3d.py:247,261-262,418-423,928)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_normalize(const float* __restrict__ tdf, float* __restrict__ dn,
                                                   const float* __restrict__ dn_prev, int th, int tw,
                                                   const DevState* st, FrameScalars* fs) {
  __shared__ double red[3][8];
  int x = blockIdx.x * 32 + (threadIdx.x & 31);
  int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  double s = 0, s2 = 0, mad = 0;
  if (x < tw && y < th) {
    size_t o = (size_t)y * tw + x;
    float d = clamp01(tdf[o]);
    float v = fs->pct_flat ? d : clamp01((d - fs->n_lo) / fs->n_den);
    dn[o] = v;
    if (y >= th / 4 && y < th * 3 / 4 && x >= tw / 4 && x < tw * 3 / 4) {
      s = (double)v;
      s2 = (double)v * (double)v;
    }
    if (st->have_prev_depth) mad = (double)fabsf(v - dn_prev[o]);
  }
  for (int off = 16; off; off >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, off);
    s2 += __shfl_xor_sync(0xffffffffu, s2, off);
    mad += __shfl_xor_sync(0xffffffffu, mad, off);
  }
  int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    red[0][w] = s;
    red[1][w] = s2;
    red[2][w] = mad;
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    double t = 0;
    for (int i = 0; i < 8; ++i) t += red[threadIdx.x][i];
    double* dst = threadIdx.x == 0 ? &fs->sum : (threadIdx.x == 1 ? &fs->sumsq : &fs->mad_sum);
    if (t != 0.0) atomicAdd(dst, t);
  }
}

// ---------------------------------------------------------------------------
// K3 d0 = clamp01(enhance_curvature(resize(depth))) (core/render_3d.py:596-601)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_d0(const float* __restrict__ src, int sh, int sw, float* __restrict__ d0,
                                            int H, int W, const float* __restrict__ xs,
                                            const float* __restrict__ ys, float strength) {
  int x = blockIdx.x * 32 + (threadIdx.x & 31);
  int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= W || y >= H) return;
  float d = bilinear_f32(src, sh, sw, H, W, y, x);
  float xx = xs[x], yy = ys[y];
  float r2 = (xx * xx) + (yy * yy);
  float curv = 1.0f - r2;
  d = d + (curv * strength);
  d0[(size_t)y * W + x] = clamp01(d);
}

// K4 shape_depth_for_pop elementwise part (core/render_3d.py:542,555-558), in place
__global__ void __launch_bounds__(256) k_shape(float* __restrict__ d, int n, const FrameScalars* fs, float mid,
                                               float gamma) {
  int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  float v = d[i];  // already clamped
  float ds = fs->st_flat ? v : clamp01((v - fs->st_lo) / fs->st_den);
  float centered = (ds - fs->st_subj) + mid;
  float x = centered - mid;
  float ax = fabsf(x);
  // |x|^gamma, correctly rounded (fp64 pow then one rounding) so that the CUDA path and the
  // oracle agree bit for bit; torch's Sleef powf is within 1 ulp of the same value
  float pw = (float)pow((double)ax, (double)gamma);
  float sg = (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f);
  d[i] = clamp01((sg * pw) + mid);
}

// ---------------------------------------------------------------------------
// K5 shift map + suppress_artifacts_with_edge_mask (core/render_3d.py:198-216,620-680)
// ---------------------------------------------------------------------------
// FAST: fp32 SFU exp / sqrt instead of the correctly rounded fp64 forms (<= 2e-7 on the mask and the fg weight)
template <bool FAST>
__global__ void __launch_bounds__(256) k_shift(const float* __restrict__ d, float* __restrict__ shift, int H, int W,
                                               const FrameScalars* fs, int edge_mask, float feather) {
  __shared__ float sd[13][38];   // d over x in [bx-3, bx+34), y in [by-3, by+10)
  __shared__ float sm[12][36];   // 1 - sigmoid(...) over x in [bx-2, bx+34), y in [by-2, by+10)
  const int bx = blockIdx.x * 32, by = blockIdx.y * 8;
  const int tid = threadIdx.x;
  if (edge_mask) {
    for (int i = tid; i < 13 * 37; i += 256) {
      int ty = i / 37, tx = i % 37;
      int gy = by - 3 + ty, gx = bx - 3 + tx;
      float v = 0.f;
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = d[(size_t)gy * W + gx];
      sd[ty][tx] = v;
    }
    __syncthreads();
    for (int i = tid; i < 12 * 36; i += 256) {
      int ty = i / 36, tx = i % 36;
      int gy = by - 2 + ty, gx = bx - 2 + tx;
      float m = 0.f;  // zero padding of avg_pool2d
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
        float c = sd[ty + 1][tx + 1];
        float dx = (gx > 0) ? fabsf(c - sd[ty + 1][tx]) : 0.f;
        float dy = (gy > 0) ? fabsf(c - sd[ty][tx + 1]) : 0.f;
        float g = sqrtf((dx * dx) + (dy * dy));
        float z = ((g - 0.02f) * feather) * 5.0f;
        float e = FAST ? (1.0f / (1.0f + __expf(-z)))
                       : (1.0f / (1.0f + (float)exp((double)(-z))));  // exp correctly rounded via fp64
        m = 1.0f - e;
      }
      sm[ty][tx] = m;
    }
    __syncthreads();
  }
  int lx = tid & 31, ly = tid >> 5;
  int x = bx + lx, y = by + ly;
  if (x >= W || y >= H) return;
  float v = edge_mask ? sd[ly + 3][lx + 3] : d[(size_t)y * W + x];
  float fgw;
  if (FAST) {
    float o1 = 1.0f - v;
    fgw = clamp01(o1 * sqrtf(o1));
  } else {
    double omv = (double)(1.0f - v);
    fgw = clamp01((float)(omv * sqrt(omv)));  // (1-d)^1.5, correctly rounded via fp64
  }
  float mgw = clamp01(1.0f - (fabsf(v - fs->c_mid) * 3.0f));
  float bgw = clamp01(v);
  float raw = (((fgw * fs->c_fg) * fs->c_fgm) + (mgw * fs->c_mg)) + ((bgw * fs->c_bg) * fs->c_bgm);
  float total = (raw * fs->c_pb) / fs->c_half;
  if (fs->use_zpo) total = total - fs->c_zpo;
  total = fminf(fmaxf(total, -fs->c_max), fs->c_max);
  if (fs->use_conv) total = total - fs->c_conv;
  float fin = total;
  if (edge_mask) {
    float acc = 0.f;
#pragma unroll
    for (int dy = 0; dy < 5; ++dy)
#pragma unroll
      for (int dx = 0; dx < 5; ++dx) acc = acc + sm[ly + dy][lx + dx];
    float smooth = acc / 25.0f;
    float sup = total * smooth;
    fin = (fs->c_m1 * total) + (fs->c_m2 * sup);
  }
  shift[(size_t)y * W + x] = fin;
}


// K6 warped depth (both eyes) -> feather edge mask clamp(|grad| * strength)
// (core/render_3d.py:700-701, 347-352).  e2[y][x] = (left, right)
__global__ void __launch_bounds__(256) k_warp_edges(const float* __restrict__ d, const float* __restrict__ shift,
                                                    float2* __restrict__ e2, int H, int W,
                                                    const float* __restrict__ xs, const float* __restrict__ ys,
                                                    float feather) {
  __shared__ float wl[9][33], wr[9][33];
  const int bx = blockIdx.x * 32, by = blockIdx.y * 8;
  for (int i = threadIdx.x; i < 9 * 33; i += 256) {
    int ty = i / 33, tx = i % 33;
    int gy = by - 1 + ty, gx = bx - 1 + tx;
    float a = 0.f, b = 0.f;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
      float sv = shift[(size_t)gy * W + gx];
      float xv = xs[gx], yv = ys[gy];
      Tap tl = make_tap(xv + sv, yv, H, W);
      Tap tr = make_tap(xv - sv, yv, H, W);
      a = sample_plane(d, W, tl);
      b = sample_plane(d, W, tr);
    }
    wl[ty][tx] = a;
    wr[ty][tx] = b;
  }
  __syncthreads();
  int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
  int x = bx + lx, y = by + ly;
  if (x >= W || y >= H) return;
  float2 o;
  {
    float c = wl[ly + 1][lx + 1];
    float dx = (x > 0) ? (c - wl[ly + 1][lx]) : 0.f;
    float dy = (y > 0) ? (c - wl[ly][lx + 1]) : 0.f;
    float g = sqrtf((dx * dx) + (dy * dy));
    o.x = clamp01(g * feather);
  }
  {
    float c = wr[ly + 1][lx + 1];
    float dx = (x > 0) ? (c - wr[ly + 1][lx]) : 0.f;
    float dy = (y > 0) ? (c - wr[ly][lx + 1]) : 0.f;
    float g = sqrtf((dx * dx) + (dy * dy));
    o.y = clamp01(g * feather);
  }
  e2[(size_t)y * W + x] = o;
}

// ---------------------------------------------------------------------------
// K7 compose: warp RGB (both eyes), feather blend, truncate to u8, optional colour grade
// (core/render_3d.py:697-698, 355-374, 289-291, 1373-1386)
// SRC_U8: sample the BGR u8 frame directly (identity-resize path) else f32 RGB planes
// ---------------------------------------------------------------------------
// lut[i] == (float)i / 255.0f (built per block): the IEEE division costs ~10 instructions and a
// pixel needs 27 of them; the table gives the identical bits with one shared-memory load.
template <bool SRC_U8>
__device__ __forceinline__ void fetch_rgb(const ComposeArgs& a, const float* lut, int y, int x, float* rgb) {
  if (SRC_U8) {
    const uint8_t* q = a.src_u8 + ((size_t)(a.cy0 + y) * a.src_pitch + a.cx0 + x) * 3;
    rgb[0] = lut[q[2]];
    rgb[1] = lut[q[1]];
    rgb[2] = lut[q[0]];
  } else {
    size_t plane = (size_t)a.H * a.W;
    size_t o = (size_t)y * a.W + x;
    rgb[0] = a.src_f32[o];
    rgb[1] = a.src_f32[plane + o];
    rgb[2] = a.src_f32[2 * plane + o];
  }
}

template <bool SRC_U8>
__global__ void __launch_bounds__(256) k_compose(ComposeArgs a) {
  extern __shared__ float2 tile[];  // (32+k-1) x (8+k-1)
  __shared__ float lut[256];
  lut[threadIdx.x] = (float)threadIdx.x / 255.0f;
  if (!a.feather) __syncthreads();
  const int k = a.feather ? a.k : 1;
  const int p = k / 2;
  const int tw = 32 + k - 1, th = 8 + k - 1;
  const int bx = blockIdx.x * 32, by = blockIdx.y * 8;
  const int H = a.H, W = a.W;
  if (a.feather) {
    for (int i = threadIdx.x; i < tw * th; i += 256) {
      int ty = i / tw, tx = i % tw;
      int gy = by - p + ty, gx = bx - p + tx;
      float2 v = make_float2(0.f, 0.f);
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = a.e2[(size_t)gy * W + gx];
      tile[i] = v;
    }
    __syncthreads();
  }
  int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
  int x = bx + lx, y = by + ly;
  if (x >= W || y >= H) return;
  float sv = a.shift[(size_t)y * W + x];
  float xv = a.xs[x], yv = a.ys[y];
  Tap tl = make_tap(xv + sv, yv, H, W);
  Tap tr = make_tap(xv - sv, yv, H, W);
  float bl = 0.f, br = 0.f;
  if (a.feather) {
    float al = 0.f, ar = 0.f;
    for (int dy = 0; dy < k; ++dy) {
      const float2* row = tile + (ly + dy) * tw + lx;
      for (int dx = 0; dx < k; ++dx) {
        float2 v = row[dx];
        al = al + v.x;
        ar = ar + v.y;
      }
    }
    float kk = (float)(k * k);
    bl = al / kk;
    br = ar / kk;
  }
  float o[3];
  fetch_rgb<SRC_U8>(a, lut, y, x, o);
  float l00[3], l01[3], l10[3], l11[3];
  uint8_t outl[3], outr[3];
#pragma unroll
  for (int eye = 0; eye < 2; ++eye) {
    const Tap& t = eye ? tr : tl;
    float b = eye ? br : bl;
    fetch_rgb<SRC_U8>(a, lut, t.y0, t.x0, l00);
    fetch_rgb<SRC_U8>(a, lut, t.y0, t.x1, l01);
    fetch_rgb<SRC_U8>(a, lut, t.y1, t.x0, l10);
    fetch_rgb<SRC_U8>(a, lut, t.y1, t.x1, l11);
    float c[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      float s = tap_apply(t, l00[ch], l01[ch], l10[ch], l11[ch]);
      if (a.feather) s = clamp01((s * (1.0f - b)) + (o[ch] * b));
      c[ch] = s;
    }
    uint8_t* dst = eye ? outr : outl;
    uint8_t r8 = trunc_u8(c[0]), g8 = trunc_u8(c[1]), b8 = trunc_u8(c[2]);
    if (a.grade) {  // frame_to_tensor -> apply_color_grade -> tensor_to_frame
      float r = lut[r8], g = lut[g8], bb = lut[b8];
      grade_px(r, g, bb, a.sat, a.con, a.bri);
      r8 = trunc_u8(r);
      g8 = trunc_u8(g);
      b8 = trunc_u8(bb);
    }
    dst[0] = b8;
    dst[1] = g8;
    dst[2] = r8;
  }
  size_t oo = ((size_t)y * W + x) * 3;
  a.left[oo] = outl[0];
  a.left[oo + 1] = outl[1];
  a.left[oo + 2] = outl[2];
  a.right[oo] = outr[0];
  a.right[oo + 1] = outr[1];
  a.right[oo + 2] = outr[2];
}

// Register-tiled variant for the common odd pool sizes: 4 horizontally adjacent outputs per
// thread share one row segment of the mask tile (6 LDS.128 per row for K = 9 instead of 36 LDS.64),
// K is a compile-time constant (fully unrolled), and each output still accumulates its K x K taps
// in the reference's row-major order, so results are bit-identical to k_compose.
template <bool SRC_U8, int K>
__global__ void __launch_bounds__(256) k_compose4(ComposeArgs a) {
  extern __shared__ float2 tile[];
  __shared__ float lut[256];
  lut[threadIdx.x] = (float)threadIdx.x / 255.0f;
  constexpr int P = K / 2;
  constexpr int TW = 128 + K - 1 + ((128 + K - 1) & 1);  // even row pitch (float2) for 16-byte loads
  constexpr int TH = 8 + K - 1;
  constexpr int NV = 4 + K - 1 + ((4 + K - 1) & 1);
  const int bx = blockIdx.x * 128, by = blockIdx.y * 8;
  const int H = a.H, W = a.W;
  for (int i = threadIdx.x; i < TW * TH; i += 256) {
    int ty = i / TW, tx = i % TW;
    int gy = by - P + ty, gx = bx - P + tx;
    float2 v = make_float2(0.f, 0.f);
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = a.e2[(size_t)gy * W + gx];
    tile[i] = v;
  }
  __syncthreads();
  const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
  const int x0 = bx + lx * 4, y = by + ly;
  if (x0 >= W || y >= H) return;
  float al[4] = {0.f, 0.f, 0.f, 0.f}, ar[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int dy = 0; dy < K; ++dy) {
    const float4* row = (const float4*)(tile + (ly + dy) * TW + lx * 4);
    float2 v[NV];
#pragma unroll
    for (int j = 0; j < NV / 2; ++j) {
      float4 f = row[j];
      v[2 * j] = make_float2(f.x, f.y);
      v[2 * j + 1] = make_float2(f.z, f.w);
    }
#pragma unroll
    for (int o = 0; o < 4; ++o)
#pragma unroll
      for (int dx = 0; dx < K; ++dx) {
        al[o] = al[o] + v[o + dx].x;
        ar[o] = ar[o] + v[o + dx].y;
      }
  }
  const float kk = (float)(K * K);
  const float yv = a.ys[y];
  uint8_t ol[12], orr[12];
  int nvalid = min(4, W - x0);
  for (int i = 0; i < nvalid; ++i) {
    const int x = x0 + i;
    float sv = a.shift[(size_t)y * W + x];
    float xv = a.xs[x];
    Tap tl = make_tap(xv + sv, yv, H, W);
    Tap tr = make_tap(xv - sv, yv, H, W);
    float bl = al[i] / kk, br = ar[i] / kk;
    float o[3];
    fetch_rgb<SRC_U8>(a, lut, y, x, o);
    float l00[3], l01[3], l10[3], l11[3];
#pragma unroll
    for (int eye = 0; eye < 2; ++eye) {
      const Tap& t = eye ? tr : tl;
      float b = eye ? br : bl;
      fetch_rgb<SRC_U8>(a, lut, t.y0, t.x0, l00);
      fetch_rgb<SRC_U8>(a, lut, t.y0, t.x1, l01);
      fetch_rgb<SRC_U8>(a, lut, t.y1, t.x0, l10);
      fetch_rgb<SRC_U8>(a, lut, t.y1, t.x1, l11);
      float c[3];
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        float s = tap_apply(t, l00[ch], l01[ch], l10[ch], l11[ch]);
        c[ch] = clamp01((s * (1.0f - b)) + (o[ch] * b));
      }
      uint8_t r8 = trunc_u8(c[0]), g8 = trunc_u8(c[1]), b8 = trunc_u8(c[2]);
      if (a.grade) {
        float r = lut[r8], g = lut[g8], bb = lut[b8];
        grade_px(r, g, bb, a.sat, a.con, a.bri);
        r8 = trunc_u8(r);
        g8 = trunc_u8(g);
        b8 = trunc_u8(bb);
      }
      uint8_t* dst = eye ? orr : ol;
      dst[3 * i] = b8;
      dst[3 * i + 1] = g8;
      dst[3 * i + 2] = r8;
    }
  }
  size_t oo = ((size_t)y * W + x0) * 3;
  if (nvalid == 4 && (oo & 3) == 0) {
    uint32_t* pl = (uint32_t*)(a.left + oo);
    uint32_t* pr = (uint32_t*)(a.right + oo);
#pragma unroll
    for (int w = 0; w < 3; ++w) {
      pl[w] = (uint32_t)ol[4 * w] | ((uint32_t)ol[4 * w + 1] << 8) | ((uint32_t)ol[4 * w + 2] << 16) |
              ((uint32_t)ol[4 * w + 3] << 24);
      pr[w] = (uint32_t)orr[4 * w] | ((uint32_t)orr[4 * w + 1] << 8) | ((uint32_t)orr[4 * w + 2] << 16) |
              ((uint32_t)orr[4 * w + 3] << 24);
    }
  } else {
    for (int i = 0; i < nvalid * 3; ++i) {
      a.left[oo + i] = ol[i];
      a.right[oo + i] = orr[i];
    }
  }
}

// ---------------------------------------------------------------------------
// K8 DOF + colour grade on a u8 eye (core/render_3d.py:769-834, 1342-1369)
// blockIdx.z selects the eye.  Gaussian levels: row-major fma chain, reflect padding.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_dof(DofArgs a) {
  extern __shared__ float dtile[];  // 3 planes of (32+2R) x (8+2R)
  const int R = a.halo;
  const int tw = 32 + 2 * R, th = 8 + 2 * R;
  const int bx = blockIdx.x * 32, by = blockIdx.y * 8;
  const int H = a.H, W = a.W;
  const uint8_t* src = blockIdx.z ? a.src_r : a.src_l;
  uint8_t* dst = blockIdx.z ? a.dst_r : a.dst_l;
  for (int i = threadIdx.x; i < tw * th; i += 256) {
    int ty = i / tw, tx = i % tw;
    int gy = by - R + ty, gx = bx - R + tx;
    // torch reflect padding (no edge repeat); clamp afterwards for tiles past the image
    if (gy < 0) gy = -gy;
    if (gy >= H) gy = 2 * H - 2 - gy;
    if (gx < 0) gx = -gx;
    if (gx >= W) gx = 2 * W - 2 - gx;
    gy = min(max(gy, 0), H - 1);
    gx = min(max(gx, 0), W - 1);
    const uint8_t* q = src + ((size_t)gy * W + gx) * 3;
    dtile[i] = (float)q[2] / 255.0f;
    dtile[tw * th + i] = (float)q[1] / 255.0f;
    dtile[2 * tw * th + i] = (float)q[0] / 255.0f;
  }
  __syncthreads();
  int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
  int x = bx + lx, y = by + ly;
  if (x >= W || y >= H) return;
  float c[3];
  int ctr = (ly + R) * tw + lx + R;
  if (a.nlevels > 1) {
    float d = bilinear_f32(a.depth, a.dh, a.dw, H, W, y, x);
    float focal = a.fs ? (float)a.fs->focal : a.focal;  // torch.tensor(float(focal_depth))
    float diff = fabsf(d - focal);
    float bw = clamp01(diff / a.focus_w);
    float bidx = fminf(fmaxf(bw * (float)(a.nlevels - 1), 0.f), a.idx_max);
    int lo = (int)floorf(bidx);
    lo = min(max(lo, 0), a.nlevels - 2);
    float al = bidx - (float)lo;
    float one_m = 1.0f - al;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float* pl = dtile + ch * tw * th;
      float v[2];
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        int lvl = lo + s;
        int ks = a.ksize[lvl];
        if (ks <= 1) {
          v[s] = pl[ctr];
        } else {
          int pr = ks / 2;
          const float* kw = a.kern + a.koff[lvl];
          float acc = 0.f;
          for (int dy = 0; dy < ks; ++dy) {
            const float* row = pl + (ly + R - pr + dy) * tw + (lx + R - pr);
            for (int dx = 0; dx < ks; ++dx) acc = __fmaf_rn(row[dx], kw[dy * ks + dx], acc);
          }
          v[s] = acc;
        }
      }
      c[ch] = clamp01((one_m * v[0]) + (al * v[1]));
    }
  } else {
    c[0] = dtile[ctr];
    c[1] = dtile[tw * th + ctr];
    c[2] = dtile[2 * tw * th + ctr];
  }
  grade_px(c[0], c[1], c[2], a.sat, a.con, a.bri);
  size_t oo = ((size_t)y * W + x) * 3;
  dst[oo] = trunc_u8(c[2]);
  dst[oo + 1] = trunc_u8(c[1]);
  dst[oo + 2] = trunc_u8(c[0]);
}

// ---------------------------------------------------------------------------
// K9 post: floating-window bars, sharpen, eye fit, pack
// (core/render_3d.py:885-892, 717-732, 1409-1419, 837-883)
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint8_t eye_px(const uint8_t* __restrict__ eye, int W, int y, int x, int ch, int bar_lo,
                                          int bar_hi) {
  if (x >= bar_lo && x < bar_hi) return 0;  // apply_side_mask
  return eye[((size_t)y * W + x) * 3 + ch];
}

__device__ __forceinline__ int sharp_px(const uint8_t* __restrict__ eye, int H, int W, int y, int x, int ch,
                                        int bar_lo, int bar_hi, float kc, float ke, int do_sharpen) {
  if (!do_sharpen) return eye_px(eye, W, y, x, ch, bar_lo, bar_hi);
  int ym = reflect101(y - 1, H), yp = reflect101(y + 1, H);
  int xm = reflect101(x - 1, W), xp = reflect101(x + 1, W);
  float acc = 0.f;  // cv2.filter2D: row-major taps, fma chain, delta 0
  acc = __fmaf_rn((float)eye_px(eye, W, ym, x, ch, bar_lo, bar_hi), ke, acc);
  acc = __fmaf_rn((float)eye_px(eye, W, y, xm, ch, bar_lo, bar_hi), ke, acc);
  acc = __fmaf_rn((float)eye_px(eye, W, y, x, ch, bar_lo, bar_hi), kc, acc);
  acc = __fmaf_rn((float)eye_px(eye, W, y, xp, ch, bar_lo, bar_hi), ke, acc);
  acc = __fmaf_rn((float)eye_px(eye, W, yp, x, ch, bar_lo, bar_hi), ke, acc);
  return (int)rhe_u8(acc);
}

// value of the fitted (resized / padded) eye image at (ex, ey) in per-eye coordinates
__device__ __forceinline__ int fitted_px(const PostArgs& a, const uint8_t* eye, int ey, int ex, int ch, int bar_lo,
                                         int bar_hi) {
  int fx = ex - a.fit_x0, fy = ey - a.fit_y0;
  if (fx < 0 || fy < 0 || fx >= a.fit_w || fy >= a.fit_h) return 0;  // pad_to_aspect_ratio canvas
  if (a.lin) {
    // cv2 resize(INTER_AREA) with an enlarged axis: HResizeLinear on int rows, then VResizeLinear<uchar, int, short>
    const int sx0 = a.xofs[fx], sx1 = min(sx0 + 1, a.W - 1), sy0 = a.yofs[fy], sy1 = min(sy0 + 1, a.H - 1);
    const int a0 = (int)a.xal[2 * fx], a1 = (int)a.xal[2 * fx + 1];
    const int b0 = (int)a.yal[2 * fy], b1 = (int)a.yal[2 * fy + 1];
    const int r0 = sharp_px(eye, a.H, a.W, sy0, sx0, ch, bar_lo, bar_hi, a.kc, a.ke, a.sharpen) * a0 +
                   sharp_px(eye, a.H, a.W, sy0, sx1, ch, bar_lo, bar_hi, a.kc, a.ke, a.sharpen) * a1;
    const int r1 = sharp_px(eye, a.H, a.W, sy1, sx0, ch, bar_lo, bar_hi, a.kc, a.ke, a.sharpen) * a0 +
                   sharp_px(eye, a.H, a.W, sy1, sx1, ch, bar_lo, bar_hi, a.kc, a.ke, a.sharpen) * a1;
    const int v = (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2;
    return min(max(v, 0), 255);
  }
  if (a.xal) {
    // cv2 ResizeArea_ (non-integer INTER_AREA shrink): per source row buf = sum_k S * alpha_k, rows combined as
    // sum = beta_0 * buf_0 + beta_1 * buf_1 ... ; fp32, separate multiply and add (this unit is built with -fmad=false)
    const int xo = a.xofs[fx], xc = a.xcnt[fx], yo = a.yofs[fy], yc = a.ycnt[fy];
    const float* xa = a.xal + (size_t)fx * a.area_t;
    const float* ya = a.yal + (size_t)fy * a.area_t;
    float acc = 0.f;
    for (int j = 0; j < yc; ++j) {
      float buf = 0.f;
      for (int i = 0; i < xc; ++i)
        buf = buf + (float)sharp_px(eye, a.H, a.W, yo + j, xo + i, ch, bar_lo, bar_hi, a.kc, a.ke, a.sharpen) * xa[i];
      const float t = ya[j] * buf;
      acc = j ? acc + t : t;
    }
    return (int)rhe_u8(acc);
  }
  if (a.sx == 1 && a.sy == 1) return sharp_px(eye, a.H, a.W, fy, fx, ch, bar_lo, bar_hi, a.kc, a.ke, a.sharpen);
  int sum = 0;
  for (int j = 0; j < a.sy; ++j)
    for (int i = 0; i < a.sx; ++i)
      sum += sharp_px(eye, a.H, a.W, fy * a.sy + j, fx * a.sx + i, ch, bar_lo, bar_hi, a.kc, a.ke, a.sharpen);
  if (a.sx == 2 && a.sy == 2) return (sum + 2) >> 2;  // cv2 INTER_AREA 2x2 integer fast path
  return (int)rhe_u8((float)sum * a.inv_area);
}

__global__ void __launch_bounds__(256) k_post(PostArgs a) {
  int ox = blockIdx.x * 32 + (threadIdx.x & 31);
  int oy = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (ox >= a.out_w || oy >= a.out_h) return;
  int bar_lo = 0, bar_hi = 0;
  if (a.fs) {
    int bw = a.fs->bar_width;
    if (a.fs->bar_side == 1) {
      bar_lo = a.W - bw;
      bar_hi = a.W;
    } else if (a.fs->bar_side == 2) {
      bar_lo = 0;
      bar_hi = bw;
    }
  }
  uint8_t o[3];
  if (a.fmt == VD3D_FMT_HALF_SBS || a.fmt == VD3D_FMT_FULL_SBS || a.fmt == VD3D_FMT_VR) {  // hstack of the fitted eyes
    int eye = ox / a.per_eye_w;
    int ex = ox - eye * a.per_eye_w;
    const uint8_t* e = eye ? a.right : a.left;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) o[ch] = (uint8_t)fitted_px(a, e, oy, ex, ch, bar_lo, bar_hi);
  } else if (a.fmt == VD3D_FMT_INTERLACED) {
    const uint8_t* e = (oy & 1) ? a.right : a.left;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) o[ch] = (uint8_t)fitted_px(a, e, oy, ox, ch, bar_lo, bar_hi);
  } else {  // Dubois anaglyph on channel indices 0,1,2 as split from the BGR arrays (862-883)
    float l[3], r[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      l[ch] = (float)fitted_px(a, a.left, oy, ox, ch, bar_lo, bar_hi) / 255.0f;
      r[ch] = (float)fitted_px(a, a.right, oy, ox, ch, bar_lo, bar_hi) / 255.0f;
    }
    float red = ((0.4561f * l[0]) + (0.5005f * l[1])) + (0.1762f * l[2]);
    float grn = ((0.3764f * r[0]) + (0.7616f * r[1])) - (0.1876f * r[2]);
    float blu = ((-0.0401f * r[0]) - (0.1126f * r[1])) + (1.2723f * r[2]);
    o[0] = trunc_u8(clamp01(red));
    o[1] = trunc_u8(clamp01(grn));
    o[2] = trunc_u8(clamp01(blu));
  }
  size_t oo = ((size_t)oy * a.out_w + ox) * 3;
  a.out[oo] = o[0];
  a.out[oo + 1] = o[1];
  a.out[oo + 2] = o[2];
}

// ---------------------------------------------------------------------------
// heal_missing_pixels (core/render_3d.py:431-459): gradient-gated blend of the warped eye toward the
// original frame + 3x3 softening.  f32 RGB planes in/out.  One pass: gray (halo 4) -> gradient flags
// (halo 3) -> 5x5 pooled mask (halo 1) -> healed (halo 1) -> 3x3 blur -> out.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_heal(const float* __restrict__ warped, const float* __restrict__ orig,
                                              const float* __restrict__ edge, float* __restrict__ out, int H, int W,
                                              float hs) {
  __shared__ float gray[16][41];    // y in [by-4, by+12), x in [bx-4, bx+36)   (+1 pad)
  __shared__ float flag[14][39];    // grad > 0.05 over [by-3, by+11) x [bx-3, bx+35)
  __shared__ float mm[10][35];      // pooled mask over [by-1, by+9) x [bx-1, bx+33)
  __shared__ float heal[3][10][35];
  const int bx = blockIdx.x * 32, by = blockIdx.y * 8;
  const size_t plane = (size_t)H * W;
  for (int i = threadIdx.x; i < 16 * 40; i += 256) {
    int ty = i / 40, tx = i % 40, gy = by - 4 + ty, gx = bx - 4 + tx;
    float v = 0.f;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
      size_t o = (size_t)gy * W + gx;
      v = ((warped[o] + warped[plane + o]) + warped[2 * plane + o]) / 3.0f;
    }
    gray[ty][tx] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 14 * 38; i += 256) {
    int ty = i / 38, tx = i % 38, gy = by - 3 + ty, gx = bx - 3 + tx;
    float f = 0.f;  // zero padding of avg_pool2d outside the image
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
      float c = gray[ty + 1][tx + 1];
      float dx = (gx > 0) ? (c - gray[ty + 1][tx]) : 0.f;
      float dy = (gy > 0) ? (c - gray[ty][tx + 1]) : 0.f;
      f = (sqrtf((dx * dx) + (dy * dy)) > 0.05f) ? 1.f : 0.f;
    }
    flag[ty][tx] = f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 10 * 34; i += 256) {
    int ty = i / 34, tx = i % 34, gy = by - 1 + ty, gx = bx - 1 + tx;
    float m = 0.f;
    bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
    if (in) {
      float acc = 0.f;
#pragma unroll
      for (int dy = 0; dy < 5; ++dy)
#pragma unroll
        for (int dx = 0; dx < 5; ++dx) acc = acc + flag[ty + dy][tx + dx];
      m = clamp01(acc / 25.0f);
      if (edge) m = fmaxf(m, edge[(size_t)gy * W + gx]);
    }
    mm[ty][tx] = m;
    float hm = hs * m;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float hv = 0.f;  // zero padding for the 3x3 pool
      if (in) {
        size_t o = c * plane + (size_t)gy * W + gx;
        hv = ((1.0f - hm) * warped[o]) + (hm * orig[o]);
      }
      heal[c][ty][tx] = hv;
    }
  }
  __syncthreads();
  int lx = threadIdx.x & 31, ly = threadIdx.x >> 5, x = bx + lx, y = by + ly;
  if (x >= W || y >= H) return;
  float sm = 0.3f * mm[ly + 1][lx + 1];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float acc = 0.f;
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) acc = acc + heal[c][ly + dy][lx + dx];
    float soft = acc / 9.0f;
    float v = ((1.0f - sm) * heal[c][ly + 1][lx + 1]) + (sm * soft);
    out[c * plane + (size_t)y * W + x] = clamp01(v);
  }
}

// cv2.resize(u8 plane, INTER_CUBIC) (core/render_depth.py:1917): float32 bicubic, A = -0.75, rows then columns,
// round half to even -- the arithmetic of oracle.resize_cubic_u8 (pinned to the installed cv2 / IPP); taps: cubic_tap
__global__ void __launch_bounds__(256) k_resize_cubic_u8(const uint8_t* __restrict__ src, int h, int w, int ch,
                                                         uint8_t* __restrict__ dst, int oh, int ow) {
  int x = blockIdx.x * 32 + (threadIdx.x & 31);
  int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= ow || y >= oh) return;
  resize_cubic_u8_px(src, (size_t)w * ch, h, w, ch, dst, oh, ow, x, y);
}
void launch_resize_cubic_u8(const uint8_t* src, int h, int w, int ch, uint8_t* dst, int oh, int ow, cudaStream_t s) {
  dim3 g((ow + 31) / 32, (oh + 7) / 8);
  k_resize_cubic_u8<<<g, 256, 0, s>>>(src, h, w, ch, dst, oh, ow);
}

// cv2.addWeighted(a, alpha, b, beta, 0) on u8 (blend_images, core/merged_pipeline.py:233-238): cv2 4.13 evaluates
// fma(a, alpha, fl(b * beta)) in float32, rounds half to even, saturates (oracle/sr.py, pinned exact against cv2)
__global__ void __launch_bounds__(256) k_add_weighted(const uint8_t* __restrict__ a, float alpha,
                                                      const uint8_t* __restrict__ b, float beta, uint8_t* __restrict__ dst,
                                                      size_t n) {
  size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  float t = (float)b[i] * beta;
  dst[i] = rhe_u8(__fmaf_rn((float)a[i], alpha, t));
}
void launch_add_weighted(const uint8_t* a, float alpha, const uint8_t* b, float beta, uint8_t* dst, size_t n,
                         cudaStream_t s) {
  k_add_weighted<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a, alpha, b, beta, dst, n);
}

// apply_color_grade (core/render_3d.py:734-767) on planar f32 RGB
__global__ void __launch_bounds__(256) k_grade_f32(const float* __restrict__ src, float* __restrict__ dst, int n, float sat,
                                                   float con, float bri) {
  int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  float r = src[i], g = src[n + i], b = src[2 * (size_t)n + i];
  grade_px(r, g, b, sat, con, bri);
  dst[i] = r;
  dst[n + i] = g;
  dst[2 * (size_t)n + i] = b;
}

// ---------------------------------------------------------------------------
// launch wrappers
// ---------------------------------------------------------------------------
void launch_grade_f32(const float* src, float* dst, int n, float sat, float con, float bri, cudaStream_t s) {
  k_grade_f32<<<(n + 255) / 256, 256, 0, s>>>(src, dst, n, sat, con, bri);
}
void launch_heal(const float* warped, const float* orig, const float* edge, float* out, int H, int W, float hs,
                 cudaStream_t s) {
  dim3 g((W + 31) / 32, (H + 7) / 8);
  k_heal<<<g, 256, 0, s>>>(warped, orig, edge, out, H, W, hs);
}
static inline dim3 grid2d(int w, int h) { return dim3((w + 31) / 32, (h + 7) / 8); }

void launch_ingest(const IngestArgs& a, cudaStream_t s) { k_ingest<<<grid2d(a.tw, a.th), 256, 0, s>>>(a); }
void launch_black_bars(const uint8_t* frame, int h, int w, int threshold, uint32_t* words, cudaStream_t s) {
  k_black_bars<<<(h + 7) / 8, 256, 0, s>>>(frame, h, w, threshold, words);
}

void launch_resize_planar(const float* src, int C, int sh, int sw, float* dst, int oh, int ow, cudaStream_t s) {
  k_resize_planar<<<grid2d(ow, oh), 256, 0, s>>>(src, C, sh, sw, dst, oh, ow);
}

void launch_select(const SelJob& a, const SelJob* b, int nblocks, cudaStream_t s) {
  SelJob bb = b ? *b : a;
  int nb = b ? 1 : 0;
  k_sel_pass<1><<<nblocks, 256, 0, s>>>(a, bb, nb);
  k_sel_find<1><<<1 + nb, 1024, 0, s>>>(a, bb);
  k_sel_pass<2><<<nblocks, 256, 0, s>>>(a, bb, nb);
  k_sel_find<2><<<1 + nb, 1024, 0, s>>>(a, bb);
  k_sel_pass<3><<<nblocks, 256, 0, s>>>(a, bb, nb);
  k_sel_find<3><<<1 + nb, 1024, 0, s>>>(a, bb);
}

void launch_fin_pct(const SelJob& j, float w_lo, float w_hi, float alpha, float oma, DevState* st, FrameScalars* fs,
                    cudaStream_t s) {
  k_fin_pct<<<1, 1, 0, s>>>(j, w_lo, w_hi, alpha, oma, st, fs);
}
void launch_normalize(const float* tdf, float* dn, const float* dn_prev, int th, int tw, const DevState* st,
                      FrameScalars* fs, cudaStream_t s) {
  k_normalize<<<grid2d(tw, th), 256, 0, s>>>(tdf, dn, dn_prev, th, tw, st, fs);
}
void launch_fin_norm(const SelJob& j, const LoopArgs& la, DevState* st, FrameScalars* fs, cudaStream_t s) {
  k_fin_norm<<<1, 1, 0, s>>>(j, la, st, fs);
}
void launch_set_ranks(SelTarget* tg, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3, cudaStream_t s) {
  k_set_ranks<<<1, 1, 0, s>>>(tg, r0, r1, r2, r3);
}
void launch_set_shifts(FrameScalars* fs, double fg, double mg, double bg, cudaStream_t s) {
  k_set_shifts<<<1, 1, 0, s>>>(fs, fg, mg, bg);
}
void launch_d0(const float* src, int sh, int sw, float* d0, int H, int W, const float* xs, const float* ys,
               float strength, cudaStream_t s) {
  k_d0<<<grid2d(W, H), 256, 0, s>>>(src, sh, sw, d0, H, W, xs, ys, strength);
}
void launch_fin_d0(const SelJob& q, const SelJob& sj, float w_lo, float w_hi, FrameScalars* fs, cudaStream_t s) {
  k_fin_d0<<<1, 1, 0, s>>>(q, sj, w_lo, w_hi, fs);
}
void launch_shape(float* d, int n, const FrameScalars* fs, float mid, float gamma, cudaStream_t s) {
  k_shape<<<(n + 255) / 256, 256, 0, s>>>(d, n, fs, mid, gamma);
}
void launch_fin_shape(const SelJob& sj, const ShiftArgs& sa, DevState* st, FrameScalars* fs, cudaStream_t s) {
  k_fin_shape<<<1, 1, 0, s>>>(sj, sa, st, fs);
}
void launch_shift(const float* d, float* shift, int H, int W, const FrameScalars* fs, int edge_mask, float feather,
                  cudaStream_t s) {
  k_shift<false><<<grid2d(W, H), 256, 0, s>>>(d, shift, H, W, fs, edge_mask, feather);
}
void launch_warp_edges(const float* d, const float* shift, float2* e2, int H, int W, const float* xs,
                       const float* ys, float feather, cudaStream_t s) {
  k_warp_edges<<<grid2d(W, H), 256, 0, s>>>(d, shift, e2, H, W, xs, ys, feather);
}
int compose_smem_bytes(int k) { return (32 + k - 1) * (8 + k - 1) * (int)sizeof(float2); }
cudaError_t init_kernel_attributes() {
  cudaError_t e;
  e = cudaFuncSetAttribute(k_compose<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(k_compose<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(k_dof, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
  return e;
}
template <int K>
static void launch_compose4(const ComposeArgs& a, cudaStream_t s) {
  constexpr int TW = 128 + K - 1 + ((128 + K - 1) & 1);
  int smem = TW * (8 + K - 1) * (int)sizeof(float2);
  dim3 g((a.W + 127) / 128, (a.H + 7) / 8);
  if (a.src_u8)
    k_compose4<true, K><<<g, 256, smem, s>>>(a);
  else
    k_compose4<false, K><<<g, 256, smem, s>>>(a);
}
void launch_compose(const ComposeArgs& a, cudaStream_t s) {
  if (a.feather) {
    switch (a.k) {
      case 3: return launch_compose4<3>(a, s);
      case 5: return launch_compose4<5>(a, s);
      case 7: return launch_compose4<7>(a, s);
      case 9: return launch_compose4<9>(a, s);
      default: break;
    }
  }
  int smem = a.feather ? compose_smem_bytes(a.k) : 0;
  if (a.src_u8)
    k_compose<true><<<grid2d(a.W, a.H), 256, smem, s>>>(a);
  else
    k_compose<false><<<grid2d(a.W, a.H), 256, smem, s>>>(a);
}
void launch_dof(const DofArgs& a, int eyes, cudaStream_t s) {
  int smem = 3 * (32 + 2 * a.halo) * (8 + 2 * a.halo) * (int)sizeof(float);
  dim3 g = grid2d(a.W, a.H);
  g.z = eyes;
  k_dof<<<g, 256, smem, s>>>(a);
}
void launch_post(const PostArgs& a, cudaStream_t s) { k_post<<<grid2d(a.out_w, a.out_h), 256, 0, s>>>(a); }

}  // namespace vd3d
