// dibr_fast.cu -- the bandwidth-oriented form of the DIBR stage (default; the one-kernel-per-op form in
// dibr_kernels.cu stays selectable with vd3d_set_exact() and is what the bit-for-bit oracle tests drive).
//
// One frame of the render_sbs_3d loop body (core/render_3d.py:1227-1419) is three launches:
//   k_stats   persistent cooperative kernel (one CTA per SM, grid-wide barriers between phases): ingest +
//             TemporalDepthFilter, the four radix selects (torch.quantile x2, torch.median + histc x3), percentile
//             normalise + centre statistics + motion metric, curvature, pop shaping, and every scalar tracker of the
//             reference computed redundantly by thread 0 of every CTA from the same global histograms (identical
//             results, no extra barrier); CTA 0 publishes DevState / FrameScalars at the end.  Pass 1 of every select
//             rides on the phase that PRODUCES the plane, so a select costs two extra reads (from L2), not three.
//   k_shift_fast  shift map + edge-mask suppression: 4 pixels per thread, ex2 / rcp / sqrt approximations, separable pool.
//   k_render  per 64x32 tile: warped depth of both eyes (tile + halo) -> gradient edge mask -> separable KxK box
//             sum in shared memory -> 4-tap RGB gather, feather blend, truncation, colour grade -> u8 eye tile in
//             shared memory -> [floating-window bars, 3x3 sharpen, INTER_AREA 1:1 / 2:1 eye fit, SBS pack] -> output.
//             Replaces k_warp_edges + k_compose (+ k_post for the two SBS fits) and their e2 / eye round trips.
//
// Numerics: same op order as the exact path everywhere except (i) |x|^gamma, sigmoid and (1-d)^1.5 use fp32 hardware
// approximations instead of correctly rounded fp64 (<= 3e-7 relative), (ii) the KxK box sum is separable (row sums
// then column sums) instead of row-major over all K*K taps.  Both are far inside the north-star tolerances (1e-3 on
// float intermediates, 1 LSB on the u8 eyes); tests/test_dibr_gpu.py gates them against the oracle.
#include "dibr_device.cuh"
#include "dibr_launch.h"

namespace vd3d {

namespace {

constexpr int NT = 1024;  // threads per CTA of k_stats
constexpr int UNR = 4;    // independent elements in flight per thread

// ---------------------------------------------------------------------------------------------------------------
// k_stats shared memory
// ---------------------------------------------------------------------------------------------------------------
struct SelState {  // bookkeeping of one selection job; every CTA computes the same values
  int nt;
  uint32_t count;
  uint32_t rank[4], p1[4], r1[4], p2[4], r2[4], bits[4];
  int g1[4], g2[4];  // histogram group of target t in pass 2 / pass 3
  int ng1, ng2;
  uint32_t gp1[4];           // pass-2 groups: first-level bin
  uint32_t gq1[4], gq2[4];   // pass-3 groups: (first, second)-level bins
};

struct StatsSmem {
  uint32_t sh1[2][4096];
  uint32_t cum[4096];
  uint32_t sh64[2][64];
  uint32_t h64[64];
  uint32_t wsum[32];
  float lut[256];     // i / 255.0f (the IEEE division costs ~10 issue slots; ingest needs 16 per pixel)
  double red[3][32];
  SelState sel[3];
  DevState st;
  FrameScalars fs;
  int crop[4];        // ingest source rectangle {x0, y0, w, h} of this frame (the fixed crop, or auto_crop_black_bars)
};

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// grid-wide barrier on a monotone counter (zeroed by the host before the launch); the launch is cooperative, so all
// CTAs are co-resident
__device__ __forceinline__ void grid_barrier(unsigned* bar, unsigned& epoch) {
  __syncthreads();
  if (threadIdx.x == 0) {
    epoch += gridDim.x;
    __threadfence();
    atomicAdd(bar, 1u);
    while (ld_acquire(bar) < epoch) {
    }
    __threadfence();
  }
  __syncthreads();
}

// histogram increment, all 32 lanes call it.  Depth planes are smooth, so the lanes of a warp mostly hit one bin: the
// lanes that share the first participating lane's bin are counted with one ballot and added once; the rest fall back
// to per-lane atomics (few, and on distinct addresses for noisy content).  Replaces __match_any_sync, whose cost
// (~32 dependent steps) dominated the streaming phases.
__device__ __forceinline__ void hist_add(uint32_t* hist, bool on, uint32_t bin) {
  const unsigned ballot = __ballot_sync(0xffffffffu, on);
  if (!ballot) return;
  const int leader = __ffs(ballot) - 1;
  const uint32_t b0 = __shfl_sync(0xffffffffu, bin, leader);
  const bool mine = on && bin == b0;
  const unsigned grp = __ballot_sync(0xffffffffu, mine);
  if ((int)(threadIdx.x & 31) == leader) atomicAdd(&hist[b0], (uint32_t)__popc(grp));
  if (on && !mine) atomicAdd(&hist[bin], 1u);
}

// idx / d for idx < 2^24 (every plane up to 16.7 Mpx) by a 40-bit reciprocal; plain division beyond
struct FastDiv {
  uint32_t d;
  uint64_t m;
  bool ok;
};
__device__ __forceinline__ FastDiv fast_div(uint32_t d, uint32_t max_idx) {
  FastDiv f;
  f.d = d;
  f.m = ((1ull << 40) / d) + 1ull;
  f.ok = max_idx < (1u << 24) && d < (1u << 15);
  return f;
}
__device__ __forceinline__ void divmod(const FastDiv& f, int idx, int& q, int& r) {
  uint32_t qq = f.ok ? (uint32_t)(((uint64_t)(uint32_t)idx * f.m) >> 40) : (uint32_t)idx / f.d;
  q = (int)qq;
  r = idx - (int)(qq * f.d);
}

__device__ __forceinline__ uint32_t key_of(float v01) { return __float_as_uint(v01) & 0x7FFFFFFFu; }

__device__ __forceinline__ void zero_pass1(StatsSmem& S) {
  for (int i = threadIdx.x; i < 2 * 4096; i += NT) (&S.sh1[0][0])[i] = 0;
  if (threadIdx.x < 128) (&S.sh64[0][0])[threadIdx.x] = 0;
  __syncthreads();
}

__device__ __forceinline__ void flush_pass1(StatsSmem& S, int slot, const JobMem& jm, bool want64) {
  for (int i = threadIdx.x; i < 4096; i += NT) {
    uint32_t v = S.sh1[slot][i];
    if (v) atomicAdd(&jm.hist1[i], v);
  }
  if (want64 && threadIdx.x < 64) {
    uint32_t v = S.sh64[slot][threadIdx.x];
    if (v) atomicAdd(&jm.hist64[threadIdx.x], v);
  }
}

// inclusive scan of a 4096-bin global histogram into S.cum; returns the total
__device__ uint32_t scan4096(StatsSmem& S, const uint32_t* gh) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint4 v = __ldcg(reinterpret_cast<const uint4*>(gh) + tid);
  uint32_t a = v.x, b = a + v.y, c = b + v.z, d = c + v.w;
  uint32_t s = d;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, s, off);
    if (lane >= off) s += t;
  }
  __syncthreads();  // previous users of wsum / cum are done
  if (lane == 31) S.wsum[warp] = s;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = S.wsum[lane];
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      uint32_t t = __shfl_up_sync(0xffffffffu, w, off);
      if (lane >= off) w += t;
    }
    S.wsum[lane] = w;
  }
  __syncthreads();
  uint32_t base = (warp ? S.wsum[warp - 1] : 0u) + (s - d);
  S.cum[4 * tid] = base + a;
  S.cum[4 * tid + 1] = base + b;
  S.cum[4 * tid + 2] = base + c;
  S.cum[4 * tid + 3] = base + d;
  __syncthreads();
  return S.wsum[31];
}

__device__ void scan64(StatsSmem& S, const uint32_t* gh) {
  const int tid = threadIdx.x;
  __syncthreads();
  if (tid < 32) {
    uint32_t a = __ldcg(gh + 2 * tid), b = a + __ldcg(gh + 2 * tid + 1);
    uint32_t s = b;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      uint32_t t = __shfl_up_sync(0xffffffffu, s, off);
      if (tid >= off) s += t;
    }
    S.cum[2 * tid] = s - b + a;
    S.cum[2 * tid + 1] = s;
  }
  __syncthreads();
}

// for every target t in `mask`: the bin of S.cum[0..nb) that holds rank r[t], and the residual rank inside it
__device__ void find_bins(StatsSmem& S, int nb, const uint32_t* r, uint32_t* outbin, uint32_t* outres, int nt,
                          unsigned mask) {
  for (int i = threadIdx.x; i < nb; i += NT) {
    uint32_t lo = i ? S.cum[i - 1] : 0u, hi = S.cum[i];
    for (int t = 0; t < nt; ++t)
      if (((mask >> t) & 1u) && r[t] >= lo && r[t] < hi) {
        outbin[t] = (uint32_t)i;
        outres[t] = r[t] - lo;
      }
  }
  __syncthreads();
}

__device__ void after_pass1(StatsSmem& S, SelState& q, const JobMem& jm, bool rank_from_count) {
  uint32_t total = scan4096(S, jm.hist1);
  if (threadIdx.x == 0) {
    q.count = total;
    if (rank_from_count) q.rank[0] = total ? (total - 1) / 2 : 0u;  // torch.median: lower middle
    for (int t = 0; t < 4; ++t) q.p1[t] = q.r1[t] = q.p2[t] = q.r2[t] = q.bits[t] = 0u;
  }
  __syncthreads();
  find_bins(S, 4096, q.rank, q.p1, q.r1, q.nt, 0xFu);
  if (threadIdx.x == 0) {
    q.ng1 = 0;
    for (int t = 0; t < q.nt; ++t) {
      int g = -1;
      for (int u = 0; u < t; ++u)
        if (q.p1[u] == q.p1[t]) {
          g = q.g1[u];
          break;
        }
      if (g < 0) {
        g = q.ng1++;
        q.gp1[g] = q.p1[t];
      }
      q.g1[t] = g;
    }
  }
  __syncthreads();
}

__device__ void after_pass2(StatsSmem& S, SelState& q, const JobMem& jm) {
  for (int g = 0; g < q.ng1; ++g) {
    scan4096(S, jm.hist2 + g * 4096);
    unsigned mask = 0;
    for (int t = 0; t < q.nt; ++t)
      if (q.g1[t] == g) mask |= 1u << t;
    find_bins(S, 4096, q.r1, q.p2, q.r2, q.nt, mask);
  }
  if (threadIdx.x == 0) {
    q.ng2 = 0;
    for (int t = 0; t < q.nt; ++t) {
      int g = -1;
      for (int u = 0; u < t; ++u)
        if (q.p1[u] == q.p1[t] && q.p2[u] == q.p2[t]) {
          g = q.g2[u];
          break;
        }
      if (g < 0) {
        g = q.ng2++;
        q.gq1[g] = q.p1[t];
        q.gq2[g] = q.p2[t];
      }
      q.g2[t] = g;
    }
  }
  __syncthreads();
}

__device__ void after_pass3(StatsSmem& S, SelState& q, const JobMem& jm) {
  __shared__ uint32_t b3[4], r3[4];
  for (int g = 0; g < q.ng2; ++g) {
    scan64(S, jm.hist3 + g * 64);
    unsigned mask = 0;
    for (int t = 0; t < q.nt; ++t)
      if (q.g2[t] == g) mask |= 1u << t;
    if (threadIdx.x < 4) b3[threadIdx.x] = 0;
    __syncthreads();
    find_bins(S, 64, q.r2, b3, r3, q.nt, mask);
    if (threadIdx.x == 0)
      for (int t = 0; t < q.nt; ++t)
        if ((mask >> t) & 1u) q.bits[t] = (q.p1[t] << 18) | (q.p2[t] << 6) | b3[t];
    __syncthreads();
  }
}

// bins selected so far, held in registers for the streaming passes
struct Grp {
  int n;
  uint32_t a[4], b[4];
};
template <int PASS>
__device__ __forceinline__ Grp load_groups(const SelState& q) {
  Grp g;
  g.n = PASS == 2 ? q.ng1 : q.ng2;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    g.a[i] = PASS == 2 ? q.gp1[i] : q.gq1[i];
    g.b[i] = PASS == 2 ? 0u : q.gq2[i];
  }
  return g;
}
template <int PASS>
__device__ __forceinline__ void pass_add(const Grp& gr, const JobMem& jm, bool on, uint32_t key) {
  int g = -1;
  const uint32_t top = key >> 18, mid = (key >> 6) & 4095u;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (i < gr.n && top == gr.a[i] && (PASS == 2 || mid == gr.b[i])) g = i;
  on = on && g >= 0;
  if (PASS == 2)
    hist_add(jm.hist2, on, (uint32_t)(g < 0 ? 0 : g) * 4096u + mid);
  else
    hist_add(jm.hist3, on, (uint32_t)(g < 0 ? 0 : g) * 64u + (key & 63u));
}

__device__ __forceinline__ bool in_region(const int* rg, int y, int x) {  // rg = {x0, x1, y0, y1}
  return x >= rg[0] && x < rg[1] && y >= rg[2] && y < rg[3];
}
__device__ __forceinline__ bool subj_keep(float v) { return (v > 0.05f) && (v < 0.95f); }
__device__ __forceinline__ int bin64(float v) {
  int b = (int)(v * 64.0f);
  return b > 63 ? 63 : b;
}

// pass 2 or 3 of up to two jobs over a plane: job A over the whole plane (or null), job B over the subject crop with
// the 0.05 < v < 0.95 mask (or null).  Values are read from L2 (written by other CTAs in an earlier phase).
template <int PASS>
__device__ void select_pass(const float* plane, int W, int H, const SelState* qa, const JobMem* ja, const SelState* qb,
                            const JobMem* jb, const int* crop) {
  Grp ga, gb;
  ga.n = gb.n = 0;
  if (qa) ga = load_groups<PASS>(*qa);
  if (qb) gb = load_groups<PASS>(*qb);
  if (qa) {
    const int n = W * H;
    const FastDiv fdw = fast_div((uint32_t)W, (uint32_t)n);
    for (int base = blockIdx.x * (NT * UNR); base < n; base += gridDim.x * (NT * UNR)) {
      float v[UNR];
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        int idx = base + u * NT + threadIdx.x;
        v[u] = idx < n ? clamp01(__ldcg(plane + idx)) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        int idx = base + u * NT + threadIdx.x;
        bool inb = idx < n;
        uint32_t key = key_of(v[u]);
        pass_add<PASS>(ga, *ja, inb, key);
        if (qb) {
          int y, x;
          divmod(fdw, idx, y, x);
          bool on = inb && in_region(crop, y, x) && subj_keep(v[u]);
          pass_add<PASS>(gb, *jb, on, key);
        }
      }
    }
  } else if (qb) {
    const int rw = crop[1] - crop[0], rh = crop[3] - crop[2];
    const int n = rw * rh;
    const FastDiv fdr = fast_div((uint32_t)rw, (uint32_t)n);
    for (int base = blockIdx.x * (NT * UNR); base < n; base += gridDim.x * (NT * UNR)) {
      float v[UNR];
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        int idx = base + u * NT + threadIdx.x;
        int y, x;
        divmod(fdr, idx, y, x);
        v[u] = idx < n ? clamp01(__ldcg(plane + (size_t)(crop[2] + y) * W + crop[0] + x)) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        int idx = base + u * NT + threadIdx.x;
        bool on = idx < n && subj_keep(v[u]);
        uint32_t key = key_of(v[u]);
        pass_add<PASS>(gb, *jb, on, key);
      }
    }
  }
}

__device__ __forceinline__ float ldcg_bilinear(const float* src, int sh, int sw, int oh, int ow, int y, int x) {
  if (sh == oh && sw == ow) return __ldcg(src + (size_t)y * sw + x);
  RsAxis ax = rs_axis(x, sw, ow), ay = rs_axis(y, sh, oh);
  const float* r0 = src + (size_t)ay.i0 * sw;
  const float* r1 = src + (size_t)ay.i1 * sw;
  return rs_combine(__ldcg(r0 + ax.i0), __ldcg(r0 + ax.i1), __ldcg(r1 + ax.i0), __ldcg(r1 + ax.i1), ax, ay);
}

__device__ __forceinline__ float subject_of(StatsSmem& S, const SelState& q, const JobMem& jm) {
  // every thread returns the same value; hist64 is staged through shared memory
  __syncthreads();
  if (threadIdx.x < 64) S.h64[threadIdx.x] = __ldcg(jm.hist64 + threadIdx.x);
  __syncthreads();
  return subject_core(q.count, S.h64, __uint_as_float(q.bits[0]));
}

// depth_to_tensor on one source pixel (cv2 BGR2GRAY fixed point, then / 255 through the table)
__device__ __forceinline__ float depth_lut01(const float* lut, const uint8_t* __restrict__ p, int ch, int pitch_px, int y,
                                             int x) {
  const uint8_t* q = p + ((size_t)y * pitch_px + x) * ch;
  int g = (ch == 1) ? (int)q[0] : ((q[0] * 3735 + q[1] * 19235 + q[2] * 9798 + (1 << 14)) >> 15);
  return lut[g];
}

// ---------------------------------------------------------------------------------------------------------------
// k_stats
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT, 1) k_stats(StatsArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  StatsSmem& S = *reinterpret_cast<StatsSmem*>(smem_raw);
  const int tid = threadIdx.x;
  unsigned epoch = 0;
  const int W = a.W, H = a.H;
  const int crop_d[4] = {W / 5, W * 4 / 5, H / 5, H * 4 / 5};  // estimate_subject_depth centre crop (145-172)

  // ---- private copy of the temporal state; FrameScalars start from zero like begin_frame() does
  if (tid == 0) S.st = *a.st;
  if (tid < 256) S.lut[tid] = (float)tid / 255.0f;
  for (int i = tid; i < (int)(sizeof(FrameScalars) / 4); i += NT) reinterpret_cast<uint32_t*>(&S.fs)[i] = 0u;
  __syncthreads();
  if (tid == 0) {
    S.sel[0].nt = 4;
    S.sel[1].nt = 1;
    S.sel[2].nt = 1;
    if (!a.loop) {
      S.fs.fg = a.sa.p.fg_shift;
      S.fs.mg = a.sa.p.mg_shift;
      S.fs.bg = a.sa.p.bg_shift;
    }
  }
  __syncthreads();

  const int crop_n[4] = {a.ia.tw / 5, a.ia.tw * 4 / 5, a.ia.th / 5, a.ia.th * 4 / 5};  // loop mode only
  if (a.loop) {
    const int tw = a.ia.tw, th = a.ia.th;
    const int ntp = tw * th;
    // ================= ingest + TemporalDepthFilter + pass 1 of q(.02/.98) =================
    zero_pass1(S);
    {
      const IngestArgs& ia = a.ia;
      if (tid == 0) {
        if (ia.bars) {  // auto_crop_black_bars: this frame's rectangle from the words of k_black_bars
          int top, bottom;
          black_bar_crop(ia.src_w, ia.src_h, ia.bars[0], ia.bars[1], ia.aspect, S.crop, &top, &bottom);
          if (blockIdx.x == 0 && ia.crop_out) {
            ia.crop_out[0] = top;
            ia.crop_out[1] = bottom;
          }
        } else {
          S.crop[0] = ia.cx0;
          S.crop[1] = ia.cy0;
          S.crop[2] = ia.cw;
          S.crop[3] = ia.ch;
        }
      }
      __syncthreads();
      const int cx0 = S.crop[0], cy0 = S.crop[1], cw = S.crop[2], ch = S.crop[3];
      const bool ident = (ia.tw == cw && ia.th == ch);
      const int tdf_init = S.st.tdf_init;
      const FastDiv fdt = fast_div((uint32_t)tw, (uint32_t)ntp);
      for (int base = blockIdx.x * (NT * UNR); base < ntp; base += gridDim.x * (NT * UNR)) {
#pragma unroll 1
        for (int u = 0; u < UNR; ++u) {
          int idx = base + u * NT + tid;
          bool inb = idx < ntp;
          float nv = 0.f;
          if (inb) {
            int y, x;
            divmod(fdt, idx, y, x);
            float cur;
            RsAxis ax, ay;
            if (ident && !a.rgbx_s) {
              cur = depth_lut01(S.lut, ia.depth, ia.depth_ch, ia.src_w, cy0 + y, cx0 + x);
            } else {
              ax = rs_axis(x, cw, ia.tw);
              ay = rs_axis(y, ch, ia.th);
              float v00 = depth_lut01(S.lut, ia.depth, ia.depth_ch, ia.src_w, cy0 + ay.i0, cx0 + ax.i0);
              float v01 = depth_lut01(S.lut, ia.depth, ia.depth_ch, ia.src_w, cy0 + ay.i0, cx0 + ax.i1);
              float v10 = depth_lut01(S.lut, ia.depth, ia.depth_ch, ia.src_w, cy0 + ay.i1, cx0 + ax.i0);
              float v11 = depth_lut01(S.lut, ia.depth, ia.depth_ch, ia.src_w, cy0 + ay.i1, cx0 + ax.i1);
              cur = rs_combine(v00, v01, v10, v11, ax, ay);
            }
            float prev = tdf_init ? __ldcg(ia.tdf + idx) : cur;
            nv = (ia.alpha * prev) + (ia.one_minus_alpha * cur);
            ia.tdf[idx] = nv;
            if (a.rgbx_s) {  // frame_to_tensor + F.interpolate to target_eye (1250-1259)
              float c[3];
#pragma unroll
              for (int ch = 0; ch < 3; ++ch) {  // ch: 0=R 1=G 2=B ; source is BGR
                const uint8_t* f = ia.frame + (2 - ch);
                float v00 = S.lut[f[((size_t)(cy0 + ay.i0) * ia.src_w + cx0 + ax.i0) * 3]];
                float v01 = S.lut[f[((size_t)(cy0 + ay.i0) * ia.src_w + cx0 + ax.i1) * 3]];
                float v10 = S.lut[f[((size_t)(cy0 + ay.i1) * ia.src_w + cx0 + ax.i0) * 3]];
                float v11 = S.lut[f[((size_t)(cy0 + ay.i1) * ia.src_w + cx0 + ax.i1) * 3]];
                c[ch] = rs_combine(v00, v01, v10, v11, ax, ay);
              }
              a.rgbx_s[idx] = make_float4(c[0], c[1], c[2], 0.f);
            }
          }
          hist_add(S.sh1[0], inb, key_of(clamp01(nv)) >> 18);
        }
      }
    }
    __syncthreads();
    flush_pass1(S, 0, a.jm[0], false);
    grid_barrier(a.bar, epoch);

    // ================= pass 2 (+ bilinear RGB upsample to the warp resolution, pixel_shift_cuda:595) =================
    if (tid < 4) S.sel[0].rank[tid] = a.pct_rank[tid];
    __syncthreads();
    after_pass1(S, S.sel[0], a.jm[0], false);
    select_pass<2>(a.ia.tdf, tw, th, &S.sel[0], &a.jm[0], nullptr, nullptr, nullptr);
    if (a.rgbx) {
      const int n = W * H;
      const FastDiv fdw = fast_div((uint32_t)W, (uint32_t)n);
      for (int idx = blockIdx.x * NT + tid; idx < n; idx += gridDim.x * NT) {
        int y, x;
        divmod(fdw, idx, y, x);
        RsAxis ax = rs_axis(x, tw, W), ay = rs_axis(y, th, H);
        const float4* r0 = a.rgbx_s + (size_t)ay.i0 * tw;
        const float4* r1 = a.rgbx_s + (size_t)ay.i1 * tw;
        float4 v00 = __ldcg(r0 + ax.i0), v01 = __ldcg(r0 + ax.i1), v10 = __ldcg(r1 + ax.i0), v11 = __ldcg(r1 + ax.i1);
        a.rgbx[idx] = make_float4(rs_combine(v00.x, v01.x, v10.x, v11.x, ax, ay),
                                  rs_combine(v00.y, v01.y, v10.y, v11.y, ax, ay),
                                  rs_combine(v00.z, v01.z, v10.z, v11.z, ax, ay), 0.f);
      }
    }
    grid_barrier(a.bar, epoch);

    // ================= pass 3 =================
    after_pass2(S, S.sel[0], a.jm[0]);
    select_pass<3>(a.ia.tdf, tw, th, &S.sel[0], &a.jm[0], nullptr, nullptr, nullptr);
    grid_barrier(a.bar, epoch);

    // ====== DepthPercentileEMA + normalise + centre statistics + motion + pass 1 of the subject estimate ======
    after_pass3(S, S.sel[0], a.jm[0]);
    if (tid == 0) {
      const SelState& q = S.sel[0];
      fin_pct_core(__uint_as_float(q.bits[0]), __uint_as_float(q.bits[1]), __uint_as_float(q.bits[2]),
                   __uint_as_float(q.bits[3]), a.pct_wlo, a.pct_whi, 0.92f, (float)(1 - 0.92), &S.st, &S.fs);
    }
    zero_pass1(S);
    {
      const int pct_flat = S.fs.pct_flat;
      const float n_lo = S.fs.n_lo, n_den = S.fs.n_den;
      const int have_prev = S.st.have_prev_depth;
      double s = 0, s2 = 0, mad = 0;
      const FastDiv fdt = fast_div((uint32_t)tw, (uint32_t)ntp);
      for (int base = blockIdx.x * (NT * UNR); base < ntp; base += gridDim.x * (NT * UNR)) {
        float tv[UNR], pv[UNR];
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
          int idx = base + u * NT + tid;
          tv[u] = idx < ntp ? __ldcg(a.ia.tdf + idx) : 0.f;
          pv[u] = (idx < ntp && have_prev) ? __ldcg(a.dn_prev + idx) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
          int idx = base + u * NT + tid;
          bool inb = idx < ntp;
          int y, x;
          divmod(fdt, idx, y, x);
          float d = clamp01(tv[u]);
          float v = pct_flat ? d : clamp01((d - n_lo) / n_den);
          if (inb) {
            a.dn[idx] = v;
            if (y >= th / 4 && y < th * 3 / 4 && x >= tw / 4 && x < tw * 3 / 4) {
              s += (double)v;
              s2 += (double)v * (double)v;
            }
            if (have_prev) mad += (double)fabsf(v - pv[u]);
          }
          bool on = inb && in_region(crop_n, y, x) && subj_keep(v);
          hist_add(S.sh1[0], on, key_of(v) >> 18);
          hist_add(S.sh64[0], on, (uint32_t)bin64(v));
        }
      }
      for (int off = 16; off; off >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, off);
        s2 += __shfl_xor_sync(0xffffffffu, s2, off);
        mad += __shfl_xor_sync(0xffffffffu, mad, off);
      }
      if ((tid & 31) == 0) {
        S.red[0][tid >> 5] = s;
        S.red[1][tid >> 5] = s2;
        S.red[2][tid >> 5] = mad;
      }
      __syncthreads();
      if (tid < 3) {
        double t = 0;
        for (int i = 0; i < NT / 32; ++i) t += S.red[tid][i];
        double* dst = tid == 0 ? &a.fs->sum : (tid == 1 ? &a.fs->sumsq : &a.fs->mad_sum);
        if (t != 0.0) atomicAdd(dst, t);
      }
    }
    flush_pass1(S, 0, a.jm[1], true);
    grid_barrier(a.bar, epoch);

    // ===== subject estimate of the normalised plane, pass 2 -- shares its phase with d0 below: d0 only needs dn,
    // ===== not the scalars of fin_norm, so the two selects interleave and two grid barriers disappear
    after_pass1(S, S.sel[2], a.jm[1], true);
    select_pass<2>(a.dn, a.ia.tw, a.ia.th, nullptr, nullptr, &S.sel[2], &a.jm[1], crop_n);
  }

  // ================= d0 = clamp01(enhance_curvature(resize(depth))) + pass 1 of q(.05/.95) and of the subject =====
  zero_pass1(S);
  {
    const int n = W * H;
    const FastDiv fdw = fast_div((uint32_t)W, (uint32_t)n);
    for (int base = blockIdx.x * (NT * UNR); base < n; base += gridDim.x * (NT * UNR)) {
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        int idx = base + u * NT + tid;
        bool inb = idx < n;
        int y, x;
        divmod(fdw, idx, y, x);
        float v = 0.f;
        if (inb) {
          float d = ldcg_bilinear(a.core_depth, a.sh, a.sw, H, W, y, x);
          float xx = a.xs[x], yy = a.ys[y];
          float r2 = (xx * xx) + (yy * yy);
          float curv = 1.0f - r2;
          d = d + (curv * 0.08f);
          v = clamp01(d);
          a.d[idx] = v;
        }
        uint32_t key = key_of(v);
        hist_add(S.sh1[0], inb, key >> 18);
        bool on = inb && in_region(crop_d, y, x) && subj_keep(v);
        hist_add(S.sh1[1], on, key >> 18);
        hist_add(S.sh64[1], on, (uint32_t)bin64(v));
      }
    }
  }
  __syncthreads();
  flush_pass1(S, 0, a.jm[2], false);
  flush_pass1(S, 1, a.jm[3], true);
  grid_barrier(a.bar, epoch);

  if (a.loop) {  // subject estimate of the normalised plane, pass 3
    after_pass2(S, S.sel[2], a.jm[1]);
    select_pass<3>(a.dn, a.ia.tw, a.ia.th, nullptr, nullptr, &S.sel[2], &a.jm[1], crop_n);
  }
  if (tid < 4) S.sel[0].rank[tid] = a.q_rank[tid];
  __syncthreads();
  after_pass1(S, S.sel[0], a.jm[2], false);
  after_pass1(S, S.sel[1], a.jm[3], true);
  select_pass<2>(a.d, W, H, &S.sel[0], &a.jm[2], &S.sel[1], &a.jm[3], crop_d);
  grid_barrier(a.bar, epoch);
  if (a.loop) {  // ShiftSmoother / dynamic scale / FocalDepthTracker / bars: the scalars of the loop level
    after_pass3(S, S.sel[2], a.jm[1]);
    float sd = subject_of(S, S.sel[2], a.jm[1]);
    if (tid == 0) {
      S.fs.sum = __ldcg(&a.fs->sum);
      S.fs.sumsq = __ldcg(&a.fs->sumsq);
      S.fs.mad_sum = __ldcg(&a.fs->mad_sum);
      fin_norm_core(sd, a.la, &S.st, &S.fs);
    }
    __syncthreads();
  }
  after_pass2(S, S.sel[0], a.jm[2]);
  after_pass2(S, S.sel[1], a.jm[3]);
  select_pass<3>(a.d, W, H, &S.sel[0], &a.jm[2], &S.sel[1], &a.jm[3], crop_d);
  grid_barrier(a.bar, epoch);

  // ================= shape_depth_for_pop (in place) + pass 1 of the subject estimate of the shaped plane ===========
  after_pass3(S, S.sel[0], a.jm[2]);
  after_pass3(S, S.sel[1], a.jm[3]);
  {
    float subj = subject_of(S, S.sel[1], a.jm[3]);
    if (tid == 0) {
      const SelState& q = S.sel[0];
      fin_d0_core(subj, __uint_as_float(q.bits[0]), __uint_as_float(q.bits[1]), __uint_as_float(q.bits[2]),
                  __uint_as_float(q.bits[3]), a.q_wlo, a.q_whi, &S.fs);
    }
  }
  zero_pass1(S);
  {
    const int n = W * H;
    const int st_flat = S.fs.st_flat;
    const float st_lo = S.fs.st_lo, st_den = S.fs.st_den, st_subj = S.fs.st_subj;
    const float mid = (float)a.sa.p.depth_pop_mid, gamma = (float)a.sa.p.depth_pop_gamma;
    const FastDiv fdw = fast_div((uint32_t)W, (uint32_t)n);
    for (int base = blockIdx.x * (NT * UNR); base < n; base += gridDim.x * (NT * UNR)) {
      float dv[UNR];
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        int idx = base + u * NT + tid;
        dv[u] = idx < n ? __ldcg(a.d + idx) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        int idx = base + u * NT + tid;
        bool inb = idx < n;
        int y, x;
        divmod(fdw, idx, y, x);
        float v = dv[u];
        float ds = st_flat ? v : clamp01((v - st_lo) / st_den);
        float centered = (ds - st_subj) + mid;
        float xr = centered - mid;
        float ax = fabsf(xr);
        // |x|^gamma = 2^(gamma*log2|x|) on the SFU: <= ~3e-7 relative (exact path: fp64 pow, one rounding)
        float pw = (ax > 0.f) ? exp2f(gamma * __log2f(ax)) : (gamma == 0.f ? 1.f : 0.f);
        float sg = (xr > 0.f) ? 1.f : ((xr < 0.f) ? -1.f : 0.f);
        float o = clamp01((sg * pw) + mid);
        if (inb) a.d[idx] = o;
        bool on = inb && in_region(crop_d, y, x) && subj_keep(o);
        hist_add(S.sh1[0], on, key_of(o) >> 18);
        hist_add(S.sh64[0], on, (uint32_t)bin64(o));
      }
    }
  }
  __syncthreads();
  flush_pass1(S, 0, a.jm[4], true);
  grid_barrier(a.bar, epoch);

  after_pass1(S, S.sel[1], a.jm[4], true);
  select_pass<2>(a.d, W, H, nullptr, nullptr, &S.sel[1], &a.jm[4], crop_d);
  grid_barrier(a.bar, epoch);
  after_pass2(S, S.sel[1], a.jm[4]);
  select_pass<3>(a.d, W, H, nullptr, nullptr, &S.sel[1], &a.jm[4], crop_d);
  grid_barrier(a.bar, epoch);
  after_pass3(S, S.sel[1], a.jm[4]);
  {
    float subj = subject_of(S, S.sel[1], a.jm[4]);
    if (tid == 0 && blockIdx.x == 0) {
      fin_shape_core(subj, a.sa, &S.st, &S.fs);
      *a.st = S.st;
      *a.fs = S.fs;
    }
  }
}


// ---------------------------------------------------------------------------------------------------------------
// k_shift_fast: shift map + suppress_artifacts_with_edge_mask (core/render_3d.py:198-216, 620-680), fast arithmetic.
// 64 x 16 pixels per CTA (4 per thread), sigmoid through ex2 / rcp approximations, the 5 x 5 pool as row sums then
// column sums.  ~1/3 of the instructions of the one-pixel-per-thread exact kernel (385 thread-instructions per
// pixel, issue bound).
// ---------------------------------------------------------------------------------------------------------------
constexpr int SHX = 64, SHY = 16;
__device__ __forceinline__ float sqrt_approx(float x) {
  float r;
  asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__global__ void __launch_bounds__(256) k_shift_fast(const float* __restrict__ d, float* __restrict__ shift, int H, int W,
                                                    const FrameScalars* __restrict__ fs, int edge_mask, float feather) {
  __shared__ float sd[SHY + 6][SHX + 6 + 2];  // d over [by-3, by+SHY+3) x [bx-3, bx+SHX+3)
  __shared__ float sm[SHY + 4][SHX + 4];      // 1 - sigmoid over [by-2, by+SHY+2) x [bx-2, bx+SHX+2)
  __shared__ float hs[SHY + 4][SHX];          // row sums of 5
  const int bx = blockIdx.x * SHX, by = blockIdx.y * SHY;
  const int tid = threadIdx.x;
  if (edge_mask) {
    for (int i = tid; i < (SHY + 6) * (SHX + 6); i += 256) {
      int ty = i / (SHX + 6), tx = i - ty * (SHX + 6);
      int gy = by - 3 + ty, gx = bx - 3 + tx;
      float v = 0.f;
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = __ldg(d + (size_t)gy * W + gx);
      sd[ty][tx] = v;
    }
    __syncthreads();
    const float f5 = feather * 5.0f;
    for (int i = tid; i < (SHY + 4) * (SHX + 4); i += 256) {
      int ty = i / (SHX + 4), tx = i - ty * (SHX + 4);
      int gy = by - 2 + ty, gx = bx - 2 + tx;
      float m = 0.f;  // zero padding of avg_pool2d
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
        float c = sd[ty + 1][tx + 1];
        float dx = (gx > 0) ? (c - sd[ty + 1][tx]) : 0.f;
        float dy = (gy > 0) ? (c - sd[ty][tx + 1]) : 0.f;
        float g = sqrt_approx((dx * dx) + (dy * dy));
        float t = __expf(-((g - 0.02f) * f5));   // 1 - 1/(1+t) = t/(1+t)
        m = __fdividef(t, 1.0f + t);
        if (!(t < 3.0e38f)) m = 1.0f;             // exp overflow: sigmoid -> 0, mask -> 1
      }
      sm[ty][tx] = m;
    }
    __syncthreads();
    for (int i = tid; i < (SHY + 4) * SHX; i += 256) {
      int r = i / SHX, x = i - r * SHX;
      const float* row = &sm[r][x];
      hs[r][x] = (((row[0] + row[1]) + row[2]) + row[3]) + row[4];
    }
    __syncthreads();
  }
  const float c_fg = fs->c_fg * fs->c_fgm, c_mg = fs->c_mg, c_bg = fs->c_bg * fs->c_bgm;
  const float c_mid = fs->c_mid, c_pb = fs->c_pb, c_half = fs->c_half, c_zpo = fs->c_zpo, c_max = fs->c_max;
  const float c_conv = fs->c_conv, c_m1 = fs->c_m1, c_m2 = fs->c_m2;
  const int use_zpo = fs->use_zpo, use_conv = fs->use_conv;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int i = tid + k * 256;
    const int ly = i / SHX, lx = i - ly * SHX;
    const int x = bx + lx, y = by + ly;
    if (x >= W || y >= H) continue;
    float v = edge_mask ? sd[ly + 3][lx + 3] : __ldg(d + (size_t)y * W + x);
    float o1 = 1.0f - v;
    float fgw = clamp01(o1 * sqrt_approx(o1));
    float mgw = clamp01(1.0f - (fabsf(v - c_mid) * 3.0f));
    float bgw = clamp01(v);
    float raw = ((fgw * c_fg) + (mgw * c_mg)) + (bgw * c_bg);
    float total = (raw * c_pb) / c_half;
    if (use_zpo) total = total - c_zpo;
    total = fminf(fmaxf(total, -c_max), c_max);
    if (use_conv) total = total - c_conv;
    float fin = total;
    if (edge_mask) {
      float acc = (((hs[ly][lx] + hs[ly + 1][lx]) + hs[ly + 2][lx]) + hs[ly + 3][lx]) + hs[ly + 4][lx];
      float sup = total * (acc * (1.0f / 25.0f));
      fin = (c_m1 * total) + (c_m2 * sup);
    }
    shift[(size_t)y * W + x] = fin;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// k_render
// ---------------------------------------------------------------------------------------------------------------
constexpr int RT = 256;           // threads
constexpr int TX = 64, TY = 32;   // eye pixels per tile

template <int K, int FUSE>
struct RenderGeom {
  static constexpr int P = K / 2;
  static constexpr int HL = FUSE ? 1 : 0;
  static constexpr int CX = TX + 2 * HL, CY = TY + 2 * HL;  // composed region (tile + sharpen halo)
  static constexpr int EX = CX + 2 * P, EY = CY + 2 * P;    // edge-mask region
  static constexpr int WX = EX + 1, WY = EY + 1;            // warped-depth region (gradient looks left / up)
  static constexpr int A_BYTES = (K > 0) ? ((WX * WY > EY * CX ? WX * WY : EY * CX) * 8) : 16;
  static constexpr int B_E = (K > 0) ? EX * EY * 8 : 0;
  static constexpr int B_EYE = 2 * CX * CY * 4;
  static constexpr int B_BYTES = B_E > B_EYE ? B_E : B_EYE;
  static constexpr int A_PAD = (A_BYTES + 15) & ~15;
  static constexpr int SMEM = A_PAD + B_BYTES;
};

template <int SRC>
__device__ __forceinline__ void fetch3(const RenderArgs& a, const float* lut, int y, int x, float* rgb) {
  if (SRC == 0) {
    const uint8_t* q = a.c.src_u8 + ((size_t)(a.c.cy0 + y) * a.c.src_pitch + a.c.cx0 + x) * 3;
    rgb[0] = lut[q[2]];
    rgb[1] = lut[q[1]];
    rgb[2] = lut[q[0]];
  } else if (SRC == 1) {
    float4 v = __ldg(a.src_rgbx + (size_t)y * a.c.W + x);
    rgb[0] = v.x;
    rgb[1] = v.y;
    rgb[2] = v.z;
  } else {
    size_t plane = (size_t)a.c.H * a.c.W, o = (size_t)y * a.c.W + x;
    rgb[0] = a.c.src_f32[o];
    rgb[1] = a.c.src_f32[plane + o];
    rgb[2] = a.c.src_f32[2 * plane + o];
  }
}

// K: box size of feather_shift_edges (odd, <= 9; 0 = feathering off).  SRC: 0 = BGR u8 frame, 1 = RGBx float4 plane,
// 2 = planar f32 RGB.  FUSE: 0 = write the two u8 eyes; 1 = bars + sharpen + identity fit + SBS pack;
// 2 = bars + sharpen + 2:1 horizontal INTER_AREA + SBS pack.
template <int K, int SRC, int FUSE>
__global__ void __launch_bounds__(RT) k_render(RenderArgs a) {
  using G = RenderGeom<K, FUSE>;
  constexpr int P = G::P, HL = G::HL, CX = G::CX, CY = G::CY, EX = G::EX, EY = G::EY, WX = G::WX, WY = G::WY;
  extern __shared__ __align__(16) unsigned char rsm[];
  float2* bufA = reinterpret_cast<float2*>(rsm);                 // warped depths, then row sums
  float2* bufE = reinterpret_cast<float2*>(rsm + G::A_PAD);      // edge mask, then the eye tile
  uchar4* eyes = reinterpret_cast<uchar4*>(rsm + G::A_PAD);      // [2][CY][CX]  (B, G, R, -)
  __shared__ float lut[256];
  const int tid = threadIdx.x;
  lut[tid] = (float)tid / 255.0f;  // == frame_to_tensor's u8 / 255.0f bit for bit
  const int H = a.c.H, W = a.c.W;
  const int bx = blockIdx.x * TX, by = blockIdx.y * TY;
  const float* __restrict__ shift = a.c.shift;
  const float* __restrict__ xs = a.c.xs;
  const float* __restrict__ ys = a.c.ys;

  if (K > 0) {
    // ---- A: warped depth of both eyes (core/render_3d.py:700-701)
    const int wx0 = bx - HL - P - 1, wy0 = by - HL - P - 1;
    for (int i = tid; i < WX * WY; i += RT) {
      int ty = i / WX, tx = i - ty * WX;
      int gy = wy0 + ty, gx = wx0 + tx;
      float2 w = make_float2(0.f, 0.f);
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
        float sv = __ldg(shift + (size_t)gy * W + gx);
        float xv = __ldg(xs + gx), yv = __ldg(ys + gy);
        Tap tl = make_tap(xv + sv, yv, H, W);
        Tap tr = make_tap(xv - sv, yv, H, W);
        w.x = sample_plane(a.d, W, tl);
        w.y = sample_plane(a.d, W, tr);
      }
      bufA[i] = w;
    }
    __syncthreads();
    // ---- B: e = clamp(|grad| * feather_strength, 0, 1) (347-352); zero outside the image (avg_pool2d padding)
    const int ex0 = bx - HL - P, ey0 = by - HL - P;
    for (int i = tid; i < EX * EY; i += RT) {
      int ty = i / EX, tx = i - ty * EX;
      int gy = ey0 + ty, gx = ex0 + tx;
      float2 e = make_float2(0.f, 0.f);
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
        float2 c = bufA[(ty + 1) * WX + tx + 1];
        float2 l = bufA[(ty + 1) * WX + tx];
        float2 u = bufA[ty * WX + tx + 1];
        {
          float dx = (gx > 0) ? (c.x - l.x) : 0.f;
          float dy = (gy > 0) ? (c.x - u.x) : 0.f;
          e.x = clamp01(sqrtf((dx * dx) + (dy * dy)) * a.feather_strength);
        }
        {
          float dx = (gx > 0) ? (c.y - l.y) : 0.f;
          float dy = (gy > 0) ? (c.y - u.y) : 0.f;
          e.y = clamp01(sqrtf((dx * dx) + (dy * dy)) * a.feather_strength);
        }
      }
      bufE[i] = e;
    }
    __syncthreads();
    // ---- C: row sums hs[r][x] = sum_{dx<K} e[r][x+dx]  (bufA is free again)
    for (int i = tid; i < EY * CX; i += RT) {
      int r = i / CX, x = i - r * CX;
      const float2* row = bufE + r * EX + x;
      float2 s = row[0];
#pragma unroll
      for (int dx = 1; dx < K; ++dx) {
        float2 v = row[dx];
        s.x = s.x + v.x;
        s.y = s.y + v.y;
      }
      bufA[i] = s;
    }
    __syncthreads();
  } else {
    __syncthreads();  // lut
  }

  // bars of the floating window (apply_side_mask, 885-892; both eyes)
  int bar_lo = 0, bar_hi = 0;
  if (FUSE && a.fs) {
    int bw = a.fs->bar_width;
    if (a.fs->bar_side == 1) {
      bar_lo = W - bw;
      bar_hi = W;
    } else if (a.fs->bar_side == 2) {
      bar_lo = 0;
      bar_hi = bw;
    }
  }

  // ---- D: column sums -> blend weight; 4-tap RGB gather for both eyes; blend; truncate; grade -> eye tile
  const int cx0 = bx - HL, cy0 = by - HL;
  constexpr float kk = (float)(K > 0 ? K * K : 1);
  for (int i = tid; i < CX * CY; i += RT) {
    int ty = i / CX, tx = i - ty * CX;
    int gy = cy0 + ty, gx = cx0 + tx;
    uchar4 ol = make_uchar4(0, 0, 0, 0), orr = make_uchar4(0, 0, 0, 0);
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
      float bl = 0.f, br = 0.f;
      if (K > 0) {
        const float2* col = bufA + ty * CX + tx;
        float2 s = col[0];
#pragma unroll
        for (int dy = 1; dy < K; ++dy) {
          float2 v = col[dy * CX];
          s.x = s.x + v.x;
          s.y = s.y + v.y;
        }
        bl = s.x / kk;
        br = s.y / kk;
      }
      float sv = __ldg(shift + (size_t)gy * W + gx);
      float xv = __ldg(xs + gx), yv = __ldg(ys + gy);
      Tap tl = make_tap(xv + sv, yv, H, W);
      Tap tr = make_tap(xv - sv, yv, H, W);
      float o[3];
      if (K > 0) fetch3<SRC>(a, lut, gy, gx, o);
      float l00[3], l01[3], l10[3], l11[3];
#pragma unroll
      for (int eye = 0; eye < 2; ++eye) {
        const Tap& t = eye ? tr : tl;
        const float b = eye ? br : bl;
        fetch3<SRC>(a, lut, t.y0, t.x0, l00);
        fetch3<SRC>(a, lut, t.y0, t.x1, l01);
        fetch3<SRC>(a, lut, t.y1, t.x0, l10);
        fetch3<SRC>(a, lut, t.y1, t.x1, l11);
        float c[3];
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
          float s = tap_apply(t, l00[ch], l01[ch], l10[ch], l11[ch]);
          if (K > 0) s = clamp01((s * (1.0f - b)) + (o[ch] * b));
          c[ch] = s;
        }
        uint8_t r8 = trunc_u8(c[0]), g8 = trunc_u8(c[1]), b8 = trunc_u8(c[2]);
        if (a.c.grade) {  // frame_to_tensor -> apply_color_grade -> tensor_to_frame (1373-1386)
          float r = lut[r8], g = lut[g8], bb = lut[b8];
          grade_px(r, g, bb, a.c.sat, a.c.con, a.c.bri);
          r8 = trunc_u8(r);
          g8 = trunc_u8(g);
          b8 = trunc_u8(bb);
        }
        if (FUSE && gx >= bar_lo && gx < bar_hi) r8 = g8 = b8 = 0;
        if (eye)
          orr = make_uchar4(b8, g8, r8, 0);
        else
          ol = make_uchar4(b8, g8, r8, 0);
      }
    }
    eyes[i] = ol;
    eyes[CX * CY + i] = orr;
  }
  __syncthreads();

  // ---- E: write out
  if (FUSE == 0) {
    // the two eyes, BGR interleaved: 4 pixels (12 bytes) per thread and iteration
    for (int i = tid; i < 2 * TY * (TX / 4); i += RT) {
      int eye = i / (TY * (TX / 4));
      int r = i - eye * (TY * (TX / 4));
      int ty = r / (TX / 4), q = r - ty * (TX / 4);
      int gy = by + ty, gx = bx + q * 4;
      if (gy >= H || gx >= W) continue;
      const uchar4* src = eyes + eye * CX * CY + ty * CX + q * 4;
      uint8_t* dst = (eye ? a.c.right : a.c.left) + ((size_t)gy * W + gx) * 3;
      int nv = min(4, W - gx);
      if (nv == 4 && (((uintptr_t)dst) & 3) == 0) {
        uchar4 p0 = src[0], p1 = src[1], p2 = src[2], p3 = src[3];
        uint32_t* d32 = reinterpret_cast<uint32_t*>(dst);
        d32[0] = (uint32_t)p0.x | ((uint32_t)p0.y << 8) | ((uint32_t)p0.z << 16) | ((uint32_t)p1.x << 24);
        d32[1] = (uint32_t)p1.y | ((uint32_t)p1.z << 8) | ((uint32_t)p2.x << 16) | ((uint32_t)p2.y << 24);
        d32[2] = (uint32_t)p2.z | ((uint32_t)p3.x << 8) | ((uint32_t)p3.y << 16) | ((uint32_t)p3.z << 24);
      } else {
        for (int k = 0; k < nv; ++k) {
          uchar4 p = src[k];
          dst[3 * k] = p.x;
          dst[3 * k + 1] = p.y;
          dst[3 * k + 2] = p.z;
        }
      }
    }
  } else {
    // apply_sharpening (717-732: cv2.filter2D u8, REFLECT_101, fma chain, round-half-even) on the eye tile, then the
    // eye fit (1409-1417) and the SBS hstack (837-860)
    constexpr int SXF = (FUSE == 2) ? 2 : 1;     // horizontal INTER_AREA factor
    constexpr int OX = TX / SXF;                 // output pixels per tile row and eye
    const int obx = bx / SXF;
    for (int i = tid; i < 2 * TY * (OX / 4); i += RT) {
      int eye = i / (TY * (OX / 4));
      int r = i - eye * (TY * (OX / 4));
      int ty = r / (OX / 4), q = r - ty * (OX / 4);
      int gy = by + ty;
      int ox = obx + q * 4;  // first of 4 output pixels (per-eye coordinates)
      if (gy >= H || ox >= a.per_eye_w) continue;
      const uchar4* et = eyes + eye * CX * CY;
      const int rym = reflect101(gy - 1, H) - cy0, ryp = reflect101(gy + 1, H) - cy0, ryc = gy - cy0;
      uint8_t o8[12];
      int nv = min(4, a.per_eye_w - ox);
      for (int k = 0; k < nv; ++k) {
        int acc3[3] = {0, 0, 0};
#pragma unroll
        for (int sx = 0; sx < SXF; ++sx) {
          int gx = (ox + k) * SXF + sx;
          int rxc = gx - cx0, rxm = reflect101(gx - 1, W) - cx0, rxp = reflect101(gx + 1, W) - cx0;
          uchar4 up = et[rym * CX + rxc], lf = et[ryc * CX + rxm], ce = et[ryc * CX + rxc], rt = et[ryc * CX + rxp],
                 dn = et[ryp * CX + rxc];
          if (a.sharpen) {
            float f;
            f = __fmaf_rn((float)up.x, a.ke, 0.f);
            f = __fmaf_rn((float)lf.x, a.ke, f);
            f = __fmaf_rn((float)ce.x, a.kc, f);
            f = __fmaf_rn((float)rt.x, a.ke, f);
            f = __fmaf_rn((float)dn.x, a.ke, f);
            acc3[0] += (int)rhe_u8(f);
            f = __fmaf_rn((float)up.y, a.ke, 0.f);
            f = __fmaf_rn((float)lf.y, a.ke, f);
            f = __fmaf_rn((float)ce.y, a.kc, f);
            f = __fmaf_rn((float)rt.y, a.ke, f);
            f = __fmaf_rn((float)dn.y, a.ke, f);
            acc3[1] += (int)rhe_u8(f);
            f = __fmaf_rn((float)up.z, a.ke, 0.f);
            f = __fmaf_rn((float)lf.z, a.ke, f);
            f = __fmaf_rn((float)ce.z, a.kc, f);
            f = __fmaf_rn((float)rt.z, a.ke, f);
            f = __fmaf_rn((float)dn.z, a.ke, f);
            acc3[2] += (int)rhe_u8(f);
          } else {
            acc3[0] += ce.x;
            acc3[1] += ce.y;
            acc3[2] += ce.z;
          }
        }
#pragma unroll
        for (int ch = 0; ch < 3; ++ch)
          o8[3 * k + ch] = (SXF == 1) ? (uint8_t)acc3[ch] : rhe_u8((float)acc3[ch] * 0.5f);  // cv2 INTER_AREA 2:1
      }
      uint8_t* dst = a.out + ((size_t)gy * a.out_w + (size_t)eye * a.per_eye_w + ox) * 3;
      if (nv == 4 && (((uintptr_t)dst) & 3) == 0) {
        uint32_t* d32 = reinterpret_cast<uint32_t*>(dst);
#pragma unroll
        for (int w = 0; w < 3; ++w)
          d32[w] = (uint32_t)o8[4 * w] | ((uint32_t)o8[4 * w + 1] << 8) | ((uint32_t)o8[4 * w + 2] << 16) |
                   ((uint32_t)o8[4 * w + 3] << 24);
      } else {
        for (int k = 0; k < nv * 3; ++k) dst[k] = o8[k];
      }
    }
  }
}

template <int K, int SRC, int FUSE>
cudaError_t render_launch(const RenderArgs& a, cudaStream_t s) {
  using G = RenderGeom<K, FUSE>;
  static bool attr_done = false;
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(k_render<K, SRC, FUSE>, cudaFuncAttributeMaxDynamicSharedMemorySize, G::SMEM);
    if (e != cudaSuccess) return e;
    attr_done = true;
  }
  dim3 g((a.c.W + TX - 1) / TX, (a.c.H + TY - 1) / TY);
  k_render<K, SRC, FUSE><<<g, RT, G::SMEM, s>>>(a);
  return cudaGetLastError();
}

template <int K, int SRC>
cudaError_t render_fuse(const RenderArgs& a, cudaStream_t s) {
  switch (a.fuse) {
    case 0: return render_launch<K, SRC, 0>(a, s);
    case 1: return render_launch<K, SRC, 1>(a, s);
    default: return render_launch<K, SRC, 2>(a, s);
  }
}

template <int K>
cudaError_t render_src(const RenderArgs& a, cudaStream_t s) {
  if (a.c.src_u8) return render_fuse<K, 0>(a, s);
  if (a.src_rgbx) return render_fuse<K, 1>(a, s);
  return render_fuse<K, 2>(a, s);
}

}  // namespace

void launch_shift_fast(const float* d, float* shift, int H, int W, const FrameScalars* fs, int edge_mask, float feather,
                       cudaStream_t s) {
  dim3 g((W + SHX - 1) / SHX, (H + SHY - 1) / SHY);
  k_shift_fast<<<g, 256, 0, s>>>(d, shift, H, W, fs, edge_mask, feather);
}

bool render_supports(int feather, int k) { return !feather || (k >= 1 && k <= 9 && (k & 1)); }

cudaError_t launch_render(const RenderArgs& a, cudaStream_t s) {
  const int k = a.c.feather ? a.c.k : 0;
  switch (k) {
    case 0: return render_src<0>(a, s);
    case 1: return render_src<1>(a, s);
    case 3: return render_src<3>(a, s);
    case 5: return render_src<5>(a, s);
    case 7: return render_src<7>(a, s);
    case 9: return render_src<9>(a, s);
    default: return cudaErrorInvalidValue;
  }
}

// grid of the persistent kernel: one CTA per SM (all co-resident: cooperative launch)
cudaError_t stats_grid(int device, int* blocks) {
  static int cached[64] = {0};
  if (device >= 0 && device < 64 && cached[device]) {
    *blocks = cached[device];
    return cudaSuccess;
  }
  cudaError_t e = cudaFuncSetAttribute(k_stats, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(StatsSmem));
  if (e != cudaSuccess) return e;
  int sms = 0, per = 0;
  if ((e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device)) != cudaSuccess) return e;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, k_stats, NT, sizeof(StatsSmem))) != cudaSuccess) return e;
  if (per < 1) return cudaErrorLaunchOutOfResources;
  *blocks = sms;
  if (device >= 0 && device < 64) cached[device] = sms;
  return cudaSuccess;
}

cudaError_t launch_stats(const StatsArgs& a, int blocks, cudaStream_t s) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.gridDim = dim3(blocks);
  cfg.blockDim = dim3(NT);
  cfg.dynamicSmemBytes = sizeof(StatsSmem);
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative;
  at[0].val.cooperative = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, k_stats, a);
}

}  // namespace vd3d
