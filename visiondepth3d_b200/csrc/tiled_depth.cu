// tiled_depth.cu -- the reference's tiled depth path on the device (core/render_depth.py:102-194): the tile crops fed
// to the depth engine, the Hann-weighted blend of the per-tile predictions and the percentile normalisation to u8.
// Compiled with -fmad=false: every product and sum below is rounded on its own, as numpy's float32 arithmetic is.
#include "dibr_device.cuh"
#include "tiled_launch.h"

namespace vd3d {

namespace {

constexpr int kHistWords = 4 * kSelTargets * 256;  // one 256-bin histogram per radix pass and target
constexpr int kStateWords = 32;                    // prefix[6], remaining rank[6], mode, offset, divisor
constexpr int kFrameWords = kHistWords + kStateWords;

// order-preserving 32-bit key of a float (NaN excluded by the callers)
__device__ __forceinline__ uint32_t fkey(float f) {
  uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float kfloat(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
// np.nan_to_num(d, nan=0.0, posinf=0.0, neginf=0.0)
__device__ __forceinline__ float finite_or0(float v) { return isfinite(v) ? v : 0.0f; }

}  // namespace

__global__ void __launch_bounds__(256) k_tile_gather(const TileJob* __restrict__ jobs, int fw) {
  const TileJob j = jobs[blockIdx.z];
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= j.rw || y >= j.rh) return;
  const uint8_t* src = j.frame + ((size_t)j.yp0 * fw + j.xp0) * 3;
  if (j.rh == j.pch && j.rw == j.pcw) {  // already a multiple of 14: the reference hands the crop over as it is
    const uint8_t* p = src + (size_t)y * fw * 3 + x * 3;
    uint8_t* q = j.crop + ((size_t)y * j.rw + x) * 3;
    q[0] = p[0];
    q[1] = p[1];
    q[2] = p[2];
  } else {
    resize_cubic_u8_px(src, (size_t)fw * 3, j.pch, j.pcw, 3, j.crop, j.rh, j.rw, x, y);
  }
}

__global__ void __launch_bounds__(256) k_tile_blend(const TileJob* __restrict__ jobs, int h, int w, int step, int tile,
                                                    int nx, int ny, float* __restrict__ out,
                                                    uint32_t* __restrict__ mm_keys) {
  const int f = blockIdx.z;
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  uint32_t kmin = 0xffffffffu, kmax = 0u;
  if (x < w && y < h) {
    const TileJob* J = jobs + (size_t)f * nx * ny;
    const int i_lo = y >= tile ? (y - tile) / step + 1 : 0, i_hi = min(y / step, ny - 1);
    const int j_lo = x >= tile ? (x - tile) / step + 1 : 0, j_hi = min(x / step, nx - 1);
    float acc = 0.0f, wacc = 0.0f;
    for (int i = i_lo; i <= i_hi; ++i)
      for (int jj = j_lo; jj <= j_hi; ++jj) {
        const TileJob& t = J[i * nx + jj];
        const int ly = y - t.y0, lx = x - t.x0;
        // center = pred[yc0:yc0+ch, xc0:xc0+cw], indexed in the un-rounded crop's coordinates (as the reference does)
        const float c = t.pred[(size_t)(y - t.yp0) * t.rw + (x - t.xp0)];
        const float wv = t.wgt[(size_t)ly * t.cw + lx];
        acc = acc + c * wv;
        wacc = wacc + wv;
      }
    const float v = acc / fmaxf(wacc, 1e-8f);
    out[((size_t)f * h + y) * w + x] = v;
    if (!isnan(v)) kmin = kmax = fkey(v);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, o));
    kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMin(mm_keys + 2 * f, kmin);
    atomicMax(mm_keys + 2 * f + 1, kmax);
  }
}

__global__ void k_mm_init(uint32_t* mm_keys, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    mm_keys[2 * i] = 0xffffffffu;
    mm_keys[2 * i + 1] = 0u;
  }
}

__global__ void k_keys_to_float(const uint32_t* __restrict__ keys, int count, float* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) out[i] = kfloat(keys[i]);
}

// radix pass `pass` (8 bits from the top) of the six selections of frame blockIdx.y: histogram of the keys that share
// each target's prefix so far
__global__ void __launch_bounds__(256) k_sel_hist(const float* __restrict__ d, int64_t npix, int pass,
                                                  uint32_t* __restrict__ scratch) {
  __shared__ uint32_t sh[kSelTargets][256];
  __shared__ uint32_t pre[kSelTargets];
  const int f = blockIdx.y;
  uint32_t* fw = scratch + (size_t)f * kFrameWords;
  for (int i = threadIdx.x; i < kSelTargets * 256; i += 256) (&sh[0][0])[i] = 0;
  if (threadIdx.x < kSelTargets) pre[threadIdx.x] = fw[kHistWords + threadIdx.x];
  __syncthreads();
  const int shift = 24 - 8 * pass;
  const uint32_t mask = pass ? (0xffffffffu << (shift + 8)) : 0u;
  const float* df = d + (size_t)f * npix;
  const int lane = threadIdx.x & 31;
  // warp-uniform trip count, so every lane takes part in the match below.  Depth values share their top key bytes,
  // so the lanes of a warp mostly hit the same bin: one shared atomic per distinct (target, bin) in the warp.
  for (int64_t base = (int64_t)blockIdx.x * 256 + (threadIdx.x & ~31); base < npix; base += (int64_t)gridDim.x * 256) {
    const int64_t i = base + lane;
    const bool valid = i < npix;
    const uint32_t k = valid ? fkey(finite_or0(df[i])) : 0u;
    const uint32_t bin = (k >> shift) & 255u;
#pragma unroll
    for (int t = 0; t < kSelTargets; ++t) {
      const bool m = valid && ((k ^ pre[t]) & mask) == 0;
      const unsigned peers = __match_any_sync(0xffffffffu, m ? bin : 0x100u + lane);
      if (m && lane == __ffs(peers) - 1) atomicAdd(&sh[t][bin], (uint32_t)__popc(peers));
    }
  }
  __syncthreads();
  uint32_t* gh = fw + pass * kSelTargets * 256;
  for (int i = threadIdx.x; i < kSelTargets * 256; i += 256) {
    const uint32_t v = (&sh[0][0])[i];
    if (v) atomicAdd(gh + i, v);
  }
}

// the bin holding each target's remaining rank: extends the prefix by 8 bits
__global__ void k_sel_pick(int pass, NormArgs a, uint32_t* __restrict__ scratch) {
  const int t = threadIdx.x;
  if (t >= kSelTargets) return;
  uint32_t* fw = scratch + (size_t)blockIdx.x * kFrameWords;
  uint32_t* pre = fw + kHistWords;
  uint32_t* rem = pre + kSelTargets;
  const uint32_t* hist = fw + (pass * kSelTargets + t) * 256;
  uint32_t r = pass ? rem[t] : a.rank[t], cum = 0;
  int b = 0;
  for (; b < 255; ++b) {
    if (cum + hist[b] > r) break;
    cum += hist[b];
  }
  pre[t] |= (uint32_t)b << (24 - 8 * pass);
  rem[t] = r - cum;
}

// numpy's _lerp(a, b, t) in float32: a + (b - a) * t, or b - (b - a) * (1 - t) where t >= 0.5
__device__ __forceinline__ float np_lerp(float a, float b, float t) {
  const float diff = b - a;
  return t >= 0.5f ? b - diff * (1.0f - t) : a + diff * t;
}

// the scalars of _normalize_to_u8: mode 0 percentile clip (offset lo, divisor hi - lo), 1 min-max (offset min, divisor
// float32(max - min + 1e-6) of the float64 operands), 2 flat 128
__global__ void k_norm_finish(NormArgs a, uint32_t* __restrict__ scratch, float* __restrict__ stats) {
  uint32_t* fw = scratch + (size_t)blockIdx.x * kFrameWords;
  const uint32_t* pre = fw + kHistWords;
  const float lo = np_lerp(kfloat(pre[0]), kfloat(pre[1]), a.gamma_lo);
  const float hi = np_lerp(kfloat(pre[2]), kfloat(pre[3]), a.gamma_hi);
  const float mn = kfloat(pre[4]), mx = kfloat(pre[5]);
  int mode = 0;
  float off = lo, div = hi - lo;
  if (hi - lo < 1e-6f) {
    const double dmn = mn, dmx = mx;
    if (dmx - dmn < 1e-6) {
      mode = 2;
    } else {
      mode = 1;
      off = mn;
      div = (float)(dmx - dmn + 1e-6);
    }
  }
  fw[kHistWords + 12] = (uint32_t)mode;
  fw[kHistWords + 13] = __float_as_uint(off);
  fw[kHistWords + 14] = __float_as_uint(div);
  if (stats) {
    float* st = stats + 4 * blockIdx.x;
    st[0] = lo;
    st[1] = hi;
    st[2] = mn;
    st[3] = mx;
  }
}

__global__ void __launch_bounds__(256) k_norm_u8(const float* __restrict__ d, int64_t npix,
                                                 const uint32_t* __restrict__ scratch, int invert,
                                                 uint8_t* __restrict__ u8) {
  const int f = blockIdx.y;
  const uint32_t* st = scratch + (size_t)f * kFrameWords + kHistWords;
  const int mode = (int)st[12];
  const float off = __uint_as_float(st[13]), div = __uint_as_float(st[14]);
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < npix; i += (int64_t)gridDim.x * 256) {
    const float v = finite_or0(d[(size_t)f * npix + i]);
    int q = 128;
    if (mode == 0) {
      float t = (v - off) / div;
      t = t < 0.0f ? 0.0f : (t > 1.0f ? 1.0f : t);  // np.clip: NaN stays NaN
      q = (uint8_t)(int)(t * 255.0f);
    } else if (mode == 1) {
      q = (uint8_t)(int)(((v - off) / div) * 255.0f);
    }
    u8[(size_t)f * npix + i] = (uint8_t)(invert ? 255 - q : q);
  }
}

static int grid_for(int64_t n) {
  int64_t b = (n + 4095) / 4096;
  return (int)(b < 1 ? 1 : (b > 264 ? 264 : b));
}

void launch_tile_gather(const TileJob* jobs, int njobs, int max_rh, int max_rw, int fw, cudaStream_t s) {
  constexpr int kMaxZ = 65535;  // gridDim.z limit: small tiles on large batches make more jobs than that
  for (int j0 = 0; j0 < njobs; j0 += kMaxZ) {
    dim3 g((max_rw + 31) / 32, (max_rh + 7) / 8, njobs - j0 < kMaxZ ? njobs - j0 : kMaxZ);
    k_tile_gather<<<g, 256, 0, s>>>(jobs + j0, fw);
  }
}

void launch_tile_blend(const TileJob* jobs, int n, int h, int w, int step, int tile, int nx, int ny, float* out,
                       uint32_t* mm_keys, cudaStream_t s) {
  k_mm_init<<<(n + 127) / 128, 128, 0, s>>>(mm_keys, n);
  dim3 g((w + 31) / 32, (h + 7) / 8, n);
  k_tile_blend<<<g, 256, 0, s>>>(jobs, h, w, step, tile, nx, ny, out, mm_keys);
}

void launch_keys_to_float(const uint32_t* keys, int count, float* out, cudaStream_t s) {
  k_keys_to_float<<<(count + 127) / 128, 128, 0, s>>>(keys, count, out);
}

size_t normalize_scratch_words() { return kFrameWords; }

void launch_normalize_u8(const float* d, int n, int64_t npix, const NormArgs& a, uint32_t* scratch, uint8_t* u8,
                         float* stats, cudaStream_t s) {
  cudaMemsetAsync(scratch, 0, (size_t)n * kFrameWords * 4, s);
  dim3 g(grid_for(npix), n);
  for (int pass = 0; pass < 4; ++pass) {
    k_sel_hist<<<g, 256, 0, s>>>(d, npix, pass, scratch);
    k_sel_pick<<<n, 32, 0, s>>>(pass, a, scratch);
  }
  k_norm_finish<<<n, 1, 0, s>>>(a, scratch, stats);
  k_norm_u8<<<g, 256, 0, s>>>(d, npix, scratch, a.invert, u8);
}

}  // namespace vd3d
