// letterbox.cu -- the pixel work of the reference's LetterboxTracker (core/render_depth.py:273-392) and of the depth
// re-pad of process_video2 (1919-1933), on the GPU.  Only a handful of scalars per frame go back to the host, where
// the tracker's decisions are made.
//
// Per-row float32 statistics equal numpy's bit for bit.  numpy reduces a contiguous float32 axis by pairwise
// summation: below 8 elements a plain loop, up to 128 elements eight interleaved accumulators, above that a split at
// n/2 rounded down to a multiple of 8.  A warp evaluates the <= 128-element leaves of that tree in parallel and one
// lane combines them along the fixed tree.  Products and sums are spelled __fmul_rn / __fadd_rn, so no contraction
// can change a rounding (the unit is also compiled with -fmad=false).
//
// Canny follows cv2.Canny(gray, low, high, apertureSize=3, L2gradient=True): replicated-border Sobel, integer
// squared magnitude, cv2's fixed-point tan(22.5 deg) non-maximum suppression, then hysteresis.  Hysteresis keeps every
// above-low survivor that is 8-connected to an above-high one; it is a connected-components problem, solved with a
// lock-free union-find (atomicMin on the parent array) in a fixed number of launches.
#include <cuda_runtime.h>
#include <stdint.h>

#include "letterbox_launch.h"

namespace vd3d {

namespace {

constexpr int kPwBlock = 128;     // numpy PW_BLOCKSIZE
constexpr int kMaxLeaves = 256;   // leaves of a node of <= 8192 elements (each leaf holds > 56 of them)
constexpr int kRowWarps = 2;      // rows per block of k_lb_rows

// leaves (start, length) of numpy's pairwise tree over n elements, left to right
__device__ int pw_leaves(int n, int* ls, int* ll) {
  int ss[32], sn[32];
  int d = 1, cnt = 0;
  ss[0] = 0;
  sn[0] = n;
  while (d) {
    --d;
    const int s0 = ss[d], m = sn[d];
    if (m <= kPwBlock) {
      ls[cnt] = s0;
      ll[cnt] = m;
      ++cnt;
      continue;
    }
    int m2 = m / 2;
    m2 -= m2 % 8;
    ss[d] = s0 + m2;  // right child below the left one: the left pops first
    sn[d] = m - m2;
    ++d;
    ss[d] = s0;
    sn[d] = m2;
    ++d;
  }
  return cnt;
}

// one leaf: numpy's pairwise_sum for n <= 128
__device__ float pw_leaf(const float* a, int n) {
  if (n < 8) {
    float r = 0.f;
    for (int i = 0; i < n; ++i) r = __fadd_rn(r, a[i]);
    return r;
  }
  float r0 = a[0], r1 = a[1], r2 = a[2], r3 = a[3], r4 = a[4], r5 = a[5], r6 = a[6], r7 = a[7];
  int i;
  for (i = 8; i < n - (n % 8); i += 8) {
    r0 = __fadd_rn(r0, a[i + 0]);
    r1 = __fadd_rn(r1, a[i + 1]);
    r2 = __fadd_rn(r2, a[i + 2]);
    r3 = __fadd_rn(r3, a[i + 3]);
    r4 = __fadd_rn(r4, a[i + 4]);
    r5 = __fadd_rn(r5, a[i + 5]);
    r6 = __fadd_rn(r6, a[i + 6]);
    r7 = __fadd_rn(r7, a[i + 7]);
  }
  float res = __fadd_rn(__fadd_rn(__fadd_rn(r0, r1), __fadd_rn(r2, r3)), __fadd_rn(__fadd_rn(r4, r5), __fadd_rn(r6, r7)));
  for (; i < n; ++i) res = __fadd_rn(res, a[i]);
  return res;
}

// the pairwise tree over n elements whose nodes of <= t elements are already summed (vals, left to right)
__device__ float pw_combine(int64_t n, int64_t t, const float* vals) {
  int64_t rn[48];
  float lv[48];
  bool right[48];
  int d = 0, k = 0;
  int64_t m = n;
  for (;;) {
    while (m > t) {
      int64_t m2 = m / 2;
      m2 -= m2 % 8;
      rn[d] = m - m2;
      right[d] = false;
      ++d;
      m = m2;
    }
    float v = vals[k++];
    for (;;) {
      if (d == 0) return v;
      if (!right[d - 1]) {
        right[d - 1] = true;
        lv[d - 1] = v;
        m = rn[d - 1];
        break;
      }
      v = __fadd_rn(lv[d - 1], v);
      --d;
    }
  }
}

// numpy's mean division: float32 sum / intp count is evaluated in float64 and stored back to float32
__device__ __forceinline__ float np_div(float sum, int64_t n) {
  return __double2float_rn(__ddiv_rn((double)sum, (double)n));
}

// numpy 2: 0.2126 * r + 0.7152 * g + 0.0722 * b on float32 planes (each constant rounded to float32)
__device__ __forceinline__ float luma709(int b, int g, int r) {
  return __fadd_rn(__fadd_rn(__fmul_rn(0.2126f, (float)r), __fmul_rn(0.7152f, (float)g)), __fmul_rn(0.0722f, (float)b));
}

// cv2 COLOR_BGR2GRAY on u8 (15-bit fixed point)
__device__ __forceinline__ int gray_cv(int b, int g, int r) { return (b * 3735 + g * 19235 + r * 9798 + (1 << 14)) >> 15; }

// S of cv2 COLOR_BGR2HSV on u8: sdiv_table[v] = round((255 << 12) / v) (no ties occur for v <= 255)
__device__ __forceinline__ int sat_cv(int b, int g, int r) {
  const int v = max(b, max(g, r)), diff = v - min(b, min(g, r));
  const int sdiv = v ? (2 * (255 << 12) + v) / (2 * v) : 0;
  return (diff * sdiv + (1 << 11)) >> 12;
}

struct RowSmem {
  int ls[kMaxLeaves], ll[kMaxLeaves + 1];
  float lv[kMaxLeaves];
  uint32_t hist[64];
  float bcast;
};

// one warp per row: pairwise mean/var of the luma, saturation sum, gray plane + histogram + |gray - prev gray|
__global__ void __launch_bounds__(32 * kRowWarps) k_lb_rows(LbRowArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t per_warp = sizeof(RowSmem) + (((size_t)a.w * 4 + 15) & ~(size_t)15);
  RowSmem& S = *reinterpret_cast<RowSmem*>(smem + warp * per_warp);
  float* luma = reinterpret_cast<float*>(smem + warp * per_warp + sizeof(RowSmem));
  const int64_t row = (int64_t)blockIdx.x * kRowWarps + warp;
  if (row >= (int64_t)a.n * a.h) return;
  const int f = (int)(row / a.h), y = (int)(row % a.h), w = a.w;
  const uint8_t* p = a.frames + (size_t)row * w * 3;
  const uint8_t* pf = f > 0 ? a.frames + ((size_t)row - a.h) * w * 3 : nullptr;
  const uint8_t* pg = (f == 0 && a.prev_gray) ? a.prev_gray + (size_t)y * w : nullptr;
  for (int j = lane; j < 64; j += 32) S.hist[j] = 0;
  __syncwarp();
  uint32_t s_sum = 0, ad = 0;
  uint8_t* gout = a.gray + (size_t)row * w;
  for (int x = lane; x < w; x += 32) {
    const int b = p[3 * x], g = p[3 * x + 1], r = p[3 * x + 2];
    luma[x] = luma709(b, g, r);
    const int gv = gray_cv(b, g, r);
    gout[x] = (uint8_t)gv;
    atomicAdd(&S.hist[gv >> 2], 1u);
    s_sum += sat_cv(b, g, r);
    if (pf) ad += abs(gv - gray_cv(pf[3 * x], pf[3 * x + 1], pf[3 * x + 2]));
    else if (pg) ad += abs(gv - (int)pg[x]);
  }
  for (int o = 16; o; o >>= 1) {
    s_sum += __shfl_xor_sync(0xffffffffu, s_sum, o);
    ad += __shfl_xor_sync(0xffffffffu, ad, o);
  }
  if (lane == 0) S.ll[0] = pw_leaves(w, S.ls, S.ll + 1);
  __syncwarp();
  // S.ll[0] holds the leaf count, lengths follow at S.ll + 1
  const int cnt = S.ll[0];
  const int* lens = S.ll + 1;
  for (int k = lane; k < cnt; k += 32) S.lv[k] = pw_leaf(luma + S.ls[k], lens[k]);
  __syncwarp();
  if (lane == 0) S.bcast = np_div(pw_combine(w, kPwBlock, S.lv), w);
  __syncwarp();
  const float mean = S.bcast;
  for (int x = lane; x < w; x += 32) {
    const float d = __fsub_rn(luma[x], mean);
    luma[x] = __fmul_rn(d, d);
  }
  __syncwarp();
  for (int k = lane; k < cnt; k += 32) S.lv[k] = pw_leaf(luma + S.ls[k], lens[k]);
  __syncwarp();
  if (lane == 0) {
    a.y_mean[row] = mean;
    a.y_var[row] = np_div(pw_combine(w, kPwBlock, S.lv), w);
    a.s_mean[row] = np_div((float)s_sum, w);  // the saturation sum is an integer below 2^24: exact in float32
    if (pf || pg) atomicAdd(a.absdiff + f, (unsigned long long)ad);
  }
  for (int j = lane; j < 64; j += 32)
    if (S.hist[j]) atomicAdd(a.hist + (size_t)f * 64 + j, S.hist[j]);
}

struct NodeSmem {
  int ls[kMaxLeaves], ll[kMaxLeaves + 1];
  float lv[kMaxLeaves];
  float luma[kLbCutNode];
};

// one warp per (cut node, frame) of the frame-wide pairwise tree
__global__ void __launch_bounds__(32) k_lb_nodes(const uint8_t* __restrict__ frames, int64_t npix,
                                                  const int64_t* __restrict__ node_start, const int* __restrict__ node_len,
                                                  int nodes, float* __restrict__ node_sum) {
  __shared__ NodeSmem S;
  const int lane = threadIdx.x, c = blockIdx.x, f = blockIdx.y;
  const int len = node_len[c];
  const uint8_t* p = frames + ((size_t)f * npix + node_start[c]) * 3;
  for (int i = lane; i < len; i += 32) S.luma[i] = luma709(p[3 * i], p[3 * i + 1], p[3 * i + 2]);
  if (lane == 0) S.ll[0] = pw_leaves(len, S.ls, S.ll + 1);
  __syncwarp();
  const int cnt = S.ll[0];
  for (int k = lane; k < cnt; k += 32) S.lv[k] = pw_leaf(S.luma + S.ls[k], S.ll[1 + k]);
  __syncwarp();
  if (lane == 0) node_sum[(size_t)f * nodes + c] = pw_combine(len, kPwBlock, S.lv);
}

__global__ void k_lb_frame_combine(const float* __restrict__ node_sum, int nodes, int64_t npix, float* __restrict__ y_mean) {
  const int f = blockIdx.x;
  if (threadIdx.x == 0) y_mean[f] = np_div(pw_combine(npix, kLbCutNode, node_sum + (size_t)f * nodes), npix);
}

// ---- Canny ----
struct CannyArgs {
  const uint8_t* gray;
  int h, w, low2, high2;
  int32_t* mag;
  int32_t* label;
  uint8_t* strong;  // [N]
  uint8_t* rflag;   // [N]: the component rooted here holds a strong pixel
  uint8_t* edges;
  int32_t* row_count;
};

__device__ __forceinline__ void sobel3(const uint8_t* g, int h, int w, int x, int y, int& dx, int& dy) {
  const int xm = max(x - 1, 0), xp = min(x + 1, w - 1);
  const uint8_t* r0 = g + (size_t)max(y - 1, 0) * w;
  const uint8_t* r1 = g + (size_t)y * w;
  const uint8_t* r2 = g + (size_t)min(y + 1, h - 1) * w;
  dx = ((int)r0[xp] - r0[xm]) + 2 * ((int)r1[xp] - r1[xm]) + ((int)r2[xp] - r2[xm]);
  dy = ((int)r2[xm] - r0[xm]) + 2 * ((int)r2[x] - r0[x]) + ((int)r2[xp] - r0[xp]);
}

// blockIdx.x: row of the n*h stacked planes, blockIdx.y: 256-column segment
__global__ void __launch_bounds__(256) k_canny_mag(CannyArgs a) {
  const int row = blockIdx.x, x = blockIdx.y * 256 + threadIdx.x;
  if (x >= a.w) return;
  const int f = row / a.h, y = row % a.h;
  int dx, dy;
  sobel3(a.gray + (size_t)f * a.h * a.w, a.h, a.w, x, y, dx, dy);
  a.mag[(size_t)row * a.w + x] = dx * dx + dy * dy;
}

// non-maximum suppression: candidates (above low) get label = own index, others -1
__global__ void __launch_bounds__(256) k_canny_nms(CannyArgs a) {
  const int row = blockIdx.x, x = blockIdx.y * 256 + threadIdx.x;
  if (x >= a.w) return;
  const int f = row / a.h, y = row % a.h, w = a.w;
  const size_t i = (size_t)row * w + x;
  const int m = a.mag[i];
  bool keep = false;
  if (m > a.low2) {
    int xs, ys;
    sobel3(a.gray + (size_t)f * a.h * w, a.h, w, x, y, xs, ys);
    const int32_t* mc = a.mag + (size_t)row * w;
    auto M = [&](int dyo, int xx) -> int {  // zero outside the plane, as cv2's padded magnitude rows
      const int yy = y + dyo;
      if (yy < 0 || yy >= a.h || xx < 0 || xx >= w) return 0;
      return mc[(ptrdiff_t)dyo * w + xx];
    };
    const int ax = abs(xs), ay = abs(ys) << 15;
    const int tg22x = ax * 13573;
    if (ay < tg22x) {
      keep = m > M(0, x - 1) && m >= M(0, x + 1);
    } else {
      const int tg67x = tg22x + (ax << 16);
      if (ay > tg67x) {
        keep = m > M(-1, x) && m >= M(1, x);
      } else {
        const int s = (xs ^ ys) < 0 ? -1 : 1;
        keep = m > M(-1, x - s) && m > M(1, x + s);
      }
    }
  }
  a.label[i] = keep ? (int32_t)i : -1;
  a.strong[i] = keep && m > a.high2;
  a.rflag[i] = 0;
}

__device__ __forceinline__ int uf_find(const int32_t* L, int x) {
  int p = ((volatile const int32_t*)L)[x];
  while (p != x) {
    x = p;
    p = ((volatile const int32_t*)L)[x];
  }
  return x;
}

// parents only decrease, so a stale read still names an ancestor; atomicMin on a root links it to the smaller root
__device__ void uf_unite(int32_t* L, int a, int b) {
  for (;;) {
    a = uf_find(L, a);
    b = uf_find(L, b);
    if (a == b) return;
    if (a > b) {
      const int t = a;
      a = b;
      b = t;
    }
    const int old = atomicMin(L + b, a);
    if (old == b) return;
    b = old;
  }
}

__global__ void __launch_bounds__(256) k_canny_union(CannyArgs a) {
  const int row = blockIdx.x, x = blockIdx.y * 256 + threadIdx.x;
  if (x >= a.w) return;
  const int y = row % a.h, w = a.w;
  const int i = row * w + x;
  if (a.label[i] < 0) return;
  if (x + 1 < w && a.label[i + 1] >= 0) uf_unite(a.label, i, i + 1);
  if (y + 1 < a.h) {
    const int j = i + w;
    if (x > 0 && a.label[j - 1] >= 0) uf_unite(a.label, i, j - 1);
    if (a.label[j] >= 0) uf_unite(a.label, i, j);
    if (x + 1 < w && a.label[j + 1] >= 0) uf_unite(a.label, i, j + 1);
  }
}

__global__ void __launch_bounds__(256) k_canny_compress(CannyArgs a) {
  const int row = blockIdx.x, x = blockIdx.y * 256 + threadIdx.x;
  if (x >= a.w) return;
  const int i = row * a.w + x;
  if (a.label[i] < 0) return;
  const int r = uf_find(a.label, i);
  a.label[i] = r;
  if (a.strong[i]) a.rflag[r] = 1;
}

__global__ void __launch_bounds__(256) k_canny_out(CannyArgs a) {
  const int row = blockIdx.x, x = blockIdx.y * 256 + threadIdx.x;
  const int i = row * a.w + x;
  bool e = false;
  if (x < a.w) {
    const int r = a.label[i];
    e = r >= 0 && a.rflag[r];
    if (a.edges) a.edges[i] = e ? 255 : 0;
  }
  if (a.row_count) {
    const int c = __syncthreads_count(e);
    if (threadIdx.x == 0 && c) atomicAdd(a.row_count + row, c);
  }
}

// ---- re-pad ----
__global__ void __launch_bounds__(256) k_lb_hist(const uint8_t* __restrict__ src, size_t count, uint32_t* __restrict__ hist) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < count; i += (size_t)gridDim.x * 256) atomicAdd(&h[src[i]], 1u);
  __syncthreads();
  if (h[threadIdx.x]) atomicAdd(hist + threadIdx.x, h[threadIdx.x]);
}

// value of rank k (0-based) of the histogram
__device__ int hist_rank(const uint32_t* hist, uint64_t k) {
  uint64_t c = 0;
  for (int v = 0; v < 256; ++v) {
    c += hist[v];
    if (c > k) return v;
  }
  return 255;
}

// int(np.median(core)): for an even count the float mean of the two middle values, truncated
__global__ void __launch_bounds__(256) k_lb_fill(uint8_t* __restrict__ dst, int h, int w, int top, int core_h,
                                                 const uint32_t* __restrict__ hist) {
  __shared__ int neutral;
  if (threadIdx.x == 0) {
    const uint64_t n = (uint64_t)core_h * w;
    neutral = (n & 1) ? hist_rank(hist, n / 2) : (hist_rank(hist, n / 2 - 1) + hist_rank(hist, n / 2)) / 2;
  }
  __syncthreads();
  const size_t bar_top = (size_t)top * w, bot0 = (size_t)(top + core_h) * w, total = (size_t)h * w;
  const size_t nbar = bar_top + (total - bot0);
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < nbar; i += (size_t)gridDim.x * 256)
    dst[i < bar_top ? i : bot0 + (i - bar_top)] = (uint8_t)neutral;
}

int blocks_for(size_t n) {
  size_t b = (n + 255) / 256;
  return (int)(b < 1024 ? (b ? b : 1) : 1024);
}

}  // namespace

void lb_cut_nodes(int64_t n, int64_t* starts, int* lens, int* count, int cap) {
  int64_t ss[64], sn[64];
  int d = 1, cnt = 0;
  ss[0] = 0;
  sn[0] = n;
  while (d) {
    --d;
    const int64_t s0 = ss[d], m = sn[d];
    if (m <= kLbCutNode) {
      if (cnt < cap) {
        starts[cnt] = s0;
        lens[cnt] = (int)m;
      }
      ++cnt;
      continue;
    }
    int64_t m2 = m / 2;
    m2 -= m2 % 8;
    ss[d] = s0 + m2;
    sn[d] = m - m2;
    ++d;
    ss[d] = s0;
    sn[d] = m2;
    ++d;
  }
  *count = cnt;
}

void launch_lb_rows(const LbRowArgs& a, cudaStream_t s) {
  const size_t per_warp = sizeof(RowSmem) + (((size_t)a.w * 4 + 15) & ~(size_t)15);
  const size_t smem = per_warp * kRowWarps;
  cudaFuncSetAttribute(k_lb_rows, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  const int64_t rows = (int64_t)a.n * a.h;
  k_lb_rows<<<(unsigned)((rows + kRowWarps - 1) / kRowWarps), 32 * kRowWarps, smem, s>>>(a);
}

void launch_lb_frame_mean(const uint8_t* frames, int n, int64_t npix, const int64_t* node_start, const int* node_len,
                          int nodes, float* node_sum, float* y_mean, cudaStream_t s) {
  k_lb_nodes<<<dim3(nodes, n), 32, 0, s>>>(frames, npix, node_start, node_len, nodes, node_sum);
  k_lb_frame_combine<<<n, 32, 0, s>>>(node_sum, nodes, npix, y_mean);
}

void launch_canny(const uint8_t* gray, int n, int h, int w, int low2, int high2, int32_t* mag, int32_t* label,
                  uint8_t* flag, uint8_t* edges, int32_t* row_count, cudaStream_t s) {
  CannyArgs a;
  a.gray = gray;
  a.h = h;
  a.w = w;
  a.low2 = low2;
  a.high2 = high2;
  a.mag = mag;
  a.label = label;
  a.strong = flag;
  a.rflag = flag + (size_t)n * h * w;
  a.edges = edges;
  a.row_count = row_count;
  const dim3 grid((unsigned)(n * h), (w + 255) / 256);
  k_canny_mag<<<grid, 256, 0, s>>>(a);
  k_canny_nms<<<grid, 256, 0, s>>>(a);
  k_canny_union<<<grid, 256, 0, s>>>(a);
  k_canny_compress<<<grid, 256, 0, s>>>(a);
  k_canny_out<<<grid, 256, 0, s>>>(a);
}

void launch_lb_pad(uint8_t* dst, int h, int w, int top, int core_h, uint32_t* hist, cudaStream_t s) {
  const size_t core = (size_t)core_h * w;
  k_lb_hist<<<blocks_for(core), 256, 0, s>>>(dst + (size_t)top * w, core, hist);
  k_lb_fill<<<blocks_for((size_t)(h - core_h) * w), 256, 0, s>>>(dst, h, w, top, core_h, hist);
}

}  // namespace vd3d
