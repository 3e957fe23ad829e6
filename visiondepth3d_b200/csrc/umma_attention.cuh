// umma_attention.cuh -- fused multi-head attention for the ViT blocks on Hopper wgmma.
//
//   O[m, :] = softmax_n(q[m] . k[n]) v[n]      head_dim 64, q pre-scaled by 1/sqrt(64)
//
// One CTA per (128-query block, head): two consumer warpgroups own 64 query rows each.  Scores never leave
// the registers: S = Q K^T (wgmma m64n128k16, Q and K from shared memory) is accumulated in registers, the
// online softmax runs on that fragment, and the probabilities are converted in place into f16 A fragments
// of the second wgmma, O += P V (m64n64k16, A from registers, V^T from shared memory).
// Online softmax in log2 units with an exact running maximum per row; each row lives in the four threads of
// a quad, so row reductions are two shuffles.  Probabilities are expressed against (maximum - 8), so they lie in
// (0, 256]: small weights stay out of the f16 subnormal range, and the row sum adds the same f16-rounded values that
// enter P V, so numerator and denominator agree.
//
// warp 0: TMA producer (Q once; K and V^T tiles through a two-deep ring)   warps 4-11: two consumer warpgroups
//
// Replaces Dinov2SelfAttention (transformers 5.5 models/dinov2/modeling_dinov2.py) inside the depth
// forward called from core/render_depth.py:1106-1119.
#pragma once
#include "umma_gemm.cuh"

namespace vd3d {

struct AttnArgs {
  int ntok;     // valid tokens (queries == keys)
  int dmodel;   // row stride of the output (elements)
  __half* out;  // [images * npad, dmodel], head h of image i writes rows i*npad + token, columns [64h, 64h+64)
  int heads;    // blockIdx.y = image * heads + head (the tensor maps' third coordinate)
  int npad;     // rows per image in `out`
};

constexpr int kAttnThreads = 384;
constexpr int kAttnKS = 2;  // K / V^T ring depth (128 keys per stage)
constexpr int kAttnSmem = 16384 /*Q*/ + kAttnKS * (16384 /*K*/ + 16384 /*V^T*/) + 1024 /*align*/ + 256 /*barriers*/;

namespace umma {
// reductions over the four threads of a quad: one fragment row
__device__ __forceinline__ float quad_max(float x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  return fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
}
__device__ __forceinline__ float quad_sum(float x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  return x + __shfl_xor_sync(0xffffffffu, x, 2);
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *(uint32_t*)&h;
}
}  // namespace umma

__global__ void __launch_bounds__(kAttnThreads, 1)
k_umma_attention(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV, const AttnArgs g) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sm = (umma::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = sm, sK = sm + 16384, sV = sK + kAttnKS * 16384;
  const uint32_t bars = sV + kAttnKS * 16384;
  const uint32_t q_full = bars, kv_full = bars + 8, kv_empty = kv_full + 8 * kAttnKS;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qblk = blockIdx.x, zq = blockIdx.y, h = zq % g.heads, img = zq / g.heads;
  const int T = (g.ntok + 127) / 128;

  if (warp == 0 && lane == 0) {
    umma::prefetch_tmap(&tmQ);
    umma::prefetch_tmap(&tmK);
    umma::prefetch_tmap(&tmV);
    umma::mbar_init(q_full, 1);
    for (int i = 0; i < kAttnKS; ++i) {
      umma::mbar_init(kv_full + 8 * i, 1);
      umma::mbar_init(kv_empty + 8 * i, 2);  // one arrive per consumer warpgroup
    }
    umma::fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    if (warp == 0 && lane == 0) {
      umma::mbar_expect_tx(q_full, 16384);
      umma::tma_load_3d(sQ, &tmQ, q_full, 0, qblk * 128, zq);
      for (int t = 0; t < T; ++t) {
        const int ks = t % kAttnKS;
        umma::mbar_wait(kv_empty + 8 * ks, ((t / kAttnKS) & 1) ^ 1);
        const uint32_t fb = kv_full + 8 * ks;
        umma::mbar_expect_tx(fb, 32768);
        umma::tma_load_3d(sK + ks * 16384, &tmK, fb, 0, t * 128, zq);
        const uint32_t dst = sV + ks * 16384;  // V^T: [64 dims][64 keys] twice (keys 0..63, 64..127 of the tile)
        umma::tma_load_3d(dst, &tmV, fb, t * 128, 0, zq);
        umma::tma_load_3d(dst + 8192, &tmV, fb, t * 128 + 64, 0, zq);
      }
    }
    return;
  }

  const int wg = (warp >> 2) - 1;
  const int wq = warp & 3;
  const float L2E = 1.4426950408889634f;
  // this thread's rows of the fragments: 64 wg + 16 wq + lane/4 (+8); its key / dim columns: 8 j + 2 (lane & 3) (+1)
  const int cq = 2 * (lane & 3);
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  umma::mbar_wait(q_full, 0);
  const uint64_t dq = umma::make_desc(sQ + (uint32_t)(wg * 64 * 128));
  for (int t = 0; t < T; ++t) {
    const int ks = t % kAttnKS;
    umma::mbar_wait(kv_full + 8 * ks, (t / kAttnKS) & 1);
    float s[64];
    {
      const uint64_t dk = umma::make_desc(sK + ks * 16384);
      umma::wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) umma::wgmma_m64n128_ss(s, dq + (uint64_t)(2 * k), dk + (uint64_t)(2 * k), k ? 1u : 0u);
      umma::wgmma_commit();
      umma::wgmma_wait<0>();
      umma::fence_regs(s);
    }
    const int nvalid = g.ntok - t * 128;  // keys of this tile that exist
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (nvalid < 128 && 8 * j + cq + (i & 1) >= nvalid) s[4 * j + i] = -INFINITY;
        mx[i >> 1] = fmaxf(mx[i >> 1], s[4 * j + i]);
      }
    float scale[2], mref[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const float m_new = fmaxf(m_run[rr], umma::quad_max(mx[rr]) * L2E);  // tile 0 always holds a valid key: finite
      scale[rr] = umma::ex2_fast(m_run[rr] - m_new);                      // -inf - finite -> 0
      m_run[rr] = m_new;
      mref[rr] = m_new - 8.0f;
    }
    float ls[2] = {0.f, 0.f};
    uint32_t p[32];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float p0 = umma::ex2_fast(fmaf(s[4 * j + 0], L2E, -mref[0]));
      const float p1 = umma::ex2_fast(fmaf(s[4 * j + 1], L2E, -mref[0]));
      const float p2 = umma::ex2_fast(fmaf(s[4 * j + 2], L2E, -mref[1]));
      const float p3 = umma::ex2_fast(fmaf(s[4 * j + 3], L2E, -mref[1]));
      p[2 * j] = umma::pack_h2(p0, p1);      // row r
      p[2 * j + 1] = umma::pack_h2(p2, p3);  // row r + 8
      const float2 h0 = __half22float2(*(const __half2*)&p[2 * j]), h1 = __half22float2(*(const __half2*)&p[2 * j + 1]);
      ls[0] += h0.x + h0.y;
      ls[1] += h1.x + h1.y;
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) l_run[rr] = l_run[rr] * scale[rr] + ls[rr];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[4 * j + 0] *= scale[0];
      o[4 * j + 1] *= scale[0];
      o[4 * j + 2] *= scale[1];
      o[4 * j + 3] *= scale[1];
    }
    // O += P V: k-slice kk covers keys 16 kk .. 16 kk + 15 of the tile; its A fragment is S columns 16 kk + cq (+1)
    // and 16 kk + 8 + cq (+1) of rows r and r + 8 -- the accumulator fragments j = 2 kk and 2 kk + 1
    umma::fence_regs(o);
    umma::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const uint32_t a[4] = {p[4 * kk], p[4 * kk + 1], p[4 * kk + 2], p[4 * kk + 3]};
      const uint64_t db = umma::make_desc(sV + ks * 16384 + (kk >> 2) * 8192) + (uint64_t)(2 * (kk & 3));
      umma::wgmma_m64n64_rs(o, a, db, 1u);
    }
    umma::wgmma_commit();
    umma::wgmma_wait<0>();
    umma::fence_regs(o);
    if ((threadIdx.x & 127) == 0) umma::mbar_arrive(kv_empty + 8 * ks);
  }

  // ---- epilogue: O / sum -> out[m, 64h .. 64h + 63] ----
  float inv[2];
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) inv[rr] = 1.0f / umma::quad_sum(l_run[rr]);
  const int r0 = qblk * 128 + wg * 64 + wq * 16 + (lane >> 2);
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int m = r0 + 8 * rr;
    if (m >= g.ntok) continue;
    __half* dst = g.out + ((size_t)img * g.npad + m) * g.dmodel + h * 64 + cq;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *(uint32_t*)(dst + 8 * j) = umma::pack_h2(o[4 * j + 2 * rr] * inv[rr], o[4 * j + 2 * rr + 1] * inv[rr]);
  }
}

}  // namespace vd3d
