// umma_gemm.cuh -- hand-written sm_90a GEMM on the Hopper tensor cores (wgmma).
//
//   D[M,N] (fp32 in registers) = A[M,K] (f16, K-major) x B[N,K]^T (f16, K-major)
//
// * operands staged by TMA (cp.async.bulk.tensor, 128B swizzle) into a STAGES-deep
//   shared-memory ring guarded by mbarriers; one producer warp issues the loads;
// * two consumer warpgroups each own 64 rows of the 128 x BN tile and issue
//   wgmma.mma_async m64nBNk16 (A and B read from shared memory through matrix descriptors),
//   accumulating in registers; a ring slot is released once the wgmmas reading it retired;
// * the finished accumulator is staged through shared memory and handed (mbarriers) to a
//   dedicated epilogue warpgroup, which runs the fused epilogue (bias, GELU, LayerScale+residual,
//   QKV head split with V transposed, pixel-shuffle for ConvTranspose, ReLU / residual for convs,
//   DPT head) while the consumers already run the next tile's mainloop: a warp per tile row
//   (coalesced) for the token GEMMs, one thread per tile row otherwise.
// * A can also be an NHWC activation read through a 3-D tensor map (C, W, H): the K loop
//   then walks the 3x3 taps and channel blocks (implicit GEMM); out-of-image taps are
//   zero-filled by TMA, so no im2col buffer and no padding copies exist.
//
// Used for the Depth-Anything-V2 forward (the dense contraction of the hot path):
// transformers' DepthAnythingForDepthEstimation as called from core/render_depth.py:1106-1119.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vd3d {

enum Epi : int {
  EPI_F16 = 0,        // out_f16[m, n] = act(acc + bias) (+ res_f16), optional second relu copy
  EPI_F32 = 1,        // out_f32[m, n] = acc (+bias)                       (attention scores)
  EPI_RESID_LS = 2,   // x_f32[m, n] += ls[n] * (acc + bias[n])            (proj / fc2)
  EPI_QKV = 3,        // split heads: q (x scale), k -> [h][m][64]; v -> vT [h][64][m]
  EPI_PATCH = 4,      // x_f32[m+1, n] = acc + bias[n] + pos[m+1, n]       (patch embedding)
  EPI_CONVT = 5,      // ConvTranspose2d(k=s): pixel-shuffle scatter into NHWC f16
  EPI_HEAD = 6,       // depth[m] = relu(s) or head_max * sigmoid(s), s = sum_n relu(acc+bias)[n] * w3[n] + b3
  EPI_SR = 7,         // RRDBNet convs (k_umma_gemm<.., .., true> only): see sr_epilogue_chunk
  EPI_READOUT = 8,    // out_f16[m, n] = GELU(acc + img_bias[m / npad, n])  (DPT project readout, per-image CLS term)
};

struct GemmArgs {
  int M, N, K;            // logical sizes (K = total reduction length)
  int nt, mt, nz;         // tile counts along N, M and batch (filled by launch_gemm)
  int epi;
  int act;                // 0 none, 1 GELU(erf), 2 ReLU, 3 PReLU (slopes in ls)
  // conv mode (implicit GEMM over a (C, W, H) activation map)
  int conv;               // 0 = plain GEMM, 1 = 3x3 pad 1, 2 = 1x1 over the same map
  int cin;                // channels per tap (multiple of 64)
  int imgW, imgH;         // output == input spatial size (stride 1)
  int tw, th;             // pixel tile: tw * th == 128
  // outputs / epilogue operands
  __half* out_f16;
  __half* out2_f16;       // optional relu(out) copy (pre-activation consumers)
  const __half* res_f16;  // optional residual added before the activation
  float* out_f32;
  const float* bias;      // [N] or null
  const float* ls;        // LayerScale lambda [N]
  const float* pos;       // position embeddings [(M+1), N]
  int ldc;                // leading dimension of out (elements)
  long long out_batch_stride;  // per blockIdx.z
  // EPI_QKV
  __half* q;
  __half* k;
  __half* vt;
  int heads, npad, dmodel;
  float qscale;
  // EPI_CONVT
  int ct_k, ct_cout, ct_w;  // kernel(=stride), Cout, input width (tokens per row)
  // EPI_HEAD
  const float* w3;
  const float* b3p;
  float head_max;  // 0: relative head (ReLU); > 0: metric head, max_depth * sigmoid in fp32 with an accurate expf
  // EPI_SR: second scaled residual and the two residual scales (act 4 = LeakyReLU(0.2) there)
  const __half* res2_f16;
  float rs, rs2;
  // EPI_READOUT: [images, N] f32, the image of row m is m / npad (npad = patch rows per image)
  const float* img_bias;
};

namespace umma {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"((uint64_t)tm), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)tm) : "memory");
}

// K-major, 128B-swizzle wgmma matrix descriptor: start>>4 | LBO(=1, unused for swizzled K-major)<<16 |
// SBO(1024 B = 8 rows of 128 B)>>4 <<32 | layout SWIZZLE_128B (1) <<62.  Advancing 16 f16 along K inside the
// swizzle atom adds 32 B (+2 in 16-byte units) to the start address.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across a wgmma_wait
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// eight consecutive accumulator registers as read-write asm operands
#define VD3D_ACC8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                     "+f"(d[i + 6]), "+f"(d[i + 7])
// D[64 x 32] (+)= A[64 x 16] (smem desc) * B[32 x 16]^T (smem desc); both operands K-major
__device__ __forceinline__ void wgmma_m64n32_ss(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, p, 1, 1, 0, 0;\n"
      "}\n"
      : VD3D_ACC8(0), VD3D_ACC8(8)
      : "l"(da), "l"(db), "r"(accumulate));
}
// D[64 x 64] (+)= A[64 x 16] (smem desc) * B[64 x 16]^T (smem desc); both operands K-major
__device__ __forceinline__ void wgmma_m64n64_ss(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n"
      "}\n"
      : VD3D_ACC8(0), VD3D_ACC8(8), VD3D_ACC8(16), VD3D_ACC8(24)
      : "l"(da), "l"(db), "r"(accumulate));
}
// D[64 x 128] (+)= A[64 x 16] (smem desc) * B[128 x 16]^T (smem desc); both operands K-major
__device__ __forceinline__ void wgmma_m64n128_ss(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n"
      "}\n"
      : VD3D_ACC8(0), VD3D_ACC8(8), VD3D_ACC8(16), VD3D_ACC8(24), VD3D_ACC8(32), VD3D_ACC8(40), VD3D_ACC8(48), VD3D_ACC8(56)
      : "l"(da), "l"(db), "r"(accumulate));
}
// D[64 x 64] (+)= A[64 x 16] (f16 registers, accumulator fragment layout) * B[64 x 16]^T (smem desc, K-major)
__device__ __forceinline__ void wgmma_m64n64_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %37, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n"
      "}\n"
      : VD3D_ACC8(0), VD3D_ACC8(8), VD3D_ACC8(16), VD3D_ACC8(24)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
}

// accumulator tile (64 x N) of one warpgroup, K = 16 per instruction, both operands in shared memory
template <int N>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (N == 32) wgmma_m64n32_ss(d, da, db, accumulate);
  else if constexpr (N == 64) wgmma_m64n64_ss(d, da, db, accumulate);
  else wgmma_m64n128_ss(d, da, db, accumulate);
}

__device__ __forceinline__ float ex2_fast(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// GELU(x) = 0.5 x (1 + erf(x / sqrt 2)), exact-erf form as in HF's "gelu".  erfc(z) for z >= 0 from Abramowitz-Stegun
// 7.1.26 (|error| <= 1.5e-7): erfc(z) = t (a1 + t (a2 + t (a3 + t (a4 + t a5)))) exp(-z^2), t = 1 / (1 + p z), and
// GELU(x) = max(x, 0) - 0.5 |x| erfc(|x| / sqrt 2)  (no cancellation for x < 0).  ~14 FP32 ops + 2 MUFU instead of
// the ~45 of erff(): the fc1 epilogue is ALU bound on erff.  Output is stored as f16.
__device__ __forceinline__ float gelu_erf(float x) {
  const float ax = fabsf(x);
  const float z = ax * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  float p = fmaf(t, 1.061405429f, -1.453152027f);
  p = fmaf(t, p, 1.421413741f);
  p = fmaf(t, p, -0.284496736f);
  p = fmaf(t, p, 0.254829592f);
  p *= t;
  const float e = ex2_fast(x * x * -0.72134752044448170368f);  // exp(-x^2 / 2)
  return fmaf(-0.5f * ax * p, e, fmaxf(x, 0.f));
}

// 32-byte global accesses as two 128-bit instructions (the widest Hopper has)
__device__ __forceinline__ void ldg_v8(const void* p, uint32_t (&r)[8]) {
  asm volatile("ld.global.v4.b32 {%0, %1, %2, %3}, [%8];\n\t"
               "ld.global.v4.b32 {%4, %5, %6, %7}, [%8+16];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]), "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7])
               : "l"(p));
}
__device__ __forceinline__ void ldg_nc_v8(const void* p, uint32_t (&r)[8]) {
  asm volatile("ld.global.nc.v4.b32 {%0, %1, %2, %3}, [%8];\n\t"
               "ld.global.nc.v4.b32 {%4, %5, %6, %7}, [%8+16];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]), "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7])
               : "l"(p));
}
__device__ __forceinline__ void stg_v8(void* p, const uint32_t (&r)[8]) {
  asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};\n\t"
               "st.global.v4.b32 [%0+16], {%5, %6, %7, %8};" ::"l"(p), "r"(r[0]), "r"(r[1]), "r"(r[2]),
               "r"(r[3]), "r"(r[4]), "r"(r[5]), "r"(r[6]), "r"(r[7])
               : "memory");
}
// 16 fp32 -> 16 f16 (32 bytes) starting at a[base]
__device__ __forceinline__ void pack16(const float (&a)[32], int base, bool relu, uint32_t (&u)[8]) {
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    float x = a[base + 2 * t], y = a[base + 2 * t + 1];
    if (relu) {
      x = fmaxf(x, 0.f);
      y = fmaxf(y, 0.f);
    }
    __half2 h = __floats2half2_rn(x, y);
    u[t] = *(uint32_t*)&h;
  }
}

}  // namespace umma

// EPI_SR, the epilogue of the RRDBNet convs (a = acc + bias of one 32-column chunk):
//   out_f32 set:  out_f32[m, n] = a                                  (conv_last, ldc floats per row)
//   otherwise:    a = res + rs a (res_f16 set); a = res2 + rs2 a (res2_f16 set); a = LeakyReLU_0.2(a) (act 4);
//                 f16 at out_f16[m, n] (ldc), or with ct_k the pixel-shuffle scatter of EPI_CONVT (nearest x2 + conv
//                 as four phase convs).  The residuals are read at the output's own offset, so out may alias a
//                 residual (the RRDB add writes in place): each element is read and then written by one thread.
__device__ __forceinline__ void sr_epilogue_chunk(const GemmArgs& g, float (&a)[32], const int m, const int n0,
                                                  const int nvalid, const bool full) {
  if (g.out_f32) {
    float* dst = g.out_f32 + (size_t)m * g.ldc + n0;
    if (full && ((((size_t)m * g.ldc + n0) & 3) == 0)) {
#pragma unroll
      for (int j = 0; j < 8; ++j) ((float4*)dst)[j] = make_float4(a[4 * j], a[4 * j + 1], a[4 * j + 2], a[4 * j + 3]);
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j < nvalid) dst[j] = a[j];
    }
    return;
  }
  size_t o;
  if (g.ct_k) {
    const int tap = n0 / g.ct_cout, co = n0 % g.ct_cout;
    const int dy = tap / g.ct_k, dx = tap % g.ct_k;
    const int y = m / g.ct_w, x = m % g.ct_w;
    o = ((size_t)(y * g.ct_k + dy) * (g.ct_w * g.ct_k) + (x * g.ct_k + dx)) * g.ct_cout + co;
  } else {
    o = (size_t)m * g.ldc + n0;
  }
  const bool vec = full && ((o & 15) == 0);
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const __half* res = q == 0 ? g.res_f16 : g.res2_f16;
    if (!res) continue;
    const float sc = q == 0 ? g.rs : g.rs2;
    float rv[32];
    if (vec) {
      uint32_t u[2][8];
      umma::ldg_v8(res + o, u[0]);
      umma::ldg_v8(res + o + 16, u[1]);
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const float2 f = __half22float2(*(const __half2*)&u[j][t]);
          rv[16 * j + 2 * t] = f.x;
          rv[16 * j + 2 * t + 1] = f.y;
        }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) rv[j] = (j < nvalid) ? __half2float(res[o + j]) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) a[j] = rv[j] + sc * a[j];
  }
  if (g.act == 4) {
#pragma unroll
    for (int j = 0; j < 32; ++j) a[j] = a[j] > 0.f ? a[j] : 0.2f * a[j];
  }
  if (vec) {
    uint32_t u[8];
    umma::pack16(a, 0, false, u);
    umma::stg_v8(g.out_f16 + o, u);
    umma::pack16(a, 16, false, u);
    umma::stg_v8(g.out_f16 + o + 16, u);
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j)
      if (j < nvalid) g.out_f16[o + j] = __float2half_rn(a[j]);
  }
}

// EPI_QKV, V columns: 32 values of head dimension d0 .. d0 + 31 of token tok into vT [image][head][64][npad] (zh =
// image * heads + head); transposed, so the lanes of a warp (consecutive rows) write consecutive tokens
__device__ __forceinline__ void qkv_store_vt(const GemmArgs& g, const float (&a)[32], const size_t zh, const int d0,
                                             const int tok) {
  __half* dst = g.vt + (zh * 64 + d0) * g.npad + tok;
#pragma unroll
  for (int j = 0; j < 32; ++j) dst[(size_t)j * g.npad] = __float2half_rn(a[j]);
}

// Fused epilogue of one 32-column chunk of one accumulator row (thread == row): v = raw fp32 accumulator bits,
// m = logical output row, n0 = first output column.  Every
// register array is indexed with compile-time constants only so the chunk stays in registers.  kSr: the RRDBNet
// instantiations, whose only epilogue is EPI_SR (the others compile exactly as without it).
template <bool kSr>
__device__ __forceinline__ void gemm_epilogue_chunk(const GemmArgs& g, const uint32_t (&v)[32], const int m, const int z,
                                                    const int n0, const bool row_ok, float& head_acc) {
  if (!row_ok || n0 >= g.N) return;
  const int nvalid = min(32, g.N - n0);
  const bool full = (nvalid == 32);
  float a[32];
  if (g.bias) {
    if (full) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float4 b4 = __ldg((const float4*)(g.bias + n0) + j);
        a[4 * j + 0] = __uint_as_float(v[4 * j + 0]) + b4.x;
        a[4 * j + 1] = __uint_as_float(v[4 * j + 1]) + b4.y;
        a[4 * j + 2] = __uint_as_float(v[4 * j + 2]) + b4.z;
        a[4 * j + 3] = __uint_as_float(v[4 * j + 3]) + b4.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) a[j] = __uint_as_float(v[j]) + ((j < nvalid) ? g.bias[n0 + j] : 0.f);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j) a[j] = __uint_as_float(v[j]);
  }
  if constexpr (kSr) {
    sr_epilogue_chunk(g, a, m, n0, nvalid, full);
    return;
  }
  switch (g.epi) {
    case EPI_F16: {
      const size_t o = (size_t)z * g.out_batch_stride + (size_t)m * g.ldc + n0;
      const bool vec = full && ((o & 15) == 0);  // 32-byte aligned: 256-bit accesses
      if (g.res_f16) {
        if (vec) {
          uint32_t rv[2][8];
          umma::ldg_nc_v8(g.res_f16 + o, rv[0]);
          umma::ldg_nc_v8(g.res_f16 + o + 16, rv[1]);
#pragma unroll
          for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int t = 0; t < 8; ++t) {
              float2 f = __half22float2(*(const __half2*)&rv[j][t]);
              a[16 * j + 2 * t] += f.x;
              a[16 * j + 2 * t + 1] += f.y;
            }
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (j < nvalid) a[j] += __half2float(g.res_f16[o + j]);
        }
      }
      if (g.act == 1) {
#pragma unroll
        for (int j = 0; j < 32; ++j) a[j] = umma::gelu_erf(a[j]);
      } else if (g.act == 2) {
#pragma unroll
        for (int j = 0; j < 32; ++j) a[j] = fmaxf(a[j], 0.f);
      } else if (g.act == 3) {  // PReLU, per-channel slopes in g.ls (SRVGGNetCompact)
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (j < nvalid) a[j] = a[j] > 0.f ? a[j] : a[j] * __ldg(g.ls + n0 + j);
      }
      if (vec) {
        uint32_t u[8];
        umma::pack16(a, 0, false, u);
        umma::stg_v8(g.out_f16 + o, u);
        umma::pack16(a, 16, false, u);
        umma::stg_v8(g.out_f16 + o + 16, u);
        if (g.out2_f16) {
          umma::pack16(a, 0, true, u);
          umma::stg_v8(g.out2_f16 + o, u);
          umma::pack16(a, 16, true, u);
          umma::stg_v8(g.out2_f16 + o + 16, u);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (j < nvalid) {
            g.out_f16[o + j] = __float2half_rn(a[j]);
            if (g.out2_f16) g.out2_f16[o + j] = __float2half_rn(fmaxf(a[j], 0.f));
          }
      }
    } break;
    case EPI_F32: {
      float* dst = g.out_f32 + (size_t)z * g.out_batch_stride + (size_t)m * g.ldc + n0;
      if (full && ((((size_t)m * g.ldc + n0) & 3) == 0) && ((g.out_batch_stride & 3) == 0)) {
#pragma unroll
        for (int j = 0; j < 8; ++j) ((float4*)dst)[j] = make_float4(a[4 * j], a[4 * j + 1], a[4 * j + 2], a[4 * j + 3]);
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (j < nvalid) dst[j] = a[j];
      }
    } break;
    case EPI_RESID_LS: {
      // read-modify-write of the fp32 residual stream: issue all loads before the first store
      // (a load/store-per-element loop serialises on possible aliasing: ~800 cycles per element);
      // 256-bit accesses: every instruction moves whole 32-byte sectors
      float* dst = g.out_f32 + (size_t)m * g.ldc + n0;
      if (full && ((((size_t)m * g.ldc + n0) & 7) == 0)) {
        uint32_t x8[4][8];
        float4 l4[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) umma::ldg_v8(dst + 8 * j, x8[j]);
#pragma unroll
        for (int j = 0; j < 8; ++j) l4[j] = __ldg((const float4*)(g.ls + n0) + j);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
#pragma unroll
          for (int t = 0; t < 2; ++t) {
            const float4 l = l4[2 * j + t];
            x8[j][4 * t + 0] = __float_as_uint(fmaf(l.x, a[8 * j + 4 * t + 0], __uint_as_float(x8[j][4 * t + 0])));
            x8[j][4 * t + 1] = __float_as_uint(fmaf(l.y, a[8 * j + 4 * t + 1], __uint_as_float(x8[j][4 * t + 1])));
            x8[j][4 * t + 2] = __float_as_uint(fmaf(l.z, a[8 * j + 4 * t + 2], __uint_as_float(x8[j][4 * t + 2])));
            x8[j][4 * t + 3] = __float_as_uint(fmaf(l.w, a[8 * j + 4 * t + 3], __uint_as_float(x8[j][4 * t + 3])));
          }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) umma::stg_v8(dst + 8 * j, x8[j]);
      } else {
        float xv[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) xv[j] = (j < nvalid) ? dst[j] : 0.f;
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (j < nvalid) dst[j] = xv[j] + g.ls[n0 + j] * a[j];
      }
    } break;
    case EPI_QKV: {
      // n0 is a multiple of 32 and head_dim is 64: the 32 columns lie in one (which, head)
      const int which = n0 / g.dmodel;
      const int rem = n0 - which * g.dmodel;
      const int h = rem >> 6, d0 = rem & 63;
      // batched forward: row m = image * npad + token; q, k are [image][head][npad][64], vT [image][head][64][npad]
      const int img = m / g.npad, tok = m - img * g.npad;
      const size_t zh = (size_t)img * g.heads + h;
      if (which < 2) {
        __half* dst = (which == 0 ? g.q : g.k) + (zh * g.npad + tok) * 64 + d0;
        const float sc = which == 0 ? g.qscale : 1.0f;
#pragma unroll
        for (int j = 0; j < 32; ++j) a[j] *= sc;
        uint32_t u[8];
        umma::pack16(a, 0, false, u);
        umma::stg_v8(dst, u);
        umma::pack16(a, 16, false, u);
        umma::stg_v8(dst + 16, u);
      } else {
        qkv_store_vt(g, a, zh, d0, tok);
      }
    } break;
    case EPI_PATCH: {
      float* dst = g.out_f32 + (size_t)(m + 1) * g.ldc + n0;
      const float* pe = g.pos + (size_t)(m + 1) * g.ldc + n0;
      float pv[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) pv[j] = (j < nvalid) ? __ldg(pe + j) : 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j < nvalid) dst[j] = a[j] + pv[j];
    } break;
    case EPI_CONVT: {
      // n = (dy*k + dx)*Cout + co ; m = y*ct_w + x ; out NHWC [(H*k), (W*k), Cout]
      const int tap = n0 / g.ct_cout, co = n0 % g.ct_cout;
      const int dy = tap / g.ct_k, dx = tap % g.ct_k;
      const int y = m / g.ct_w, x = m % g.ct_w;
      size_t o = ((size_t)(y * g.ct_k + dy) * (g.ct_w * g.ct_k) + (x * g.ct_k + dx)) * g.ct_cout + co;
      if (full && ((o & 15) == 0)) {
        uint32_t u[8];
        umma::pack16(a, 0, false, u);
        umma::stg_v8(g.out_f16 + o, u);
        umma::pack16(a, 16, false, u);
        umma::stg_v8(g.out_f16 + o + 16, u);
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (j < nvalid) g.out_f16[o + j] = __float2half_rn(a[j]);
      }
    } break;
    case EPI_HEAD: {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j < nvalid) head_acc += fmaxf(a[j], 0.f) * __ldg(g.w3 + n0 + j);
    } break;
    case EPI_READOUT: {
      // the token half of Linear(cat(tok, cls)) is this GEMM; the CLS half plus the bias arrives per image
      const float* cb = g.img_bias + (size_t)(m / g.npad) * g.N + n0;
      const size_t o = (size_t)m * g.ldc + n0;
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j < nvalid) a[j] = umma::gelu_erf(a[j] + __ldg(cb + j));
      if (full && ((o & 15) == 0)) {
        uint32_t u[8];
        umma::pack16(a, 0, false, u);
        umma::stg_v8(g.out_f16 + o, u);
        umma::pack16(a, 16, false, u);
        umma::stg_v8(g.out_f16 + o + 16, u);
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (j < nvalid) g.out_f16[o + j] = __float2half_rn(a[j]);
      }
    } break;
  }
}

// The row-per-warp epilogue (gemm_epilogue_rows) serves the plain-GEMM epilogues whose global accesses become
// contiguous when a warp walks a row: EPI_RESID_LS, EPI_F16, EPI_QKV and EPI_READOUT.  It is decided per launch:
// 128-column tiles that all lie inside N (N a multiple of 128), no conv row mapping, and every pointer and row pitch
// aligned for the 4-column vectors of a lane.  Every other launch keeps the thread-per-row epilogue.
template <int BN, bool kSr>
__device__ __forceinline__ bool gemm_launch_by_rows(const GemmArgs& g) {
  if constexpr (BN != 128 || kSr) {
    return false;
  } else {
    auto al = [](const void* p, int bytes) { return ((uintptr_t)p & (uintptr_t)(bytes - 1)) == 0; };
    if (g.conv || (g.N & 127) || !al(g.bias, 16)) return false;
    switch (g.epi) {
      case EPI_RESID_LS: return (g.ldc & 3) == 0 && al(g.out_f32, 16) && al(g.ls, 16);
      case EPI_F16:
        return (g.ldc & 3) == 0 && (g.out_batch_stride & 3) == 0 && al(g.out_f16, 8) && al(g.out2_f16, 8) &&
               al(g.res_f16, 8) && (g.act != 3 || al(g.ls, 16));
      case EPI_QKV: return (g.dmodel & 127) == 0 && al(g.q, 8) && al(g.k, 8);
      case EPI_READOUT: return (g.ldc & 3) == 0 && al(g.out_f16, 8) && al(g.img_bias, 16);
      default: return false;
    }
  }
}

// rows per warp in flight: their global loads all issue before the first store (8 do not fit the 120 registers)
constexpr int kEpiRows = 4;

namespace umma {
// 4 fp32 -> 4 f16 (8 bytes), each element rounded on its own as in pack16
__device__ __forceinline__ uint2 pack4(const float4 a) {
  __half2 lo = __floats2half2_rn(a.x, a.y), hi = __floats2half2_rn(a.z, a.w);
  return make_uint2(*(uint32_t*)&lo, *(uint32_t*)&hi);
}
__device__ __forceinline__ float4 lds_f4(const uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ float4 relu4(const float4 a) {
  return make_float4(fmaxf(a.x, 0.f), fmaxf(a.y, 0.f), fmaxf(a.z, 0.f), fmaxf(a.w, 0.f));
}
}  // namespace umma

// Row-per-warp fused epilogue of one 128 x 128 tile of a plain GEMM, every column inside N: warp w of the epilogue
// warpgroup takes tile rows w, w + 4, ..., w + 124, lane l columns 4 l .. 4 l + 3.  A staging read is one contiguous
// 512-byte row (conflict-free at pitch 132), the bias / LayerScale of the lane's columns are loaded once per tile, and a
// warp's global access is one contiguous piece of an output row: 512 bytes of the fp32 residual, 256 bytes of an f16
// output, two 128-byte head rows of q or k (where a thread per row touched 32 rows per instruction).  Rows come in
// groups of kEpiRows whose global loads are issued before the group's first store.  The arithmetic per element is that
// of gemm_epilogue_chunk (same operations, same order, same roundings), so both paths write the same bits.
__device__ __forceinline__ void gemm_epilogue_rows(const GemmArgs& g, const float* tile, const int pitch,
                                                   const int m_blk, const int n_blk, const int z) {
  const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int n = n_blk * 128 + 4 * lane;
  const int nrows = min(128, g.M - m_blk * 128);  // rows of the tile inside M
  const size_t row0 = (size_t)m_blk * 128;
  const uint32_t srow = umma::smem_u32(tile) + 16 * lane;
  const float4 b4 = g.bias ? __ldg((const float4*)(g.bias + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
  // acc (+ bias) of the lane's 4 columns of tile row r; without a bias the accumulator is taken as it is
  auto row_acc = [&](const int r) {
    float4 a = umma::lds_f4(srow + r * pitch * 4);
    if (g.bias) {
      a.x += b4.x;
      a.y += b4.y;
      a.z += b4.z;
      a.w += b4.w;
    }
    return a;
  };
  switch (g.epi) {
    case EPI_RESID_LS: {
      const float4 l4 = __ldg((const float4*)(g.ls + n));
      float* const x0 = g.out_f32 + n;
#pragma unroll 1
      for (int r0 = w; r0 < nrows; r0 += 4 * kEpiRows) {
        float4 x[kEpiRows];
#pragma unroll
        for (int i = 0; i < kEpiRows; ++i)
          if (r0 + 4 * i < nrows) x[i] = *(const float4*)(x0 + (row0 + r0 + 4 * i) * g.ldc);
#pragma unroll
        for (int i = 0; i < kEpiRows; ++i) {
          if (r0 + 4 * i >= nrows) break;
          const float4 a = row_acc(r0 + 4 * i);
          x[i].x = fmaf(l4.x, a.x, x[i].x);
          x[i].y = fmaf(l4.y, a.y, x[i].y);
          x[i].z = fmaf(l4.z, a.z, x[i].z);
          x[i].w = fmaf(l4.w, a.w, x[i].w);
          *(float4*)(x0 + (row0 + r0 + 4 * i) * g.ldc) = x[i];
        }
      }
    } break;
    case EPI_F16: {
      const float4 s4 = g.act == 3 ? __ldg((const float4*)(g.ls + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
      const size_t o0 = (size_t)z * g.out_batch_stride + n;
#pragma unroll 1
      for (int r0 = w; r0 < nrows; r0 += 4 * kEpiRows) {
        uint2 rv[kEpiRows];
        if (g.res_f16) {
#pragma unroll
          for (int i = 0; i < kEpiRows; ++i)
            if (r0 + 4 * i < nrows) rv[i] = __ldg((const uint2*)(g.res_f16 + o0 + (row0 + r0 + 4 * i) * g.ldc));
        }
#pragma unroll
        for (int i = 0; i < kEpiRows; ++i) {
          if (r0 + 4 * i >= nrows) break;
          const size_t o = o0 + (row0 + r0 + 4 * i) * g.ldc;
          float4 a = row_acc(r0 + 4 * i);
          if (g.res_f16) {
            const float2 f0 = __half22float2(*(const __half2*)&rv[i].x), f1 = __half22float2(*(const __half2*)&rv[i].y);
            a.x += f0.x;
            a.y += f0.y;
            a.z += f1.x;
            a.w += f1.y;
          }
          if (g.act == 1) {
            a = make_float4(umma::gelu_erf(a.x), umma::gelu_erf(a.y), umma::gelu_erf(a.z), umma::gelu_erf(a.w));
          } else if (g.act == 2) {
            a = umma::relu4(a);
          } else if (g.act == 3) {
            a.x = a.x > 0.f ? a.x : a.x * s4.x;
            a.y = a.y > 0.f ? a.y : a.y * s4.y;
            a.z = a.z > 0.f ? a.z : a.z * s4.z;
            a.w = a.w > 0.f ? a.w : a.w * s4.w;
          }
          *(uint2*)(g.out_f16 + o) = umma::pack4(a);
          if (g.out2_f16) *(uint2*)(g.out2_f16 + o) = umma::pack4(umma::relu4(a));
        }
      }
    } break;
    case EPI_QKV: {
      const int which = n_blk * 128 / g.dmodel;
      if (which == 2) {
        // V: thread t keeps tile row t, whose transposed stores are already coalesced across the lanes
        const int r = threadIdx.x & 127;
        if (r >= nrows) break;
        const int m = m_blk * 128 + r, img = m / g.npad, tok = m - img * g.npad;
#pragma unroll 1
        for (int ci = 0; ci < 4; ++ci) {
          const int n0 = n_blk * 128 + 32 * ci;
          float a[32];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            float4 f = umma::lds_f4(umma::smem_u32(tile + r * pitch + 32 * ci + 4 * i));
            if (g.bias) {
              const float4 bb = __ldg((const float4*)(g.bias + n0) + i);
              f.x += bb.x;
              f.y += bb.y;
              f.z += bb.z;
              f.w += bb.w;
            }
            a[4 * i] = f.x;
            a[4 * i + 1] = f.y;
            a[4 * i + 2] = f.z;
            a[4 * i + 3] = f.w;
          }
          const int rem = n0 - 2 * g.dmodel;
          qkv_store_vt(g, a, (size_t)img * g.heads + (rem >> 6), rem & 63, tok);
        }
        break;
      }
      // q or k: the tile's 128 columns are heads h0 and h0 + 1, lanes 0-15 write 128 contiguous bytes of a row of head
      // h0, lanes 16-31 of head h0 + 1
      const int h = (n_blk * 128 - which * g.dmodel + 4 * lane) >> 6, d0 = (4 * lane) & 63;
      __half* const base = which == 0 ? g.q : g.k;
      const float sc = which == 0 ? g.qscale : 1.0f;
#pragma unroll 4
      for (int r = w; r < nrows; r += 4) {
        const int m = m_blk * 128 + r;
        const int img = m / g.npad, tok = m - img * g.npad;
        float4 a = row_acc(r);
        a.x *= sc;
        a.y *= sc;
        a.z *= sc;
        a.w *= sc;
        *(uint2*)(base + (((size_t)img * g.heads + h) * g.npad + tok) * 64 + d0) = umma::pack4(a);
      }
    } break;
    case EPI_READOUT: {
#pragma unroll 1
      for (int r0 = w; r0 < nrows; r0 += 4 * kEpiRows) {
        float4 cb[kEpiRows];
#pragma unroll
        for (int i = 0; i < kEpiRows; ++i)
          if (r0 + 4 * i < nrows)
            cb[i] = __ldg((const float4*)(g.img_bias + (size_t)((m_blk * 128 + r0 + 4 * i) / g.npad) * g.N + n));
#pragma unroll
        for (int i = 0; i < kEpiRows; ++i) {
          if (r0 + 4 * i >= nrows) break;
          const float4 a = row_acc(r0 + 4 * i);
          const float4 y = make_float4(umma::gelu_erf(a.x + cb[i].x), umma::gelu_erf(a.y + cb[i].y),
                                       umma::gelu_erf(a.z + cb[i].z), umma::gelu_erf(a.w + cb[i].w));
          *(uint2*)(g.out_f16 + (row0 + r0 + 4 * i) * g.ldc + n) = umma::pack4(y);
        }
      }
    } break;
  }
}

// Four warpgroups:
//   WG0 (warps 0-3)   TMA producer; warp 0 issues, warps 1-3 only make the other warpgroups whole and aligned;
//   WG1 (warps 4-7)   epilogue: warp w walks rows w, w + 4, ... of the 128 x BN tile (gemm_epilogue_rows), or thread
//                     t owns row t (every launch gemm_launch_by_rows turns down);
//   WG2-3 (warps 8-15) MMA consumers, 64 accumulator rows each.
// The consumers hand each finished tile to the epilogue warpgroup through the fp32 staging tile and go straight on to
// the next tile's mainloop, so the tensor cores stay busy while the epilogue of the previous tile runs.
constexpr int kGemmThreads = 512;
constexpr int kBK = 64;  // 64 f16 = 128 B = one swizzle row
constexpr int kPromote = 4;  // k-blocks (K = 256) per tensor-core accumulation group
// setmaxnreg split of the 64 K-register file: 128 x producer + 128 x epilogue + 256 x consumer <= 65536.  A consumer
// holds acc + tot (BN registers) and the loop state; the epilogue holds one 32-column chunk (~100 live values for the
// LayerScale + residual read-modify-write).
constexpr int kProducerRegs = 40;
constexpr int kEpilogueRegs = 120;
constexpr int kConsumerRegs = 176;
static_assert(128 * kProducerRegs + 128 * kEpilogueRegs + 256 * kConsumerRegs <= 65536, "register file overcommitted");

template <int BN, int STAGES>
struct GemmSmem {
  static constexpr int kABytes = 128 * kBK * 2;
  static constexpr int kBBytes = BN * kBK * 2;
  static constexpr int kStage = kABytes + kBBytes;
  static constexpr int kPitch = BN + 4;  // floats per staged row (+4: no bank conflicts on the row reads)
  static constexpr int kEpi = 128 * kPitch * 4;  // the 128 x BN fp32 staging tile (consumers -> epilogue warpgroup)
  static constexpr int kTotal = STAGES * kStage + kEpi + 1024 /*align*/ + 256 /*barriers*/;
};

template <int BN, int STAGES, bool kSr = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
k_umma_gemm(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmArgs g) {
  using S = GemmSmem<BN, STAGES>;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment for SWIZZLE_128B
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  float* epi_buf = (float*)(smem + STAGES * S::kStage);
  uint64_t* bars = (uint64_t*)(smem + STAGES * S::kStage + S::kEpi);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;
  uint64_t* epi_full = bars + 2 * STAGES;  // staging tile written by both consumer warpgroups
  uint64_t* epi_empty = epi_full + 1;      // staging tile read by the epilogue warpgroup

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // persistent: this CTA walks tiles blockIdx.x, +gridDim.x, ...; n fastest so co-resident CTAs share A in L2
  const int total_tiles = g.nt * g.mt * g.nz;
  const int nkb = (g.K + kBK - 1) / kBK;

  if (warp == 0 && lane == 0) {
    umma::prefetch_tmap(&tmA);
    umma::prefetch_tmap(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      umma::mbar_init(umma::smem_u32(&full[s]), 1);
      umma::mbar_init(umma::smem_u32(&empty[s]), 2);  // one arrive per consumer warpgroup
    }
    umma::mbar_init(umma::smem_u32(epi_full), 256);  // every consumer thread, after its own staging stores
    umma::mbar_init(umma::smem_u32(epi_empty), 128);  // every epilogue thread, after its own staging reads
    umma::fence_barrier_init();
  }
  __syncthreads();

  auto decode = [&](int tile, int& n_blk, int& m_blk, int& z, int& px0, int& py0) {
    n_blk = tile % g.nt;
    int rem = tile / g.nt;
    m_blk = rem % g.mt;
    z = rem / g.mt;
    px0 = py0 = 0;
    if (g.conv) {  // pixel tile origin for conv mode
      int tiles_x = (g.imgW + g.tw - 1) / g.tw;
      py0 = (m_blk / tiles_x) * g.th;
      px0 = (m_blk % tiles_x) * g.tw;
    }
  };

  if (warp < 4) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));  // registers go to the consumers
    if (warp == 0 && lane == 0) {
      int kit = 0;  // k-block counter across tiles (ring position)
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int n_blk, m_blk, z, px0, py0;
        decode(tile, n_blk, m_blk, z, px0, py0);
        for (int kb = 0; kb < nkb; ++kb, ++kit) {
          const int s = kit % STAGES;
          const uint32_t ph = (kit / STAGES) & 1;
          umma::mbar_wait(umma::smem_u32(&empty[s]), ph ^ 1);
          const uint32_t fb = umma::smem_u32(&full[s]);
          umma::mbar_expect_tx(fb, S::kStage);
          const uint32_t sa = umma::smem_u32(smem + s * S::kStage);
          const uint32_t sb = sa + S::kABytes;
          if (g.conv == 0) {
            umma::tma_load_3d(sa, &tmA, fb, kb * kBK, m_blk * 128, z);
          } else {
            const int cblocks = g.cin / kBK;
            const int tap = kb / cblocks, cb = kb % cblocks;
            int dx = 0, dy = 0;
            if (g.conv == 1) {
              dy = tap / 3 - 1;
              dx = tap % 3 - 1;
            }
            umma::tma_load_3d(sa, &tmA, fb, cb * kBK, px0 + dx, py0 + dy);
          }
          umma::tma_load_3d(sb, &tmB, fb, kb * kBK, n_blk * BN, z);
        }
      }
    }
  } else if (warp < 8) {
    // ===================== epilogue warpgroup =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kEpilogueRegs));
    // One tile loop per epilogue mapping (decided for the whole launch), so that neither constrains the other's
    // registers under the 120 of this warpgroup
    if (gemm_launch_by_rows<BN, kSr>(g)) {
      int j = 0;  // staging round (tiles of this CTA)
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++j) {
        int n_blk, m_blk, z, px0, py0;
        decode(tile, n_blk, m_blk, z, px0, py0);
        umma::mbar_wait(umma::smem_u32(epi_full), j & 1);
        gemm_epilogue_rows(g, epi_buf, S::kPitch, m_blk, n_blk, z);
        umma::mbar_arrive(umma::smem_u32(epi_empty));
      }
      return;
    }
    const int r = threadIdx.x & 127;  // accumulator row inside the tile
    int j = 0;                        // staging round (tiles of this CTA)
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++j) {
      int n_blk, m_blk, z, px0, py0;
      decode(tile, n_blk, m_blk, z, px0, py0);
      int m;  // logical output row
      bool row_ok;
      if (g.conv) {
        int ly = r / g.tw, lx = r % g.tw;
        int y = py0 + ly, x = px0 + lx;
        row_ok = (y < g.imgH) && (x < g.imgW);
        m = y * g.imgW + x;
      } else {
        m = m_blk * 128 + r;
        row_ok = m < g.M;
      }
      umma::mbar_wait(umma::smem_u32(epi_full), j & 1);
      // the fused epilogue on the row's BN / 32 chunks of 32 consecutive columns, in column order
      float head_acc = 0.f;
#pragma unroll 1
      for (int ci = 0; ci < BN / 32; ++ci) {
        uint32_t v[32];
        const float4* src = (const float4*)(epi_buf + r * S::kPitch + ci * 32);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 f = src[i];
          v[4 * i] = __float_as_uint(f.x);
          v[4 * i + 1] = __float_as_uint(f.y);
          v[4 * i + 2] = __float_as_uint(f.z);
          v[4 * i + 3] = __float_as_uint(f.w);
        }
        gemm_epilogue_chunk<kSr>(g, v, m, z, n_blk * BN + ci * 32, row_ok, head_acc);
      }
      // DPT head: N == 32 is a single chunk
      if (g.epi == EPI_HEAD && row_ok && n_blk == 0) {
        const float s = head_acc + g.b3p[0];
        g.out_f32[m] = g.head_max > 0.f ? g.head_max * (1.f / (1.f + expf(-s))) : fmaxf(s, 0.f);
      }
      umma::mbar_arrive(umma::smem_u32(epi_empty));
    }
  } else {
    // ===================== consumers: MMA, then hand the tile to the epilogue warpgroup =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
    const int wg = (warp >> 2) - 2;      // consumer warpgroup: accumulator rows 64 wg .. 64 wg + 63
    const int t = threadIdx.x & 127;     // thread in the warpgroup
    const int wq = t >> 5;               // warp in the warpgroup: fragment rows 16 wq .. 16 wq + 15
    float* ebuf = epi_buf + wg * 64 * S::kPitch;
    int kit = 0;
    int j = 0;  // staging round
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++j) {
      // The tensor core adds each k16 product sum into its accumulator with truncation, so over long reductions (fc2:
      // K = 4D) the error grows with K.  Each group of kPromote k-blocks is therefore accumulated from zero in `acc`
      // and then added into the fp32 total `tot` in the FP32 pipe.
      float acc[BN / 2];  // the first k-block of a group overwrites it (scale-d = 0)
      float tot[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) tot[i] = 0.f;
      int prev = -1;  // ring slot still read by the wgmmas in flight
      // groups of kPromote k-blocks: the loop structure, not a data-dependent branch, decides where a group ends, and the
      // accumulator is only read after the group's wgmma.wait_group 0
      for (int kb0 = 0; kb0 < nkb; kb0 += kPromote) {
        const int kend = min(nkb, kb0 + kPromote);
        for (int kb = kb0; kb < kend; ++kb, ++kit) {
          const int s = kit % STAGES;
          const uint32_t ph = (kit / STAGES) & 1;
          umma::mbar_wait(umma::smem_u32(&full[s]), ph);
          const uint32_t sa = umma::smem_u32(smem + s * S::kStage) + (uint32_t)(wg * 64 * 128);
          const uint32_t sb = umma::smem_u32(smem + s * S::kStage) + S::kABytes;
          const uint64_t da = umma::make_desc(sa), db = umma::make_desc(sb);
          umma::wgmma_fence();
#pragma unroll
          for (int k = 0; k < kBK / 16; ++k)
            umma::wgmma_ss<BN>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), ((kb - kb0) | k) ? 1u : 0u);
          umma::wgmma_commit();
          umma::wgmma_wait<1>();  // the previous k-block's wgmmas have retired: its slot may be refilled
          if (prev >= 0 && t == 0) umma::mbar_arrive(umma::smem_u32(&empty[prev]));
          prev = s;
        }
        umma::wgmma_wait<0>();
        umma::fence_regs(acc);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) tot[i] += acc[i];
      }
      if (prev >= 0 && t == 0) umma::mbar_arrive(umma::smem_u32(&empty[prev]));

      // ---- hand-off: once the epilogue warpgroup has read the previous tile, stage this one ----
      umma::mbar_wait(umma::smem_u32(epi_empty), (j & 1) ^ 1);
      // fragment of m64nN: tot[4 i + q] is row 16 wq + lane/4 + 8 (q >> 1), column 8 i + 2 (lane & 3) + (q & 1)
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const int c = 8 * i + 2 * (lane & 3);
        const int r0 = 16 * wq + (lane >> 2);
        *(float2*)(ebuf + r0 * S::kPitch + c) = make_float2(tot[4 * i], tot[4 * i + 1]);
        *(float2*)(ebuf + (r0 + 8) * S::kPitch + c) = make_float2(tot[4 * i + 2], tot[4 * i + 3]);
      }
      umma::mbar_arrive(umma::smem_u32(epi_full));
    }
  }
}

}  // namespace vd3d
