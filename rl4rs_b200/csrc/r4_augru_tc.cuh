// r4_augru_tc.cuh -- common ground of the tensor-core kernels (GRU-1 / AUGRU recurrences, attention scores, GEMM):
// constants of the AUGRU problem, the PTX wrappers (wgmma, mbarrier, bulk copy), the bf16 hi/lo split, the quad-layout
// input loads and the parameter structs of the AUGRU kernel (r4_recur.cuh).
//
// fp32 parity on a bf16 tensor pipe: every fp32 operand x is split x = hi + lo (both bf16, lo = bf16(x - hi)) and each
// product is issued as hi*hi + lo*hi + hi*lo (3 MMAs, fp32 accumulate): relative error ~2^-16 per term, inside the 1e-4
// parity bound on the 64-step recurrence.  The state h itself stays fp32 in registers; only the MMA operand copies are rounded.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <string.h>
#include <algorithm>

namespace r4tc {

constexpr int TM = 128;                 // rows per lane-major input tile
constexpr int HID = 256;                // AUGRU hidden = GEMM N and K
constexpr int STEPS = 64;
constexpr int KB = 32;                  // K elements per B stage
constexpr int NKB = HID / KB;           // 8 K blocks per matrix
constexpr int LBO = 128;                             // K-adjacent core matrices
constexpr int B_SBO = (KB / 8) * 128;                // 512:  8-row groups inside a 32-deep weight block
constexpr int XT_COLS = 3 * HID;                     // transposed input halves: [r | u | c] rows of 128 lanes

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Shared-memory matrix descriptor of a wgmma operand in the SWIZZLE_NONE K-major layout: 8-row x 16-byte core matrices,
// `lbo` = byte distance of K-adjacent core matrices, `sbo` = byte distance of 8-row groups (layout type 0 in bits 62-63).
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((saddr >> 4) & 0x3fff) | ((uint64_t)((lbo >> 4) & 0x3fff) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3fff) << 32);
}
// D[64 x N] (+)= A[64 x 16] . B[16 x N]^T, bf16 in, fp32 accumulators in the registers of the issuing warpgroup.  Register
// i of a thread (warp w of the warpgroup, lane l) holds row 16 w + l / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (l % 4) + i % 2.
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(da), "l"(db), "r"(1) : "memory");
}
__device__ __forceinline__ void wgmma_m64n16k16_rs(float (&d)[8], const uint32_t (&a)[4], uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1, 0;\n\t}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(1) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile("{\n\t.reg .pred p;\n\tWAIT_LOOP:\n\t"
               "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
               "@p bra DONE;\n\tbra WAIT_LOOP;\n\tDONE:\n\t}\n"
               :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// generic-proxy shared-memory stores -> visible to the async proxy (wgmma operand reads, bulk copies)
__device__ __forceinline__ void proxy_fence() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(nthreads) : "memory");
}
// two fp32 -> bf16 pair words (low half = first value): hi = bf16(x), lo = bf16(x - hi)
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
  const __nv_bfloat162 l = __floats2bfloat162_rn(x0 - __bfloat162float(h.x), x1 - __bfloat162float(h.y));
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// MUFU-based gate functions: ex2.approx (rel. error 2^-22) + rcp.approx (1 ulp); saturate correctly
// (ex2 -> +inf gives rcp -> 0).  No slow-path calls (the IEEE __frcp_rn costs a CALL per element).
__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float fast_sigmoid(float x) { return rcp_approx(1.0f + ex2_approx(-1.4426950408889634f * x)); }
__device__ __forceinline__ float fast_tanh(float x) { return fmaf(-2.0f, rcp_approx(1.0f + ex2_approx(2.8853900817779268f * x)), 1.0f); }

// split 8 consecutive fp32 into bf16 hi / lo vectors (16 B each)
__device__ __forceinline__ void split8(const float* x, uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __nv_bfloat162 hh = __floats2bfloat162_rn(x[2 * i], x[2 * i + 1]);
    float r0 = x[2 * i] - __bfloat162float(hh.x), r1 = x[2 * i + 1] - __bfloat162float(hh.y);
    __nv_bfloat162 ll = __floats2bfloat162_rn(r0, r1);
    h[i] = *reinterpret_cast<uint32_t*>(&hh);
    l[i] = *reinterpret_cast<uint32_t*>(&ll);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}

// 16 consecutive columns (colbase % 16 == 0) of one lane of a lane-major tile-step in the quad layout
// [col / 4][lane][col % 4] (r4_gemm_tc.cuh: xt_index): four 128-bit loads.  `ts` = tile-step base, `ln4` = lane * 4.
#ifndef R4_LDG_NOALLOC
#define R4_LDG_NOALLOC 0     // 1: the input halves are read once per CTA -> ld.global.nc.L1::no_allocate (probe switch)
#endif
__device__ __forceinline__ float4 ldg_x4(const float* p) {
#if R4_LDG_NOALLOC
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
#else
  return __ldg(reinterpret_cast<const float4*>(p));
#endif
}
__device__ __forceinline__ void load_x16(float* dst, const float* ts, int colbase, int ln4) {
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const float4 v = ldg_x4(ts + (size_t)(colbase + 4 * g) * TM + ln4);
    dst[4 * g] = v.x; dst[4 * g + 1] = v.y; dst[4 * g + 2] = v.z; dst[4 * g + 3] = v.w;
  }
}

struct AugruTcSeq {
  const float* XT;        // transposed input halves [n_tiles_cached, 64, 768 / 4, 128, 4]  (tile, step, column quad, lane, column % 4)
  const uint8_t* Wimg;    // pre-tiled bf16 hi/lo weight stream (r4_recur.cuh: build_recur_image)
  const float* scoresT;   // [n_row_tiles, 64, 128]
  float* out;             // final state, row stride out_ld
  int shared;             // 1: every row reads cached sequence 0
};
struct AugruTcParams {
  AugruTcSeq s[2];
  int R, row0, div, out_ld;
};

// host-side bf16 rounding (round to nearest even) shared by the weight-image builders
inline uint16_t host_bf16_bits(float x) {
  uint32_t u; memcpy(&u, &x, 4);
  if ((u & 0x7f800000u) == 0x7f800000u) return (uint16_t)(u >> 16);
  u = (u + 0x7fffu + ((u >> 16) & 1u)) >> 16; return (uint16_t)u;
}
inline float host_bf16_val(uint16_t b) { uint32_t u = (uint32_t)b << 16; float f; memcpy(&f, &u, 4); return f; }
}  // namespace r4tc
