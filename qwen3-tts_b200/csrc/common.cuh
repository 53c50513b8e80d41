// Shared device/host helpers for the H100 (sm_90a) Qwen3-TTS hot-path kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>

typedef __nv_bfloat16 bf16;

// ------------------------------------------------------------------------------------------------
// host-side error plumbing (thread-local message returned by q3_last_error())
// ------------------------------------------------------------------------------------------------
extern thread_local std::string g_q3_err;
int q3_set_err(const char* fmt, ...);

#define Q3_CUDA(call)                                                                              \
  do {                                                                                             \
    cudaError_t _e = (call);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      return q3_set_err("%s:%d CUDA error %d (%s) in %s", __FILE__, __LINE__, (int)_e,             \
                        cudaGetErrorString(_e), #call);                                            \
  } while (0)

#define Q3_REQUIRE(cond, ...)                                                                      \
  do {                                                                                             \
    if (!(cond)) return q3_set_err(__VA_ARGS__);                                                   \
  } while (0)

// ------------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------------
#ifdef __CUDACC__

__device__ __forceinline__ float bf16lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
__device__ __forceinline__ float bf2f(bf16 x) { return __bfloat162float(x); }
__device__ __forceinline__ bf16 f2bf(float x) { return __float2bfloat16_rn(x); }
// round-trip through bf16 (mimics a PyTorch bf16 intermediate)
__device__ __forceinline__ float rbf(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// streaming weight load: read-only path, do not pollute L1
__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
// cross-CTA activations: L2-coherent loads (bypass the non-coherent L1)
__device__ __forceinline__ uint4 ldcg16(const void* p) {
  uint4 r;
  asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint2 ldcg8(const void* p) {
  uint2 r;
  asm volatile("ld.global.cg.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ uint32_t ldcg4(const void* p) {
  uint32_t r;
  asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ float ldcgf(const float* p) {
  float r;
  asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ bf16 ldcg_bf16(const bf16* p) {
  unsigned short r;
  asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(r) : "l"(p));
  return __ushort_as_bfloat16(r);
}
__device__ __forceinline__ int ldcgi(const int* p) {
  int r;
  asm volatile("ld.global.cg.s32 %0, [%1];" : "=r"(r) : "l"(p));
  return r;
}

// L2 prefetch of a contiguous byte range through the bulk-copy (TMA) unit; bytes % 16 == 0
__device__ __forceinline__ void l2_prefetch_bulk(const void* p, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}

// D[16x8] += A[16x16] * B[16x8], bf16 inputs, fp32 accumulate
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Philox4x32-10 (Salmon et al. SC'11) — must match oracle/philox.py bit for bit.
__device__ __forceinline__ uint32_t philox_u32(uint64_t seed, uint32_t c0, uint32_t c1, uint32_t c2) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  uint32_t c3 = 0;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c0;
}
__device__ __forceinline__ float philox_uniform(uint64_t seed, uint32_t row, uint32_t frame, uint32_t group) {
  return (float)(philox_u32(seed, row, frame, group) >> 8) * (1.0f / 16777216.0f);
}

#endif  // __CUDACC__
