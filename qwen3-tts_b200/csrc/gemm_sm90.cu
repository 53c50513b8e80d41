// wgmma tap-GEMM kernel (see gemm_sm90.cuh).  Warp-specialised and PERSISTENT: a CTA walks 128 x bn output tiles
// (tile = blockIdx.x, += gridDim.x); the TMA ring keeps running across tiles, so the loads of tile i+1 overlap the
// epilogue of tile i:
//   warps 0-7 : two consumer warpgroups, each owning 64 rows of the tile: wgmma.mma_async m64 x bn x k16 (bf16 -> fp32
//               in registers) straight from the swizzled shared-memory stages, then the epilogue (bias / LayerScale /
//               residual / SnakeBeta / GELU / SwiGLU, bf16 stores) from the accumulator fragments
//   warp 8    : TMA producer (A tile via a 3-D map with a per-tap row shift, W tile via a 2-D map)
#include "gemm_sm90.cuh"
#include <algorithm>
#include <cstring>

namespace {

constexpr int BM = 128;
constexpr int BK = 64;           // 64 bf16 = 128 B = one SWIZZLE_128B row
constexpr int MAX_STAGES = 6;
constexpr int A_BYTES = BM * BK * 2;        // 16 KB
constexpr int SMEM_OPTIN = 232448;          // 227 KB
constexpr int BAR_BYTES = 256;              // full[S], empty[S]
constexpr int CONSUMER_WGS = 2;             // rows [64 * wg, +64) of the tile
constexpr int PRODUCER_WARP = 4 * CONSUMER_WGS;
constexpr int GEMM_THREADS = 128 * CONSUMER_WGS + 32;  // consumer warpgroups first (wgmma needs aligned warpgroups)
__host__ __device__ inline int stage_bytes_for(int bn) { return A_BYTES + ((bn * BK * 2 + 1023) & ~1023); }
inline int stages_for(int bn) { return std::min(MAX_STAGES, (SMEM_OPTIN - 1024 - BAR_BYTES) / stage_bytes_for(bn)); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  long long t0 = clock64();
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) break;
    if (clock64() - t0 > 4000000000LL) __trap();  // never hang the box on a protocol bug
  }
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}
// K-major, SWIZZLE_128B wgmma shared-memory matrix descriptor: 8-row groups 1024 B apart
__device__ __forceinline__ uint64_t make_sdesc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);        // start address
  d |= (uint64_t)1 << 16;                          // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;                // stride byte offset
  d |= (uint64_t)1 << 62;                          // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x BN] (+)= A[64 x 16] * W[BN x 16]^T, both operands K-major in shared memory; accum == 0 overwrites D
template <int BN>
__device__ __forceinline__ void wgmma_bf16(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t accum);
template <>
__device__ __forceinline__ void wgmma_bf16<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accum));
}
template <>
__device__ __forceinline__ void wgmma_bf16<128>(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accum));
}

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

// sin for the SnakeBeta epilogue: Cody-Waite reduction to [-pi, pi] (k * 6.28125 is exact for |k| < 2^15), then the SFU
// (MUFU.SIN, abs error 2^-21.4 on that interval).  The result is squared, scaled and rounded to bf16 (2^-9 relative), so
// this is far inside the output's resolution for every argument below ~1e4; sinf()'s 20-instruction polynomial would
// make the epilogue of the short-K decoder convolutions as long as their mainloop.
__device__ __forceinline__ float snake_sin(float a) {
  const float k = (fmaf(a, 0.15915494309189535f, 12582912.f)) - 12582912.f;  // rint for |a/2pi| < 2^22, on the FMA pipe (FRND is quarter-rate)
  float r = fmaf(-k, 6.28125f, a);
  r = fmaf(-k, 1.9353071795864769e-3f, r);
  return __sinf(r);
}

// round a pair to bf16 and back (a PyTorch bf16 intermediate); returns the packed pair
__device__ __forceinline__ uint32_t round2(float& x0, float& x1) {
  const uint32_t xp = pack_bf16(x0, x1);
  x0 = bf16lo(xp);
  x1 = bf16hi(xp);
  return xp;
}

// ACT and BN are template parameters on purpose: the wgmma shape is part of the instruction, and with a run-time
// activation code ptxas if-converts the activation branches and evaluates erff() AND sin() for every element.
template <int BN, int ACT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) tap_gemm_kernel(const __grid_constant__ GemmPlan p) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  constexpr int STAGE_BYTES = A_BYTES + BN * BK * 2;
  static_assert(BN % 64 == 0 && STAGE_BYTES % 1024 == 0, "SWIZZLE_128B operand tiles must stay 1024-byte aligned");
  const int STAGES = p.nst;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);  // full[S], empty[S]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kpb = p.Kp / BK;
  const int nkb = p.ntaps * kpb;
  const int mtiles = (p.T + BM - 1) / BM, ntiles = (p.N + BN - 1) / BN;
  const int total = mtiles * ntiles * p.B;
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + MAX_STAGES);

  if (warp == PRODUCER_WARP && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&p.tmW) : "memory");
    for (int s = 0; s < STAGES; ++s) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, CONSUMER_WGS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      int s = 0, round = 0;  // ring slot and how many times the ring has wrapped, over all tiles
      for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        const int nt = tile % ntiles, mt = (tile / ntiles) % mtiles, b = tile / (ntiles * mtiles);
        const int m0 = mt * BM, n0 = nt * BN;
        for (int kb = 0; kb < nkb; ++kb) {
          if (round > 0) mbar_wait(empty0 + 8 * s, (round - 1) & 1);
          const int tap = kb / kpb, k0 = (kb - tap * kpb) * BK;
          const uint32_t sa = smem_u32(smem + s * STAGE_BYTES), sb = sa + A_BYTES;
          mbar_expect_tx(full0 + 8 * s, STAGE_BYTES);
          tma_load_3d(sa, &p.tmA, k0, m0 + p.shift[tap] + p.a_row0, b, full0 + 8 * s);
          tma_load_2d(sb, &p.tmW, tap * p.Kp + k0, n0, full0 + 8 * s);
          if (++s == STAGES) { s = 0; ++round; }
        }
      }
    }
    return;
  }

  // ---- consumers.  Accumulator fragment of m64nBNk16 (per warpgroup): register 4j + 2h + e holds row
  // 16 * (warp % 4) + lane / 4 + 8h, column 8j + 2 * (lane % 4) + e.
  const int wg = warp >> 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const GemmEpilogue& E = p.ep;
  float acc[BN / 2];
  int s = 0, round = 0;
  for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
    const int nt = tile % ntiles, mt = (tile / ntiles) % mtiles, b = tile / (ntiles * mtiles);
    const int m0 = mt * BM, n0 = nt * BN;
    int prev = 0;
    for (int kb = 0; kb < nkb; ++kb) {
      mbar_wait(full0 + 8 * s, round & 1);
      const uint32_t sa = smem_u32(smem + s * STAGE_BYTES);
      const uint64_t ad = make_sdesc(sa + wg * 64 * 128), bd = make_sdesc(sa + A_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        // advance 16 bf16 = 32 B inside the 128 B swizzle row: +2 in the (>>4) start-address field
        wgmma_bf16<BN>(acc, ad + (uint64_t)(k * 2), bd + (uint64_t)(k * 2), (kb | k) != 0);
      }
      wgmma_commit();
      if (kb > 0) {  // the previous stage's MMAs are complete: hand its slot back to the producer
        wgmma_wait<1>();
        if (wg_leader) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(empty0 + 8 * prev) : "memory");
      }
      prev = s;
      if (++s == STAGES) { s = 0; ++round; }
    }
    wgmma_wait<0>();
    if (wg_leader) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(empty0 + 8 * prev) : "memory");

    const int c_lane = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * h;
      if (m >= p.T) continue;
      if constexpr (ACT == ACT_SWIGLU_PAIR) {  // columns (2i, 2i+1) = (gate_i, up_i)
        bf16* orow = E.out_act + (size_t)b * (size_t)p.act_bs + (size_t)m * (size_t)(p.N / 2);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int n = n0 + 8 * j + c_lane;
          if (n >= p.N) continue;
          const int ch = n % E.cmod;
          const float gt = rbf(acc[4 * j + 2 * h] + (E.bias ? E.bias[ch] : 0.f));
          const float u = rbf(acc[4 * j + 2 * h + 1] + (E.bias ? E.bias[ch + 1] : 0.f));
          orow[n / 2] = f2bf(rbf(gt / (1.f + __expf(-gt))) * u);
        }
      } else if constexpr (ACT == ACT_SWIGLU_BLK8) {  // 16 columns = gate[8i..8i+7] | up[8i..8i+7] (the AR engine's gate_up row interleave)
        bf16* orow = E.out_act + (size_t)b * (size_t)p.act_bs + (size_t)m * (size_t)(p.N / 2);
#pragma unroll
        for (int j = 0; j < BN / 16; ++j) {
          const int n = n0 + 16 * j;
          if (n >= p.N) continue;
          const int ch = n % E.cmod + c_lane;
          float y[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float gt = rbf(acc[8 * j + 2 * h + e] + (E.bias ? E.bias[ch + e] : 0.f));
            const float u = rbf(acc[8 * j + 4 + 2 * h + e] + (E.bias ? E.bias[ch + 8 + e] : 0.f));
            y[e] = rbf(gt / (1.f + __expf(-gt))) * u;
          }
          *reinterpret_cast<uint32_t*>(orow + n / 2 + c_lane) = pack_bf16(y[0], y[1]);
        }
      } else {
        const size_t row = (size_t)m * (size_t)p.N;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int n = n0 + 8 * j + c_lane;
          if (n >= p.N) continue;  // N % 16 == 0: n + 1 < N as well
          const int ch = n % E.cmod;
          float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
          if (E.bias) {
            const float2 bv = __ldg(reinterpret_cast<const float2*>(E.bias + ch));
            x0 += bv.x; x1 += bv.y;
          }
          uint32_t xp = round2(x0, x1);  // the reference's layer output is bf16
          if (E.scale) {
            const float2 sv = __ldg(reinterpret_cast<const float2*>(E.scale + ch));
            x0 *= sv.x; x1 *= sv.y;
            xp = round2(x0, x1);
          }
          if (E.resid) {  // plain load: the residual may be the tensor this launch writes (in-place update)
            const uint32_t r = *reinterpret_cast<const uint32_t*>(E.resid + (size_t)b * (size_t)p.resid_bs + row + n);
            x0 += bf16lo(r); x1 += bf16hi(r);
            xp = round2(x0, x1);
          }
          if (E.out_raw) *reinterpret_cast<uint32_t*>(E.out_raw + (size_t)b * (size_t)p.raw_bs + row + n) = xp;
          if (E.out_act) {
            float y0 = x0, y1 = x1;
            if constexpr (ACT == ACT_SNAKE) {
              const float2 ea = __ldg(reinterpret_cast<const float2*>(E.snake_ea + ch));
              const float2 ib = __ldg(reinterpret_cast<const float2*>(E.snake_ib + ch));
              const float s0 = snake_sin(x0 * ea.x), s1 = snake_sin(x1 * ea.y);
              y0 = x0 + ib.x * s0 * s0;
              y1 = x1 + ib.y * s1 * s1;
            } else if constexpr (ACT == ACT_GELU) {
              y0 = gelu_erf(x0);
              y1 = gelu_erf(x1);
            }
            *reinterpret_cast<uint32_t*>(E.out_act + (size_t)b * (size_t)p.act_bs + row + n) = pack_bf16(y0, y1);
          }
        }
      }
    }
  }
}

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                             const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeFn g_encode = nullptr;
int g_sm_count = 0;

template <int BN>
int set_smem_attrs() {
  Q3_CUDA(cudaFuncSetAttribute(tap_gemm_kernel<BN, ACT_NONE>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_OPTIN));
  Q3_CUDA(cudaFuncSetAttribute(tap_gemm_kernel<BN, ACT_SNAKE>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_OPTIN));
  Q3_CUDA(cudaFuncSetAttribute(tap_gemm_kernel<BN, ACT_GELU>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_OPTIN));
  Q3_CUDA(cudaFuncSetAttribute(tap_gemm_kernel<BN, ACT_SWIGLU_PAIR>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_OPTIN));
  Q3_CUDA(cudaFuncSetAttribute(tap_gemm_kernel<BN, ACT_SWIGLU_BLK8>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_OPTIN));
  return 0;
}

template <int BN>
int launch_bn(const GemmPlan& plan, int grid, int smem_bytes, cudaStream_t stream) {
  switch (plan.ep.act) {
    case ACT_NONE: tap_gemm_kernel<BN, ACT_NONE><<<grid, GEMM_THREADS, smem_bytes, stream>>>(plan); break;
    case ACT_SNAKE: tap_gemm_kernel<BN, ACT_SNAKE><<<grid, GEMM_THREADS, smem_bytes, stream>>>(plan); break;
    case ACT_GELU: tap_gemm_kernel<BN, ACT_GELU><<<grid, GEMM_THREADS, smem_bytes, stream>>>(plan); break;
    case ACT_SWIGLU_PAIR: tap_gemm_kernel<BN, ACT_SWIGLU_PAIR><<<grid, GEMM_THREADS, smem_bytes, stream>>>(plan); break;
    case ACT_SWIGLU_BLK8: tap_gemm_kernel<BN, ACT_SWIGLU_BLK8><<<grid, GEMM_THREADS, smem_bytes, stream>>>(plan); break;
    default: Q3_REQUIRE(false, "unknown activation %d", plan.ep.act);
  }
  return 0;
}

}  // namespace

int gemm_init() {
  if (!g_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    Q3_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    Q3_REQUIRE(fn && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available in this driver");
    g_encode = reinterpret_cast<EncodeFn>(fn);
  }
  if (set_smem_attrs<64>() || set_smem_attrs<128>()) return 1;
  if (g_sm_count == 0) {
    int dev = 0;
    Q3_CUDA(cudaGetDevice(&dev));
    Q3_CUDA(cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, dev));
  }
  return 0;
}

int gemm_make_plan(GemmPlan* plan, const bf16* a, int B, int T, int K, int64_t lda, int64_t a_batch_stride, const bf16* w,
                   int N, int Kp, int ntaps, const int* shifts, int bn, const GemmEpilogue& ep) {
  return gemm_make_plan_v(plan, a, B, T, K, lda, a_batch_stride, w, N, Kp, ntaps, shifts, bn, ep, GemmViews{});
}

int gemm_make_plan_v(GemmPlan* plan, const bf16* a, int B, int T, int K, int64_t lda, int64_t a_batch_stride, const bf16* w,
                     int N, int Kp, int ntaps, const int* shifts, int bn, const GemmEpilogue& ep, const GemmViews& v) {
  Q3_REQUIRE(g_encode, "gemm_init() not called");
  Q3_REQUIRE(Kp % BK == 0 && Kp >= K, "Kp must be a multiple of 64 and >= K");
  Q3_REQUIRE(bn == 64 || bn == 128, "bn must be 64 or 128");
  Q3_REQUIRE(N % 16 == 0, "N must be a multiple of 16");
  Q3_REQUIRE(ntaps >= 1 && ntaps <= 8, "ntaps out of range");
  Q3_REQUIRE(ep.cmod % 16 == 0 && ((uintptr_t)ep.bias % 16) == 0 && ((uintptr_t)ep.scale % 16) == 0 &&
                 ((uintptr_t)ep.snake_ea % 16) == 0 && ((uintptr_t)ep.snake_ib % 16) == 0,
             "per-channel epilogue vectors must be 16-byte aligned and the channel count a multiple of 16");
  Q3_REQUIRE(!((ep.act == ACT_SWIGLU_PAIR || ep.act == ACT_SWIGLU_BLK8) && (ep.resid || ep.out_raw || ep.scale)),
             "gated epilogues write out_act only");
  Q3_REQUIRE((lda * 2) % 16 == 0 && (a_batch_stride * 2) % 16 == 0 && ((uintptr_t)a % 16) == 0, "A alignment");
  memset(plan, 0, sizeof(*plan));
  plan->B = B; plan->T = T; plan->N = N; plan->Kp = Kp; plan->ntaps = ntaps; plan->bn = bn; plan->ep = ep;
  const bool half = ep.act == ACT_SWIGLU_PAIR || ep.act == ACT_SWIGLU_BLK8;
  plan->a_row0 = v.a_row0;
  plan->nst = stages_for(bn);
  plan->raw_bs = v.raw_bs ? v.raw_bs : (long long)T * N;
  plan->act_bs = v.act_bs ? v.act_bs : (long long)T * (half ? N / 2 : N);
  plan->resid_bs = v.resid_bs ? v.resid_bs : (long long)T * N;
  const int a_rows = v.a_rows ? v.a_rows : T;
  for (int i = 0; i < ntaps; ++i) plan->shift[i] = shifts[i];
  {
    cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)a_rows, (cuuint64_t)B};
    cuuint64_t strides[2] = {(cuuint64_t)lda * 2, (cuuint64_t)a_batch_stride * 2};
    cuuint32_t box[3] = {(cuuint32_t)BK, (cuuint32_t)BM, 1};
    cuuint32_t es[3] = {1, 1, 1};
    CUresult r = g_encode(&plan->tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, (void*)a, dims, strides, box, es,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    Q3_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(A) failed: %d (K=%d T=%d B=%d lda=%lld)", (int)r, K, T, B, (long long)lda);
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)ntaps * Kp, (cuuint64_t)N};
    cuuint64_t strides[1] = {(cuuint64_t)ntaps * Kp * 2};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)bn};
    cuuint32_t es[2] = {1, 1};
    CUresult r = g_encode(&plan->tmW, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void*)w, dims, strides, box, es,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    Q3_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(W) failed: %d (N=%d Kp=%d taps=%d)", (int)r, N, Kp, ntaps);
  }
  return 0;
}

int gemm_pick_bn(int N, int mtiles, int B) {
  // a 128-wide tile reads each A tile half as often; a 64-wide one gives small problems enough tiles for every SM
  if (N > 64 && (long long)mtiles * ((N + 127) / 128) * B >= g_sm_count) return 128;
  return 64;
}

int gemm_launch(const GemmPlan& plan, cudaStream_t stream) {
  const long long total = (long long)((plan.T + BM - 1) / BM) * ((plan.N + plan.bn - 1) / plan.bn) * plan.B;
  const int grid = (int)std::min<long long>(total, g_sm_count);  // persistent: one CTA per SM walks the tiles
  const int smem_bytes = 1024 + plan.nst * stage_bytes_for(plan.bn) + BAR_BYTES;
  if (plan.bn == 128) {
    if (launch_bn<128>(plan, grid, smem_bytes, stream)) return 1;
  } else {
    if (launch_bn<64>(plan, grid, smem_bytes, stream)) return 1;
  }
  Q3_CUDA(cudaGetLastError());
  return 0;
}
