// Attention phase: per-head q/k RMSNorm + RoPE, KV append, single-query GQA with cross-CTA split-K combine.
// Part of the ar_engine.cu translation unit (include order: ar_program, ar_gemv, ar_attention, ar_sampler,
// the persistent kernel in ar_step, ar_prefill).
#pragma once

namespace {

// ------------------------------------------------------------------------------------------------
// attention phase (per (sequence, kv head, split) unit): q/k RMSNorm + RoPE, KV append, single-query GQA
// ------------------------------------------------------------------------------------------------
// one warp normalises + rotates one 128-vector; lane owns dims {l, l+32, l+64, l+96}
__device__ __noinline__ void norm_rope_vec(const bf16* src, const bf16* nw, float eps, const bf16* cosr, const bf16* sinr,
                                           float* out_f32, bf16* out_bf16, bf16* out_bf16_b = nullptr) {
  const int lane = threadIdx.x & 31;
  float x[4], w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) x[i] = bf2f(ldcg_bf16(src + lane + 32 * i));
#pragma unroll
  for (int i = 0; i < 4; ++i) w[i] = bf2f(nw[lane + 32 * i]);
  // rotate_half pairs: (l, l+64) and (l+32, l+96); cos/sin tables are [64] (emb = cat(freqs, freqs))
  const float c0 = bf2f(cosr[lane]), s0 = bf2f(sinr[lane]);
  const float c1 = bf2f(cosr[lane + 32]), s1 = bf2f(sinr[lane + 32]);
  float ss = x[0] * x[0] + x[1] * x[1] + x[2] * x[2] + x[3] * x[3];
  ss = warp_sum(ss);
  const float inv = rsqrtf(ss / (float)HD + eps);
#pragma unroll
  for (int i = 0; i < 4; ++i) x[i] = rbf(rbf(x[i] * inv) * w[i]);
  float o[4];
  o[0] = rbf(rbf(x[0] * c0) + rbf(-x[2] * s0));
  o[2] = rbf(rbf(x[2] * c0) + rbf(x[0] * s0));
  o[1] = rbf(rbf(x[1] * c1) + rbf(-x[3] * s1));
  o[3] = rbf(rbf(x[3] * c1) + rbf(x[1] * s1));
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (out_f32) out_f32[lane + 32 * i] = o[i];
    else {
      out_bf16[lane + 32 * i] = f2bf(o[i]);
      if (out_bf16_b) out_bf16_b[lane + 32 * i] = f2bf(o[i]);
    }
  }
}

// ---- unit geometry: one (sequence, kv head, context split) per CTA-iteration
struct AttnUnit {
  int seq, kvh, sp, nsplit, q0, nq, qstride, ctx_end, s0, s1, units;
};
__shared__ AttnUnit s_au;  // geometry of the unit whose K/V window is (being) loaded; written by attn_window_issue

constexpr int KVWIN = 60;                                   // cached K/V rows per unit held in shared memory
constexpr int ATT_QS_BYTES = 2 * RMAX * HD * 4;             // fp32 queries [nq<=2][RMAX][128]
constexpr int ATT_RED_BYTES = 32 * RMAX * 130 * 4;          // per-half-warp partials
constexpr int ATT_WIN_OFF = ATT_QS_BYTES + ATT_RED_BYTES;   // K window, then V window (bf16 [KVWIN][128] each)
static_assert(ATT_WIN_OFF % 16 == 0 && ATT_WIN_OFF + 2 * KVWIN * HD * 2 <= ATT_SMEM, "attention shared-memory layout");

// Geometry of `unit` -> s_au, and its cached K/V rows [s0, min(s1, first new position, s0+KVWIN)) -> the shared-memory
// window, asynchronously (cp.async, L2 -> smem).  Those rows were written in earlier phases, so for a CTA's first unit
// this runs BEFORE the grid barrier that precedes the attention phase: by the time q/k of the new token are
// normalised the cached rows are on chip.  One copy of this code (noinline): it is called from the pre-barrier hook
// and from the unit loop, and instruction-cache footprint is what bounds the frame loop's phase overheads.
__device__ __noinline__ void attn_window_issue(const Phase& ph, const KParams& P, unsigned char* smem, int frame, int unit) {
  const StackDev& S = ph.stack == 0 ? P.talker : P.cp;
  int nsplit = 1;
  if (ph.seqmode == SEQ_DECODE) {
    const int cmax = P.max_len0 + frame + 1;
    nsplit = max(1, min(min((cmax + 127) >> 7, (int)gridDim.x / (P.B * S.nkv)), MAXSPLIT));
  }
  AttnUnit u;
  u.nsplit = nsplit;
  u.units = P.B * S.nkv * nsplit;
  u.sp = unit % nsplit;
  u.kvh = (unit / nsplit) % S.nkv;
  const int si = min(unit / (nsplit * S.nkv), P.B - 1);
  u.seq = si; u.q0 = si;
  if (ph.seqmode == SEQ_CP) { u.nq = ph.nq; u.qstride = P.B; u.ctx_end = ph.ctx_end; }
  else { u.nq = 1; u.qstride = 0; u.ctx_end = max(1, min(P.len0[si] + frame + 1, S.cap)); }  // (clamp: finished rows of a session keep stepping)
  const int SL = (u.ctx_end + nsplit - 1) / nsplit;
  u.s0 = u.sp * SL;
  u.s1 = min(u.ctx_end, u.s0 + SL);
  if (threadIdx.x == 0) s_au = u;
  if (unit < u.units) {
    const int hi = min(min(u.s1, u.ctx_end - u.nq), u.s0 + KVWIN);
    const int n = hi - u.s0;
    const size_t base = ((((size_t)u.seq * S.layers + ph.layer) * S.nkv + u.kvh) * (size_t)S.cap + u.s0) * HD;
    const char* kg = reinterpret_cast<const char*>(S.kc + base);
    const char* vg = reinterpret_cast<const char*>(S.vc + base);
    const uint32_t kw = smem_addr(smem + ATT_WIN_OFF), vw = kw + KVWIN * HD * 2;
#pragma unroll 1
    for (int c = threadIdx.x; c < n * 16; c += NTHREADS) {
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(kw + c * 16), "l"(kg + (size_t)c * 16) : "memory");
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(vw + c * 16), "l"(vg + (size_t)c * 16) : "memory");
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}

__device__ __forceinline__ void attn_prefetch(const Phase& ph, const KParams& P, unsigned char* smem, int frame) {
  attn_window_issue(ph, P, smem, frame, (int)blockIdx.x);
}

template <bool DEV>
__device__ __forceinline__ void attn_phase(const Phase& ph, const KParams& P, unsigned char* smem, int frame) {
  const StackDev& S = ph.stack == 0 ? P.talker : P.cp;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nh = S.nh, nkv = S.nkv, layers = S.layers, cap = S.cap;
  const int R = nh / nkv;  // <= RMAX
  const int B = P.B;
  const int qkv_ld = (nh + 2 * nkv) * HD;
  const int layer = ph.layer;
  const float eps = S.eps;
  const bf16 *qn = ph.qn, *kn = ph.kn;

  float* qs = reinterpret_cast<float*>(smem);                 // [nq<=2][RMAX][128]
  float* red = qs + 2 * RMAX * HD;                            // [32 halfwarps][RMAX][130]
  bf16* kwin = reinterpret_cast<bf16*>(smem + ATT_WIN_OFF);   // [KVWIN][128]
  bf16* vwin = kwin + KVWIN * HD;
  __shared__ int s_ticket;

  // s_au holds the geometry of this CTA's first unit (written before the preceding grid barrier, which ended in a
  // CTA-wide sync); later units (B*nkv*nsplit > grid) compute theirs and fetch their window inside the loop
#pragma unroll 1
  for (int unit = blockIdx.x; unit < s_au.units; unit += gridDim.x) {
    if (unit != (int)blockIdx.x) {
      cta_sync();
      attn_window_issue(ph, P, smem, frame, unit);
      cta_sync();
    }
    const AttnUnit U = s_au;
    const int nsplit = U.nsplit;
    const int sp = U.sp, kvh = U.kvh, seq = U.seq, q0 = U.q0, nq = U.nq, qstride = U.qstride, ctx_end = U.ctx_end;
    const int s0 = U.s0, s1 = U.s1;
    bf16* kc = S.kc + (((size_t)seq * layers + layer) * nkv + kvh) * (size_t)cap * HD;
    bf16* vc = S.vc + (((size_t)seq * layers + layer) * nkv + kvh) * (size_t)cap * HD;

    // ---- per query token: q heads -> smem (fp32), k (norm+rope) and v -> cache (owner split only)
    const int nvec = nq * (R + 2);
#pragma unroll 1
    for (int v = warp; v < nvec; v += NWARPS) {
      const int j = v / (R + 2), which = v - j * (R + 2);
      const int col = q0 + j * qstride;
      const int pos = ctx_end - nq + j;
      const bool owner = (pos >= s0 && pos < s1);
      const bf16* base = S.qkv + (size_t)col * qkv_ld;
      const bf16* cosr = S.rope_cos + (size_t)pos * 64;
      const bf16* sinr = S.rope_sin + (size_t)pos * 64;
      if (which < R) {
        norm_rope_vec(base + (kvh * R + which) * HD, qn, eps, cosr, sinr, qs + (j * RMAX + which) * HD, nullptr);
      } else if (owner) {
        const bool inwin = pos - s0 < KVWIN;  // the new row is used from shared memory by this very phase
        if (which == R) {
          norm_rope_vec(base + (nh + kvh) * HD, kn, eps, cosr, sinr, nullptr, kc + (size_t)pos * HD, inwin ? kwin + (pos - s0) * HD : nullptr);
        } else {
          const bf16* vsrc = base + (nh + nkv + kvh) * HD;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const bf16 vv = ldcg_bf16(vsrc + lane + 32 * i);
            vc[(size_t)pos * HD + lane + 32 * i] = vv;
            if (inwin) vwin[(pos - s0) * HD + lane + 32 * i] = vv;
          }
        }
      }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
    __threadfence_block();
    cta_sync();
    PROF_MARK(2);

    const float scale = rsqrtf((float)HD);
    const int hw = warp * 2 + (lane >> 4), l16 = lane & 15;
    const int rr_ = tid >> 7, dd = tid & (HD - 1);
#pragma unroll 1
    for (int j = 0; j < nq; ++j) {
      const int col = q0 + j * qstride;
      const int pos = ctx_end - nq + j;
      const int e1 = min(s1, pos + 1);
      float q[RMAX][8];
#pragma unroll
      for (int r = 0; r < RMAX; ++r)
#pragma unroll
        for (int i = 0; i < 8; ++i) q[r][i] = (r < R) ? qs[(j * RMAX + r) * HD + l16 * 8 + i] : 0.f;
      float m[RMAX], l[RMAX], o[RMAX][8];
#pragma unroll
      for (int r = 0; r < RMAX; ++r) {
        m[r] = -INFINITY; l[r] = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) o[r][i] = 0.f;
      }
      // warp-uniform trip count (full-mask shuffles below); each half-warp handles 2 tokens per iteration so
      // that 4 independent 16-byte loads are in flight before the dependent softmax update
#pragma unroll 1
      for (int tb = s0 + warp * 4; tb < e1; tb += NWARPS * 4) {
        const int tk0 = tb + (lane >> 4), tk1 = tk0 + 2;
        uint4 kv[2], vv[2];
        kv[0] = kv[1] = vv[0] = vv[1] = make_uint4(0, 0, 0, 0);
        if (tk0 < e1) {
          if (tk0 - s0 < KVWIN) {
            kv[0] = *reinterpret_cast<const uint4*>(kwin + (tk0 - s0) * HD + l16 * 8);
            vv[0] = *reinterpret_cast<const uint4*>(vwin + (tk0 - s0) * HD + l16 * 8);
          } else { kv[0] = ldcg16(kc + (size_t)tk0 * HD + l16 * 8); vv[0] = ldcg16(vc + (size_t)tk0 * HD + l16 * 8); }
        }
        if (tk1 < e1) {
          if (tk1 - s0 < KVWIN) {
            kv[1] = *reinterpret_cast<const uint4*>(kwin + (tk1 - s0) * HD + l16 * 8);
            vv[1] = *reinterpret_cast<const uint4*>(vwin + (tk1 - s0) * HD + l16 * 8);
          } else { kv[1] = ldcg16(kc + (size_t)tk1 * HD + l16 * 8); vv[1] = ldcg16(vc + (size_t)tk1 * HD + l16 * 8); }
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {  // fully unrolled: register arrays must keep compile-time indices (no local memory)
          const bool valid = (u == 0 ? tk0 : tk1) < e1;
          const uint4 kk = kv[u], v4 = vv[u];
          const float kf[8] = {bf16lo(kk.x), bf16hi(kk.x), bf16lo(kk.y), bf16hi(kk.y),
                               bf16lo(kk.z), bf16hi(kk.z), bf16lo(kk.w), bf16hi(kk.w)};
          const float vf[8] = {bf16lo(v4.x), bf16hi(v4.x), bf16lo(v4.y), bf16hi(v4.y),
                               bf16lo(v4.z), bf16hi(v4.z), bf16lo(v4.w), bf16hi(v4.w)};
#pragma unroll
          for (int r = 0; r < RMAX; ++r) {
            if (r < R) {
              float d = 0.f;
#pragma unroll
              for (int i = 0; i < 8; ++i) d += q[r][i] * kf[i];
              d += __shfl_xor_sync(0xffffffffu, d, 8);
              d += __shfl_xor_sync(0xffffffffu, d, 4);
              d += __shfl_xor_sync(0xffffffffu, d, 2);
              d += __shfl_xor_sync(0xffffffffu, d, 1);
              if (valid) {
                d *= scale;
                const float mn = fmaxf(m[r], d);
                const float corr = __expf(m[r] - mn);  // exp(-inf)=0 on the first token
                const float p = __expf(d - mn);
                l[r] = l[r] * corr + p;
#pragma unroll
                for (int i = 0; i < 8; ++i) o[r][i] = o[r][i] * corr + p * vf[i];
                m[r] = mn;
              }
            }
          }
        }
      }
      // ---- combine the 32 half-warps
      PROF_MARK(3);
      cta_sync();
#pragma unroll
      for (int r = 0; r < RMAX; ++r) {
        if (r < R) {
          float* rr = red + ((size_t)hw * RMAX + r) * 130;
          if (l16 == 0) { rr[0] = m[r]; rr[1] = l[r]; }
#pragma unroll
          for (int i = 0; i < 8; ++i) rr[2 + l16 * 8 + i] = o[r][i];
        }
      }
      cta_sync();
      float M = -INFINITY, L = 0.f, O = 0.f;
      // token t of this split maps to half-warp ((t>>2)<<1) | (t&1): only the first nhw half-warps hold data
      const int ntok = max(e1 - s0, 0);
      const int nhw = min(2 * NWARPS, ((ntok + 3) >> 2) << 1);
      if (rr_ < R) {
#pragma unroll 2
        for (int h2 = 0; h2 < nhw; ++h2) M = fmaxf(M, red[((size_t)h2 * RMAX + rr_) * 130]);
#pragma unroll 2
        for (int h2 = 0; h2 < nhw; ++h2) {
          const float* rp = red + ((size_t)h2 * RMAX + rr_) * 130;
          const float wgt = (rp[0] == -INFINITY) ? 0.f : __expf(rp[0] - M);
          L += rp[1] * wgt;
          O += rp[2 + dd] * wgt;
        }
      }
      PROF_MARK(4);
      bf16* outp = S.attn + (size_t)col * (nh * HD) + (kvh * R + rr_) * HD + dd;
      if (nsplit == 1) {
        if (rr_ < R) *outp = f2bf(O / L);
      } else {
        // cross-CTA split combine: publish (M,L,O) and let the last arriver finish (deterministic order)
        float* sb0 = P.split_buf + (((size_t)(seq * nkv + kvh) * MAXSPLIT) * RMAX) * 130;
        float* sb = sb0 + ((size_t)sp * RMAX) * 130;
        if (rr_ < R) {
          if (dd == 0) { sb[rr_ * 130] = M; sb[rr_ * 130 + 1] = L; }
          sb[rr_ * 130 + 2 + dd] = O;
        }
        __threadfence();
        cta_sync();
        if (tid == 0) s_ticket = (int)atomicAdd(&P.st->split_cnt[seq * nkv + kvh], 1u);
        cta_sync();
        if (s_ticket == nsplit - 1) {
          __threadfence();
          if (rr_ < R) {
            float M2 = -INFINITY, L2 = 0.f, O2 = 0.f;
#pragma unroll 1
            for (int s2 = 0; s2 < nsplit; ++s2) M2 = fmaxf(M2, ldcgf(sb0 + ((size_t)s2 * RMAX + rr_) * 130));
#pragma unroll 1
            for (int s2 = 0; s2 < nsplit; ++s2) {
              const float* rp = sb0 + ((size_t)s2 * RMAX + rr_) * 130;
              const float mm = ldcgf(rp);
              const float wgt = (mm == -INFINITY) ? 0.f : __expf(mm - M2);
              L2 += ldcgf(rp + 1) * wgt;
              O2 += ldcgf(rp + 2 + dd) * wgt;
            }
            *outp = f2bf(O2 / L2);
          }
          if (tid == 0) P.st->split_cnt[seq * nkv + kvh] = 0;
        }
      }
      cta_sync();
    }
  }
}

}  // namespace
