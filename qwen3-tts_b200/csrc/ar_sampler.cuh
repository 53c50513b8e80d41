// Sample phase: HF logits processors, argmax / inverse-CDF sampling with Philox uniforms, next-input embedding.
// Part of the ar_engine.cu translation unit (include order: ar_program, ar_gemv, ar_attention, ar_sampler,
// the persistent kernel in ar_step, ar_prefill).
#pragma once

namespace {

// ------------------------------------------------------------------------------------------------
// sample phase: HF logits processors + argmax / inverse-CDF sampling + next-embed (one CTA per row)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned int fkey(float f) {
  unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// k-th largest of sv[0..V) (block-wide radix select over 4x8 bits); returns the threshold value
__device__ __noinline__ float kth_largest(const float* sv, int V, int k, unsigned int* hist, int* sh) {
  unsigned int prefix = 0, mask = 0;
#pragma unroll 1
  for (int pass = 3; pass >= 0; --pass) {
    const int shift = pass * 8;
    if (threadIdx.x < 256) hist[threadIdx.x] = 0;
    cta_sync();
#pragma unroll 1
    for (int i = threadIdx.x; i < V; i += NTHREADS) {
      const unsigned int key = fkey(sv[i]);
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
    }
    cta_sync();
    // suffix counts over the 256 bins (8 warps)
    unsigned int cnt = 0, incl = 0;
    if (threadIdx.x < 256) {
      cnt = hist[threadIdx.x];
      incl = cnt;
      const int ln = threadIdx.x & 31;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        unsigned int n = __shfl_down_sync(0xffffffffu, incl, o);
        if (ln + o < 32) incl += n;
      }
      if (ln == 0) sh[threadIdx.x >> 5] = (int)incl;  // warp totals
    }
    cta_sync();
    if (threadIdx.x < 256) {
      unsigned int above = 0;
#pragma unroll 1
      for (int w = (threadIdx.x >> 5) + 1; w < 8; ++w) above += (unsigned int)sh[w];
      incl += above;                       // elements with digit >= d
      const unsigned int excl = incl - cnt;  // elements with digit > d
      if ((int)excl < k && k <= (int)incl) { sh[8] = threadIdx.x; sh[9] = k - (int)excl; }
    }
    cta_sync();
    prefix |= ((unsigned int)sh[8]) << shift;
    mask |= 255u << shift;
    k = sh[9];
    cta_sync();
  }
  const unsigned int u = (prefix & 0x80000000u) ? (prefix & 0x7fffffffu) : ~prefix;
  return __uint_as_float(u);
}

// Fast path of the default sampling configuration (top-k with k <= 128, no top-p): exact top-k threshold from ONE
// histogram pass over a monotone 2048-bin key of (score - max) plus a rank count among the few scores of the
// threshold bin, then softmax + inverse CDF over the <= 384 kept scores in token-id order.  ~10 CTA syncs instead of
// the ~30 of the generic path (4-pass radix select + full-vocabulary scan); returns false (nothing decided) when a
// degenerate input (hundreds of ties, fewer than k finite scores) needs the generic path.
__device__ __noinline__ bool sample_fast(const float* sv, int V, int k, float u, float* scratch, float* red, int* ired, int* tok_out) {
  int* hist = reinterpret_cast<int*>(scratch);                      // [2048]
  float* cand = scratch + 2048;                                     // [256]
  int* kidx = reinterpret_cast<int*>(scratch + 2048 + 256);         // [384]
  float* kp = scratch + 2048 + 256 + 384;                           // [384]
  int* sidx = reinterpret_cast<int*>(scratch + 2048 + 256 + 768);   // [384]
  float* spp = scratch + 2048 + 256 + 1152;                         // [384]
  __shared__ int s_misc[8];  // 0 threshold bin, 1 rank inside it, 2 #candidates, 3 #kept, 4 threshold bits, 5 token
  const int tid = threadIdx.x, lane = tid & 31, wp = tid >> 5;
  float mx = -INFINITY;
#pragma unroll 1
  for (int i = tid; i < V; i += NTHREADS) mx = fmaxf(mx, sv[i]);
  mx = block_reduce(mx, red, 0);
#pragma unroll 1
  for (int i = tid; i < 2048; i += NTHREADS) hist[i] = 0;
  if (tid == 0) { s_misc[0] = -1; s_misc[2] = 0; s_misc[3] = 0; s_misc[4] = __float_as_int(-INFINITY); }
  cta_sync();
  const float lo = mx - 32.f;
#pragma unroll 1
  for (int i = tid; i < V; i += NTHREADS) {
    const float sc = sv[i];
    if (sc > -INFINITY) atomicAdd(&hist[min(2047, max(0, (int)((sc - lo) * 64.f)))], 1);
  }
  cta_sync();
  // thread t owns bins [8t, 8t+8); scores in a higher bin are strictly larger
  int hb[8], S = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) { hb[j] = hist[8 * tid + j]; S += hb[j]; }
  int incl = S;  // inclusive SUFFIX sum inside the warp (threads above me own larger scores)
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int n = __shfl_down_sync(0xffffffffu, incl, o);
    if (lane + o < 32) incl += n;
  }
  if (lane == 0) ired[wp] = incl;
  cta_sync();
  int above = incl - S;
#pragma unroll 1
  for (int w = wp + 1; w < NWARPS; ++w) above += ired[w];
  {
    int run = above;
#pragma unroll
    for (int j = 7; j >= 0; --j) {
      if (run < k && k <= run + hb[j]) { s_misc[0] = 8 * tid + j; s_misc[1] = k - run; }
      run += hb[j];
    }
  }
  cta_sync();
  const int tb = s_misc[0], kk = s_misc[1];
  if (tb < 0) return false;  // fewer than k finite scores
#pragma unroll 1
  for (int i = tid; i < V; i += NTHREADS) {
    const float sc = sv[i];
    if (sc > -INFINITY && min(2047, max(0, (int)((sc - lo) * 64.f))) == tb) {
      const int p = atomicAdd(&s_misc[2], 1);
      if (p < 256) cand[p] = sc;
    }
  }
  cta_sync();
  const int nc = s_misc[2];
  if (nc > 256) return false;
  if (tid < nc) {
    const float v = cand[tid];
    int gt = 0, ge = 0;
#pragma unroll 1
    for (int j = 0; j < nc; ++j) { const float w = cand[j]; gt += w > v; ge += w >= v; }
    if (gt < kk && kk <= ge) s_misc[4] = __float_as_int(v);  // (ties write the same value)
  }
  cta_sync();
  const float thr = __int_as_float(s_misc[4]);
  // kept set (HF keeps everything >= the k-th largest: ties at the threshold stay)
#pragma unroll 1
  for (int i = tid; i < V; i += NTHREADS) {
    const float sc = sv[i];
    if (sc > -INFINITY && sc >= thr) {
      const int p = atomicAdd(&s_misc[3], 1);
      if (p < 384) { kidx[p] = i; kp[p] = __expf(sc - mx); }
    }
  }
  cta_sync();
  const int m = s_misc[3];
  if (m > 384 || m == 0) return false;
  // token-id order by rank counting (the arrival order of the atomics is not deterministic, the ids are)
#pragma unroll 1
  for (int e = tid; e < m; e += NTHREADS) {
    const int id = kidx[e];
    int r = 0;
#pragma unroll 1
    for (int j = 0; j < m; ++j) r += kidx[j] < id;
    sidx[r] = id;
    spp[r] = kp[e];
  }
  cta_sync();
  if (tid < 32) {  // inverse CDF over the sorted kept set
    const int per = (m + 31) >> 5;
    const int a = min(m, lane * per), bnd = min(m, a + per);
    float loc = 0.f;
#pragma unroll 1
    for (int j = a; j < bnd; ++j) loc += spp[j];
    float inc = loc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float n = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += n;
    }
    const float total = __shfl_sync(0xffffffffu, inc, 31);
    const float target = u * total;
    float run = inc - loc;
    int cnd = 0x7fffffff;
#pragma unroll 1
    for (int j = a; j < bnd; ++j) {
      run += spp[j];
      if (run > target && cnd == 0x7fffffff && spp[j] > 0.f) cnd = j;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnd = min(cnd, __shfl_xor_sync(0xffffffffu, cnd, o));
    if (cnd == 0x7fffffff) {  // rounding pushed the target past the last partial sum: take the last token with p > 0
      int last = -1;
#pragma unroll 1
      for (int j = a; j < bnd; ++j)
        if (spp[j] > 0.f) last = j;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
      cnd = max(last, 0);
    }
    if (lane == 0) s_misc[5] = sidx[cnd];
  }
  cta_sync();
  *tok_out = s_misc[5];
  return true;
}

__device__ __forceinline__ void sample_phase(const Phase& ph, const KParams& P, unsigned char* smem, int frame, bool in_prefill) {
  const int b = blockIdx.x;
  DevState* st = P.st;
  const int B = P.B;
  if (b >= B) return;
  if (in_prefill && !((P.admit_mask >> b) & 1u)) return;  // admission prefill: rows already running keep their state
  frame -= P.frame0[b];  // the row's own frame counter (continuous batching admits rows at different global frames)
  const int tid = threadIdx.x;
  const int group = ph.group;
  const bool talker = group == 0;
  const StackDev& S = talker ? P.talker : P.cp;
  const int V = S.vocab;
  const int H = P.talker.hidden;
  if (talker && !in_prefill && ((P.text_open >> b) & 1u) && frame >= P.trailing_len[b]) {
    // held step (live text): this step's talker input needed trailing[frame], which has not arrived.  Nothing of the
    // sample is committed; the code predictor's input is put back to what the last committed sample left (its passes
    // may have run in place on it), so the step can run again, bit for bit, once the text is there.
    const bf16* e = P.emb_t + (size_t)ldcgi(&st->c0[b]) * H;
    const bf16* k = P.past_keep + (size_t)b * H;
#pragma unroll 1
    for (int i = tid * 8; i < H; i += NTHREADS * 8) {
      *reinterpret_cast<uint4*>(P.x_cp + ((size_t)B + b) * H + i) = *reinterpret_cast<const uint4*>(e + i);
      *reinterpret_cast<uint4*>(P.x_cp + (size_t)b * H + i) = ldcg16(k + i);
    }
    return;
  }
  float* sv = reinterpret_cast<float*>(smem);       // [MAXV]
  float* pv = sv + MAXV;                            // [MAXV]
  float* red = pv + MAXV;                           // [32]
  int* ired = reinterpret_cast<int*>(red + 32);     // [32]
  unsigned int* hist = reinterpret_cast<unsigned int*>(ired + 32);  // [256]
  // frame index of the token being sampled
  const int fidx = talker ? (in_prefill ? 0 : frame + 1) : frame;
  // this row's parameters: its own entry of the per-row table (each request of a session samples with its own), or the
  // launch-wide set.  Every choice below (greedy, fast or generic path) is made per row.
  const q3_sampling& sp = P.row_sampling ? P.row_sp[b] : P.sp;
  const bool do_sample = talker ? sp.do_sample : sp.subtalker_dosample;
  const float temperature = talker ? sp.temperature : sp.subtalker_temperature;
  const int top_k = talker ? sp.top_k : sp.subtalker_top_k;
  const float top_p = talker ? sp.top_p : sp.subtalker_top_p;
  const float* lg = S.logits + (size_t)b * V;
  const int n_gen_b = talker ? ldcgi(&st->n_gen[b]) : 0;

  // raw logits -> smem with all loads of a thread in flight, then a rolled processing pass
  {
    float lreg[MAXV / NTHREADS];
#pragma unroll
    for (int r = 0; r < MAXV / NTHREADS; ++r) { const int i = tid + r * NTHREADS; if (i < V) lreg[r] = ldcgf(lg + i); }
#pragma unroll
    for (int r = 0; r < MAXV / NTHREADS; ++r) { const int i = tid + r * NTHREADS; if (i < V) sv[i] = lreg[r]; }
  }
  float* dbg = talker ? (P.dbg_tlogits ? P.dbg_tlogits + ((size_t)fidx * B + b) * V : nullptr)
                      : (P.dbg_clogits ? P.dbg_clogits + (((size_t)frame * (P.G - 1) + (group - 1)) * B + b) * V : nullptr);
  const float rp = sp.repetition_penalty;
  const float inv_t = (do_sample && temperature != 1.0f) ? temperature : 1.0f;
#pragma unroll 1
  for (int i = tid; i < V; i += NTHREADS) {
    float s = sv[i];
    if (dbg) dbg[i] = s;
    if (talker) {
      // 1. repetition penalty over generated codebook-0 tokens
      if (rp != 1.0f && __ldcg(P.seen + (size_t)b * V + i)) s = s < 0.f ? s * rp : s / rp;
      // 2. min_new_tokens (and the fixed-horizon benchmark switch)
      if (i == P.eos && (n_gen_b < sp.min_new_tokens || sp.suppress_eos)) s = -INFINITY;
      // 3. suppress [V-1024, V) \ {eos}
      if (i >= V - 1024 && i != P.eos) s = -INFINITY;
    }
    if (inv_t != 1.0f) s = s / inv_t;
    sv[i] = s;
  }
  cta_sync();

  int tok;
  if (!do_sample) {
    float mx = -INFINITY;
#pragma unroll 1
    for (int i = tid; i < V; i += NTHREADS) mx = fmaxf(mx, sv[i]);
    mx = block_reduce(mx, red, 0);
    int idx = 0x7fffffff;
#pragma unroll 1
    for (int i = tid; i < V; i += NTHREADS)
      if (sv[i] == mx) idx = min(idx, i);
    tok = block_min_int(idx, ired);
  } else if (top_p >= 1.0f && top_k > 0 && top_k < V && top_k <= 128 &&
             sample_fast(sv, V, top_k, philox_uniform(sp.seed, P.row_key[b], (uint32_t)fidx, (uint32_t)group), pv, red, ired, &tok)) {
    // (decided by the fast path)
  } else {
    if (top_k > 0 && top_k < V) {
      const float thr = kth_largest(sv, V, top_k, hist, ired);
#pragma unroll 1
      for (int i = tid; i < V; i += NTHREADS)
        if (sv[i] < thr) sv[i] = -INFINITY;
      cta_sync();
    }
    float mx = -INFINITY;
#pragma unroll 1
    for (int i = tid; i < V; i += NTHREADS) mx = fmaxf(mx, sv[i]);
    mx = block_reduce(mx, red, 0);
    if (top_p < 1.0f) {
      // ascending-order cumulative softmax <= 1-p is removed, highest kept (O(n^2) over the kept set)
      float tot = 0.f;
#pragma unroll 1
      for (int i = tid; i < V; i += NTHREADS) { const float p = __expf(sv[i] - mx); pv[i] = p; tot += p; }
      tot = block_reduce(tot, red, 1);
      cta_sync();
      unsigned int rm_mask = 0;  // removal flags stay in registers until every thread has finished reading pv/sv
      int slot = 0;
#pragma unroll 1
      for (int i = tid; i < V; i += NTHREADS, ++slot) {
        const float si = sv[i];
        bool rm = false;
        if (si != -INFINITY) {
          float cum = 0.f;
          bool is_top = true;
#pragma unroll 1
          for (int j = 0; j < V; ++j) {
            const float sj = sv[j];
            if (sj == -INFINITY) continue;
            if (sj < si || (sj == si && j <= i)) cum += pv[j];
            if (sj > si || (sj == si && j > i)) is_top = false;
          }
          rm = (cum / tot <= 1.0f - top_p) && !is_top;
        }
        if (rm) rm_mask |= 1u << slot;
      }
      cta_sync();
      slot = 0;
#pragma unroll 1
      for (int i = tid; i < V; i += NTHREADS, ++slot)
        if (rm_mask & (1u << slot)) sv[i] = -INFINITY;
      cta_sync();
    }
    // softmax + inverse CDF in token-id order (blocked mapping for the scan)
    const int E = (V + NTHREADS - 1) / NTHREADS;
    const int i0 = tid * E, i1 = min(V, i0 + E);
    float loc = 0.f;
#pragma unroll 1
    for (int i = i0; i < i1; ++i) { const float p = __expf(sv[i] - mx); pv[i] = p; loc += p; }
    // block inclusive scan of loc
    float incl = loc;
    const int ln = tid & 31, wp = tid >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float n = __shfl_up_sync(0xffffffffu, incl, o);
      if (ln >= o) incl += n;
    }
    cta_sync();
    if (ln == 31) red[wp] = incl;
    cta_sync();
    float base = 0.f, total = 0.f;
#pragma unroll 1
    for (int w = 0; w < NWARPS; ++w) { if (w < wp) base += red[w]; total += red[w]; }
    const float excl = base + incl - loc;
    const float u = philox_uniform(sp.seed, P.row_key[b], (uint32_t)fidx, (uint32_t)group);
    const float target = u * total;
    int cand = 0x7fffffff, lastpos = -1;
    float run = excl;
#pragma unroll 1
    for (int i = i0; i < i1; ++i) {
      run += pv[i];
      if (pv[i] > 0.f) { lastpos = i; if (run > target && cand == 0x7fffffff) cand = i; }
    }
    cand = block_min_int(cand, ired);
    if (cand == 0x7fffffff) cand = -block_min_int(-lastpos, ired);
    tok = cand;
  }
  // teacher forcing (tests)
  if (P.forced && fidx < P.n_forced) {
    const int f = P.forced[((size_t)b * P.n_forced + fidx) * P.G + group];
    if (f >= 0) tok = f;
  }

  if (talker) {
    const int was_finished = ldcgi(&st->finished[b]);
    if (was_finished) tok = P.eos;  // HF pads finished rows with pad_token_id (= eos)
    cta_sync();
    if (tid == 0) {
      if (!was_finished) {
        if (tok == P.eos) { st->finished[b] = 1; st->n_valid[b] = fidx; }
        else { P.seen[(size_t)b * V + tok] = 1; }
        st->n_gen[b] = n_gen_b + 1;
      }
      st->c0[b] = tok;
      st->cur[b][0] = tok;
    }
    // CP input for the next frame: token 0 = past_hidden (already saved by the head phase), token 1 = E0[c0]
    bf16* x1 = P.x_cp + ((size_t)B + b) * H;
    bf16* x0 = P.x_cp + (size_t)b * H;
    const bf16* e = P.emb_t + (size_t)tok * H;
    const bf16* ph_ = P.past_hidden + (size_t)b * H;
    bf16* keep = P.past_keep ? P.past_keep + (size_t)b * H : nullptr;  // (a caller that never opens a row may leave it unset)
#pragma unroll 1
    for (int i = tid * 8; i < H; i += NTHREADS * 8) {
      *reinterpret_cast<uint4*>(x1 + i) = *reinterpret_cast<const uint4*>(e + i);
      const uint4 v = ldcg16(ph_ + i);
      *reinterpret_cast<uint4*>(x0 + i) = v;
      if (keep) *reinterpret_cast<uint4*>(keep + i) = v;
    }
  } else {
    const int j = group;  // codebook index 1..G-1
    if (tid == 0) {
      st->cur[b][j] = tok;
      if (P.codes_out && frame >= 0 && frame < P.codes_stride) {
        int* row = P.codes_out + ((size_t)b * P.codes_stride + frame) * P.G;
        row[j] = tok;
        if (j == 1) row[0] = ldcgi(&st->cur[b][0]);
      }
    }
    cta_sync();
    const int Vc = P.cp.vocab;
    if (j < P.G - 1) {
      // input of the next pass: codec_embedding[j-1](c_j)  (:1281)
      // (with the projection table the row is small_to_mtp_projection(embedding) already, :1283, and lands in cp.h)
      const int Wn = P.cp_next_w;
      const bf16* e = P.cp_next + ((size_t)(j - 1) * Vc + tok) * Wn;
      bf16* x = P.cp_next_dst + (size_t)b * Wn;
#pragma unroll 1
      for (int i = tid * 8; i < Wn; i += NTHREADS * 8)
        *reinterpret_cast<uint4*>(x + i) = *reinterpret_cast<const uint4*>(e + i);
    } else {
      // next talker input: sum of the 16 codebook embeddings (fp32 sum, one bf16 rounding) + text (:1682-1692)
      const bf16* txt = (frame < P.trailing_len[b])
                            ? P.trailing + ((size_t)b * P.trailing_stride + frame) * H
                            : P.tts_pad;
      int* codes = reinterpret_cast<int*>(hist);  // smem scratch: the 16 codes of this frame
      if (tid < P.G) codes[tid] = (tid == j) ? tok : ldcgi(&st->cur[b][tid]);
      cta_sync();
#pragma unroll 1
      for (int i = tid; i < H; i += NTHREADS) {
        float s = bf2f(P.emb_t[(size_t)codes[0] * H + i]);
#pragma unroll 4
        for (int g2 = 1; g2 < P.G; ++g2) s += bf2f(P.emb_cp[((size_t)(g2 - 1) * Vc + codes[g2]) * H + i]);
        P.talker.h[(size_t)b * H + i] = f2bf(rbf(s) + bf2f(txt[i]));
      }
    }
  }
}

}  // namespace
