// The persistent frame-step kernel and the host-side plan of a program it runs: tile assignment, shared-memory plan,
// weight-ring run table and the dynamic shared-memory budget.  The engine (ar_engine.cu) and the GEMV test shim
// (tests/csrc/gemv_shim.cu) both build their launches with these functions, so a test runs the same plan as the engine.
// Part of the ar_engine.cu translation unit (include order: ar_program, ar_gemv, ar_attention, ar_sampler, ar_step,
// ar_prefill).
#pragma once
#include <algorithm>
#include <vector>

namespace {

// ------------------------------------------------------------------------------------------------
// the persistent kernel
// ------------------------------------------------------------------------------------------------
// VAR: 0 = production, 1 = production + per-step hidden-state capture, 2 = profiled (hidden capture + device-timestamp
// marks).  See gemv_phase for why these are separate instantiations.
template <int NT, int VAR>
__global__ void __launch_bounds__(CTA_THREADS, 1) q3_step_kernel(const __grid_constant__ KParams P) {
  extern __shared__ __align__(1024) unsigned char smem[];
  __shared__ Phase s_ph[2];
  __shared__ RoundTab s_tab;
  DevState* st = P.st;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr bool HID = VAR >= 1, DEV = VAR == 2;
  unsigned int epoch = 0;  // host resets bar_count to 0 before every launch
  PMeta* meta = reinterpret_cast<PMeta*>(smem + P.plan.meta_off);
  const int R = P.plan.nslots, SB = P.plan.slot_blocks;
  const uint32_t full0 = smem_addr(smem + P.plan.bar_off);      // [NWARPS][R] full barriers, then the x barrier
  const uint32_t xbar = full0 + 8u * (NWARPS * R);
  uint32_t xpar = 0;
  const int niter = P.mode == 1 ? P.max_iters : 1;

  // ---- per-CTA phase metas: how many tiles of every phase this CTA owns
#pragma unroll 1
  for (int i = tid; i < P.n_phases; i += CTA_THREADS) {
    const Phase* gp = P.prog + i;
    PMeta m;
    m.woff16 = 0; m.ntc = 0; m.kb = 0;
    if (gp->type == PH_GEMV) {
      int t0, ntc;
      q3ring::cta_tiles(gp->tq, gp->tr, (int)blockIdx.x, t0, ntc);
      m.ntc = (uint16_t)ntc;
      m.kb = (uint16_t)gp->kb;
    }
    meta[i] = m;
  }
  if (tid == 0) {
    for (int i = 0; i < NWARPS * R + 1; ++i) mbar_init(full0 + 8u * i, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async;" ::: "memory");
    g_prof_row = nullptr;
  }
  if (tid < (int)(sizeof(Phase) / 4))
    reinterpret_cast<uint32_t*>(&s_ph[0])[tid] = reinterpret_cast<const uint32_t*>(P.prog)[tid];
  __syncthreads();
  if (s_ph[0].type == PH_GEMV && s_ph[0].norm_w != nullptr && tid < s_ph[0].kb * 4)
    reinterpret_cast<uint4*>(smem + P.plan.nw_off)[tid] = reinterpret_cast<const uint4*>(s_ph[0].norm_w)[tid];

  // L2 eviction priorities of the weight stream (createpolicy): the talker and the 15 heads are read once per
  // frame-step -> evict_first; the code predictor's layer weights (157 MB) are re-read on each of its 15 passes -> a
  // fixed, address-hashed fraction of their lines is evict_last, i.e. stays in L2 between passes and is not
  // re-fetched from HBM.  The kernel is latency-bound, so the effect is on DRAM traffic rather than on time.
  uint64_t pol_stream, pol_keep;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_stream));
  asm volatile("createpolicy.fractional.L2::evict_last.L2::evict_first.b64 %0, %1;" : "=l"(pol_keep) : "f"(P.keep_fraction));

  // ---- this warp's weight ring: start streaming before anything else happens
  Ring rg;
  rg.SB = SB; rg.R = R;
  rg.slots = smem_addr(smem + P.plan.ring_off) + (uint32_t)(warp * R * SB) * 1024u;
  rg.full = full0 + 8u * (warp * R);
  rg.c_slot = 0; rg.c_par = 0; rg.p_slot = 0; rg.outstanding = 0;
  {
    const uint32_t o0 = P.run_off[blockIdx.x * NWARPS + warp], o1 = P.run_off[blockIdx.x * NWARPS + warp + 1];
    ring_init(rg, P.runs + o0, (int)(o1 - o0), (long long)(o1 - o0) * niter);
  }
#pragma unroll 1
  for (int i = 0; i < R; ++i) ring_issue(rg, P, lane, pol_stream, pol_keep);
  __syncthreads();

  const int step_base = st->step;
  int iters_done = 0;
  int slot = 0;
#pragma unroll 1
  for (int it = 0; it < niter; ++it) {
    const int frame = step_base + it;
    if (P.mode == 1) {
      bool all = true;
      for (int b = 0; b < P.B; ++b) all = all && (ldcgi(&st->finished[b]) != 0);
      if (all) break;
    }
#pragma unroll 1
    for (int pi = 0; pi < P.n_phases; ++pi) {
      // descriptor of this phase sits in s_ph[slot] (fetched one phase ahead).  The load of the NEXT descriptor is
      // issued now into a register and only stored to smem after the body, so its L2 round trip is hidden.
      int nx = pi + 1;
      if (nx >= P.n_phases) nx = (P.mode == 1) ? 0 : -1;
      const bool dhave = nx >= 0 && tid < (int)(sizeof(Phase) / 4);
      uint32_t dreg = 0;
      if (dhave) dreg = reinterpret_cast<const uint32_t*>(P.prog + nx)[tid];
      const Phase& ph = s_ph[slot];
      if (tid == 0) {
        if constexpr (DEV) g_prof_row = (P.prof && it == 0) ? P.prof + ((size_t)pi * gridDim.x + blockIdx.x) * 16 : nullptr;
        PROF_MARK(6);
      }
      const int type = ph.type;
      if (type == PH_GEMV) xpar = gemv_phase<NT, HID, DEV>(ph, meta[pi], P, rg, smem, &s_tab, xbar, xpar, pol_stream, pol_keep, frame);
      else if (type == PH_ATTN) attn_phase<DEV>(ph, P, smem + P.plan.x_off, frame);
      else sample_phase(ph, P, smem + P.plan.x_off, frame, P.mode == 0);
      if (dhave) reinterpret_cast<uint32_t*>(&s_ph[slot ^ 1])[tid] = dreg;
      cta_sync();  // body done (global writes of every thread precede thread 0's release), next descriptor visible
      PROF_MARK(0);
      grid_arrive(st, epoch);
      // work that does not depend on the other CTAs, between arrive and wait: the next GEMV's RMSNorm weights
      // (load now, store after the wait) and the KV rows the next attention phase will need
      uint4 nwv = make_uint4(0, 0, 0, 0);
      bool nw_have = false;
      if (nx >= 0) {
        const Phase& nph = s_ph[slot ^ 1];
        if (nph.type == PH_GEMV && nph.norm_w != nullptr && tid < nph.kb * 4) {
          nwv = reinterpret_cast<const uint4*>(nph.norm_w)[tid];
          nw_have = true;
        } else if (nph.type == PH_ATTN) {
          attn_prefetch(nph, P, smem + P.plan.x_off, pi + 1 >= P.n_phases ? frame + 1 : frame);
        }
      }
      grid_wait(st, epoch);
      slot ^= 1;
      if (nw_have) reinterpret_cast<uint4*>(smem + P.plan.nw_off)[tid] = nwv;
      cta_sync();
      PROF_MARK(1);
    }
    ++iters_done;
  }
  // never leave with bulk copies in flight into this CTA's shared memory (early exit: every row finished)
#pragma unroll 1
  while (rg.outstanding > 0) {
    mbar_wait(rg.full + 8u * rg.c_slot, (uint32_t)rg.c_par, st);
    if (++rg.c_slot == rg.R) { rg.c_slot = 0; rg.c_par ^= 1; }
    --rg.outstanding;
  }
  if (P.mode == 1 && blockIdx.x == 0 && tid == 0) st->step = step_base + iters_done;
}

// every instantiation, by variant (rows) and batch class 1 / 2 / 4 (columns)
const void* const kStepKernels[3][3] = {
    {(const void*)q3_step_kernel<1, 0>, (const void*)q3_step_kernel<2, 0>, (const void*)q3_step_kernel<4, 0>},
    {(const void*)q3_step_kernel<1, 1>, (const void*)q3_step_kernel<2, 1>, (const void*)q3_step_kernel<4, 1>},
    {(const void*)q3_step_kernel<1, 2>, (const void*)q3_step_kernel<2, 2>, (const void*)q3_step_kernel<4, 2>}};


// ------------------------------------------------------------------------------------------------
// host-side plan of a program (plain arguments: the engine uploads the results through its DevStore)
// ------------------------------------------------------------------------------------------------
// Balanced contiguous split of every GEMV phase's tiles over `grid` CTAs (q3ring::cta_tiles reads it back).
void assign_tiles(std::vector<Phase>& prog, int grid) {
  for (Phase& p : prog)
    if (p.type == PH_GEMV) { p.tq = p.n_tiles / grid; p.tr = p.n_tiles % grid; }
}

// Run table of a program: for every (CTA, warp) the sequence of contiguous weight runs (offset from the weight arena
// base `wbase` in 16-byte units, number of 1 KB blocks) of ONE pass over the program, enumerated with the same iterator
// the model check in tests/test_ring_model.py exercises.  The kernel's consumer loop derives the same runs from
// run_geom().  `runs` gets the runs, `off` the [grid * NWARPS + 1] start of each (CTA, warp) list.
int build_run_table(const std::vector<Phase>& prog, int grid, const char* wbase, int keep_phases, std::vector<uint2>* runs,
                    std::vector<uint32_t>* off) {
  const int n = (int)prog.size();
  std::vector<uint2>& pieces = *runs;
  pieces.clear();
  off->clear();
  off->reserve((size_t)grid * NWARPS + 1);
  std::vector<q3ring::PMeta> meta(n);
  for (int cta = 0; cta < grid; ++cta) {
    for (int i = 0; i < n; ++i) {
      q3ring::PMeta m{0, 0, 0};
      if (prog[i].type == PH_GEMV) {
        int t0, ntc;
        q3ring::cta_tiles(prog[i].tq, prog[i].tr, cta, t0, ntc);
        m.ntc = (uint16_t)ntc;
        m.kb = (uint16_t)prog[i].kb;
        const size_t byte_off = (size_t)(reinterpret_cast<const char*>(prog[i].w) - wbase) + (size_t)t0 * prog[i].kb * 1024;
        Q3_REQUIRE((byte_off >> 4) < ((size_t)1 << 32) && (byte_off & 15) == 0, "weight offset out of range / unaligned");
        m.woff16 = (uint32_t)(byte_off >> 4);
      }
      meta[i] = m;
    }
    for (int warp = 0; warp < NWARPS; ++warp) {
      off->push_back((uint32_t)pieces.size());
      q3ring::ProdIter it;
      q3ring::prod_init(it);
      q3ring::prod_next_run(it, meta.data(), n, 1, warp);
      while (!it.done) {
        // bit 31 of the length: the run belongs to weights that are re-read within a frame-step (the code predictor's
        // LAYERS: phases before keep_phases that are not an LM head / projection) -> L2 evict_last fraction
        const Phase& ph = prog[it.pi];
        const bool keep = it.pi < keep_phases && ph.epi != EPI_LOGITS && ph.epi != EPI_BIAS;
        pieces.push_back(make_uint2((uint32_t)(q3ring::prod_piece_offset(it) >> 4), (uint32_t)(it.u1 - it.u) | (keep ? 0x80000000u : 0u)));
        q3ring::prod_next_run(it, meta.data(), n, 1, warp);
      }
    }
  }
  off->push_back((uint32_t)pieces.size());
  return 0;
}

// Shared-memory plan of one program at one batch class (layout: ar_program.cuh) within `max_dyn_smem` bytes of dynamic
// shared memory.  Marks every GEMV phase as staged (activations copied to the x area once, B fragments read from shared
// memory) or not (B fragments straight from L2: only inputs that do not fit, i.e. K = intermediate_size at B > 8).
int make_smem_plan(std::vector<Phase>& prog, int B, int nt, int max_dyn_smem, SmemPlan* out) {
  const int budget = x_budget_nt(nt);
  int xneed = X_MIN_BYTES;
  for (Phase& p : prog) {
    if (p.type != PH_GEMV) continue;
    const int nc = p.ncmode == NC_B ? B : 2 * B;
    const int need = xs_stride_bytes(p.kb * 32) * ((nc + 7) / 8 * 8);
    p.staged = need <= budget ? 1 : 0;
    Q3_REQUIRE(p.staged || p.norm_w == nullptr, "normed GEMV input of %d columns x K=%d does not fit the x area", nc, p.kb * 32);
    if (p.staged) xneed = std::max(xneed, need);
  }
  SmemPlan pl{};
  auto up = [](int v, int a) { return (v + a - 1) / a * a; };
  pl.x_off = 0; pl.x_bytes = up(xneed, 1024);
  pl.part_off = pl.x_off + pl.x_bytes;
  pl.nw_off = pl.part_off + part_bytes_nt(nt);
  pl.ring_off = up(pl.nw_off + NW_BYTES, 1024);
  const int meta_bytes = up((int)prog.size() * (int)sizeof(q3ring::PMeta), 16);
  const int bar_bytes = 8 * (NWARPS * MAX_SLOTS + 1) + 8;  // one full barrier per ring slot, the x barrier
  // batch classes 1-2 stay under the 196 KB carve-out (195 KB per CTA) so that 32 KB of the SM remain L1: the phase
  // functions' stack traffic then hits L1 instead of making an L2 round trip each
  int limit = max_dyn_smem;
  if (nt <= 2) limit = std::min(limit, 195 * 1024 - (SMEM_OPTIN - max_dyn_smem) - 256);
  const int avail = limit - pl.ring_off - meta_bytes - bar_bytes;
  pl.slot_blocks = 0;
  const int sb_first = nt == 4 ? 2 : 4;  // the largest batch class keeps its B fragments of a piece in registers: 2-block pieces
  for (int sb : {sb_first, 2, 1}) {
    const int r = avail / (NWARPS * sb * 1024);
    if (r >= 2) { pl.slot_blocks = sb; pl.nslots = std::min(r, MAX_SLOTS); break; }
  }
  Q3_REQUIRE(pl.slot_blocks > 0, "no shared memory left for the weight rings (x area %d B, batch class %d)", pl.x_bytes, nt);
  pl.meta_off = pl.ring_off + NWARPS * pl.nslots * pl.slot_blocks * 1024;
  pl.bar_off = pl.meta_off + meta_bytes;
  pl.total = pl.bar_off + bar_bytes;
  Q3_REQUIRE(pl.total <= max_dyn_smem, "shared-memory plan of %d B exceeds %d B", pl.total, max_dyn_smem);
  *out = pl;
  return 0;
}

// Dynamic shared-memory budget of the plans: all opt-in shared memory minus the largest static part of any
// instantiation, and every instantiation allowed to request it.
int step_kernels_set_max_dyn_smem(int* max_dyn_smem) {
  int stat = 0;
  for (const auto& row : kStepKernels)
    for (const void* fn : row) {
      cudaFuncAttributes fa;
      Q3_CUDA(cudaFuncGetAttributes(&fa, fn));
      stat = std::max(stat, (int)fa.sharedSizeBytes);
    }
  *max_dyn_smem = SMEM_OPTIN - (stat + 127) / 128 * 128;
  for (const auto& row : kStepKernels)
    for (const void* fn : row) Q3_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, *max_dyn_smem));
  return 0;
}

}  // namespace
