// AR hot path of Qwen3-TTS on H100 (sm_90a): talker + 15-pass code predictor + logits processing + sampling
// + next-embed as ONE persistent cooperative kernel per group of frame-steps.
//
// Replaces (reference, paths relative to /root/reference/qwen_tts/core/models/modeling_qwen3_tts.py):
//   decode step  :1669-1744   code predictor :1250-1312 / :1671-1680   layers :1393-1424, :985-1012
//   attention    :761-805, :916-958, :634-657   RMSNorm :605-610   RoPE :660-724, :858-882   MLP :853-855
//   sampling     HF processors configured at :2044-2066 (semantics restated in oracle/sampler.py)
//
// Design (see DESIGN.md):
//   * the step is a "phase program": GEMV / attention / sample phases separated by a software grid barrier;
//     one CTA per SM, all CTAs walk the same program (cooperative launch guarantees co-residency).
//   * GEMV phases stream weights exactly once per step, straight from HBM/L2 into mma.sync A-fragments
//     (weights are re-packed at load into 8x32 bf16 sub-tiles = 512 B contiguous per warp load; a K
//     permutation shared by A and B lets every lane use one 16-byte vector load per 8 k-values), batch
//     columns ride in the N dimension (n8 tiles), fp32 accumulate, cross-warp split-K reduced in smem.
//   * the next phase's weight slice is pulled into L2 with cp.async.bulk.prefetch.L2 before a CTA waits on
//     the barrier, so HBM keeps streaming across the dependency bubbles.
//   * rounding points mirror the PyTorch bf16 path (linear outputs, RMSNorm, RoPE, residual adds are
//     rounded to bf16 exactly where the reference rounds).
#include "common.cuh"
#include "dev_store.h"
#include "gemm_sm90.cuh"
#include "../../include/qwen3tts_b200.h"

#include <cooperative_groups.h>
#include <stdarg.h>
#include <algorithm>
#include <cmath>
#include <map>
#include <memory>
#include <vector>

thread_local std::string g_q3_err;
int q3_set_err(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_q3_err = buf;
  return 1;
}

#include "ar_ring.cuh"
#include "ar_program.cuh"
#include "ar_gemv.cuh"
#include "ar_attention.cuh"
#include "ar_sampler.cuh"
#include "ar_step.cuh"  // the persistent kernel q3_step_kernel and the host-side plan of its programs
#include "ar_prefill.cuh"

// =================================================================================================
// host side
// =================================================================================================
struct PackedW {
  uint4* w = nullptr;
  int n = 0, k = 0;
};

// device copy of a program's ring-piece table (see ar_gemv.cuh: weight rings)
struct PieceTable {
  uint2* runs = nullptr;
  uint32_t* off = nullptr;
  size_t n_runs = 0;
};

// the weights one talker layer of the prefill reads: its norms and the plain [N][K] copies of its GEMM weights
struct PfLayer {
  const bf16 *ln1, *ln2, *qn, *kn, *qkv, *o, *gate_up, *down;
};

constexpr char kEngineName[] = "AR engine";

struct q3_engine {
  q3_engine_cfg cfg;
  int sm_count = 0;
  size_t l2_bytes = 0;
  cudaStream_t copy_stream = nullptr;
  // every device block: norms, biases, embeddings, rope tables and the plain [N][K] copies of the talker layer weights
  // for the wgmma prefill GEMMs as named tensors; the packed GEMV weights and the buffers below as blocks
  DevStore store{kEngineName};
  std::map<std::string, PackedW> packed;   // GEMV weights
  std::vector<PfLayer> pf_layers;          // resolved at finalize
  const bf16 *emb_t = nullptr, *emb_cp = nullptr;  // talker / code-predictor codec embeddings, resolved at finalize
  bf16 *pf_x = nullptr, *pf_xn = nullptr, *pf_qkv = nullptr, *pf_attn = nullptr, *pf_act = nullptr;
  int *pf_seq = nullptr, *pf_pos = nullptr;
  int pf_cap = 0;
  // device buffers
  DevState* st = nullptr;
  StackDev talker{}, cp{};
  bf16 *x_cp = nullptr, *past_hidden = nullptr, *past_keep = nullptr, *h_last = nullptr;
  bf16 *trailing = nullptr, *tts_pad = nullptr;
  int trailing_cap = 0;
  size_t trailing_alloc = 0;
  int max_len0 = 0, frames_issued = 0;
  int len0[MAXB] = {0}, trailing_len[MAXB] = {0};   // len0 is stored as prompt length - frame0 (see KParams)
  int frame0[MAXB] = {0};
  unsigned int row_key[MAXB] = {0};
  bool active[MAXB] = {false};
  // live text (q3_set_trailing_open): rows whose text may still grow, and rows whose last decode ended held at a step
  // whose text row had not arrived (that step's code-predictor half, i.e. one more frame of codes, is done)
  bool text_open[MAXB] = {false}, held[MAXB] = {false};
  bool session = false;       // continuous-batching session (q3_session_begin / q3_admit_with_sampling)
  unsigned int admit_mask = 0xffffffffu;
  unsigned char* seen = nullptr;
  float* split_buf = nullptr;
  Phase* prog_dev = nullptr;
  int prog_cap = 0;
  // programs (host copies) for the current batch size
  int prog_B = -1;
  const char* wbase = nullptr;  // lowest packed-weight address (PMeta offsets)
  float keep_fraction = 0.5f;
  int cp_phases = 0;
  int nt_frame = 1, nt_head = 1, max_dyn_smem = 0;
  SmemPlan plan_frame{}, plan_head{};
  PieceTable pt_frame{}, pt_head{};
  bf16* proj_tab = nullptr;   // small_to_mtp_projection(cp.codec_embedding) [(G-1)*Vc][Hc], built once at finalize
  std::vector<Phase> prog_head, prog_frame;
  int off_head = 0, off_frame = 0;
  q3_sampling sp{};           // default parameters: those of a static batch / a session's, and of rows without a request
  q3_sampling row_sp[MAXB]{}; // each admitted row's own parameters
  bool finalized = false;
  int B = 0;
  int codes_stride = 0;
  const int* forced = nullptr;
  bf16* hid_out = nullptr;
  int hid_stride = 0;
  int n_forced = 0;
  float *dbg_t = nullptr, *dbg_c = nullptr;
  unsigned long long* prof = nullptr;
  size_t smem_bytes = 0;
  double w_talker_bytes = 0, w_cp_unique_bytes = 0, w_cp_stream_bytes = 0;
  // registered prompt prefixes (q3_prefix_create): their talker K/V, [2 (K, V)][layers][nkv][len][HD]
  struct Prefix { bf16* kv; int len; };
  std::map<int, Prefix> prefixes;
  int next_prefix = 0;
  // parked rows of the current session (q3_row_park): a device block each, laid out by record_layout, and the host state
  // that resume restores.  Ids count on across sessions; first_record is the first id of the current one.
  struct Record {
    unsigned char* blk;
    int pos, f, trailing_len;  // position of the row's next step, its committed frames, its trailing rows
    unsigned int key;
    q3_sampling sp;
    bool text_open, held;
  };
  std::map<int, Record> records;
  int next_record = 0, first_record = 0;

  ~q3_engine() {
    if (copy_stream) cudaStreamDestroy(copy_stream);
  }
};

// the engine's own blocks are zero-filled (allocation is a load-time or growth-time event; nothing on the per-step
// path allocates)
static int stack_alloc(q3_engine* e, StackDev& S, const q3_stack_cfg& c, int nseq, int cap, int cols) {
  S.hidden = c.hidden_size; S.layers = c.num_layers; S.nh = c.num_heads; S.nkv = c.num_kv_heads;
  S.inter = c.intermediate_size; S.vocab = c.vocab_size; S.eps = c.rms_eps; S.cap = cap;
  DevStore& store = e->store;
  if (store.alloc(&S.h, (size_t)cols * c.hidden_size, true)) return 1;
  if (store.alloc(&S.qkv, (size_t)cols * (c.num_heads + 2 * c.num_kv_heads) * HD, true)) return 1;
  if (store.alloc(&S.attn, (size_t)cols * c.num_heads * HD, true)) return 1;
  if (store.alloc(&S.act, (size_t)cols * c.intermediate_size, true)) return 1;
  const size_t kv = (size_t)nseq * c.num_layers * c.num_kv_heads * cap * HD;
  if (store.alloc(&S.kc, kv, true)) return 1;
  if (store.alloc(&S.vc, kv, true)) return 1;
  if (store.alloc(&S.logits, (size_t)MAXB * c.vocab_size, true)) return 1;
  return 0;
}

extern "C" int q3_abi_version(void) { return Q3_ABI_VERSION; }
extern "C" const char* q3_last_error(void) { return g_q3_err.c_str(); }

extern "C" int q3_engine_create(const q3_engine_cfg* cfg, q3_engine** out) {
  Q3_REQUIRE(cfg && out, "null argument");
  Q3_REQUIRE(cfg->talker.head_dim == HD && cfg->cp.head_dim == HD, "head_dim must be 128");
  Q3_REQUIRE(cfg->max_batch >= 1 && cfg->max_batch <= MAXB, "max_batch must be in [1,%d]", MAXB);
  Q3_REQUIRE(cfg->num_code_groups >= 2 && cfg->num_code_groups <= Q3_NUM_GROUPS_MAX, "bad num_code_groups");
  Q3_REQUIRE(cfg->talker.vocab_size <= MAXV && cfg->cp.vocab_size <= MAXV, "vocab > %d unsupported", MAXV);
  Q3_REQUIRE(cfg->talker.vocab_size >= 1024, "talker vocab must be >= 1024 (suppress range)");
  for (const q3_stack_cfg* s : {&cfg->talker, &cfg->cp}) {
    Q3_REQUIRE(s->hidden_size % 32 == 0 && s->intermediate_size % 32 == 0 && s->vocab_size % 16 == 0,
               "hidden/intermediate must be multiples of 32 and vocab of 16");
    Q3_REQUIRE(s->num_heads % s->num_kv_heads == 0 && s->num_heads / s->num_kv_heads <= RMAX, "GQA group (heads / kv_heads) must be <= 2");
    Q3_REQUIRE(xs_stride_bytes(s->hidden_size) * MAXCOLS <= x_budget_nt(4) && s->hidden_size <= 2048,
               "hidden_size above 2048 unsupported");
  }
  Q3_REQUIRE(cfg->has_cp_projection || cfg->talker.hidden_size == cfg->cp.hidden_size,
             "Identity projection requires equal hidden sizes");
  Q3_CUDA(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  Q3_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
  Q3_REQUIRE(prop.major == 9 && prop.minor == 0, "this library is built for sm_90a (H100); device is sm_%d%d", prop.major, prop.minor);
  std::unique_ptr<q3_engine> e(new q3_engine());  // deleted on every failure below
  e->cfg = *cfg;
  e->sm_count = prop.multiProcessorCount;
  e->l2_bytes = (size_t)prop.l2CacheSize;
  Q3_CUDA(cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
  if (gemm_init()) return 1;
  DevStore& store = e->store;
  if (store.alloc(&e->st, 1, true)) return 1;
  if (stack_alloc(e.get(), e->talker, cfg->talker, cfg->max_batch, cfg->max_ctx, MAXCOLS)) return 1;
  if (stack_alloc(e.get(), e->cp, cfg->cp, cfg->max_batch, 32, MAXCOLS)) return 1;
  const int H = cfg->talker.hidden_size;
  if (store.alloc(&e->x_cp, (size_t)2 * MAXB * H, true)) return 1;
  if (store.alloc(&e->past_hidden, (size_t)MAXB * H, true)) return 1;
  if (store.alloc(&e->past_keep, (size_t)MAXB * H, true)) return 1;
  if (store.alloc(&e->h_last, (size_t)MAXB * H, true)) return 1;
  if (store.alloc(&e->tts_pad, (size_t)H, true)) return 1;
  if (store.alloc(&e->seen, (size_t)MAXB * cfg->talker.vocab_size, true)) return 1;
  if (store.alloc(&e->split_buf, (size_t)MAXB * cfg->talker.num_kv_heads * MAXSPLIT * RMAX * 130, true)) return 1;
  static_assert(SAMPLER_SMEM <= X_MIN_BYTES && ATT_SMEM <= X_MIN_BYTES, "attention / sampler scratch must fit the x area");
  Q3_REQUIRE((size_t)SMEM_OPTIN <= (size_t)prop.sharedMemPerBlockOptin, "not enough shared memory per block");
  *out = e.release();
  return 0;
}

extern "C" void q3_engine_destroy(q3_engine* e) { delete e; }

static bool is_gemv_weight(const std::string& n) {
  auto ends = [&](const char* s) { size_t l = strlen(s); return n.size() >= l && n.compare(n.size() - l, l, s) == 0; };
  if (ends(".qkv") || ends(".gate_up") || ends(".o") || ends(".down")) return true;
  if (n == "talker.codec_head" || n == "cp.proj") return true;
  if (n.rfind("cp.lm_head.", 0) == 0) return true;
  return false;
}

extern "C" int q3_engine_load_tensor(q3_engine* e, const char* name, const void* dev, int64_t rows, int64_t cols) {
  Q3_REQUIRE(e && name && dev, "null argument");
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  const std::string n(name);
  const int64_t shape[2] = {rows, cols};
  if (!is_gemv_weight(n)) return e->store.load(n, dev, shape, 2, DT_BF16);
  Q3_REQUIRE(rows % 16 == 0 && cols % 32 == 0, "%s: GEMV weight must be [16a][32b], got [%lld][%lld]", name,
             (long long)rows, (long long)cols);
  // `dev` may still be being produced on the caller's stream (a cat / cast queued by the framework): the ABI has
  // no stream argument here, so wait for the device once per tensor — a load-time cost only
  Q3_CUDA(cudaDeviceSynchronize());
  PackedW pw;
  pw.n = (int)rows; pw.k = (int)cols;
  if (e->store.alloc(&pw.w, (size_t)rows * cols / 8, false)) return 1;  // the pack kernel writes every element
  pack_weight_kernel<<<1024, 256, 0, e->copy_stream>>>(reinterpret_cast<const bf16*>(dev), pw.w, (int)rows, (int)cols);
  Q3_CUDA(cudaGetLastError());
  Q3_CUDA(cudaStreamSynchronize(e->copy_stream));
  e->packed[n] = pw;
  if (n.rfind("talker.layers.", 0) == 0 || (n == "cp.proj" && cols % 64 == 0)) {  // wgmma GEMM operand: [N][K] is already K-major
    Q3_REQUIRE(cols % 64 == 0, "%s: K must be a multiple of 64 for the prefill GEMM", name);
    return e->store.load(n, dev, shape, 2, DT_BF16);
  }
  return 0;
}

static int need_packed(q3_engine* e, const std::string& n, int rows, int cols, PackedW* out) {
  auto it = e->packed.find(n);
  Q3_REQUIRE(it != e->packed.end(), "%s: tensor %s is missing, expected shape [%d][%d]", kEngineName, n.c_str(), rows, cols);
  Q3_REQUIRE(it->second.n == rows && it->second.k == cols, "%s: tensor %s has shape [%d][%d], expected [%d][%d]", kEngineName,
             n.c_str(), it->second.n, it->second.k, rows, cols);
  *out = it->second;
  return 0;
}

// ---- program construction ------------------------------------------------------------------------
static Phase gemv(const PackedW& w, const bf16* src, int src_ld, const bf16* norm_w, float eps, void* dst, int dst_ld,
                  int epi, int ncmode, const bf16* bias = nullptr, bf16* save_normed = nullptr) {
  Phase p{};
  p.type = PH_GEMV; p.epi = epi; p.ncmode = ncmode;
  p.w = w.w; p.n_tiles = w.n / 16; p.kb = w.k / 32;
  p.src = src; p.src_ld = src_ld; p.norm_w = norm_w; p.eps = eps; p.dst = dst; p.dst_ld = dst_ld; p.bias = bias;
  p.save_normed = save_normed;
  return p;
}

static int add_layers(q3_engine* e, std::vector<Phase>& prog, const char* pfx, StackDev& S, bf16* hbuf, int ncmode,
                      int seqmode, int nq, int ctx_end) {
  const int Hh = S.hidden, QKV = (S.nh + 2 * S.nkv) * HD;
  for (int l = 0; l < S.layers; ++l) {
    std::string p = std::string(pfx) + ".layers." + std::to_string(l);
    PackedW wqkv, wo, wgu, wd;
    const bf16 *ln1, *ln2, *qn, *kn;
    if (need_packed(e, p + ".qkv", QKV, Hh, &wqkv) || need_packed(e, p + ".o", Hh, S.nh * HD, &wo) ||
        need_packed(e, p + ".gate_up", 2 * S.inter, Hh, &wgu) || need_packed(e, p + ".down", Hh, S.inter, &wd) ||
        !(ln1 = e->store.need<bf16>(p + ".ln1", Hh)) || !(ln2 = e->store.need<bf16>(p + ".ln2", Hh)) ||
        !(qn = e->store.need<bf16>(p + ".q_norm", HD)) || !(kn = e->store.need<bf16>(p + ".k_norm", HD)))
      return 1;
    prog.push_back(gemv(wqkv, hbuf, Hh, ln1, S.eps, S.qkv, QKV, EPI_STORE, ncmode));
    Phase a{};
    a.type = PH_ATTN; a.stack = (&S == &e->talker) ? 0 : 1; a.layer = l; a.seqmode = seqmode; a.nq = nq; a.ctx_end = ctx_end;
    a.qn = qn; a.kn = kn;
    prog.push_back(a);
    prog.push_back(gemv(wo, S.attn, S.nh * HD, nullptr, 0.f, hbuf, Hh, EPI_RESID, ncmode));
    prog.push_back(gemv(wgu, hbuf, Hh, ln2, S.eps, S.act, S.inter, EPI_SWIGLU, ncmode));
    prog.push_back(gemv(wd, S.act, S.inter, nullptr, 0.f, hbuf, Hh, EPI_RESID, ncmode));
  }
  return 0;
}

// Run table of a program (build_run_table, ar_step.cuh) in the engine's device store
static int build_piece_table(q3_engine* e, const std::vector<Phase>& prog, PieceTable* out, int keep_phases = 0) {
  std::vector<uint2> pieces;
  std::vector<uint32_t> off;
  if (build_run_table(prog, e->sm_count, e->wbase, keep_phases, &pieces, &off)) return 1;
  // the caller has drained the device: no launch still reads the old tables
  if (e->store.grow(&out->runs, (pieces.size() + 8) * sizeof(uint2), e->copy_stream, true) ||
      e->store.grow(&out->off, off.size() * sizeof(uint32_t), e->copy_stream, true))
    return 1;
  out->n_runs = pieces.size();
  Q3_CUDA(cudaMemcpy(out->runs, pieces.data(), pieces.size() * sizeof(uint2), cudaMemcpyHostToDevice));
  Q3_CUDA(cudaMemcpy(out->off, off.data(), off.size() * 4, cudaMemcpyHostToDevice));
  return 0;
}

static int build_programs(q3_engine* e, int B) {
  if (e->prog_B == B) return 0;
  const q3_engine_cfg& c = e->cfg;
  StackDev &T = e->talker, &C = e->cp;
  const int H = T.hidden, Hc = C.hidden, G = c.num_code_groups;
  const bf16 *tnorm, *cnorm;
  PackedW whead;
  if (!(tnorm = e->store.need<bf16>("talker.norm", H)) || !(cnorm = e->store.need<bf16>("cp.norm", Hc)) ||
      need_packed(e, "talker.codec_head", T.vocab, H, &whead))
    return 1;
  PackedW wproj{};
  const bf16* bproj = nullptr;
  if (c.has_cp_projection) {
    if (need_packed(e, "cp.proj", Hc, H, &wproj) || !(bproj = e->store.need<bf16>("cp.proj_bias", Hc))) return 1;
  }
  // ---- prefill-head program: final norm + codec_head on the last token of each row, sample frame-0 codebook-0
  e->prog_head.clear();
  {
    Phase hd = gemv(whead, e->h_last, H, tnorm, T.eps, T.logits, T.vocab, EPI_LOGITS, NC_B, nullptr, e->past_hidden);
    e->prog_head.push_back(hd);
    Phase s{}; s.type = PH_SAMPLE; s.group = 0;
    e->prog_head.push_back(s);
  }
  // ---- frame program
  std::vector<Phase>& F = e->prog_frame;
  F.clear();
  const bool joint = (2 * B <= MAXCOLS);
  // The CP input x lives token-major as [2][B][H]: block 0 = past_hidden (pass 0) or the previous codebook's
  // embedding (passes >= 1), block 1 = E0[c0] (pass 0 only).  With a projection (1.7B) x is e->x_cp and a
  // bias-GEMV writes the projected rows into cp.h; with the Identity projection (0.6B, H == Hc) x IS cp.h
  // (e->x_cp_ptr() aliases it) and the layers run in place on the block they need.
  bf16* xin = c.has_cp_projection ? e->x_cp : C.h;
  auto cp_pass = [&](int ncmode, int nq, int ctx_end, int block, bool from_table = false) -> bf16* {
    bf16* hb = C.h;
    if (from_table) {
      // the previous sample phase already wrote the projected embedding rows into cp.h
    } else if (c.has_cp_projection) {
      F.push_back(gemv(wproj, xin + (size_t)block * B * H, H, nullptr, 0.f, C.h, Hc, EPI_BIAS, ncmode, bproj));
    } else {
      hb = C.h + (size_t)block * B * Hc;
    }
    if (add_layers(e, F, "cp", C, hb, ncmode, SEQ_CP, nq, ctx_end)) return nullptr;
    return hb;
  };
  for (int j = 0; j < G - 1; ++j) {
    PackedW wlm;
    if (need_packed(e, "cp.lm_head." + std::to_string(j), C.vocab, Hc, &wlm)) return 1;
    bf16* hb;
    if (j == 0) {
      if (joint) {
        if (!(hb = cp_pass(NC_2B, 2, 2, 0))) return 1;
        hb += (size_t)B * Hc;  // logits come from the second token's rows
      } else {
        if (!cp_pass(NC_B, 1, 1, 0)) return 1;
        if (!(hb = cp_pass(NC_B, 1, 2, 1))) return 1;
      }
    } else {
      if (!(hb = cp_pass(NC_B, 1, j + 2, 0, e->proj_tab != nullptr))) return 1;
    }
    F.push_back(gemv(wlm, hb, Hc, cnorm, C.eps, C.logits, C.vocab, EPI_LOGITS, NC_B));
    Phase s{}; s.type = PH_SAMPLE; s.group = j + 1;
    F.push_back(s);
  }
  e->cp_phases = (int)F.size();
  if (add_layers(e, F, "talker", T, T.h, NC_B, SEQ_DECODE, 1, 0)) return 1;
  F.push_back(gemv(whead, T.h, H, tnorm, T.eps, T.logits, T.vocab, EPI_LOGITS, NC_B, nullptr, e->past_hidden));
  {
    Phase s{}; s.type = PH_SAMPLE; s.group = 0;
    F.push_back(s);
  }
  assign_tiles(e->prog_head, e->sm_count);
  assign_tiles(e->prog_frame, e->sm_count);
  // shared-memory plans: which phases stage their activations, how large the x area is, what is left for the rings
  e->nt_frame = (joint ? 2 * B : B) <= 8 ? 1 : (joint ? 2 * B : B) <= 16 ? 2 : 4;
  e->nt_head = B <= 8 ? 1 : B <= 16 ? 2 : 4;
  if (make_smem_plan(e->prog_head, B, e->nt_head, e->max_dyn_smem, &e->plan_head) ||
      make_smem_plan(e->prog_frame, B, e->nt_frame, e->max_dyn_smem, &e->plan_frame))
    return 1;
  Q3_REQUIRE((int)F.size() <= MAX_PHASES, "frame program has %d phases (max %d)", (int)F.size(), MAX_PHASES);
  // launches may still walk the old program and its piece tables: wait for them before replacing either (a batch-size
  // change is rare)
  Q3_CUDA(cudaDeviceSynchronize());
  if (build_piece_table(e, e->prog_head, &e->pt_head) || build_piece_table(e, e->prog_frame, &e->pt_frame, e->cp_phases))
    return 1;
  const size_t total = e->prog_head.size() + F.size();
  if ((int)total > e->prog_cap) {
    if (e->store.grow(&e->prog_dev, (total + 64) * sizeof(Phase), e->copy_stream, true)) return 1;
    e->prog_cap = (int)total + 64;
  }
  e->off_head = 0;
  e->off_frame = (int)e->prog_head.size();
  Q3_CUDA(cudaMemcpy(e->prog_dev + e->off_head, e->prog_head.data(), e->prog_head.size() * sizeof(Phase), cudaMemcpyHostToDevice));
  Q3_CUDA(cudaMemcpy(e->prog_dev + e->off_frame, F.data(), F.size() * sizeof(Phase), cudaMemcpyHostToDevice));
  e->prog_B = B;
  return 0;
}

extern "C" int q3_engine_finalize(q3_engine* e) {
  Q3_REQUIRE(e, "null engine");
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  const q3_engine_cfg& c = e->cfg;
  const DevStore& S = e->store;
  const q3_stack_cfg& tc = c.talker;
  if (!(e->emb_t = S.need<bf16>("talker.codec_embedding", (int64_t)tc.vocab_size * tc.hidden_size)) ||
      !(e->talker.rope_cos = S.need<bf16>("talker.rope_cos", (int64_t)c.max_ctx * 64)) ||
      !(e->talker.rope_sin = S.need<bf16>("talker.rope_sin", (int64_t)c.max_ctx * 64)) ||
      !(e->cp.rope_cos = S.need<bf16>("cp.rope_cos", (int64_t)32 * 64)) ||
      !(e->cp.rope_sin = S.need<bf16>("cp.rope_sin", (int64_t)32 * 64)) ||
      !(e->emb_cp = S.need<bf16>("cp.codec_embedding", (int64_t)(c.num_code_groups - 1) * c.cp.vocab_size * tc.hidden_size)))
    return 1;
  const int64_t H = tc.hidden_size, A = (int64_t)tc.num_heads * HD, QKV = A + 2LL * tc.num_kv_heads * HD, I = tc.intermediate_size;
  e->pf_layers.resize(tc.num_layers);
  for (int l = 0; l < tc.num_layers; ++l) {
    const std::string p = "talker.layers." + std::to_string(l);
    PfLayer& L = e->pf_layers[l];
    if (!(L.ln1 = S.need<bf16>(p + ".ln1", H)) || !(L.ln2 = S.need<bf16>(p + ".ln2", H)) ||
        !(L.qn = S.need<bf16>(p + ".q_norm", HD)) || !(L.kn = S.need<bf16>(p + ".k_norm", HD)) ||
        !(L.qkv = S.need<bf16>(p + ".qkv", QKV * H)) || !(L.o = S.need<bf16>(p + ".o", H * A)) ||
        !(L.gate_up = S.need<bf16>(p + ".gate_up", 2 * I * H)) || !(L.down = S.need<bf16>(p + ".down", H * I)))
      return 1;
  }
  // projection table: passes >= 1 of the code predictor feed small_to_mtp_projection(codec_embedding[j-1](c_j)) (:1281-1283),
  // a function of the sampled id only -> one wgmma GEMM over all (G-1)*Vc embedding rows here, no GEMV phase per pass
  // (without a GEMM copy of cp.proj, i.e. a talker hidden size that is not a multiple of 64, each pass keeps its projection GEMV)
  if (c.has_cp_projection && H % 64 == 0 && !e->proj_tab) {
    const int Hc = c.cp.hidden_size;
    const int rows = (c.num_code_groups - 1) * c.cp.vocab_size;
    const bf16 *bproj, *wproj;
    if (!(bproj = S.need<bf16>("cp.proj_bias", Hc)) || !(wproj = S.need<bf16>("cp.proj", (int64_t)Hc * H))) return 1;
    float* bias_f = nullptr;
    if (e->store.alloc(&bias_f, (size_t)Hc, true) || e->store.alloc(&e->proj_tab, (size_t)rows * Hc, true)) return 1;
    bf16_to_f32_kernel<<<(Hc + 255) / 256, 256, 0, e->copy_stream>>>(bproj, bias_f, Hc);
    GemmEpilogue ep{};
    ep.bias = bias_f; ep.cmod = Hc; ep.out_raw = e->proj_tab;
    GemmPlan plan;
    const int zero = 0;
    if (gemm_make_plan(&plan, e->emb_cp, 1, rows, H, H, (int64_t)rows * H, wproj, Hc, H, 1, &zero,
                       gemm_pick_bn(Hc, (rows + 127) / 128, 1), ep))
      return 1;
    if (gemm_launch(plan, e->copy_stream)) return 1;
    Q3_CUDA(cudaStreamSynchronize(e->copy_stream));
  }
  // kernel attributes: all opt-in shared memory minus the kernel's static part is the dynamic budget of the plans
  if (step_kernels_set_max_dyn_smem(&e->max_dyn_smem)) return 1;
  {  // weight arena base for the 32-bit (x16 B) offsets of the phase metas
    const char *lo = nullptr, *hi = nullptr;
    for (auto& kv : e->packed) {
      const char* a = reinterpret_cast<const char*>(kv.second.w);
      const char* b = a + (size_t)kv.second.n * kv.second.k * 2;
      if (!lo || a < lo) lo = a;
      if (!hi || b > hi) hi = b;
    }
    Q3_REQUIRE(lo && (size_t)(hi - lo) < ((size_t)1 << 36), "packed weights span more than 64 GB of address space");
    e->wbase = lo;
  }
  if (build_programs(e, 1)) return 1;
  // algorithmic bytes (SURVEY §8d)
  auto lw = [](const q3_stack_cfg& s) {
    return (double)s.hidden_size * (s.num_heads * HD) * 2 + 2.0 * s.hidden_size * (s.num_kv_heads * HD) +
           3.0 * s.hidden_size * s.intermediate_size + 2.0 * s.hidden_size + 2.0 * HD;
  };
  const double wt = c.talker.num_layers * lw(c.talker) + c.talker.hidden_size + (double)c.talker.vocab_size * c.talker.hidden_size;
  const double proj = c.has_cp_projection ? ((double)c.talker.hidden_size * c.cp.hidden_size + c.cp.hidden_size) : 0.0;
  const double heads = (double)(c.num_code_groups - 1) * c.cp.hidden_size * c.cp.vocab_size;
  const double cpl = c.cp.num_layers * lw(c.cp) + c.cp.hidden_size;
  e->w_talker_bytes = 2.0 * wt;
  e->w_cp_unique_bytes = 2.0 * (cpl + proj + heads);
  e->w_cp_stream_bytes = 2.0 * ((c.num_code_groups - 1) * (cpl + proj) + heads);
  // L2 residency of the code predictor's layer weights (re-read on each of its passes): keep a bit over half of the
  // L2 (27 MB of H100's 50 MB) of them at evict_last priority beside the talker's evict_first stream; much more than
  // that and the evict_last lines evict each other
  e->keep_fraction = (float)std::min(1.0, 0.54 * (double)e->l2_bytes / (2.0 * cpl));
  e->finalized = true;
  return 0;
}

// field by field: q3_sampling has padding before `seed`, which memcmp would compare
static bool same_sampling(const q3_sampling& a, const q3_sampling& b) {
  return a.do_sample == b.do_sample && a.top_k == b.top_k && a.top_p == b.top_p && a.temperature == b.temperature &&
         a.repetition_penalty == b.repetition_penalty && a.subtalker_dosample == b.subtalker_dosample &&
         a.subtalker_top_k == b.subtalker_top_k && a.subtalker_top_p == b.subtalker_top_p &&
         a.subtalker_temperature == b.subtalker_temperature && a.min_new_tokens == b.min_new_tokens &&
         a.suppress_eos == b.suppress_eos && a.seed == b.seed;
}

static int launch_program(q3_engine* e, int off, int n, int mode, int max_iters, int nt, const SmemPlan& plan,
                          const PieceTable& pt, int* codes_dev, cudaStream_t stream) {
  KParams P{};
  P.prog = e->prog_dev + off; P.n_phases = n; P.mode = mode; P.max_iters = max_iters; P.st = e->st;
  P.talker = e->talker; P.cp = e->cp; P.G = e->cfg.num_code_groups; P.eos = e->cfg.codec_eos_token_id;
  P.has_proj = e->cfg.has_cp_projection; P.sp = e->sp;
  // rows sample with their own request's parameters; a row without a running request (never admitted, finished,
  // released) with the default's, so that a request's settings stop costing the others once it has left.  The per-row
  // table is used only when some running row's parameters differ from the default: otherwise every row reads P.sp.
  for (int b = 0; b < e->B; ++b)
    if (e->active[b] && !same_sampling(e->row_sp[b], e->sp)) P.row_sampling = 1;
  if (P.row_sampling)
    for (int b = 0; b < MAXB; ++b) P.row_sp[b] = e->active[b] ? e->row_sp[b] : e->sp;
  P.B = e->B;
  for (int b = 0; b < MAXB; ++b) { P.len0[b] = e->len0[b]; P.trailing_len[b] = e->trailing_len[b]; }
  P.max_len0 = e->max_len0;
  for (int b = 0; b < MAXB; ++b) { P.frame0[b] = e->frame0[b]; P.row_key[b] = e->row_key[b]; }
  P.admit_mask = e->admit_mask;
  for (int b = 0; b < e->B; ++b)
    if (e->active[b] && e->text_open[b]) P.text_open |= 1u << b;
  P.emb_t = e->emb_t; P.emb_cp = e->emb_cp;
  P.x_cp = e->cfg.has_cp_projection ? e->x_cp : e->cp.h; P.past_hidden = e->past_hidden; P.past_keep = e->past_keep; P.trailing = e->trailing; P.trailing_stride = e->trailing_cap;
  if (e->proj_tab) { P.cp_next = e->proj_tab; P.cp_next_dst = e->cp.h; P.cp_next_w = e->cfg.cp.hidden_size; }
  else { P.cp_next = P.emb_cp; P.cp_next_dst = P.x_cp; P.cp_next_w = e->cfg.talker.hidden_size; }
  P.tts_pad = e->tts_pad; P.seen = e->seen; P.codes_out = codes_dev; P.codes_stride = e->codes_stride;
  P.split_buf = e->split_buf; P.forced = e->forced; P.n_forced = e->n_forced; P.dbg_tlogits = e->dbg_t; P.dbg_clogits = e->dbg_c; P.prof = (mode == 1) ? e->prof : nullptr;
  P.wbase = e->wbase; P.keep_fraction = e->keep_fraction;
  P.hid_out = e->hid_out; P.hid_stride = e->hid_stride;
  P.runs = pt.runs; P.run_off = pt.off;
  P.plan = plan;
  Q3_REQUIRE(n <= MAX_PHASES, "program of %d phases exceeds %d", n, MAX_PHASES);
  Q3_CUDA(cudaMemsetAsync(&e->st->bar_count, 0, sizeof(unsigned int), stream));
  void* args[] = {&P};
  const int var = P.prof ? 2 : P.hid_out ? 1 : 0;
  const void* fn = kStepKernels[var][nt == 1 ? 0 : nt == 2 ? 1 : 2];
  Q3_CUDA(cudaLaunchCooperativeKernel(fn, dim3(e->sm_count), dim3(CTA_THREADS), args, (size_t)plan.total, stream));
  return 0;
}

// One admission of n requests: request r enters engine slot slots[r] with the Philox row key keys[r] and the sampling
// parameters sp[r] (sp == nullptr: the default e->sp); its prompt is the prefix prefix[r] (prefix == nullptr or an id
// of -1: none) followed by lens[r] rows of embeds (packed back to back), its trailing text the first tl[r] rows of
// trailing[r] ([n][stride][H]; tl == nullptr: none).
struct Admission {
  int n;
  const int32_t* slots;
  const uint32_t* keys;
  const q3_sampling* sp;
  const int32_t* prefix;
  const void* embeds;
  const int32_t* lens;
  const void* trailing;
  const int32_t* tl;
  int stride;
};

// the prefix of request r of A (checked by check_admission), or null
static const q3_engine::Prefix* admission_prefix(const q3_engine* e, const Admission& A, int r) {
  if (!A.prefix || A.prefix[r] < 0) return nullptr;
  const auto it = e->prefixes.find(A.prefix[r]);
  return it == e->prefixes.end() ? nullptr : &it->second;
}

// room in the prefill scratch for ntok packed rows
static int ensure_prefill_rows(q3_engine* e, int ntok, cudaStream_t stream) {
  if (ntok <= e->pf_cap) return 0;
  const q3_stack_cfg& tc = e->cfg.talker;
  const int H = tc.hidden_size, nh = tc.num_heads, I = tc.intermediate_size, QKV = (nh + 2 * tc.num_kv_heads) * HD;
  const size_t cap = std::max(ntok + ntok / 4, 1024);
  DevStore& store = e->store;
  e->pf_cap = 0;  // until every block has grown: a failed growth leaves a freed block behind
  if (store.grow(&e->pf_x, cap * H * sizeof(bf16), stream, true) || store.grow(&e->pf_xn, cap * H * sizeof(bf16), stream, true) ||
      store.grow(&e->pf_qkv, cap * QKV * sizeof(bf16), stream, true) ||
      store.grow(&e->pf_attn, cap * nh * HD * sizeof(bf16), stream, true) ||
      store.grow(&e->pf_act, cap * I * sizeof(bf16), stream, true) || store.grow(&e->pf_seq, cap * sizeof(int), stream, true) ||
      store.grow(&e->pf_pos, cap * sizeof(int), stream, true))
    return 1;
  e->pf_cap = (int)cap;
  return 0;
}

// The talker layers over the ntok packed rows of pf_x, whose sequence and position are in pf_seq / pf_pos: wgmma GEMMs
// over all rows at once, K/V of every row into kc / vc ([seq][layers][nkv][cap][HD]), attention over each sequence's
// keys up to the row's position.  Every stage is row-wise or causal within one sequence.
static int prefill_layers(q3_engine* e, int ntok, bf16* kc, bf16* vc, int cap, cudaStream_t stream) {
  const q3_stack_cfg& tc = e->cfg.talker;
  const int H = tc.hidden_size, nh = tc.num_heads, nkv = tc.num_kv_heads, I = tc.intermediate_size, QKV = (nh + 2 * nkv) * HD;
  const int mt = (ntok + 127) / 128;
  const int zero = 0;
  auto gemm = [&](const bf16* a, int K, const bf16* w, int N, GemmEpilogue ep) -> int {
    ep.cmod = N;
    GemmPlan plan;
    if (gemm_make_plan(&plan, a, 1, ntok, K, K, (int64_t)ntok * K, w, N, K, 1, &zero, gemm_pick_bn(N, mt, 1), ep)) return 1;
    return gemm_launch(plan, stream);
  };
  const int rows_per_blk = 8;
  for (int l = 0; l < tc.num_layers; ++l) {
    const PfLayer& L = e->pf_layers[l];
    pf_rmsnorm_kernel<<<(ntok + rows_per_blk - 1) / rows_per_blk, 256, 0, stream>>>(e->pf_x, L.ln1, e->pf_xn, ntok, H, tc.rms_eps);
    { GemmEpilogue ep{}; ep.out_raw = e->pf_qkv; if (gemm(e->pf_xn, H, L.qkv, QKV, ep)) return 1; }
    pf_qkv_post_kernel<<<(ntok * (nh + 2 * nkv) + 7) / 8, 256, 0, stream>>>(e->pf_qkv, ntok, e->pf_seq, e->pf_pos, nh, nkv, L.qn, L.kn, tc.rms_eps,
                                                                         e->talker.rope_cos, e->talker.rope_sin, kc, vc, l,
                                                                         tc.num_layers, cap);
    pf_attention_kernel<<<(ntok * nh + 7) / 8, 256, 0, stream>>>(e->pf_qkv, e->pf_attn, ntok, e->pf_seq, e->pf_pos, nh, nkv, kc, vc, l,
                                                                 tc.num_layers, cap);
    { GemmEpilogue ep{}; ep.resid = e->pf_x; ep.out_raw = e->pf_x; if (gemm(e->pf_attn, nh * HD, L.o, H, ep)) return 1; }
    pf_rmsnorm_kernel<<<(ntok + rows_per_blk - 1) / rows_per_blk, 256, 0, stream>>>(e->pf_x, L.ln2, e->pf_xn, ntok, H, tc.rms_eps);
    { GemmEpilogue ep{}; ep.act = ACT_SWIGLU_BLK8; ep.out_act = e->pf_act; if (gemm(e->pf_xn, H, L.gate_up, 2 * I, ep)) return 1; }
    { GemmEpilogue ep{}; ep.resid = e->pf_x; ep.out_raw = e->pf_x; if (gemm(e->pf_act, I, L.down, H, ep)) return 1; }
  }
  Q3_CUDA(cudaGetLastError());
  return 0;
}

// Prefill of an admission into its slots: the index kernel resets the rows' device state, gathers their trailing text
// and copies their prefixes' K/V into the slots' caches; the layers run over the rows' own (suffix) tokens, whose K/V
// go into the slots' cache rows behind the prefix; then the head GEMV + the first codebook-0 sample of exactly those
// rows (`mask`: the admitted slots).
static int prefill_rows(q3_engine* e, const Admission& A, unsigned int mask, cudaStream_t stream) {
  const int n = A.n, H = e->cfg.talker.hidden_size;
  const q3_stack_cfg& tc = e->cfg.talker;
  PfLens pl{};
  PfRows pr{};
  PfPrefix px{};
  pl.B = n;
  pr.src = reinterpret_cast<const bf16*>(A.trailing); pr.dst = e->trailing; pr.stride = A.stride; pr.cap = e->trailing_cap; pr.H = H;
  px.kc = reinterpret_cast<uint4*>(e->talker.kc); px.vc = reinterpret_cast<uint4*>(e->talker.vc);
  px.lh = tc.num_layers * tc.num_kv_heads; px.cap = e->talker.cap;
  const int V = tc.vocab_size;
  int row_work = V;  // index-kernel threads per row: its seen bytes, its trailing elements or its prefix K chunks
  for (int r = 0; r < n; ++r) {
    pl.start[r + 1] = pl.start[r] + A.lens[r]; pl.slot[r] = A.slots[r];
    pr.trailing_len[r] = A.tl ? A.tl[r] : 0;
    row_work = std::max(row_work, pr.trailing_len[r] * H);
    if (const q3_engine::Prefix* p = admission_prefix(e, A, r)) {
      pl.p0[r] = p->len;
      px.kv[r] = reinterpret_cast<const uint4*>(p->kv);
      row_work = std::max(row_work, px.lh * p->len * (HD / 8));
    }
  }
  const int ntok = pl.start[n];
  if (ensure_prefill_rows(e, ntok, stream)) return 1;
  pf_index_kernel<<<dim3((std::max(ntok, row_work) + 255) / 256, n), 256, 0, stream>>>(pl, pr, px, e->st, e->seen, V, e->pf_seq, e->pf_pos);
  Q3_CUDA(cudaMemcpyAsync(e->pf_x, A.embeds, (size_t)ntok * H * 2, cudaMemcpyDeviceToDevice, stream));
  if (prefill_layers(e, ntok, e->talker.kc, e->talker.vc, e->talker.cap, stream)) return 1;
  pf_gather_last_kernel<<<n, 128, 0, stream>>>(pl, e->pf_x, e->h_last, H);
  // head + sample codebook-0 of the rows' first frame (codes are materialised by the following q3_decode via st->c0)
  e->admit_mask = mask;
  const int rc = launch_program(e, e->off_head, (int)e->prog_head.size(), 0, 1, e->nt_head, e->plan_head, e->pt_head, nullptr, stream);
  e->admit_mask = 0xffffffffu;
  return rc;
}

static int ensure_trailing(q3_engine* e, int stride, cudaStream_t stream) {
  const size_t need = (size_t)MAXB * stride * e->cfg.talker.hidden_size;
  if (need > e->trailing_alloc) {  // (re)allocate the engine-owned copy of trailing_text_hidden
    e->trailing_alloc = 0;  // until the block has grown
    if (e->store.grow(&e->trailing, need * sizeof(bf16), stream, true)) return 1;
    e->trailing_alloc = need;
  }
  return 0;
}

// The ranges HF's processors accept, plus finiteness where the sample phase needs it: a temperature of 0, a negative or
// non-finite one, or a repetition penalty of 0 turns scores into NaN, and the phase would then find no token at all.
static int check_sampling(const q3_sampling& s) {
  Q3_REQUIRE(!s.do_sample || (std::isfinite(s.temperature) && s.temperature > 0.f),
             "sampling: temperature %g must be finite and > 0 when do_sample is set", (double)s.temperature);
  Q3_REQUIRE(!s.subtalker_dosample || (std::isfinite(s.subtalker_temperature) && s.subtalker_temperature > 0.f),
             "sampling: subtalker_temperature %g must be finite and > 0 when subtalker_dosample is set",
             (double)s.subtalker_temperature);
  Q3_REQUIRE(s.top_k >= 0, "sampling: top_k %d must be >= 0", s.top_k);
  Q3_REQUIRE(s.subtalker_top_k >= 0, "sampling: subtalker_top_k %d must be >= 0", s.subtalker_top_k);
  Q3_REQUIRE(s.top_p >= 0.f && s.top_p <= 1.f, "sampling: top_p %g must be in [0, 1]", (double)s.top_p);
  Q3_REQUIRE(s.subtalker_top_p >= 0.f && s.subtalker_top_p <= 1.f, "sampling: subtalker_top_p %g must be in [0, 1]",
             (double)s.subtalker_top_p);
  Q3_REQUIRE(std::isfinite(s.repetition_penalty) && s.repetition_penalty > 0.f,
             "sampling: repetition_penalty %g must be finite and > 0", (double)s.repetition_penalty);
  Q3_REQUIRE(s.min_new_tokens >= 0, "sampling: min_new_tokens %d must be >= 0", s.min_new_tokens);
  return 0;
}

// Every check of admission A into a batch of B slots with a trailing capacity of cap rows, where `running` marks the
// slots whose request is still generating.  Writes nothing, so a rejected admission leaves the engine as it was.
static int check_admission(const q3_engine* e, const Admission& A, int B, int cap, unsigned int running) {
  for (int r = 0; r < A.n; ++r) {
    const int b = A.slots[r], tl = A.tl ? A.tl[r] : 0;
    Q3_REQUIRE(b >= 0 && b < B, "slot %d out of range", b);
    Q3_REQUIRE(!((running >> b) & 1u), "slot %d is still running (q3_release_slots it first)", b);
    for (int q = 0; q < r; ++q) Q3_REQUIRE(A.slots[q] != b, "slot %d admitted twice", b);
    const int id = A.prefix ? A.prefix[r] : -1;
    Q3_REQUIRE(id == -1 || e->prefixes.count(id), "request %d: prefix %d does not exist (never created, or freed)", r, id);
    const int P = id == -1 ? 0 : e->prefixes.at(id).len, S = A.lens[r];
    Q3_REQUIRE(S >= 1 && P + S < e->cfg.max_ctx,
               "request %d: prompt length %d out of range (a prefix of %d rows and %d rows of its own, at least 1, below max_ctx %d)",
               r, P + S, P, S, e->cfg.max_ctx);
    Q3_REQUIRE(tl >= 0 && tl <= A.stride && tl <= cap, "trailing length %d exceeds the stride %d or the capacity %d", tl, A.stride, cap);
    Q3_REQUIRE(tl == 0 || A.trailing, "request %d has a trailing length of %d but no trailing text", r, tl);
  }
  return 0;
}

// Free every parked row's record: a park's gather may still be queued on `stream`
static int free_records(q3_engine* e, cudaStream_t stream) {
  if (!e->records.empty()) Q3_CUDA(cudaStreamSynchronize(stream));
  for (auto& kv : e->records)
    if (e->store.release(kv.second.blk)) return 1;
  e->records.clear();
  e->first_record = e->next_record;
  return 0;
}

// A batch of B slots, every row finished (an empty slot is a finished row: it keeps stepping, like HF's padded rows, and
// is ignored), sampling with the default sp, room for max_trailing rows of trailing text per slot.  Records of parked
// rows belong to the session they were parked in and are freed.
static int reset_rows(q3_engine* e, int B, int max_trailing, const void* tts_pad_dev, const q3_sampling& sp, bool session,
                      cudaStream_t stream) {
  if (free_records(e, stream)) return 1;
  if (build_programs(e, B)) return 1;
  e->B = B; e->sp = sp; e->session = session;
  DevState hs;
  memset(&hs, 0, sizeof(hs));
  hs.B = B;
  for (int b = 0; b < MAXB; ++b) {
    hs.finished[b] = 1; hs.len0[b] = 1;
    e->len0[b] = 1; e->frame0[b] = 0; e->row_key[b] = (unsigned int)b; e->trailing_len[b] = 0; e->active[b] = false;
    e->text_open[b] = false; e->held[b] = false;
  }
  e->max_len0 = 1;
  Q3_CUDA(cudaMemcpyAsync(e->st, &hs, sizeof(hs), cudaMemcpyHostToDevice, stream));
  Q3_CUDA(cudaMemsetAsync(e->seen, 0, (size_t)MAXB * e->cfg.talker.vocab_size, stream));
  Q3_CUDA(cudaMemcpyAsync(e->tts_pad, tts_pad_dev, (size_t)e->cfg.talker.hidden_size * 2, cudaMemcpyDeviceToDevice, stream));
  if (max_trailing > 0 && ensure_trailing(e, max_trailing, stream)) return 1;
  e->trailing_cap = max_trailing;
  return 0;
}

// Admission A at global frame F (frames completed so far): all rows are checked before any state changes.  `running`
// marks the slots whose request is still generating; they keep their state.
static int admit_rows(q3_engine* e, const Admission& A, int F, unsigned int running, cudaStream_t stream) {
  if (check_admission(e, A, e->B, e->trailing_cap, running)) return 1;
  unsigned int admitted = 0;
  for (int r = 0; r < A.n; ++r) {
    const int b = A.slots[r];
    const q3_engine::Prefix* p = admission_prefix(e, A, r);
    e->len0[b] = (p ? p->len : 0) + A.lens[r] - F; e->frame0[b] = F; e->row_key[b] = A.keys[r]; e->trailing_len[b] = A.tl ? A.tl[r] : 0;
    e->row_sp[b] = A.sp ? A.sp[r] : e->sp;
    e->text_open[b] = false; e->held[b] = false;  // every admission starts closed: q3_set_trailing_open opens it
    admitted |= 1u << b;
  }
  e->frames_issued = F;
  e->max_len0 = 1;
  for (int b = 0; b < e->B; ++b) {
    e->active[b] = ((running | admitted) >> b) & 1u;
    if (e->active[b]) e->max_len0 = std::max(e->max_len0, e->len0[b]);
  }
  return prefill_rows(e, A, admitted, stream);
}

// A static batch is a session of B slots whose rows are all admitted at frame 0 with the Philox keys 0..B-1.
extern "C" int q3_prefill(q3_engine* e, int32_t B, const void* embeds_dev, const int32_t* lens_host,
                          const void* trailing_dev, const int32_t* trailing_lens_host, int32_t trailing_stride,
                          const void* tts_pad_dev, const q3_sampling* sp, void* stream_) {
  Q3_REQUIRE(e && e->finalized, "engine not finalized");
  Q3_REQUIRE(sp, "null argument");
  if (check_sampling(*sp)) return 1;
  Q3_REQUIRE(B >= 1 && B <= e->cfg.max_batch, "batch %d out of range", B);
  Q3_REQUIRE(embeds_dev && lens_host && tts_pad_dev, "null argument");
  int32_t slots[MAXB]; uint32_t keys[MAXB];
  for (int b = 0; b < B; ++b) { slots[b] = b; keys[b] = (uint32_t)b; }
  const Admission A{B, slots, keys, nullptr, nullptr, embeds_dev, lens_host, trailing_dev, trailing_lens_host, trailing_stride};
  if (check_admission(e, A, B, trailing_stride, 0)) return 1;
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  cudaStream_t stream = (cudaStream_t)stream_;
  if (reset_rows(e, B, trailing_stride, tts_pad_dev, *sp, false, stream)) return 1;
  return admit_rows(e, A, 0, 0, stream);
}

// ---- continuous batching (SURVEY §8f-4): a session of n_slots rows that start and finish independently ------------
extern "C" int q3_session_begin(q3_engine* e, int32_t n_slots, int32_t max_trailing, const void* tts_pad_dev, const q3_sampling* sp,
                                void* stream_) {
  Q3_REQUIRE(e && e->finalized, "engine not finalized");
  Q3_REQUIRE(sp, "bad argument");
  if (check_sampling(*sp)) return 1;
  Q3_REQUIRE(n_slots >= 1 && n_slots <= e->cfg.max_batch, "n_slots %d out of range", n_slots);
  Q3_REQUIRE(tts_pad_dev && sp && max_trailing >= 0, "bad argument");
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  return reset_rows(e, n_slots, max_trailing, tts_pad_dev, *sp, true, (cudaStream_t)stream_);
}

extern "C" int q3_sampling_check(const q3_sampling* sp) {
  Q3_REQUIRE(sp, "null argument");
  return check_sampling(*sp);
}

// sp_host == nullptr: every request samples with the session's parameters; prefix_ids_host == nullptr: no prefixes
extern "C" int q3_admit_with_prefix(q3_engine* e, int32_t n, const int32_t* slots_host, const uint32_t* keys_host,
                                    const q3_sampling* sp_host, const int32_t* prefix_ids_host, const void* embeds_dev,
                                    const int32_t* lens_host, const void* trailing_dev, const int32_t* trailing_lens_host,
                                    int32_t trailing_stride, void* stream_) {
  Q3_REQUIRE(e && e->finalized && e->session, "q3_session_begin first");
  Q3_REQUIRE(n >= 1 && n <= e->B && slots_host && keys_host && embeds_dev && lens_host, "bad argument");
  // every request's parameters before anything else: one bad entry fails the whole admission before any device work
  for (int r = 0; sp_host && r < n; ++r)
    if (check_sampling(sp_host[r])) {
      const std::string why = g_q3_err;
      return q3_set_err("request %d: %s", r, why.c_str());
    }
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  cudaStream_t stream = (cudaStream_t)stream_;
  // the global frame at which these rows start = frames completed so far (a decode may have stopped early)
  DevState hs;
  Q3_CUDA(cudaStreamSynchronize(stream));
  Q3_CUDA(cudaMemcpy(&hs, e->st, sizeof(hs), cudaMemcpyDeviceToHost));
  Q3_REQUIRE(hs.error == 0, "device-side error %d", hs.error);
  unsigned int running = 0;
  for (int b = 0; b < e->B; ++b)
    if (e->active[b] && !hs.finished[b]) running |= 1u << b;
  const Admission A{n, slots_host, keys_host, sp_host, prefix_ids_host, embeds_dev, lens_host, trailing_dev, trailing_lens_host,
                    trailing_stride};
  return admit_rows(e, A, hs.step, running, stream);
}

extern "C" int q3_admit_with_sampling(q3_engine* e, int32_t n, const int32_t* slots_host, const uint32_t* keys_host,
                                      const q3_sampling* sp_host, const void* embeds_dev, const int32_t* lens_host,
                                      const void* trailing_dev, const int32_t* trailing_lens_host, int32_t trailing_stride,
                                      void* stream_) {
  return q3_admit_with_prefix(e, n, slots_host, keys_host, sp_host, nullptr, embeds_dev, lens_host, trailing_dev,
                              trailing_lens_host, trailing_stride, stream_);
}

// ---- registered prompt prefixes: the talker K/V of rows that many requests' prompts begin with ---------------------
extern "C" int q3_prefix_create(q3_engine* e, const void* embeds_dev, int32_t len, void* stream_, int32_t* id_out) {
  Q3_REQUIRE(e && e->finalized, "engine not finalized");
  Q3_REQUIRE(len >= 1 && len < e->cfg.max_ctx - 1, "prefix length %d out of range [1, %d)", len, e->cfg.max_ctx - 1);
  Q3_REQUIRE(embeds_dev && id_out, "null argument");
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  cudaStream_t stream = (cudaStream_t)stream_;
  const q3_stack_cfg& tc = e->cfg.talker;
  const size_t half = (size_t)tc.num_layers * tc.num_kv_heads * len * HD;
  bf16* kv = nullptr;
  if (e->store.alloc(&kv, 2 * half, false)) return 1;  // the layers write every element
  int rc = ensure_prefill_rows(e, len, stream);
  if (!rc) {
    pf_prefix_index_kernel<<<(len + 255) / 256, 256, 0, stream>>>(len, e->pf_seq, e->pf_pos);
    Q3_CUDA(cudaMemcpyAsync(e->pf_x, embeds_dev, (size_t)len * tc.hidden_size * 2, cudaMemcpyDeviceToDevice, stream));
    rc = prefill_layers(e, len, kv, kv + half, len, stream);
  }
  if (rc) {  // the error stays the one recorded; launches already queued may still write the block
    cudaStreamSynchronize(stream);
    e->store.release(kv);
    return 1;
  }
  const int id = e->next_prefix++;
  e->prefixes[id] = q3_engine::Prefix{kv, len};
  *id_out = id;
  return 0;
}

extern "C" int q3_prefix_free(q3_engine* e, int32_t id, void* stream_) {
  Q3_REQUIRE(e, "null engine");
  const auto it = e->prefixes.find(id);
  Q3_REQUIRE(it != e->prefixes.end(), "prefix %d does not exist (never created, or freed)", id);
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  Q3_CUDA(cudaStreamSynchronize((cudaStream_t)stream_));  // an admission's copy of the block may still be queued
  bf16* kv = it->second.kv;
  e->prefixes.erase(it);
  return e->store.release(kv);
}

extern "C" int q3_prefix_length(q3_engine* e, int32_t id) {
  if (e) {
    const auto it = e->prefixes.find(id);
    if (it != e->prefixes.end()) return it->second.len;
  }
  q3_set_err("prefix %d does not exist", id);
  return -1;
}

extern "C" int q3_decode(q3_engine* e, int32_t max_frames, int32_t* codes_dev, int32_t codes_stride, void* stream_) {
  Q3_REQUIRE(e && e->finalized && e->B > 0, "prefill first");
  Q3_REQUIRE(codes_dev && codes_stride > 0 && max_frames > 0, "bad arguments");
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  cudaStream_t stream = (cudaStream_t)stream_;
  e->codes_stride = codes_stride;
  for (int b = 0; b < e->B; ++b)  // len0 holds prompt length - frame0: position of the last frame = len0 + frames issued
    if (e->active[b])
      Q3_REQUIRE(e->len0[b] + e->frames_issued + max_frames <= e->cfg.max_ctx,
                 "KV capacity exceeded: row %d would reach position %d > max_ctx %d", b, e->len0[b] + e->frames_issued + max_frames, e->cfg.max_ctx);
  for (int b = 0; b < e->B; ++b)
    Q3_REQUIRE(!(e->active[b] && e->text_open[b] && e->hid_out), "row %d is open for live text while hidden-state capture is set", b);
  const int F = e->frames_issued;
  e->frames_issued += max_frames;
  if (launch_program(e, e->off_frame, (int)e->prog_frame.size(), 1, max_frames, e->nt_frame, e->plan_frame, e->pt_frame, codes_dev, stream))
    return 1;
  // Live text: an open row held at step f (its row frame f >= trailing_len) stays held for the rest of the launch, so
  // of the n steps only the first `avail` committed.  Moving its admission frame by the held steps makes its row frame
  // (frame - frame0) and its position (len0 + frame) those of its committed steps again: the next launch runs step f
  // anew.  A held row is not finished, so the launch ran all n steps whenever this applies.  No device state changes.
  bool rebased = false;
  for (int b = 0; b < e->B; ++b) {
    e->held[b] = false;
    if (!e->active[b] || !e->text_open[b]) continue;
    const int avail = std::max(0, e->trailing_len[b] - (F - e->frame0[b]));
    const int held = max_frames - std::min(max_frames, avail);
    e->frame0[b] += held;
    e->len0[b] -= held;
    e->held[b] = held > 0;
    rebased = rebased || held > 0;
  }
  if (rebased) {  // still the largest (prompt - frame0) of the running rows: the attention split count of the batch
    e->max_len0 = 1;
    for (int b = 0; b < e->B; ++b)
      if (e->active[b]) e->max_len0 = std::max(e->max_len0, e->len0[b]);
  }
  return 0;
}

// Streaming TEXT input (SURVEY §8f-2): more trailing_text_hidden rows for a row that is already generating.  Frame t of a
// row adds trailing[t] while t < its trailing length and tts_pad afterwards (modeling_qwen3_tts.py:1689-1692), so rows
// appended before the frame that needs them are indistinguishable from rows given at prefill.
extern "C" int q3_append_trailing(q3_engine* e, int32_t slot, const void* rows_dev, int32_t n, void* stream_) {
  Q3_REQUIRE(e && e->B > 0 && rows_dev && n >= 1, "bad argument");
  Q3_REQUIRE(slot >= 0 && slot < e->B, "slot %d out of range", slot);
  Q3_REQUIRE(e->trailing && e->trailing_len[slot] + n <= e->trailing_cap, "trailing text of row %d would exceed its capacity %d", slot,
             e->trailing_cap);
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  const int H = e->cfg.talker.hidden_size;
  Q3_CUDA(cudaMemcpyAsync(e->trailing + ((size_t)slot * e->trailing_cap + e->trailing_len[slot]) * H, rows_dev, (size_t)n * H * 2,
                          cudaMemcpyDeviceToDevice, (cudaStream_t)stream_));
  e->trailing_len[slot] += n;
  return 0;
}

// Live text (SURVEY §8f-2): while a row is open its text may still grow, and a step whose text row has not arrived is
// held instead of reading tts_pad (see q3_decode).  Closing puts the row back on the reference's semantics.
extern "C" int q3_set_trailing_open(q3_engine* e, int32_t slot, int32_t open) {
  Q3_REQUIRE(e && e->B > 0, "prefill or q3_session_begin first");
  Q3_REQUIRE(slot >= 0 && slot < e->B, "slot %d out of range", slot);
  Q3_REQUIRE(e->active[slot], "slot %d has no running request", slot);
  Q3_REQUIRE(!open || !e->hid_out, "live text is not available while hidden-state capture is set");
  e->text_open[slot] = open != 0;
  return 0;
}

extern "C" int q3_release_slots(q3_engine* e, int32_t n, const int32_t* slots_host, void* stream_) {
  Q3_REQUIRE(e && e->session && slots_host && n >= 0 && n <= MAXB, "bad argument");
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  SlotList A{};
  A.n = n;
  for (int r = 0; r < n; ++r) {
    Q3_REQUIRE(slots_host[r] >= 0 && slots_host[r] < e->B, "slot %d out of range", slots_host[r]);
    A.slot[r] = slots_host[r];
    e->active[slots_host[r]] = false;
    e->text_open[slots_host[r]] = false;
    e->held[slots_host[r]] = false;
  }
  if (n > 0) release_state_kernel<<<1, 32, 0, (cudaStream_t)stream_>>>(e->st, A);
  return 0;
}

// ---- parked rows: a running request's state moves out of its slot into a record and back into any free slot --------
// Record block: [2][layers * nkv][pos][HD] bf16 talker K/V (a registered prefix's layout), then the x_cp rows of blocks
// 0 and 1, past_hidden and past_keep ([4][H] bf16), the trailing text [trailing_len][H] bf16, the seen bytes [V] and the
// DevState ints.  Every piece starts on a 16-byte boundary (H % 32 == 0, V % 16 == 0).
struct RecordLayout { size_t kv, rows, text, seen, ints, bytes; };
static RecordLayout record_layout(const q3_engine* e, int pos, int trailing_len) {
  const q3_stack_cfg& tc = e->cfg.talker;
  const size_t H = tc.hidden_size;
  RecordLayout L;
  L.kv = 0;
  L.rows = L.kv + (size_t)2 * tc.num_layers * tc.num_kv_heads * pos * HD * sizeof(bf16);
  L.text = L.rows + 4 * H * sizeof(bf16);
  L.seen = L.text + (size_t)trailing_len * H * sizeof(bf16);
  L.ints = L.seen + (size_t)tc.vocab_size;
  L.bytes = L.ints + kRowInts * sizeof(int);
  return L;
}

// The one launch of a park (kResume false) or a resume of record R in slot b
template <bool kResume>
static int launch_row_move(q3_engine* e, const q3_engine::Record& R, int b, cudaStream_t stream) {
  const q3_stack_cfg& tc = e->cfg.talker;
  const int H = tc.hidden_size, V = tc.vocab_size;
  const RecordLayout L = record_layout(e, R.pos, R.trailing_len);
  bf16* xcp = e->cfg.has_cp_projection ? e->x_cp : e->cp.h;  // what KParams::x_cp points at: [2][B][H]
  const bf16* rows[4] = {xcp + (size_t)b * H, xcp + ((size_t)e->B + b) * H, e->past_hidden + (size_t)b * H,
                         e->past_keep + (size_t)b * H};
  RowMove M{};
  for (int k = 0; k < 4; ++k)
    M.span[k] = RowSpan{(uint4*)rows[k], (uint4*)(R.blk + L.rows + (size_t)k * H * sizeof(bf16)), H / 8};
  M.span[4] = RowSpan{(uint4*)(e->trailing + (size_t)b * e->trailing_cap * H), (uint4*)(R.blk + L.text), R.trailing_len * H / 8};
  M.span[5] = RowSpan{(uint4*)(e->seen + (size_t)b * V), (uint4*)(R.blk + L.seen), V / 16};
  M.kc = reinterpret_cast<uint4*>(e->talker.kc); M.vc = reinterpret_cast<uint4*>(e->talker.vc);
  M.kv = reinterpret_cast<uint4*>(R.blk + L.kv);
  M.lh = tc.num_layers * tc.num_kv_heads; M.cap = e->talker.cap; M.pos = R.pos; M.slot = b;
  M.ints = reinterpret_cast<int*>(R.blk + L.ints);
  const size_t work = std::max<size_t>((size_t)M.lh * R.pos * (HD / 8), (size_t)std::max(V / 16, R.trailing_len * H / 8));
  const int grid = (int)std::min<size_t>((work + 255) / 256, (size_t)e->sm_count * 8);
  row_move_kernel<kResume><<<std::max(grid, 1), 256, 0, stream>>>(M, e->st);
  Q3_CUDA(cudaGetLastError());
  return 0;
}

// The rules park and resume share: a session without hidden-state capture or teacher forcing (the rules of live text)
static int check_row_move(const q3_engine* e, const char* what) {
  Q3_REQUIRE(e && e->finalized && e->session, "%s: q3_session_begin first (rows are parked only in a session)", what);
  Q3_REQUIRE(!e->hid_out && !e->forced, "%s: not available while hidden-state capture or teacher forcing is set", what);
  return 0;
}

static int record_missing(const q3_engine* e, int id) {
  if (id >= 0 && id < e->first_record) return q3_set_err("record %d belongs to an earlier session", id);
  return q3_set_err("record %d does not exist (never parked, or already resumed or discarded)", id);
}

extern "C" int q3_row_park(q3_engine* e, int32_t slot, void* stream_, int32_t* id_out) {
  if (check_row_move(e, "q3_row_park")) return 1;
  Q3_REQUIRE(id_out, "null argument");
  Q3_REQUIRE(slot >= 0 && slot < e->B, "q3_row_park: slot %d out of range", slot);
  Q3_REQUIRE(e->active[slot], "q3_row_park: slot %d has no running request (never admitted, finished, released or parked)", slot);
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  q3_engine::Record R{};
  R.pos = e->len0[slot] + e->frames_issued;
  R.f = e->frames_issued - e->frame0[slot];
  R.trailing_len = e->trailing_len[slot];
  R.key = e->row_key[slot]; R.sp = e->row_sp[slot]; R.text_open = e->text_open[slot]; R.held = e->held[slot];
  // no zero fill: the launch writes every byte that resume reads, and a zeroed block would drain the device
  if (e->store.alloc(&R.blk, record_layout(e, R.pos, R.trailing_len).bytes, false)) return 1;
  if (launch_row_move<false>(e, R, slot, (cudaStream_t)stream_)) {
    cudaStreamSynchronize((cudaStream_t)stream_);
    e->store.release(R.blk);
    return 1;
  }
  e->active[slot] = e->text_open[slot] = e->held[slot] = false;
  const int id = e->next_record++;
  e->records[id] = R;
  *id_out = id;
  return 0;
}

extern "C" int q3_row_resume(q3_engine* e, int32_t id, int32_t slot, void* stream_) {
  if (check_row_move(e, "q3_row_resume")) return 1;
  const auto it = e->records.find(id);
  if (it == e->records.end()) return record_missing(e, id);
  const q3_engine::Record R = it->second;
  Q3_REQUIRE(slot >= 0 && slot < e->B, "q3_row_resume: slot %d out of range", slot);
  Q3_REQUIRE(R.pos < e->cfg.max_ctx, "record %d: its next position %d does not fit max_ctx %d", id, R.pos, e->cfg.max_ctx);
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  cudaStream_t stream = (cudaStream_t)stream_;
  // the global frame at which the row continues = frames completed so far, as for an admission
  DevState hs;
  Q3_CUDA(cudaStreamSynchronize(stream));
  Q3_CUDA(cudaMemcpy(&hs, e->st, sizeof(hs), cudaMemcpyDeviceToHost));
  Q3_REQUIRE(hs.error == 0, "device-side error %d", hs.error);
  Q3_REQUIRE(!(e->active[slot] && !hs.finished[slot]), "q3_row_resume: slot %d is still running (park or release it first)", slot);
  const int F = hs.step;
  if (launch_row_move<true>(e, R, slot, stream)) return 1;
  // the row's frame counter (frame - frame0) and position (len0 + frame) continue from where they were at the park
  e->frame0[slot] = F - R.f; e->len0[slot] = R.pos - F; e->trailing_len[slot] = R.trailing_len;
  e->row_key[slot] = R.key; e->row_sp[slot] = R.sp; e->text_open[slot] = R.text_open; e->held[slot] = R.held;
  e->active[slot] = true;
  e->frames_issued = F;
  e->max_len0 = 1;
  for (int b = 0; b < e->B; ++b)
    if (e->active[b]) e->max_len0 = std::max(e->max_len0, e->len0[b]);
  // the record is freed once the launch that reads it is done
  Q3_CUDA(cudaStreamSynchronize(stream));
  e->records.erase(id);
  return e->store.release(R.blk);
}

extern "C" int q3_row_discard(q3_engine* e, int32_t id, void* stream_) {
  Q3_REQUIRE(e && e->finalized && e->session, "q3_row_discard: q3_session_begin first");
  const auto it = e->records.find(id);
  if (it == e->records.end()) return record_missing(e, id);
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  Q3_CUDA(cudaStreamSynchronize((cudaStream_t)stream_));  // the park's gather may still be queued
  unsigned char* blk = it->second.blk;
  e->records.erase(it);
  return e->store.release(blk);
}

extern "C" int q3_get_progress(q3_engine* e, int32_t* frames_done, int32_t* n_valid, int32_t* finished) {
  Q3_REQUIRE(e, "null engine");
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  DevState hs;
  Q3_CUDA(cudaMemcpy(&hs, e->st, sizeof(hs), cudaMemcpyDeviceToHost));
  Q3_REQUIRE(hs.error == 0, "device-side error %d (grid barrier timeout)", hs.error);
  if (frames_done) *frames_done = hs.step;
  for (int b = 0; b < e->B; ++b) {
    // the row's own frame count; a held row has one frame more: its held step's code-predictor half is done
    if (n_valid) n_valid[b] = hs.finished[b] ? hs.n_valid[b] : hs.step - e->frame0[b] + (e->held[b] ? 1 : 0);
    if (hs.finished[b]) e->active[b] = e->text_open[b] = e->held[b] = false;
    if (finished) finished[b] = hs.finished[b];
  }
  return 0;
}

extern "C" int q3_set_debug(q3_engine* e, const int32_t* forced_dev, int32_t n_frames, float* talker_logits_dev,
                            float* cp_logits_dev) {
  Q3_REQUIRE(e, "null engine");
  e->forced = forced_dev; e->n_forced = forced_dev ? n_frames : 0;
  e->dbg_t = talker_logits_dev; e->dbg_c = cp_logits_dev;
  return 0;
}

// Per-step hidden states (the second return value of Qwen3TTSForConditionalGeneration.generate, :2281): hid_dev bf16
// [B][stride][H] receives, for row b, the final-norm output of its last position at step s (s = 0: the prefill) at
// [b][s][:].  NULL disables.  Set before q3_prefill.
extern "C" int q3_set_hidden_capture(q3_engine* e, void* hid_dev, int32_t stride) {
  Q3_REQUIRE(e, "null engine");
  e->hid_out = reinterpret_cast<bf16*>(hid_dev);
  e->hid_stride = hid_dev ? stride : 0;
  return 0;
}

extern "C" int q3_set_profile(q3_engine* e, unsigned long long* prof_dev) {
  Q3_REQUIRE(e, "null engine");
  e->prof = prof_dev;
  return 0;
}

// phase kinds of the frame program (0 GEMV, 1 ATTN, 2 SAMPLE) + stack (0 talker, 1 cp) + epilogue, for profiling
extern "C" int q3_describe_frame_program(q3_engine* e, int32_t* kinds, int32_t capacity) {
  Q3_REQUIRE(e && e->prog_B > 0, "no program built yet");
  const int n = (int)e->prog_frame.size();
  if (kinds) {
    for (int i = 0; i < n && i < capacity; ++i) {
      const Phase& p = e->prog_frame[i];
      int stack = p.stack;
      if (p.type == PH_GEMV) stack = (p.kb * 32 == e->cfg.talker.hidden_size || p.kb * 32 == e->cfg.talker.intermediate_size ||
                                      p.kb * 32 == e->cfg.talker.num_heads * HD) && !(p.src == e->cp.h || p.src == e->cp.attn || p.src == e->cp.act) ? 0 : 1;
      if (p.type == PH_SAMPLE) stack = p.group == 0 ? 0 : 1;
      kinds[i] = p.type * 100 + stack * 10 + (p.type == PH_GEMV ? p.epi : 0);
    }
  }
  return -n;  // negative = count (0 is reserved for success elsewhere); callers use abs()
}

extern "C" int q3_algorithmic_bytes(q3_engine* e, int32_t B, int32_t S, double* a_bytes, double* a_stream_bytes) {
  Q3_REQUIRE(e && e->finalized, "engine not finalized");
  const q3_engine_cfg& c = e->cfg;
  const double kv_tok = (double)c.talker.num_layers * 2 * c.talker.num_kv_heads * HD * 2;
  const double kv = (double)B * (S + 1) * kv_tok;
  if (a_bytes) *a_bytes = e->w_talker_bytes + e->w_cp_unique_bytes + kv;
  if (a_stream_bytes) *a_stream_bytes = e->w_talker_bytes + e->w_cp_stream_bytes + kv;
  return 0;
}
