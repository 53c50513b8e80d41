// Data model of the fused frame-step kernel: tile constants, the phase descriptor, device-side state and launch parameters.
// Part of the ar_engine.cu translation unit (include order: ar_program, ar_gemv, ar_attention, ar_sampler,
// the persistent kernel in ar_step, ar_prefill).
#pragma once

namespace {

constexpr int NTHREADS = 256;                 // worker threads (8 consumer warps)
constexpr int NWARPS = NTHREADS / 32;
constexpr int CTA_THREADS = NTHREADS;
constexpr int HD = 128;          // head_dim (required)
constexpr int MAXB = Q3_MAX_BATCH;
constexpr int MAXCOLS = 32;      // columns per pass (batch rows or prefill tokens)
constexpr int MAXSPLIT = 16;
constexpr int RMAX = 2;          // max GQA group size (q heads per kv head)
constexpr int PCOL = 20;         // padded row count of a partial column (bank-conflict-free)
// ---- shared-memory plan of the frame-step kernel (host-computed per launch class, see make_smem_plan) -------------
//   [ x area | part | nw | weight rings | phase metas | mbarriers + round tables ]
// x area : staged activations [cols][K] bf16 (rows skewed by 64 B), aliased by the attention / sampler phases
// part   : split-K partial sums [warp][seg][col][PCOL] fp32
// nw     : RMSNorm weights of the current GEMV phase (<= 2048 bf16)
// rings  : per warp R slots of SB KB, filled by cp.async.bulk (TMA) ahead of the consumer, across phases
constexpr int SMEM_OPTIN = 232448;             // 227 KB per CTA on sm_90
constexpr int MAX_PHASES = 640;                // phases per program (meta table)
constexpr int ATT_SMEM = (2 * 2 * 128 + 32 * 2 * 130) * 4 + 2 * 60 * 128 * 2;  // attention: fp32 queries + half-warp partials + 60-row K and V windows
constexpr int SAMPLER_SMEM = (2 * 4096 + 64 + 256) * 4;
constexpr int X_MIN_BYTES = 65 * 1024;         // >= ATT_SMEM, SAMPLER_SMEM
constexpr int NW_BYTES = 4096;
constexpr int MAX_SLOTS = 8;
// x-area budget: 16 columns x K <= 2048 for batch classes 1-2 (8 x 4160 B ... 16 x 4160 B), 32 x 4160 B for class 4.  Inputs
// with a larger K (the down projections) are read un-staged.  Keeping the whole plan of classes 1-2 under 195 KB
// leaves the SM a 32 KB L1, which is what absorbs the stack traffic of the phase functions (with a 227 KB request
// every local-memory access is an L2 round trip).
__host__ __device__ constexpr int x_budget_nt(int nt) { return (nt <= 2 ? 16 : 32) * (2 * 2048 + 64); }
__host__ __device__ constexpr int part_bytes_nt(int nt) { return NWARPS * 2 * nt * 8 * PCOL * 4; }

struct SmemPlan {
  int x_off, x_bytes, part_off, nw_off, ring_off, slot_blocks, nslots, meta_off, bar_off, total;
};
constexpr int MAXV = 4096;       // max vocab handled by the sampler

enum PhaseType { PH_GEMV = 0, PH_ATTN = 1, PH_SAMPLE = 2 };
enum Epi { EPI_STORE = 0, EPI_BIAS = 1, EPI_RESID = 2, EPI_SWIGLU = 3, EPI_LOGITS = 4 };
enum NcMode { NC_B = 0, NC_2B = 1 };
enum SeqMode { SEQ_CP = 0, SEQ_DECODE = 1 };

struct Phase {
  int type, epi, ncmode, stack;
  // ---- GEMV
  const uint4* w;      // packed weights
  int n_tiles, kb;     // rows/16, K/32
  int tq, tr;          // n_tiles = tq*grid + tr: CTA c owns tq (+1 if c < tr) consecutive tiles
  const bf16* src;     // [nc][src_ld]
  int src_ld;
  const bf16* norm_w;  // RMSNorm weight applied while staging (nullable)
  float eps;
  void* dst;
  int dst_ld;
  const bf16* bias;
  bf16* save_normed;   // optional copy of the normed input (past_hidden), ld = K
  // ---- ATTN
  int layer, seqmode, nq, ctx_end;
  const bf16* qn;
  const bf16* kn;
  // ---- SAMPLE
  int group;           // 0 = talker codebook-0; j>=1 = code predictor codebook j
  int staged;          // GEMV: activations are staged in the x area (else B fragments come straight from L2)
};

struct StackDev {
  int hidden, layers, nh, nkv, inter, vocab;
  float eps;
  bf16 *h, *qkv, *attn, *act;  // activations [cols][...]
  bf16 *kc, *vc;               // KV cache [seq][layer][nkv][cap][128]
  int cap;
  const bf16 *rope_cos, *rope_sin;  // [cap][64]
  float* logits;               // [MAXB][vocab]
};

struct DevState {
  unsigned int bar_count;        // grid barrier counter (every CTA's arrive and poll hit it)
  // Keeps the fields below, and the buffers allocated after DevState, where the kernel was tuned: without this 1 KB the
  // frame-step measured 0.3-0.5% slower at B = 8 with identical kernel code, and a 128-byte pad did not recover it
  // (one H100 80GB HBM3 SXM, 700 W limit)
  unsigned int bar_pad[256];
  int error;
  int B;
  int step;            // frames whose 16 codes are complete
  int len0[MAXB];
  int finished[MAXB];
  int n_valid[MAXB];
  int n_gen[MAXB];
  int c0[MAXB];
  int trailing_len[MAXB];
  int cur[MAXB][Q3_NUM_GROUPS_MAX];
  unsigned int split_cnt[MAXB * 16];
};

struct KParams {
  const Phase* prog;
  int n_phases;
  int mode;        // 0 = one pass over the program (prefill chunk / prefill head), 1 = frame loop
  int max_iters;
  DevState* st;
  StackDev talker, cp;
  int G, eos, has_proj;
  int B;                    // sequences in this request (constant per launch)
  int len0[MAXB];           // prompt lengths
  int max_len0;             // longest (prompt - frame0) of the batch (attention split count)
  int frame0[MAXB];         // global frame index at which row b was admitted (continuous batching; 0 for a static batch):
                            // the row's own frame counter is frame - frame0[b]; len0[b] is stored as prompt_len - frame0[b]
  unsigned int row_key[MAXB];  // Philox row key (the request's identity, not its slot: an admitted row samples what it would alone)
  unsigned int admit_mask;  // prefill-head program only: rows whose first token is sampled / whose hidden state is saved
  unsigned int text_open;   // rows whose text may still grow: such a row is HELD at a step whose text row has not
                            // arrived (row frame >= trailing_len[b]) and its talker sample commits nothing (live text)
  int trailing_len[MAXB];
  q3_sampling sp;           // sampling parameters of every row, unless row_sampling is set
  int row_sampling;         // 1: row b samples with row_sp[b] (continuous batching: per-request parameters); 0: with sp
  q3_sampling row_sp[MAXB];
  // sampler / embed resources
  const bf16* emb_t;        // talker codec_embedding [V][H]
  const bf16* emb_cp;       // cp codec_embedding [G-1][Vc][H]
  bf16* x_cp;               // CP input [2][B][H]
  const bf16* cp_next;      // rows fed to passes >= 1: projected embedding table [(G-1)*Vc][Hc] or emb_cp itself
  bf16* cp_next_dst;        // where they go: cp.h (table / Identity projection) or x_cp (projection phase follows)
  int cp_next_w;            // row width of cp_next / cp_next_dst
  bf16* past_hidden;        // [B][H]
  bf16* past_keep;          // [B][H] past_hidden as the row's last committed talker sample copied it into x_cp: a held
                            // step puts x_cp back from it (the code predictor's passes may overwrite x_cp in place)
  const bf16* trailing;     // [B][stride][H]
  int trailing_stride;
  const bf16* tts_pad;      // [H]
  unsigned char* seen;      // [B][V]
  int* codes_out;           // [B][codes_stride][G]
  int codes_stride;
  float* split_buf;         // [MAXB*nkv*MAXSPLIT][RMAX][130]
  bf16* hid_out;            // optional [B][hid_stride][H]: the normed last hidden state of every step (generate()'s 2nd return)
  int hid_stride;
  // debug hooks
  const int* forced;
  int n_forced;
  float* dbg_tlogits;
  float* dbg_clogits;
  float keep_fraction;      // share of the code predictor's weight lines fetched with L2 evict_last priority
  SmemPlan plan;
  const char* wbase;        // lowest address of the packed GEMV weights (piece offsets are relative to it)
  const uint2* runs;        // run table of this program: per (CTA, warp) the (offset/16, blocks) of every weight run of ONE pass
  const uint32_t* run_off;  // [grid*NWARPS + 1] start of each (CTA, warp) list in `runs`
  unsigned long long* prof;  // [n_phases][grid][16]: globaltimer ns [0] phase end, [1] barrier passed, [2..4] inner marks, [6] start, [7],[8] warp-0 marks; cycles [5]
};
// passed by value to the kernel: stays within the classic 4 KB kernel-parameter limit
static_assert(sizeof(KParams) <= 4096, "KParams exceeds 4 KB");

}  // namespace
