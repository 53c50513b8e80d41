/*
 * qwen3tts_b200.h — C ABI of the H100-native Qwen3-TTS hot-path library (libqwen3tts_b200.so).
 *
 * The reference (QwenLM/Qwen3-TTS) is pure Python with no FFI/plugin interface (SURVEY.md §8b), so the
 * boundary below is defined at the two narrowest seams of the reference and each entry point cites the
 * reference interface it replaces (paths relative to /root/reference/qwen_tts/):
 *
 *   seam B (AR)   : Qwen3TTSTalkerForConditionalGeneration.generate(inputs_embeds, attention_mask,
 *                   trailing_text_hidden, tts_pad_embed, **talker_kwargs)
 *                   as called at core/models/modeling_qwen3_tts.py:2272-2278, including the per-frame
 *                   forward :1636-1744, the nested code-predictor generate :1671-1680 / :1250-1312 and the
 *                   HF logits processors + sampling configured at :2044-2066.
 *   seam C (codec): Qwen3TTSTokenizerV2Decoder.forward / chunked_decode
 *                   core/tokenizer_12hz/modeling_qwen3_tts_tokenizer_v2.py:869-896 (called by
 *                   Qwen3TTSTokenizerV2Model.decode :993-1024).
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on error; q3_last_error() gives the message
 *     (thread-local).
 *   - all `dev` pointers are CUDA device pointers on the engine's device; the caller (PyTorch) OWNS them.
 *     The engine owns only what it allocates itself (packed weights, KV cache, workspaces).
 *   - `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream); work is
 *     enqueued on it, calls do not synchronise unless documented.  One engine = one device, not re-entrant.
 *     Apart from the debug and hidden-capture buffers, which must stay valid until cleared, the engine reads caller
 *     memory only in work it queues on `stream` during the call.
 *   - bf16 tensors are raw uint16 storage (torch.bfloat16).  No torch types cross this boundary.
 */
#ifndef QWEN3TTS_B200_H
#define QWEN3TTS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define Q3_ABI_VERSION 2
#define Q3_MAX_BATCH 32        /* sequences per engine pass (reference batches = padded batch on one GPU) */
#define Q3_NUM_GROUPS_MAX 32

typedef struct q3_engine q3_engine; /* AR engine: talker + code predictor + sampler */
typedef struct q3_codec q3_codec;   /* 12 Hz codec decoder */

/* One decoder stack.  Mirrors Qwen3TTSTalkerConfig / Qwen3TTSTalkerCodePredictorConfig
 * (core/models/configuration_qwen3_tts.py:370-404, :187-212); values come from the loaded config. */
typedef struct {
  int32_t hidden_size, num_layers, num_heads, num_kv_heads, head_dim, intermediate_size, vocab_size;
  float rms_eps;
} q3_stack_cfg;

typedef struct {
  q3_stack_cfg talker, cp;
  int32_t num_code_groups;   /* 16 */
  int32_t has_cp_projection; /* small_to_mtp_projection is a Linear (1.7B) or Identity (0.6B), :1171-1174 */
  int32_t codec_eos_token_id;
  int32_t max_batch;         /* <= Q3_MAX_BATCH */
  int32_t max_ctx;           /* talker KV capacity per sequence (prompt + frames) */
  int32_t device;            /* CUDA ordinal */
} q3_engine_cfg;

/* Generation kwargs of seam B (modeling_qwen3_tts.py:2044-2066; defaults inference/qwen3_tts_model.py:287-352).
 * Accepted ranges (HF's processors, plus finiteness where the sampler needs it); q3_prefill, q3_session_begin and
 * q3_admit_with_sampling reject anything else with an error naming the field, before any device work (q3_sampling_check
 * applies the same rules on its own):
 *   temperature / subtalker_temperature: finite and > 0 when do_sample / subtalker_dosample is set (ignored otherwise);
 *   top_k, subtalker_top_k >= 0 (0 = off); 0 <= top_p, subtalker_top_p <= 1 (1 = off);
 *   repetition_penalty finite and > 0 (1 = off); min_new_tokens >= 0. */
typedef struct {
  int32_t do_sample, top_k;
  float top_p, temperature, repetition_penalty;
  int32_t subtalker_dosample, subtalker_top_k;
  float subtalker_top_p, subtalker_temperature;
  int32_t min_new_tokens;  /* 2 */
  int32_t suppress_eos;    /* benchmark-only: fixed horizon (EOS never sampled) */
  uint64_t seed;           /* Philox key; u = philox(seed; row, frame, group) */
} q3_sampling;

int q3_abi_version(void);
const char* q3_last_error(void);

/* ---------------------------------------------------------------- AR engine (seam B) */
int q3_engine_create(const q3_engine_cfg* cfg, q3_engine** out);
void q3_engine_destroy(q3_engine* e);

/* Copy+repack one weight from device memory (bf16, row-major [rows][cols], i.e. nn.Linear/nn.Embedding
 * layout).  `name` is one of the engine tensor names documented in INTEGRATION.md, e.g.
 *   "talker.layers.<i>.qkv"  = cat(q_proj,k_proj,v_proj).weight          (:740-748)
 *   "talker.layers.<i>.gate_up" = gate/up rows interleaved in blocks of 8 (:848-849)
 *   "talker.layers.<i>.o", ".down", ".ln1", ".ln2", ".q_norm", ".k_norm"
 *   "talker.norm", "talker.codec_head", "talker.codec_embedding", "talker.rope_cos", "talker.rope_sin"
 *   "cp.layers.<i>.*", "cp.norm", "cp.proj", "cp.proj_bias", "cp.lm_head.<j>", "cp.codec_embedding.<j>",
 *   "cp.rope_cos", "cp.rope_sin".
 * The source may be freed after the call returns (the copy is complete by then). */
int q3_engine_load_tensor(q3_engine* e, const char* name, const void* dev_bf16, int64_t rows, int64_t cols);
int q3_engine_finalize(q3_engine* e); /* verifies that every tensor is present */

/* Prefill = first `talker.generate` forward (modeling_qwen3_tts.py:1665-1667 -> :1457-1561).
 * embeds: bf16 [sum(lens)][H], rows of sequence 0 first (NO padding: the reference's left-pad+mask,
 * :2239-2254, is equivalent to per-sequence positions 0..len-1).  lens: host int32[B].
 * trailing: bf16 [B][trailing_stride][H] (row b valid for trailing_lens[b] steps, then tts_pad, :1689-1692);
 * tts_pad: bf16 [H].  Resets all per-request state (per request, never on a module: SURVEY F10) and samples
 * codebook-0 of frame 0: the batch is a session of B slots whose rows are all admitted at frame 0 with the Philox row
 * keys 0..B-1 and the parameters sp.  Every row is checked before any state changes: a rejected call leaves the
 * running batch as it was. */
int q3_prefill(q3_engine* e, int32_t B, const void* embeds_dev, const int32_t* lens_host,
               const void* trailing_dev, const int32_t* trailing_lens_host, int32_t trailing_stride,
               const void* tts_pad_dev, const q3_sampling* sp, void* stream);

/* Run up to `max_frames` further frame-steps (code predictor x15 -> embed -> talker -> head -> sample),
 * stopping early once every row has sampled EOS.  No host sync per token (HF syncs every token).
 * codes_dev: int32 [B][codes_stride][num_code_groups], frame f of row b at [b][f][:]; frames accumulate
 * across calls (streaming = repeated calls with small max_frames).  Asynchronous. */
int q3_decode(q3_engine* e, int32_t max_frames, int32_t* codes_dev, int32_t codes_stride, void* stream);

/* ---- continuous batching (SURVEY §8f-4; the reference has only the static padded batch of
 * modeling_qwen3_tts.py:2239-2254 behind a Gradio queue, cli/demo.py:629).  A session owns n_slots rows; a finished or
 * never-used slot is a row that keeps stepping and is ignored (exactly what HF does with finished rows of a batch).
 * q3_admit_with_sampling prefills n new requests into free slots WHILE the others keep their state: their K/V,
 * positions, sampling history and Philox streams are per row, so a request admitted at any frame generates what it
 * would generate alone (keys_host[r] is the request's Philox row key).  q3_decode / q3_get_progress are shared with the
 * static path; n_valid[b] counts the row's OWN frames, and the row's codes land at codes[b][0..n_valid).
 * q3_admit_with_sampling synchronises `stream` (it needs the frame counter).  embeds_dev: the n prompts packed back to
 * back; trailing_dev: [n][stride][H]. */
int q3_session_begin(q3_engine* e, int32_t n_slots, int32_t max_trailing, const void* tts_pad_dev, const q3_sampling* sp,
                     void* stream);
/* Request r samples (its prefill head and every frame-step) with sp_host[r] (host array [n]; NULL = the session's sp
 * for all) and the Philox key (sp_host[r].seed, keys_host[r]), so it generates what it would generate alone in a
 * session whose parameters are sp_host[r].  A row without a running request (never admitted, finished, released)
 * samples with the session's sp.
 * All n entries are checked (q3_sampling_check) before any other argument and any device work; a bad one fails the
 * whole call with an error naming the request index and the field.  Then every row (slot, prompt and trailing length,
 * trailing text) is checked before any state changes: a rejected call admits no row, and no slot, key or parameter
 * changes. */
int q3_admit_with_sampling(q3_engine* e, int32_t n, const int32_t* slots_host, const uint32_t* keys_host,
                           const q3_sampling* sp_host, const void* embeds_dev, const int32_t* lens_host,
                           const void* trailing_dev, const int32_t* trailing_lens_host, int32_t trailing_stride,
                           void* stream);
/* ---- registered prompt prefixes: rows that many requests' prompts begin with (a voice's instruct, role and codec
 * prefix rows, an ICL clone's reference).  q3_prefix_create runs the talker layers over `len` rows embeds_dev bf16
 * [len][H] on `stream` and keeps their K and V ([2][layers][nkv][len][128] bf16, 114,688 B per row at the 1.7B shape) in
 * a device block of the engine; *id_out receives its id.  1 <= len < max_ctx - 1.  It writes no slot's K/V and no
 * row's state, so it may run between two decodes of a session.  Prefixes survive q3_session_begin and q3_prefill, and
 * live until q3_prefix_free or q3_engine_destroy.  q3_prefix_free synchronises `stream` (an admission's copy of the
 * block may be queued on it) and releases the block; the id is never reused.  q3_prefix_length: the prefix's rows, or
 * -1 when no such prefix exists. */
int q3_prefix_create(q3_engine* e, const void* embeds_dev, int32_t len, void* stream, int32_t* id_out);
int q3_prefix_free(q3_engine* e, int32_t id, void* stream);
int q3_prefix_length(q3_engine* e, int32_t id);
/* q3_admit_with_sampling where request r's prompt is the prefix prefix_ids_host[r] (-1: none; prefix_ids_host == NULL:
 * none for all) followed by lens_host[r] rows of its own (at least 1).  The prefix's K/V are copied into the slot's
 * cache at positions [0, P) (P its length) and only the request's own rows are prefilled, at positions P.., so the
 * request generates exactly what q3_admit_with_sampling of cat(prefix rows, own rows) generates: every prefill stage is
 * row-wise or causal within one sequence.  Besides the checks of q3_admit_with_sampling, each request's prefix must
 * exist and P + lens_host[r] < max_ctx; a rejected call admits no row.  Errors name the request index.
 * q3_admit_with_sampling is this call with prefix_ids_host == NULL. */
int q3_admit_with_prefix(q3_engine* e, int32_t n, const int32_t* slots_host, const uint32_t* keys_host,
                         const q3_sampling* sp_host, const int32_t* prefix_ids_host, const void* embeds_dev,
                         const int32_t* lens_host, const void* trailing_dev, const int32_t* trailing_lens_host,
                         int32_t trailing_stride, void* stream);
/* The range check q3_prefill, q3_session_begin and q3_admit_with_sampling apply (see q3_sampling): 0 if sp is
 * accepted, else non-zero with q3_last_error() naming the field.  Host only: needs no engine and no GPU. */
int q3_sampling_check(const q3_sampling* sp);
/* Streaming text input: append n rows [n][H] bf16 to the trailing_text_hidden of a running row (static batch or session);
 * frame t adds trailing[t] while t < the row's trailing length and tts_pad afterwards (modeling_qwen3_tts.py:1689-1692).
 * The capacity is the trailing stride given at q3_prefill / max_trailing of q3_session_begin. */
int q3_append_trailing(q3_engine* e, int32_t slot, const void* rows_dev, int32_t n, void* stream);
/* Live text: open = 1 marks a running row (admitted, not released, of a static batch or a session) whose text may
 * still grow.  A step of an open row whose text row has not arrived (row frame >= trailing length) is HELD instead of
 * reading tts_pad: it commits nothing, and q3_decode moves the row back onto its committed steps before it returns, so
 * the next decode runs that step again.  An open row therefore generates exactly what it generates with the whole text
 * given up front, however its rows arrive.  open = 0 closes the row: past its text it reads tts_pad again.  Every
 * admission starts closed.  Refused while hidden-state capture is set (q3_decode refuses the combination too). */
int q3_set_trailing_open(q3_engine* e, int32_t slot, int32_t open);
/* give up rows that reached their frame horizon without EOS (their slots become free) */
int q3_release_slots(q3_engine* e, int32_t n, const int32_t* slots_host, void* stream);
/* ---- parked rows (session only): a running request leaves its slot and later continues in any free slot.
 * q3_row_park moves the request of `slot` (admitted, not finished, released or parked) into a record, a device block of
 * the engine: its talker K/V at positions [0, pos) (pos = the position its next step writes) in the layout of a
 * registered prefix, and every per-row state a frame-step reads before it writes it (the row's DevState fields, its
 * repetition-penalty row, its code-predictor input rows, past_hidden / past_keep, its trailing text), plus on the host its
 * committed frames, Philox key, sampling parameters and live-text flags.  One launch on `stream`, no host sync; the slot
 * is then free as after q3_release_slots, and *id_out receives the record's id (never reused).  The caller's codes
 * buffer is not saved.  q3_row_resume synchronises `stream` (it needs the frame counter, like an admission), puts record
 * `id` into the free slot `slot` with one launch, synchronises again and frees the record: the request then generates
 * exactly the frames it would have generated never parked, and q3_get_progress reports the same n_valid as before the
 * park (committed frames + 1 for a row the last decode left held).  q3_row_discard frees a record without resuming it
 * (after synchronising `stream`).  Records belong to their session: q3_session_begin, q3_prefill and q3_engine_destroy
 * free them all.  Refused, before any device work and with every row, record and position unchanged, with an error
 * naming the slot or id: not a session; a slot out of range or without a running request; hidden-state capture or
 * teacher forcing set; resume into a running slot; an unknown, resumed or discarded id, or one of an earlier session;
 * a record whose position would not fit max_ctx; a failed allocation (the row keeps running). */
int q3_row_park(q3_engine* e, int32_t slot, void* stream, int32_t* id_out);
int q3_row_resume(q3_engine* e, int32_t id, int32_t slot, void* stream);
int q3_row_discard(q3_engine* e, int32_t id, void* stream);

/* After synchronising `stream`: frames_done = frames whose 16 codes are complete (same for all rows);
 * n_valid[b] = frames of row b before its first EOS (== modeling_qwen3_tts.py:2283-2290 trim); for a row the last
 * decode left held, its committed frames + 1 (the held step's 16 codes are final: they do not depend on its text);
 * finished[b] = 1 once row b sampled EOS.  Host pointers (may be NULL). */
int q3_get_progress(q3_engine* e, int32_t* frames_done, int32_t* n_valid, int32_t* finished);

/* Per-step hidden states = the second return value of generate() (modeling_qwen3_tts.py:2281: the last layer's normed
 * output of the newest position of every step): hid_dev bf16 [B][stride][hidden] gets row b's step s at [b][s][:]
 * (s = 0 is the prefill).  NULL disables the capture.  Call before q3_prefill. */
int q3_set_hidden_capture(q3_engine* e, void* hid_dev, int32_t stride);

/* Test hooks (used by tests/ only): teacher forcing and raw-logit capture.
 * forced: int32 [B][n_frames][G] device (or NULL to disable); talker_logits: fp32 [n_frames+1][B][V];
 * cp_logits: fp32 [n_frames][G-1][B][Vc].  Pointers must stay valid until cleared. */
int q3_set_debug(q3_engine* e, const int32_t* forced_dev, int32_t n_frames, float* talker_logits_dev,
                 float* cp_logits_dev);

/* Profiling hooks (tools/profile_frame.py): prof_dev = uint64 [n_phases][grid][16], written by thread 0 of EVERY CTA
 * during the first frame of each q3_decode while it is set (the decode then runs the profiled kernel instantiation).
 * %globaltimer ns: [0] phase body end, [1] barrier passed, [2..4] inner marks of the phase body (GEMV: activations
 * staged, main loop done, epilogue done; attention: K/V window loaded, partials done, combine done), [6] phase start, [8] / [7] start / end of
 * warp 0's GEMV main loop; [5] clock cycles warp 0 waited for ring data in a GEMV phase; slots 9..15 are not written.
 * q3_describe_frame_program returns -n_phases and fills kinds[i] = type*100 + stack*10 + epilogue. */
int q3_set_profile(q3_engine* e, unsigned long long* prof_dev);
int q3_describe_frame_program(q3_engine* e, int32_t* kinds, int32_t capacity);

/* Bytes the fused frame-step kernel must stream per step for batch B at mean context S
 * (SURVEY §8d: W_talker + W_cp_unique + B*(S+1)*KV_tok), and the no-residency figure. */
int q3_algorithmic_bytes(q3_engine* e, int32_t B, int32_t S, double* a_bytes, double* a_stream_bytes);

/* ---------------------------------------------------------------- codec decoder (seam C) */
/* Mirrors Qwen3TTSTokenizerV2DecoderConfig (core/tokenizer_12hz/configuration_qwen3_tts_tokenizer_v2.py:72-93). */
typedef struct {
  int32_t codebook_size, codebook_dim, hidden_size, latent_dim;
  int32_t num_heads, num_kv_heads, head_dim, sliding_window, intermediate_size, num_layers, num_quantizers;
  int32_t n_upsample_rates;    int32_t upsample_rates[8];    /* (8,5,4,3) */
  int32_t n_upsampling_ratios; int32_t upsampling_ratios[8]; /* (2,2)     */
  int32_t decoder_dim;
  float rms_eps, rope_theta;
  int32_t max_frames;  /* per forward (chunk_size + left_context = 325 in the reference) */
  int32_t max_batch;
  int32_t device;
} q3_codec_cfg;

int q3_codec_create(const q3_codec_cfg* cfg, q3_codec** out);
void q3_codec_destroy(q3_codec* c);
/* Engine-native tensors, converted from the reference decoder's state_dict by the host
 * (qwen3-tts_b200/codec.py documents every name; INTEGRATION.md lists the mapping).  GEMM weights are bf16
 * [N][ntaps*Kp] (K-major per tap, Kp = K rounded up to 64; Conv1d taps in kernel order, ConvTranspose1d as
 * N = stride*Cout with 2 taps), biases / SnakeBeta / LayerScale / LayerNorm parameters fp32.  dtype is implied
 * by the name (".w", ".table", ".proj", ".norm", ".ln1", ".ln2", ".cos", ".sin" = bf16; the rest fp32). */
int q3_codec_load_tensor(q3_codec* c, const char* name, const void* dev, const int64_t* shape, int32_t ndim);
int q3_codec_finalize(q3_codec* c);
/* One full causal forward == Qwen3TTSTokenizerV2Decoder.forward (…v2.py:869-884).
 * codes: int32 [B][K][T] device; wav: fp32 [B][T*upsample] device.  Asynchronous. */
int q3_codec_forward(q3_codec* c, const int32_t* codes_dev, int32_t B, int32_t T, float* wav_dev, void* stream);

/* ---- stateful streaming decoder (SURVEY §8b / §8f-2).  The reference decodes whole utterances, or chunks with 25
 * re-decoded frames of left context (chunked_decode, tokenizer_12hz/modeling_qwen3_tts_tokenizer_v2.py:886-896); this
 * handle carries the decoder's causal state instead (conv tails, ConvTranspose overlap row, 71 frames of rotated K/V
 * per transformer layer), so pushing packets of any sizes yields exactly the waveform of the full causal forward
 * (…v2.py:869-884) over everything pushed, with only the NEW frames' work per packet.
 * open: B rows, packets of <= max_packet_frames frames.  A row's position (frames pushed since its reset) may not pass
 * the engine's max_frames (RoPE table).  Every row has its own position (continuous batching: rows start and end at
 * different frames, slots are reused):
 * step_rows: codes_dev int32 [B][num_quantizers][n] (the next n frames of every row) -> wav_dev fp32
 *   [B][n * total_upsample]; asynchronous on `stream`.  Row b takes only the first counts_host[b] (0 <= counts_host[b]
 *   <= n, host int32 [B]) of the n frames; its audio is wav_dev[b][0, counts_host[b] * total_upsample) and the rest of
 *   its row is zeros.  Codes past a row's count are never read (any value, -1 included).  A row with count 0 keeps its
 *   state and position.
 * reset_rows: the n rows in rows_host (host int32, each in [0, B), no repeats) start new utterances at position 0;
 *   the other rows are untouched.
 * row_position: frames pushed to one row since its reset.
 * Bad arguments (a count outside [0, n], position + count > max_frames, a reset row out of range or listed twice, null
 * pointers) are rejected with an error naming the row before any device work, and leave every position unchanged. */
typedef struct q3_codec_stream q3_codec_stream;
int q3_codec_stream_open(q3_codec* c, int32_t B, int32_t max_packet_frames, q3_codec_stream** out);
int q3_codec_stream_step_rows(q3_codec_stream* s, const int32_t* codes_dev, int32_t n, const int32_t* counts_host,
                              float* wav_dev, void* stream);
int q3_codec_stream_reset_rows(q3_codec_stream* s, int32_t n, const int32_t* rows_host, void* stream);
int q3_codec_stream_row_position(q3_codec_stream* s, int32_t row);
/* copy_rows: for i < n, row dst_rows_host[i] of dst becomes exactly row src_rows_host[i] of src (host int32 [n]): its
 *   decoder state (the history of every buffer: conv tails, ConvTranspose overlap rows, each layer's K/V window) and
 *   its position.  The destination row's previous state is replaced, so a running row needs no reset first.  Both
 *   streams come from the same codec; their B and max_packet_frames may differ.  A source row may be listed more than
 *   once (it is forked); a destination row may not.  One kernel launch, asynchronous on `stream`, no host sync.
 *   Voice cloning decodes cat(ref_code, generated codes) and keeps the generated part (qwen3_tts_model.py:612-631):
 *   decode the reference prefix once in a private stream, then copy its rows into the serving stream's rows.
 *   Bad arguments (null or equal streams, different codecs, n outside [0, dst B], a row out of range, a destination
 *   row listed twice) are rejected before any device work and change nothing. */
int q3_codec_stream_copy_rows(q3_codec_stream* dst, const q3_codec_stream* src, int32_t n, const int32_t* src_rows_host,
                              const int32_t* dst_rows_host, void* stream);
void q3_codec_stream_close(q3_codec_stream* s);
int q3_codec_total_upsample(q3_codec* c);
/* kernels launched by the last q3_codec_forward or q3_codec_stream_step_rows (bench.py's gpu_launches bookkeeping) */
int q3_codec_last_launch_count(q3_codec* c);
/* Test hook (tests/ only): per-stage capture of the DECODER, so that an error in one small kernel cannot hide behind the
 * waveform SNR.  The following q3_codec_forward calls copy the bf16 [B][T_stage][C_stage] tensor of `stage` into dst_dev
 * (at most `capacity` elements): 0 pre_conv output (…v2.py:874), 1 pre-transformer output (:875-876), 2 output of the
 * upsample stack (:878-880), 3 SnakeBeta(decoder.0 output) as fed to block 0 (:857,:646), 4+i output of decoder block i
 * (:638-658).  stage < 0 clears all captures. */
int q3_codec_debug_capture(q3_codec* c, int32_t stage, void* dst_dev, int64_t capacity);

/* ---------------------------------------------------------------- codec ENCODER (Qwen3TTSTokenizer.encode)
 * Replaces Qwen3TTSTokenizerV2Model.encode (core/tokenizer_12hz/modeling_qwen3_tts_tokenizer_v2.py:961-991), i.e.
 * transformers MimiModel._encode_frame (modeling_mimi.py:1455-1488), restricted to the first
 * `encoder_valid_num_quantizers` levels (the reference computes 32 and keeps 16, :981-983).  fp32 end to end:
 * the output is discrete (nearest-centroid indices), see csrc/codec_encoder.cu. */
typedef struct {
  int32_t num_filters, kernel_size, last_kernel_size, residual_kernel_size, compress; /* MimiConfig SEANet fields */
  int32_t n_ratios, ratios[8];        /* downsampling strides in encoder order = reversed(upsampling_ratios): 4,5,6,8 */
  int32_t hidden_size, num_layers, num_heads, head_dim, intermediate_size, sliding_window;
  float norm_eps;
  int32_t codebook_size, codebook_dim;
  int32_t num_semantic_quantizers;    /* 1 */
  int32_t num_quantizers;             /* levels to compute = encoder_valid_num_quantizers (16) */
  int32_t downsample_stride;          /* encodec_frame_rate / frame_rate = 2 */
  int32_t max_frames;                 /* rows of the RoPE tables (transformer frames, 25 Hz) */
  int32_t device;
} q3_codec_enc_cfg;
typedef struct q3_codec_enc q3_codec_enc;

int q3_codec_enc_create(const q3_codec_enc_cfg* cfg, q3_codec_enc** out);
void q3_codec_enc_destroy(q3_codec_enc* e);
/* fp32 device tensors, engine-native names (qwen3-tts_b200/codec_encoder.py::_load maps MimiModel's state_dict):
 *   "enc.conv0|enc.res<i>.a|enc.res<i>.b|enc.down<i>|enc.conv_last" + ".w" [Cout][Cin][k] / ".b" [Cout];
 *   "tr.<l>.ln1.w/.b", "tr.<l>.qkv.w" [3C][C] = cat(q,k,v), "tr.<l>.o.w", "tr.<l>.ls1", "tr.<l>.ln2.w/.b",
 *   "tr.<l>.fc1.w" [I][C], "tr.<l>.fc2.w" [C][I], "tr.<l>.ls2"; "rope.cos|sin" [max_frames][head_dim/2];
 *   "down.w" [C][C][2*stride]; "rvq.sem.proj.w|rvq.ac.proj.w" [D][C]; per level q (0 = semantic):
 *   "rvq.<q>.e" [K][D] = embed_sum / clamp(cluster_usage, 1e-5), "rvq.<q>.et" [D][K], "rvq.<q>.e2" [K] = |e|^2. */
int q3_codec_enc_load_tensor(q3_codec_enc* e, const char* name, const float* dev, const int64_t* shape, int32_t ndim);
int q3_codec_enc_finalize(q3_codec_enc* e);
/* wav: fp32 [B][T] device (rows right-padded with zeros: every layer is causal, so padding never reaches earlier
 * frames); codes: int32 [B][num_quantizers][q3_codec_enc_frames(T)] device.  Asynchronous. */
int q3_codec_enc_encode(q3_codec_enc* e, const float* wav_dev, int32_t B, int32_t T, int32_t* codes_dev, void* stream);
int q3_codec_enc_frames(q3_codec_enc* e, int32_t T);   /* ceil-chain through every stride */
int q3_codec_enc_hop(q3_codec_enc* e);                 /* samples per frame (1920) */
int q3_codec_enc_last_launch_count(q3_codec_enc* e);
/* Test hook: copy the activation [B][C][T] after stage `stage` (conv0, per ratio [res, down], conv_last, one per
 * transformer layer, downsample) of the next encode into dst; stage < 0 clears all captures. */
int q3_codec_enc_debug_capture(q3_codec_enc* e, int32_t stage, float* dst_dev, int64_t capacity);

/* ---- stateful streaming encoder.  The encoder is causal (causal convolutions, a causal sliding-window transformer,
 * a causal stride-2 downsample), so whole 1920-sample frames can be encoded as they arrive: this handle carries each
 * row's causal state (the conv tails, the transformer's residual stream tail for the downsample, window - 1 columns of
 * rotated K and V per transformer layer) and runs the one-shot's kernels over only the new frames.  The codes of a clip
 * pushed in packets of any sizes and ended with finish_rows equal q3_codec_enc_encode of that clip alone (B = 1) bit
 * for bit.  Only the clip's final partial frame needs the clip's end: the one-shot pads every layer on the right, which
 * is not the same as encoding zero audio, so finish_rows encodes it on its own path.
 * open: B rows (<= Q3_MAX_BATCH), packets of <= max_packet_frames frames.  A row's 25 Hz position (2 x its 12.5 Hz
 * frames since reset) may not pass the encoder's max_frames (RoPE table), as in the one-shot.
 * step_rows: wav_dev fp32 [B][n * hop]; row b takes its first counts_host[b] frames (0..n, host int32 [B]);
 *   codes_dev int32 [B][num_quantizers][n], row b's codes past counts_host[b] are -1.  Samples past a row's count are
 *   never read.  A row with count 0 keeps its state and position.  Asynchronous on `stream`, no host sync.
 * finish_rows: for i < n, row rows_host[i] ends its clip with tail_host[i] (0..hop-1) samples at wav_dev[i][0..tail)
 *   (wav_dev fp32 [n][hop]); codes_dev int32 [n][num_quantizers] = its last frame (-1 when the tail is 0).  The row is
 *   then reset.  Asynchronous.
 * reset_rows: the n rows in rows_host (host int32, each in [0, B), no repeats) start new clips at position 0.
 * row_position: 12.5 Hz frames encoded for one row since its reset (-1 for a bad row).
 * Bad arguments (a count outside [0, n], n > max_packet_frames, a tail outside [0, hop), a row out of range or listed
 * twice, null pointers, a row whose 25 Hz position would pass max_frames) are rejected with an error naming the row
 * before any device work, and leave every position unchanged. */
typedef struct q3_codec_enc_stream q3_codec_enc_stream;
int q3_codec_enc_stream_open(q3_codec_enc* e, int32_t B, int32_t max_packet_frames, q3_codec_enc_stream** out);
int q3_codec_enc_stream_step_rows(q3_codec_enc_stream* s, const float* wav_dev, int32_t n, const int32_t* counts_host,
                                  int32_t* codes_dev, void* stream);
int q3_codec_enc_stream_finish_rows(q3_codec_enc_stream* s, int32_t n, const int32_t* rows_host, const int32_t* tail_host,
                                    const float* wav_dev, int32_t* codes_dev, void* stream);
int q3_codec_enc_stream_reset_rows(q3_codec_enc_stream* s, int32_t n, const int32_t* rows_host, void* stream);
int q3_codec_enc_stream_row_position(q3_codec_enc_stream* s, int32_t row);
void q3_codec_enc_stream_close(q3_codec_enc_stream* s);

/* ---------------------------------------------------------------- audio rate and encoding (streaming resampler)
 * Stands beside the reference's librosa.resample / scipy.signal.resample_poly calls (qwen3_tts_tokenizer.py:156,204):
 * the polyphase FIR rate conversion of resample_poly, streamed over many rows, with an encoding epilogue.  For a rate
 * pair up/down (reduced) and taps h[0..ntaps), ntaps = 2*hl + 1 (resample_poly's firwin(2*hl+1, 1/max(up,down),
 * ("kaiser", 5.0)) * up, designed by the caller; [1.0] for equal rates), output j of a clip x[0..n) is
 *   y[j] = sum_m x[m] * h[hl + j*down - m*up]  over 0 <= m < n, 0 <= hl + j*down - m*up <= 2*hl,
 * an fp32 sum in ascending m, and the clip has ceil(n*up/down) outputs.  Output j is emitted once input
 * floor((hl + j*down)/up) has arrived, so after n inputs without an end a row has emitted
 * E(n) = max(0, floor((n*up - 1 - hl)/down) + 1); the end emits the rest, with x = 0 past the clip.  A clip streamed in
 * pushes of any sizes equals the clip pushed at once, bit for bit.  Encodings of y: F32 as is; S16 =
 * clamp(rint(y*32768), -32768, 32767) (round half to even); ULAW = G.711 mu-law of that S16 value as
 * audioop.lin2ulaw(..., 2) computes it.
 * open: `rows` rows; a step gives each row at most max_in inputs; each row's output capacity is max_out samples
 *   (4*max_out bytes).  Device memory of the object is its own.
 * add_filter: copies the device taps (fp32 [ntaps]) into the object and returns their id in *id_out.  A filter may
 *   not read more than Q3_RESAMPLE_HIST inputs back (floor(2*hl/up)), nor emit more than max_out samples from a push of
 *   max_in inputs plus its end (ceil(max_in*up/down) + ceil(hl/down) + 1).  At most 64 filters at a time; a new filter
 *   takes the lowest free id, so an id dropped by drop_filter may come back for another filter.
 * drop_filter: frees filter `id` and its id.  Refused while any row uses it (reset or loaded with it and not released
 *   since).  Drains the device first, as launches queued on any stream may read its taps.
 * release_rows: the n rows in rows_host no longer use their filters; they may take neither inputs nor an end until they
 *   are reset or loaded again.  Host state only.
 * reset_rows: the n rows in rows_host start new clips with filter filters_host[i] and encoding encodings_host[i]
 *   (Q3_RESAMPLE_F32 / S16 / ULAW).  Host state only, no device work.
 * step_rows: one launch over every row.  Row r takes counts_host[r] (0..max_in) fp32 inputs at in_dev + r*ld and, when
 *   end_host[r] != 0, ends its clip (it then starts a new one with the same filter and encoding).  Its new outputs go
 *   to out_dev + r*4*max_out bytes in its encoding (4, 2 or 1 bytes each), and their count to nout_host[r], known
 *   without a sync.  A row with count 0 and no end is untouched.  A row never reset may take neither inputs nor an end.
 *   Asynchronous on `stream`; the rows' histories move on the device.
 * save_rows: the n listed rows' state (filter id, encoding, inputs so far, history) to dst_dev, Q3_RESAMPLE_ROW_BYTES
 *   bytes per row in list order.  Asynchronous.
 * load_rows: the n listed rows continue the states saved at src_dev (by this object): reads the records' headers back
 *   to the host (synchronises `stream`), then copies the histories asynchronously.  A record's filter id (its first 4
 *   bytes) must name a live filter: a caller that dropped the filter since the save adds it again and writes its new
 *   id there first.
 * Bad arguments (a row out of range or listed twice, a count outside [0, max_in] or above ld, an unknown filter or
 *   encoding, a row never reset, null pointers) are rejected before any device work and change nothing. */
#define Q3_RESAMPLE_HIST 128
#define Q3_RESAMPLE_ROW_BYTES 528
#define Q3_RESAMPLE_F32 0
#define Q3_RESAMPLE_S16 1
#define Q3_RESAMPLE_ULAW 2
typedef struct q3_resampler q3_resampler;
int q3_resample_open(int32_t rows, int32_t max_in, int32_t max_out, int32_t device, q3_resampler** out);
void q3_resample_close(q3_resampler* s);
int q3_resample_add_filter(q3_resampler* s, int32_t up, int32_t down, const float* taps_dev, int32_t ntaps, int32_t* id_out);
int q3_resample_reset_rows(q3_resampler* s, int32_t n, const int32_t* rows_host, const int32_t* filters_host,
                           const int32_t* encodings_host);
int q3_resample_drop_filter(q3_resampler* s, int32_t id);
int q3_resample_release_rows(q3_resampler* s, int32_t n, const int32_t* rows_host);
int q3_resample_step_rows(q3_resampler* s, const float* in_dev, int64_t ld, const int32_t* counts_host,
                          const int32_t* end_host, void* out_dev, int32_t* nout_host, void* stream);
int q3_resample_save_rows(q3_resampler* s, int32_t n, const int32_t* rows_host, void* dst_dev, void* stream);
int q3_resample_load_rows(q3_resampler* s, int32_t n, const int32_t* rows_host, const void* src_dev, void* stream);

/* ---------------------------------------------------------------- speaking rate (streaming WSOLA time-stretch)
 * Waveform-similarity overlap-add at the codec's 24 kHz with fixed geometry: frame N = 960, synthesis hop Hs = 480,
 * search tolerance D = 240, analysis hop Ha in [240, 960] (Ha = floor(speed*480 + 0.5)), window w[n] = sin^2(pi*n/960)
 * (fp32, designed by the caller).  Frame k has nominal position a_k = k*Ha and chosen position p_k = a_k + d_k, d_0 = 0;
 * for k >= 1, d_k in [-D, D] maximises C_k(d) = sum_{n<480} x[p_{k-1} + 480 + n] * x[a_k + d + n] (fp32, acc = 0 then
 * one fused multiply-add per n in ascending n), ties to the smallest |d|, then to the negative d.  Output:
 *   y[m] = x[m]  (m < 480);  y[k*480 + i] = fl(fl(w[i]*x[p_k + i]) + fl(w[i+480]*x[p_{k-1} + i + 480]))  (k >= 1, i < 480),
 * and a clip x[0..n) gives M(n) = ceil(n*480/Ha) samples, with x = 0 past n.  Frame k is done once input
 * a_k + D + N - 1 has arrived, so after n inputs without an end a row has emitted E(n) = 480*(floor((n - 1200)/Ha) + 1)
 * (0 for n < 1200); an end emits [E(n), M(n)).  A clip streamed in pushes of any sizes equals the clip pushed at once.
 * open: `rows` rows; a step gives each row at most max_in (1 .. 32768) inputs; each row's output capacity is max_out fp32
 *   samples, at least ceil((max_in + 1199)*480/240).  Device memory of the object is its own.
 * set_window: copies the device window (fp32 [960]) into the object.  Required before the first step.
 * reset_rows: the n rows in rows_host start new clips with analysis hop hops_host[i].  Host state only.
 * step_rows: one launch, one CTA per row with inputs or an end.  Row r takes counts_host[r] (0..max_in) fp32 inputs at
 *   in_dev + r*ld and, when end_host[r] != 0, ends its clip (it then starts a new one with the same hop).  Its new
 *   outputs go to out_dev + r*max_out (fp32), their count to nout_host[r], known without a sync.  A row with count 0 and
 *   no end is untouched.  A row never reset may take neither inputs nor an end.  Asynchronous on `stream`.
 * save_rows / load_rows: as q3_resample_save_rows / load_rows, Q3_STRETCH_ROW_BYTES per row (hop, inputs so far, frames
 *   done, p of the last frame done, its windowed second half, the last Q3_STRETCH_HIST inputs).  load synchronises.
 * Bad arguments are rejected before any device work and change nothing. */
#define Q3_STRETCH_HIST 2048
#define Q3_STRETCH_ROW_BYTES 10144
typedef struct q3_stretcher q3_stretcher;
int q3_stretch_open(int32_t rows, int32_t max_in, int32_t max_out, int32_t device, q3_stretcher** out);
void q3_stretch_close(q3_stretcher* s);
int q3_stretch_set_window(q3_stretcher* s, const float* window_dev);
int q3_stretch_reset_rows(q3_stretcher* s, int32_t n, const int32_t* rows_host, const int32_t* hops_host);
int q3_stretch_step_rows(q3_stretcher* s, const float* in_dev, int64_t ld, const int32_t* counts_host,
                         const int32_t* end_host, float* out_dev, int32_t* nout_host, void* stream);
int q3_stretch_save_rows(q3_stretcher* s, int32_t n, const int32_t* rows_host, void* dst_dev, void* stream);
int q3_stretch_load_rows(q3_stretcher* s, int32_t n, const int32_t* rows_host, const void* src_dev, void* stream);

/* ---------------------------------------------------------------- volume (streaming look-ahead limiter)
 * A gain that cannot clip, at the codec's 24 kHz, with peaks held at c = fp32(10^(-1/20)) (-1 dBFS).  Row gain g (fp32,
 * designed by the caller), u[n] = g*x[n] (x = 0 before the clip and past its end):
 *   a[n] = 1 if |u[n]| <= c, else c/|u[n]|;   b[m] = min a[m .. m+119];
 *   s[n] = min(a[n], (b[n] + b[n-1] + ... + b[n-119]) * fp32(1/120))   summed from b[n] down;
 *   G[n] = min over m in [max(0, n-1200), n] of s[m] + fp32(n-m) * fp32(1/1200);   y[n] = u[n] * G[n],
 * every operation fp32 round-to-nearest in that order, without contraction.  A clip of n samples gives n samples; output
 * n reads inputs up to n + 119, so after n inputs without an end a row has emitted E(n) = max(0, n - 119), and an end
 * emits the rest.  A clip streamed in pushes of any sizes equals the clip pushed at once, bit for bit.
 * open: `rows` rows; a step gives each row at most max_in inputs; each row's output capacity is max_out fp32 samples, at
 *   least max_in + 119.  Device memory of the object is its own.
 * reset_rows: the n rows in rows_host start new clips with gain gains_host[i] (positive, finite).  Host state only.
 * step_rows: one launch over every row.  Row r takes counts_host[r] (0..max_in) fp32 inputs at in_dev + r*ld and, when
 *   end_host[r] != 0, ends its clip (it then starts a new one with the same gain).  Its new outputs go to
 *   out_dev + r*max_out, their count to nout_host[r], known without a sync.  A row with count 0 and no end is
 *   untouched.  A row never reset may take neither inputs nor an end.  Asynchronous on `stream`.
 * save_rows / load_rows: as q3_resample_save_rows / load_rows, Q3_LIMIT_ROW_BYTES per row (gain, inputs so far, the last
 *   Q3_LIMIT_HIST inputs).  load synchronises.
 * Bad arguments are rejected before any device work and change nothing. */
#define Q3_LIMIT_HIST 1536
#define Q3_LIMIT_ROW_BYTES 6160
typedef struct q3_limiter q3_limiter;
int q3_limit_open(int32_t rows, int32_t max_in, int32_t max_out, int32_t device, q3_limiter** out);
void q3_limit_close(q3_limiter* s);
int q3_limit_reset_rows(q3_limiter* s, int32_t n, const int32_t* rows_host, const float* gains_host);
int q3_limit_step_rows(q3_limiter* s, const float* in_dev, int64_t ld, const int32_t* counts_host,
                       const int32_t* end_host, float* out_dev, int32_t* nout_host, void* stream);
int q3_limit_save_rows(q3_limiter* s, int32_t n, const int32_t* rows_host, void* dst_dev, void* stream);
int q3_limit_load_rows(q3_limiter* s, int32_t n, const int32_t* rows_host, const void* src_dev, void* stream);

/* ---------------------------------------------------------------- loudness (streaming BS.1770 normaliser)
 * A gain towards a target integrated loudness T (LUFS), decided while the audio streams, at the codec's 24 kHz.  The
 * input x is K-weighted (BS.1770-4 shelf then high-pass, fp32 in transposed direct form II, designed by the caller) over
 * complete segments s = [2400s, 2400s + 2400) only; z_s is the fp64 sum of a segment's squared K-weighted samples, block
 * j covers segments max(0, j-3) .. j with ms_j = (z_{j-3} + ... + z_j) / (2400*min(j+1, 4)) and l_j = -0.691 +
 * 10*log10(ms_j).  When segment s completes: Ja = {j <= s : l_j > -70}; if Ja is empty A_s = A_{s-1}, else
 * Gr = -0.691 + 10*log10(mean_Ja ms) - 10, J = {j in Ja : l_j > Gr}, I_s = -0.691 + 10*log10(mean_J ms) and
 * A_s = fp32(10^(clamp(T - I_s, -30, 30)/20)), all in fp64; A_{-1} = A_{-2} = 1.  Output n = 2400k + i:
 *   y[n] = x[n] * (A_{k-2} + (A_{k-1} - A_{k-2}) * fp32((i+1)/2400)),   fp32 round-to-nearest without contraction,
 * so a clip of n samples gives n samples with no delay, and an end emits nothing more.  A clip may hold at most
 * Q3_LOUD_MAX_BLOCKS segments (2400 * Q3_LOUD_MAX_BLOCKS samples).  A clip streamed in pushes of any sizes equals the
 * clip pushed at once, bit for bit.
 * open: `rows` rows; a step gives each row at most max_in (1 .. 32768) inputs; each row's output capacity is max_out fp32
 *   samples, at least max_in.  Device memory of the object is its own.
 * set_filter: the K-weighting, fp32 host sos[12]: two rows b0 b1 b2 a0 a1 a2 (shelf, then high-pass), a0 = 1.  Required
 *   before the first step.
 * reset_rows: the n rows in rows_host start new clips at target targets_host[i] (finite).  Host state only.
 * step_rows: one launch, one CTA per row with inputs.  Row r takes counts_host[r] (0..max_in) fp32 inputs at
 *   in_dev + r*ld and, when end_host[r] != 0, ends its clip (it then starts a new one at the same target).  Its new
 *   outputs go to out_dev + r*max_out, their count (counts_host[r]) to nout_host[r].  A row with count 0 and no end is
 *   untouched.  A row never reset may take neither inputs nor an end; a row whose clip would pass Q3_LOUD_MAX_BLOCKS
 *   segments is refused.  Asynchronous on `stream`.
 * save_rows / load_rows: as q3_resample_save_rows / load_rows, Q3_LOUD_ROW_BYTES per row: a Q3_LOUD_HEADER_BYTES header
 *   (target fp64, inputs so far int64, A_{k-1} and A_{k-2} fp32, the filter state fp32[4], z_{k-3..k-1} fp64[3]), the
 *   partial segment's inputs fp32[2400] and the block mean squares fp64[Q3_LOUD_MAX_BLOCKS].  load synchronises.
 * Bad arguments are rejected before any device work and change nothing. */
#define Q3_LOUD_MAX_BLOCKS 16384
#define Q3_LOUD_HEADER_BYTES 64
#define Q3_LOUD_ROW_BYTES 140736
typedef struct q3_loudness q3_loudness;
int q3_loud_open(int32_t rows, int32_t max_in, int32_t max_out, int32_t device, q3_loudness** out);
void q3_loud_close(q3_loudness* s);
int q3_loud_set_filter(q3_loudness* s, const float* sos_host);
int q3_loud_reset_rows(q3_loudness* s, int32_t n, const int32_t* rows_host, const double* targets_host);
int q3_loud_step_rows(q3_loudness* s, const float* in_dev, int64_t ld, const int32_t* counts_host,
                      const int32_t* end_host, float* out_dev, int32_t* nout_host, void* stream);
int q3_loud_save_rows(q3_loudness* s, int32_t n, const int32_t* rows_host, void* dst_dev, void* stream);
int q3_loud_load_rows(q3_loudness* s, int32_t n, const int32_t* rows_host, const void* src_dev, void* stream);

/* ---------------------------------------------------------------- speaker x-vector (voice cloning)
 * Replaces Qwen3TTSForConditionalGeneration.extract_speaker_embedding (core/models/modeling_qwen3_tts.py:1941-1954):
 * mel_spectrogram (:396-448) + Qwen3TTSSpeakerEncoder.forward (:371-393).  fp32. */
typedef struct {
  int32_t mel_dim, enc_dim;                 /* Qwen3TTSSpeakerEncoderConfig (configuration_qwen3_tts.py:47-57) */
  int32_t n_blocks;                         /* len(enc_channels) */
  int32_t channels[8], kernel_sizes[8], dilations[8];
  int32_t attention_channels, res2net_scale, se_channels;
  int32_t n_fft, hop, win;                  /* 1024, 256, 1024 at the reference call site (:1943-1951) */
  int32_t device;
} q3_spk_cfg;
typedef struct q3_spk q3_spk;

int q3_spk_create(const q3_spk_cfg* cfg, q3_spk** out);
void q3_spk_destroy(q3_spk* e);
/* fp32 device tensors: the reference's own `speaker_encoder.` state_dict names with the prefix stripped
 * ("blocks.0.conv.weight", "blocks.<i>.tdnn1.conv.weight", "blocks.<i>.res2net_block.blocks.<j>.conv.weight",
 * "blocks.<i>.se_block.conv1.weight", "mfa.conv.weight", "asp.tdnn.conv.weight", "asp.conv.weight", "fc.weight", and
 * the matching ".bias"), plus the host-computed front-end tables "mel.window" [n_fft] (Hann), "mel.cos" / "mel.sin"
 * [n_fft] = cos/sin(2*pi*j/n_fft), "mel.fbT" [n_fft/2+1][mel_dim] (librosa-style Slaney filterbank, transposed). */
int q3_spk_load_tensor(q3_spk* e, const char* name, const float* dev, const int64_t* shape, int32_t ndim);
int q3_spk_finalize(q3_spk* e);
int q3_spk_frames(q3_spk* e, int32_t T);    /* STFT frames of a T-sample waveform */
/* wav fp32 [B][T] -> log-mel fp32 [B][mel_dim][frames] */
int q3_spk_mel(q3_spk* e, const float* wav_dev, int32_t B, int32_t T, float* mel_dev, void* stream);
/* wav fp32 [B][T] (or, when mel_dev != NULL, a ready mel [B][mel_dim][frames]) -> emb fp32 [B][enc_dim] */
int q3_spk_embed(q3_spk* e, const float* wav_dev, int32_t B, int32_t T, const float* mel_dev, int32_t frames,
                 float* emb_dev, void* stream);
int q3_spk_last_launch_count(q3_spk* e);

#ifdef __cplusplus
}
#endif
#endif /* QWEN3TTS_B200_H */
