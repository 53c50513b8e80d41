"""Host side of the AR hot path: drives libqwen3tts_b200.so through its C ABI.

Mirrors seam B of the reference — `talker.generate(inputs_embeds, attention_mask, trailing_text_hidden,
tts_pad_embed, **talker_kwargs)` at core/models/modeling_qwen3_tts.py:2272-2278 and the stack/trim at
:2280-2290 — with per-request state inside the engine (never on a module, SURVEY F10).
PyTorch is used only for device memory and streams.
"""
import ctypes as C
from typing import Optional, Sequence

import torch

from . import _lib
from .config import SamplingParams, TTSConfig


def _rope_tables(n_pos, head_dim, theta, device):
    """fp32 tables cast to bf16, exactly like modeling_qwen3_tts.py:546-559 / :581-592."""
    inv = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.int64).to(torch.float32) / head_dim))
    freqs = torch.arange(n_pos, dtype=torch.float32)[:, None] * inv[None, :]
    return (freqs.cos().to(torch.bfloat16).to(device).contiguous(),
            freqs.sin().to(torch.bfloat16).to(device).contiguous())


class AREngine:
    """Talker + code predictor + sampler on one H100.  `weights` maps the reference's state_dict names
    (`talker.model.layers.0.self_attn.q_proj.weight`, …) to tensors."""

    def __init__(self, cfg: TTSConfig, weights, device="cuda:0", max_batch=32, max_ctx=4096):
        self.lib = _lib.load()
        self.cfg = cfg
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("AREngine needs a CUDA device (no CPU fallback)")
        self.max_batch, self.max_ctx = max_batch, max_ctx
        t, c = cfg.talker, cfg.cp
        ec = _lib.EngineCfg()
        for dst, s in ((ec.talker, t), (ec.cp, c)):
            dst.hidden_size, dst.num_layers, dst.num_heads, dst.num_kv_heads = s.hidden_size, s.num_layers, s.num_heads, s.num_kv_heads
            dst.head_dim, dst.intermediate_size, dst.vocab_size, dst.rms_eps = s.head_dim, s.intermediate_size, s.vocab_size, s.rms_eps
        ec.num_code_groups = cfg.num_code_groups
        self.has_proj = "talker.code_predictor.small_to_mtp_projection.weight" in weights
        assert self.has_proj == (t.hidden_size != c.hidden_size), "projection is Identity iff hidden sizes match"
        ec.has_cp_projection = int(self.has_proj)
        ec.codec_eos_token_id = cfg.codec_eos_token_id
        ec.max_batch, ec.max_ctx, ec.device = max_batch, max_ctx, self.device.index or 0
        h = C.c_void_p()
        _lib.check(self.lib.q3_engine_create(C.byref(ec), C.byref(h)))
        self.h = h
        self._load(weights)
        _lib.check(self.lib.q3_engine_finalize(self.h))
        self._dbg = None

    # ------------------------------------------------------------------ weights
    def _put(self, name, x):
        x = x.detach().to(device=self.device, dtype=torch.bfloat16).contiguous()
        if x.dim() == 1:
            x = x[None]
        _lib.check(self.lib.q3_engine_load_tensor(self.h, name.encode(), x.data_ptr(), x.shape[0], x.shape[1]))

    @staticmethod
    def _gate_up_blk8(gate, up):
        """gate, up [I][K] -> [2I][K] in blocks of 16 rows: gate rows 8i..8i+7, then up rows 8i..8i+7 (ACT_SWIGLU_BLK8)."""
        I, K = gate.shape
        return torch.stack([gate.view(I // 8, 8, K), up.view(I // 8, 8, K)], 1).reshape(2 * I, K)

    def _load(self, W):
        cfg = self.cfg

        def stack(src, dst, s):
            for i in range(s.num_layers):
                p, q = f"{src}.layers.{i}", f"{dst}.layers.{i}"
                g = lambda n: W[f"{p}.{n}.weight"].to(self.device, torch.bfloat16)  # noqa: E731
                self._put(f"{q}.qkv", torch.cat([g("self_attn.q_proj"), g("self_attn.k_proj"), g("self_attn.v_proj")], 0))
                self._put(f"{q}.o", g("self_attn.o_proj"))
                self._put(f"{q}.gate_up", self._gate_up_blk8(g("mlp.gate_proj"), g("mlp.up_proj")))
                self._put(f"{q}.down", g("mlp.down_proj"))
                self._put(f"{q}.ln1", g("input_layernorm"))
                self._put(f"{q}.ln2", g("post_attention_layernorm"))
                self._put(f"{q}.q_norm", g("self_attn.q_norm"))
                self._put(f"{q}.k_norm", g("self_attn.k_norm"))
            self._put(f"{dst}.norm", W[f"{src}.norm.weight"])

        stack("talker.model", "talker", cfg.talker)
        self._put("talker.codec_head", W["talker.codec_head.weight"])
        self._put("talker.codec_embedding", W["talker.model.codec_embedding.weight"])
        cos, sin = _rope_tables(self.max_ctx, cfg.talker.head_dim, cfg.talker.rope_theta, self.device)
        self._put("talker.rope_cos", cos)
        self._put("talker.rope_sin", sin)
        stack("talker.code_predictor.model", "cp", cfg.cp)
        cos, sin = _rope_tables(32, cfg.cp.head_dim, cfg.cp.rope_theta, self.device)
        self._put("cp.rope_cos", cos)
        self._put("cp.rope_sin", sin)
        G = cfg.num_code_groups
        for j in range(G - 1):
            self._put(f"cp.lm_head.{j}", W[f"talker.code_predictor.lm_head.{j}.weight"])
        emb = torch.cat([W[f"talker.code_predictor.model.codec_embedding.{j}.weight"].to(self.device, torch.bfloat16)
                         for j in range(G - 1)], 0)
        self._put("cp.codec_embedding", emb)
        if self.has_proj:
            self._put("cp.proj", W["talker.code_predictor.small_to_mtp_projection.weight"])
            self._put("cp.proj_bias", W["talker.code_predictor.small_to_mtp_projection.bias"])

    def close(self):
        if getattr(self, "h", None):
            self.lib.q3_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ low level
    @staticmethod
    def _sampling(sp: SamplingParams):
        s = _lib.Sampling()
        s.do_sample, s.top_k, s.top_p, s.temperature = int(sp.do_sample), int(sp.top_k or 0), float(sp.top_p), float(sp.temperature)
        s.repetition_penalty = float(sp.repetition_penalty)
        s.subtalker_dosample, s.subtalker_top_k = int(sp.subtalker_dosample), int(sp.subtalker_top_k or 0)
        s.subtalker_top_p, s.subtalker_temperature = float(sp.subtalker_top_p), float(sp.subtalker_temperature)
        s.min_new_tokens, s.suppress_eos, s.seed = int(sp.min_new_tokens), int(sp.suppress_eos), int(sp.seed)
        return s

    @staticmethod
    def check_sampling(sp: SamplingParams):
        """Raise ValueError with the library's message when `sp` is outside the ranges the engine accepts
        (q3_sampling_check: the rules q3_prefill / q3_session_begin / q3_admit_with_sampling apply).  Needs no GPU."""
        lib = _lib.load()
        s = AREngine._sampling(sp)
        if lib.q3_sampling_check(C.byref(s)) != 0:
            raise ValueError(lib.q3_last_error().decode())

    def _pack(self, inputs_embeds, trailing_text, stride=0):
        """The prompts packed back to back [sum(lens)][H] with their lengths, and the trailing texts as [n][stride][H]
        (stride at least the longest) with their lengths.  The engine reads row i's first tl[i] rows only."""
        H = self.cfg.talker.hidden_size
        n = len(inputs_embeds)
        emb = torch.cat([e.reshape(-1, H) for e in inputs_embeds], 0).to(self.device, torch.bfloat16).contiguous()
        lens = (C.c_int32 * n)(*[int(e.reshape(-1, H).shape[0]) for e in inputs_embeds])
        tl = [int(t.reshape(-1, H).shape[0]) for t in trailing_text]
        stride = max([int(stride)] + tl)
        tr = torch.zeros(n, stride, H, dtype=torch.bfloat16, device=self.device)  # stride 0: empty, no row is read
        for i, t in enumerate(trailing_text):
            tr[i, :tl[i]] = t.reshape(-1, H).to(self.device, torch.bfloat16)
        return emb, lens, tr, (C.c_int32 * n)(*tl), stride

    def prefill(self, inputs_embeds: Sequence[torch.Tensor], trailing_text: Sequence[torch.Tensor],
                tts_pad_embed: torch.Tensor, sp: SamplingParams, trailing_capacity: int = 0):
        """`trailing_capacity` > longest trailing text reserves room for append_trailing() (streaming text input)."""
        B = len(inputs_embeds)
        emb, lens, tr, tl, stride = self._pack(inputs_embeds, trailing_text, trailing_capacity)
        pad = tts_pad_embed.reshape(self.cfg.talker.hidden_size).to(self.device, torch.bfloat16).contiguous()
        s = self._sampling(sp)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.q3_prefill(self.h, B, emb.data_ptr(), lens, tr.data_ptr(), tl, stride,
                                       pad.data_ptr(), C.byref(s), C.c_void_p(stream)))
        self._B = B

    # ------------------------------------------------------------------ continuous batching (low level)
    def session_begin(self, n_slots: int, tts_pad_embed: torch.Tensor, sp: SamplingParams, max_trailing: int = 0):
        """Start a session of `n_slots` independent rows (all empty).  See include/qwen3tts_b200.h: q3_session_begin."""
        H = self.cfg.talker.hidden_size
        pad = tts_pad_embed.reshape(H).to(self.device, torch.bfloat16).contiguous()
        s = self._sampling(sp)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        self._B = n_slots
        self._session_sp = sp
        _lib.check(self.lib.q3_session_begin(self.h, int(n_slots), int(max_trailing), pad.data_ptr(), C.byref(s), C.c_void_p(stream)))

    def admit(self, slots: Sequence[int], keys: Sequence[int], inputs_embeds: Sequence[torch.Tensor],
              trailing_text: Sequence[torch.Tensor], sampling: Optional[Sequence[Optional[SamplingParams]]] = None,
              prefixes: Optional[Sequence[Optional[int]]] = None):
        """Prefill new requests into free slots of the running session (q3_admit_with_sampling).  `sampling`: None
        (every request samples with the session's parameters) or one entry per request, a SamplingParams or None for
        the session's; a bad entry fails the whole admission before anything changes.  Of each entry the fields of
        q3_sampling are used, max_new_tokens is the caller's horizon.  `prefixes`: None, or one entry per request, a
        prefix id of create_prefix or None; request r's prompt is then that prefix followed by inputs_embeds[r]
        (q3_admit_with_prefix), and it generates what the admission of the whole prompt generates."""
        n = len(slots)
        sps = None
        if sampling is not None:
            if len(sampling) != n:
                raise ValueError(f"sampling has {len(sampling)} entries for {n} requests")
            sps = (_lib.Sampling * n)(*[self._sampling(self._session_sp if s is None else s) for s in sampling])
        emb, lens, tr, tl, stride = self._pack(inputs_embeds, trailing_text)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        sl, ks = (C.c_int32 * n)(*[int(x) for x in slots]), (C.c_uint32 * n)(*[int(k) & 0xffffffff for k in keys])
        if prefixes is None:
            _lib.check(self.lib.q3_admit_with_sampling(self.h, n, sl, ks, sps, emb.data_ptr(), lens, tr.data_ptr(), tl, stride,
                                                       C.c_void_p(stream)))
            return
        if len(prefixes) != n:
            raise ValueError(f"prefixes has {len(prefixes)} entries for {n} requests")
        ids = (C.c_int32 * n)(*[-1 if p is None else int(p) for p in prefixes])
        _lib.check(self.lib.q3_admit_with_prefix(self.h, n, sl, ks, sps, ids, emb.data_ptr(), lens, tr.data_ptr(), tl, stride,
                                                 C.c_void_p(stream)))

    def create_prefix(self, embeds: torch.Tensor) -> int:
        """Register prompt rows (n, H) that requests' prompts begin with (q3_prefix_create): their talker K/V are
        computed once and kept on the device, and admit(..., prefixes=[id]) copies them into a request's slot instead of
        prefilling them again.  May be called while a session runs: no running row changes.  Returns the prefix id."""
        H = self.cfg.talker.hidden_size
        e = embeds.reshape(-1, H).to(self.device, torch.bfloat16).contiguous()
        out = C.c_int32()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.q3_prefix_create(self.h, e.data_ptr(), int(e.shape[0]), C.c_void_p(stream), C.byref(out)))
        return out.value

    def free_prefix(self, prefix_id: int):
        """Release a prefix of create_prefix (q3_prefix_free).  Rows admitted with it keep their copy of its K/V."""
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.q3_prefix_free(self.h, int(prefix_id), C.c_void_p(stream)))

    def prefix_length(self, prefix_id: int) -> int:
        """Rows of a live prefix, -1 when there is none of that id."""
        return int(self.lib.q3_prefix_length(self.h, int(prefix_id)))

    def append_trailing(self, slot: int, rows: torch.Tensor):
        """Streaming text input: more trailing_text_hidden rows (n, H) for a row that is already generating."""
        H = self.cfg.talker.hidden_size
        r = rows.reshape(-1, H).to(self.device, torch.bfloat16).contiguous()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.q3_append_trailing(self.h, int(slot), r.data_ptr(), int(r.shape[0]), C.c_void_p(stream)))

    def set_text_open(self, slot: int, open: bool):
        """Live text (q3_set_trailing_open): while `slot` is open its text may still grow, and a step whose text row
        has not arrived is held (the row waits) instead of reading tts_pad.  Closing returns the row to reading tts_pad
        past its text.  Every admission starts closed."""
        _lib.check(self.lib.q3_set_trailing_open(self.h, int(slot), int(bool(open))))

    def release_slots(self, slots: Sequence[int]):
        n = len(slots)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.q3_release_slots(self.h, n, (C.c_int32 * max(n, 1))(*[int(x) for x in slots]), C.c_void_p(stream)))

    def park(self, slot: int) -> int:
        """Move the running request of `slot` out of the session into a record on the device (q3_row_park): its talker
        K/V and every per-row state the frame-step reads.  The slot is free afterwards, as after release_slots.  The
        caller keeps the request's codes, which live in its own buffer.  Returns the record id for resume / discard."""
        out = C.c_int32()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.q3_row_park(self.h, int(slot), C.c_void_p(stream), C.byref(out)))
        return out.value

    def resume(self, record: int, slot: int):
        """Continue a parked request in the free slot `slot` of the same session (q3_row_resume): it generates exactly
        what it would have generated never parked.  The record is consumed."""
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.q3_row_resume(self.h, int(record), int(slot), C.c_void_p(stream)))

    def discard(self, record: int):
        """Free a parked request's record without resuming it (q3_row_discard)."""
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.q3_row_discard(self.h, int(record), C.c_void_p(stream)))

    def decode(self, max_frames: int, codes: torch.Tensor):
        """codes: int32 [B][stride][G] device tensor that accumulates frames across calls."""
        assert codes.dtype == torch.int32 and codes.is_cuda and codes.is_contiguous()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.q3_decode(self.h, int(max_frames), codes.data_ptr(), codes.shape[1], C.c_void_p(stream)))

    def progress(self):
        B = self._B
        fd = C.c_int32()
        nv = (C.c_int32 * _lib.MAXB)()
        fin = (C.c_int32 * _lib.MAXB)()
        _lib.check(self.lib.q3_get_progress(self.h, C.byref(fd), nv, fin))
        return fd.value, list(nv[:B]), list(fin[:B])

    def set_debug(self, forced: Optional[torch.Tensor] = None, n_frames=0, talker_logits=None, cp_logits=None):
        self._dbg = (forced, talker_logits, cp_logits)
        _lib.check(self.lib.q3_set_debug(self.h, forced.data_ptr() if forced is not None else None, int(n_frames),
                                         talker_logits.data_ptr() if talker_logits is not None else None,
                                         cp_logits.data_ptr() if cp_logits is not None else None))

    def profile_frame(self, max_frames, codes):
        """Per-phase device timestamps of the first frame of one decode launch (CTA 0).  Returns
        (kinds[n], t_phase_end[n], t_barrier_end[n]) in ns."""
        n = -self.lib.q3_describe_frame_program(self.h, None, 0)
        kinds = (C.c_int32 * n)()
        self.lib.q3_describe_frame_program(self.h, kinds, n)
        G = torch.cuda.get_device_properties(self.device).multi_processor_count
        buf = torch.zeros(n, G, 16, dtype=torch.int64, device=self.device)
        _lib.check(self.lib.q3_set_profile(self.h, buf.data_ptr()))
        self.decode(max_frames, codes)
        torch.cuda.current_stream(self.device).synchronize()
        _lib.check(self.lib.q3_set_profile(self.h, None))
        t = buf.cpu().numpy()
        self.last_profile_all = t  # [phase][cta][16]: 0 end, 1 barrier passed, 2..4 inner marks, 6 start, 7/8 warp-0 marks, 5/9/10 cycle counts
        return list(kinds), t[:, 0, 0], t[:, 0, 1], t[:, 0, 2:6]

    def algorithmic_bytes(self, B, S):
        a, s = C.c_double(), C.c_double()
        _lib.check(self.lib.q3_algorithmic_bytes(self.h, B, S, C.byref(a), C.byref(s)))
        return a.value, s.value

    # ------------------------------------------------------------------ seam B
    def _frame_budget(self, inputs_embeds, sp: SamplingParams) -> int:
        """Frames this request may generate: HF emits max_new_tokens-1 complete frames; the KV cache holds
        max_ctx positions per row, so the horizon is clamped to max_ctx - longest prompt (the reference runs to EOS
        under max_position_embeddings=32768; an engine built with a smaller max_ctx says so instead of failing
        after the prefill).  Checked BEFORE any device work."""
        H = self.cfg.talker.hidden_size
        longest = max(int(e.reshape(-1, H).shape[0]) for e in inputs_embeds)
        if longest >= self.max_ctx:
            raise ValueError(f"prompt of {longest} positions does not fit max_ctx={self.max_ctx}")
        want = max(int(sp.max_new_tokens) - 1, 0)
        room = self.max_ctx - longest
        if want > room:
            if not getattr(self, "_warned_clamp", False):
                import warnings
                warnings.warn(f"max_new_tokens={sp.max_new_tokens} exceeds the KV capacity (max_ctx={self.max_ctx}, longest "
                              f"prompt {longest}): generation is capped at {room} frames; build the engine with a larger "
                              f"max_ctx to lift the cap", RuntimeWarning, stacklevel=3)
                self._warned_clamp = True
            want = room
        return want

    @torch.no_grad()
    def generate(self, inputs_embeds, trailing_text, tts_pad_embed, sp: SamplingParams, return_hidden: bool = False):
        """Returns per-row LongTensor (N_i, G) trimmed at the first EOS (modeling_qwen3_tts.py:2283-2290).
        HF emits max_new_tokens-1 complete frames when no EOS is sampled.  With return_hidden also the per-step
        hidden states (N_i, H) of :2281/:2290 (the reference's second return value)."""
        B = len(inputs_embeds)
        G = self.cfg.num_code_groups
        H = self.cfg.talker.hidden_size
        max_frames = self._frame_budget(inputs_embeds, sp)
        hid = None
        if return_hidden:
            hid = torch.zeros(B, max(max_frames, 1) + 1, H, dtype=torch.bfloat16, device=self.device)
            _lib.check(self.lib.q3_set_hidden_capture(self.h, hid.data_ptr(), hid.shape[1]))
        try:
            self.prefill(inputs_embeds, trailing_text, tts_pad_embed, sp)
            codes = torch.zeros(B, max(max_frames, 1), G, dtype=torch.int32, device=self.device)
            if max_frames > 0:
                self.decode(max_frames, codes)
            torch.cuda.current_stream(self.device).synchronize()
        finally:
            if return_hidden:
                _lib.check(self.lib.q3_set_hidden_capture(self.h, None, 0))
        _, n_valid, _ = self.progress()
        out = [codes[b, :min(n_valid[b], max_frames)].to(torch.int64) for b in range(B)]
        if return_hidden:
            return out, [hid[b, :o.shape[0]].clone() for b, o in enumerate(out)]
        return out
