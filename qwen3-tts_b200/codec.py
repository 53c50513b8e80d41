"""Host side of the codec hot path (seam C): Qwen3TTSTokenizerV2Decoder.forward / chunked_decode /
Qwen3TTSTokenizerV2Model.decode (core/tokenizer_12hz/modeling_qwen3_tts_tokenizer_v2.py:869-896, :993-1024)
on libqwen3tts_b200.so.  The reference state_dict is re-laid-out here into the engine-native tensors:

  rvq.table  bf16 [K][bins][D]      embedding_sum / clamp(cluster_usage, 1e-5), precomputed once (SURVEY B.3)
  rvq.proj   bf16 [Cq][Kp(2D)]      [rvq_first.output_proj | rvq_rest.output_proj] side by side
  <conv>.w   bf16 [Cout][k*Kp]      Conv1d weight, tap-major (tap j multiplies x[t-(k-1-j)*dil])
  <convT>.w  bf16 [r*Cout][2*Kp]    ConvTranspose1d(k=2r, stride r): row m*Cout+co, tap 0 = w[:,co,m], tap 1 = w[:,co,m+r]
  *.b, snake_ea/ib, ls*, gamma, ln.*, dw.*  fp32
"""
import ctypes as C
import math
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib
from .config import CodecConfig


def _kpad(k):
    return (k + 63) // 64 * 64


SEED_PACKET_FRAMES = 32   # capacity of the private stream that decodes reference prefixes (CodecStream.seed)


def check_ref_codes(cfg: CodecConfig, codes, max_len: int, what: str = "reference codes") -> int:
    """Validate an utterance prefix in the layout of VoiceClonePromptItem.ref_code / encode().audio_codes: an integer
    (L, num_quantizers) tensor with 1 <= L <= max_len and every code in [0, codebook_size) (an out-of-range code would
    index past the codebook in the RVQ gather).  Raises ValueError; returns L."""
    K = int(cfg.num_quantizers)
    if not isinstance(codes, torch.Tensor) or codes.dim() != 2 or int(codes.shape[1]) != K:
        shape = tuple(codes.shape) if isinstance(codes, torch.Tensor) else type(codes).__name__
        raise ValueError(f"{what}: expected an (L, {K}) tensor, got {shape}")
    if codes.dtype.is_floating_point or codes.dtype.is_complex or codes.dtype == torch.bool:
        raise ValueError(f"{what}: expected integer codes, got {codes.dtype}")
    L = int(codes.shape[0])
    if not 1 <= L <= max_len:
        raise ValueError(f"{what}: {L} frames outside [1, {max_len}]")
    lo, hi = (int(v) for v in torch.aminmax(codes.to(torch.int64)))
    if lo < 0 or hi >= int(cfg.codebook_size):
        raise ValueError(f"{what}: codes must lie in [0, {cfg.codebook_size}), got values in [{lo}, {hi}]")
    return L


class CodecDecoder:
    def __init__(self, cfg: CodecConfig, weights, device="cuda:0", max_frames=1024, max_batch=32):
        self.lib = _lib.load()
        self.cfg = cfg
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("CodecDecoder needs a CUDA device (no CPU fallback)")
        self.max_frames = max_frames
        self.max_batch = int(max_batch)
        cc = _lib.CodecCfg()
        for n in ("codebook_size", "codebook_dim", "hidden_size", "latent_dim", "num_heads", "num_kv_heads", "head_dim",
                  "sliding_window", "intermediate_size", "num_layers", "num_quantizers", "decoder_dim"):
            setattr(cc, n, int(getattr(cfg, n)))
        cc.n_upsample_rates = len(cfg.upsample_rates)
        cc.n_upsampling_ratios = len(cfg.upsampling_ratios)
        for i, r in enumerate(cfg.upsample_rates):
            cc.upsample_rates[i] = int(r)
        for i, r in enumerate(cfg.upsampling_ratios):
            cc.upsampling_ratios[i] = int(r)
        cc.rms_eps, cc.rope_theta = float(cfg.rms_eps), float(cfg.rope_theta)
        cc.max_frames, cc.max_batch, cc.device = int(max_frames), int(max_batch), self.device.index or 0
        h = C.c_void_p()
        _lib.check(self.lib.q3_codec_create(C.byref(cc), C.byref(h)))
        self.h = h
        self._load(weights)
        _lib.check(self.lib.q3_codec_finalize(self.h))
        self.total_upsample = self.lib.q3_codec_total_upsample(self.h)
        assert self.total_upsample == cfg.total_upsample
        self._banks: List[Optional["CodecStream"]] = []   # bank_reference's streams and their rows in use
        self._bank_used: List[set] = []

    # ------------------------------------------------------------------ weight conversion
    def _put(self, name, x, bf16):
        x = x.detach().to(self.device, torch.bfloat16 if bf16 else torch.float32).contiguous()
        shape = (C.c_int64 * x.dim())(*x.shape)
        _lib.check(self.lib.q3_codec_load_tensor(self.h, name.encode(), x.data_ptr(), shape, x.dim()))

    def _w(self, name, x):
        self._put(name, x, True)

    def _f(self, name, x):
        self._put(name, x, False)

    @staticmethod
    def _conv_w(w):
        """Conv1d [Cout][Cin][k] -> [Cout][k*Kp]."""
        co, ci, k = w.shape
        kp = _kpad(ci)
        out = torch.zeros(co, k, kp, dtype=torch.float32, device=w.device)
        out[:, :, :ci] = w.permute(0, 2, 1)
        return out.reshape(co, k * kp)

    @staticmethod
    def _convT_w(w, stride):
        """ConvTranspose1d [Cin][Cout][k] (k == stride or k == 2*stride) -> [stride*Cout][taps*Kp]."""
        ci, co, k = w.shape
        taps = k // stride
        assert taps in (1, 2) and taps * stride == k
        kp = _kpad(ci)
        out = torch.zeros(stride, co, taps, kp, dtype=torch.float32, device=w.device)
        for tap in range(taps):
            # out[m, co, tap, ci] = w[ci, co, m + tap*stride]
            out[:, :, tap, :ci] = w[:, :, tap * stride:(tap + 1) * stride].permute(2, 1, 0)
        return out.reshape(stride * co, taps * kp)

    @staticmethod
    def _lin_w(w):
        n, k = w.shape
        kp = _kpad(k)
        out = torch.zeros(n, kp, dtype=torch.float32, device=w.device)
        out[:, :k] = w
        return out

    @staticmethod
    def _gate_up_pair(gate, up):
        """gate, up [I][K] -> [2I][K] with rows (gate_i, up_i) adjacent (ACT_SWIGLU_PAIR)."""
        return torch.stack([gate, up], 1).reshape(2 * gate.shape[0], gate.shape[1])

    def _snake(self, name, alpha, beta):
        self._f(name + "_ea", torch.exp(alpha.float()))
        self._f(name + "_ib", 1.0 / (torch.exp(beta.float()) + 1e-9))

    def _load(self, W):
        cfg = self.cfg
        g = lambda n: W[n].to(self.device, torch.float32)  # noqa: E731
        # mirror the reference's parameter dtype when it was loaded in bf16 (values are then already bf16)
        D = cfg.codebook_dim // 2
        tabs = []
        for pfx, n in (("quantizer.rvq_first", 1), ("quantizer.rvq_rest", cfg.num_quantizers - 1)):
            for i in range(n):
                es, cu = g(f"{pfx}.vq.layers.{i}._codebook.embedding_sum"), g(f"{pfx}.vq.layers.{i}._codebook.cluster_usage")
                tabs.append(es / cu.clamp(min=1e-5)[:, None])
        self._w("rvq.table", torch.stack(tabs, 0))
        proj = torch.cat([g("quantizer.rvq_first.output_proj.weight")[:, :, 0], g("quantizer.rvq_rest.output_proj.weight")[:, :, 0]], 1)
        self._w("rvq.proj", self._lin_w(proj))
        self._w("pre_conv.w", self._conv_w(g("pre_conv.conv.weight")))
        self._f("pre_conv.b", g("pre_conv.conv.bias"))
        p = "pre_transformer"
        self._w("tr.in.w", self._lin_w(g(f"{p}.input_proj.weight")))
        self._f("tr.in.b", g(f"{p}.input_proj.bias"))
        self._w("tr.out.w", self._lin_w(g(f"{p}.output_proj.weight")))
        self._f("tr.out.b", g(f"{p}.output_proj.bias"))
        self._w("tr.norm", g(f"{p}.norm.weight"))
        for i in range(cfg.num_layers):
            lp, q = f"{p}.layers.{i}", f"tr.{i}"
            qkv = torch.cat([g(f"{lp}.self_attn.q_proj.weight"), g(f"{lp}.self_attn.k_proj.weight"), g(f"{lp}.self_attn.v_proj.weight")], 0)
            self._w(f"{q}.qkv.w", self._lin_w(qkv))
            self._w(f"{q}.o.w", self._lin_w(g(f"{lp}.self_attn.o_proj.weight")))
            gu = self._gate_up_pair(g(f"{lp}.mlp.gate_proj.weight"), g(f"{lp}.mlp.up_proj.weight"))
            self._w(f"{q}.gate_up.w", self._lin_w(gu))
            self._w(f"{q}.down.w", self._lin_w(g(f"{lp}.mlp.down_proj.weight")))
            self._w(f"{q}.ln1", g(f"{lp}.input_layernorm.weight"))
            self._w(f"{q}.ln2", g(f"{lp}.post_attention_layernorm.weight"))
            self._f(f"{q}.ls1", g(f"{lp}.self_attn_layer_scale.scale"))
            self._f(f"{q}.ls2", g(f"{lp}.mlp_layer_scale.scale"))
        hd = cfg.head_dim
        inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.int64).to(torch.float32) / hd))
        fr = torch.arange(self.max_frames, dtype=torch.float32)[:, None] * inv[None]
        self._w("rope.cos", fr.cos())
        self._w("rope.sin", fr.sin())
        for i, f in enumerate(cfg.upsampling_ratios):
            q = f"up.{i}"
            self._w(f"{q}.ct.w", self._convT_w(g(f"upsample.{i}.0.conv.weight"), f))
            self._f(f"{q}.ct.b", g(f"upsample.{i}.0.conv.bias"))
            self._f(f"{q}.dw.w", g(f"upsample.{i}.1.dwconv.conv.weight")[:, 0, :])
            self._f(f"{q}.dw.b", g(f"upsample.{i}.1.dwconv.conv.bias"))
            self._f(f"{q}.ln_g", g(f"upsample.{i}.1.norm.weight"))
            self._f(f"{q}.ln_beta", g(f"upsample.{i}.1.norm.bias"))
            self._w(f"{q}.pw1.w", self._lin_w(g(f"upsample.{i}.1.pwconv1.weight")))
            self._f(f"{q}.pw1.b", g(f"upsample.{i}.1.pwconv1.bias"))
            self._w(f"{q}.pw2.w", self._lin_w(g(f"upsample.{i}.1.pwconv2.weight")))
            self._f(f"{q}.pw2.b", g(f"upsample.{i}.1.pwconv2.bias"))
            self._f(f"{q}.gamma", g(f"upsample.{i}.1.gamma"))
        self._w("dec.in.w", self._conv_w(g("decoder.0.conv.weight")))
        self._f("dec.in.b", g("decoder.0.conv.bias"))
        nb = len(cfg.upsample_rates)
        for bi, r in enumerate(cfg.upsample_rates):
            bp, q = f"decoder.{bi + 1}.block", f"dec.{bi}"
            self._snake(f"{q}.snake", g(f"{bp}.0.alpha"), g(f"{bp}.0.beta"))
            self._w(f"{q}.ct.w", self._convT_w(g(f"{bp}.1.conv.weight"), r))
            self._f(f"{q}.ct.b", g(f"{bp}.1.conv.bias"))
            for u in range(3):
                up, uq = f"{bp}.{u + 2}", f"{q}.{u}"
                self._snake(f"{uq}.s1", g(f"{up}.act1.alpha"), g(f"{up}.act1.beta"))
                self._w(f"{uq}.c1.w", self._conv_w(g(f"{up}.conv1.conv.weight")))
                self._f(f"{uq}.c1.b", g(f"{up}.conv1.conv.bias"))
                self._snake(f"{uq}.s2", g(f"{up}.act2.alpha"), g(f"{up}.act2.beta"))
                self._w(f"{uq}.c2.w", self._conv_w(g(f"{up}.conv2.conv.weight")))
                self._f(f"{uq}.c2.b", g(f"{up}.conv2.conv.bias"))
        self._snake("dec.out.snake", g(f"decoder.{nb + 1}.alpha"), g(f"decoder.{nb + 1}.beta"))
        self._f("dec.out.w", g(f"decoder.{nb + 2}.conv.weight")[0].t().contiguous())  # [7][C]
        self._f("dec.out.b", g(f"decoder.{nb + 2}.conv.bias"))

    def last_launches(self):
        return int(self.lib.q3_codec_last_launch_count(self.h))

    def close(self):
        for st in getattr(self, "_banks", []):
            if st is not None:
                st.close()
        self._banks = []
        if getattr(self, "h", None):
            self.lib.q3_codec_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ seam C
    @torch.no_grad()
    def forward(self, codes: torch.Tensor) -> torch.Tensor:
        """codes (B,K,T) integer -> wav (B,1,T*upsample) fp32, == Qwen3TTSTokenizerV2Decoder.forward."""
        if codes.shape[1] != self.cfg.num_quantizers:
            raise ValueError(f"Expected {self.cfg.num_quantizers} layer of codes, got {codes.shape[1]}")
        B, K, T = codes.shape
        c = codes.to(self.device, torch.int32).contiguous()
        wav = torch.empty(B, T * self.total_upsample, dtype=torch.float32, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.q3_codec_forward(self.h, c.data_ptr(), B, T, wav.data_ptr(), C.c_void_p(stream)))
        self._keep = c
        return wav[:, None, :]

    def stage_shapes(self, B: int, T: int):
        """(name, (B, T_stage, C_stage)) of the stages q3_codec_debug_capture can copy, in stage-ordinal order."""
        g = self.cfg
        out = [("pre_conv", (B, T, g.latent_dim)), ("pre_transformer", (B, T, g.latent_dim))]
        Tc = T
        for f in g.upsampling_ratios:
            Tc *= int(f)
        out.append(("upsample", (B, Tc, g.latent_dim)))
        C_ = g.decoder_dim
        out.append(("decoder0_act", (B, Tc, C_)))
        for i, r in enumerate(g.upsample_rates):
            Tc *= int(r)
            C_ //= 2
            out.append((f"block{i}", (B, Tc, C_)))
        return out

    @torch.no_grad()
    def forward_with_stages(self, codes: torch.Tensor):
        """Test hook: forward() plus the bf16 channels-last tensor of every capturable stage (dict name -> (B,T,C))."""
        B, K, T = codes.shape
        bufs = {}
        _lib.check(self.lib.q3_codec_debug_capture(self.h, -1, None, 0))
        for i, (name, shp) in enumerate(self.stage_shapes(B, T)):
            bufs[name] = torch.zeros(shp, dtype=torch.bfloat16, device=self.device)
            _lib.check(self.lib.q3_codec_debug_capture(self.h, i, bufs[name].data_ptr(), bufs[name].numel()))
        try:
            wav = self.forward(codes)
            torch.cuda.current_stream(self.device).synchronize()
        finally:
            _lib.check(self.lib.q3_codec_debug_capture(self.h, -1, None, 0))
        return wav, bufs

    def open_stream(self, batch: int, max_packet_frames: int = 8) -> "CodecStream":
        """Stateful streaming decoder over `batch` rows (q3_codec_stream_*): push packets, get exactly the waveform of
        the full causal forward over everything pushed, for the cost of the new frames only."""
        return CodecStream(self, batch, max_packet_frames)

    # ------------------------------------------------------------------ state bank (registered voices, parked requests)
    def bank_reference(self, codes: torch.Tensor) -> Tuple[int, int]:
        """Decode reference codes ((L, K), the layout of VoiceClonePromptItem.ref_code) once into a row of a bank
        stream of this decoder and return (bank, row).  A row copied from it (CodecStream.copy_from(bank_stream(bank),
        [row], [slot])) has exactly the state CodecStream.seed with these codes leaves.  A bank holds up to max_batch
        rows; it grows by opening a larger stream and copying its rows over, so (bank, row) stays valid until
        bank_release.  Bank streams take no packets: they are opened with packets of one frame."""
        check_ref_codes(self.cfg, codes, self.max_frames, "reference codes")
        bank, row = self._bank_row()
        st = self._banks[bank]
        try:
            st.seed([row], [codes])
        except Exception:
            self.bank_release(bank, row)
            raise
        st._seeder.close()      # registration is rare: the private seed stream is not kept
        st._seeder = None
        return bank, row

    def bank_copy(self, src: "CodecStream", src_row: int) -> Tuple[int, int]:
        """Copy row `src_row` of a stream of this decoder, its whole causal state and position, into a bank row and
        return (bank, row), as bank_reference does for a reference (a parked request's codec row).  Copying it back with
        CodecStream.copy_from(bank_stream(bank), [row], [slot]) restores exactly that state; bank_release frees it."""
        if not 0 <= int(src_row) < src.B:
            raise ValueError(f"source row {src_row} out of range [0, {src.B})")
        bank, row = self._bank_row()
        try:
            self._banks[bank].copy_from(src, [int(src_row)], [row])
        except Exception:
            self.bank_release(bank, row)
            raise
        return bank, row

    def _bank_row(self) -> Tuple[int, int]:
        """A free row of a bank stream, growing a bank or adding one when every row is in use; marked used."""
        bank = next((i for i, used in enumerate(self._bank_used) if len(used) < self.max_batch), None)
        if bank is None:
            self._banks.append(None)
            self._bank_used.append(set())
            bank = len(self._banks) - 1
        used, old = self._bank_used[bank], self._banks[bank]
        if old is None or len(used) == old.B:
            grown = CodecStream(self, min(max(2 * len(used), 1), self.max_batch), 1)
            if used:
                grown.copy_from(old, sorted(used), sorted(used))
            if old is not None:
                torch.cuda.current_stream(self.device).synchronize()   # the copy reads the old stream
                old.close()
            self._banks[bank] = grown
        row = min(set(range(self._banks[bank].B)) - used)
        used.add(row)
        return bank, row

    def bank_stream(self, bank: int) -> "CodecStream":
        return self._banks[bank]

    def bank_release(self, bank: int, row: int):
        """Free a row of bank_reference; the bank's stream stays open for later references."""
        self._bank_used[bank].discard(int(row))

    @torch.no_grad()
    def chunked_decode(self, codes, chunk_size=300, left_context_size=25):
        """…v2.py:886-896, replicated exactly (chunks with 25 frames of left context)."""
        wavs = []
        start = 0
        T = codes.shape[-1]
        while start < T:
            end = min(start + chunk_size, T)
            ctx = left_context_size if start - left_context_size > 0 else start
            wav = self.forward(codes[..., start - ctx:end])
            wavs.append(wav[..., ctx * self.total_upsample:])
            start = end
        return torch.cat(wavs, dim=-1)

    @torch.no_grad()
    def decode(self, audio_codes: torch.Tensor) -> List[torch.Tensor]:
        """Qwen3TTSTokenizerV2Model.decode (…v2.py:993-1024): (B,T,K) padded with -1 -> list of 1-D wavs."""
        lengths = (audio_codes[..., 0] > -1).sum(1) * self.total_upsample
        codes = torch.clamp(audio_codes, min=0)
        wav = self.chunked_decode(codes.transpose(1, 2)).squeeze(1)
        return [a[:int(l)] for a, l in zip(wav, lengths)]


class CodecStream:
    """Handle on a q3_codec_stream (conv tails, ConvTranspose overlap rows and 71 frames of rotated K/V per transformer
    layer live on the device).  `push(codes (B,K,n))` -> wav (B,1,n*upsample) of those n frames.  Every row has its
    own position: `push(codes, counts)` advances row b by counts[b] frames only, and `reset(rows)` restarts some rows."""

    def __init__(self, dec: CodecDecoder, batch: int, max_packet_frames: int = 8):
        self.dec, self.B, self.nmax = dec, int(batch), int(max_packet_frames)
        h = C.c_void_p()
        _lib.check(dec.lib.q3_codec_stream_open(dec.h, self.B, self.nmax, C.byref(h)))
        self.h = h
        self._seeder: Optional["CodecStream"] = None   # private stream of seed(), opened on first use

    @property
    def positions(self) -> List[int]:
        """Frames pushed to each row since its last reset."""
        return [int(self.dec.lib.q3_codec_stream_row_position(self.h, b)) for b in range(self.B)]

    @torch.no_grad()
    def push(self, codes: torch.Tensor, counts: Optional[Sequence[int]] = None) -> torch.Tensor:
        """codes (B,K,n) -> wav (B,1,n*upsample).  With `counts`, row b takes only its first counts[b] frames
        (0 <= counts[b] <= n; the codes past them are never read): its audio is wav[b, 0, :counts[b]*upsample] and
        the rest of its row is zeros.  Without, every row takes all n."""
        dec = self.dec
        if codes.dim() != 3 or codes.shape[0] != self.B or codes.shape[1] != dec.cfg.num_quantizers:
            raise ValueError(f"expected codes of shape ({self.B}, {dec.cfg.num_quantizers}, n), got {tuple(codes.shape)}")
        n = int(codes.shape[2])
        counts = [n] * self.B if counts is None else [int(k) for k in counts]
        if len(counts) != self.B:
            raise ValueError(f"expected {self.B} counts, got {len(counts)}")
        for b, k in enumerate(counts):
            if not 0 <= k <= n:
                raise ValueError(f"row {b}: count {k} outside [0, {n}]")
        out = []
        for s0 in range(0, n, self.nmax):  # longer pushes are cut into packets of the stream's capacity
            c = codes[:, :, s0:s0 + self.nmax].to(dec.device, torch.int32).contiguous()
            m = int(c.shape[2])
            wav = torch.empty(self.B, m * dec.total_upsample, dtype=torch.float32, device=dec.device)
            stream = C.c_void_p(torch.cuda.current_stream(dec.device).cuda_stream)
            # a row's frames fill the packets in order: this packet holds frames s0 .. s0+m of the push
            k = (C.c_int32 * self.B)(*[min(max(kb - s0, 0), m) for kb in counts])
            _lib.check(dec.lib.q3_codec_stream_step_rows(self.h, c.data_ptr(), m, k, wav.data_ptr(), stream))
            self._keep = c
            out.append(wav)
        return torch.cat(out, 1)[:, None, :] if out else torch.zeros(self.B, 1, 0, device=dec.device)

    def reset(self, rows: Optional[Sequence[int]] = None):
        """Start new utterances in `rows` (all rows when None); the other rows keep their state."""
        stream = C.c_void_p(torch.cuda.current_stream(self.dec.device).cuda_stream)
        rows = range(self.B) if rows is None else [int(r) for r in rows]
        _lib.check(self.dec.lib.q3_codec_stream_reset_rows(self.h, len(rows), (C.c_int32 * max(len(rows), 1))(*rows), stream))

    @torch.no_grad()
    def seed(self, rows: Sequence[int], codes: Sequence[torch.Tensor]):
        """Start utterances in `rows` that continue the prefixes `codes` ((L_i, K) integer tensors, the layout of
        VoiceClonePromptItem.ref_code): afterwards row rows[i] is at position L_i with exactly the state of reset +
        a push of those L_i frames, so its next push decodes as cat(codes[i], next codes) would, and the prefix's own
        audio is never produced here.  The prefixes are decoded together in a private stream of packets of
        SEED_PACKET_FRAMES frames, whose rows are then copied over (q3_codec_stream_copy_rows); the other rows of this
        stream are untouched.  Bad input raises ValueError before any device work."""
        dec = self.dec
        rows = [int(r) for r in rows]
        if len(rows) != len(codes):
            raise ValueError(f"{len(rows)} rows for {len(codes)} code prefixes")
        for r in rows:
            if not 0 <= r < self.B:
                raise ValueError(f"seed row {r} out of range [0, {self.B})")
        if len(set(rows)) != len(rows):
            raise ValueError(f"seed rows {rows} are not distinct")
        lens = [check_ref_codes(dec.cfg, c, dec.max_frames, f"row {r}: reference codes") for r, c in zip(rows, codes)]
        n = len(rows)
        if n == 0:
            return
        if self._seeder is None or self._seeder.B < n:
            if self._seeder is not None:
                self._seeder.close()
            self._seeder = CodecStream(dec, n, min(SEED_PACKET_FRAMES, dec.max_frames))
        sd = self._seeder
        pkt = torch.zeros(sd.B, dec.cfg.num_quantizers, max(lens), dtype=torch.int32, device=dec.device)
        for i, c in enumerate(codes):
            pkt[i, :, :lens[i]] = c.to(dec.device, torch.int32).T
        sd.reset()
        sd.push(pkt, lens + [0] * (sd.B - n))   # the prefixes' audio is discarded
        self.copy_from(sd, range(n), rows)

    def copy_from(self, src: "CodecStream", src_rows: Sequence[int], rows: Sequence[int]):
        """Row rows[i] of this stream becomes row src_rows[i] of `src`, a stream of the same decoder of any size
        (q3_codec_stream_copy_rows): its whole causal state and its position.  The other rows are untouched."""
        src_rows, rows = [int(r) for r in src_rows], [int(r) for r in rows]
        if len(src_rows) != len(rows):
            raise ValueError(f"{len(src_rows)} source rows for {len(rows)} rows")
        n = len(rows)
        stream = C.c_void_p(torch.cuda.current_stream(self.dec.device).cuda_stream)
        _lib.check(self.dec.lib.q3_codec_stream_copy_rows(self.h, src.h, n, (C.c_int32 * max(n, 1))(*src_rows),
                                                          (C.c_int32 * max(n, 1))(*rows), stream))

    def close(self):
        if getattr(self, "_seeder", None) is not None:
            self._seeder.close()
            self._seeder = None
        if getattr(self, "h", None):
            self.dec.lib.q3_codec_stream_close(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
