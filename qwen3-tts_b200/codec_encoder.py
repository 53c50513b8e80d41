"""Host side of the codec ENCODER (Qwen3TTSTokenizerV2Model.encode, core/tokenizer_12hz/
modeling_qwen3_tts_tokenizer_v2.py:961-991 -> transformers MimiModel._encode_frame) on libqwen3tts_b200.so.

`weights` is a flat dict keyed by MimiModel's own state_dict names (the encoder half: `encoder.*`,
`encoder_transformer.*`, `downsample.*`, `quantizer.*`), any float dtype; everything is converted to fp32 — the
encoder's output is discrete, see csrc/codec_encoder.cu.  Engine-native tensors built here:

  enc.conv0 / enc.res<i>.a|.b / enc.down<i> / enc.conv_last   .w [Cout][Cin][k], .b [Cout]
  tr.<l>.qkv.w = cat(q_proj, k_proj, v_proj) [3C][C];  .o.w, .fc1.w, .fc2.w, .ln1/.ln2 .w/.b, .ls1/.ls2
  rope.cos / rope.sin [max_frames][head_dim/2]   fp32 tables, computed exactly as MimiRotaryEmbedding does
  down.w [C][C][2*stride];  rvq.sem|ac.proj.w [D][C]
  rvq.<q>.e = embed_sum / clamp(cluster_usage, 1e-5) [K][D], .et = its transpose, .e2 = squared norms
"""
import ctypes as C
from typing import Dict, List, Tuple

import numpy as np
import torch

from . import _lib
from .config import EncoderConfig


class CodecEncoder:
    def __init__(self, cfg: EncoderConfig, weights: Dict[str, torch.Tensor], device="cuda:0", max_frames=None):
        self.lib = _lib.load()
        self.cfg = cfg
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("CodecEncoder needs a CUDA device (no CPU fallback)")
        self.max_frames = int(max_frames or cfg.max_position_embeddings)
        cc = _lib.CodecEncCfg()
        for n in ("num_filters", "kernel_size", "last_kernel_size", "residual_kernel_size", "compress", "hidden_size",
                  "num_layers", "num_heads", "head_dim", "intermediate_size", "sliding_window", "codebook_size",
                  "codebook_dim", "num_semantic_quantizers", "downsample_stride"):
            setattr(cc, n, int(getattr(cfg, n)))
        cc.n_ratios = len(cfg.ratios)
        for i, r in enumerate(cfg.ratios):
            cc.ratios[i] = int(r)
        cc.norm_eps = float(cfg.norm_eps)
        cc.num_quantizers = int(cfg.valid_num_quantizers)
        cc.max_frames, cc.device = self.max_frames, self.device.index or 0
        h = C.c_void_p()
        _lib.check(self.lib.q3_codec_enc_create(C.byref(cc), C.byref(h)))
        self.h = h
        self._load(weights)
        _lib.check(self.lib.q3_codec_enc_finalize(self.h))
        self.hop = self.lib.q3_codec_enc_hop(self.h)
        # stage ordinals of q3_codec_enc_debug_capture (tests)
        self.stage_names = ["conv0"] + [n for i in range(len(cfg.ratios)) for n in (f"res{i}", f"down{i}")] + \
                           ["conv_last"] + [f"tr{l}" for l in range(cfg.num_layers)] + ["downsample"]

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.q3_codec_enc_destroy(self.h)
                self.h = None
        except Exception:
            pass

    # ------------------------------------------------------------------ weight conversion
    def _put(self, name, x):
        x = x.detach().to(self.device, torch.float32).contiguous()
        shape = (C.c_int64 * x.dim())(*x.shape)
        _lib.check(self.lib.q3_codec_enc_load_tensor(self.h, name.encode(), x.data_ptr(), shape, x.dim()))

    def _load(self, W):
        cfg = self.cfg

        def conv(dst, src, bias=True):
            self._put(dst + ".w", W[f"{src}.conv.weight"])
            if bias:
                self._put(dst + ".b", W[f"{src}.conv.bias"])

        # module indices of MimiEncoder.layers (modeling_mimi.py:457-485): conv, then per ratio [resblock, ELU, conv], ELU, conv
        idx = 0
        conv("enc.conv0", f"encoder.layers.{idx}")
        idx += 1
        for i in range(len(cfg.ratios)):
            conv(f"enc.res{i}.a", f"encoder.layers.{idx}.block.1")
            conv(f"enc.res{i}.b", f"encoder.layers.{idx}.block.3")
            idx += 2
            conv(f"enc.down{i}", f"encoder.layers.{idx}")
            idx += 1
        idx += 1
        conv("enc.conv_last", f"encoder.layers.{idx}")
        for l in range(cfg.num_layers):
            p = f"encoder_transformer.layers.{l}."
            qkv = torch.cat([W[p + f"self_attn.{n}_proj.weight"].float() for n in ("q", "k", "v")], 0)
            self._put(f"tr.{l}.qkv.w", qkv[:, :, None])
            self._put(f"tr.{l}.o.w", W[p + "self_attn.o_proj.weight"][:, :, None])
            self._put(f"tr.{l}.fc1.w", W[p + "mlp.fc1.weight"][:, :, None])
            self._put(f"tr.{l}.fc2.w", W[p + "mlp.fc2.weight"][:, :, None])
            self._put(f"tr.{l}.ln1.w", W[p + "input_layernorm.weight"])
            self._put(f"tr.{l}.ln1.b", W[p + "input_layernorm.bias"])
            self._put(f"tr.{l}.ln2.w", W[p + "post_attention_layernorm.weight"])
            self._put(f"tr.{l}.ln2.b", W[p + "post_attention_layernorm.bias"])
            self._put(f"tr.{l}.ls1", W[p + "self_attn_layer_scale.scale"])
            self._put(f"tr.{l}.ls2", W[p + "mlp_layer_scale.scale"])
        # MimiRotaryEmbedding (modeling_mimi.py:515-578): fp32 inv_freq x position, computed on the CPU like the reference
        inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, cfg.head_dim, 2, dtype=torch.int64).float() / cfg.head_dim))
        fr = torch.arange(self.max_frames).float()[:, None] * inv[None, :]
        self._put("rope.cos", fr.cos())
        self._put("rope.sin", fr.sin())
        self._put("down.w", W["downsample.conv.weight"])
        nsem = cfg.num_semantic_quantizers
        for which, tag in (("semantic", "sem"), ("acoustic", "ac")):
            self._put(f"rvq.{tag}.proj.w", W[f"quantizer.{which}_residual_vector_quantizer.input_proj.weight"])
        for q in range(cfg.valid_num_quantizers):
            which, qi = ("semantic", q) if q < nsem else ("acoustic", q - nsem)
            p = f"quantizer.{which}_residual_vector_quantizer.layers.{qi}.codebook."
            # MimiEuclideanCodebook.embed (:1192-1195), divided on the CPU in fp32 exactly like the reference
            E = W[p + "embed_sum"].float().cpu() / W[p + "cluster_usage"].float().cpu().clamp(min=1e-5)[:, None]
            self._put(f"rvq.{q}.e", E)
            self._put(f"rvq.{q}.et", E.t().contiguous())
            self._put(f"rvq.{q}.e2", (E * E).sum(1))

    # ------------------------------------------------------------------ forward
    def frames(self, n_samples: int) -> int:
        return self.lib.q3_codec_enc_frames(self.h, int(n_samples))

    def forward(self, wav: torch.Tensor) -> torch.Tensor:
        """wav: (B, T) float -> codes (B, valid_num_quantizers, ceil-chain(T)) int64, like MimiModel.encode(...)[:, :16]."""
        if wav.dim() != 2:
            raise ValueError(f"Expected wav with shape (B, T), got {tuple(wav.shape)}")
        wav = wav.to(self.device, torch.float32).contiguous()
        B, T = wav.shape
        n = self.frames(T)
        codes = torch.empty(B, self.cfg.valid_num_quantizers, n, dtype=torch.int32, device=self.device)
        st = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.q3_codec_enc_encode(self.h, wav.data_ptr(), B, T, codes.data_ptr(), C.c_void_p(st)))
        return codes.long()

    def encode(self, wavs: List[torch.Tensor]) -> List[torch.Tensor]:
        """Qwen3TTSTokenizerV2Model.encode (…v2.py:961-991) on a list of 1-D waveforms: right-pad to the longest,
        encode, trim row i to ceil(len_i / encode_downsample_rate) frames; returns [(T_i, n_q) int64]."""
        L = max(int(w.shape[0]) for w in wavs)
        x = torch.zeros(len(wavs), L, dtype=torch.float32, device=self.device)
        for i, w in enumerate(wavs):
            x[i, : w.shape[0]] = w.to(self.device, torch.float32)
        codes = self.forward(x)
        rate = self.cfg.encode_downsample_rate
        return [codes[i, :, : -(-int(w.shape[0]) // rate)].transpose(0, 1).contiguous() for i, w in enumerate(wavs)]

    def last_launches(self) -> int:
        return self.lib.q3_codec_enc_last_launch_count(self.h)

    def open_stream(self, batch: int, max_packet_frames: int = 8, sample_rate=None):
        """A streaming encoder of `batch` rows (see EncoderStream): codes come back as each 1920-sample frame completes,
        and a clip ended with end() has exactly the codes of forward() on that clip alone.  `sample_rate` (None: the
        encoder's 24 kHz) other than 24 kHz: pushes are resampled on the device first (audio.ResampledEncoderStream),
        and a clip's codes equal forward(Resampler.oneshot(clip))."""
        from . import audio
        if sample_rate is None or sample_rate == audio.CODEC_RATE:
            return EncoderStream(self, batch, max_packet_frames)
        return audio.ResampledEncoderStream(self, batch, max_packet_frames, sample_rate)

    def forward_with_stages(self, wav: torch.Tensor):
        """Test helper: one forward that also returns every stage activation (name -> (B, C, T) fp32)."""
        wav = wav.to(self.device, torch.float32).contiguous()
        B, T = wav.shape
        cfg = self.cfg
        shapes, t, c = [], T, cfg.num_filters
        shapes.append((c, t))
        for r in cfg.ratios:
            shapes.append((c, t))
            t = -(-t // r)
            c *= 2
            shapes.append((c, t))
        shapes.append((cfg.hidden_size, t))
        shapes += [(cfg.hidden_size, t)] * cfg.num_layers
        shapes.append((cfg.hidden_size, -(-t // cfg.downsample_stride)))
        bufs = [torch.zeros(B, cc, tt, dtype=torch.float32, device=self.device) for cc, tt in shapes]
        _lib.check(self.lib.q3_codec_enc_debug_capture(self.h, -1, None, 0))
        for i, b in enumerate(bufs):
            _lib.check(self.lib.q3_codec_enc_debug_capture(self.h, i, b.data_ptr(), b.numel()))
        codes = self.forward(wav)
        torch.cuda.current_stream(self.device).synchronize()
        _lib.check(self.lib.q3_codec_enc_debug_capture(self.h, -1, None, 0))
        return codes, dict(zip(self.stage_names, bufs))


# ---------------------------------------------------------------------------------------------- streaming encoder
def split_frames(buffered: int, new: int, hop: int) -> Tuple[int, int]:
    """`buffered` samples held back plus `new` ones -> (whole frames ready to encode, samples left over, < hop)."""
    total = int(buffered) + int(new)
    return total // hop, total % hop


def check_chunks(chunks: Dict, batch: int) -> Dict[int, torch.Tensor]:
    """Validate push() input before any native call: {row: 1-D finite samples} with rows in [0, batch).  Returns the
    chunks as fp32 CPU-or-device tensors (numpy arrays are converted)."""
    if not isinstance(chunks, dict):
        raise ValueError("push expects a dict {row: 1-D samples}")
    out = {}
    for row, x in chunks.items():
        if isinstance(row, bool) or not isinstance(row, (int, np.integer)) or not 0 <= int(row) < batch:
            raise ValueError(f"row {row!r} is not a row of this stream (0..{batch - 1})")
        t = torch.from_numpy(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else x
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"row {row}: samples must be a numpy array or a torch tensor, got {type(x).__name__}")
        if t.dim() != 1:
            raise ValueError(f"row {row}: expected 1-D samples, got shape {tuple(t.shape)}")
        if not (t.is_floating_point() or t.numel() == 0):
            raise ValueError(f"row {row}: expected floating-point samples, got {t.dtype}")
        t = t.to(torch.float32)
        if not bool(torch.isfinite(t).all()):
            raise ValueError(f"row {row}: samples are not all finite")
        out[int(row)] = t
    return out


def check_rows(rows, batch: int) -> List[int]:
    rows = [rows] if isinstance(rows, (int, np.integer)) else list(rows)
    for r in rows:
        if isinstance(r, bool) or not isinstance(r, (int, np.integer)) or not 0 <= int(r) < batch:
            raise ValueError(f"row {r!r} is not a row of this stream (0..{batch - 1})")
    if len(set(int(r) for r in rows)) != len(rows):
        raise ValueError(f"rows listed twice: {rows}")
    return [int(r) for r in rows]


class EncoderStream:
    """Stateful streaming encoder over `batch` rows (q3_codec_enc_stream_*).  push({row: samples}) takes chunks of any
    length at the encoder's input rate, holds back each row's partial frame, encodes every completed frame in packets of
    at most `max_packet_frames` and returns {row: LongTensor (n_i, nq)} for the frames this push completed.  end(rows)
    encodes each row's held-back partial frame exactly as the one-shot encoder pads a clip's end and returns its
    (0 or 1, nq) codes; the rows then start new clips.  The concatenation of a clip's pushes and its end equals
    CodecEncoder.forward of the whole clip alone, bit for bit."""

    def __init__(self, enc: CodecEncoder, batch: int, max_packet_frames: int = 8):
        self.enc, self.lib = enc, enc.lib
        self.batch, self.max_packet_frames = int(batch), int(max_packet_frames)
        self.hop, self.nq = enc.hop, enc.cfg.valid_num_quantizers
        self.device = enc.device
        h = C.c_void_p()
        _lib.check(self.lib.q3_codec_enc_stream_open(enc.h, self.batch, self.max_packet_frames, C.byref(h)))
        self.h = h
        self._pending = [torch.zeros(0, dtype=torch.float32, device=self.device) for _ in range(self.batch)]

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def close(self):
        if getattr(self, "h", None):
            self.lib.q3_codec_enc_stream_close(self.h)
            self.h = None

    def _stream(self):
        if not self.h:
            raise RuntimeError("encoder stream is closed")
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    @property
    def positions(self) -> List[int]:
        """12.5 Hz frames encoded per row since its reset (held-back samples not counted)."""
        return [self.lib.q3_codec_enc_stream_row_position(self.h, b) for b in range(self.batch)]

    def push(self, chunks: Dict) -> Dict[int, torch.Tensor]:
        chunks = check_chunks(chunks, self.batch)
        st = self._stream()
        todo, frames = {}, {}
        for b, x in chunks.items():
            n, _ = split_frames(self._pending[b].numel(), x.numel(), self.hop)
            todo[b] = torch.cat([self._pending[b], x.to(self.device)])
            frames[b] = n
        pos, ds = self.positions, self.enc.cfg.downsample_stride
        for b, n in frames.items():
            if (pos[b] + n) * ds > self.enc.max_frames:
                raise ValueError(f"row {b}: 25 Hz position {pos[b] * ds} + {n * ds} frames exceeds the encoder's "
                                 f"max_frames {self.enc.max_frames}")
        out = {b: [] for b in chunks}
        done = {b: 0 for b in chunks}
        while any(done[b] < frames[b] for b in chunks):
            n = min(self.max_packet_frames, max(frames[b] - done[b] for b in chunks))
            counts = (C.c_int32 * self.batch)()
            wav = torch.zeros(self.batch, n * self.hop, dtype=torch.float32, device=self.device)
            for b in chunks:
                k = min(n, frames[b] - done[b])
                counts[b] = k
                wav[b, : k * self.hop] = todo[b][done[b] * self.hop: (done[b] + k) * self.hop]
            codes = torch.empty(self.batch, self.nq, n, dtype=torch.int32, device=self.device)
            _lib.check(self.lib.q3_codec_enc_stream_step_rows(self.h, wav.data_ptr(), n, counts, codes.data_ptr(), st))
            for b in chunks:
                if counts[b]:
                    out[b].append(codes[b, :, : counts[b]].transpose(0, 1))
                done[b] += counts[b]
        for b in chunks:
            self._pending[b] = todo[b][frames[b] * self.hop:].clone()
        return {b: (torch.cat(v).long() if v else torch.zeros(0, self.nq, dtype=torch.long, device=self.device))
                for b, v in out.items()}

    def end(self, rows) -> Dict[int, torch.Tensor]:
        """Encode each row's held-back partial frame (the clip's last frame) and start new clips on these rows."""
        rows = check_rows(rows, self.batch)
        if not rows:
            return {}
        st = self._stream()
        n = len(rows)
        wav = torch.zeros(n, self.hop, dtype=torch.float32, device=self.device)
        tails = (C.c_int32 * n)()
        for i, b in enumerate(rows):
            tails[i] = self._pending[b].numel()
            wav[i, : tails[i]] = self._pending[b]
        codes = torch.empty(n, self.nq, dtype=torch.int32, device=self.device)
        _lib.check(self.lib.q3_codec_enc_stream_finish_rows(self.h, n, (C.c_int32 * n)(*rows), tails, wav.data_ptr(),
                                                            codes.data_ptr(), st))
        for b in rows:
            self._pending[b] = self._pending[b][:0]
        return {b: codes[i: i + 1].long() if tails[i] else codes[i: i].long() for i, b in enumerate(rows)}

    def reset(self, rows):
        """Drop the rows' clips (state and held-back samples); they start new clips at position 0."""
        rows = check_rows(rows, self.batch)
        if not rows:
            return
        _lib.check(self.lib.q3_codec_enc_stream_reset_rows(self.h, len(rows), (C.c_int32 * len(rows))(*rows), self._stream()))
        for b in rows:
            self._pending[b] = self._pending[b][:0]
