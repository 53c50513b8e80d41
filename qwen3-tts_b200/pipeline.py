"""End-to-end hot path on one GPU: prefill -> fused frame-step decode -> codec decode.

`TTSEngine.synthesize` is the call a user of seam B + seam C makes: prefill embeddings in (host or device),
waveforms out (host numpy, like Qwen3TTSTokenizer.decode -> `.to(float32).cpu().numpy()`,
inference/qwen3_tts_tokenizer.py:364)."""
from typing import List, Sequence

import numpy as np
import torch

from .codec import CodecDecoder, check_ref_codes
from .config import CodecConfig, SamplingParams, TTSConfig
from .engine import AREngine
from .scheduler import ContinuousBatcher


class TTSEngine:
    def __init__(self, cfg: TTSConfig, weights, codec_cfg: CodecConfig, codec_weights, device="cuda:0", max_batch=32,
                 max_ctx=4096, codec_max_frames=1024):
        self.device = torch.device(device)
        self.ar = AREngine(cfg, weights, device=device, max_batch=max_batch, max_ctx=max_ctx)
        self.codec = CodecDecoder(codec_cfg, codec_weights, device=device, max_frames=codec_max_frames, max_batch=max_batch)
        self.cfg, self.codec_cfg = cfg, codec_cfg
        self.timing = {}

    @torch.no_grad()
    def generate_codes(self, inputs_embeds, trailing_text, tts_pad_embed, sp: SamplingParams) -> List[torch.Tensor]:
        return self.ar.generate(inputs_embeds, trailing_text, tts_pad_embed, sp)

    @torch.no_grad()
    def decode_codes(self, codes: Sequence[torch.Tensor]) -> List[torch.Tensor]:
        """List[(T_i,K)] -> List[(T_i*1920,)] fp32 on device; == Qwen3TTSTokenizer.decode's padding with -1 +
        Qwen3TTSTokenizerV2Model.decode (inference/qwen3_tts_tokenizer.py:329, …v2.py:993-1024)."""
        B = len(codes)
        Tm = max(max(int(c.shape[0]) for c in codes), 1)
        K = self.codec_cfg.num_quantizers
        ac = torch.full((B, Tm, K), -1, dtype=torch.int64, device=self.device)
        for i, c in enumerate(codes):
            ac[i, :c.shape[0]] = c.to(self.device)
        return self.codec.decode(ac)

    @torch.no_grad()
    def synthesize(self, inputs_embeds, trailing_text, tts_pad_embed, sp: SamplingParams, to_host=True):
        """inputs_embeds / trailing_text / tts_pad_embed may live in (pinned) host memory: they are copied to the
        device here, and the waveforms are copied back — both inside the caller's timed region."""
        dev = self.device
        emb = [e.to(dev, non_blocking=True) for e in inputs_embeds]
        tr = [t.to(dev, non_blocking=True) for t in trailing_text]
        pad = tts_pad_embed.to(dev, non_blocking=True)
        codes = self.ar.generate(emb, tr, pad, sp)
        wavs = self.decode_codes(codes)
        if not to_host:
            return wavs, codes
        out = [w.to(torch.float32).cpu().numpy() for w in wavs]
        return out, codes

    @torch.no_grad()
    def stream_synthesize(self, inputs_embeds, trailing_text, tts_pad_embed, sp: SamplingParams, packet_frames: int = 4,
                          left_context="stateful", ref_codes=None):
        """Streaming OUTPUT (new surface: the reference returns audio whole, SURVEY F1).  Yields, per packet of
        `packet_frames` frames (4 frames = 320 ms, Qwen3-TTS report §3.4), a list with one fp32 numpy waveform chunk per
        row (empty for a row without new frames).  The rows run as one ContinuousBatcher session.  Default: the
        STATEFUL codec stream (q3_codec_stream_*) — each packet costs its own frames only and the concatenated chunks
        equal the one-shot causal decode.  `left_context=25` decodes every packet together with 25
        already-emitted frames, exactly like the reference's chunked_decode does between chunks (…v2.py:886-896);
        `left_context=None` re-decodes the whole prefix.
        `ref_codes`: one entry per row, the (L, K) reference codes of a voice-clone row (VoiceClonePromptItem.ref_code)
        or None.  A row's audio is then decoded as cat(ref_codes, generated codes) is (qwen3_tts_model.py:612-631):
        the stateful stream seeds the row with its reference (and caps its horizon at the codec's max_frames minus the
        reference's length), the windowed modes start its history with it.  The chunks hold the generated audio only."""
        dev = self.device
        emb = [e.to(dev, non_blocking=True) for e in inputs_embeds]
        tr = [t.to(dev, non_blocking=True) for t in trailing_text]
        pad = tts_pad_embed.to(dev, non_blocking=True)
        K = self.codec_cfg.num_quantizers
        up = self.codec.total_upsample
        B = len(emb)
        refs = [None] * B
        if ref_codes is not None:
            if len(ref_codes) != B:
                raise ValueError(f"ref_codes has {len(ref_codes)} entries for {B} rows")
            for b, r in enumerate(ref_codes):
                if r is not None:
                    check_ref_codes(self.codec_cfg, r, self.codec.max_frames, f"row {b}: ref_codes")
                    refs[b] = r.to(dev, torch.int64)
        budget = self.ar._frame_budget(emb, sp)
        stateful = left_context == "stateful"
        cs = None
        if stateful:
            key = (B, int(packet_frames))
            if getattr(self, "_cstream_key", None) != key:
                if getattr(self, "_cstream", None) is not None:
                    self._cstream.close()
                self._cstream = self.codec.open_stream(B, max_packet_frames=int(packet_frames))
                self._cstream_key = key
            cs = self._cstream
        # the static batch is a session of B slots whose rows are all admitted in the first step, row b with Philox key b
        H = self.ar.cfg.talker.hidden_size
        cb = ContinuousBatcher(self.ar, pad, sp, n_slots=B, packet_frames=packet_frames,
                               max_trailing=max(int(t.reshape(-1, H).shape[0]) for t in tr), codec=cs)
        for b in range(B):
            cb.submit(emb[b], tr[b], key=b, max_frames=budget, ref_codes=refs[b] if stateful else None)
        if budget == 0:
            return
        if stateful:
            for chunks, _ in cb.stream():
                yield [chunks.get(b, np.zeros(0, dtype=np.float32)) for b in range(B)]
            return
        hist = [torch.zeros(0, K, dtype=torch.int64, device=dev) if r is None else r for r in refs]
        for new, _ in cb.packets():
            out = [np.zeros(0, dtype=np.float32) for _ in range(B)]
            # rows whose window has the same shape (the normal case: every live row got `packet_frames` new frames on top
            # of the same history) go through ONE batched codec call — rows are independent in the decoder, so this is
            # bit-identical to decoding them one by one, at 1/B of the launches
            groups = {}
            for b, codes in new.items():
                ctx = hist[b].shape[0] if left_context is None else min(left_context, hist[b].shape[0])
                groups.setdefault((ctx, int(codes.shape[0])), []).append(b)
            for (ctx, n_new), rows in groups.items():
                windows = torch.stack([torch.cat([hist[b][hist[b].shape[0] - ctx:], new[b]], 0) for b in rows], 0)  # (n, T, K)
                wav = self.codec.forward(windows.transpose(1, 2).contiguous())[:, 0, ctx * up:]
                wav = wav.to(torch.float32).cpu().numpy()
                for i, b in enumerate(rows):
                    out[b] = wav[i]
            for b, codes in new.items():
                hist[b] = torch.cat([hist[b], codes], 0)
            yield out

    def close(self):
        self.ar.close()
        self.codec.close()
