"""Reference arm of bench.py: the reference's OWN modules timed on the host cores.

`Qwen3TTSTalkerForConditionalGeneration` (talker + code predictor, core/models/modeling_qwen3_tts.py) and
`Qwen3TTSTokenizerV2Decoder` (tokenizer_12hz/modeling_qwen3_tts_tokenizer_v2.py) are imported from the unmodified
package installed in baseline/_ref (baseline/install_reference.sh) through the three probe-only shims of
oracle/ref_shims.py, loaded with the SAME seeded synthetic weights as the GPU arm, and driven by the restated
generation loop (:1665-1744, :1250-1312 — the reference's HF `generate()` cannot execute under the installed
transformers 5.5.0, SURVEY §8c): prefill, then per frame 15 code-predictor forwards + sampling + one talker step,
then `chunked_decode` of the generated frames.  fp32, eager attention, all usable host threads.

When baseline/_ref is absent the same loop runs on the oracle port (oracle/talker.py, oracle/codec.py) and the
result says `kind: "port"`.  This module is bench infrastructure: the product never imports it.
"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_ROOT = os.path.join(ROOT, "baseline", "_ref")


def reference_installed() -> bool:
    return os.path.isdir(os.path.join(REF_ROOT, "qwen_tts"))


class _no_random_init:
    """Skip torch's default random initialisation while the reference modules are constructed (2 G parameters of
    kaiming/normal draws that load_state_dict overwrites anyway).  Touches torch.nn only, not the reference."""

    def __enter__(self):
        self.saved = []
        for cls in (torch.nn.Linear, torch.nn.Embedding, torch.nn.Conv1d, torch.nn.ConvTranspose1d):
            self.saved.append((cls, cls.reset_parameters))
            cls.reset_parameters = lambda self_: None
        self.init = {n: getattr(torch.nn.init, n) for n in ("normal_", "trunc_normal_", "kaiming_uniform_", "uniform_", "xavier_uniform_")}
        for n in self.init:
            setattr(torch.nn.init, n, lambda t, *a, **k: t)
        return self

    def __exit__(self, *exc):
        for cls, fn in self.saved:
            cls.reset_parameters = fn
        for n, fn in self.init.items():
            setattr(torch.nn.init, n, fn)
        return False


class ReferenceArm:
    def __init__(self, ocfg, occfg, W_f32, CW_f32, threads):
        torch.set_num_threads(threads)
        self.ocfg, self.occfg, self.W, self.CW = ocfg, occfg, W_f32, CW_f32
        self.kind = "port"
        self.talker = self.decoder = None
        if reference_installed():
            try:
                os.environ["QWEN3TTS_REFERENCE_ROOT"] = REF_ROOT
                from oracle import ref_shims, ref_driver as R
                ref_shims.REFERENCE_ROOT = REF_ROOT
                with _no_random_init():  # every parameter is overwritten by the seeded synthetic weights below
                    self.talker = R.build_reference_talker(ocfg)
                    self.decoder = R.build_reference_codec_decoder(occfg)
                R.load_weights_into_reference(self.talker, W_f32)
                self.decoder.load_state_dict(CW_f32, strict=False)
                self.kind = "reference"
            except Exception as e:  # an import problem must not take the bench line down
                print(f"[bench] reference modules unavailable ({e!r}); using the oracle port", file=sys.stderr)
                self.talker = self.decoder = None

    # ------------------------------------------------------------------ bounded samples of the workload
    @torch.no_grad()
    def start(self, embs, trail, pad, sp_kwargs, seed=1234, horizon=4096):
        """Prefill of the batch + codebook-0 of frame 0.  Returns the seconds it took; keeps the generation state
        (KV cache, past_hidden, sampled history) so that step_frames() continues the same utterances."""
        from oracle import talker as OT
        self.sp = OT.SamplingCfg(max_new_tokens=horizon, suppress_eos=True, **sp_kwargs)
        self.embs, self.trail, self.pad, self.seed = embs, trail, pad, seed
        self.B = len(embs)
        self.frame = 0
        if self.kind == "port":
            sp0 = OT.SamplingCfg(max_new_tokens=1, suppress_eos=True, **sp_kwargs)
            t0 = time.perf_counter()
            OT.generate(self.W, self.ocfg, [e.float() for e in embs], [t.float() for t in trail], pad.float(), sp0)
            self.t_prefill = time.perf_counter() - t0
            self.sp_kwargs = sp_kwargs
            return self.t_prefill
        from transformers.cache_utils import DynamicCache
        m, cfg = self.talker, self.ocfg
        B, H = self.B, cfg.talker.hidden_size
        self.lp = OT.talker_logits_processors(cfg, self.sp)
        lens = [int(e.shape[0]) for e in embs]
        self.Lmax = max(lens)
        t0 = time.perf_counter()
        x = torch.zeros(B, self.Lmax, H)
        mask = torch.zeros(B, self.Lmax, dtype=torch.long)
        for i, e in enumerate(embs):  # left padding (:2239-2254)
            x[i, self.Lmax - lens[i]:] = e.float()
            mask[i, self.Lmax - lens[i]:] = 1
        self.cache = DynamicCache()
        m.rope_deltas = None
        out = m(inputs_embeds=x, attention_mask=mask, past_key_values=self.cache, use_cache=True,
                cache_position=torch.arange(self.Lmax))
        self.mask = mask
        self.past_hidden = out.past_hidden
        self.gen = [[] for _ in range(B)]
        self.c0 = self._pick_talker(out.logits[:, -1].float().numpy(), 0)
        self.t_prefill = time.perf_counter() - t0
        return self.t_prefill

    def _pick_talker(self, logits, frame):
        from oracle import sampler as OS, philox
        toks = []
        for b in range(self.B):
            s = OS.process_logits(logits[b], generated_ids=self.gen[b], **self.lp)
            s[self.ocfg.codec_eos_token_id] = -np.inf  # fixed horizon (suppress_eos), like the GPU arm
            tok, _ = OS.sample_from_scores(s, do_sample=self.sp.do_sample, u=philox.uniform(self.seed, b, frame, 0))
            self.gen[b].append(int(tok))
            toks.append(tok)
        return torch.tensor(toks)

    def _pick_cp(self, logits, frame, group):
        from oracle import sampler as OS, philox
        sp = self.sp
        toks = []
        for b in range(self.B):
            s = OS.process_logits(logits[b], do_sample=sp.subtalker_dosample, temperature=sp.subtalker_temperature,
                                  top_k=sp.subtalker_top_k, top_p=sp.subtalker_top_p)
            tok, _ = OS.sample_from_scores(s, do_sample=sp.subtalker_dosample, u=philox.uniform(self.seed, b, frame, group))
            toks.append(tok)
        return torch.tensor(toks)

    @torch.no_grad()
    def step_frames(self, n_frames):
        """n_frames more frame-steps of the running utterances (15 code-predictor forwards + sampling + one talker
        step each) and `chunked_decode` of exactly those frames.  Returns ({frames: [s...], codec: s}, codes)."""
        if self.kind == "port":
            return self._port_frames(n_frames)
        m, cfg = self.talker, self.ocfg
        B, H, G = self.B, cfg.talker.hidden_size, cfg.num_code_groups
        padv = self.pad.float().view(1, 1, H)
        codes = torch.zeros(B, n_frames, G, dtype=torch.long)
        from transformers.cache_utils import DynamicCache
        t_frames = []
        for k in range(n_frames):
            step = self.frame
            t0 = time.perf_counter()
            c0 = self.c0
            codes[:, k, 0] = c0
            cpc = DynamicCache()  # code predictor: 15 forwards on a fresh cache (:1250-1312)
            e0 = m.get_input_embeddings()(c0[:, None])
            o = m.code_predictor(inputs_embeds=torch.cat((self.past_hidden, e0), dim=1), past_key_values=cpc, use_cache=True)
            gs = o.generation_steps
            for j in range(1, G):
                cj = self._pick_cp(o.logits[:, -1].float().numpy(), step, j)
                codes[:, k, j] = cj
                if j < G - 1:
                    o = m.code_predictor(input_ids=cj[:, None], past_key_values=cpc, use_cache=True, generation_steps=gs)
                    gs = o.generation_steps
            # talker decode step (:1682-1727)
            hid = [e0] + [m.code_predictor.get_input_embeddings()[i](codes[:, k, i + 1:i + 2]) for i in range(G - 1)]
            xe = torch.cat(hid, dim=1).sum(1, keepdim=True)
            tr = torch.stack([t[step].float() if step < t.shape[0] else self.pad.float() for t in self.trail])[:, None] \
                if any(step < t.shape[0] for t in self.trail) else padv
            xe = xe + tr
            self.mask = torch.cat((self.mask, torch.ones(B, 1, dtype=torch.long)), dim=1)
            cp = torch.tensor([self.Lmax + step])
            pos = (cp[0] + m.rope_deltas).view(1, B, 1).expand(3, -1, -1)
            mo = m.model(inputs_embeds=xe, attention_mask=self.mask, position_ids=pos, past_key_values=self.cache,
                         use_cache=True, cache_position=cp)
            logits = m.codec_head(mo.last_hidden_state)[:, -1].float().numpy()
            self.past_hidden = mo.last_hidden_state[:, -1:]
            self.frame += 1
            self.c0 = self._pick_talker(logits, self.frame)
            t_frames.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        wav = self.decoder.chunked_decode(codes.transpose(1, 2).contiguous())
        t_codec = time.perf_counter() - t0
        assert tuple(wav.shape) == (B, 1, n_frames * self.occfg.total_upsample) and bool(torch.isfinite(wav).all())
        return {"prefill": self.t_prefill, "frames": t_frames, "codec": t_codec}, codes

    @torch.no_grad()
    def _port_frames(self, n_frames):
        """Oracle-port fallback: its generate() is not resumable, so a sample re-runs prefill + n_frames and the
        prefill time measured by start() is subtracted."""
        from oracle import talker as OT, codec as OC
        spn = OT.SamplingCfg(max_new_tokens=n_frames + 1, suppress_eos=True, **self.sp_kwargs)
        t0 = time.perf_counter()
        r = OT.generate(self.W, self.ocfg, [e.float() for e in self.embs], [t.float() for t in self.trail], self.pad.float(), spn)
        per = max(time.perf_counter() - t0 - self.t_prefill, 1e-9) / n_frames
        codes = torch.stack(r.codes)
        t0 = time.perf_counter()
        OC.decoder_forward(self.CW, self.occfg, codes.transpose(1, 2).contiguous())
        t_codec = time.perf_counter() - t0
        return {"prefill": self.t_prefill, "frames": [per] * n_frames, "codec": t_codec}, codes


def workload_rate(timing, batch, full_frames):
    """frames/s of the full workload (prefill + full_frames frame-steps + codec decode of them) from one sample:
    the measured prefill, the MEDIAN measured frame-step and the measured codec time per frame."""
    n = len(timing["frames"])
    per_frame = float(np.median(timing["frames"])) + timing["codec"] / n
    total = timing["prefill"] + full_frames * per_frame
    return batch * full_frames / total, {"prefill_s": timing["prefill"], "per_frame_step_s_median": float(np.median(timing["frames"])),
                                         "per_frame_step_s_min": float(np.min(timing["frames"])),
                                         "per_frame_step_s_max": float(np.max(timing["frames"])),
                                         "codec_s_per_frame": timing["codec"] / n, "frames_sampled": n,
                                         "full_workload_s": total}
