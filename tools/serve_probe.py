"""Serving probe: continuous batching with audio out (ContinuousBatcher(..., codec=...).stream()).

Full 1.7B talker and default codec shapes with seeded random weights, suppress_eos, 4-frame packets, horizons
staggered so that requests leave at different steps and new ones are admitted into running sessions.  For each
n_slots it reports the AR and codec milliseconds per step, the time from submit() to a request's first audio chunk,
and the aggregate audio seconds produced per wall second, with the card name and power limit read in the same run.
With --mix the requests carry their own sampling parameters: every fourth one top-p 0.8 (talker and subtalker, the
generic sampler path), every fourth one greedy, the rest the session's; comparing with a run without it gives what
such rows cost the whole session.

    python tools/serve_probe.py [--slots 8 32] [--requests-per-slot 3] [--packet 4] [--mix]

Prints one JSON line.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HORIZONS = (40, 64, 88, 112)   # frames; staggered so that slots free up at different steps
SAMPLE_RATE = 24000


def card():
    name, limit = torch.cuda.get_device_name(), None
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits",
                              f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30).stdout
        name, limit = [x.strip() for x in out.strip().split(",")][:2]
        limit = float(limit)
    except Exception as e:  # the figure is then reported as unknown, never guessed
        limit = f"not read ({e!r})"
    return {"name": name, "power_limit_w": limit}


def mixed_sampling(sp, i):
    """--mix: request i's own parameters (None = the session's)."""
    import dataclasses
    if i % 4 == 0:
        return dataclasses.replace(sp, top_p=0.8, subtalker_top_p=0.8, seed=sp.seed + i)
    if i % 4 == 1:
        return dataclasses.replace(sp, do_sample=False, subtalker_dosample=False)
    return None


def run_session(eng, codec, pad, sp, prompts, n_slots, packet, horizons, timed, mix=False):
    """One session: n_slots requests at once, then one more per step until all are in.  Returns the measurements."""
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cb = ContinuousBatcher(eng, pad, sp, n_slots=n_slots, packet_frames=packet, codec=codec)
    t_ar, t_codec = [], []

    def clocked(fn, acc):
        def call(*a, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn(*a, **k)
            torch.cuda.synchronize()
            acc.append(time.perf_counter() - t0)
            return r
        return call

    if timed:
        eng.decode = clocked(type(eng).decode.__get__(eng), t_ar)
        cb.cstream.push = clocked(cb.cstream.push, t_codec)
    submitted, first, samples = {}, {}, 0
    todo = list(range(len(prompts)))

    def submit(i):
        rid = cb.submit(prompts[i], None, key=i, max_frames=horizons[i % len(horizons)],
                        sampling=mixed_sampling(sp, i) if mix else None)
        submitted[rid] = time.perf_counter()

    for i in todo[:n_slots]:
        submit(i)
    todo = todo[n_slots:]
    t0 = time.perf_counter()
    try:
        for chunks, _ in cb.stream():
            now = time.perf_counter()
            for rid, a in chunks.items():
                first.setdefault(rid, now - submitted[rid])
                samples += a.shape[0]
            if todo:
                submit(todo.pop(0))
    finally:
        if timed:
            del eng.decode
        cb.cstream.close()
    wall = time.perf_counter() - t0
    ms = lambda v: {"median": float(np.median(v)) * 1e3, "p90": float(np.percentile(v, 90)) * 1e3}  # noqa: E731
    return {"requests": len(prompts), "steps": len(t_ar), "ar_ms_per_step": ms(t_ar) if t_ar else None,
            "codec_ms_per_step": ms(t_codec) if t_codec else None,
            "first_chunk_ms": ms(list(first.values())), "audio_s": samples / SAMPLE_RATE, "wall_s": wall,
            "audio_s_per_wall_s": samples / SAMPLE_RATE / wall}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--requests-per-slot", type=int, default=3)
    ap.add_argument("--packet", type=int, default=4)
    ap.add_argument("--prompt-len", type=int, default=24)
    ap.add_argument("--mix", action="store_true", help="per-request parameters: 1/4 top-p 0.8, 1/4 greedy, the rest the session's")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("serve_probe needs a CUDA device")
    import qwen3_tts_b200 as q
    from qwen3_tts_b200 import synthetic
    from qwen3_tts_b200.codec import CodecDecoder
    from qwen3_tts_b200.engine import AREngine
    dev = "cuda:0"
    cfg, ccfg = synthetic.cfg_1p7b(), q.CodecConfig()
    max_b = max(args.slots)
    eng = AREngine(cfg, synthetic.random_tts_weights(cfg, device="cpu", seed=0), device=dev, max_batch=max_b,
                   max_ctx=args.prompt_len + max(HORIZONS) + 8)
    codec = CodecDecoder(ccfg, synthetic.random_codec_weights(ccfg, device="cpu", seed=0), device=dev,
                         max_frames=max(HORIZONS) + 8, max_batch=max_b)
    H = cfg.talker.hidden_size
    g = torch.Generator().manual_seed(0)
    pad = (torch.randn(H, generator=g) * 0.1).bfloat16()
    sp = q.SamplingParams(do_sample=True, subtalker_dosample=True, max_new_tokens=max(HORIZONS) + 1, suppress_eos=True, seed=7)
    out = {"what": "ContinuousBatcher.stream(): 1.7B talker + default codec, seeded random weights, suppress_eos, "
                   f"{args.packet}-frame packets, horizons {list(HORIZONS)} frames, n_slots requests at once then one "
                   "more per step", "sampling": "mixed: 1/4 top-p 0.8, 1/4 greedy, 1/2 session (top-k 50, T 0.9)" if args.mix
           else "uniform: top-k 50, T 0.9", "card": card(), "results": {}}
    for S in args.slots:
        n_req = S * args.requests_per_slot
        prompts = [(torch.randn(args.prompt_len, H, generator=g) * 0.5).bfloat16() for _ in range(n_req)]
        run_session(eng, codec, pad, sp, prompts[:S], S, args.packet, (8,), timed=False, mix=args.mix)   # warm-up: every shape
        out["results"][f"n_slots={S}"] = run_session(eng, codec, pad, sp, prompts, S, args.packet, HORIZONS, timed=True,
                                                     mix=args.mix)
    out["card_after"] = card()
    print(json.dumps(out))
    codec.close()
    eng.close()


if __name__ == "__main__":
    main()
