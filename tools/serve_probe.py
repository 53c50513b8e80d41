"""Serving probe: continuous batching with audio out (ContinuousBatcher(..., codec=...).stream()).

Full 1.7B talker and default codec shapes with seeded random weights, suppress_eos, 4-frame packets, horizons
staggered so that requests leave at different steps and new ones are admitted into running sessions.  For each
n_slots it reports the AR and codec milliseconds per step, the time from submit() to a request's first audio chunk,
and the aggregate audio seconds produced per wall second, with the card name and power limit read in the same run.
With --mix the requests carry their own sampling parameters: every fourth one top-p 0.8 (talker and subtalker, the
generic sampler path), every fourth one greedy, the rest the session's; comparing with a run without it gives what
such rows cost the whole session.
With --voice-clone every second request carries a 3 s reference (38 frames of random valid codes) and a prompt longer
by those frames, as an ICL voice-clone prompt is: its codec row is seeded with the reference at admission
(CodecStream.seed).  The probe then also reports the seed time per admission, the first-chunk times of voice-clone and
plain requests apart, and, for comparison in the same run, the time to push one reference through an n_slots-row
stream of the session's packet size, which is what seeding through the session's own stream would stall it for.
With --live-text TOKENS_PER_S every request is live (submit(text_open=True)): its prompt holds the first text token,
and its other text rows (horizon // 3 of them, then tts_eos) are appended between steps at that rate from its submit
time, after which it is closed.  The probe then also reports the share of row-steps held (the host's count of the
engine's hold rule); first_chunk_ms is then the time from the first text token to the first audio chunk.
With --park (with --live-text) the batcher parks live requests that wait for text when another request needs a slot
(ContinuousBatcher(park_waiting=True)).  The probe then also reports parks and resumes per wall second, the time of an
engine park and resume (host clock around the call, ending in a device synchronise), the park kernel's time (CUDA
events around the call, which only enqueues it) and the record bytes it gathers over that time.
With --voices K the requests are drawn from K registered voices, alternately ICL clones (a 38-frame reference and a
24-token reference text: a 33-row prefix of 3 role, 6 codec-prefix and 24 reference rows, 15 rows of its own) and
VoiceDesign voices (a 48-token instruct: a 56-row prefix, 1 row of its own), with the engine's random rows of those
lengths.  Every request set runs registered (submit(voice=)) and unregistered (the whole prompt, and ref_codes for the
clones), the two sessions alternated twice in one run.  The probe reports for each the median admission time (a host
clock around the engine's admission and the codec-row setup of every step that admits, each ending in a device
synchronise), the AR step and the first-chunk latency.
With --live-clone (with --live-text) every request is a live ICL voice clone (a 38-frame reference and a 24-token
reference text, so K = 39 - 24 = 15 prompt rows wait for target text), alternately unregistered (the known prompt rows
and ref_codes) and of a registered voice (no rows of its own but the overlay).  Its first text row is given at submit,
the next K + horizon // 3 rows and tts_eos arrive at TOKENS_PER_S from then, and it is then closed.  The probe reports
the AR step, the time from the first text row to the admission (host clock after the engine's admission and a device
synchronise) and from the admission to the first audio chunk, over all requests and for each kind.

    python tools/serve_probe.py [--slots 8 32] [--requests-per-slot 3] [--packet 4] [--mix] [--voice-clone]
                                [--live-text TOKENS_PER_S [--park | --live-clone]] [--voices K]

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
REF_FRAMES = 38                # a 3 s voice-clone reference at 12.5 frames/s
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


def record_bytes(eng, pos, trailing):
    """Bytes of a parked row's record (q3_row_park): talker K/V of pos positions, 4 hidden rows, the trailing text,
    the seen bytes and the DevState ints."""
    t, G = eng.cfg.talker, 16
    return 2 * t.num_layers * t.num_kv_heads * pos * t.head_dim * 2 + (4 + trailing) * t.hidden_size * 2 + t.vocab_size + (6 + G) * 4


def run_session(eng, codec, pad, sp, prompts, n_slots, packet, horizons, timed, mix=False, refs=None, live=None, texts=None,
                park=False):
    """One session: n_slots requests at once, then one more per step until all are in.  refs[i]: request i's
    reference codes or None.  live: text rows per second (texts[i]: request i's rows after the first token, tts_eos
    last), or None.  Returns the measurements."""
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cb = ContinuousBatcher(eng, pad, sp, n_slots=n_slots, packet_frames=packet, codec=codec, park_waiting=park)
    t_ar, t_codec, t_seed = [], [], []
    t_park, t_resume, k_park, b_park = [], [], [], []
    refs = refs or [None] * len(prompts)

    def clocked(fn, acc):
        def call(*a, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn(*a, **k)
            torch.cuda.synchronize()
            acc.append(time.perf_counter() - t0)
            return r
        return call

    held = [0, 0]     # row-steps held, row-steps run (live text)
    committed = {}    # request id -> steps committed, by the engine's hold rule

    def count_holds(fn):
        def call(n, codes):
            for r in cb.running.values():
                c = committed.get(r.rid, 0)
                k = n if r.closed else min(n, max(0, r.n_text - c))
                committed[r.rid] = c + k
                held[0] += n - k
                held[1] += n
            return fn(n, codes)
        return call

    moving = [None]   # the request the batcher is parking or resuming

    def watch(fn):
        def call(*a):
            moving[0] = cb.running[a[0]] if fn.__name__ == "_park" else a[0]
            return fn(*a)
        return call

    def clocked_park(fn):
        def call(slot):
            r = moving[0]
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record()
            out = fn(slot)
            e1.record()
            torch.cuda.synchronize()
            t_park.append(time.perf_counter() - t0)
            k_park.append(e0.elapsed_time(e1) * 1e-3)
            b_park.append(record_bytes(eng, prompts[r.rid].shape[0] + committed.get(r.rid, 0), r.n_text))
            return out
        return call

    decode = type(eng).decode.__get__(eng)
    if timed:
        decode = clocked(decode, t_ar)
        if park:
            cb._park, cb._resume = watch(cb._park), watch(cb._resume)
            eng.park = clocked_park(type(eng).park.__get__(eng))
            eng.resume = clocked(type(eng).resume.__get__(eng), t_resume)
    if live:
        decode = count_holds(decode)
    if timed or live:
        eng.decode = decode
        cb.cstream.push = clocked(cb.cstream.push, t_codec)
        cb.cstream.seed = clocked(cb.cstream.seed, t_seed)
    submitted, first, samples = {}, {}, 0
    todo = list(range(len(prompts)))
    fed = {}

    def submit(i):
        rid = cb.submit(prompts[i], texts[i][:0] if live else None, key=i, max_frames=horizons[i % len(horizons)],
                        sampling=mixed_sampling(sp, i) if mix else None, ref_codes=refs[i], text_open=bool(live))
        submitted[rid] = time.perf_counter()
        if live:
            fed[rid] = 0

    def feed(now):
        for rid in list(fed):
            if rid in cb.done:
                del fed[rid]
                continue
            due = min(int((now - submitted[rid]) * live), texts[rid].shape[0])
            if due > fed[rid]:
                cb.append_text(rid, texts[rid][fed[rid]:due])
                fed[rid] = due
            if fed[rid] == texts[rid].shape[0]:
                cb.close_text(rid)
                del fed[rid]

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
            if live:
                feed(time.perf_counter())
    finally:
        if timed or live:
            del eng.decode
        if timed and park:
            del eng.park, eng.resume
        cb.cstream.close()
    wall = time.perf_counter() - t0
    ms = lambda v: {"median": float(np.median(v)) * 1e3, "p90": float(np.percentile(v, 90)) * 1e3} if v else None  # noqa: E731
    out = {"requests": len(prompts), "steps": len(t_ar), "ar_ms_per_step": ms(t_ar), "codec_ms_per_step": ms(t_codec),
           "first_chunk_ms": ms(list(first.values())), "audio_s": samples / SAMPLE_RATE, "wall_s": wall,
           "audio_s_per_wall_s": samples / SAMPLE_RATE / wall}
    if live:
        out["held_row_step_share"] = held[0] / max(held[1], 1)
    if park:
        out.update({"parks": len(t_park), "resumes": len(t_resume), "parks_per_s": len(t_park) / wall,
                    "resumes_per_s": len(t_resume) / wall, "park_ms": ms(t_park), "resume_ms": ms(t_resume),
                    "park_kernel_ms": ms(k_park), "park_record_mb": ms([b / 1e9 for b in b_park]),   # (ms() scales by 1e3)
                    "park_gb_per_s": ms([b / k / 1e12 for b, k in zip(b_park, k_park)])})
    if any(r is not None for r in refs):
        out["first_chunk_ms_voice_clone"] = ms([t for rid, t in first.items() if refs[rid] is not None])
        out["first_chunk_ms_plain"] = ms([t for rid, t in first.items() if refs[rid] is None])
        # the first admission also opens the private seed stream (device allocation): reported apart
        out["seed_ms_first_admission"] = t_seed[0] * 1e3 if t_seed else None
        out["seed_ms_per_admission"] = ms(t_seed[1:])
        out["seed_admissions"] = len(t_seed)
    return out


VOICE_REF_TEXT, VOICE_INSTRUCT = 24, 48   # tokens
VOICE_OVERLAY = 3 + 6                     # role rows and codec-prefix overlay rows (think, language, speaker, pad)


def voice_session(eng, codec, pad, sp, reqs, n_slots, packet, horizons, registered):
    """One session of `reqs` [(voice, own rows, full rows)]: registered requests submit their own rows with the voice,
    unregistered ones the full rows and the reference codes.  Returns admission, AR-step and first-chunk times."""
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cb = ContinuousBatcher(eng, pad, sp, n_slots=n_slots, packet_frames=packet, codec=codec)
    t_ar, t_admit = [], []
    admitting = [0.0]

    def clocked(fn, acc=None):
        def call(*a, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn(*a, **k)
            torch.cuda.synchronize()
            if acc is None:
                admitting[0] += time.perf_counter() - t0
            else:
                acc.append(time.perf_counter() - t0)
            return r
        return call

    eng.admit = clocked(type(eng).admit.__get__(eng))
    eng.decode = clocked(type(eng).decode.__get__(eng), t_ar)
    for name in ("seed", "copy_from", "reset"):
        setattr(cb.cstream, name, clocked(getattr(cb.cstream, name)))
    submitted, first = {}, {}

    def submit(i):
        v, own, full = reqs[i]
        h = horizons[i % len(horizons)]
        if registered:
            cb.submit(own, None, key=i, max_frames=h, voice=v)
        else:
            cb.submit(full, None, key=i, max_frames=h, ref_codes=v.ref_codes)
        submitted[i] = time.perf_counter()

    todo = list(range(len(reqs)))
    for i in todo[:n_slots]:
        submit(i)
    todo = todo[n_slots:]
    try:
        for chunks, _ in cb.stream():
            now = time.perf_counter()
            if admitting[0]:
                t_admit.append(admitting[0])
                admitting[0] = 0.0
            for rid in chunks:
                first.setdefault(rid, now - submitted[rid])
            if todo:
                submit(todo.pop(0))
    finally:
        del eng.admit, eng.decode
        cb.cstream.close()
    ms = lambda v: {"median": float(np.median(v)) * 1e3, "p90": float(np.percentile(v, 90)) * 1e3} if v else None  # noqa: E731
    return {"admissions": len(t_admit), "admission_ms": ms(t_admit), "ar_ms_per_step": ms(t_ar),
            "first_chunk_ms": ms(list(first.values()))}


def voices_probe(eng, codec, pad, sp, S, K, n_req, packet, g):
    """--voices K: K voices, requests i of voice i % K, registered and unregistered sessions alternated twice."""
    from types import SimpleNamespace
    H = eng.cfg.talker.hidden_size
    voices = []
    for k in range(K):
        icl = k % 2 == 0
        P = VOICE_OVERLAY + (VOICE_REF_TEXT if icl else VOICE_INSTRUCT)
        prefix = (torch.randn(P, H, generator=g) * 0.5).bfloat16()
        ref = torch.randint(0, codec.cfg.codebook_size, (REF_FRAMES, codec.cfg.num_quantizers), generator=g) if icl else None
        v = SimpleNamespace(engine=eng, codec=codec, prefix=prefix, prefix_len=P, prefix_id=eng.create_prefix(prefix),
                            ref_codes=ref, ref_len=REF_FRAMES if icl else 0, bank=codec.bank_reference(ref) if icl else None,
                            own=REF_FRAMES + 1 - VOICE_REF_TEXT if icl else 1, pending=0, closed=False)
        voices.append(v)
    reqs = []
    for i in range(n_req):
        v = voices[i % K]
        own = (torch.randn(v.own, H, generator=g) * 0.5).bfloat16()
        reqs.append((v, own, torch.cat([v.prefix, own], 0)))
    voice_session(eng, codec, pad, sp, reqs[:S], S, packet, (8,), True)      # warm-up: every shape
    voice_session(eng, codec, pad, sp, reqs[:S], S, packet, (8,), False)
    runs = {"registered": [], "unregistered": []}
    for _ in range(2):
        for mode in ("registered", "unregistered"):
            runs[mode].append(voice_session(eng, codec, pad, sp, reqs, S, packet, HORIZONS, mode == "registered"))
    for v in voices:
        eng.free_prefix(v.prefix_id)
        if v.bank is not None:
            codec.bank_release(*v.bank)
    return runs


def live_clone_session(eng, codec, pad, sp, reqs, n_slots, packet, horizons, rate):
    """One session of live ICL clones `reqs` [(voice or None, known prompt rows, overlay, text rows with tts_eos last,
    reference codes)]: n_slots requests at once, then one more per step; a request's first text row comes with submit,
    the others at `rate` rows per second from then, after which it is closed."""
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cb = ContinuousBatcher(eng, pad, sp, n_slots=n_slots, packet_frames=packet, codec=codec)
    t_ar, admitted = [], {}

    def clocked_admit(fn):
        def call(slots, keys, *a, **k):
            r = fn(slots, keys, *a, **k)
            torch.cuda.synchronize()
            now = time.perf_counter()
            for key in keys:
                admitted[key] = now
            return r
        return call

    def clocked(fn):
        def call(*a, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn(*a, **k)
            torch.cuda.synchronize()
            t_ar.append(time.perf_counter() - t0)
            return r
        return call

    eng.admit = clocked_admit(type(eng).admit.__get__(eng))
    eng.decode = clocked(type(eng).decode.__get__(eng))
    submitted, first, fed = {}, {}, {}

    def submit(i):
        v, known, ov, text, ref = reqs[i]
        kw = {"voice": v} if v is not None else {"ref_codes": ref}
        cb.submit(known, text[:1], key=i, max_frames=horizons[i % len(horizons)], text_open=True, overlay=ov, **kw)
        submitted[i], fed[i] = time.perf_counter(), 1

    def feed(now):
        for rid in list(fed):
            text = reqs[rid][3]
            due = min(1 + int((now - submitted[rid]) * rate), text.shape[0])
            if due > fed[rid]:
                cb.append_text(rid, text[fed[rid]:due])
                fed[rid] = due
            if fed[rid] == text.shape[0]:
                cb.close_text(rid)
                del fed[rid]

    todo = list(range(len(reqs)))
    for i in todo[:n_slots]:
        submit(i)
    todo = todo[n_slots:]
    try:
        for chunks, _ in cb.stream():
            now = time.perf_counter()
            for rid in chunks:
                first.setdefault(rid, now - admitted[rid])
            if todo:
                submit(todo.pop(0))
            feed(time.perf_counter())
    finally:
        del eng.admit, eng.decode
        cb.cstream.close()
    ms = lambda v: {"median": float(np.median(v)) * 1e3, "p90": float(np.percentile(v, 90)) * 1e3} if v else None  # noqa: E731
    out = {"requests": len(reqs), "steps": len(t_ar), "ar_ms_per_step": ms(t_ar)}
    for name, pick in (("all", lambda i: True), ("unregistered", lambda i: reqs[i][0] is None),
                       ("registered", lambda i: reqs[i][0] is not None)):
        out[name] = {"first_token_to_admission_ms": ms([admitted[i] - submitted[i] for i in admitted if pick(i)]),
                     "admission_to_first_chunk_ms": ms([t for i, t in first.items() if pick(i)])}
    return out


def live_clone_probe(eng, codec, pad, sp, S, n_req, packet, rate, g):
    """--live-clone: requests alternately unregistered and of one registered ICL voice; one warm-up session, then the
    timed one."""
    from types import SimpleNamespace
    H = eng.cfg.talker.hidden_size
    P = VOICE_OVERLAY + VOICE_REF_TEXT
    K = REF_FRAMES + 1 - VOICE_REF_TEXT
    prefix = (torch.randn(P, H, generator=g) * 0.5).bfloat16()
    ref = torch.randint(0, codec.cfg.codebook_size, (REF_FRAMES, codec.cfg.num_quantizers), generator=g)
    voice = SimpleNamespace(engine=eng, codec=codec, prefix=prefix, prefix_len=P, prefix_id=eng.create_prefix(prefix),
                            ref_codes=ref, ref_len=REF_FRAMES, bank=codec.bank_reference(ref), icl=True,
                            non_streaming_mode=False, pending=0, closed=False)
    reqs = []
    for i in range(n_req):
        v = voice if i % 2 else None
        known = prefix[:0] if v is not None else prefix
        ov = (torch.randn(K, H, generator=g) * 0.5).bfloat16()
        text = (torch.randn(K + HORIZONS[i % len(HORIZONS)] // 3 + 1, H, generator=g) * 0.1).bfloat16()
        reqs.append((v, known, ov, text, ref))
    live_clone_session(eng, codec, pad, sp, reqs[:S], S, packet, (8,), rate)   # warm-up: every shape
    res = live_clone_session(eng, codec, pad, sp, reqs, S, packet, HORIZONS, rate)
    eng.free_prefix(voice.prefix_id)
    codec.bank_release(*voice.bank)
    return res


def naive_seed_ms(codec, n_slots, packet, ref, reps=5):
    """The path seeding avoids: one reference pushed through an n_slots-row stream of the session's packet size (every
    row computed each step, the other rows with count 0).  Sync-clocked; median over `reps` after one warm-up."""
    st = codec.open_stream(n_slots, max_packet_frames=packet)
    codes = torch.zeros(n_slots, ref.shape[1], ref.shape[0], dtype=torch.int32, device=codec.device)
    codes[0] = ref.T.to(codec.device, torch.int32)
    counts = [ref.shape[0]] + [0] * (n_slots - 1)
    ts = []
    try:
        for r in range(reps + 1):
            st.reset([0])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            st.push(codes, counts)
            torch.cuda.synchronize()
            if r:
                ts.append(time.perf_counter() - t0)
    finally:
        st.close()
    return {"median": float(np.median(ts)) * 1e3, "p90": float(np.percentile(ts, 90)) * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--requests-per-slot", type=int, default=3)
    ap.add_argument("--packet", type=int, default=4)
    ap.add_argument("--prompt-len", type=int, default=24)
    ap.add_argument("--mix", action="store_true", help="per-request parameters: 1/4 top-p 0.8, 1/4 greedy, the rest the session's")
    ap.add_argument("--voice-clone", action="store_true",
                    help=f"every second request carries a {REF_FRAMES}-frame reference and a prompt longer by it")
    ap.add_argument("--live-text", type=float, default=None, metavar="TOKENS_PER_S",
                    help="every request is live: its text rows arrive at this rate after submit")
    ap.add_argument("--park", action="store_true", help="with --live-text: park requests that wait for text when a slot is needed")
    ap.add_argument("--live-clone", action="store_true",
                    help="with --live-text: every request is a live ICL voice clone, unregistered and registered")
    ap.add_argument("--voices", type=int, default=None, metavar="K",
                    help="requests of K registered voices (ICL clones and VoiceDesign), run registered and unregistered")
    args = ap.parse_args()
    if (args.park or args.live_clone) and not args.live_text:
        raise SystemExit("--park and --live-clone need --live-text")
    if args.park and args.live_clone:
        raise SystemExit("--park and --live-clone are separate probes")
    if not torch.cuda.is_available():
        raise SystemExit("serve_probe needs a CUDA device")
    import qwen3_tts_b200 as q
    from qwen3_tts_b200 import synthetic
    from qwen3_tts_b200.codec import CodecDecoder
    from qwen3_tts_b200.engine import AREngine
    dev = "cuda:0"
    cfg, ccfg = synthetic.cfg_1p7b(), q.CodecConfig()
    max_b = max(args.slots)
    extra = REF_FRAMES if (args.voice_clone or args.voices or args.live_clone) else 0   # the reference's frames in the prompt and the codec row
    if args.voices:
        extra += VOICE_OVERLAY + VOICE_INSTRUCT
    eng = AREngine(cfg, synthetic.random_tts_weights(cfg, device="cpu", seed=0), device=dev, max_batch=max_b,
                   max_ctx=args.prompt_len + extra + max(HORIZONS) + 8)
    codec = CodecDecoder(ccfg, synthetic.random_codec_weights(ccfg, device="cpu", seed=0), device=dev,
                         max_frames=extra + max(HORIZONS) + 8, max_batch=max_b)
    H = cfg.talker.hidden_size
    g = torch.Generator().manual_seed(0)
    pad = (torch.randn(H, generator=g) * 0.1).bfloat16()
    sp = q.SamplingParams(do_sample=True, subtalker_dosample=True, max_new_tokens=max(HORIZONS) + 1, suppress_eos=True, seed=7)
    out = {"what": "ContinuousBatcher.stream(): 1.7B talker + default codec, seeded random weights, suppress_eos, "
                   f"{args.packet}-frame packets, horizons {list(HORIZONS)} frames, n_slots requests at once then one "
                   "more per step", "sampling": "mixed: 1/4 top-p 0.8, 1/4 greedy, 1/2 session (top-k 50, T 0.9)" if args.mix
           else "uniform: top-k 50, T 0.9", "card": card(), "results": {}}
    if args.live_text:
        out["live_text"] = (f"every request live: {args.live_text:g} text tokens/s from submit, "
                            f"{'15 + ' if args.live_clone else ''}horizon // 3 tokens after the first, then tts_eos and close")
        out["park"] = "park_waiting=True" if args.park else "no parking"

    if args.live_clone:
        out["live_clone"] = (f"every request a live ICL clone ({REF_FRAMES}-frame reference, {VOICE_REF_TEXT}-token reference "
                             f"text: {REF_FRAMES + 1 - VOICE_REF_TEXT} rows wait for target text), alternately unregistered "
                             "and of one registered voice; first text row at submit")
        for S in args.slots:
            out["results"][f"n_slots={S}"] = live_clone_probe(eng, codec, pad, sp, S, S * args.requests_per_slot, args.packet,
                                                              args.live_text, g)
        out["card_after"] = card()
        print(json.dumps(out))
        codec.close()
        eng.close()
        return
    if args.voice_clone:
        out["voice_clone"] = (f"every second request: {REF_FRAMES}-frame reference of random valid codes, prompt "
                              f"{args.prompt_len + REF_FRAMES} positions instead of {args.prompt_len}")
    if args.voices:
        out["voices"] = (f"{args.voices} voices: ICL clones ({REF_FRAMES}-frame reference, {VOICE_REF_TEXT}-token reference "
                         f"text) and VoiceDesign ({VOICE_INSTRUCT}-token instruct); registered and unregistered sessions "
                         "alternated twice")
        for S in args.slots:
            out["results"][f"n_slots={S}"] = voices_probe(eng, codec, pad, sp, S, args.voices, S * args.requests_per_slot,
                                                          args.packet, g)
        out["card_after"] = card()
        print(json.dumps(out))
        codec.close()
        eng.close()
        return
    for S in args.slots:
        n_req = S * args.requests_per_slot
        refs = [torch.randint(0, ccfg.codebook_size, (REF_FRAMES, ccfg.num_quantizers), generator=g)
                if args.voice_clone and i % 2 == 1 else None for i in range(n_req)]
        prompts = [(torch.randn(args.prompt_len + (0 if r is None else REF_FRAMES), H, generator=g) * 0.5).bfloat16()
                   for r in refs]
        texts = [torch.cat([(torch.randn(HORIZONS[i % len(HORIZONS)] // 3, H, generator=g) * 0.1).bfloat16(),
                            (torch.randn(1, H, generator=g) * 0.1).bfloat16()]) for i in range(n_req)] if args.live_text else None
        run_session(eng, codec, pad, sp, prompts[:S], S, args.packet, (8,), timed=False, mix=args.mix,
                    refs=refs[:S], live=args.live_text, texts=texts, park=args.park)   # warm-up: every shape
        res = run_session(eng, codec, pad, sp, prompts, S, args.packet, HORIZONS, timed=True, mix=args.mix, refs=refs,
                          live=args.live_text, texts=texts, park=args.park)
        if args.voice_clone:
            res["naive_push_ms_per_admission"] = naive_seed_ms(codec, S, args.packet, refs[1])
        out["results"][f"n_slots={S}"] = res
    out["card_after"] = card()
    print(json.dumps(out))
    codec.close()
    eng.close()


if __name__ == "__main__":
    main()
