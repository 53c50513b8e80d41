"""Cost of audio formats in the continuous batcher, on the GPU: the resampler kernel's time (CUDA events around its
launches) and the batcher's _push_audio time per step (host clock ending in a synchronise), at 8 and 32 slots with the
default codec and 4-frame packets, for all rows in the default format, all rows 8 kHz mu-law and all rows 48 kHz
float32.  With --speed, the same for every row at each of the given speaking rates (24 kHz float32, so only the
time-stretch runs), and the time-stretch step (CUDA events around q3_stretch_step_rows calls of one packet per row)
instead of the resampler's.  With --pitch, every row at each of the given pitches (24 kHz float32: the time-stretch
and the pitched resampler run), timing the pitched resampler step; with --volume, every row at each of the given
volumes (only the limiter runs), timing the limiter step; with --loudness, every row at each of the given loudness
targets (the loudness normaliser and the limiter run), timing the loudness step.  Prints one JSON line, with the card's name and power limit
read in the same run.

    python tools/format_probe.py [--steps 60] [--warmup 10] [--speed 0.5 1.25 2.0] [--pitch -7 3] [--volume 6 -6]
                                 [--loudness -16]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


class _Cfg:          # the few engine fields ContinuousBatcher.__init__ reads
    class talker:
        hidden_size = 8
    num_code_groups = 16


class _Engine:
    cfg, max_ctx = _Cfg, 1 << 20

    def __init__(self, device):
        import torch
        self.device = torch.device(device)

    def session_begin(self, *a, **k):
        pass


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as e:   # the numbers stay, the card is reported as unknown
        return f"unknown ({e!r})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--speed", type=float, nargs="*", default=None)
    ap.add_argument("--pitch", type=float, nargs="*", default=None)
    ap.add_argument("--volume", type=float, nargs="*", default=None)
    ap.add_argument("--loudness", type=float, nargs="*", default=None)
    a = ap.parse_args()
    import torch
    import qwen3_tts_b200 as q
    from qwen3_tts_b200 import _lib, audio, synthetic
    from qwen3_tts_b200.codec import CodecDecoder
    from qwen3_tts_b200.scheduler import ContinuousBatcher, _Request
    if not torch.cuda.is_available():
        raise SystemExit("format_probe needs a GPU")
    dev = "cuda:0"
    ccfg = q.CodecConfig()
    dec = CodecDecoder(ccfg, synthetic.random_codec_weights(ccfg, device="cpu", seed=0), device=dev, max_frames=1024)
    P, up = 4, dec.total_upsample
    formats = {"default": None, "8k_ulaw": q.AudioFormat(8000, "ulaw"), "48k_f32": q.AudioFormat(48000, "f32")}
    if a.speed or a.pitch or a.volume or a.loudness:
        formats = {"default": None, **{f"speed_{sp}": q.AudioFormat(24000, speed=sp) for sp in a.speed or ()},
                   **{f"pitch_{p}": q.AudioFormat(24000, pitch=p) for p in a.pitch or ()},
                   **{f"volume_{v}": q.AudioFormat(24000, volume=v) for v in a.volume or ()},
                   **{f"loudness_{t}": q.AudioFormat(24000, loudness=t) for t in a.loudness or ()}}
    results = []
    g = torch.Generator().manual_seed(0)
    for S in (8, 32):
        for name, fmt in formats.items():
            cb = ContinuousBatcher(_Engine(dev), torch.zeros(8), q.SamplingParams(max_new_tokens=2048), n_slots=S,
                                   packet_frames=P, codec=dec)
            cb.codes.copy_(torch.randint(0, ccfg.codebook_size, cb.codes.shape, generator=g).to(cb.codes))
            chain = dict(audio.stages(fmt))
            reqs = [_Request(s, None, None, 2000, chain=chain) for s in range(S)]
            for s, r in enumerate(reqs):
                r.slot = s
                cb.running[s] = r
            cb.cstream.reset()
            for stage, args in chain.items():
                cb.stages[stage] = getattr(audio, stage)(dev, S, P * up)
                cb.stages[stage].reset(range(S), *args)
            times = []
            for it in range(a.warmup + a.steps):
                new = {s: (r, it * P, P) for s, r in enumerate(reqs)}
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                cb._push_audio(new)
                torch.cuda.synchronize()
                if it >= a.warmup:
                    times.append(time.perf_counter() - t0)
            row = {"slots": S, "format": name, "push_audio_ms_mean": 1e3 * sum(times) / len(times),
                   "push_audio_ms_min": 1e3 * min(times)}
            if chain:    # one step of the timed stage (its job upload and kernel) of one packet per row
                res = cb.stages[next(n for n in ("Loudness", "Limiter", "Resampler", "TimeStretch") if n in chain)]
                fn = getattr(res.lib, f"q3_{res.PREFIX}_step_rows")
                x = torch.rand(S, P * up, device=dev) * 2 - 1
                cnt, end = (C.c_int32 * S)(*[P * up] * S), (C.c_int32 * S)()
                nout = (C.c_int32 * S)()
                st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
                step = lambda: _lib.check(fn(res.h, x.data_ptr(), x.stride(0), cnt, end, res._out.data_ptr(), nout, st))  # noqa: E731
                for _ in range(a.warmup):
                    step()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                n = 200
                e0.record()
                for _ in range(n):
                    step()
                e1.record()
                torch.cuda.synchronize()
                row[res.PREFIX + "_step_us"] = 1e3 * e0.elapsed_time(e1) / n
                row["outputs_per_row"] = int(nout[0])
            for obj in cb.stages.values():
                obj.close()
            cb.cstream.close()
            results.append(row)
    name, power = _card()
    print(json.dumps({"gpu": name, "power_limit": power, "packet_frames": P, "results": results}))


if __name__ == "__main__":
    main()
