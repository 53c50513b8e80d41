"""Streaming codec encoder timing: ms per packet (CUDA events, warmed up) at B in {1, 8, 32} rows with packets of 1 and 4
frames, kernel launches per packet, and the one-shot 3 s encode at B = 1 in the same run.  Default encoder config, seeded
random weights (timing does not depend on the values).  Prints the card's name and power limit beside the numbers.

    python tools/encoder_stream_probe.py [--iters N] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from qwen3_tts_b200 import _lib, synthetic  # noqa: E402
from qwen3_tts_b200.codec_encoder import CodecEncoder  # noqa: E402
from qwen3_tts_b200.config import EncoderConfig  # noqa: E402

DEV = "cuda:0"


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return name, out or "unknown"


def _time(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    cfg = EncoderConfig()
    enc = CodecEncoder(cfg, synthetic.random_encoder_weights(cfg, seed=2), device=DEV)
    name, plim = _card()
    print(f"card: {name}, power limit {plim}")
    res = {"card": name, "power_limit": plim, "packets": []}
    lib, hop, nq = enc.lib, enc.hop, cfg.valid_num_quantizers
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for B in (1, 8, 32):
        for n in (1, 4):
            s = enc.open_stream(B, max_packet_frames=n)
            wav = (torch.randn(B, n * hop, device=DEV) * 0.1).clamp(-1, 1)
            codes = torch.empty(B, nq, n, dtype=torch.int32, device=DEV)
            counts = (C.c_int32 * B)(*([n] * B))

            def step():
                _lib.check(lib.q3_codec_enc_stream_step_rows(s.h, wav.data_ptr(), n, counts, codes.data_ptr(), st))

            # positions advance by n per packet; reset all rows before they reach the RoPE table
            rows = (C.c_int32 * B)(*range(B))
            iters = min(a.iters, (enc.max_frames // cfg.downsample_stride) // n - 2)
            for _ in range(3):
                step()
            _lib.check(lib.q3_codec_enc_stream_reset_rows(s.h, B, rows, st))
            ms = _time(step, iters)
            launches = enc.last_launches()
            audio_ms = n * hop / 24.0
            print(f"B={B:2d} packet={n} frames ({audio_ms:.0f} ms audio): {ms:.3f} ms/packet, {launches} launches/packet"
                  + ("  SLOWER THAN REAL TIME" if ms > audio_ms else ""))
            res["packets"].append({"B": B, "frames": n, "ms": ms, "launches": launches, "audio_ms": audio_ms})
            s.close()
    wav = (torch.randn(1, 72000, device=DEV) * 0.1).clamp(-1, 1)
    for _ in range(3):
        enc.forward(wav)
    ms = _time(lambda: enc.forward(wav), a.iters)
    print(f"one-shot encode B=1, 3 s: {ms:.3f} ms, {enc.last_launches()} launches")
    res["one_shot_3s_ms"], res["one_shot_launches"] = ms, enc.last_launches()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
