"""Speaking rate in the continuous batcher: every request's concatenated stream() chunks equal
Resampler.oneshot(TimeStretch.oneshot(w, speed), 24000, its rate and encoding), w the one-shot decode of its codes (at
24 kHz float32 just the stretch), while requests of mixed speeds and formats share the session's slots; a parked and
resumed request streams exactly what it streams never parked; a voice-clone request stretches its generated part."""
import numpy as np
import pytest
import torch

from tests.test_gpu_scheduler_audio_format import _model, _sp, _want as _decoded

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _fmts():
    from qwen3_tts_b200 import AudioFormat
    return [None, AudioFormat(24000, speed=0.75), AudioFormat(8000, "ulaw", 1.5), AudioFormat(24000, speed=1.0),
            AudioFormat(16000, "s16", 0.5)]


def _run(fmts, park=None):
    """Five requests through two slots (three submitted while the session runs); `park`: (rid, step to park at, step
    to resume at).  Returns (batcher, {rid: [chunks]})."""
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    eng, dec, embs, trail, pad = _model()
    horizons = [20, 3, 20, 2, 16]
    cb = ContinuousBatcher(eng, pad, _sp(), n_slots=2, packet_frames=4, codec=dec)
    sub = lambda i: cb.submit(embs[i], trail[i], key=i, max_frames=horizons[i], audio_format=fmts[i])  # noqa: E731
    sub(0)
    sub(1)
    out = {}
    for it, (chunks, _) in enumerate(cb.stream()):
        for rid, a in chunks.items():
            out.setdefault(rid, []).append(a)
        if it == 0:
            sub(2)
            sub(3)
        if it == 2:
            sub(4)
        if park is not None and it == park[1]:
            cb.park(park[0])
        if park is not None and it == park[2]:
            cb.resume(park[0])
    return cb, out


def _want(ts, res, dec, codes, fmt, ref=None):
    from qwen3_tts_b200 import AudioFormat
    wav = _decoded(res, dec, codes, None, ref=ref)
    if fmt is None:
        return wav
    y = ts.oneshot(wav, fmt.speed)
    return y if AudioFormat(fmt.sample_rate, fmt.encoding) == AudioFormat(24000) else \
        res.oneshot(y, 24000, AudioFormat(fmt.sample_rate, fmt.encoding))


def test_mixed_speeds_stream_the_oneshot_stretch_of_each_request():
    from qwen3_tts_b200.audio import Resampler, TimeStretch
    eng, dec, *_ = _model()
    fmts = _fmts()
    cb, out = _run(fmts)
    assert cb.stretcher is not None and cb.resampler is not None
    ts, res = TimeStretch(DEV, 1, 8192), Resampler(DEV, 1, 64)
    dtypes = {None: np.float32, "f32": np.float32, "s16": np.int16, "ulaw": np.uint8}
    for i, fmt in enumerate(fmts):
        if i == 3:
            continue   # speed 1 at 24 kHz float32 takes the default path: compared with a plain session below
        n = cb.done[i].shape[0]
        got = np.concatenate(out[i]) if i in out else np.zeros(0, dtypes[fmt and fmt.encoding])
        want = _want(ts, res, dec, cb.done[i], fmt) if n else np.zeros(0, got.dtype)
        assert got.dtype == want.dtype and np.array_equal(got, want), (i, fmt, got.shape, want.shape)
    # a speed-1 request streams exactly what a session without formats streams
    plain, pout = _run([None] * 5)
    assert plain.stretcher is None and plain.resampler is None
    assert len(out[3]) == len(pout[3]) and all(np.array_equal(a, b) for a, b in zip(out[3], pout[3]))
    ts.close()
    res.close()


def test_parked_request_streams_what_it_streams_never_parked():
    fmts = _fmts()
    fmts[0] = fmts[2]                  # request 0 (8 kHz mu-law at 1.5x) is parked after its first packet
    _, ref = _run(fmts)
    cb, got = _run(fmts, park=(0, 0, 2))
    assert [m[:2] for m in cb.moves] == [("park", 0), ("resume", 0)], cb.moves
    for i in range(5):
        a = np.concatenate(got[i]) if i in got else None
        b = np.concatenate(ref[i]) if i in ref else None
        assert (a is None and b is None) or np.array_equal(a, b), i
    # and a stretch-only request (24 kHz float32 at 0.75x) parked the same way
    fmts = _fmts()
    fmts[0] = fmts[1]
    _, ref = _run(fmts)
    cb, got = _run(fmts, park=(0, 0, 2))
    assert [m[:2] for m in cb.moves] == [("park", 0), ("resume", 0)], cb.moves
    assert np.array_equal(np.concatenate(got[0]), np.concatenate(ref[0]))


def test_voice_clone_request_stretches_its_generated_part():
    from qwen3_tts_b200 import AudioFormat
    from qwen3_tts_b200.audio import Resampler, TimeStretch
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    eng, dec, embs, trail, pad = _model()
    g = torch.Generator().manual_seed(7)
    ref_codes = torch.randint(0, dec.cfg.codebook_size, (6, dec.cfg.num_quantizers), generator=g)
    fmt = AudioFormat(24000, speed=1.25)
    cb = ContinuousBatcher(eng, pad, _sp(), n_slots=2, packet_frames=4, codec=dec)
    cb.submit(embs[0], trail[0], key=0, max_frames=12, ref_codes=ref_codes, audio_format=fmt)
    cb.submit(embs[1], trail[1], key=1, max_frames=9, audio_format=AudioFormat(8000, "ulaw", 0.8))
    out = {}
    for chunks, _ in cb.stream():
        for rid, a in chunks.items():
            out.setdefault(rid, []).append(a)
    ts, res = TimeStretch(DEV, 1, 8192), Resampler(DEV, 1, 64)
    assert np.array_equal(np.concatenate(out[0]), _want(ts, res, dec, cb.done[0], fmt, ref=ref_codes))
    assert np.array_equal(np.concatenate(out[1]), _want(ts, res, dec, cb.done[1], AudioFormat(8000, "ulaw", 0.8)))
    ts.close()
    res.close()
