"""Pitch and volume in the continuous batcher: every request's concatenated stream() chunks equal
Resampler.oneshot(Limiter.oneshot(TimeStretch.oneshot(w, speed, pitch), volume), 50*Lp, its rate and encoding), w the
one-shot decode of its codes and each stage skipped when the request does not use it, while requests of mixed speeds,
pitches, volumes, rates and encodings share the session's slots; a parked and resumed request streams exactly what it
streams never parked; a voice-clone request and a registered ICL voice shape their generated part."""
import numpy as np
import pytest
import torch

from tests.test_gpu_scheduler_audio_format import _model, _sp, _want as _decoded

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _fmts():
    from qwen3_tts_b200 import AudioFormat
    return [AudioFormat(24000, pitch=4.0, volume=6.0), AudioFormat(8000, "ulaw", 1.25, -3.0, -6.0),
            AudioFormat(24000, volume=12.0), AudioFormat(16000, "s16", pitch=-12.0, speed=0.6),
            AudioFormat(44100, "f32", 0.8, 2.5, 3.0)]


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


def _want(dec, codes, fmt, ref=None):
    """The documented composition of one request's whole audio."""
    from qwen3_tts_b200 import AudioFormat
    from qwen3_tts_b200.audio import Limiter, Resampler, TimeStretch
    ts, lim, res = TimeStretch(DEV, 1, 8192), Limiter(DEV, 1, 64), Resampler(DEV, 1, 64)
    try:
        y = _decoded(res, dec, codes, None, ref=ref)
        if fmt.hop != 480:
            y = ts.oneshot(y, fmt.speed, fmt.pitch)
        if fmt.volume != 0:
            y = lim.oneshot(y, fmt.volume)
        out = AudioFormat(fmt.sample_rate, fmt.encoding)
        if fmt.pitch_step != 480 or out != AudioFormat(24000):
            y = res.oneshot(y, 50 * fmt.pitch_step, out)
        return y
    finally:
        ts.close()
        lim.close()
        res.close()


def test_mixed_pitches_and_volumes_stream_the_oneshot_composition_of_each_request():
    eng, dec, *_ = _model()
    fmts = _fmts()
    cb, out = _run(fmts)
    assert cb.stretcher is not None and cb.limiter is not None and cb.resampler is not None
    dtypes = {"f32": np.float32, "s16": np.int16, "ulaw": np.uint8}
    for i, fmt in enumerate(fmts):
        n = cb.done[i].shape[0]
        got = np.concatenate(out[i]) if i in out else np.zeros(0, dtypes[fmt.encoding])
        want = _want(dec, cb.done[i], fmt) if n else np.zeros(0, got.dtype)
        assert got.dtype == want.dtype and np.array_equal(got, want), (i, fmt, got.shape, want.shape)


def test_parked_request_streams_what_it_streams_never_parked():
    fmts = _fmts()
    for src in (1, 2):                 # every stage, and the limiter alone
        fmts[0] = fmts[src]
        _, ref = _run(fmts)
        cb, got = _run(fmts, park=(0, 0, 2))
        assert [m[:2] for m in cb.moves] == [("park", 0), ("resume", 0)], cb.moves
        for i in range(5):
            a = np.concatenate(got[i]) if i in got else None
            b = np.concatenate(ref[i]) if i in ref else None
            assert (a is None and b is None) or np.array_equal(a, b), (src, i)


def test_voice_clone_request_and_a_registered_voice_shape_their_generated_part():
    from qwen3_tts_b200 import AudioFormat
    from qwen3_tts_b200.model import VoiceClonePromptItem
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    from tests.test_gpu_live_text import _sampling
    from tests.test_gpu_scheduler_audio import _codec
    from tests.test_gpu_voice_prefix import _voice_model
    eng, dec, embs, trail, pad = _model()
    g = torch.Generator().manual_seed(7)
    ref_codes = torch.randint(0, dec.cfg.codebook_size, (6, dec.cfg.num_quantizers), generator=g)
    fa, fb = AudioFormat(22050, "s16", 1.1, -5.0, 8.0), AudioFormat(24000, pitch=7.0)
    cb = ContinuousBatcher(eng, pad, _sp(), n_slots=2, packet_frames=4, codec=dec)
    cb.submit(embs[0], trail[0], key=0, max_frames=12, ref_codes=ref_codes, audio_format=fa)
    cb.submit(embs[1], trail[1], key=1, max_frames=9, audio_format=fb)
    out = {}
    for chunks, _ in cb.stream():
        for rid, a in chunks.items():
            out.setdefault(rid, []).append(a)
    assert np.array_equal(np.concatenate(out[0]), _want(dec, cb.done[0], fa, ref=ref_codes))
    assert np.array_equal(np.concatenate(out[1]), _want(dec, cb.done[1], fb))
    # a registered ICL voice: its codec row is copied from the reference bank, its audio shaped as any request's
    dec2 = _codec()
    w = _voice_model(dec2)
    H = w.model.cfg.talker.hidden_size
    it = VoiceClonePromptItem(torch.randint(0, 2000, (5, 16), generator=g), (torch.randn(H, generator=g) * 0.3).bfloat16(),
                              False, True, "a reference text")
    v = w.register_voice(voice_clone_prompt=it, language="English")
    suf, tr, vpad = w.build_voice_request("Hello there.", v)
    fv = AudioFormat(8000, "ulaw", 0.9, 2.0, -12.0)
    cb = ContinuousBatcher(w.model.engine, vpad, _sampling("sampled", 24), n_slots=2, packet_frames=4, codec=dec2)
    cb.submit(suf, tr, key=0, max_frames=10, voice=v, audio_format=fv)
    out = {}
    for chunks, _ in cb.stream():
        for rid, a in chunks.items():
            out.setdefault(rid, []).append(a)
    assert cb.limiter is not None
    assert np.array_equal(np.concatenate(out[0]), _want(dec2, cb.done[0], fv, ref=v.ref_codes))
    cb.cstream.close()
