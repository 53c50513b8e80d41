"""Audio formats in the continuous batcher: every request's concatenated stream() chunks equal Resampler.oneshot of the
one-shot decode of its codes, in its own rate and encoding, while requests of mixed formats share the session's slots;
default-format requests stream exactly what a session without formats streams; a voice-clone request and a parked and
resumed request stream in their formats exactly what they stream otherwise."""
import numpy as np
import pytest
import torch

from tests.test_gpu_scheduler import _setup
from tests.test_gpu_scheduler_audio import _codec

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
UP = 1920
_M = []


def _model():
    """The batcher audio test's talker (EOS made likely, so some requests leave at EOS) and codec, built once."""
    if not _M:
        from qwen3_tts_b200.engine import AREngine
        from oracle import talker as OT
        from tests import helpers as Hh
        cfg, eng, embs, trail, pad = _setup()
        eng.close()
        W = OT.random_weights(cfg, seed=3)
        W["talker.codec_head.weight"][cfg.codec_eos_token_id] *= 30.0
        Wb, _ = Hh.bf16_weights(W)
        eng = AREngine(Hh.to_pkg_cfg(cfg), Wb, device=DEV, max_batch=4, max_ctx=160)
        _M.append((eng, _codec(), embs, trail, pad))
    return _M[0]


def _sp():
    import qwen3_tts_b200 as q
    return q.SamplingParams(do_sample=True, subtalker_dosample=True, top_k=50, temperature=0.9, subtalker_top_k=50,
                            subtalker_temperature=0.9, repetition_penalty=1.05, max_new_tokens=21, suppress_eos=False,
                            min_new_tokens=4, seed=5)


def _fmts():
    from qwen3_tts_b200 import AudioFormat
    return [None, AudioFormat(16000, "s16"), AudioFormat(8000, "ulaw"), AudioFormat(48000, "f32"), AudioFormat(22050, "s16")]


def _run(fmts, park=None, **kw):
    """Five requests through two slots (three submitted while the session runs); `park`: (rid, step to park at, step
    to resume at).  Returns (batcher, {rid: [chunks]})."""
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    eng, dec, embs, trail, pad = _model()
    horizons = [20, 3, 20, 2, 16]
    cb = ContinuousBatcher(eng, pad, _sp(), n_slots=2, packet_frames=4, codec=dec, **kw)
    sub = lambda i: cb.submit(embs[i], trail[i], key=i, max_frames=horizons[i], audio_format=fmts[i])  # noqa: E731
    sub(0)
    sub(1)
    out = {}
    for it, (chunks, finished) in enumerate(cb.stream()):
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


def _want(res, dec, codes, fmt, ref=None):
    full = codes if ref is None else torch.cat([ref.to(codes.device), codes])
    wav = dec.forward(full.T[None].to(DEV))[0, 0].cpu().numpy()[(0 if ref is None else ref.shape[0] * UP):]
    return wav if fmt is None else res.oneshot(wav, 24000, fmt)


def test_mixed_formats_stream_the_oneshot_conversion_of_each_request():
    from qwen3_tts_b200.audio import Resampler
    eng, dec, *_ = _model()
    fmts = _fmts()
    cb, out = _run(fmts)
    lens = [cb.done[i].shape[0] for i in range(5)]
    assert any(n < h for n, h in zip(lens, [20, 3, 20, 2, 16])) and any(n == h for n, h in zip(lens, [20, 3, 20, 2, 16])), lens
    res = Resampler(DEV, 1, 64)
    dtypes = {None: np.float32, "f32": np.float32, "s16": np.int16, "ulaw": np.uint8}
    for i, fmt in enumerate(fmts):
        assert all(a.dtype == dtypes[fmt and fmt.encoding] for a in out.get(i, []))
        got = np.concatenate(out[i]) if i in out else np.zeros(0, dtypes[fmt and fmt.encoding])
        want = _want(res, dec, cb.done[i], fmt) if lens[i] else np.zeros(0, got.dtype)
        assert got.dtype == want.dtype and np.array_equal(got, want), (i, fmt, got.shape, want.shape)
    assert cb.resampler is not None
    # the default-format request streams exactly what a session without formats streams
    plain, pout = _run([None] * 5)
    assert plain.resampler is None
    assert len(out[0]) == len(pout[0]) and all(np.array_equal(a, b) for a, b in zip(out[0], pout[0]))
    # a session default applies to requests submitted without a format
    from qwen3_tts_b200 import AudioFormat
    dflt, dout = _run([None] * 5, audio_format=AudioFormat(8000, "ulaw"))
    assert np.array_equal(np.concatenate(dout[2]), np.concatenate(out[2]))
    res.close()


def test_parked_request_streams_in_its_format_what_it_streams_never_parked():
    fmts = _fmts()
    fmts[0] = fmts[2]                  # request 0 (8 kHz mu-law) is parked after its first packet, resumed two steps later
    _, ref = _run(fmts)
    cb, got = _run(fmts, park=(0, 0, 2))
    assert [m[:2] for m in cb.moves] == [("park", 0), ("resume", 0)], cb.moves
    for i in range(5):
        a = np.concatenate(got[i]) if i in got else None
        b = np.concatenate(ref[i]) if i in ref else None
        assert (a is None and b is None) or np.array_equal(a, b), i


def test_voice_clone_request_streams_its_generated_part_in_its_format():
    from qwen3_tts_b200 import AudioFormat
    from qwen3_tts_b200.audio import Resampler
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    eng, dec, embs, trail, pad = _model()
    g = torch.Generator().manual_seed(7)
    ref_codes = torch.randint(0, dec.cfg.codebook_size, (6, dec.cfg.num_quantizers), generator=g)
    fmt = AudioFormat(16000, "s16")
    cb = ContinuousBatcher(eng, pad, _sp(), n_slots=2, packet_frames=4, codec=dec)
    cb.submit(embs[0], trail[0], key=0, max_frames=12, ref_codes=ref_codes, audio_format=fmt)
    cb.submit(embs[1], trail[1], key=1, max_frames=9, audio_format=AudioFormat(8000, "ulaw"))
    out = {}
    for chunks, _ in cb.stream():
        for rid, a in chunks.items():
            out.setdefault(rid, []).append(a)
    res = Resampler(DEV, 1, 64)
    assert np.array_equal(np.concatenate(out[0]), _want(res, dec, cb.done[0], fmt, ref=ref_codes))
    assert np.array_equal(np.concatenate(out[1]), _want(res, dec, cb.done[1], AudioFormat(8000, "ulaw")))
    res.close()


def test_bad_format_is_refused_at_submit():
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    eng, dec, embs, trail, pad = _model()
    cb = ContinuousBatcher(eng, pad, _sp(), n_slots=2, packet_frames=4, codec=dec)
    with pytest.raises(ValueError):
        cb.submit(embs[0], trail[0], audio_format="ulaw")
    assert not cb.pending
