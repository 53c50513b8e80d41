"""Loudness targets in the continuous batcher: in a session mixing the default format, loudness -16, loudness -23 at
speed 1.25, 8 kHz mu-law and volume -3, each shaped request's concatenated stream() chunks equal
Resampler.oneshot(Limiter.oneshot(Loudness.oneshot(TimeStretch.oneshot(w, speed, pitch), target), volume), 50*Lp, its
rate and encoding) bit for bit, the other requests stream exactly what they stream in the same session without the
loudness requests, and a loudness request parked and resumed mid-segment streams what it streams never parked."""
import numpy as np
import pytest

from tests.test_gpu_scheduler_audio_format import _model, _sp, _want as _decoded

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _fmts():
    from qwen3_tts_b200 import AudioFormat
    return [None, AudioFormat(24000, loudness=-16.0), AudioFormat(24000, speed=1.25, loudness=-23.0),
            AudioFormat(8000, "ulaw"), AudioFormat(24000, volume=-3.0)]


def _run(fmts, keep=range(5), park=None):
    """The requests `keep` of five through two slots (some submitted while the session runs); `park`: (rid, step to park
    at, step to resume at).  Returns (batcher, {rid: concatenated chunks})."""
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    eng, dec, embs, trail, pad = _model()
    horizons = [6, 20, 16, 5, 12]
    cb = ContinuousBatcher(eng, pad, _sp(), n_slots=2, packet_frames=4, codec=dec)

    def sub(i):
        if i in keep:
            cb.submit(embs[i], trail[i], key=i, max_frames=horizons[i], audio_format=fmts[i])
    sub(1)
    sub(0)
    out = {}
    for it, (chunks, _) in enumerate(cb.stream()):
        for rid, a in chunks.items():
            out.setdefault(rid, []).append(a)
        if it == 0:
            sub(2)
            sub(3)
        if it == 1:
            sub(4)
        if park is not None and it == park[1]:
            cb.park(park[0])
        if park is not None and it == park[2]:
            cb.resume(park[0])
    return cb, {rid: np.concatenate(v) for rid, v in out.items()}


def _want(dec, codes, fmt):
    from qwen3_tts_b200 import AudioFormat
    from qwen3_tts_b200.audio import Limiter, Loudness, Resampler, TimeStretch
    ts, ld, lim, res = TimeStretch(DEV, 1, 8192), Loudness(DEV, 1, 64), Limiter(DEV, 1, 64), Resampler(DEV, 1, 64)
    try:
        y = _decoded(res, dec, codes, None)
        if fmt is None:
            return y
        if fmt.hop != 480:
            y = ts.oneshot(y, fmt.speed, fmt.pitch)
        if fmt.loudness is not None:
            y = ld.oneshot(y, fmt.loudness)
        if fmt.volume != 0 or fmt.loudness is not None:
            y = lim.oneshot(y, fmt.volume)
        out = AudioFormat(fmt.sample_rate, fmt.encoding)
        if fmt.pitch_step != 480 or out != AudioFormat(24000):
            y = res.oneshot(y, 50 * fmt.pitch_step, out)
        return y
    finally:
        for o in (ts, ld, lim, res):
            o.close()


def test_mixed_session_streams_each_requests_composition_and_leaves_the_others_alone():
    eng, dec, *_ = _model()
    fmts = _fmts()
    cb, out = _run(fmts)
    assert cb.loudness is not None and cb.limiter is not None
    for i, fmt in enumerate(fmts):
        assert cb.done[i].shape[0] > 0, i
        want = _want(dec, cb.done[i], fmt)
        assert out[i].dtype == want.dtype and np.array_equal(out[i], want), (i, fmt, out[i].shape, want.shape)
    assert any(out[i].shape[0] > 2400 * 2 for i in (1, 2))     # a measured gain was applied
    cb2, out2 = _run(fmts, keep=(0, 3, 4))
    assert cb2.loudness is None
    for i in (0, 3, 4):
        assert np.array_equal(out2[i], out[i]), i


def test_a_loudness_request_parked_mid_segment_streams_what_it_streams_never_parked():
    fmts = _fmts()
    _, ref = _run(fmts)
    cb, got = _run(fmts, park=(1, 0, 2))      # parked after one 4-frame packet: 7680 samples, mid-segment
    assert [m[:2] for m in cb.moves] == [("park", 1), ("resume", 1)], cb.moves
    for i in range(5):
        assert np.array_equal(got[i], ref[i]), i
