"""Audio formats without a GPU: the resampler's count formulas against a brute-force restatement for every supported
pair, AudioFormat validation, the G.711 restatement against audioop, and the continuous batcher's format handling
(default sessions untouched, bad formats refused at submit, a final chunk for a request that ends without new frames,
park / resume / cancel carrying and dropping the row's state) against fake engines, codec and stages."""
import numpy as np
import pytest
import torch

from qwen3_tts_b200 import audio
from qwen3_tts_b200.config import SUPPORTED_RATES, AudioFormat, SamplingParams
from tests.fake_stages import install
from tests.test_scheduler_cpu import FakeEngine, _mock_sync
from tests.test_scheduler_park_cpu import H, UP, BankCodec, ParkingEngine

PAIRS = [(a, b) for a in SUPPORTED_RATES for b in SUPPORTED_RATES]


@pytest.mark.parametrize("sr_in,sr_out", PAIRS)
def test_count_formulas_against_brute_force(sr_in, sr_out):
    up, down = audio.ratio(sr_in, sr_out)
    hl = audio.half_len(up, down)
    ns = np.arange(0, 3001)
    j = np.arange(0, 6 * 3001 + 64)
    last_input = (hl + j * down) // up            # output j is emitted once this input has arrived
    E = np.searchsorted(last_input, ns - 1, side="right")
    N = np.searchsorted(j * down, ns * up, side="left")   # j with j*down < n*up: the clip's outputs
    assert all(audio.emitted(int(n), up, down) == E[n] for n in ns)
    assert all(audio.total(int(n), up, down) == N[n] for n in ns)
    assert (E <= N).all()
    # the earliest input of the first output not yet emitted lies within the native history (Q3_RESAMPLE_HIST = 128)
    first_in = np.maximum(0, -(-(j * down - hl) // up))
    assert (ns[ns > 0] - first_in[E[ns > 0]] <= 128).all()
    # one push of max_in inputs plus an end never exceeds the capacity the resampler is opened with
    for n0 in (0, 1, 57, 1000):
        for c in (0, 1, 7680):
            worst = audio.total(n0 + c, up, down) - audio.emitted(n0, up, down)
            assert worst <= audio.out_bound(7680, up, down)
    if up != down:
        from scipy.signal import resample_poly
        for n in (1, 2, 37, 1001):
            assert len(resample_poly(np.ones(n), up, down)) == audio.total(n, up, down)


def test_audio_format_validation():
    assert AudioFormat(8000, "ulaw").sample_rate == 8000
    assert AudioFormat(np.int64(16000)).sample_rate == 16000
    for bad in (12345, 0, 16000.0, "16000", True, None):
        with pytest.raises(ValueError):
            AudioFormat(bad)
    for bad in ("alaw", "mp3", "F32", None, 1):
        with pytest.raises(ValueError):
            AudioFormat(24000, bad)
    with pytest.raises(ValueError):
        audio.ratio(24000, 96000)


def _ulaw(s16):
    v = s16.astype(np.int32) >> 2
    mask = np.where(v < 0, 0x7F, 0xFF)
    v = np.minimum(np.abs(v), 8159) + 33
    seg = np.searchsorted(np.array([0x3F, 0x7F, 0xFF, 0x1FF, 0x3FF, 0x7FF, 0xFFF, 0x1FFF]), v)
    u = np.where(seg >= 8, 0x7F, (seg << 4) | ((v >> (seg + 1)) & 0xF))
    return (u ^ mask).astype(np.uint8)


def test_ulaw_restatement_equals_audioop_on_every_int16():
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        audioop = pytest.importorskip("audioop")
    x = np.arange(-32768, 32768, dtype=np.int16)
    want = np.frombuffer(audioop.lin2ulaw(x.tobytes(), 2), dtype=np.uint8)
    assert np.array_equal(_ulaw(x), want)


# ---------------------------------------------------------------------------------------------- the batcher
@pytest.fixture
def fakes(monkeypatch):
    return install(monkeypatch)


def _batcher(codec=True, eng=None, **kw):
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    eng = eng or ParkingEngine()
    cb = ContinuousBatcher(eng, torch.zeros(H), SamplingParams(max_new_tokens=21), n_slots=2, packet_frames=4,
                           max_trailing=32, codec=BankCodec() if codec else None, **kw)
    return eng, cb


def _drain(cb):
    out = {}
    for chunks, _ in cb.stream():
        for rid, a in chunks.items():
            out.setdefault(rid, []).append(a)
    return out


def _want(n_frames, fmt):
    up, down = audio.ratio(24000, fmt.sample_rate)
    n = audio.total(n_frames * UP, up, down)
    return (np.arange(n) % 251).astype({"f32": np.float32, "s16": np.int16, "ulaw": np.uint8}[fmt.encoding])


def test_session_without_formats_opens_no_resampler(monkeypatch, fakes):
    _mock_sync(monkeypatch)
    for kw in ({}, {"audio_format": AudioFormat(24000)}):
        eng, cb = _batcher(**kw)
        a = cb.submit(torch.zeros(4, H), torch.zeros(2, H), key=1, max_frames=6)
        b = cb.submit(torch.zeros(4, H), torch.zeros(2, H), key=2, max_frames=3, audio_format=AudioFormat(24000, "f32"))
        out = _drain(cb)
        assert cb.resampler is None and cb.stages == {} and all(f.made == [] for f in fakes.values())
        for rid, n in ((a, 6), (b, 3)):
            assert all(c.dtype == np.float32 and c.shape[0] > 0 for c in out[rid])
            assert np.concatenate(out[rid]).shape == (n * UP,)


def test_bad_formats_are_refused_at_submit(monkeypatch, fakes):
    _mock_sync(monkeypatch)
    eng, cb = _batcher()
    for bad in ("ulaw", 8000, (8000, "ulaw"), {"sample_rate": 8000}):
        with pytest.raises(ValueError):
            cb.submit(torch.zeros(4, H), audio_format=bad)
    assert not cb.pending
    with pytest.raises(ValueError):
        _batcher(audio_format="s16")
    eng, plain = _batcher(codec=False)
    with pytest.raises(ValueError):
        plain.submit(torch.zeros(4, H), audio_format=AudioFormat(8000))


def test_a_request_ending_without_new_frames_gets_its_tail(monkeypatch, fakes):
    _mock_sync(monkeypatch)
    # EOS right after the first packet: the next step has no new frame
    eng, cb = _batcher(eng=FakeEngine(eos_at={1: 4, 2: 4}))
    fmt = AudioFormat(8000, "ulaw")
    a = cb.submit(torch.zeros(4, H), key=1, max_frames=10, audio_format=fmt)
    b = cb.submit(torch.zeros(4, H), key=2, max_frames=10)
    steps = list(cb.stream())
    assert len(steps) == 2 and sorted(steps[1][1]) == [a, b]
    assert a in steps[1][0] and b not in steps[1][0]        # the default request gets no entry, as before
    got = np.concatenate([c[a] for c, _ in steps if a in c])
    assert np.array_equal(got, _want(4, fmt))
    res = fakes["Resampler"].made[0]
    assert res.log[-1] == ("push", {}, [0], True)
    assert cb.done[a].shape[0] == 4


def test_park_resume_and_cancel_carry_and_drop_the_resampler_state(monkeypatch, fakes):
    _mock_sync(monkeypatch)
    eng, cb = _batcher()
    fmt = AudioFormat(16000, "s16")
    a = cb.submit(torch.zeros(4, H), torch.zeros(20, H), key=1, max_frames=12, audio_format=fmt)
    c = cb.submit(torch.zeros(4, H), torch.zeros(20, H), key=2, max_frames=12, audio_format=AudioFormat(8000))
    out = {}
    for it, (chunks, _) in enumerate(cb.stream()):
        for rid, y in chunks.items():
            out.setdefault(rid, []).append(y)
        if it == 0:
            cb.park(a)
            cb.park(c)
        if it == 1:
            assert cb.parked[a].res_state is not None and cb.parked[c].res_state is not None
            rc = cb.parked[c]
            assert cb.cancel(c) and rc.res_state is None
            cb.resume(a)
    assert np.array_equal(np.concatenate(out[a]), _want(12, fmt))
    res = fakes["Resampler"].made[0]
    assert ("save", [0]) in res.log and ("save", [1]) in res.log and ("load", [0]) in res.log
    assert len([e for e in res.log if e[0] == "load"]) == 1       # the cancelled request's state was never loaded
    assert c not in cb.done
