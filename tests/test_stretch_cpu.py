"""Speaking rate without a GPU: the time-stretch's count formulas and history bound against brute force for every
analysis hop, the output capacity, AudioFormat.speed validation, the reference being a time-stretch (a tone keeps its
pitch at every speed) and the continuous batcher's speed handling (no stretcher without speeds, a tail for a request
that ends without new frames, park / resume / cancel carrying and dropping the row's state, speed before a resampler)
against fake engines, codec and stages."""
import numpy as np
import pytest
import torch

from qwen3_tts_b200 import audio
from qwen3_tts_b200.config import AudioFormat
from tests import stretch_ref as S
from tests.fake_stages import install
from tests.test_audio_format_cpu import _batcher, _drain
from tests.test_scheduler_cpu import FakeEngine, _mock_sync
from tests.test_scheduler_park_cpu import H, UP

TS = audio.TimeStretch


def test_count_formulas_and_history_bound_against_brute_force():
    assert TS.hop(0.5) == 240 and TS.hop(2.0) == 960 and TS.hop(1.0) == 480 and TS.hop(1.25) == 600
    assert TS.hop(1.001) == 480 and TS.hop(1.0011) == 481
    ns = np.arange(0, 6001)
    for ha in range(240, 961):
        assert ha >= S.DELTA                      # the first search (k = 1) reads from ha - 240 >= 0
        k = np.arange(0, 6001 // 240 + 8)
        need = k * ha + S.DELTA + S.N - 1         # frame k reads inputs through need[k]
        frames = np.searchsorted(need, ns - 1, side="right")   # frames done after n inputs: need[k] <= n - 1
        E = np.array([TS.emitted(int(n), ha) for n in ns])
        M = np.array([TS.total(int(n), ha) for n in ns])
        assert np.array_equal(E, 480 * frames), ha
        assert np.array_equal(M, -(-ns * 480 // ha)), ha
        assert (E <= M).all()
        # an end emits up to frame ceil(M/480) - 1, whose reads end below n + 1199 (the kernel's zero padding)
        K = -(-M // 480)
        last = np.where(K > 0, (K - 1) * ha + S.DELTA + S.N - 1, -1)
        assert (last <= ns + 1198).all(), ha
        # the earliest input the next frame may read (its search or the previous frame's second half) lies within
        # the 2048 inputs a row keeps: n - earliest < 2*240 + 960 + max(0, ha - 480) <= 1920
        f = frames[ns > 0]
        p_low = np.maximum(0, (f - 1) * ha - S.DELTA)          # the lowest position the last frame done may have
        earliest = np.where(f == 0, 0, np.minimum(p_low + S.HS, f * ha - S.DELTA))
        span = ns[ns > 0] - earliest
        assert span.max() < 2 * S.DELTA + S.N + max(0, ha - S.HS) <= 1920 < TS.HIST, ha
        assert all(TS.emitted(int(n), ha) == S.emitted(int(n), ha) for n in (0, 1199, 1200, 1200 + ha, 5000))


def test_one_push_and_its_end_never_exceed_out_bound():
    for ha in (240, 241, 359, 480, 481, 600, 959, 960):
        for max_in in (1, 7, 480, 7680):
            bound = TS.out_bound(max_in, ha)
            assert bound <= TS.out_bound(max_in)          # the slowest speed is the widest
            worst = max(TS.total(n0 + c, ha) - TS.emitted(n0, ha)
                        for n0 in range(0, 1200 + 2 * ha + 3) for c in (0, 1, max_in // 2, max_in))
            assert worst <= bound, (ha, max_in, worst, bound)


def test_audio_format_speed_validation():
    assert AudioFormat(24000).speed == 1.0 and AudioFormat(8000, "ulaw", 1.25).speed == 1.25
    assert AudioFormat(24000, speed=np.float32(0.75)).speed == 0.75 and AudioFormat(24000, speed=2).speed == 2.0
    assert AudioFormat(24000) == AudioFormat(24000, "f32", 1.0)
    for bad in (0.49, 2.01, 0, -1.0, float("nan"), float("inf"), True, "1.2", None, 1 + 0j):
        with pytest.raises(ValueError):
            AudioFormat(24000, speed=bad)
    with pytest.raises(ValueError):
        TS.hop(3.0)


@pytest.mark.parametrize("speed", [0.5, 0.8, 1.3, 2.0])
def test_reference_stretches_a_tone_and_keeps_its_pitch(speed):
    ha = S.hop(speed)
    n = 24000
    tone = np.sin(2 * np.pi * 200 * np.arange(n) / 24000).astype(np.float32)   # a 120-sample period
    y, p, _ = S.stretch(tone, ha)
    assert y.shape == (TS.total(n, ha),)
    # every chosen frame lies a whole number of periods from its nominal continuation, so the tone goes on unbroken:
    # away from the end (where the zeros past the clip come in) y is the same tone, not a resampled one
    m = (len(p) - 4) * 480
    want = np.sin(2 * np.pi * 200 * np.arange(m) / 24000)
    assert m > 4800 and np.abs(y[:m] - want).max() <= 1e-5, (speed, np.abs(y[:m] - want).max())
    # and the clip's duration changed by the speed
    assert abs(len(y) / n - 480 / ha) < 1e-3


# ---------------------------------------------------------------------------------------------- the batcher
@pytest.fixture
def fakes(monkeypatch):
    return install(monkeypatch)


def _want(n_frames, speed):
    return (1000 + np.arange(TS.total(n_frames * UP, TS.hop(speed)))).astype(np.float32)


def test_no_stretcher_without_speeds(monkeypatch, fakes):
    _mock_sync(monkeypatch)
    for fmt in (None, AudioFormat(24000), AudioFormat(24000, speed=1.0005), AudioFormat(8000, "ulaw")):
        eng, cb = _batcher(audio_format=fmt)
        a = cb.submit(torch.zeros(4, H), torch.zeros(2, H), key=1, max_frames=6)
        _drain(cb)
        assert cb.stretcher is None and fakes["TimeStretch"].made == [] and cb.done[a].shape[0] == 6


def test_a_request_ending_without_new_frames_gets_its_tail(monkeypatch, fakes):
    _mock_sync(monkeypatch)
    eng, cb = _batcher(eng=FakeEngine(eos_at={1: 4, 2: 4}))
    a = cb.submit(torch.zeros(4, H), key=1, max_frames=10, audio_format=AudioFormat(24000, speed=0.75))
    b = cb.submit(torch.zeros(4, H), key=2, max_frames=10)
    steps = list(cb.stream())
    assert len(steps) == 2 and sorted(steps[1][1]) == [a, b]
    assert a in steps[1][0] and b not in steps[1][0]
    got = np.concatenate([c[a] for c, _ in steps if a in c])
    assert got.dtype == np.float32 and np.array_equal(got, _want(4, 0.75))
    st = fakes["TimeStretch"].made[0]
    assert st.log[0] == ("reset", [0], 0.75) and st.log[-1] == ("push", {}, [0], True)
    assert fakes["Resampler"].made == []             # 24 kHz f32: no resampler row


def test_park_resume_and_cancel_carry_and_drop_the_stretch_state(monkeypatch, fakes):
    _mock_sync(monkeypatch)
    eng, cb = _batcher()
    a = cb.submit(torch.zeros(4, H), torch.zeros(20, H), key=1, max_frames=12, audio_format=AudioFormat(24000, speed=1.5))
    c = cb.submit(torch.zeros(4, H), torch.zeros(20, H), key=2, max_frames=12, audio_format=AudioFormat(24000, speed=0.6))
    out = {}
    for it, (chunks, _) in enumerate(cb.stream()):
        for rid, y in chunks.items():
            out.setdefault(rid, []).append(y)
        if it == 0:
            cb.park(a)
            cb.park(c)
        if it == 1:
            assert cb.parked[a].st_state is not None and cb.parked[c].st_state is not None
            rc = cb.parked[c]
            assert cb.cancel(c) and rc.st_state is None
            cb.resume(a)
    assert np.array_equal(np.concatenate(out[a]), _want(12, 1.5))
    st = fakes["TimeStretch"].made[0]
    assert ("save", [0]) in st.log and ("save", [1]) in st.log and ("load", [0]) in st.log
    assert len([e for e in st.log if e[0] == "load"]) == 1
    assert c not in cb.done


def test_speed_composes_with_a_resampled_format(monkeypatch, fakes):
    _mock_sync(monkeypatch)
    eng, cb = _batcher(eng=FakeEngine(eos_at={1: 8}))
    fmt = AudioFormat(8000, "s16", 1.25)
    a = cb.submit(torch.zeros(4, H), key=1, max_frames=10, audio_format=fmt)
    b = cb.submit(torch.zeros(4, H), key=2, max_frames=6, audio_format=AudioFormat(16000, "ulaw"))
    out = _drain(cb)
    st, res = fakes["TimeStretch"].made[0], fakes["Resampler"].made[0]
    assert st.log[0] == ("reset", [0], 1.25)
    assert ("reset", [0], 24000, AudioFormat(8000, "s16")) in res.log      # the resampler converts rate and encoding only
    # the stretched samples go into the resampler: its row 0 took exactly the stretch's outputs, and its end came in
    # the step the stretch's tail did
    n_st = TS.total(8 * UP, TS.hop(1.25))
    assert sum(e[1].get(0, 0) for e in res.log if e[0] == "push") == n_st
    ends = [i for i, e in enumerate(res.log) if e[0] == "push" and 0 in e[2]]
    assert len(ends) == 1 and all(e[3] is False for e in st.log if e[0] == "push" and (e[1].get(0) or 0 in e[2]))
    up, down = audio.ratio(24000, 8000)
    want = (np.arange(audio.total(n_st, up, down)) % 251).astype(np.int16)
    assert np.array_equal(np.concatenate(out[a]), want)
    # the resample-only request is untouched by the stretch
    upb, downb = audio.ratio(24000, 16000)
    assert np.array_equal(np.concatenate(out[b]), (np.arange(audio.total(6 * UP, upb, downb)) % 251).astype(np.uint8))
    assert all(1 not in e[1] and 1 not in e[2] for e in st.log if e[0] == "push")
