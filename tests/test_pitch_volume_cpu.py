"""Pitch and volume without a GPU: AudioFormat's pitch / volume validation and the combined hop range; the pitch step
and hop rules (pitch 0 keeps today's hop at every speed); the pitched resampler filters' bounds for every pitch step and
rate; the limiter's counts and history bound against brute force on the reference (tests/limiter_ref.py) and the
reference's properties (ceiling, identity on quiet audio, the 119-sample delay, a loud tone settling at the ceiling);
the resampler's filter lifetime (drop the least recently used unused filter, re-add it on load) against a fake
library; and the continuous batcher's routing through the time-stretch, the limiter and the resampler against fakes."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from qwen3_tts_b200 import audio
from qwen3_tts_b200.config import SUPPORTED_RATES, AudioFormat
from tests import limiter_ref as LR
from tests.fake_stages import install
from tests.test_audio_format_cpu import _batcher, _drain
from tests.test_scheduler_cpu import FakeEngine, _mock_sync
from tests.test_scheduler_park_cpu import H, UP

TS = audio.TimeStretch
LIM = audio.Limiter


# ------------------------------------------------------------------------------------------------- AudioFormat
def test_audio_format_pitch_and_volume_validation():
    f = AudioFormat(24000)
    assert f.pitch == 0.0 and f.volume == 0.0 and f.pitch_step == 480 and f.hop == 480
    assert AudioFormat(8000, "ulaw", 1.25, 3, -6).volume == -6.0 and AudioFormat(24000, pitch=np.float32(2)).pitch == 2.0
    assert AudioFormat(24000, pitch=12).pitch_step == 960 and AudioFormat(24000, pitch=-12).pitch_step == 240
    assert AudioFormat(24000, volume=12).volume == 12 and AudioFormat(24000, volume=-30).volume == -30
    for bad in (-12.01, 12.01, float("nan"), float("inf"), -float("inf"), True, "1", None, 1j):
        with pytest.raises(ValueError):
            AudioFormat(24000, pitch=bad)
    for bad in (-30.01, 12.01, float("nan"), float("inf"), False, "0", None):
        with pytest.raises(ValueError):
            AudioFormat(24000, volume=bad)
    # speed / pitch factor outside [0.5, 2]: the hop leaves [240, 960]
    for speed, pitch in ((2.0, -12), (0.5, 12), (1.1, -12.0), (1.5, -7), (0.6, 5)):
        with pytest.raises(ValueError, match="pitch factor"):
            AudioFormat(24000, speed=speed, pitch=pitch)
    assert AudioFormat(24000, speed=2.0, pitch=12).hop == 480 and AudioFormat(24000, speed=0.5, pitch=-12).hop == 480


def test_pitch_step_and_hop_rules():
    for pitch in np.linspace(-12, 12, 2401):
        lp = AudioFormat(24000, pitch=float(pitch)).pitch_step
        assert lp == math.floor(480 * 2 ** (float(pitch) / 12) + 0.5) and 240 <= lp <= 960
        assert 50 * lp % 50 == 0 and 12000 <= 50 * lp <= 48000
    # 3.6 cents per step at pitch 0
    assert abs(1200 * math.log2(481 / 480) - 3.6) < 0.01
    g = np.random.default_rng(0)
    speeds = np.concatenate([np.linspace(0.5, 2.0, 30001), g.uniform(0.5, 2.0, 20000), (np.arange(240, 960) + 0.5) / 480])
    for s in speeds:
        s = float(s)
        assert AudioFormat(24000, speed=s).hop == int(np.floor(s * 480 + 0.5)) == TS.hop(s)   # today's hop
    for s, pitch in ((1.0, 3), (1.3, -7), (1.2, 10), (2.0, 11.99)):
        f = AudioFormat(24000, speed=s, pitch=pitch)
        assert f.hop == math.floor(s * 480 * 480 / f.pitch_step + 0.5) == TS.hop(s, pitch)
        assert abs(f.hop * f.pitch_step / 480 ** 2 - s) <= 480 / (2 * 480 ** 2) * 2 + 1e-12   # effective speed


def test_pitched_resampler_filters_fit_the_table_history_and_outputs():
    max_in = 4 * 1920
    cap = max(audio.out_bound(max_in, *audio.ratio(a, b)) for a in SUPPORTED_RATES for b in SUPPORTED_RATES)
    worst, reach, per_out, taps = (0, 0, 0), 0, 0, 0
    for lp in range(240, 961):
        for sr in SUPPORTED_RATES:
            up, down = audio.ratio(50 * lp, sr, pitched=True)
            hl = audio.half_len(up, down)
            worst = max(worst, (max(up, down), lp, sr))
            taps = max(taps, 2 * hl + 1)
            reach = max(reach, 2 * hl // up)
            per_out = max(per_out, -(-(2 * hl + 1) // up))
            for mi in (1, 7, 480, max_in):
                c = max(audio.out_bound(mi, *audio.ratio(a, b)) for a in SUPPORTED_RATES for b in SUPPORTED_RATES) \
                    if mi != max_in else cap
                assert audio.out_bound(mi, up, down) <= c, (lp, sr, mi)
    assert worst == (1916, 958, 11025) and taps == 38321 and taps * 4 < 150 * 1024
    assert per_out <= 121 and reach == 120 <= 128          # Q3_RESAMPLE_HIST
    assert audio.MAX_FILTERS * taps * 4 < 10 * 2 ** 20
    # only rates the resampler takes as input
    for bad in (12345, 11950, 48050, 8000 * 0 + 60000):
        with pytest.raises(ValueError):
            audio.ratio(bad, 24000, pitched=True)
    with pytest.raises(ValueError):
        audio.ratio(12050, 24000)                          # a pitched rate only where asked for
    with pytest.raises(ValueError):
        audio.ratio(24000, 12050, pitched=True)            # never as output


# ------------------------------------------------------------------------------------------------- limiter
def test_limiter_counts_and_history_bound_against_brute_force():
    assert LIM.DELAY == LR.DELAY == 119 and LR.REACH == 1438 < LIM.HIST == 1536
    for n in (0, 1, 118, 119, 120, 121, 5000):
        assert LIM.emitted(n) == LR.emitted(n) == max(0, n - 119) and LIM.total(n) == n
    # output n reads inputs [n - 1319, n + 119] exactly: perturb one input and see which outputs move
    g = np.random.default_rng(1)
    x = (g.uniform(-1, 1, 4000) * 0.6).astype(np.float32)
    x[1500:1510] *= 3
    gain = LR.gain(6.0)
    y = LR.limit(x, gain)
    for p in (0, 700, 2000, 3999):
        x2 = x.copy()
        x2[p] = np.float32(9.0)
        d = np.nonzero(LR.limit(x2, gain) != y)[0]
        assert d.min() >= p - 119 and d.max() <= p + 1319, p
    # on quiet audio the look-ahead reaches exactly 119 back
    q = (x * np.float32(0.1)).astype(np.float32)
    yq = LR.limit(q, gain)
    for p in (700, 2000):
        q2 = q.copy()
        q2[p] = np.float32(9.0)
        assert np.nonzero(LR.limit(q2, gain) != yq)[0].min() == p - 119
    # E(n): the outputs emitted after n inputs read none past them, so a prefix gives them bit for bit
    for n in (119, 120, 500, 1438, 1439, 3000):
        e = LR.emitted(n)
        assert np.array_equal(LR.limit(x[:n], gain)[:e], y[:e]), n
    # the first pending output after n inputs reads back 1438 inputs, which the 1536 kept hold
    for n in range(119, 6000):
        assert n - (LR.emitted(n) - 1319) <= LR.REACH <= LIM.HIST


def test_limiter_reference_properties():
    c = LR.C
    ulp2 = 2 * np.spacing(c)
    g = np.random.default_rng(2)
    # the ceiling on loud noise and impulses
    for vol in (12.0, 6.0, 0.0):
        x = g.uniform(-1, 1, 6000).astype(np.float32)
        x[1000] = 1.0
        x[3000:3003] = [-1.0, 1.0, -1.0]
        y = LR.limit(x, LR.gain(vol))
        assert y.shape == x.shape and np.abs(y).max() <= c + ulp2, vol
    # identity on quiet stretches: wherever a = 1 on [n - 1319, n + 119], y = u bit for bit
    x = (g.uniform(-1, 1, 8000) * 0.2).astype(np.float32)
    x[4000] = 0.99
    gain = LR.gain(3.0)
    y = LR.limit(x, gain)
    u = x * gain
    loud = np.nonzero(np.abs(u) > c)[0]
    assert loud.tolist() == [4000]
    quiet = [n for n in range(8000) if not (n - 1319 <= 4000 <= n + 119)]
    assert np.array_equal(y[quiet], u[quiet])
    # the 119-sample delay: the gain starts down exactly 119 samples before the peak
    assert np.array_equal(y[:4000 - 119], u[:4000 - 119]) and abs(y[4000 - 119]) < abs(u[4000 - 119])
    assert c * np.float32(1 - 1e-5) <= abs(y[4000]) <= c + ulp2
    # a tone pushed +12 dB settles with its peaks at c
    t = np.arange(24000)
    tone = (0.5 * np.sin(2 * np.pi * 200 * t / 24000)).astype(np.float32)
    y = LR.limit(tone, LR.gain(12.0))
    late = np.abs(y[6000:-2000])
    assert late.max() <= c + ulp2 and late.max() >= c * 0.999
    # below the ceiling a gain is just a gain
    y = LR.limit(tone, LR.gain(-6.0))
    assert np.array_equal(y, tone * LR.gain(-6.0))


# ------------------------------------------------------------------------------------------------- filter lifetime
class FakeLib:
    """q3_resample_* entries of a resampler table: ids are reused lowest first; drop refuses a filter a row uses."""

    def __init__(self, rows):
        self.ids, self.fid, self.log = {}, [-1] * rows, []

    def q3_resample_add_filter(self, h, up, down, taps, n, out):
        i = min(set(range(audio.MAX_FILTERS)) - set(self.ids))
        self.ids[i] = (up, down)
        out._obj.value = i
        self.log.append(("add", (up, down), i))
        return 0

    def q3_resample_drop_filter(self, h, i):
        assert i in self.ids and i not in self.fid, i
        self.log.append(("drop", self.ids.pop(i), i))
        return 0

    def q3_resample_reset_rows(self, h, n, rows, fids, encs):
        for k in range(n):
            assert fids[k] in self.ids
            self.fid[rows[k]] = fids[k]
        return 0

    def q3_resample_release_rows(self, h, n, rows):
        for k in range(n):
            self.fid[rows[k]] = -1
        return 0

    def q3_resample_save_rows(self, h, n, rows, dst, st):
        C.memset(dst, 0, n * audio.ROW_BYTES)      # filter id 0, encoding f32
        return 0

    def q3_resample_load_rows(self, h, n, rows, src, st):
        self.loaded = [C.c_int32.from_address(src + k * audio.ROW_BYTES).value for k in range(n)]
        for k in range(n):
            self.fid[rows[k]] = self.loaded[k]
        return 0


def _fake_resampler(monkeypatch, rows):
    monkeypatch.setattr(audio, "design", lambda up, down: np.ones(3))
    res = object.__new__(audio.Resampler)
    res.lib, res.device, res.rows, res.h = FakeLib(rows), torch.device("cpu"), rows, C.c_void_p(1)
    res._filters, res._pair, res._enc = {}, [None] * rows, [None] * rows
    res._stream = lambda: None
    return res


def test_filters_are_dropped_least_recently_used_first_and_re_added_on_load(monkeypatch):
    res = _fake_resampler(monkeypatch, 4)
    lib = res.lib
    fmts = [(50 * lp, AudioFormat(sr)) for lp in range(300, 320) for sr in (8000, 16000, 44100, 48000)]   # 80 pairs
    res.reset([0], *fmts[0])
    state = res.save([0])
    assert state.pairs == [audio.ratio(fmts[0][0], 8000, pitched=True)] and state.records.shape == (1, audio.ROW_BYTES)
    res.reset([1], *fmts[1])
    res.release([0])
    assert lib.fid[0] == -1 and res._pair[0] is None
    for rate, fmt in fmts[2:]:
        res.reset([2], rate, fmt)
    assert len(res._filters) == audio.MAX_FILTERS and len(lib.ids) == audio.MAX_FILTERS
    drops = [e for e in lib.log if e[0] == "drop"]
    assert len(drops) == len(fmts) - audio.MAX_FILTERS
    # row 1's pair is in use and never dropped; row 0's (released) pair went first
    p1 = audio.ratio(fmts[1][0], 16000, pitched=True)
    assert drops[0][1] == state.pairs[0] and all(d[1] != p1 for d in drops)
    assert lib.ids[lib.fid[1]] == p1
    # a dropped id is reused by the next add
    adds = [e for e in lib.log if e[0] == "add"]
    assert adds[audio.MAX_FILTERS][2] == drops[0][2]
    # loading the saved row adds its filter again and writes the new id into the record's header
    n_add = len(adds)
    res.load([3], state)
    adds = [e for e in lib.log if e[0] == "add"]
    assert len(adds) == n_add + 1 and adds[-1][1] == state.pairs[0]
    assert res._pair[3] == state.pairs[0] and res._enc[3] == "f32" and lib.loaded == [adds[-1][2]]
    # every id on the table is live once; rows 1, 2, 3 use theirs
    assert sorted(res._filters.values()) == sorted(lib.ids) and all(lib.fid[r] in lib.ids for r in (1, 2, 3))
    # a state that is not a ResamplerState is refused
    with pytest.raises(ValueError):
        res.load([0], state.records)


def test_a_full_table_of_filters_in_use_is_refused(monkeypatch):
    res = _fake_resampler(monkeypatch, audio.MAX_FILTERS + 1)
    for r in range(audio.MAX_FILTERS):
        res.reset([r], 50 * (300 + r), AudioFormat(8000))
    with pytest.raises(RuntimeError, match="in use"):
        res.reset([audio.MAX_FILTERS], 50 * 900, AudioFormat(8000))


# ------------------------------------------------------------------------------------------------- the batcher
@pytest.fixture
def fakes(monkeypatch):
    return install(monkeypatch)


def _chain(n_frames, fmt):
    """The fakes' composition for a whole clip of n_frames frames: its output length and values."""
    n = n_frames * UP
    if fmt.hop != 480:
        n = TS.total(n, fmt.hop)
        y = (1000 + np.arange(n)).astype(np.float32)
    if fmt.volume != 0:
        y = (5000 + np.arange(n)).astype(np.float32)
    if fmt.pitch_step != 480 or fmt.sample_rate != 24000 or fmt.encoding != "f32":
        up, down = audio.ratio(50 * fmt.pitch_step, fmt.sample_rate, pitched=True)
        y = (np.arange(audio.total(n, up, down)) % 251).astype({"f32": np.float32, "s16": np.int16, "ulaw": np.uint8}[fmt.encoding])
    return y


def test_sessions_without_pitch_or_volume_open_no_limiter_and_reset_as_before(monkeypatch, fakes):
    _mock_sync(monkeypatch)
    fmts = (AudioFormat(8000, "ulaw", 1.25), AudioFormat(24000, speed=0.75), AudioFormat(16000, "s16"),
            AudioFormat(24000, pitch=0.001, volume=0.0))      # a pitch below half a step is no pitch
    eng, cb = _batcher()
    ids = [cb.submit(torch.zeros(4, H), key=i + 1, max_frames=6 + i, audio_format=f) for i, f in enumerate(fmts)]
    out = _drain(cb)
    assert cb.limiter is None and fakes["Limiter"].made == []
    st, res = fakes["TimeStretch"].made[0], fakes["Resampler"].made[0]
    assert all(len(e) == 3 for e in st.log if e[0] == "reset")          # reset(rows, speed), as before
    assert all(e[2] == 24000 for e in res.log if e[0] == "reset")       # resampled from 24 kHz, as before
    for rid, f in zip(ids, fmts):
        if f.hop == 480 and f.sample_rate == 24000:
            assert rid in out and out[rid][0].dtype == np.float32        # the codec's own audio
        else:
            assert np.array_equal(np.concatenate(out[rid]), _chain(cb.done[rid].shape[0], f)), f


def test_pitch_and_volume_route_through_stretch_limiter_and_resampler(monkeypatch, fakes):
    _mock_sync(monkeypatch)
    eng, cb = _batcher(eng=FakeEngine(eos_at={1: 9, 2: 5}))
    fa = AudioFormat(8000, "s16", 1.1, 3.0, -4.0)
    fb = AudioFormat(24000, pitch=-2.0)
    a = cb.submit(torch.zeros(4, H), key=1, max_frames=12, audio_format=fa)
    b = cb.submit(torch.zeros(4, H), key=2, max_frames=12, audio_format=fb)
    out = _drain(cb)
    st, lim, res = (fakes[n].made[0] for n in ("TimeStretch", "Limiter", "Resampler"))
    assert ("reset", [0], 1.1, 3.0) in st.log and ("reset", [1], 1.0, -2.0) in st.log
    assert lim.log[0] == ("reset", [0], -4.0)
    assert ("reset", [0], 50 * fa.pitch_step, AudioFormat(8000, "s16")) in res.log
    assert ("reset", [1], 50 * fb.pitch_step, AudioFormat(24000)) in res.log
    assert all(1 not in e[1] and 1 not in e[2] for e in lim.log if e[0] == "push")
    # the limiter took exactly the stretch's output of row 0 and the resampler exactly the limiter's; the ends came in
    # one step
    n_st = TS.total(9 * UP, fa.hop)
    assert sum(e[1].get(0, 0) for e in lim.log if e[0] == "push") == n_st
    assert sum(e[1].get(0, 0) for e in res.log if e[0] == "push") == n_st
    ends = [[i for i, e in enumerate(o.log) if e[0] == "push" and 0 in e[2]] for o in (st, lim, res)]
    assert all(len(e) == 1 for e in ends)
    assert all(e[3] is False for e in st.log + lim.log if e[0] == "push" and (0 in e[1] or 0 in e[2]))
    assert np.array_equal(np.concatenate(out[a]), _chain(9, fa))
    assert np.array_equal(np.concatenate(out[b]), _chain(5, fb))


def test_volume_alone_and_its_park_resume_and_cancel(monkeypatch, fakes):
    _mock_sync(monkeypatch)
    eng, cb = _batcher()
    fa, fc = AudioFormat(24000, volume=6.0), AudioFormat(16000, "ulaw", volume=-10.0)
    a = cb.submit(torch.zeros(4, H), torch.zeros(20, H), key=1, max_frames=12, audio_format=fa)
    c = cb.submit(torch.zeros(4, H), torch.zeros(20, H), key=2, max_frames=12, audio_format=fc)
    out = {}
    for it, (chunks, _) in enumerate(cb.stream()):
        for rid, y in chunks.items():
            out.setdefault(rid, []).append(y)
        if it == 0:
            cb.park(a)
            cb.park(c)
        if it == 1:
            assert cb.parked[a].lim_state is not None and cb.parked[c].lim_state is not None
            rc = cb.parked[c]
            assert cb.cancel(c) and rc.lim_state is None and rc.res_state is None
            cb.resume(a)
    assert fakes["TimeStretch"].made == []
    lim = fakes["Limiter"].made[0]
    assert ("save", [0]) in lim.log and ("save", [1]) in lim.log and ("load", [0]) in lim.log
    assert len([e for e in lim.log if e[0] == "load"]) == 1 and c not in cb.done
    # volume alone at 24 kHz f32 has no resampler row: its chunks are the limiter's, host arrays
    assert all(0 not in e[1] and 0 not in e[2] for e in fakes["Resampler"].made[0].log if e[0] == "push")
    assert all(y.dtype == np.float32 and isinstance(y, np.ndarray) for y in out[a])
    assert np.array_equal(np.concatenate(out[a]), _chain(12, fa))


def test_bad_pitch_or_volume_raise_at_submit(monkeypatch, fakes):
    _mock_sync(monkeypatch)
    eng, cb = _batcher()
    with pytest.raises(ValueError):
        cb.submit(torch.zeros(4, H), key=1, audio_format=AudioFormat(24000, pitch=13))
    with pytest.raises(ValueError):
        cb.submit(torch.zeros(4, H), key=1, audio_format=AudioFormat(24000, volume=20))
    with pytest.raises(ValueError):
        cb.submit(torch.zeros(4, H), key=1, audio_format=AudioFormat(24000, speed=2.0, pitch=-1))
    eng, cb = _batcher(codec=False)
    with pytest.raises(ValueError, match="codec"):
        cb.submit(torch.zeros(4, H), key=1, audio_format=AudioFormat(24000, volume=3))
    assert not cb.pending
