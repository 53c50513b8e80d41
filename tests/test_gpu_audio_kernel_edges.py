"""The three streaming audio stages' kernels (resample_poly / resample_move, wsola / stretch_move, limit / limit_move)
run directly through their shims (tests/csrc/{resample,stretch,limit}_shim.cu) at the edges the per-kernel tests leave
open, against an fp64 polyphase sum, tests/stretch_ref.py and tests/limiter_ref.py:

A. every launch with poison in what it must not read or write: each row's input past its count and rows without a
   job, the history half a launch writes, history before a clip's first sample, outputs past each row's count up to
   the row stride; ended clips of 0, 1 and about kStPad samples, rows resumed at their deepest read, idle rows, all
   shared.  The poison is a NaN with a payload, except in the limiter's inputs and histories: a NaN drops out of its
   window minima (fminf) exactly as the zero it stands for, so those hold +-64, which |g*x| > c at every gain makes
   audible;
B. every real resampler filter (every supported pair, the pitched pairs of whole semitones, the pitched pairs that
   maximise the history reach, hl, up and down) through full 64-entry filter tables, each resumed at its deepest read
   and ended; the one-shot of each of those pairs against scipy.signal.resample_poly;
C. the s16 and mu-law epilogues on every int16 value, every half-way value and its fp32 neighbours, and clamp values;
D. counters past 2^31 and 2^32: a row shifted by a whole period equals its unshifted twin bit for bit;
E. launch limits: a 32768-sample stretch push, 4096 resampler rows that fill each row's output stride to its last
   byte, limiter rows whose only blocks write history, next to many output tiles, with ceiling and subnormal inputs;
F. save / load records with NaN in every record byte and history half the call must not touch, headers past 2^32.

A NaN written by a kernel is the canonical 0x7fffffff; the poison carries a payload, so a poisoned value that is
still there afterwards was never written.  Sizes come from the C header and the kernels (tests/audio_shims.py)."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy.signal import resample_poly

from tests import audio_shims as A
from tests import limiter_ref as LR
from tests import stretch_ref as S
from tests.test_gpu_resample import _s16, _ulaw

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RH, SH, LH = A.RESAMPLE_HIST, A.STRETCH_HIST, A.LIMIT_HIST
ST_PAD, ST_MAX_IN = A.STRETCH_PAD, A.STRETCH_MAX_IN
POISON = 0x7FC0BEEF                   # a quiet NaN with a payload
POISON64 = 0x7FC0BEEF7FC0BEEF
LOUD = 64.0                           # the limiter's input poison: |g*x| > c at every gain, so a read changes its output
WIDTH = (4, 2, 1)                     # bytes per output of Q3_RESAMPLE_F32 / S16 / ULAW
U = 2.0 ** -24


@pytest.fixture(scope="module")
def shims(tmp_path_factory):
    return A.build(str(tmp_path_factory.mktemp("audio_shims")), ["resample_shim", "stretch_shim", "limit_shim"])


@pytest.fixture(scope="module")
def rlib(shims):
    return shims["resample_shim"]


@pytest.fixture(scope="module")
def slib(shims):
    return shims["stretch_shim"]


@pytest.fixture(scope="module")
def llib(shims):
    return shims["limit_shim"]


def _arr(t, xs):
    return (t * len(xs))(*xs)


def _poison(*shape) -> np.ndarray:
    return np.full(shape, POISON, np.uint32).view(np.float32)


def _dev(a) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _same(a, b) -> bool:
    """Bit for bit (NaN payloads included)."""
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def _loud(*shape) -> np.ndarray:
    """The limiter's input poison: +-LOUD alternating.  A NaN read by the limiter drops out of its window minima (fminf
    returns the other operand) and leaves the output as a zero would, so its inputs are poisoned with finite values."""
    return (LOUD * (1 - 2 * (np.arange(int(np.prod(shape))) % 2))).astype(np.float32).reshape(shape)


def _past(clip, n0, hist_len, fill=_poison) -> np.ndarray:
    """A row's current history after n0 inputs: clip[n0 - hist_len .. n0), poison (`fill`) before sample 0."""
    h = fill(hist_len)
    k = min(n0, hist_len)
    h[hist_len - k:] = clip[n0 - k:n0]
    return h


# ---------------------------------------------------------------- resampler

def _rcounts(n0, c, end, up, down, hl):
    """(out0, nout) of a row as q3_resample_step_rows computes them."""
    def e(n):
        return max(0, (n * up - 1 - hl) // down + 1)
    upto = -(-(n0 + c) * up // down) if end else e(n0 + c)
    return e(n0), upto - e(n0)


def _reach(up, down, hl, n0):
    """How far back the first output not yet emitted after n0 inputs reads."""
    j = max(0, (n0 * up - 1 - hl) // down + 1)
    c = hl + j * down
    return n0 - max(0, -(-(c - 2 * hl) // up))


def _deepest(up, down, hl):
    """The first n_in >= floor(2*hl/up) whose first pending output reads exactly floor(2*hl/up) back."""
    d = 2 * hl // up
    for n0 in range(max(d, 1), d + hl // up + down + 2):
        if _reach(up, down, hl, n0) == d:
            return n0
    raise AssertionError((up, down, hl))


def _poly_ref(h, up, down, hl, clip, j):
    """fp64 y[j] for the output indices j of clip (x = 0 past its end) through the taps h, and the error bound
    gamma_T * sum |x*h| of a sequential fp32 sum of its T products."""
    j = np.asarray(j, np.int64)
    if j.size == 0 or len(clip) == 0:
        return np.zeros(j.size), np.zeros(j.size)
    h, x = np.asarray(h, np.float64), np.asarray(clip, np.float64)
    c = hl + j * down
    m0 = np.maximum(0, -(-(c - 2 * hl) // up))
    m1 = np.minimum(c // up, len(x) - 1)
    T = max(1, int((m1 - m0 + 1).max()))
    m = m0[:, None] + np.arange(T)[None]
    ok = m <= m1[:, None]
    mm = np.where(ok, m, 0)
    p = np.where(ok, x[mm] * h[np.where(ok, c[:, None] - mm * up, 0)], 0.0)
    t = ok.sum(1)
    return p.sum(1), t * U / (1 - t * U) * np.abs(p).sum(1)


def _filters(pairs):
    """[(up, down, hl, fp32 taps)] designed as audio.Resampler designs them."""
    from qwen3_tts_b200 import audio
    return [(up, down, audio.half_len(up, down), audio.design(up, down).astype(np.float32)) for up, down in pairs]


def _res_launch(lib, filters, jobs, x, hist, cap, out_extra=0):
    """One resample_poly_kernel launch.  filters: [(up, down, hl, taps)]; jobs: per row (n_in, count, end, fid, enc,
    cur), counts as the host computes them; x fp32 [rows][ld]; hist fp32 [2][rows][128].  The outputs start poisoned
    ([rows][cap] bytes, then out_extra more).  Returns (outputs, next hist, [(out0, nout)])."""
    taps = _dev(np.concatenate([f[3] for f in filters]))
    offs = np.cumsum([0] + [len(f[3]) for f in filters])
    n_in, out0, fields, counts = [], [], [], []
    for n0, c, end, fid, enc, cur in jobs:
        up, down, hl, _ = filters[fid]
        e0, k = _rcounts(n0, c, end, up, down, hl)
        n_in.append(n0)
        out0.append(e0)
        fields += [c, k, int(end), fid, enc, cur]
        counts.append((e0, k))
        assert k * WIDTH[enc] <= cap
    R = len(jobs)
    out = _dev(_poison((R * cap + out_extra) // 4).view(np.uint8))
    xd, hd = _dev(x), _dev(hist)
    rc = lib.resample_shim_poly(len(filters), _arr(C.c_void_p, [taps.data_ptr() + 4 * int(o) for o in offs[:-1]]),
                                _arr(C.c_int, [f[0] for f in filters]), _arr(C.c_int, [f[1] for f in filters]),
                                _arr(C.c_int, [f[2] for f in filters]), R, _arr(C.c_longlong, n_in),
                                _arr(C.c_longlong, out0), _arr(C.c_int, fields), xd.data_ptr(), x.shape[1],
                                hd.data_ptr(), out.data_ptr(), cap)
    assert rc == 0
    return out.cpu().numpy(), hd.cpu().numpy(), counts


def _res_rows(rows, R, ld):
    """Buffers of a launch.  rows: {row: (fid, enc, n_in, count, end, cur, clip)}; the other rows have no job.
    Returns (x, hist, jobs) with everything a launch must not read poisoned."""
    x, hist, jobs = _poison(R, ld), _poison(2, R, RH), []
    for r in range(R):
        if r not in rows:
            jobs.append((0, 0, False, 0, 0, r % 2))
            continue
        fid, enc, n0, c, end, cur, clip = rows[r]
        hist[cur, r] = _past(clip, n0, RH)
        x[r, :c] = clip[n0:n0 + c]
        jobs.append((n0, c, end, fid, enc, cur))
    return x, hist, jobs


def _check_res(filters, rows, jobs, hist, o, hn, counts, cap):
    """Every row of a launch: outputs against fp64 in their encoding, poison past them, both history halves."""
    pois = _poison(cap // 4).view(np.uint8)
    for r, (n0, c, end, fid, enc, cur) in enumerate(jobs):
        e0, k = counts[r]
        nb = k * WIDTH[enc]
        assert _same(o[r * cap + nb:(r + 1) * cap], pois[nb:]), ("written past nout", r)
        assert _same(hn[cur, r], hist[cur, r]), ("current half", r)
        if r not in rows:
            assert nb == 0 and _same(hn[1 - cur, r], hist[1 - cur, r]), ("idle row", r)
            continue
        clip = rows[r][6]
        up, down, hl, h = filters[fid]
        want, bound = _poly_ref(h, up, down, hl, clip[:n0 + c], e0 + np.arange(k))
        got = o[r * cap:r * cap + nb]
        if enc == 0:
            y = got.view(np.float32)
            assert not np.isnan(y).any() and (np.abs(y - want) <= bound).all(), (r, np.abs(y - want).max(initial=0))
        else:
            lo, hi = _s16((want - bound).astype(np.float32)), _s16((want + bound).astype(np.float32))
            if enc == 1:
                g = got.view(np.int16)
                assert ((lo <= g) & (g <= hi)).all(), r
            else:
                assert ((got == _ulaw(lo)) | (got == _ulaw(hi))).all(), r
        nh = hn[1 - cur, r]
        if c == 0 and not end:
            assert _same(nh, hist[1 - cur, r]), ("idle row", r)
        elif end:
            assert _same(nh, np.zeros(RH, np.float32)), ("ended row", r)
        else:
            n1 = n0 + c
            want_h = np.array([clip[n1 - RH + i] if n1 - RH + i >= 0 else 0 for i in range(RH)], np.float32)
            assert _same(nh, want_h), ("next half", r)


def test_resampler_poisoned_buffers(rlib):
    from qwen3_tts_b200 import audio
    g = np.random.default_rng(0)
    pairs = [audio.ratio(24000, 8000), audio.ratio(16000, 24000), audio.ratio(24000, 44100), (1, 1),
             audio.ratio(48000, 8000)]
    F = _filters(pairs)
    specs = []   # (fid, enc, n_in, count, end)
    for fid, (up, down, hl, _) in enumerate(F):
        d = _deepest(up, down, hl)
        specs += [(fid, fid % 3, d, 300, False),          # resumed at its deepest read
                  (fid, (fid + 1) % 3, 0, 0, True),       # an ended clip of 0 samples
                  (fid, (fid + 2) % 3, 0, 1, True),       # of 1
                  (fid, 0, 0, 57, True),                  # a fresh clip ended in one launch
                  (fid, 1, d + 11, 0, True),              # resumed and ended with no new input
                  (fid, 2, 3, 5, False),                  # a short history
                  (fid, 0, 500, 0, False)]                # idle with a job entry
    R, ld, cap = len(specs) + 3, 400, 4 * 1100
    rows = {}
    for i, (fid, enc, n0, c, end) in enumerate(specs):
        r = i + 1                                         # rows 0, R - 2 and R - 1 have no job
        amp = 3.0 if enc else 1.0                         # past the s16 clamp
        rows[r] = (fid, enc, n0, c, end, r % 2, g.uniform(-amp, amp, n0 + c).astype(np.float32))
    x, hist, jobs = _res_rows(rows, R, ld)
    o, hn, counts = _res_launch(rlib, F, jobs, x, hist, cap)
    assert any(k > 0 for _, k in counts)
    _check_res(F, rows, jobs, hist, o, hn, counts, cap)


# ---------------------------------------------------------------- B: every kind of real filter

def _real_pairs():
    """{(up, down): (sr_in, sr_out)}: every supported pair, the pitched pairs 50*Lp -> rate at whole semitones, and
    the pitched pairs that maximise floor(2*hl/up), hl, up and down over every Lp x rate."""
    from qwen3_tts_b200 import audio
    from qwen3_tts_b200.config import SUPPORTED_RATES, AudioFormat
    out = {}
    for a in SUPPORTED_RATES:
        for b in SUPPORTED_RATES:
            out.setdefault(audio.ratio(a, b), (a, b))
    for b in SUPPORTED_RATES:
        for st in range(-12, 13):
            a = 50 * AudioFormat(b, pitch=st).pitch_step
            out.setdefault(audio.ratio(a, b, pitched=True), (a, b))
    every = [(audio.ratio(50 * lp, b, pitched=True), (50 * lp, b)) for lp in range(240, 961) for b in SUPPORTED_RATES]

    def key(p):
        up, down = p
        hl = audio.half_len(up, down)
        return 2 * hl // up, hl, up, down
    for i in range(4):
        top = max(key(p)[i] for p, _ in every)
        for p, sr in every:
            if key(p)[i] == top:
                out.setdefault(p, sr)
    return out


def test_every_real_filter_through_full_tables(rlib):
    pairs = _real_pairs()
    F = _filters(sorted(pairs))
    reach = [2 * hl // up for up, down, hl, _ in F]
    assert max(reach) == 120 <= RH and max(len(f[3]) for f in F) == 38321
    F += F[:-len(F) % 64]                                 # whole launches of 64 filters: id 63 is always used
    g = np.random.default_rng(1)
    ld, cap = 1024, 4 * 1024
    for b in range(0, len(F), 64):
        T = F[b:b + 64]
        rows = {}
        for fid, (up, down, hl, _) in enumerate(T):
            d = _deepest(up, down, hl)
            assert _reach(up, down, hl, d) == 2 * hl // up
            c = min(ld, max(16, -(-100 * down // up)))
            rows[2 * fid] = (fid, 0, d, c, False, fid % 2, g.uniform(-1, 1, d + c).astype(np.float32))
            n0 = d // 2 + 3
            rows[2 * fid + 1] = (fid, 0, n0, 37, True, 1 - fid % 2, g.uniform(-1, 1, n0 + 37).astype(np.float32))
        x, hist, jobs = _res_rows(rows, 128, ld)
        o, hn, counts = _res_launch(rlib, T, jobs, x, hist, cap)
        assert all(counts[2 * i][1] > 0 for i in range(64))
        _check_res(T, rows, jobs, hist, o, hn, counts, cap)


def test_oneshot_of_every_real_pair_matches_resample_poly():
    from qwen3_tts_b200.audio import Resampler
    from qwen3_tts_b200.config import AudioFormat
    res = Resampler(DEV, 1, 64)
    g = np.random.default_rng(2)
    try:
        for (up, down), (a, b) in sorted(_real_pairs().items()):
            for n in (a // 20 + 3, 1):
                x = g.uniform(-1, 1, n).astype(np.float32)
                y = res.oneshot(x, a, AudioFormat(b))
                ref = resample_poly(x.astype(np.float64), up, down) if up != down else x.astype(np.float64)
                assert y.dtype == np.float32 and y.shape == (-(-n * up // down),) == ref.shape, (a, b, n)
                assert np.abs(y - ref).max() <= 1e-5, (a, b, n, np.abs(y - ref).max())
    finally:
        res.close()


# ---------------------------------------------------------------- C: exhaustive encodings

def test_every_int16_and_half_way_value_through_the_copy_filter(rlib):
    half = ((np.arange(-32769, 32768) + 0.5) / 32768).astype(np.float32)
    assert np.array_equal(half.astype(np.float64) * 32768, np.arange(-32769, 32768) + 0.5)   # exact
    vals = np.concatenate([np.arange(-32768, 32768) / 32768, half, np.nextafter(half, np.float32(-np.inf)),
                           np.nextafter(half, np.float32(np.inf)),
                           np.array([2 ** 15 + 1, 2 ** 15 - 1, -2 ** 15 + 1, -2 ** 15 - 1, 2 ** 20, -2 ** 20]) / 32768])
    vals = vals.astype(np.float32)
    n = vals.size
    F = [(1, 1, 0, np.ones(1, np.float32))]
    x = np.stack([vals] * 3)
    hist = _poison(2, 3, RH)
    o, hn, counts = _res_launch(rlib, F, [(0, n, True, 0, enc, 0) for enc in range(3)], x, hist, 4 * n)
    assert [k for _, k in counts] == [n] * 3
    assert _same(o[:4 * n].view(np.float32), vals)
    s16 = np.clip(np.rint(vals.astype(np.float64) * 32768), -32768, 32767).astype(np.int16)
    got = o[4 * n:6 * n].view(np.int16)
    bad = np.flatnonzero(got != s16)
    assert bad.size == 0, (vals[bad[:5]] * 32768, got[bad[:5]], s16[bad[:5]])
    u = o[8 * n:9 * n]
    want = _ulaw(s16)
    assert np.array_equal(u, want) and np.unique(u).size == np.unique(_ulaw(np.arange(-32768, 32768))).size


# ---------------------------------------------------------------- D: counters past 2^31 and 2^32

def test_resampler_rows_shifted_past_2_32_equal_their_twins(rlib):
    from qwen3_tts_b200 import audio
    pairs = [(1, 1), audio.ratio(24000, 8000), audio.ratio(8000, 48000), audio.ratio(47950, 8000, pitched=True),
             audio.ratio(47900, 11025, pitched=True)]
    F = _filters(pairs)
    g = np.random.default_rng(3)
    x, hist = _poison(len(F) * 6, 512), _poison(2, len(F) * 6, RH)
    jobs, twins = [], []
    for fid, (up, down, hl, _) in enumerate(F):
        for end in (False, True):
            n0, c = 300 + fid, 400
            clip = g.uniform(-1.5, 1.5, n0 + c).astype(np.float32)
            base = len(jobs)
            for lim in (0, 2 ** 31, 2 ** 32):
                K = 0 if lim == 0 else lim // min(up, down) + 3
                m = n0 + K * down
                e0, k = _rcounts(m, c, end, up, down, hl)
                e00, k0 = _rcounts(n0, c, end, up, down, hl)
                assert (e0, k) == (audio.emitted(n0, up, down) + K * up, k0) == (e00 + K * up, k0)
                assert audio.total(m + c, up, down) == audio.total(n0 + c, up, down) + K * up
                assert min(m, e0) > lim
                r = len(jobs)
                hist[r % 2, r] = _past(clip, n0, RH)
                x[r, :c] = clip[n0:]
                jobs.append((m, c, end, fid, (fid + end) % 3, r % 2))
            twins.append(base)
    cap = 4 * 4096
    o, hn, counts = _res_launch(rlib, F, jobs, x, hist, cap)
    for b in twins:
        assert counts[b][1] > 0
        for r in (b + 1, b + 2):
            assert counts[r][1] == counts[b][1]
            assert _same(o[r * cap:(r + 1) * cap], o[b * cap:(b + 1) * cap]), (b, r)
            assert _same(hn[1 - r % 2, r], hn[1 - b % 2, b]), (b, r)


def test_stretch_rows_shifted_past_2_32_equal_their_twins(slib):
    g = np.random.default_rng(4)
    jobs, state, twins = [], [], []
    for ha in (240, 481, 960):
        for end in (False, True):
            n0, c = S.READY + 3 * ha - 1, 2500
            clip = (g.integers(-8, 9, n0 + c) / 16).astype(np.float32)
            f, pk, tail, hist = S.state_after(clip, n0, ha)
            assert f >= 1
            twins.append(len(jobs))
            for lim in (0, 2 ** 31, 2 ** 32):
                K = 0 if lim == 0 else lim // ha + 1
                m = n0 + K * ha
                assert S.frames_done(m, ha) == f + K and S.frames_done(m + c, ha) == S.frames_done(n0 + c, ha) + K
                assert S.emitted(m + c, ha) - S.emitted(m, ha) == S.emitted(n0 + c, ha) - S.emitted(n0, ha)
                assert S.total(m + c, ha) == S.total(n0 + c, ha) + 480 * K
                assert min(m, pk + K * ha) > lim
                jobs.append((len(jobs), m, c, end, ha))
                state.append((hist, tail, pk + K * ha, clip[n0:]))
    R = len(jobs)
    st = _StRows(R, 8192, 2500)
    for r, (hist, tail, p, xs) in enumerate(state):
        st.hist[r], st.tail[r], st.plast[r], st.x[r, :len(xs)] = hist, tail, p, xs
    o, nouts = st.launch(slib, jobs)
    for b, (_, n0, c, end, ha) in zip(twins, [jobs[t] for t in twins]):
        K = [0, 2 ** 31 // ha + 1, 2 ** 32 // ha + 1]
        assert nouts[b] > 0
        for i, r in ((1, b + 1), (2, b + 2)):
            assert nouts[r] == nouts[b] and _same(o[r], o[b]), (ha, end, r)
            assert _same(st.h[r], st.h[b]) and _same(st.t[r], st.t[b]), (ha, end, r)
            assert st.p[r] == st.p[b] + K[i] * ha, (ha, end, r)


def test_limiter_rows_shifted_past_2_32_equal_their_twins(llib):
    g = np.random.default_rng(5)
    rows, twins = [], []
    for n0, c, vol in ((LH, 700, 12.0), (LH + 17, 3000, -6.0), (5000, 300, 3.0)):
        for end in (False, True):
            clip = g.uniform(-1, 1, n0 + c).astype(np.float32)
            twins.append(len(rows))
            for lim in (0, 2 ** 31, 2 ** 32):
                K = 0 if lim == 0 else lim + 12345
                m = n0 + K
                assert LR.emitted(m) == LR.emitted(n0) + K and LR.emitted(m + c) - LR.emitted(m) == c
                assert min(m, LR.emitted(m)) > lim
                rows.append((m, c, end, LR.gain(vol), clip, n0))
    st = _LimRows(len(rows), 4096, 3008)
    for r, (m, c, end, gn, clip, n0) in enumerate(rows):
        st.set_row(r, r % 2, _past(clip, n0, LH, _loud), clip[n0:])
    o, hn, nouts = st.launch(llib, {r: (m, c, end, gn) for r, (m, c, end, gn, _, _) in enumerate(rows)})
    for b in twins:
        assert nouts[b] > 0
        for r in (b + 1, b + 2):
            assert nouts[r] == nouts[b] and _same(o[r], o[b]), r
            assert _same(hn[1 - r % 2, r], hn[1 - b % 2, b]), r


# ---------------------------------------------------------------- time-stretch

class _StRows:
    """Host images of `rows` stretch rows (history, tail, last frame position, inputs), all poisoned, and one
    launch: what comes back is in .h, .t, .p and the returned outputs."""

    def __init__(self, rows, cap, ld):
        self.rows, self.cap = rows, cap
        self.hist, self.tail = _poison(rows, SH), _poison(rows, 480)
        self.plast = np.full(rows, POISON64, np.uint64).view(np.int64)
        self.x = _poison(rows, ld)

    def launch(self, lib, jobs):
        """jobs: [(row, n_in, count, end, ha)]; counts as q3_stretch_step_rows computes them.  Returns (outputs fp32
        [rows][cap], {row: nout})."""
        n_in, f0, fields, nouts = [], [], [], {}
        self.jobs = {}
        for row, n0, c, end, ha in jobs:
            n = n0 + c
            a = S.frames_done(n0, ha)
            upto = S.total(n, ha) if end else S.emitted(n, ha)
            f1 = -(-upto // 480) if end else S.frames_done(n, ha)
            n_in.append(n0)
            f0.append(a)
            fields += [row, c, f1 - a, upto - 480 * a, int(end), ha]
            nouts[row] = upto - 480 * a
            self.jobs[row] = (a, f1)
            assert nouts[row] <= self.cap
        w = _dev(S.window32())
        xd, hd, td, pd = _dev(self.x), _dev(self.hist), _dev(self.tail), _dev(self.plast)
        out = _dev(_poison(self.rows, self.cap))
        rc = lib.stretch_shim_wsola(len(jobs), _arr(C.c_longlong, n_in), _arr(C.c_longlong, f0), _arr(C.c_int, fields),
                                    w.data_ptr(), xd.data_ptr(), self.x.shape[1], hd.data_ptr(), td.data_ptr(),
                                    pd.data_ptr(), out.data_ptr(), self.cap)
        assert rc == 0
        self.h, self.t, self.p = hd.cpu().numpy(), td.cpu().numpy(), pd.cpu().numpy()
        return out.cpu().numpy(), nouts


def _check_stretch(st, o, nouts, specs):
    """specs: {row: (ha, n0, count, end, clip)}; rows not in specs had no job."""
    w = S.window32()
    for r in range(st.rows):
        k = nouts.get(r, 0)
        assert _same(o[r, k:], _poison(st.cap - k)), ("written past nout", r)
        if r not in specs:
            assert _same(st.h[r], st.hist[r]) and _same(st.t[r], st.tail[r]) and st.p[r] == st.plast[r], r
            continue
        ha, n0, c, end, clip = specs[r]
        n = n0 + c
        y, p, _ = S.stretch(clip[:n], ha)
        assert not np.isnan(o[r, :k]).any() and np.array_equal(o[r, :k], y[S.emitted(n0, ha):S.emitted(n0, ha) + k]), (r, ha, n0, c)
        a, f1 = st.jobs[r]
        if end:          # an ended row writes none of its state
            assert _same(st.h[r], st.hist[r]) and _same(st.t[r], st.tail[r]) and st.p[r] == st.plast[r], r
            continue
        lo = max(0, SH - n)
        assert np.array_equal(st.h[r, lo:], clip[n - SH + lo:n]), r
        if f1 > a:
            pk = p[f1 - 1]
            assert st.p[r] == pk and np.array_equal(st.t[r], w[480:] * clip[pk + 480:pk + 960]), r
        else:
            assert _same(st.t[r], st.tail[r]) and st.p[r] == st.plast[r], r


def test_stretch_poisoned_buffers(slib):
    g = np.random.default_rng(6)
    specs = {}
    r = 1                                                     # row 0 and the last row have no job
    for ha in (240, 481, 960):
        for n in (0, 1, ST_PAD - 1, ST_PAD, ST_PAD + 1, 2 * ST_PAD + 1):
            specs[r] = (ha, 0, n, True, (g.integers(-8, 9, n) / 16).astype(np.float32))
            r += 1
        clip = (g.integers(-8, 9, 9000) / 16).astype(np.float32)
        d = S.READY + 3 * ha - 1                              # the next frame reads furthest back
        specs[r] = (ha, d, 2500, False, clip)
        specs[r + 1] = (ha, d, 1300, True, clip)
        specs[r + 2] = (ha, d + 1, ha - 1, False, clip)       # no frame completes: tail and p stay
        specs[r + 3] = (ha, 5000, 0, True, clip)              # ended with no new input
        r += 4
    R = r + 1
    st = _StRows(R, 8192, 2500 + ST_PAD + 8)
    for row, (ha, n0, c, end, clip) in specs.items():
        st.x[row, :c] = clip[n0:n0 + c]
        f, pk, tail, _ = S.state_after(clip, n0, ha)
        st.hist[row] = _past(clip, n0, SH)
        if f:
            st.tail[row], st.plast[row] = tail, pk
    o, nouts = st.launch(slib, [(row, n0, c, end, ha) for row, (ha, n0, c, end, _) in specs.items()])
    _check_stretch(st, o, nouts, specs)


@pytest.mark.parametrize("ha", [240, 960])
def test_stretch_push_of_max_in_samples(slib, ha):
    g = np.random.default_rng(ha)
    specs = {}
    d = S.READY + 3 * ha - 1
    for row, end in enumerate((False, True)):
        specs[row] = (ha, d, ST_MAX_IN, end, (g.integers(-8, 9, d + ST_MAX_IN) / 16).astype(np.float32))
    st = _StRows(2, -(-(ST_MAX_IN + ST_PAD - 1) * 480 // 240), ST_MAX_IN + ST_PAD + 8)
    for row, (_, n0, c, end, clip) in specs.items():
        f, pk, tail, _ = S.state_after(clip, n0, ha)
        st.hist[row], st.tail[row], st.plast[row], st.x[row, :c] = _past(clip, n0, SH), tail, pk, clip[n0:]
    o, nouts = st.launch(slib, [(row, n0, c, end, ha) for row, (_, n0, c, end, _) in specs.items()])
    assert nouts[1] > nouts[0] > 0
    _check_stretch(st, o, nouts, specs)


# ---------------------------------------------------------------- limiter

class _LimRows:
    """Host images of `rows` limiter rows (both history halves and inputs, all LOUD; set_row fills them) and one
    launch, whose outputs start as NaN poison."""

    def __init__(self, rows, cap, ld):
        self.rows, self.cap = rows, cap
        self.hist, self.x = _loud(2, rows, LH), _loud(rows, ld)
        self.cur = [0] * rows

    def set_row(self, r, cur, hist, xs):
        self.cur[r] = cur
        self.hist[cur, r] = hist
        self.x[r, :len(xs)] = xs

    def launch(self, lib, jobs):
        """jobs: {row: (n_in, count, end, gain)}, other rows idle; counts as q3_limit_step_rows computes them.
        Returns (outputs fp32 [rows][cap], next hist, {row: nout})."""
        n_in, out0, fields, gains, nouts = [], [], [], [], {}
        for r in range(self.rows):
            n0, c, end, gn = jobs.get(r, (0, 0, False, 1.0))
            nout = ((n0 + c) if end else LR.emitted(n0 + c)) - LR.emitted(n0) if (c or end) else 0
            n_in.append(n0)
            out0.append(LR.emitted(n0))
            fields += [c, nout, int(end), self.cur[r]]
            gains.append(float(gn))
            nouts[r] = nout
        xd, hd = _dev(self.x), _dev(self.hist)
        out = _dev(_poison(self.rows, self.cap))
        rc = lib.limit_shim_step(self.rows, _arr(C.c_longlong, n_in), _arr(C.c_longlong, out0), _arr(C.c_int, fields),
                                 _arr(C.c_float, gains), xd.data_ptr(), self.x.shape[1], hd.data_ptr(), out.data_ptr(),
                                 self.cap)
        assert rc == 0
        return out.cpu().numpy(), hd.cpu().numpy(), nouts


def _check_limit(st, o, hn, nouts, specs):
    """specs: {row: (n0, count, end, gain, clip)}; rows not in specs had no job."""
    for r in range(st.rows):
        k, cur = nouts[r], st.cur[r]
        assert _same(o[r, k:], _poison(st.cap - k)), ("written past nout", r)
        assert _same(hn[cur, r], st.hist[cur, r]), ("current half", r)
        if r not in specs:
            assert k == 0 and _same(hn[1 - cur, r], st.hist[1 - cur, r]), r
            continue
        n0, c, end, gn, clip = specs[r]
        n = n0 + c
        y = LR.limit(clip[:n], gn)
        e0 = LR.emitted(n0)
        assert not np.isnan(o[r, :k]).any() and _same(o[r, :k], y[e0:e0 + k]), (r, n0, c, end)
        if c == 0 or end:        # the other half is written only by a row that takes inputs and goes on
            assert _same(hn[1 - cur, r], st.hist[1 - cur, r]), r
        else:
            want = np.zeros(LH, np.float32)
            m = min(n, LH)
            want[LH - m:] = clip[n - m:n]
            assert _same(hn[1 - cur, r], want), ("next half", r)


def test_limiter_poisoned_buffers(llib):
    g = np.random.default_rng(7)
    specs = {}
    r = 1
    for n in (0, 1, 119, 120, 257, 1700):
        specs[r] = (0, n, True, LR.gain(9.0), (g.uniform(-1, 1, n)).astype(np.float32))
        r += 1
    clip = g.uniform(-1, 1, 9000).astype(np.float32)
    for n0, c, end in ((LR.REACH, 600, False), (LR.REACH, 600, True), (LH + 5, 1000, False), (3000, 0, True),
                       (40, 30, False), (4000, 0, False)):
        specs[r] = (n0, c, end, LR.gain(-6.0 if end else 12.0), clip)
        r += 1
    R = r + 1
    st = _LimRows(R, 2048, 1708)
    for row, (n0, c, end, gn, cl) in specs.items():
        st.set_row(row, row % 2, _past(cl, n0, LH, _loud), cl[n0:n0 + c])
    for row in range(R):
        if row not in specs:
            st.cur[row] = row % 2
    o, hn, nouts = st.launch(llib, {row: s[:4] for row, s in specs.items()})
    _check_limit(st, o, hn, nouts, specs)


def _ceiling_clip(g, n, gn):
    """Noise with inputs x where fl(g*x) is exactly the ceiling, their fp32 neighbours, and subnormals."""
    x = g.uniform(-0.6, 0.6, n).astype(np.float32)
    c = np.float32(LR.C / gn)
    assert np.float32(gn) * c == LR.C
    for i, p in enumerate(range(300, n - 300, 1000)):
        s = np.float32(1 if i % 2 else -1)
        x[p] = s * c
        x[p + 150] = s * np.nextafter(c, np.float32(np.inf))
        x[p + 400] = s * np.nextafter(c, np.float32(0))
    x[n // 3:n // 3 + 400] = (g.integers(-1000, 1000, 400) * np.float32(2.0 ** -149)).astype(np.float32)
    x[n // 2:n // 2 + 50] = np.float32(2.0 ** -130)
    assert (np.abs(x) < np.finfo(np.float32).tiny).sum() > 300
    return x


def test_limiter_history_only_rows_beside_many_tiles(llib):
    g = np.random.default_rng(8)
    lo, hi = LR.gain(-30.0), LR.gain(12.0)
    big = _ceiling_clip(g, 9000, hi)
    quiet = _ceiling_clip(g, 9000, lo)
    specs = {0: (0, 100, False, hi, big),                  # count > 0, no output: only history blocks
             1: (2000, 6000, False, hi, big),             # 24 output tiles
             2: (40, 60, False, lo, quiet),               # count > 0, no output, with a history
             3: (LH + 3, 5000, True, lo, quiet)}          # ended across 21 tiles
    st = _LimRows(5, 8192, 6008)
    for row, (n0, c, end, gn, cl) in specs.items():
        st.set_row(row, row % 2, _past(cl, n0, LH, _loud), cl[n0:n0 + c])
    o, hn, nouts = st.launch(llib, {row: s[:4] for row, s in specs.items()})
    assert nouts[0] == nouts[2] == 0 and min(nouts[1], nouts[3]) > 16 * 256
    _check_limit(st, o, hn, nouts, specs)
    # the same two history-only rows alone: a launch of history blocks only
    alone = {0: specs[0], 1: specs[2]}
    st = _LimRows(2, 256, 108)
    for row, (n0, c, end, gn, cl) in alone.items():
        st.set_row(row, 1 - row % 2, _past(cl, n0, LH, _loud), cl[n0:n0 + c])
    o, hn, nouts = st.launch(llib, {row: s[:4] for row, s in alone.items()})
    _check_limit(st, o, hn, nouts, alone)


# ---------------------------------------------------------------- E: resampler rows

def test_resampler_4096_rows_fill_their_outputs_to_the_last_byte(rlib):
    from qwen3_tts_b200 import audio
    F = _filters([(1, 1), audio.ratio(24000, 8000), audio.ratio(24000, 16000), audio.ratio(24000, 22050)])
    g = np.random.default_rng(9)
    R, ld, cap = 4096, 1664, 512
    rows = {}
    for r in range(R):
        fid, enc, end = r % 4, (r // 4) % 3, bool((r // 12) % 2)
        up, down, hl, _ = F[fid]
        n0 = int(g.integers(0, 300))
        e = _rcounts(n0, 0, False, up, down, hl)[0] + cap // WIDTH[enc] - 1   # the row's last output
        c = (e * down // up + 1 if end else -(-(e * down + 1 + hl) // up)) - n0
        assert 0 <= c < ld and _rcounts(n0, c, end, up, down, hl)[1] == cap // WIDTH[enc]
        rows[r] = (fid, enc, n0, c, end, r % 2, g.uniform(-1.2, 1.2, n0 + c).astype(np.float32))
    assert max(s[3] for s in rows.values()) < ld
    x, hist, jobs = _res_rows(rows, R, ld)
    o, hn, counts = _res_launch(rlib, F, jobs, x, hist, cap, out_extra=64)
    assert all(k * WIDTH[jobs[r][4]] == cap for r, (_, k) in enumerate(counts))
    assert _same(o[R * cap:], _poison(16)), "written past the last row"
    _check_res(F, rows, jobs, hist, o, hn, counts, cap)


# ---------------------------------------------------------------- F: move kernels

def test_resampler_move_with_poison(rlib):
    R = 6
    g = np.random.default_rng(10)
    hist = _poison(2, R, RH)
    cur = [1, 0, 1, 1, 0, 0]
    for r in range(R):
        hist[cur[r], r] = g.standard_normal(RH)
    rows, n_in = [4, 1, 2], [2 ** 32 + 5, 2 ** 40 + 3, 7]
    fids, encs = [63, 0, 17], [2, 0, 1]
    fields = sum(([0, 0, 0, fids[i], encs[i], cur[rows[i]]] for i in range(3)), [])
    rec = _dev(_poison(4, A.RESAMPLE_ROW_BYTES // 4).view(np.uint8))           # one record more than the call writes
    hd = _dev(hist)
    assert rlib.resample_shim_move(3, _arr(C.c_int, rows), _arr(C.c_longlong, n_in), _arr(C.c_int, fields),
                                   hd.data_ptr(), R, rec.data_ptr(), 0) == 0
    rc = rec.cpu().numpy()
    assert _same(hd.cpu().numpy(), hist)
    for i, r in enumerate(rows):
        assert rc[i, :8].view(np.int32).tolist() == [fids[i], encs[i]] and rc[i, 8:16].view(np.int64)[0] == n_in[i]
        assert _same(rc[i, 16:], hist[cur[r], r])
    assert _same(rc[3], _poison(A.RESAMPLE_ROW_BYTES // 4))
    # load records 0, 1, 2 into rows 0, 5, 3 (current halves 1, 0, 1): only those halves change
    dst, dcur = [0, 5, 3], [1, 0, 1]
    fields2 = sum(([0, 0, 0, 0, 0, dcur[i]] for i in range(3)), [])
    assert rlib.resample_shim_move(3, _arr(C.c_int, dst), _arr(C.c_longlong, [0] * 3), _arr(C.c_int, fields2),
                                   hd.data_ptr(), R, rec.data_ptr(), 1) == 0
    want = hist.copy()
    for i, r in enumerate(dst):
        want[dcur[i], r] = rc[i, 16:].view(np.float32)
    assert _same(hd.cpu().numpy(), want) and _same(rec.cpu().numpy(), rc)


def test_stretch_move_with_poison(slib):
    R = 5
    g = np.random.default_rng(11)
    hist, tail = g.standard_normal((R, SH)).astype(np.float32), g.standard_normal((R, 480)).astype(np.float32)
    plast = np.array([2 ** 33 + 1, 2 ** 40 + 9, POISON64, 5, 2 ** 32 + 480], np.int64)
    rows, n_in, f0, ha = [0, 1, 2], [2 ** 33 + 1200, 2 ** 41, 900], [2 ** 33 // 240, 2 ** 40 // 481, 0], [240, 481, 960]
    fields = sum(([rows[i], 0, 0, 0, 0, ha[i]] for i in range(3)), [])
    rec = _dev(_poison(4, A.STRETCH_ROW_BYTES // 4).view(np.uint8))
    hd, td, pd = _dev(hist), _dev(tail), _dev(plast)
    assert slib.stretch_shim_move(3, _arr(C.c_longlong, n_in), _arr(C.c_longlong, f0), _arr(C.c_int, fields),
                                  hd.data_ptr(), td.data_ptr(), pd.data_ptr(), rec.data_ptr(), 0) == 0
    rc = rec.cpu().numpy()
    assert _same(hd.cpu().numpy(), hist) and _same(td.cpu().numpy(), tail) and _same(pd.cpu().numpy(), plast)
    for i, r in enumerate(rows):
        assert rc[i, :8].view(np.int32).tolist() == [ha[i], 0]
        # a row with no frame done reads no p_last (row 2's is poison) and records 0
        assert rc[i, 8:32].view(np.int64).tolist() == [n_in[i], f0[i], int(plast[r]) if f0[i] else 0]
        assert _same(rc[i, 32:32 + 1920], tail[r]) and _same(rc[i, 32 + 1920:], hist[r])
    assert _same(rc[3], _poison(A.STRETCH_ROW_BYTES // 4))
    # load records 0 and 1 into rows 4 and 2 over poison: only those rows change
    hist[4], tail[4], hist[2], tail[2] = _poison(SH), _poison(480), _poison(SH), _poison(480)
    hd, td = _dev(hist), _dev(tail)
    fields2 = [4, 0, 0, 0, 0, 0, 2, 0, 0, 0, 0, 0]
    assert slib.stretch_shim_move(2, _arr(C.c_longlong, [0, 0]), _arr(C.c_longlong, [0, 0]), _arr(C.c_int, fields2),
                                  hd.data_ptr(), td.data_ptr(), pd.data_ptr(), rec.data_ptr(), 1) == 0
    wh, wt, wp = hist.copy(), tail.copy(), plast.copy()
    for i, r in ((0, 4), (1, 2)):
        wh[r], wt[r], wp[r] = rc[i, 32 + 1920:].view(np.float32), rc[i, 32:32 + 1920].view(np.float32), plast[rows[i]]
    assert _same(hd.cpu().numpy(), wh) and _same(td.cpu().numpy(), wt) and _same(pd.cpu().numpy(), wp)
    assert pd.cpu().numpy()[2] > 2 ** 32 and pd.cpu().numpy()[4] > 2 ** 32


def test_limiter_move_with_poison(llib):
    R = 6
    g = np.random.default_rng(12)
    hist = _poison(2, R, LH)
    cur = [0, 1, 1, 0, 1, 0]
    for r in range(R):
        hist[cur[r], r] = g.standard_normal(LH)
    rows, n_in, gains = [3, 0, 5], [2 ** 32 + 1, 2 ** 45 + 7, 1536], [LR.gain(12.0), LR.gain(-30.0), 1.0]
    fields = sum(([0, 0, 0, cur[rows[i]]] for i in range(3)), [])
    rec = _dev(_poison(4, A.LIMIT_ROW_BYTES // 4).view(np.uint8))
    hd = _dev(hist)
    assert llib.limit_shim_move(3, _arr(C.c_int, rows), _arr(C.c_longlong, n_in), _arr(C.c_int, fields),
                                _arr(C.c_float, [float(x) for x in gains]), hd.data_ptr(), R, rec.data_ptr(), 0) == 0
    rc = rec.cpu().numpy()
    assert _same(hd.cpu().numpy(), hist)
    for i, r in enumerate(rows):
        assert rc[i, :4].view(np.float32)[0] == gains[i] and rc[i, 4:8].view(np.int32)[0] == 0
        assert rc[i, 8:16].view(np.int64)[0] == n_in[i] and _same(rc[i, 16:], hist[cur[r], r])
    assert _same(rc[3], _poison(A.LIMIT_ROW_BYTES // 4))
    dst, dcur = [1, 4, 2], [0, 0, 1]
    fields2 = sum(([0, 0, 0, dcur[i]] for i in range(3)), [])
    assert llib.limit_shim_move(3, _arr(C.c_int, dst), _arr(C.c_longlong, [0] * 3), _arr(C.c_int, fields2),
                                _arr(C.c_float, [1.0] * 3), hd.data_ptr(), R, rec.data_ptr(), 1) == 0
    want = hist.copy()
    for i, r in enumerate(dst):
        want[dcur[i], r] = rc[i, 16:].view(np.float32)
    assert _same(hd.cpu().numpy(), want)
