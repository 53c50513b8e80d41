"""Pitch and volume on the GPU: audio.Limiter's ragged multi-row pushes equal its one-shot and the numpy restatement
(tests/limiter_ref.py) bit for bit, a saved row continues in another row, bad arguments are refused; pitch-shifted
tones come out at 200*Lp/480 Hz with the lengths the counts predict, streamed through TimeStretch and Resampler equal to
the one-shot composition; a resampler serving many more (pitch, rate) pairs than its table holds reuses filter ids and
still converts every pair exactly."""
import numpy as np
import pytest
import torch

from tests import limiter_ref as LR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _noise(n, seed, amp=1.0):
    return (np.random.default_rng(seed).uniform(-1, 1, n) * amp).astype(np.float32)


def _push_all(obj, clips, sizes):
    """Push clips {row: samples} in ragged pieces (piece k of row r has sizes[(r + k) % len]), every row in each push,
    then end them; returns {row: concatenated output}."""
    pos = {r: 0 for r in clips}
    out = {r: [] for r in clips}
    k = 0
    while any(pos[r] < len(clips[r]) for r in clips):
        chunks = {}
        for r in clips:
            n = sizes[(r + k) % len(sizes)]
            chunks[r] = clips[r][pos[r]:pos[r] + n]
            pos[r] += len(chunks[r])
        for r, y in obj.push(chunks).items():
            out[r].append(y)
        k += 1
    for r, y in obj.push({}, end=sorted(clips)).items():
        out[r].append(y)
    return {r: np.concatenate(v) for r, v in out.items()}


def test_limiter_ragged_rows_equal_oneshot_and_the_reference():
    from qwen3_tts_b200.audio import Limiter
    vols = [12.0, 6.0, 0.5, -3.0, -30.0]
    R = len(vols)
    lim = Limiter(DEV, R, 700)                 # pushes longer than max_in take several launches
    clips = {}
    for r, v in enumerate(vols):
        lim.reset([r], v)
        x = _noise(2500 + 1311 * r, r, 0.4)
        x[np.random.default_rng(10 + r).integers(0, len(x), 5)] = 0.98
        clips[r] = x
    got = _push_all(lim, clips, [0, 1, 7, 119, 120, 300, 0, 1500, 256, 2])
    for r, v in enumerate(vols):
        one = lim.oneshot(clips[r], v)
        assert np.array_equal(one, LR.limit(clips[r], LR.gain(v))), v
        assert got[r].shape == clips[r].shape and np.array_equal(got[r], one), v
        assert np.abs(got[r]).max() <= LR.C + 2 * np.spacing(LR.C)
    # a device push equals a host push
    lim.reset([0, 1], 6.0)
    a = lim.push({0: clips[0][:900]})[0]
    b = lim.push_device({1: torch.from_numpy(clips[0][:900]).to(DEV)})[1].cpu().numpy()
    assert a.shape == (900 - 119,) and np.array_equal(a, b)
    lim.close()


def test_limiter_saved_row_continues_in_another_row_and_bad_arguments_are_refused():
    from qwen3_tts_b200.audio import Limiter
    lim = Limiter(DEV, 3, 2048)
    x = _noise(6000, 1, 0.7)
    ref = lim.oneshot(x, 9.0)
    lim.reset([0, 2], 9.0)
    a = [lim.push({0: x[:2111]})[0]]
    state = lim.save([0])
    assert state.shape == (1, Limiter.ROW_BYTES)
    lim.push({0: _noise(1500, 2)})             # row 0 goes on with something else
    lim.load([1], state)
    b = lim.push({1: x[2111:]}, end=[1])[1]
    assert np.array_equal(np.concatenate(a + [b]), ref)
    lim.reset([0], 9.0)
    assert np.array_equal(lim.push({0: x}, end=[0])[0], ref)
    for bad in (lambda: lim.reset([0], 13.0), lambda: lim.reset([0], float("nan")), lambda: lim.reset([3], 0.0),
                lambda: lim.push({1: np.arange(10)}), lambda: lim.load([0, 1], state)):
        with pytest.raises(ValueError):
            bad()
    fresh = Limiter(DEV, 2, 64)
    with pytest.raises(ValueError):
        fresh.push({0: x[:10]})                 # never reset
    with pytest.raises(RuntimeError):
        fresh.load([0], torch.zeros(1, Limiter.ROW_BYTES, dtype=torch.uint8, device=DEV))   # gain 0: not a record
    fresh.close()
    lim.close()


def _freq(y, rate):
    """The dominant frequency of y, by a parabolic peak fit on a Hann-windowed spectrum."""
    y = np.asarray(y, np.float64)
    w = np.hanning(len(y))
    s = np.abs(np.fft.rfft(y * w, 8 * len(y)))
    k = int(np.argmax(s[1:])) + 1
    a, b, c = np.log(s[k - 1:k + 2])
    return (k + 0.5 * (a - c) / (a - 2 * b + c)) * rate / (8 * len(y))


@pytest.mark.parametrize("pitch", [12, -12, 3, -7])
def test_pitch_shifts_a_tone_and_streams_the_oneshot_composition(pitch):
    from qwen3_tts_b200 import AudioFormat
    from qwen3_tts_b200.audio import Resampler, TimeStretch, total
    from qwen3_tts_b200.audio import ratio as pair
    fmt = AudioFormat(24000, pitch=pitch)
    lp, ha = fmt.pitch_step, fmt.hop
    n = 48000
    tone = (0.5 * np.sin(2 * np.pi * 200 * np.arange(n) / 24000)).astype(np.float32)
    ts, res = TimeStretch(DEV, 2, 4096), Resampler(DEV, 2, 4096)
    st = ts.oneshot(tone, 1.0, pitch)
    y = res.oneshot(st, 50 * lp, AudioFormat(24000))
    up, down = pair(50 * lp, 24000, pitched=True)
    assert st.shape == (TimeStretch.total(n, ha),) and y.shape == (total(st.shape[0], up, down),)
    # the duration is kept (effective speed ha*lp/480^2) and the tone moved to 200*lp/480 Hz
    assert abs(len(y) / n - 480 ** 2 / (ha * lp)) < 1e-3
    mid = y[len(y) // 4: 3 * len(y) // 4]
    f = _freq(mid, 24000)
    assert abs(f / (200 * lp / 480) - 1) < 0.005, (pitch, f)
    # streamed in ragged pieces through both stages equals the one-shot composition
    ts.reset([1], 1.0, pitch)
    res.reset([1], 50 * lp, AudioFormat(24000))
    out, i, k = [], 0, 0
    sizes = [1, 3000, 480, 7, 2500, 960]
    while i < n:
        c = sizes[k % len(sizes)]
        s = ts.push({1: tone[i:i + c]})[1]
        out.append(res.push({1: s})[1])
        i, k = i + c, k + 1
    out.append(res.push({1: ts.push({}, end=[1])[1]}, end=[1])[1])
    assert np.array_equal(np.concatenate(out), y)
    ts.close()
    res.close()


def test_many_pitch_and_rate_pairs_reuse_the_filter_table():
    from qwen3_tts_b200 import AudioFormat
    from qwen3_tts_b200.audio import MAX_FILTERS, Resampler, ratio
    rates = (8000, 16000, 44100, 48000)
    pitches = np.linspace(-11, 11, 21)
    pairs = [(50 * AudioFormat(24000, pitch=float(p)).pitch_step, AudioFormat(sr, "s16"))
             for p in pitches for sr in rates]
    assert len({(a, f.sample_rate) for a, f in pairs}) > MAX_FILTERS
    res = Resampler(DEV, 3, 2048)
    x = _noise(3000, 5, 0.5)
    first = pairs[0]
    res.reset([2], *first)                       # row 2 starts a clip with the first pair and is parked mid-clip
    head = res.push({2: x[:1234]})[2]
    saved = res.save([2])
    res.release([2])                             # the row is parked: its filter may go
    for j, (rate, fmt) in enumerate(pairs):
        res.reset([j % 2], rate, fmt)
        got = res.push({j % 2: x}, end=[j % 2])[j % 2]
        if j % 9 == 0:
            assert np.array_equal(got, res.oneshot(x, rate, fmt)), (rate, fmt)
    assert len(res._filters) <= MAX_FILTERS
    # the parked row's pair was dropped by now; loading adds it again under its current id
    assert ratio(first[0], first[1].sample_rate, pitched=True) not in res._filters
    res.load([0], saved)
    tail = res.push({0: x[1234:]}, end=[0])[0]
    assert np.array_equal(np.concatenate([head, tail]), res.oneshot(x, *first))
    res.close()
