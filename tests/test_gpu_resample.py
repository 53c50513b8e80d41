"""Streaming resampler (q3_resample_*, audio.Resampler): the one-shot conversion matches scipy.signal.resample_poly in
fp64 for every supported rate to and from 24 kHz; ragged pushes of several rows with different pairs and encodings
sharing each launch, then end, equal the one-shot bit for bit; the encodings equal numpy's of the f32 result; a saved
row continues in another row, and a reset row starts clean."""
import numpy as np
import pytest
import torch
from scipy.signal import resample_poly

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RATES = (8000, 11025, 16000, 22050, 32000, 44100, 48000)
PAIRS = [(r, 24000) for r in RATES] + [(24000, r) for r in RATES] + [(24000, 24000)]


def _noise(n, seed):
    return np.random.default_rng(seed).uniform(-1, 1, n).astype(np.float32)


def _chirp(n, sr):
    t = np.arange(n) / sr
    return (0.9 * np.sin(2 * np.pi * (50 * t + 0.5 * (sr / 2 - 50) / t[-1] * t * t))).astype(np.float32)


def _s16(y):
    return np.clip(np.rint(y.astype(np.float32) * np.float32(32768)), -32768, 32767).astype(np.int16)


def _ulaw(s16):
    """audioop.lin2ulaw(..., 2) restated (tests/test_audio_format_cpu.py checks it against audioop)."""
    v = s16.astype(np.int32) >> 2
    mask = np.where(v < 0, 0x7F, 0xFF)
    v = np.minimum(np.abs(v), 8159) + 33
    seg = np.searchsorted(np.array([0x3F, 0x7F, 0xFF, 0x1FF, 0x3FF, 0x7FF, 0xFFF, 0x1FFF]), v)
    u = np.where(seg >= 8, 0x7F, (seg << 4) | ((v >> (seg + 1)) & 0xF))
    return (u ^ mask).astype(np.uint8)


def _res(rows=1, max_in=4096):
    from qwen3_tts_b200.audio import Resampler
    return Resampler(DEV, rows, max_in)


@pytest.mark.parametrize("sr_in,sr_out", PAIRS)
def test_oneshot_matches_resample_poly(sr_in, sr_out):
    from qwen3_tts_b200 import audio
    from qwen3_tts_b200.config import AudioFormat
    up, down = audio.ratio(sr_in, sr_out)
    res = _res()
    for n, x in ((sr_in // 10 + 3, _noise(sr_in // 10 + 3, sr_in)), (sr_in // 5, _chirp(sr_in // 5, sr_in)), (1, _noise(1, 1))):
        y = res.oneshot(x, sr_in, AudioFormat(sr_out))
        ref = resample_poly(x.astype(np.float64), up, down) if up != down else x.astype(np.float64)
        assert y.dtype == np.float32 and y.shape == (-(-n * up // down),) == ref.shape
        assert np.abs(y - ref).max() <= 1e-5, (sr_in, sr_out, n, np.abs(y - ref).max())
    res.close()


def test_ragged_rows_in_shared_launches_equal_oneshot_bit_for_bit():
    from qwen3_tts_b200.config import AudioFormat
    rows = [(24000, AudioFormat(8000, "ulaw")), (24000, AudioFormat(44100, "s16")), (16000, AudioFormat(24000)),
            (24000, AudioFormat(48000)), (11025, AudioFormat(24000, "s16")), (48000, AudioFormat(24000, "ulaw")),
            (24000, AudioFormat(24000, "s16"))]
    sizes = [0, 1, 7, 300, 0, 1, 5000, 2, 64, 999]
    res = _res(len(rows), max_in=1024)      # pushes longer than max_in take several launches
    for r, (sr, fmt) in enumerate(rows):
        res.reset([r], sr, fmt)
    R = len(rows)
    clips = [_noise(3000 + 1777 * r, r) for r in range(R)]
    plans = []                           # row r's pushes: the sizes cycled from offset r
    for r in range(R):
        cuts, i, k = [], 0, r
        while i < len(clips[r]):
            n = sizes[k % len(sizes)]
            cuts.append(clips[r][i: i + n])
            i, k = i + n, k + 1
        plans.append(cuts)
    # row r starts at step r; odd rows end in the launch of their last push, even rows one step later without input
    last = [r + len(plans[r]) - (r % 2) for r in range(R)]
    got = {r: [] for r in range(R)}
    for s in range(max(last) + 1):
        chunks = {r: plans[r][s - r] for r in range(R) if 0 <= s - r < len(plans[r])}
        out = res.push(chunks, end=[r for r in range(R) if last[r] == s])
        for r, y in out.items():
            got[r].append(y)
    for r, (sr, fmt) in enumerate(rows):
        ref = res.oneshot(clips[r], sr, fmt)
        y = np.concatenate(got[r])
        assert y.dtype == ref.dtype and np.array_equal(y, ref), (r, y.shape, ref.shape)
        if fmt.encoding != "f32":
            f = res.oneshot(clips[r], sr, AudioFormat(fmt.sample_rate))
            want = _s16(f) if fmt.encoding == "s16" else _ulaw(_s16(f))
            assert np.array_equal(ref, want), (r, fmt)
    res.close()


def test_device_push_equals_host_push():
    from qwen3_tts_b200.config import AudioFormat
    res = _res(2, 512)
    x = _noise(2000, 9)
    res.reset([0, 1], 24000, AudioFormat(16000, "s16"))
    a = res.push({0: x[:900]})[0]
    b = res.push_device({1: torch.from_numpy(x[:900]).to(DEV)})[1].cpu().numpy()
    assert a.dtype == np.int16 and np.array_equal(a, b)
    res.close()


def test_saved_row_continues_in_another_row_and_reset_row_starts_clean():
    from qwen3_tts_b200.config import AudioFormat
    fmt = AudioFormat(8000, "f32")
    res = _res(3, 2048)
    x, z = _noise(5000, 1), _noise(3000, 2)
    ref = res.oneshot(x, 24000, fmt)
    res.reset([0, 2], 24000, fmt)
    a = [res.push({0: x[:2111]})[0]]
    state = res.save([0])
    res.push({0: z[:1500]})            # row 0 goes on with something else
    res.load([1], state)               # row 1 continues row 0's clip
    b = res.push({1: x[2111:]}, end=[1])[1]
    assert np.array_equal(np.concatenate(a + [b]), ref)
    res.reset([0], 24000, fmt)          # a reset row starts clean
    c = res.push({0: x}, end=[0])[0]
    assert np.array_equal(c, ref)
    first = res.push({2: z[:100]})[2]   # row 2 was untouched by all of it
    assert np.array_equal(np.concatenate([first, res.push({2: z[100:]}, end=[2])[2]]), res.oneshot(z, 24000, fmt))
    res.close()


def test_bad_arguments_are_refused():
    from qwen3_tts_b200.config import AudioFormat
    res = _res(2, 64)
    with pytest.raises(ValueError):
        res.push({0: _noise(10, 0)})    # never reset
    res.reset([0], 24000, AudioFormat(8000))
    with pytest.raises(ValueError):
        res.push({2: _noise(10, 0)})    # no such row
    with pytest.raises(ValueError):
        res.reset([1], 12345, AudioFormat(8000))
    with pytest.raises(ValueError):
        res.push({0: np.arange(10)})    # integer samples
    res.close()
