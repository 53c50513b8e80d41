"""Streaming time-stretch (q3_stretch_*, audio.TimeStretch): ragged pushes of several rows with different speeds sharing
each launch, then ended, equal the one-shot bit for bit; the one-shot equals the fp32 reference; a device push equals
a host push; a saved row continues in another row and a reset row starts clean; bad arguments are refused before any
launch."""
import numpy as np
import pytest
import torch

from tests import stretch_ref as S

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _noise(n, seed):
    return np.random.default_rng(seed).uniform(-1, 1, n).astype(np.float32)


def _ts(rows=1, max_in=4096):
    from qwen3_tts_b200.audio import TimeStretch
    return TimeStretch(DEV, rows, max_in)


def test_ragged_rows_in_shared_launches_equal_oneshot_bit_for_bit():
    speeds = [0.5, 0.75, 1.001, 1.25, 1.5, 2.0, 0.9]
    sizes = [0, 1, 7, 300, 0, 1, 5000, 2, 1919, 999, 480]
    R = len(speeds)
    ts = _ts(R, max_in=1024)          # pushes longer than max_in take several launches
    for r, sp in enumerate(speeds):
        ts.reset([r], sp)
    clips = [_noise(3000 + 1777 * r, r) for r in range(R)]
    plans = []
    for r in range(R):
        cuts, i, k = [], 0, r
        while i < len(clips[r]):
            n = sizes[k % len(sizes)]
            cuts.append(clips[r][i: i + n])
            i, k = i + n, k + 1
        plans.append(cuts)
    last = [r + len(plans[r]) - (r % 2) for r in range(R)]
    got = {r: [] for r in range(R)}
    for s in range(max(last) + 1):
        chunks = {r: plans[r][s - r] for r in range(R) if 0 <= s - r < len(plans[r])}
        out = ts.push(chunks, end=[r for r in range(R) if last[r] == s])
        for r, y in out.items():
            got[r].append(y)
    for r, sp in enumerate(speeds):
        ref = ts.oneshot(clips[r], sp)
        y = np.concatenate(got[r])
        assert y.dtype == np.float32 and np.array_equal(y, ref), (r, y.shape, ref.shape)
        assert y.shape == (S.total(len(clips[r]), S.hop(sp)),)
    ts.close()


@pytest.mark.parametrize("speed", [0.5, 0.8, 1.3, 2.0])
def test_oneshot_equals_the_reference_and_keeps_a_tone(speed):
    ts = _ts()
    grid = (np.random.default_rng(3).integers(-8, 9, 7001) / 16).astype(np.float32)
    want, _, _ = S.stretch(grid, S.hop(speed))
    assert np.array_equal(ts.oneshot(grid, speed), want)
    tone = np.sin(2 * np.pi * 200 * np.arange(24000) / 24000).astype(np.float32)
    y = ts.oneshot(tone, speed)
    m = len(y) - 4 * 480
    assert np.abs(y[:m] - np.sin(2 * np.pi * 200 * np.arange(m) / 24000)).max() <= 1e-5
    ts.close()


def test_device_push_equals_host_push():
    ts = _ts(2, 512)
    x = _noise(4000, 9)
    ts.reset([0, 1], 1.25)
    a = ts.push({0: x[:3100]})[0]
    b = ts.push_device({1: torch.from_numpy(x[:3100]).to(DEV)})[1]
    assert isinstance(b, torch.Tensor) and b.is_cuda and a.dtype == np.float32 and np.array_equal(a, b.cpu().numpy())
    assert a.shape[0] > 0
    ts.close()


def test_saved_row_continues_in_another_row_and_reset_row_starts_clean():
    ts = _ts(3, 2048)
    x, z = _noise(9000, 1), _noise(5000, 2)
    ref = ts.oneshot(x, 0.7)
    ts.reset([0, 2], 0.7)
    a = [ts.push({0: x[:4111]})[0]]
    state = ts.save([0])
    ts.push({0: z[:1500]})           # row 0 goes on with something else
    ts.load([1], state)              # row 1 continues row 0's clip
    b = ts.push({1: x[4111:]}, end=[1])[1]
    assert np.array_equal(np.concatenate(a + [b]), ref)
    ts.reset([0], 0.7)
    assert np.array_equal(ts.push({0: x}, end=[0])[0], ref)
    first = ts.push({2: z[:100]})[2]   # row 2 was untouched by all of it
    assert np.array_equal(np.concatenate([first, ts.push({2: z[100:]}, end=[2])[2]]), ts.oneshot(z, 0.7))
    ts.close()


def test_bad_arguments_are_refused():
    ts = _ts(2, 64)
    with pytest.raises(ValueError):
        ts.push({0: _noise(10, 0)})     # never reset
    ts.reset([0], 1.5)
    with pytest.raises(ValueError):
        ts.push({2: _noise(10, 0)})     # no such row
    for bad in (0.4, 2.5, float("nan"), "1.0"):
        with pytest.raises(ValueError):
            ts.reset([1], bad)
    with pytest.raises(ValueError):
        ts.push({0: np.arange(10)})     # integer samples
    with pytest.raises(ValueError):
        ts.load([1], torch.zeros(1, 16, dtype=torch.uint8, device=DEV))
    with pytest.raises(ValueError):
        _ts(1, 1 << 20)                 # max_in beyond the native limit
    # natively: a hop outside [240, 960] and a count above max_in change nothing
    import ctypes as C
    lib = ts.lib
    assert lib.q3_stretch_reset_rows(ts.h, 1, (C.c_int32 * 1)(1), (C.c_int32 * 1)(239)) != 0
    n = (C.c_int32 * 2)()
    assert lib.q3_stretch_step_rows(ts.h, None, 0, (C.c_int32 * 2)(65, 0), (C.c_int32 * 2)(), None, n, None) != 0
    x = _noise(3000, 4)
    assert np.array_equal(np.concatenate([ts.push({0: x})[0], ts.push({}, end=[0])[0]]), ts.oneshot(x, 1.5))
    ts.close()
