"""audio.Loudness on the GPU: a clip streamed in random push sizes over several rows equals oneshot() bit for bit; a row
saved mid-segment and loaded into another normaliser continues bit for bit; on 5 s of stationary noise and tones the
standard BS.1770 meter reads the output after its first 400 ms within 0.2 LU of the target; the gain holds through
digital silence."""
import numpy as np
import pytest

from tests import loudness_ref as LR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _loud(rows, max_in):
    from qwen3_tts_b200.audio import Loudness
    return Loudness(DEV, rows, max_in)


def _at(x, lufs):
    return (x * 10 ** ((lufs - LR.integrated(x)) / 20)).astype(np.float32)


def _noise(g, n):
    return g.standard_normal(n).astype(np.float32)


def _tone(n, f=440.0):
    return np.sin(2 * np.pi * f * np.arange(n) / 24000).astype(np.float32)


def test_stream_equals_oneshot_for_random_push_sizes():
    g = np.random.default_rng(0)
    N = 24000 * 4 + 777
    clips = [_at(_noise(g, N), -30.0), _at(_tone(N), -14.0), _at(_noise(g, N) * _tone(N, 2.0), -40.0)]
    targets = [-16.0, -23.0, -10.0]
    ld = _loud(3, 5000)
    try:
        ld.reset([0], targets[0])
        ld.reset([1], targets[1])
        ld.reset([2], targets[2])
        out = {r: [] for r in range(3)}
        pos = [0, 0, 0]
        while min(pos) < N:
            chunks = {}
            for r in range(3):
                c = min(int(g.integers(0, 7000)), N - pos[r])
                if c:
                    chunks[r] = clips[r][pos[r]:pos[r] + c]
                    pos[r] += c
            end = [r for r in range(3) if pos[r] == N and r in chunks]
            for r, y in ld.push(chunks, end=end).items():
                out[r].append(y)
        for r in range(3):
            want = ld.oneshot(clips[r], targets[r])
            assert want.dtype == np.float32 and want.shape == (N,)
            assert np.array_equal(np.concatenate(out[r]), want), r
    finally:
        ld.close()


def test_save_and_load_mid_segment_continue_bit_for_bit():
    g = np.random.default_rng(1)
    x = _at(_noise(g, 24000 * 2), -25.0)
    a, b = _loud(2, 4096), _loud(3, 4096)
    try:
        a.reset([1], -18.0)
        y = [a.push({1: x[:9000]})[1]]                  # 9000: 3 segments and 1800 inputs of the 4th
        state = a.save([1])
        b.reset([0, 1, 2], -30.0)
        b.push({2: x[:100]})
        b.load([2], state)
        for i in range(9000, len(x), 4096):
            y.append(b.push({2: x[i:i + 4096]})[2])
        assert np.array_equal(np.concatenate(y), a.oneshot(x, -18.0))
        with pytest.raises(ValueError):
            b.load([0], state[:, :100])
    finally:
        a.close()
        b.close()


@pytest.mark.parametrize("kind", ["noise", "tone"])
def test_the_meter_reads_the_target_after_400_ms(kind):
    g = np.random.default_rng(2)
    N = 24000 * 5
    base = _noise(g, N) if kind == "noise" else _tone(N, 997.0)
    levels, targets = (-50.0, -38.0, -26.0, -12.0), (-40.0, -31.0, -23.0, -16.0, -10.0)
    cases = [(lv, t) for lv in levels for t in targets if abs(t - lv) <= 30]   # the +-30 dB clamp bounds the gain
    ld = _loud(1, 1)                                   # oneshot() opens a row of its own
    try:
        checked = 0
        for i, (lv, t) in enumerate(cases):
            y = ld.oneshot(_at(base, lv), t)
            if np.abs(y).max() >= 10 ** (-1 / 20):      # the limiter's job: out of scope here
                continue
            got = LR.integrated(y[9600:])
            assert abs(got - t) <= 0.2, (kind, lv, t, got)
            checked += 1
        assert checked >= len(cases) // 2
    finally:
        ld.close()


def test_the_gain_holds_through_digital_silence():
    g = np.random.default_rng(4)
    x = _at(_noise(g, 24000 * 2), -30.0)
    clip = np.concatenate([x, np.zeros(24000 * 2, np.float32), x])
    ld = _loud(1, 2400)
    try:
        ld.reset([0], -16.0)
        A = []
        for s in range(len(clip) // 2400):
            ld.push({0: clip[s * 2400:(s + 1) * 2400]})
            A.append(ld.save([0])[0, 16:20].cpu().numpy().view(np.float32)[0])
        gap = A[20 + 3:40]                             # blocks wholly inside the gap: Ja does not change
        assert len(set(gap)) == 1 and gap[0] > 1
        assert abs(20 * np.log10(gap[0]) - 14.0) < 0.5
    finally:
        ld.close()
