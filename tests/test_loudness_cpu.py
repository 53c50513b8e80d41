"""CPU checks of the loudness target: the K-weighting against the BS.1770-4 table, the reference meter on a 997 Hz sine,
AudioFormat's loudness validation, the stage chains audio.stages gives, the counts and the record size against the C
header, the reference's properties, and the batcher's capacity check and routing with fakes."""
import os
import re

import numpy as np
import pytest
import torch

from qwen3_tts_b200 import audio
from qwen3_tts_b200.config import LOUDNESS_RANGE, AudioFormat
from tests import loudness_ref as LR
from tests.fake_stages import FakeStage, install
from tests.test_audio_format_cpu import _batcher, _drain
from tests.test_scheduler_cpu import _mock_sync
from tests.test_scheduler_park_cpu import H, UP

LD = audio.Loudness
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_k_weighting_reproduces_the_bs1770_table_at_48_khz():
    table = np.array([[1.53512485958697, -2.69169618940638, 1.19839281085285, 1.0, -1.69065929318241, 0.73248077421585],
                      [1.0, -2.0, 1.0, 1.0, -1.99004745483398, 0.99007225036621]])
    assert np.abs(LD.k_weighting(48000) - table).max() < 1e-8
    assert np.array_equal(LD.k_weighting(), LD.k_weighting(24000))
    assert np.abs(LD.k_weighting() - LR.sos(24000)).max() < 1e-15
    want24 = [[1.48790022, -2.24620547, 0.90490912, 1, -1.39023461, 0.53683848], [1, -2, 1, 1, -1.98014413, 0.98024282]]
    assert np.abs(LD.k_weighting() - np.array(want24)).max() < 1e-8


@pytest.mark.parametrize("fs,want", [(48000, -3.01), (24000, -2.98)])
def test_a_full_scale_997_hz_sine_measures_its_bs1770_loudness(fs, want):
    x = np.sin(2 * np.pi * 997 * np.arange(5 * fs) / fs)
    assert abs(LR.integrated(x, fs) - want) < 0.005


def test_audio_format_loudness_validation():
    assert AudioFormat(24000).loudness is None
    assert AudioFormat(24000, loudness=-16).loudness == -16.0
    for t in LOUDNESS_RANGE:
        assert AudioFormat(8000, "ulaw", loudness=t).loudness == t
    for bad in (-40.5, -9.9, float("nan"), float("inf"), True, "-16", [-16]):
        with pytest.raises(ValueError):
            AudioFormat(24000, loudness=bad)
    # existing formats compare and hash as before, and a target makes a format of its own
    assert AudioFormat(16000, "s16", 1.25) == AudioFormat(16000, "s16", 1.25, loudness=None)
    assert len({AudioFormat(16000, "s16"), AudioFormat(16000, "s16"), AudioFormat(16000, "s16", loudness=-16)}) == 2
    assert AudioFormat(24000, loudness=-16) != AudioFormat(24000, loudness=-23)


def test_stage_chains():
    assert audio.STAGES == ("TimeStretch", "Loudness", "Limiter", "Resampler")
    assert audio.stages(AudioFormat(24000)) == ()
    assert audio.stages(AudioFormat(24000, volume=-3)) == (("Limiter", (-3.0,)),)
    # a target always brings the limiter, at volume 0 too
    assert audio.stages(AudioFormat(24000, loudness=-16)) == (("Loudness", (-16.0,)), ("Limiter", (0.0,)))
    assert audio.stages(AudioFormat(8000, "ulaw", 1.25, volume=-2, loudness=-23)) == (
        ("TimeStretch", (1.25,)), ("Loudness", (-23.0,)), ("Limiter", (-2.0,)),
        ("Resampler", (24000, AudioFormat(8000, "ulaw"))))
    for f in (AudioFormat(16000, "s16", 0.8, 3.0, 6.0), AudioFormat(24000, pitch=-2.0), AudioFormat(44100)):
        assert all(n != "Loudness" for n, _ in audio.stages(f))


def test_counts_and_the_record_size_against_the_header():
    hdr = {k: int(v) for k, v in re.findall(r"#define (Q3_LOUD_\w+) (\d+)\b",
                                            open(os.path.join(ROOT, "include", "qwen3tts_b200.h")).read())}
    assert hdr["Q3_LOUD_MAX_BLOCKS"] == LD.MAX_BLOCKS == 16384
    # header: target f64, n_in i64, A_{k-1} and A_{k-2} f32, filter state f32[4], z f64[3]; partial segment; ms
    assert hdr["Q3_LOUD_HEADER_BYTES"] == 8 + 8 + 4 + 4 + 16 + 24
    assert LD.ROW_BYTES == hdr["Q3_LOUD_ROW_BYTES"] == hdr["Q3_LOUD_HEADER_BYTES"] + 4 * LD.SEG + 8 * LD.MAX_BLOCKS
    assert LD.MAX_BLOCKS * LD.SEG == (27 * 60 + 18.4) * 24000
    for n in (0, 1, 2399, 2400, 2401, 10 ** 7):
        assert LD.emitted(n) == LD.total(n) == n


def test_reference_properties():
    g = np.random.default_rng(0)
    x = (g.standard_normal(24000 * 3) * 0.03).astype(np.float32)
    A, ms, _ = LR.measure(x, -20.0)
    assert A.shape == (30,) and ms.shape == (30,)
    # the first segment passes at unity gain, segment k ramps from A_{k-2} to A_{k-1}
    y = LR.apply(x, A)
    assert np.array_equal(y[:2400], x[:2400])
    assert np.array_equal(y[2400:4800], (x[2400:4800] * (1 + (A[0] - 1) * (np.arange(1, 2401, dtype=np.float32)
                                                                           / np.float32(2400)))).astype(np.float32))
    assert y[4799] == x[4799] * A[0]
    # a prefix's gains are the whole clip's: no look-ahead
    assert np.array_equal(LR.gains(x[:12345], -20.0), A[:5])
    # silence holds unity gain; the clamp bounds the gain
    assert np.all(LR.gains(np.zeros(24000), -16.0) == 1)
    assert LR.gains(x * 0.03, -10.0)[-1] == np.float32(10 ** 1.5)        # about -60 LUFS: +50 dB wanted


def test_a_loudness_request_that_could_pass_the_block_cap_is_refused_at_submit(monkeypatch):
    _mock_sync(monkeypatch)
    eng, cb = _batcher()             # horizon 20 frames of UP samples
    monkeypatch.setattr(audio.Loudness, "SEG", 10)
    monkeypatch.setattr(audio.Loudness, "MAX_BLOCKS", 3)    # 30 samples: 15 frames
    cb.submit(torch.zeros(4, H), key=1, audio_format=AudioFormat(24000, volume=6))          # no target: no cap
    with pytest.raises(ValueError, match="segments"):
        cb.submit(torch.zeros(4, H), key=2, audio_format=AudioFormat(24000, loudness=-16))
    cb.submit(torch.zeros(4, H), key=3, max_frames=30 // UP, audio_format=AudioFormat(24000, loudness=-16))
    with pytest.raises(ValueError, match="segments"):    # a slower speed streams more samples
        cb.submit(torch.zeros(4, H), key=4, max_frames=30 // UP, audio_format=AudioFormat(24000, speed=0.9, loudness=-16))
    assert [r.rid for r in cb.pending] == [1, 3]


class FakeLoudness(FakeStage):
    made = []
    SEG, MAX_BLOCKS = LD.SEG, LD.MAX_BLOCKS
    setting = staticmethod(lambda target: target)
    emitted = staticmethod(lambda t, n: LD.emitted(n))
    total = staticmethod(lambda t, n: LD.total(n))
    pattern = staticmethod(lambda t, j: (9000 + j).astype(np.float32))


def test_a_target_routes_through_loudness_then_the_limiter_and_parks(monkeypatch):
    _mock_sync(monkeypatch)
    fakes = install(monkeypatch)
    FakeLoudness.made = []
    monkeypatch.setattr(audio, "Loudness", FakeLoudness)
    eng, cb = _batcher()
    fa, fb = AudioFormat(24000, loudness=-16), AudioFormat(16000, "s16")
    a = cb.submit(torch.zeros(4, H), torch.zeros(20, H), key=1, max_frames=12, audio_format=fa)
    b = cb.submit(torch.zeros(4, H), key=2, max_frames=9, audio_format=fb)
    out = {}
    for it, (chunks, _) in enumerate(cb.stream()):
        for rid, y in chunks.items():
            out.setdefault(rid, []).append(y)
        if it == 0:
            cb.park(a)
        if it == 1:
            assert cb.parked[a].loud_state is not None and cb.parked[a].lim_state is not None
            cb.resume(a)
    loud, lim = FakeLoudness.made[0], fakes["Limiter"].made[0]
    assert cb.loudness is loud and list(cb.stages) == ["Loudness", "Limiter", "Resampler"]
    assert loud.log[0] == ("reset", [0], -16.0) and lim.log[0] == ("reset", [0], 0.0)
    assert ("save", [0]) in loud.log and len([e for e in loud.log if e[0] == "load"]) == 1
    # the limiter took exactly the normaliser's output, which is its input: 12 frames
    assert sum(e[1].get(0, 0) for e in loud.log if e[0] == "push") == 12 * UP
    assert sum(e[1].get(0, 0) for e in lim.log if e[0] == "push") == 12 * UP
    assert all(1 not in e[1] and 1 not in e[2] for o in (loud, lim) for e in o.log if e[0] == "push")
    assert np.array_equal(np.concatenate(out[a]), (5000 + np.arange(12 * UP)).astype(np.float32))
    assert out[b][0].dtype == np.int16


def test_sessions_without_a_target_open_no_loudness_stage(monkeypatch):
    _mock_sync(monkeypatch)
    install(monkeypatch)
    FakeLoudness.made = []
    monkeypatch.setattr(audio, "Loudness", FakeLoudness)
    eng, cb = _batcher()
    for i, f in enumerate((AudioFormat(8000, "ulaw", 1.25), AudioFormat(24000, volume=-3), None)):
        cb.submit(torch.zeros(4, H), key=i + 1, max_frames=6 + i, audio_format=f)
    _drain(cb)
    assert cb.loudness is None and FakeLoudness.made == [] and "Loudness" not in cb.stages
