"""Per-request sampling parameters in the continuous batcher, host side (no GPU): the batcher hands each admission's
parameters to the engine (None for requests without their own), a request's max_new_tokens bounds its horizon, and
bad parameters are refused at submit() by the library's own range check (q3_sampling_check, which needs no GPU)."""
import math

import pytest
import torch

from qwen3_tts_b200.config import SamplingParams
from tests.test_scheduler_cpu import FakeEngine, _mock_sync


class SamplingFakeEngine(FakeEngine):
    """FakeEngine that accepts sampling= and validates through the real library."""

    def admit(self, slots, keys, embs, trails, sampling=None):
        super().admit(slots, keys, embs, trails)
        self.log[-1] = self.log[-1] + (None if sampling is None else list(sampling),)

    @staticmethod
    def check_sampling(sp):
        from qwen3_tts_b200.engine import AREngine
        AREngine.check_sampling(sp)


def test_parameters_reach_the_engine_per_request(monkeypatch):
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    _mock_sync(monkeypatch)
    eng = SamplingFakeEngine()
    sp = SamplingParams(max_new_tokens=11)
    greedy = SamplingParams(do_sample=False, subtalker_dosample=False, max_new_tokens=11, seed=3)
    topp = SamplingParams(top_k=0, top_p=0.8, max_new_tokens=11, seed=4)
    cb = ContinuousBatcher(eng, torch.zeros(8), sp, n_slots=2, packet_frames=4)
    cb.submit(torch.zeros(4, 8), key=0, max_frames=6, sampling=greedy)
    cb.submit(torch.zeros(4, 8), key=1, max_frames=3)
    cb.submit(torch.zeros(4, 8), key=2, max_frames=3)           # no request of this admission has its own parameters
    cb.submit(torch.zeros(4, 8), key=3, max_frames=5, sampling=topp)
    out = cb.run()
    assert sorted(out) == [0, 1, 2, 3]
    admits = [e for e in eng.log if e[0] == "admit"]
    assert admits[0][1:3] == ([0, 1], [0, 1]) and admits[0][4] == [greedy, None]
    assert admits[1][2] == [2] and admits[1][4] is None             # called exactly as without the feature
    assert admits[2][2] == [3] and admits[2][4] == [topp]


def test_horizon_follows_max_new_tokens(monkeypatch):
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    _mock_sync(monkeypatch)
    eng = SamplingFakeEngine()
    cb = ContinuousBatcher(eng, torch.zeros(8), SamplingParams(max_new_tokens=11), n_slots=3, packet_frames=4)
    cb.submit(torch.zeros(4, 8), key=0, sampling=SamplingParams(max_new_tokens=5))              # 4 frames
    cb.submit(torch.zeros(4, 8), key=1, max_frames=2, sampling=SamplingParams(max_new_tokens=8))  # max_frames is lower
    cb.submit(torch.zeros(4, 8), key=2, sampling=SamplingParams(max_new_tokens=11))             # the session's 10
    out = cb.run()
    assert [int(out[k].shape[0]) for k in range(3)] == [4, 2, 10]
    with pytest.raises(ValueError, match="max_new_tokens=12 exceeds"):
        cb.submit(torch.zeros(4, 8), key=9, sampling=SamplingParams(max_new_tokens=12))
    assert not cb.pending


BAD = [
    (dict(do_sample=True, temperature=0.0), "temperature 0 must be finite and > 0 when do_sample is set"),
    (dict(do_sample=True, temperature=math.inf), "temperature inf must be finite"),
    (dict(subtalker_dosample=True, subtalker_temperature=-1.0), "subtalker_temperature -1 must be finite and > 0"),
    (dict(top_k=-1), "top_k -1 must be >= 0"),
    (dict(subtalker_top_k=-3), "subtalker_top_k -3 must be >= 0"),
    (dict(top_p=1.5), "top_p 1.5 must be in [0, 1]"),
    (dict(subtalker_top_p=-0.1), "subtalker_top_p -0.1 must be in [0, 1]"),
    (dict(repetition_penalty=math.nan), "repetition_penalty nan must be finite and > 0"),
    (dict(repetition_penalty=0.0), "repetition_penalty 0 must be finite and > 0"),
    (dict(min_new_tokens=-1), "min_new_tokens -1 must be >= 0"),
]


@pytest.mark.parametrize("kw,msg", BAD, ids=[m.split(" ")[0] + "_" + str(i) for i, (_, m) in enumerate(BAD)])
def test_library_check_names_the_field(kw, msg):
    from qwen3_tts_b200.engine import AREngine
    with pytest.raises(ValueError) as ei:
        AREngine.check_sampling(SamplingParams(**kw))
    assert msg in str(ei.value)


def test_library_check_accepts_the_edges():
    from qwen3_tts_b200.engine import AREngine
    for kw in (dict(), dict(do_sample=False, temperature=0.0), dict(subtalker_dosample=False, subtalker_temperature=0.0),
               dict(top_k=0, top_p=0.0), dict(top_p=1.0, subtalker_top_p=1.0), dict(min_new_tokens=0),
               dict(repetition_penalty=1e-3)):
        AREngine.check_sampling(SamplingParams(**kw))


def test_submit_refuses_bad_parameters_before_any_step(monkeypatch):
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    _mock_sync(monkeypatch)
    eng = SamplingFakeEngine()
    cb = ContinuousBatcher(eng, torch.zeros(8), SamplingParams(max_new_tokens=11), n_slots=2, packet_frames=4)
    cb.submit(torch.zeros(4, 8), key=0, max_frames=6)
    cb.step()
    for kw, msg in BAD:
        with pytest.raises(ValueError, match="sampling: "):
            cb.submit(torch.zeros(4, 8), key=7, sampling=SamplingParams(**kw))
    assert not cb.pending
    out = cb.run()
    assert sorted(out) == [0] and int(out[0].shape[0]) == 6
