"""Host logic of the continuous batcher's audio path (no GPU): row resets on admission, per-row counts of the codec
stream, and the chunks handed out per request — against the fake engine of test_scheduler_cpu.py and a fake codec
stream whose "audio" of a frame is `up` copies of the frame's first code."""
import numpy as np
import torch

from qwen3_tts_b200.config import SamplingParams
from tests.test_scheduler_cpu import FakeEngine, _mock_sync

UP = 3


class FakeStream:
    def __init__(self, B, nmax, log):
        self.B, self.nmax, self.log = B, nmax, log
        self.pos = [0] * B

    def reset(self, rows=None):
        rows = list(range(self.B)) if rows is None else list(rows)
        for r in rows:
            self.pos[r] = 0
        self.log.append(("reset", rows))

    def push(self, codes, counts=None):
        B, K, n = codes.shape
        counts = [n] * B if counts is None else list(counts)
        assert B == self.B and all(0 <= k <= n for k in counts)
        wav = torch.zeros(B, 1, n * UP)
        for b, k in enumerate(counts):
            wav[b, 0, :k * UP] = codes[b, 0, :k].float().repeat_interleave(UP)
            self.pos[b] += k
        self.log.append(("push", list(counts), list(self.pos)))
        return wav


class FakeCodec:
    total_upsample = UP

    def __init__(self, max_frames=64):
        self.max_frames = max_frames
        self.log = []

    def open_stream(self, batch, max_packet_frames=8):
        self.stream = FakeStream(batch, max_packet_frames, self.log)
        return self.stream


def _run(monkeypatch, eos_at, horizons, n_slots=2, packet=4, codec_max=64):
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    _mock_sync(monkeypatch)
    eng, codec = FakeEngine(eos_at=eos_at), FakeCodec(codec_max)
    cb = ContinuousBatcher(eng, torch.zeros(8), SamplingParams(max_new_tokens=11), n_slots=n_slots, packet_frames=packet,
                           codec=codec)
    for i, h in enumerate(horizons):
        cb.submit(torch.zeros(4, 8), key=i, max_frames=h)
    audio, order = {}, []
    for chunks, finished in cb.stream():
        for rid, a in chunks.items():
            assert a.dtype == np.float32
            audio.setdefault(rid, []).append(a)
        order += finished
    return cb, eng, codec, {k: np.concatenate(v) for k, v in audio.items()}, order


def test_resets_counts_and_chunks_follow_the_slots(monkeypatch):
    cb, eng, codec, audio, order = _run(monkeypatch, {1: 3, 3: 0}, [10, 10, 6, 10, 2])
    assert sorted(order) == [0, 1, 2, 3, 4]
    frames = {rid: int(c.shape[0]) for rid, c in cb.done.items()}
    assert frames == {0: 10, 1: 3, 2: 6, 3: 0, 4: 2}
    for rid, n in frames.items():
        got = audio.get(rid, np.zeros(0, np.float32))
        assert got.shape == (n * UP,), (rid, got.shape)                       # chunk lengths add up to the frames
        assert (got == cb.done[rid][:, 0].numpy().repeat(UP)).all()           # and carry the request's own frames
    # every admission resets exactly the admitted slots before their first push, and a reused slot again
    admits = [e for e in eng.log if e[0] == "admit"]
    resets = [e[1] for e in codec.log if e[0] == "reset"]
    assert resets == [a[1] for a in admits]
    slot_of = {k: s for a in admits for s, k in zip(a[1], a[2])}
    assert slot_of[2] == slot_of[1] and sum(slot_of[1] in r for r in resets) >= 2  # the reused slot is reset again
    # replayed from the log: the stream's rows advance by the new frames only, from 0 after their reset
    pushed = {0: 0, 1: 0}
    for e in codec.log:
        if e[0] == "reset":
            for s in e[1]:
                pushed[s] = 0
        else:
            for s in (0, 1):
                pushed[s] += e[1][s]
            assert e[2] == [pushed[0], pushed[1]]


def test_counts_equal_the_new_frames_and_idle_slots_push_zero(monkeypatch):
    """One request in a two-slot session: slot 1 stays idle and pushes 0 every step; slot 0 pushes its new frames."""
    cb, eng, codec, audio, order = _run(monkeypatch, {}, [7])
    pushes = [e[1] for e in codec.log if e[0] == "push"]
    assert [p[1] for p in pushes] == [0] * len(pushes)
    assert sum(p[0] for p in pushes) == 7 and all(p[0] <= 4 for p in pushes)
    assert audio[0].shape == (7 * UP,)


def test_horizon_is_capped_at_the_codec_table(monkeypatch):
    cb, eng, codec, audio, order = _run(monkeypatch, {}, [10, 10], codec_max=5)
    assert {rid: int(c.shape[0]) for rid, c in cb.done.items()} == {0: 5, 1: 5}
    assert max(max(e[2]) for e in codec.log if e[0] == "push") <= 5


def test_without_a_codec_stream_is_refused_and_step_is_unchanged(monkeypatch):
    import pytest
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    _mock_sync(monkeypatch)
    cb = ContinuousBatcher(FakeEngine(), torch.zeros(8), SamplingParams(max_new_tokens=11), n_slots=2, packet_frames=4)
    cb.submit(torch.zeros(4, 8), key=0, max_frames=3)
    with pytest.raises(ValueError, match="codec"):
        next(cb.stream())
    assert cb.step() == [0]


def test_an_open_stream_must_fit_the_session(monkeypatch):
    """A CodecStream is taken as the session's stream when it has n_slots rows and room for a packet; anything that is
    neither a stream nor a decoder is refused."""
    import pytest
    from qwen3_tts_b200.codec import CodecStream
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    _mock_sync(monkeypatch)

    class OpenStream(FakeStream, CodecStream):
        def __init__(self, B, nmax, dec):
            super().__init__(B, nmax, dec.log)
            self.dec = dec

    codec = FakeCodec()
    make = lambda c: ContinuousBatcher(FakeEngine(), torch.zeros(8), SamplingParams(max_new_tokens=11), n_slots=2,  # noqa: E731
                                       packet_frames=4, codec=c)
    for bad, msg in ((OpenStream(3, 4, codec), "3 rows"), (OpenStream(2, 3, codec), "up to 3 frames"),
                     (object(), "CodecDecoder or a CodecStream")):
        with pytest.raises(ValueError, match=msg):
            make(bad)
    st = OpenStream(2, 8, codec)
    cb = make(st)
    assert cb.cstream is st and cb.codec is codec
    cb.submit(torch.zeros(4, 8), key=0, max_frames=3)
    assert [sorted(c) for c, _ in cb.stream()] == [[0]] and st.pos == [3, 0]
