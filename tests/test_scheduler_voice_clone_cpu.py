"""Host logic of the continuous batcher's voice-clone admissions (no GPU): slots whose request carries reference codes
are seeded with them (one seed call per admission) instead of reset, the horizon leaves the codec's RoPE table room
for the reference, chunks and `done` hold the generated part only, and bad references are refused at submit().
Fakes: the engine of test_scheduler_cpu.py and the codec stream of test_scheduler_audio_cpu.py, given a `seed`."""
import numpy as np
import pytest
import torch

from qwen3_tts_b200.config import SamplingParams
from tests.test_scheduler_audio_cpu import UP, FakeStream
from tests.test_scheduler_cpu import FakeEngine, _mock_sync

K, BINS = 3, 16


class SeedingStream(FakeStream):
    def seed(self, rows, codes):
        rows = list(rows)
        for r, c in zip(rows, codes):
            self.pos[r] = int(c.shape[0])
        self.log.append(("seed", rows, [c.clone() for c in codes]))


class SeedingCodec:
    total_upsample = UP

    class cfg:
        num_quantizers, codebook_size = K, BINS

    def __init__(self, max_frames=64):
        self.max_frames = max_frames
        self.log = []

    def open_stream(self, batch, max_packet_frames=8):
        self.stream = SeedingStream(batch, max_packet_frames, self.log)
        return self.stream


def _ref(L, v):
    return torch.full((L, K), v, dtype=torch.int64)


def _run(monkeypatch, reqs, n_slots=2, codec_max=64, eos_at=None):
    """reqs: list of (horizon, reference or None); requests 0 .. n_slots-1 are submitted first, the rest one per step."""
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    _mock_sync(monkeypatch)
    eng, codec = FakeEngine(eos_at=eos_at), SeedingCodec(codec_max)
    cb = ContinuousBatcher(eng, torch.zeros(8), SamplingParams(max_new_tokens=11), n_slots=n_slots, packet_frames=4,
                           codec=codec)
    todo = list(enumerate(reqs))
    for i, (h, ref) in todo[:n_slots]:
        cb.submit(torch.zeros(4, 8), key=i, max_frames=h, ref_codes=ref)
    todo = todo[n_slots:]
    audio = {}
    for chunks, _ in cb.stream():
        for rid, a in chunks.items():
            audio.setdefault(rid, []).append(a)
        if todo:
            i, (h, ref) = todo.pop(0)
            cb.submit(torch.zeros(4, 8), key=i, max_frames=h, ref_codes=ref)
    return cb, eng, codec, {k: np.concatenate(v) for k, v in audio.items()}


def test_seeded_slots_are_seeded_not_reset(monkeypatch):
    reqs = [(6, _ref(5, 7)), (3, None), (4, _ref(2, 9)), (5, _ref(3, 1)), (2, None)]
    cb, eng, codec, audio = _run(monkeypatch, reqs, eos_at={4: 1})
    admits = [e for e in eng.log if e[0] == "admit"]
    slot_of = {k: s for a in admits for s, k in zip(a[1], a[2])}
    # the stream's calls between two pushes belong to one admission: one reset of the plain slots, one seed of the others
    groups, cur = [], []
    for e in codec.log:
        if e[0] == "push":
            if cur:
                groups.append(cur)
            cur = []
        else:
            cur.append(e)
    assert len(groups) == len(admits)
    for a, g in zip(admits, groups):
        plain = [s for s, k in zip(a[1], a[2]) if reqs[k][1] is None]
        seeded = [(s, k) for s, k in zip(a[1], a[2]) if reqs[k][1] is not None]
        assert [e[0] for e in g] == (["reset"] if plain else []) + (["seed"] if seeded else [])
        if plain:
            assert g[0][1] == plain
        if seeded:
            assert g[-1][1] == [s for s, _ in seeded]
            assert all(torch.equal(c, reqs[k][1]) for c, (_, k) in zip(g[-1][2], seeded))
    # a seeded row continues from its reference's length; the chunks and done carry the generated frames only
    for rid, (h, ref) in enumerate(reqs):
        codes = cb.done[rid]
        assert codes.shape[0] == (1 if rid == 4 else h)
        got = audio.get(rid, np.zeros(0, np.float32))
        assert (got == codes[:, 0].numpy().repeat(UP)).all() and got.shape == (codes.shape[0] * UP,)
    pos = {0: 0, 1: 0}
    for e in codec.log:
        if e[0] == "reset":
            for s in e[1]:
                pos[s] = 0
        elif e[0] == "seed":
            for s, c in zip(e[1], e[2]):
                pos[s] = int(c.shape[0])
        else:
            for s in (0, 1):
                pos[s] += e[1][s]
            assert e[2] == [pos[0], pos[1]]
    assert slot_of[0] != slot_of[1]


def test_without_references_the_admission_path_is_unchanged(monkeypatch):
    cb, eng, codec, audio = _run(monkeypatch, [(5, None), (3, None), (4, None)])
    assert not any(e[0] == "seed" for e in codec.log)
    assert [e[1] for e in codec.log if e[0] == "reset"] == [e[1] for e in eng.log if e[0] == "admit"]


def test_horizon_leaves_the_codec_table_room_for_the_reference(monkeypatch):
    cb, eng, codec, audio = _run(monkeypatch, [(10, _ref(7, 1)), (10, None), (10, _ref(11, 2))], codec_max=12)
    assert {rid: int(c.shape[0]) for rid, c in cb.done.items()} == {0: 5, 1: 10, 2: 1}
    assert max(max(e[2]) for e in codec.log if e[0] == "push") <= 12


def test_submit_rejects_bad_references(monkeypatch):
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    _mock_sync(monkeypatch)
    cb = ContinuousBatcher(FakeEngine(), torch.zeros(8), SamplingParams(max_new_tokens=11), n_slots=2, packet_frames=4,
                           codec=SeedingCodec(12))
    bad = [
        (torch.zeros(4, K + 1, dtype=torch.int64), "expected an \\(L, 3\\) tensor"),
        (torch.zeros(4, dtype=torch.int64), "expected an \\(L, 3\\) tensor"),
        (torch.zeros(0, K, dtype=torch.int64), "0 frames outside \\[1, 11\\]"),
        (_ref(12, 0), "12 frames outside \\[1, 11\\]"),
        (_ref(3, BINS), "codes must lie in \\[0, 16\\)"),
        (_ref(3, -1), "codes must lie in \\[0, 16\\)"),
        (torch.zeros(3, K), "integer codes"),
        ([[0] * K], "expected an \\(L, 3\\) tensor"),
    ]
    for ref, msg in bad:
        with pytest.raises(ValueError, match=msg):
            cb.submit(torch.zeros(4, 8), max_frames=3, ref_codes=ref)
    assert not cb.pending
    cb.submit(torch.zeros(4, 8), max_frames=3, ref_codes=_ref(11, BINS - 1))   # L = max_frames - 1 leaves one frame
    assert cb.pending[0].max_frames == 1
    plain = ContinuousBatcher(FakeEngine(), torch.zeros(8), SamplingParams(max_new_tokens=11), n_slots=2, packet_frames=4)
    with pytest.raises(ValueError, match="codec"):
        plain.submit(torch.zeros(4, 8), ref_codes=_ref(2, 0))
    assert not plain.pending
