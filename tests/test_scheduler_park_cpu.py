"""Parking in the continuous batcher without a GPU: when rows are parked and resumed (only when another request needs a
slot, only rows that wait for text, resumes before admissions, oldest park first), park(rid) / resume(rid), stream()
while requests are parked, append_text / close_text / cancel of a parked request, and the errors — against the holding
fake engine of test_live_text_cpu.py extended with records, and a fake codec whose audio shows each row's position."""
import numpy as np
import pytest
import torch

from qwen3_tts_b200.config import SamplingParams
from tests.test_live_text_cpu import HoldingEngine
from tests.test_scheduler_cpu import _mock_sync

H = 8
UP = 2


class ParkingEngine(HoldingEngine):
    """Records hold a row's frame counter, key, text length and live-text flags; the slot is free after a park."""

    def session_begin(self, n_slots, pad, sp, max_trailing=0):
        super().session_begin(n_slots, pad, sp, max_trailing)
        self.records, self.next_record = {}, 0

    def park(self, slot):
        assert not self.fin[slot], "parked a slot without a running request"
        rid = self.next_record
        self.next_record += 1
        self.records[rid] = (self.local[slot], self.key[slot], self.T[slot], self.open[slot], self.held[slot])
        self.fin[slot], self.nv[slot] = 1, 0
        self.open[slot] = self.held[slot] = False
        self.log.append(("park", slot, rid))
        return rid

    def resume(self, record, slot):
        assert self.fin[slot] == 1, "resumed into a running slot"
        self.local[slot], self.key[slot], self.T[slot], self.open[slot], self.held[slot] = self.records.pop(record)
        self.fin[slot] = 0
        self.log.append(("resume", slot, record))

    def discard(self, record):
        del self.records[record]
        self.log.append(("discard", record))


class PosStream:
    """Frame i of a row sounds as its first code + 10000 * the row's position: a row that continued from the wrong
    state would sound different."""

    def __init__(self, B):
        self.B, self.pos = B, [0] * B

    def reset(self, rows=None):
        for r in (range(self.B) if rows is None else rows):
            self.pos[r] = 0

    def push(self, codes, counts):
        B, K, n = codes.shape
        wav = torch.zeros(B, 1, n * UP)
        for b, k in enumerate(counts):
            for i in range(k):
                wav[b, 0, i * UP:(i + 1) * UP] = float(codes[b, 0, i]) + 10000 * (self.pos[b] + i)
            self.pos[b] += k
        return wav

    def copy_from(self, src, src_rows, rows):
        for s, d in zip(src_rows, rows):
            self.pos[d] = src.pos[s]


class BankCodec:
    total_upsample = UP

    def __init__(self, max_frames=64):
        self.max_frames, self.bank, self.used = max_frames, PosStream(32), set()

    def open_stream(self, batch, max_packet_frames=8):
        self.stream = PosStream(batch)
        return self.stream

    def bank_copy(self, src, src_row):
        row = min(set(range(self.bank.B)) - self.used)
        self.used.add(row)
        self.bank.copy_from(src, [src_row], [row])
        return 0, row

    def bank_stream(self, bank):
        return self.bank

    def bank_release(self, bank, row):
        self.used.discard(row)


def _batcher(n_slots=2, packet=4, codec=None, park_waiting=True):
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    eng = ParkingEngine()
    return eng, ContinuousBatcher(eng, torch.zeros(H), SamplingParams(max_new_tokens=21), n_slots=n_slots, packet_frames=packet,
                                  max_trailing=32, codec=codec, park_waiting=park_waiting)


def _rows(n):
    return torch.zeros(n, H)


def _codes_ok(out, rid, n):
    return out[rid].shape[0] == n and bool((out[rid][:, 0] == torch.arange(n) + 100 * rid).all())


def test_park_only_waiting_rows_and_only_when_a_slot_is_needed(monkeypatch):
    _mock_sync(monkeypatch)
    eng, cb = _batcher()
    a = cb.submit(torch.zeros(4, H), _rows(0), key=1, max_frames=6, text_open=True)
    cb.step()                                            # a holds at frame 0; slot 1 is free
    c = cb.submit(torch.zeros(4, H), _rows(2), key=3, max_frames=8)
    cb.step()                                            # c takes the free slot: nothing is parked
    assert cb.moves == [] and sorted(r.rid for r in cb.running.values()) == [a, c]
    d = cb.submit(torch.zeros(4, H), _rows(2), key=4, max_frames=5)
    cb.step()                                            # every slot is taken and a waits: a is parked, d takes slot 0
    assert cb.moves == [("park", a, 0)] and cb.running[0].rid == d and a in cb.parked
    assert c in cb.done                                  # c reached its horizon: slot 1 is free, but a still waits
    cb.step()
    assert len(cb.moves) == 1 and a in cb.parked and d in cb.done
    cb.append_text(a, _rows(8))                          # a can step again: it resumes into the lowest free slot
    cb.close_text(a)
    out = cb.run()
    assert cb.moves[1:] == [("resume", a, 0)]
    assert _codes_ok(out, a, 6) and _codes_ok(out, d, 5) and _codes_ok(out, c, 8)
    assert eng.records == {}


def test_resumes_come_before_admissions_oldest_park_first(monkeypatch):
    _mock_sync(monkeypatch)
    eng, cb = _batcher()
    a = cb.submit(torch.zeros(4, H), _rows(0), key=1, max_frames=7, text_open=True)
    b = cb.submit(torch.zeros(4, H), _rows(0), key=2, max_frames=7, text_open=True)
    cb.step()                                            # both hold at frame 0
    c = cb.submit(torch.zeros(4, H), _rows(1), key=3, max_frames=4)
    d = cb.submit(torch.zeros(4, H), _rows(1), key=4, max_frames=4)
    cb.step()                                            # two slots needed: both are parked, a first
    assert cb.moves == [("park", a, 0), ("park", b, 1)] and list(cb.parked) == [a, b]
    cb.append_text(b, _rows(7))
    cb.close_text(b)
    cb.append_text(a, _rows(7))
    cb.close_text(a)
    e = cb.submit(torch.zeros(4, H), _rows(1), key=5, max_frames=3)
    cb.step()                                            # c and d finish: a and b come back before e is admitted
    assert cb.moves[2:] == [("resume", a, 0), ("resume", b, 1)] and [r.rid for r in cb.pending] == [e]
    out = cb.run()
    assert all(_codes_ok(out, r, n) for r, n in ((a, 7), (b, 7), (c, 4), (d, 4), (e, 3)))


def test_resume_into_another_slot_with_audio_and_text_while_parked(monkeypatch):
    """stream() keeps running while a request is parked; text appended while parked reaches the engine at resume; the
    request's codes and chunks continue where they stopped (its codec row's position travels through the bank)."""
    _mock_sync(monkeypatch)
    codec = BankCodec()
    eng, cb = _batcher(codec=codec)
    a = cb.submit(torch.zeros(4, H), _rows(2), key=1, max_frames=8, text_open=True)
    b = cb.submit(torch.zeros(4, H), _rows(2), key=2, max_frames=4)
    audio = {}
    gen = cb.stream()
    parked_steps = 0
    for it, (chunks, _) in enumerate(gen):
        for rid, w in chunks.items():
            audio.setdefault(rid, []).append(w)
        if it == 0:   # a waits after 2 frames + 1 held, b has finished: one of c and d needs a's slot
            c = cb.submit(torch.zeros(4, H), _rows(3), key=3, max_frames=12)
            d = cb.submit(torch.zeros(4, H), _rows(3), key=4, max_frames=3)
        if a in cb.parked:
            parked_steps += 1
            if parked_steps == 2:
                cb.append_text(a, _rows(6))       # arrives while parked
                cb.close_text(a)
        assert it < 50
    assert ("park", a, 0) in cb.moves and ("resume", a, 1) in cb.moves and parked_steps >= 2
    assert ("append", 1, 6) in eng.log and ("open", 1, False) in eng.log
    for rid, n in ((a, 8), (b, 4), (c, 12), (d, 3)):
        assert _codes_ok(cb.done, rid, n)
        want = np.repeat(np.arange(n) + 100 * rid + 10000 * np.arange(n), UP).astype(np.float32)
        assert np.array_equal(np.concatenate(audio[rid]), want), f"request {rid}: chunks differ"
    assert codec.used == set()


def test_explicit_park_resume_and_cancel(monkeypatch):
    _mock_sync(monkeypatch)
    codec = BankCodec()
    eng, cb = _batcher(codec=codec, park_waiting=False)
    a = cb.submit(torch.zeros(4, H), _rows(1), key=1, max_frames=10)
    b = cb.submit(torch.zeros(4, H), _rows(1), key=2, max_frames=20)
    p = cb.submit(torch.zeros(4, H), _rows(1), key=3, max_frames=3)
    cb.park(p)                                           # pending: not admitted while paused
    cb.step()
    cb.park(a)
    assert a in [r.rid for r in cb.running.values()]     # parked at the next step boundary
    cb.step()
    assert a in cb.parked and 0 not in cb.running and [r.rid for r in cb.pending] == [p]
    cb.resume(p)                                         # p may be admitted now: it takes a's slot
    cb.step()
    assert any(e[:3] == ("admit", [0], [p]) for e in eng.log) and p in cb.done and a in cb.parked
    cb.park(b)
    cb.step()
    assert b in cb.parked and len(codec.used) == 2
    assert cb.cancel(b) and b not in cb.parked and ("discard", 1) in eng.log and len(codec.used) == 1
    for _ in range(3):
        cb.step()
    assert a in cb.parked                                # a paused request is not resumed while slots are free
    cb.resume(a)
    cb.step()
    assert ("resume", a, 0) in cb.moves and codec.used == set()
    out = cb.run()
    assert sorted(out) == [a, p] and _codes_ok(out, a, 10) and _codes_ok(out, p, 3) and eng.records == {}


def test_errors_and_run(monkeypatch):
    _mock_sync(monkeypatch)
    eng, cb = _batcher(n_slots=1)
    for f in (cb.park, cb.resume):
        with pytest.raises(ValueError, match="is unknown"):
            f(42)
    done = cb.submit(torch.zeros(4, H), _rows(1), key=1, max_frames=2)
    cb.run()
    gone = cb.submit(torch.zeros(4, H), _rows(1), key=2, max_frames=2)
    assert cb.cancel(gone)
    with pytest.raises(ValueError, match="has finished"):
        cb.park(done)
    with pytest.raises(ValueError, match="was cancelled"):
        cb.park(gone)
    # a parked live request: its text may grow and close; run() raises only when nothing can make progress
    a = cb.submit(torch.zeros(4, H), _rows(1), key=3, max_frames=6, text_open=True)
    cb.step()
    cb.park(a)
    cb.step()
    assert a in cb.parked
    with pytest.raises(ValueError, match="waits for text"):
        cb.run()
    cb.append_text(a, _rows(6))
    cb.close_text(a)
    with pytest.raises(ValueError, match="already closed"):
        cb.close_text(a)
    cb.resume(a)
    out = cb.run()
    assert _codes_ok(out, a, 6) and cb.parked == {}
