"""Live text without a GPU: the batcher's launch rule, horizons, append / close on pending and running requests, cancel
and errors against a fake engine that models held steps; and the live-request rows of the model API against the
streaming-layout prefill of the same ids."""
import pytest
import torch

from qwen3_tts_b200.config import SamplingParams
from tests.test_scheduler_cpu import FakeEngine, _mock_sync

H = 8


class HoldingEngine(FakeEngine):
    """A row open for live text holds at a step whose text row has not arrived: the step's frame is produced (as the
    code-predictor half does) but not committed, and the row reports its committed frames + 1 while held."""

    def session_begin(self, n_slots, pad, sp, max_trailing=0):
        super().session_begin(n_slots, pad, sp, max_trailing)
        self.T, self.open, self.held = [0] * n_slots, [False] * n_slots, [False] * n_slots
        self.launches = 0

    def admit(self, slots, keys, embs, trails):
        super().admit(slots, keys, embs, trails)
        for s, t in zip(slots, trails):
            self.T[s], self.open[s], self.held[s] = int(t.reshape(-1, H).shape[0]), False, False

    def append_trailing(self, slot, rows):
        assert not self.fin[slot]
        self.T[slot] += int(rows.shape[0])
        self.log.append(("append", slot, int(rows.shape[0])))

    def set_text_open(self, slot, open):
        assert not self.fin[slot]
        self.open[slot] = bool(open)
        self.log.append(("open", slot, bool(open)))

    def release_slots(self, slots):
        super().release_slots(slots)
        for s in slots:
            self.open[s] = self.held[s] = False

    def decode(self, n, codes):
        self.launches += 1
        self.held = [False] * self.n
        for _ in range(n):
            for s in range(self.n):
                if not self.fin[s]:
                    codes[s, self.local[s]] = self.key[s] * 100 + self.local[s]
                    if self.open[s] and self.local[s] >= self.T[s]:
                        self.held[s] = True
                    else:
                        self.local[s] += 1
            self.step += 1

    def progress(self):
        return self.step, [self.local[s] + int(self.held[s]) if not self.fin[s] else self.nv[s] for s in range(self.n)], list(self.fin)


def _batcher(n_slots=2, packet=4, max_trailing=16):
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    eng = HoldingEngine()
    return eng, ContinuousBatcher(eng, torch.zeros(H), SamplingParams(max_new_tokens=13), n_slots=n_slots,
                                  packet_frames=packet, max_trailing=max_trailing)


def _rows(n):
    return torch.zeros(n, H)


def test_launch_rule_and_horizons(monkeypatch):
    _mock_sync(monkeypatch)
    eng, cb = _batcher()
    a = cb.submit(torch.zeros(4, H), _rows(0), key=1, max_frames=6, text_open=True)
    assert cb.step() == [] and eng.launches == 1
    _, nv, _ = eng.progress()
    assert nv[0] == 1                                   # held at frame 0: the held step's frame is reported
    for _ in range(3):                                  # waiting for text: no launch, no frames
        new, fin = cb._advance()
        assert new == {} and fin == [] and eng.launches == 1 and cb.frames_total == 4
    cb.append_text(a, _rows(1))                         # text covers the one reported frame: runnable
    cb.step()
    assert eng.launches == 2 and eng.progress()[1][0] == 2
    cb.append_text(a, _rows(2))
    cb.step()
    assert eng.progress()[1][0] == 4
    cb.append_text(a, _rows(5))
    cb.close_text(a)
    assert ("open", 0, False) in eng.log
    out = cb.run()
    assert out[a].shape[0] == 6 and (out[a][:, 0] == torch.arange(6) + 100).all()   # the horizon, codes in order


def test_pending_append_and_close(monkeypatch):
    """Text appended to a pending request is concatenated on the host; a request closed while pending is admitted
    closed; an open one is opened at admission."""
    _mock_sync(monkeypatch)
    eng, cb = _batcher(n_slots=1)
    busy = cb.submit(torch.zeros(4, H), _rows(2), key=7, max_frames=3)
    a = cb.submit(torch.zeros(4, H), _rows(1), key=1, max_frames=5, text_open=True)
    b = cb.submit(torch.zeros(4, H), _rows(0), key=2, max_frames=5, text_open=True)
    cb.append_text(a, _rows(3))
    cb.append_text(b, _rows(2))
    cb.close_text(b)
    assert cb.pending[1].trailing.shape == (4, H) and cb.pending[2].trailing.shape == (2, H)
    cb.step()                       # request 7 runs to its horizon and frees the slot
    assert busy in cb.done
    cb.step()                       # request 1 admitted with 4 rows, opened
    assert ("open", 0, True) in eng.log and eng.T[0] == 4
    cb.append_text(a, _rows(1))
    cb.close_text(a)
    cb.run()
    assert sorted(cb.done) == [1, 2, 7]
    assert [e for e in eng.log if e[0] == "open"] == [("open", 0, True), ("open", 0, False)]   # request 2: never opened


def test_cancel(monkeypatch):
    _mock_sync(monkeypatch)
    eng, cb = _batcher(n_slots=2)
    held = cb.submit(torch.zeros(4, H), _rows(0), key=1, max_frames=8, text_open=True)
    run = cb.submit(torch.zeros(4, H), _rows(3), key=2, max_frames=12)
    pend = cb.submit(torch.zeros(4, H), _rows(3), key=3, max_frames=4)
    cb.step()
    assert cb.cancel(pend) and cb.cancel(held)
    assert ("release", [0]) in eng.log and 0 not in cb.running
    nxt = cb.submit(torch.zeros(4, H), _rows(3), key=4, max_frames=5)
    cb.step()
    assert cb.running[0].rid == nxt                      # the cancelled request's slot is reused
    assert cb.cancel(run) and not cb.cancel(run) and not cb.cancel(123)
    out = cb.run()
    assert sorted(out) == [nxt] and (out[nxt][:, 0] == torch.arange(5) + 400).all()


def test_errors(monkeypatch):
    _mock_sync(monkeypatch)
    eng, cb = _batcher(n_slots=1, max_trailing=4)
    live = cb.submit(torch.zeros(4, H), _rows(2), key=1, max_frames=8, text_open=True)
    plain = cb.submit(torch.zeros(4, H), _rows(1), key=2, max_frames=2)
    with pytest.raises(ValueError, match="max_trailing"):
        cb.append_text(live, _rows(3))
    with pytest.raises(ValueError, match="max_trailing"):
        cb.submit(torch.zeros(4, H), _rows(5), key=9, text_open=True)
    for f in (cb.append_text, cb.close_text):
        with pytest.raises(ValueError, match="is unknown"):
            f(55, _rows(1)) if f == cb.append_text else f(55)
        with pytest.raises(ValueError, match="not submitted with text_open"):
            f(plain, _rows(1)) if f == cb.append_text else f(plain)
    cb.step()                                           # live request admitted and running
    with pytest.raises(ValueError, match="max_trailing"):
        cb.append_text(live, _rows(3))
    cb.close_text(live)
    with pytest.raises(ValueError, match="already closed"):
        cb.close_text(live)
    with pytest.raises(ValueError, match="already closed"):
        cb.append_text(live, _rows(1))
    cb.run()
    with pytest.raises(ValueError, match="has finished"):
        cb.append_text(live, _rows(1))
    gone = cb.submit(torch.zeros(4, H), _rows(0), key=3, text_open=True)
    assert cb.cancel(gone)
    with pytest.raises(ValueError, match="was cancelled"):
        cb.close_text(gone)
    stuck = cb.submit(torch.zeros(4, H), _rows(0), key=4, text_open=True)
    with pytest.raises(ValueError, match="waits for text"):
        cb.run()
    assert cb.running[0].rid == stuck


def test_live_request_rows_equal_streaming_prefill():
    """build_live_prefill + text_rows + tts_eos_row give exactly build_prefill(non_streaming_mode=False) of the same
    ids, however the later ids are split; the public wrapper's build_live_request / live_text_rows / live_text_end
    likewise; an ICL prompt and a text without tokens raise."""
    from oracle import talker as OT
    from tests import helpers as Hh
    from qwen3_tts_b200.model import Qwen3TTSForConditionalGenerationB200 as M, Qwen3TTSModel
    cfg = OT.cfg_tiny()
    W = OT.random_weights(cfg, seed=4, with_text=True, text_vocab=1000)
    m = M.__new__(M)
    M.__init__(m, Hh.to_pkg_cfg(cfg), {k: v.to(torch.bfloat16) for k, v in W.items()}, device="cpu", spk_id={"alice": 3000},
               spk_is_dialect={"alice": False}, codec_language_id={"english": 2050}, engine=object())
    # one text token per ResizeMLP call on both sides (a CPU BLAS may round a row differently with the call's row count)
    tp = m._tp
    m._tp = lambda t: torch.cat([tp(t[:, j:j + 1]) for j in range(t.shape[1])], dim=1) if t.shape[1] else tp(t)  # noqa: E731
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 990, (1, 20), generator=g)   # 3 role tokens, 12 text tokens, 5 closing tokens
    vcp = dict(ref_spk_embedding=[torch.randn(cfg.talker.hidden_size, generator=g)], x_vector_only_mode=[True],
               icl_mode=[False], ref_code=[None])
    for kw in (dict(instruct_ids=[torch.randint(0, 990, (1, 5), generator=g)], speakers=["alice"]), dict(voice_clone_prompt=vcp)):
        e, t, p = m.build_prefill([ids], languages=["English"], non_streaming_mode=False, **kw)
        known = torch.cat([ids[:, :5], ids[:, -5:]], 1)   # the first two text tokens so far
        le, lt, lp = m.build_live_prefill([known], languages=["English"], **kw)
        assert torch.equal(le[0], e[0]) and torch.equal(lp, p)
        rows = torch.cat([lt[0], m.text_rows(ids[0, 5:9]), m.text_rows(ids[0, 9:-5]), m.tts_eos_row()], 0)
        assert rows.shape == t[0].shape and torch.equal(rows, t[0])
    icl = dict(vcp, icl_mode=[True], x_vector_only_mode=[False], ref_code=[torch.randint(0, 2000, (5, 16), generator=g)])
    with pytest.raises(ValueError, match="ICL"):
        m.build_live_prefill([ids], voice_clone_prompt=icl, languages=["English"])
    with pytest.raises(ValueError, match="at least one text token"):
        m.build_live_prefill([torch.cat([ids[:, :3], ids[:, -5:]], 1)], languages=["English"])

    # the public wrapper, with a processor that has 3 ids for the chat wrapper's head, 5 for its tail and one per
    # character of the text: the chat wrapper goes around the first piece only
    head, tail = "<|im_start|>assistant\n", "<|im_end|>\n<|im_start|>assistant\n"

    def processor(text=None, **kw):
        out = []
        if text.startswith(head):
            out, text = [980, 981, 982], text[len(head):]
        end = [983, 984, 985, 986, 987] if text.endswith(tail) else []
        text = text[:len(text) - len(tail)] if end else text
        return {"input_ids": torch.tensor([out + [ord(ch) % 900 for ch in text] + end])}
    m.tts_model_type, m.tts_model_size = "custom_voice", "1b7"
    m.supported_languages = ["auto", "english"]
    w = Qwen3TTSModel(m, processor)
    e, t, p = w.build_live_request("Hi", speaker="alice", language="English")
    whole = w._tokenize_texts([w._build_assistant_text("Hi there.")])
    re_, rt, rp = m.build_prefill(whole, instruct_ids=[None], languages=["English"], speakers=["alice"], non_streaming_mode=False)
    rows = torch.cat([t, w.live_text_rows(" there."), w.live_text_end()], 0)
    assert torch.equal(e, re_[0]) and torch.equal(rows, rt[0]) and torch.equal(p, rp)
