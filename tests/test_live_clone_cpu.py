"""Live text of ICL voice clones without a GPU: the rows of build_live_icl_prefill / build_live_clone_request, completed
through the batcher's overlay by later text rows, tts_eos and the tts_pad fill, are exactly build_prefill's streaming
rows of the whole ids (unregistered and registered voices, every split of the text); and the batcher's policy for a
request whose overlay waits for text (admission, parking, run(), cancel, park, refusals) against the fake engines of the
other batcher tests."""
from types import SimpleNamespace

import pytest
import torch

from qwen3_tts_b200.config import SamplingParams
from tests.test_live_text_cpu import HoldingEngine
from tests.test_scheduler_cpu import _mock_sync
from tests.test_scheduler_park_cpu import ParkingEngine
from tests.test_voice_prefix_cpu import BankCodec, _model, _voice

H = 8


class RecordingEngine(HoldingEngine):
    """Keeps each admitted request's prompt rows and its trailing rows, those appended later included."""

    def __init__(self, hidden=H):
        super().__init__()
        self.cfg = SimpleNamespace(talker=SimpleNamespace(hidden_size=hidden), num_code_groups=3)
        self.rows = {}

    def admit(self, slots, keys, embs, trails, **kw):
        super().admit(slots, keys, embs, trails)
        self.log.append(("kw", kw))
        hid = self.cfg.talker.hidden_size
        for s, k, e, t in zip(slots, keys, embs, trails):
            self.rows[k] = [e.reshape(-1, hid).clone(), t.reshape(-1, hid).clone()]
            self.T[s] = self.rows[k][1].shape[0]

    def append_trailing(self, slot, rows):
        super().append_trailing(slot, rows)
        r = self.rows[self.key[slot]]
        r[1] = torch.cat([r[1], rows.to(r[1].dtype)], 0)


def _batcher(eng, pad, n_slots=2, max_trailing=64, park_waiting=False, codec=None):
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    return ContinuousBatcher(eng, pad, SamplingParams(max_new_tokens=9), n_slots=n_slots, packet_frames=4,
                             max_trailing=max_trailing, park_waiting=park_waiting, codec=codec)


# ---------------------------------------------------------------------------------------------- rows
CASES = [   # (reference text, reference frames, target text): R = len(reference text), Lc = frames + 1, K = max(0, Lc - R)
    ("abcd", 9, "Hello there, friend."),   # R < Lc, T = 20 > K = 6
    ("abcd", 9, "Hello!"),                 # T = K: tts_eos is the first trailing row
    ("abcd", 9, "Hello"),                  # T = K - 1: tts_eos lands on the last overlay row
    ("abcd", 9, "Hi"),                     # shorter: the overlay ends in tts_pad rows
    ("a longer ref", 5, "Hi there."),      # R >= Lc: K = 0, an ordinary live request
]


def _whole(w, item, text):
    """build_prefill(non_streaming_mode=False) of the whole request."""
    input_ids = w._tokenize_texts([w._build_assistant_text(text)])
    ref_ids = [w._tokenize_texts([w._build_ref_text(item.ref_text)])[0]]
    vcp = w._prompt_items_to_voice_clone_prompt([item])
    e, t, p = w.model.build_prefill(input_ids, ref_ids=ref_ids, voice_clone_prompt=vcp, languages=["English"],
                                    non_streaming_mode=False)
    return e[0], t[0], p


def _complete(w, emb, tr, pad, ov, rest, up_front):
    """Submit a live request of `emb`, `tr`, `ov` to a batcher, feed the rest of its text (two pieces and tts_eos,
    appended, or all given at submit) and close it; returns the prompt and trailing rows the engine received."""
    eng = RecordingEngine(w.model.cfg.talker.hidden_size)
    cb = _batcher(eng, pad, n_slots=1)
    half = len(rest) // 2
    later = [w.live_text_rows(rest[:half]), w.live_text_rows(rest[half:]), w.live_text_end()]
    if up_front:
        rid = cb.submit(emb, torch.cat([tr] + later, 0), key=5, text_open=True, overlay=ov)
    else:
        rid = cb.submit(emb, tr, key=5, text_open=True, overlay=ov)
        for rows in later:
            cb.append_text(rid, rows)
    cb.close_text(rid)
    cb.run()
    return eng.rows[rid]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_live_clone_rows_equal_streaming_prefill(case, monkeypatch):
    from qwen3_tts_b200.model import VoiceClonePromptItem
    _mock_sync(monkeypatch)
    ref_text, L, text = CASES[case]
    w = _model("base")
    g = torch.Generator().manual_seed(3 + case)
    item = VoiceClonePromptItem(torch.randint(0, 2000, (L, 16), generator=g), torch.randn(w.model.cfg.talker.hidden_size,
                                generator=g).bfloat16(), False, True, ref_text)
    voice = w.register_voice(voice_clone_prompt=[item], language="English")
    R, Lc, T = len(ref_text), L + 1, len(text)
    K = max(0, Lc - R)
    E, Tr, P = _whole(w, item, text)
    eos_on_overlay = R + T + 1 == Lc
    for t in range(T + 1):
        for registered in (False, True):
            if registered:
                suf, tr, pad, ov = w.build_live_clone_request(text[:t], voice=voice)
                emb = torch.cat([voice.prefix, suf], 0)
            else:
                emb, tr, pad, ov = w.build_live_clone_request(text[:t], voice_clone_prompt=item, language="English")
            assert ov.shape[0] == K - min(K, t) and emb.shape[0] + ov.shape[0] == E.shape[0] and torch.equal(pad, P)
            assert torch.equal(emb, E[:emb.shape[0]]), (t, registered)
            assert tr.shape[0] == max(0, R + t - Lc)
            for up_front in (False, True):
                rows, trailing = _complete(w, emb, tr, pad, ov, text[t:], up_front)
                assert torch.equal(rows, E), (t, registered, up_front)
                if eos_on_overlay:
                    # the text's last row completed the overlay: build_prefill's trailing [tts_pad] is what the engine
                    # reads past the end of a closed text
                    assert trailing.shape[0] == 0 and torch.equal(Tr, P.reshape(1, -1))
                else:
                    assert torch.equal(trailing, Tr), (t, registered, up_front)
    with pytest.raises(ValueError, match="ICL"):
        w.build_voice_request(text, voice, live=True)
    voice.close()


def test_model_refusals():
    from qwen3_tts_b200.model import VoiceClonePromptItem
    w = _model("base")
    g = torch.Generator().manual_seed(9)
    Hm = w.model.cfg.talker.hidden_size
    icl = VoiceClonePromptItem(torch.randint(0, 2000, (6, 16), generator=g), torch.randn(Hm, generator=g).bfloat16(),
                               False, True, "ab")
    xv = VoiceClonePromptItem(None, torch.randn(Hm, generator=g).bfloat16(), True, False)
    with pytest.raises(ValueError, match="build_live_request"):
        w.build_live_clone_request("Hi", voice_clone_prompt=xv)
    with pytest.raises(ValueError, match="one of"):
        w.build_live_clone_request("Hi")
    with pytest.raises(ValueError, match="one text"):
        w.build_live_clone_request(["Hi", "there"], voice_clone_prompt=icl)
    with pytest.raises(ValueError, match="build_voice_request"):
        w.build_live_clone_request("Hi", voice=w.register_voice(voice_clone_prompt=xv))
    with pytest.raises(ValueError, match="non_streaming_mode"):
        w.build_live_clone_request("Hi", voice=w.register_voice(voice_clone_prompt=icl, non_streaming_mode=True))
    v = w.register_voice(voice_clone_prompt=icl, language="English")
    with pytest.raises(ValueError, match="fixes its language"):
        w.build_live_clone_request("Hi", voice=v, language="English")
    v.close()
    with pytest.raises(ValueError, match="closed"):
        w.build_live_clone_request("Hi", voice=v)
    # the calls of the other prompts keep refusing ICL
    with pytest.raises(ValueError, match="ICL"):
        w.build_live_request("Hi", language="English", voice_clone_prompt=[icl])
    vcp = w._prompt_items_to_voice_clone_prompt([xv])
    ids = w._tokenize_texts([w._build_assistant_text("Hi")])
    with pytest.raises(ValueError, match="not an ICL"):
        w.model.build_live_icl_prefill(ids, [None], vcp, ["English"])


# ---------------------------------------------------------------------------------------------- batcher policy
def _rows(n, v=0.0):
    return torch.full((n, H), float(v))


def _overlay(k):
    return torch.arange(k * H, dtype=torch.float32).reshape(k, H)


def test_admission_waits_for_the_overlay(monkeypatch):
    """A request is admitted once its overlay is full (text rows summed onto it, the rest trailing, opened) or its text
    is closed (tts_pad fill, trailing [tts_pad], never opened); meanwhile other requests are admitted and run."""
    _mock_sync(monkeypatch)
    eng = RecordingEngine()
    pad = torch.full((H,), 0.5)
    cb = _batcher(eng, pad)
    a = cb.submit(_rows(3, 1), _rows(1, 7), key=1, max_frames=5, text_open=True, overlay=_overlay(4))
    b = cb.submit(_rows(2, 2), _rows(0), key=2, max_frames=4, text_open=True, overlay=_overlay(5))
    plain = cb.submit(_rows(4), _rows(2), key=3, max_frames=3)
    assert [r.n_text for r in cb.pending] == [0, 0, 2]
    cb.step()
    assert [e[2] for e in eng.log if e[0] == "admit"] == [[plain]] and len(cb.pending) == 2
    cb.append_text(a, _rows(2, 10))
    cb.append_text(b, _rows(2, 20))
    cb.step()
    assert [e[2] for e in eng.log if e[0] == "admit"] == [[plain]]
    cb.append_text(a, _rows(3, 30))                      # one row completes the overlay, two are trailing
    assert cb.pending[0].n_text == 2 and cb.pending[0].overlay is None
    cb.close_text(b)                                     # b ends inside its overlay
    cb.step()
    assert [e[2] for e in eng.log if e[0] == "admit"][1] == [a, b]
    ov = _overlay(4)
    want_a = torch.cat([_rows(3, 1), ov + torch.cat([_rows(1, 7), _rows(2, 10), _rows(1, 30)])])
    assert torch.equal(eng.rows[a][0], want_a) and torch.equal(eng.rows[a][1], _rows(2, 30))
    ov = _overlay(5)
    want_b = torch.cat([_rows(2, 2), ov[:2] + 20, ov[2:] + pad])
    assert torch.equal(eng.rows[b][0], want_b) and torch.equal(eng.rows[b][1], pad.reshape(1, H))
    opens = [e for e in eng.log if e[0] == "open"]
    assert opens == [("open", 0, True)]                  # a is open, b was closed before its admission
    cb.append_text(a, _rows(5, 40))
    cb.close_text(a)
    out = cb.run()
    assert sorted(out) == [a, b, plain]


def test_requests_without_overlay_make_the_same_calls(monkeypatch):
    """A session with an overlay request that never completes, or with an empty overlay, makes exactly the engine calls
    of the same session without it."""
    _mock_sync(monkeypatch)

    def session(extra):
        eng = RecordingEngine()
        cb = _batcher(eng, torch.zeros(H))
        live = cb.submit(_rows(4), _rows(1), key=1, max_frames=6, text_open=True)
        cb.submit(_rows(3), _rows(2), key=2, max_frames=5)
        if extra == "waiting":
            cb.submit(_rows(2), _rows(0), key=9, text_open=True, overlay=_overlay(3))
        for i in range(6):
            if i == 1 and extra == "empty":
                cb.submit(_rows(2), _rows(1), key=4, max_frames=3, text_open=True, overlay=_overlay(0))
            elif i == 1:
                cb.submit(_rows(2), _rows(1), key=4, max_frames=3, text_open=True)
            if i == 2:
                cb.append_text(live, _rows(3))
                cb.append_text(4, _rows(2))
                cb.close_text(4)
            if i == 3:
                cb.append_text(live, _rows(2))
                cb.close_text(live)
            cb.step()
        return eng.log

    base = session(None)
    assert session("waiting") == base and session("empty") == base


def test_park_waiting_and_run_ignore_a_request_that_cannot_enter(monkeypatch):
    _mock_sync(monkeypatch)
    eng = ParkingEngine()
    cb = _batcher(eng, torch.zeros(H), n_slots=1, park_waiting=True)
    live = cb.submit(_rows(4), _rows(0), key=1, max_frames=6, text_open=True)
    cb.step()                                            # live holds at frame 0
    icl = cb.submit(_rows(2), _rows(1), key=2, max_frames=4, text_open=True, overlay=_overlay(3))
    for _ in range(3):
        cb.step()
    assert cb.moves == [] and cb.running[0].rid == live  # no park for a request that could not enter
    with pytest.raises(ValueError, match="waits for text"):
        cb.run()
    cb.append_text(icl, _rows(2))                        # the overlay is full: live is parked for it
    cb.step()
    assert cb.moves == [("park", live, 0)] and cb.running[0].rid == icl
    cb.close_text(icl)
    cb.append_text(live, _rows(6))
    cb.close_text(live)
    out = cb.run()
    assert sorted(out) == [live, icl] and out[icl].shape[0] == 4 and out[live].shape[0] == 6
    # run() drains what can run and raises when only a waiting overlay is left
    cb.submit(_rows(3), _rows(2), key=3, max_frames=3)
    cb.submit(_rows(2), _rows(0), key=4, text_open=True, overlay=_overlay(2))
    with pytest.raises(ValueError, match="waits for text"):
        cb.run()
    assert 3 in cb.done and [r.rid for r in cb.pending] == [4]


def test_cancel_and_park_a_waiting_request(monkeypatch):
    _mock_sync(monkeypatch)
    eng = RecordingEngine()
    cb = _batcher(eng, torch.zeros(H))
    a = cb.submit(_rows(2), _rows(0), key=1, max_frames=3, text_open=True, overlay=_overlay(2))
    b = cb.submit(_rows(2), _rows(1), key=2, max_frames=3, text_open=True, overlay=_overlay(2))
    cb.park(b)
    assert cb.cancel(a) and not cb.cancel(a)
    with pytest.raises(ValueError, match="was cancelled"):
        cb.append_text(a, _rows(1))
    cb.append_text(b, _rows(1))                          # b's overlay is full, but b is paused
    cb.step()
    assert not any(e[0] == "admit" for e in eng.log)
    cb.resume(b)
    cb.step()
    assert [e[2] for e in eng.log if e[0] == "admit"] == [[b]]
    cb.close_text(b)
    assert sorted(cb.run()) == [b]


def test_voice_request_with_an_overlay(monkeypatch):
    """A registered ICL voice's live request may have no rows of its own but its overlay; it is admitted with the
    voice's prefix and its codec row is copied from the bank once the overlay is full."""
    _mock_sync(monkeypatch)
    eng, codec = RecordingEngine(), BankCodec()
    cb = _batcher(eng, torch.zeros(H), codec=codec)
    v = _voice(eng, 9, 4, codec, (0, 1), ref_len=6)
    v.non_streaming_mode = False
    rid = cb.submit(_rows(0), _rows(0), key=1, max_frames=5, voice=v, text_open=True, overlay=_overlay(3))
    cb.step()
    assert not any(e[0] == "admit" for e in eng.log) and v.pending == 1
    cb.append_text(rid, _rows(4))
    cb.step()
    assert ("kw", {"prefixes": [4]}) in eng.log and v.pending == 0
    assert [e[0] for e in codec.log if e[0] in ("copy", "seed", "reset")] == ["copy"]
    cb.close_text(rid)
    assert cb.run()[rid].shape[0] == 5


def test_submit_and_append_refusals(monkeypatch):
    _mock_sync(monkeypatch)
    eng, codec = RecordingEngine(), BankCodec()
    cb = _batcher(eng, torch.zeros(H), codec=codec, max_trailing=2)
    with pytest.raises(ValueError, match="text_open=True"):
        cb.submit(_rows(2), _rows(0), overlay=_overlay(2))
    for bad in (torch.zeros(2, H + 1), torch.zeros(H)):
        with pytest.raises(ValueError, match="overlay must be"):
            cb.submit(_rows(2), _rows(0), text_open=True, overlay=bad)
    with pytest.raises(ValueError, match="does not fit max_ctx"):
        cb.submit(_rows(10), _rows(0), text_open=True, overlay=_overlay(eng.max_ctx - 10))
    design = _voice(eng, 5, 1)
    with pytest.raises(ValueError, match="ICL voice"):
        cb.submit(_rows(1), _rows(0), voice=design, text_open=True, overlay=_overlay(2))
    nsm = _voice(eng, 5, 2, codec, (0, 0), ref_len=3)
    nsm.non_streaming_mode = True
    with pytest.raises(ValueError, match="non_streaming_mode=False"):
        cb.submit(_rows(1), _rows(0), voice=nsm, text_open=True, overlay=_overlay(2))
    nsm.non_streaming_mode = False
    with pytest.raises(ValueError, match="at least one row"):
        cb.submit(_rows(0), _rows(0), voice=nsm, text_open=True, overlay=_overlay(0))
    assert not cb.pending
    # max_trailing counts trailing rows only: rows that complete the overlay are prompt positions
    rid = cb.submit(_rows(0), _rows(4), voice=nsm, text_open=True, overlay=_overlay(3))
    assert cb.pending[0].n_text == 1
    cb.append_text(rid, _rows(1))
    with pytest.raises(ValueError, match="max_trailing"):
        cb.append_text(rid, _rows(1))
    with pytest.raises(ValueError, match="max_trailing"):
        cb.submit(_rows(2), _rows(6), text_open=True, overlay=_overlay(3))
    rid2 = cb.submit(_rows(2), _rows(5), text_open=True, overlay=_overlay(3))
    assert cb.pending[-1].n_text == 2 and cb.pending[-1].overlay is None
    with pytest.raises(ValueError, match="max_trailing >= 1"):
        _batcher(RecordingEngine(), torch.zeros(H), max_trailing=0).submit(_rows(2), _rows(0), text_open=True, overlay=_overlay(1))
    assert cb.cancel(rid) and cb.cancel(rid2) and nsm.pending == 0
