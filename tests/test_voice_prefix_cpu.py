"""Registered voices without a GPU: the voice's prefix rows followed by a request's suffix rows are exactly the rows
build_prefill makes for the request, for every kind of voice and both layouts; and the batcher's host logic for voice
requests (prefixes passed to admit, codec rows copied from the reference bank instead of seeded, horizons, errors)
against the fake engine and seeding codec of the other batcher tests."""
import pytest
import torch

from qwen3_tts_b200.config import SamplingParams
from tests.test_scheduler_cpu import FakeEngine, _mock_sync
from tests.test_scheduler_voice_clone_cpu import K, SeedingCodec, SeedingStream

HEAD, TAIL, REF_TAIL = "<|im_start|>assistant\n", "<|im_end|>\n<|im_start|>assistant\n", "<|im_end|>\n"


def _processor(text=None, **kw):
    """3 ids for the chat head, 5 for the request tail, 2 for a reference text's tail, one per other character."""
    out = []
    if text.startswith(HEAD):
        out, text = [980, 981, 982], text[len(HEAD):]
    end = []
    if text.endswith(TAIL):
        end, text = [983, 984, 985, 986, 987], text[:-len(TAIL)]
    elif text.endswith(REF_TAIL):
        end, text = [983, 984], text[:-len(REF_TAIL)]
    return {"input_ids": torch.tensor([out + [ord(ch) % 900 for ch in text] + end])}


class _PrefixStore:
    def __init__(self):
        self.prefixes, self.freed = {}, []

    def create_prefix(self, rows):
        self.prefixes[len(self.prefixes)] = rows.clone()
        return len(self.prefixes) - 1

    def free_prefix(self, pid):
        self.freed.append(pid)


class _Bank:
    def __init__(self):
        self.refs = []

    def bank_reference(self, codes):
        self.refs.append(codes)
        return 0, len(self.refs) - 1

    def bank_release(self, bank, row):
        pass


def _model(model_type):
    from oracle import talker as OT
    from tests import helpers as Hh
    from qwen3_tts_b200.model import Qwen3TTSForConditionalGenerationB200 as M, Qwen3TTSModel
    from types import SimpleNamespace
    cfg = OT.cfg_tiny()
    W = OT.random_weights(cfg, seed=5, with_text=True, text_vocab=1000)
    m = M.__new__(M)
    M.__init__(m, Hh.to_pkg_cfg(cfg), {k: v.to(torch.bfloat16) for k, v in W.items()}, device="cpu",
               spk_id={"alice": 3000, "bob": 3001}, spk_is_dialect={"alice": False, "bob": "sichuan_dialect"},
               codec_language_id={"english": 2050, "chinese": 2055, "sichuan_dialect": 2060}, engine=_PrefixStore(),
               tts_model_type=model_type)
    # one text token per ResizeMLP call (a CPU BLAS may round a row differently with the call's row count)
    tp = m._tp
    m._tp = lambda t: torch.cat([tp(t[:, j:j + 1]) for j in range(t.shape[1])], dim=1) if t.shape[1] else tp(t)  # noqa: E731
    m.speech_tokenizer = SimpleNamespace(decoder=_Bank())
    return Qwen3TTSModel(m, _processor)


def _full(w, text, voice, live):
    """The rows of the request built the unregistered way (generate_* / build_live_request)."""
    if live:
        if voice.vcp is not None:
            from qwen3_tts_b200.model import VoiceClonePromptItem
            it = VoiceClonePromptItem(None, voice.vcp["ref_spk_embedding"][0], True, False)
            return w.build_live_request(text, language=voice.language, voice_clone_prompt=[it])
        return w.build_live_request(text, speaker=voice.speaker, language=voice.language, instruct=w._instruct)
    input_ids = w._tokenize_texts([w._build_assistant_text(text)])
    e, t, p = w.model.build_prefill(input_ids, voice.instruct_ids, voice.ref_ids, voice.vcp, [voice.language],
                                    [voice.speaker], voice.non_streaming_mode)
    return e[0], t[0], p


def _check(w, voice, texts=("Hello there.", "Hi"), live=False):
    for text in texts:
        suf, tr, pad = w.build_voice_request(text, voice, live=live)
        e, t, p = _full(w, text, voice, live)
        assert suf.shape[0] >= 1 and voice.prefix_len + suf.shape[0] == e.shape[0]
        assert torch.equal(torch.cat([voice.prefix, suf], 0), e), text
        assert torch.equal(tr, t) and torch.equal(pad, p)
        assert torch.equal(w.model.engine.prefixes[voice.prefix_id], voice.prefix)
    return suf


@pytest.mark.parametrize("nsm", [False, True])
def test_custom_voice_and_voice_design_rows(nsm):
    w = _model("custom_voice")
    for speaker, language, instruct in (("alice", "English", None), ("bob", "Auto", "Speak slowly."), ("bob", "English", None)):
        w._instruct = instruct
        v = w.register_voice(speaker=speaker, language=language, instruct=instruct, non_streaming_mode=nsm)
        suf = _check(w, v)
        n_ins = 0 if instruct is None else len("<|im_start|>user\n") + len(instruct) + 2
        # instruct, 3 role rows, |C| - 1 overlay rows: think ids (3, or 4 with a language id), speaker, pad
        assert v.prefix_len == n_ins + 3 + (6 if (speaker == "bob" or language != "Auto") else 5)
        assert suf.shape[0] == (len("Hi") + 2 if nsm else 1)
        if not nsm:
            _check(w, v, live=True)
    w = _model("voice_design")
    w._instruct = "A calm, low voice."
    v = w.register_voice(instruct=w._instruct, language="Chinese", non_streaming_mode=nsm)
    _check(w, v)
    if not nsm:
        _check(w, v, live=True)
    with pytest.raises(ValueError, match="Unsupported speakers"):
        _model("custom_voice").register_voice(speaker="carol")
    with pytest.raises(ValueError, match="Unsupported languages"):
        _model("custom_voice").register_voice(speaker="alice", language="Klingon")


@pytest.mark.parametrize("nsm", [False, True])
def test_voice_clone_rows(nsm):
    from qwen3_tts_b200.model import VoiceClonePromptItem
    w = _model("base")
    g = torch.Generator().manual_seed(2)
    H = w.model.cfg.talker.hidden_size
    xv = VoiceClonePromptItem(None, torch.randn(H, generator=g).bfloat16(), True, False)
    v = w.register_voice(voice_clone_prompt=xv, language="English", non_streaming_mode=nsm)
    assert v.bank is None and v.ref_len == 0
    _check(w, v)
    if not nsm:
        _check(w, v, live=True)
    for ref_text, L in (("abc", 8), ("a longer reference", 5)):   # R < Lc and R >= Lc
        it = VoiceClonePromptItem(torch.randint(0, 2000, (L, 16), generator=g), torch.randn(H, generator=g).bfloat16(),
                                  False, True, ref_text)
        v = w.register_voice(voice_clone_prompt=[it], language="English", non_streaming_mode=nsm)
        assert v.icl and v.ref_len == L and v.bank is not None
        R, Lc = len(ref_text), L + 1
        suf = _check(w, v, texts=("Hi", "Some longer text here."))
        if nsm:
            assert suf.shape[0] == (Lc + len("Some longer text here.") + 1)
        elif R < Lc:
            assert suf.shape[0] == Lc - R
        else:
            assert suf.shape[0] == 1
        with pytest.raises(ValueError, match="ICL|non_streaming_mode"):
            w.build_voice_request("Hi there", v, live=True)
        v.close()
        assert v.prefix_id in w.model.engine.freed
        with pytest.raises(ValueError, match="closed"):
            w.build_voice_request("Hi", v)


# ---------------------------------------------------------------------------------------------- batcher host logic
class PrefixEngine(FakeEngine):
    def admit(self, slots, keys, embs, trails, **kw):
        super().admit(slots, keys, embs, trails)
        self.log.append(("kw", kw))

    def free_prefix(self, pid):
        self.log.append(("free", pid))


class BankStream(SeedingStream):
    def copy_from(self, src, src_rows, rows):
        for s, r in zip(src_rows, rows):
            self.pos[r] = src.pos[s]
        self.log.append(("copy", src, list(src_rows), list(rows)))


class BankCodec(SeedingCodec):
    def __init__(self, max_frames=64):
        super().__init__(max_frames)
        self.banks = [BankStream(4, 1, []), BankStream(4, 1, [])]

    def open_stream(self, batch, max_packet_frames=8):
        self.stream = BankStream(batch, max_packet_frames, self.log)
        return self.stream

    def bank_stream(self, bank):
        return self.banks[bank]

    def bank_release(self, bank, row):
        pass


def _voice(eng, P, pid, codec=None, bank=None, ref_len=0):
    from qwen3_tts_b200.model import Voice
    v = Voice.__new__(Voice)
    v.engine, v.prefix, v.prefix_id, v.codec, v.bank = eng, torch.zeros(P, 8), pid, codec, bank
    v.ref_codes = torch.zeros(ref_len, K, dtype=torch.int64) if ref_len else None
    v.icl, v.pending, v.closed = bank is not None, 0, False
    if bank is not None:
        codec.banks[bank[0]].pos[bank[1]] = ref_len
    return v


def _batcher(eng, codec, n_slots=4):
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    return ContinuousBatcher(eng, torch.zeros(8), SamplingParams(max_new_tokens=11), n_slots=n_slots, packet_frames=4,
                             codec=codec)


def test_batcher_voice_admissions(monkeypatch):
    _mock_sync(monkeypatch)
    eng, codec = PrefixEngine(), BankCodec()
    cb = _batcher(eng, codec)
    plain = cb.submit(torch.zeros(4, 8), key=1, max_frames=3)
    cb.step()
    assert [e for e in eng.log if e[0] == "kw"] == [("kw", {})]          # no voice: exactly today's call
    design = _voice(eng, 6, 7)
    icl_a, icl_b = _voice(eng, 9, 8, codec, (0, 2), ref_len=5), _voice(eng, 9, 9, codec, (1, 0), ref_len=21)
    ids = [cb.submit(torch.zeros(1, 8), key=10, voice=design),
           cb.submit(torch.zeros(2, 8), key=11, voice=icl_a),
           cb.submit(torch.zeros(2, 8), key=12, voice=icl_b)]
    assert design.pending == 1 and icl_a.pending == 1
    with pytest.raises(ValueError, match="pending"):
        design.close()
    cb.step()
    assert eng.log[-1] == ("kw", {"prefixes": [7, 8, 9]}) and design.pending == 0
    adm = [e for e in eng.log if e[0] == "admit"][-1]
    slot = dict(zip(adm[2], adm[1]))
    after = codec.log[[i for i, e in enumerate(codec.log) if e[0] == "push"][0] + 1:]
    assert not any(e[0] == "seed" for e in after)                         # ICL voices: copied, never seeded
    copies = [e for e in after if e[0] == "copy"]
    assert [(c[1], c[2], c[3]) for c in copies] == [(codec.banks[0], [2], [slot[11]]), (codec.banks[1], [0], [slot[12]])]
    assert ("reset", [slot[10]]) in [(e[0], list(e[1])) for e in after if e[0] == "reset"]
    assert codec.stream.pos[slot[12]] >= 21
    design.close()
    assert ("free", 7) in eng.log and design.closed
    out = cb.run()
    assert sorted(out) == sorted([plain] + ids)


def test_batcher_voice_horizons_and_errors(monkeypatch):
    _mock_sync(monkeypatch)
    eng, codec = PrefixEngine(), BankCodec(max_frames=30)
    cb = _batcher(eng, codec)
    long_prefix = _voice(eng, 60, 1)                                      # max_ctx 64: P + S counts
    cb.submit(torch.zeros(2, 8), key=1, voice=long_prefix)
    assert cb.pending[-1].max_frames == 2
    with pytest.raises(ValueError, match="does not fit max_ctx"):
        cb.submit(torch.zeros(4, 8), key=2, voice=long_prefix)
    icl = _voice(eng, 3, 2, codec, (0, 0), ref_len=25)                    # codec max_frames 30: the reference counts
    cb.submit(torch.zeros(2, 8), key=3, voice=icl)
    assert cb.pending[-1].max_frames == 5
    with pytest.raises(ValueError, match="without ref_codes"):
        cb.submit(torch.zeros(2, 8), key=4, voice=icl, ref_codes=torch.zeros(3, K, dtype=torch.int64))
    with pytest.raises(ValueError, match="another engine"):
        cb.submit(torch.zeros(2, 8), key=5, voice=_voice(PrefixEngine(), 3, 3))
    with pytest.raises(ValueError, match="another codec"):
        cb.submit(torch.zeros(2, 8), key=6, voice=_voice(eng, 3, 4, BankCodec(), (0, 1), ref_len=2))
    with pytest.raises(ValueError, match="at least one row"):
        cb.submit(torch.zeros(0, 8), key=7, voice=icl)
    closed = _voice(eng, 3, 5)
    closed.close()
    with pytest.raises(ValueError, match="closed"):
        cb.submit(torch.zeros(2, 8), key=8, voice=closed)
    assert cb.cancel(1) and long_prefix.pending == 0
    no_codec = _batcher(PrefixEngine(), None)
    with pytest.raises(ValueError, match="another"):
        no_codec.submit(torch.zeros(2, 8), key=9, voice=_voice(no_codec.eng, 3, 6, codec, (0, 2), ref_len=2))
    live = _voice(no_codec.eng, 3, 7)
    rid = no_codec.submit(torch.zeros(1, 8), torch.zeros(2, 8), key=10, voice=live, text_open=True)
    no_codec.append_text(rid, torch.zeros(3, 8))
    no_codec.close_text(rid)
    assert no_codec.run()[rid].shape[0] == 10
