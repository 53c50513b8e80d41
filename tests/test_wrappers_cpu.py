"""Public wrapper semantics (inference/qwen3_tts_model.py) with a fake engine: input broadcasting, validation,
kwarg precedence, voice-clone proportional cut — no GPU needed."""
import numpy as np
import pytest
import torch

from qwen3_tts_b200.model import Qwen3TTSModel, VoiceClonePromptItem


class _FakeTok:
    def decode(self, items):
        return [np.arange(int(d["audio_codes"].shape[0]) * 1920, dtype=np.float32) for d in items], 24000


class _FakeCore:
    tts_model_type = "custom_voice"
    tts_model_size = "1b7"
    device = torch.device("cpu")

    def __init__(self):
        self.calls = []
        self.speech_tokenizer = _FakeTok()

    def get_supported_speakers(self):
        return ["Alice", "bob"]

    def get_supported_languages(self):
        return ["auto", "english", "chinese"]

    def generate(self, **kw):
        self.calls.append(kw)
        n = len(kw["input_ids"])
        return [torch.zeros(4 + i, 16, dtype=torch.long) for i in range(n)], [None] * n


def _proc(text=None, return_tensors="pt", padding=True):
    return {"input_ids": torch.tensor([[1, 2, 3] + [ord(c) % 50 for c in text][:8] + [4, 5, 6, 7, 8]])}


def test_custom_voice_broadcast_defaults_and_validation():
    core = _FakeCore()
    m = Qwen3TTSModel(core, _proc, generate_defaults={"top_k": 20, "temperature": 0.7})
    wavs, fs = m.generate_custom_voice(["hello", "world"], speaker="alice", language="English", top_k=None, temperature=0.5)
    assert fs == 24000 and [w.shape[0] for w in wavs] == [4 * 1920, 5 * 1920]
    kw = core.calls[-1]
    assert kw["speakers"] == ["alice", "alice"] and kw["languages"] == ["English", "English"]
    assert kw["instruct_ids"] == [None, None] and kw["non_streaming_mode"] is True
    # precedence: user > generate_config.json > hard defaults (:287-352)
    assert kw["top_k"] == 20 and kw["temperature"] == 0.5 and kw["repetition_penalty"] == 1.05 and kw["max_new_tokens"] == 2048
    with pytest.raises(ValueError):
        m.generate_custom_voice("x", speaker="carol")
    with pytest.raises(ValueError):
        m.generate_custom_voice("x", speaker="alice", language="klingon")
    with pytest.raises(ValueError):
        m.generate_custom_voice(["a", "b", "c"], speaker=["alice", "bob"])
    with pytest.raises(ValueError):
        m.generate_voice_design("x", instruct="y")  # wrong model type
    assert m.get_supported_speakers() == ["alice", "bob"]


def test_voice_clone_prepends_ref_codes_and_cuts_proportionally():
    core = _FakeCore()
    core.tts_model_type = "base"
    m = Qwen3TTSModel(core, _proc)
    item = VoiceClonePromptItem(ref_code=torch.ones(6, 16, dtype=torch.long), ref_spk_embedding=torch.zeros(8),
                                x_vector_only_mode=False, icl_mode=True, ref_text="ref")
    wavs, fs = m.generate_voice_clone(["t1", "t2"], language="english", voice_clone_prompt=[item])
    # decoded length (6+4)*1920, cut int(6/10*len) == 6*1920 (qwen3_tts_model.py:622-631)
    assert [w.shape[0] for w in wavs] == [4 * 1920, 5 * 1920]
    assert wavs[0][0] == 6 * 1920
    kw = core.calls[-1]
    assert kw["non_streaming_mode"] is False and len(kw["ref_ids"]) == 2 and kw["voice_clone_prompt"]["icl_mode"] == [True, True]
    with pytest.raises(ValueError):
        m.generate_voice_clone("t")


def test_tokenizer_audio_input_normalisation():
    """inference/qwen3_tts_tokenizer.py:100-207 — ndarray(+sr) / list / base64 / data-URL / wav path; error behaviour."""
    import base64
    import io
    import numpy as np
    from scipy.io import wavfile
    from qwen3_tts_b200.model import Qwen3TTSTokenizer as T
    a = (np.sin(np.arange(16000) * 0.05) * 0.3).astype(np.float32)
    out = T._normalize_audio_inputs([a, np.stack([a[:8000], a[:8000]], -1)], sr=16000)   # stereo -> mono, 16k -> 24k
    assert [o.shape for o in out] == [(24000,), (12000,)] and out[0].dtype == np.float32
    assert T._normalize_audio_inputs(a, sr=24000)[0] is not None and T._normalize_audio_inputs([], None) == []
    buf = io.BytesIO()
    wavfile.write(buf, 24000, (a * 32767).astype(np.int16))
    b64 = base64.b64encode(buf.getvalue()).decode()
    w = T._normalize_audio_inputs("data:audio/wav;base64," + b64, None)[0]
    assert w.shape == a.shape and np.abs(w - a).max() < 1e-4
    # raw base64 is only recognised when it has no '/' (the reference's heuristic, :100-107) -- same quirk here
    assert T._is_probably_base64("A" * 300) and not T._is_probably_base64("A" * 300 + "/")
    with pytest.raises(ValueError):
        T._normalize_audio_inputs(a, None)
    with pytest.raises(TypeError):
        T._normalize_audio_inputs([a, "x.wav"], 24000)
    assert T._is_url("https://example.com/a.wav") and not T._is_url("/tmp/a.wav")


def test_create_voice_clone_prompt_host_logic():
    """inference/qwen3_tts_model.py:355-458 with fake engines: broadcasting, ICL vs x-vector-only items, resampling to
    the speaker encoder's rate, single batched encode when all sampling rates agree, error behaviour."""
    from types import SimpleNamespace

    class _Tok(_FakeTok):
        def __init__(self):
            self.calls = []

        def encode(self, audios, sr=None, return_dict=True):
            lst = audios if isinstance(audios, list) else [audios]
            self.calls.append((len(lst), sr))
            return SimpleNamespace(audio_codes=[torch.full((-(-len(a) * 24000 // sr // 1920), 16), i, dtype=torch.long)
                                                for i, a in enumerate(lst)])

    core = _FakeCore()
    core.speech_tokenizer = _Tok()
    core.speaker_encoder_sample_rate = 24000
    core.tts_model_size = "1b7"
    seen = []

    def extract(audio, sr):
        seen.append((audio.shape[0], sr, audio.dtype))
        return torch.full((8,), float(audio.shape[0]))

    core.extract_speaker_embedding = extract
    m = Qwen3TTSModel(core, _proc)
    a = np.zeros(24000, np.float32)
    with pytest.raises(ValueError):                       # custom_voice models cannot build clone prompts (:400-406)
        m.create_voice_clone_prompt((a, 24000), "hi")
    core.tts_model_type = "base"
    items = m.create_voice_clone_prompt([(a, 24000), (np.zeros((12000, 2), np.float32), 24000)], ref_text=["one", None],
                                        x_vector_only_mode=[False, True])
    assert core.speech_tokenizer.calls == [(2, 24000)]   # same sr -> one batched encode (:423-425)
    assert [it.icl_mode for it in items] == [True, False] and [it.x_vector_only_mode for it in items] == [False, True]
    assert items[0].ref_code.shape == (13, 16) and items[1].ref_code is None and items[0].ref_text == "one"
    assert seen == [(24000, 24000, np.float32), (12000, 24000, np.float32)]   # stereo was mixed down
    # different sampling rates -> per-item encode, x-vector input resampled to 24 kHz (:426-445)
    seen.clear()
    core.speech_tokenizer.calls.clear()
    items = m.create_voice_clone_prompt([(a, 24000), (np.zeros(16000, np.float32), 16000)], ref_text="same text")
    assert core.speech_tokenizer.calls == [(1, 24000), (1, 16000)] and [s[0] for s in seen] == [24000, 24000]
    assert all(it.ref_text == "same text" and it.icl_mode for it in items)
    with pytest.raises(ValueError):                       # ICL needs a transcript
        m.create_voice_clone_prompt((a, 24000))
    with pytest.raises(ValueError):                       # batch mismatch
        m.create_voice_clone_prompt([(a, 24000), (a, 24000)], ref_text=["x"], x_vector_only_mode=[True, True])
    with pytest.raises(ValueError):                       # bare ndarray needs its sampling rate
        m.create_voice_clone_prompt(a, "hi")
    with pytest.raises(TypeError):
        m.create_voice_clone_prompt(123, "hi")
    # and the items feed generate_voice_clone unchanged
    wavs, fs = m.generate_voice_clone("t", language="english", ref_audio=(a, 24000), ref_text="r")
    assert fs == 24000 and len(wavs) == 1


def test_public_names_match_the_reference_package():
    """qwen_tts/__init__.py:21-22 exports exactly these three names."""
    from qwen3_tts_b200 import Qwen3TTSModel as A, Qwen3TTSTokenizer as B, VoiceClonePromptItem as C
    from qwen3_tts_b200 import model
    assert A is model.Qwen3TTSModel and B is model.Qwen3TTSTokenizer and C is model.VoiceClonePromptItem
    assert all(hasattr(A, n) for n in ("from_pretrained", "generate_custom_voice", "generate_voice_design",
                                       "generate_voice_clone", "create_voice_clone_prompt", "get_supported_speakers",
                                       "get_supported_languages"))
    assert all(hasattr(B, n) for n in ("from_pretrained", "encode", "decode", "get_model_type", "get_input_sample_rate",
                                       "get_output_sample_rate", "get_encode_downsample_rate", "get_decode_upsample_rate"))


def _stream_engine(monkeypatch, codec_max=64, eos_at=None):
    """A TTSEngine over the fake engine of test_scheduler_cpu.py (row b's frame t has every code b * 100 + t) and the
    seeding codec of test_scheduler_voice_clone_cpu.py, given a causal forward: the running sum of the codes."""
    from qwen3_tts_b200.engine import AREngine
    from qwen3_tts_b200.pipeline import TTSEngine
    from tests.test_scheduler_cpu import FakeEngine, _mock_sync
    from tests.test_scheduler_voice_clone_cpu import SeedingCodec, SeedingStream
    from qwen3_tts_b200.codec import CodecStream
    _mock_sync(monkeypatch)

    class _AR(FakeEngine):
        _frame_budget = AREngine._frame_budget

    class _Stream(SeedingStream, CodecStream):
        pass

    class _Codec(SeedingCodec):
        def open_stream(self, batch, max_packet_frames=8):
            self.stream = _Stream(batch, max_packet_frames, self.log)
            self.stream.dec = self
            return self.stream

        def forward(self, codes):                       # (B, K, T) -> (B, 1, T*up), repeated `up` times
            self.log.append(("forward", tuple(codes.shape)))
            return codes.sum(1).cumsum(-1).float().repeat_interleave(self.total_upsample, dim=-1)[:, None, :]

    eng = object.__new__(TTSEngine)
    eng.device, eng.ar, eng.codec = torch.device("cpu"), _AR(eos_at), _Codec(codec_max)
    eng.codec_cfg = eng.codec.cfg
    return eng


def test_stream_synthesize_on_the_batcher_equals_per_row_decoding(monkeypatch):
    """pipeline.TTSEngine.stream_synthesize runs the rows as one ContinuousBatcher session.  The windowed modes group
    rows with equal window shapes into one codec call, and their packets must equal what per-row decoding with the same
    left context yields; the stateful mode hands out each row's own frames of the codec stream (ragged finish)."""
    from qwen3_tts_b200.config import SamplingParams
    eng = _stream_engine(monkeypatch, eos_at={1: 7})                            # row 1 finishes early
    up, K = eng.codec.total_upsample, eng.codec_cfg.num_quantizers
    full = [(b * 100 + torch.arange(n))[:, None].expand(n, K) for b, n in enumerate((10, 7, 10))]
    z = [torch.zeros(1, 8)] * 3
    sp = SamplingParams(max_new_tokens=11)
    for lc in (None, 2, "stateful"):
        eng.codec.log.clear()
        parts = [[] for _ in full]
        for pkt in eng.stream_synthesize(z, z, torch.zeros(8), sp, packet_frames=4, left_context=lc):
            assert len(pkt) == 3 and all(w.dtype == np.float32 for w in pkt)
            for b, w in enumerate(pkt):
                parts[b].append(w)
        for b, f in enumerate(full):
            want, hist = [], 0
            for s0 in range(0, f.shape[0], 4):
                new = f[s0:s0 + 4]
                if lc == "stateful":
                    want.append(new[:, 0].float().repeat_interleave(up).numpy())
                else:
                    ctx = hist if lc is None else min(lc, hist)
                    win = torch.cat([f[hist - ctx:hist], new], 0)
                    want.append(eng.codec.forward(win.t()[None])[0, 0, ctx * up:].numpy())
                hist += new.shape[0]
            assert np.array_equal(np.concatenate(parts[b]), np.concatenate(want))
            assert np.concatenate(parts[b]).shape[0] == f.shape[0] * up
        if lc != "stateful":   # packet 0: all three rows in one codec call
            assert next(e for e in eng.codec.log if e[0] == "forward")[1][0] == 3


def test_stream_synthesize_zero_budget_and_seeded_horizon(monkeypatch):
    """A zero-frame budget yields no packet in any mode; a seeded row's horizon leaves the codec's RoPE table room for
    its reference (codec max_frames 12, reference of 7 frames: 5 frames), the other row runs to its budget."""
    from qwen3_tts_b200.config import SamplingParams
    from tests.test_scheduler_voice_clone_cpu import _ref
    eng = _stream_engine(monkeypatch, codec_max=12)
    z = [torch.zeros(1, 8)] * 2
    for lc in (None, 2, "stateful"):
        assert list(eng.stream_synthesize(z, z, torch.zeros(8), SamplingParams(max_new_tokens=1), left_context=lc)) == []
    pkts = list(eng.stream_synthesize(z, z, torch.zeros(8), SamplingParams(max_new_tokens=11), packet_frames=4,
                                      ref_codes=[_ref(7, 1), None]))
    up = eng.codec.total_upsample
    assert [sum(p[b].shape[0] for p in pkts) for b in range(2)] == [5 * up, 10 * up]
    assert [e[0] for e in eng.codec.log[:2]] == ["reset", "seed"]
    assert max(max(e[2]) for e in eng.codec.log if e[0] == "push") <= 12


def test_batched_prefill_assembly_equals_per_sample_restatement():
    """build_prefill (batched gathers / one ResizeMLP for every text token of every sample, SURVEY §8f-3) must equal the
    statement-by-statement restatement of modeling_qwen3_tts.py:2068-2237 exactly, in bf16, for every mode mix:
    instruct / no instruct, known language / auto / dialect override, speaker id / x-vector / ICL, streaming and not."""
    from oracle import talker as OT
    from tests import helpers as Hh
    from qwen3_tts_b200.model import Qwen3TTSForConditionalGenerationB200 as M
    cfg = OT.cfg_tiny()
    W = OT.random_weights(cfg, seed=4, with_text=True, text_vocab=1000)
    spk_id = {"alice": 3000, "bob": 3001}
    lang = {"english": 2050, "chinese": 2055, "sichuan_dialect": 2060}
    dial = {"alice": False, "bob": "sichuan_dialect"}
    m = M.__new__(M)
    M.__init__(m, Hh.to_pkg_cfg(cfg), {k: v.to(torch.bfloat16) for k, v in W.items()}, device="cpu", spk_id=spk_id, spk_is_dialect=dial,
               codec_language_id=lang, engine=object())
    # Both paths project one text token per ResizeMLP call: a CPU BLAS may accumulate a row of a bf16 GEMM in an order
    # that depends on how many rows the call has, and the assembly (what this test checks) must be exact regardless.
    tp = m._tp
    m._tp = lambda t: torch.cat([tp(t[:, j:j + 1]) for j in range(t.shape[1])], dim=1) if t.shape[1] else tp(t)  # noqa: E731
    g = torch.Generator().manual_seed(1)
    ids = lambda n: torch.randint(0, 990, (1, n), generator=g)  # noqa: E731
    H = cfg.talker.hidden_size

    def same(a, b):
        ea, ta, pa = a
        eb, tb, pb = b
        assert len(ea) == len(eb)
        for x, y in zip(ea + ta + [pa], eb + tb + [pb]):
            assert x.shape == y.shape and torch.equal(x, y), (x.shape, y.shape, (x.float() - y.float()).abs().max())

    for nsm in (False, True):
        # custom voice / voice design: instruct on some rows, dialect override, auto language, no speaker
        kw = dict(input_ids=[ids(14), ids(10), ids(21)], instruct_ids=[ids(6), None, ids(9)], languages=["English", "auto", "Chinese"],
                  speakers=["alice", "bob", None], non_streaming_mode=nsm)
        same(m.build_prefill(**kw), m.build_prefill_per_sample(**kw))
        # voice clone: ICL (text longer and shorter than the reference codes) and x-vector-only rows
        vcp = dict(ref_spk_embedding=[torch.randn(H, generator=g), torch.randn(H, generator=g), torch.randn(H, generator=g)],
                   x_vector_only_mode=[False, True, False], icl_mode=[True, False, True],
                   ref_code=[torch.randint(0, 2000, (5, 16), generator=g), None, torch.randint(0, 2000, (30, 16), generator=g)])
        kw = dict(input_ids=[ids(25), ids(12), ids(13)], ref_ids=[ids(11), None, ids(9)], voice_clone_prompt=vcp,
                  languages=["English", "auto", "English"], non_streaming_mode=nsm)
        same(m.build_prefill(**kw), m.build_prefill_per_sample(**kw))
