"""End-to-end on the GPU through the public mirror: Qwen3TTSModel.generate_custom_voice -> composite generate (a1,
PyTorch host) -> fused AR engine (seam B) -> codec engine (seam C) -> numpy waveforms; plus the streaming API."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _proc(text=None, return_tensors="pt", padding=True):
    body = [(ord(c) * 7) % 900 for c in text if c not in "<|>"][:12]
    return {"input_ids": torch.tensor([[1, 2, 3] + body + [4, 5, 6, 7, 8]])}


def _build():
    import qwen3_tts_b200 as q
    from qwen3_tts_b200 import synthetic
    from qwen3_tts_b200.model import Qwen3TTSForConditionalGenerationB200, Qwen3TTSModel, Qwen3TTSTokenizer
    cfg = synthetic.cfg_tiny()
    W = synthetic.random_tts_weights(cfg, device=DEV, seed=0, with_text=True, text_vocab=1000)
    ccfg = q.CodecConfig(codebook_size=2048, codebook_dim=64, hidden_size=64, latent_dim=64, num_heads=4, num_kv_heads=4,
                         head_dim=16, sliding_window=6, intermediate_size=96, num_layers=2, decoder_dim=256)
    CW = synthetic.random_codec_weights(ccfg, device=DEV, seed=0)
    core = Qwen3TTSForConditionalGenerationB200(cfg, W, device=DEV, spk_id={"alice": 3000, "bob": 3001},
                                                spk_is_dialect={"alice": False, "bob": False},
                                                codec_language_id={"english": 2050, "chinese": 2055}, max_batch=8, max_ctx=256)
    core.load_speech_tokenizer(Qwen3TTSTokenizer(ccfg, CW, device=DEV, max_frames=128))
    return cfg, core, Qwen3TTSModel(core, _proc)


def test_custom_voice_end_to_end_and_determinism():
    cfg, core, m = _build()
    kw = dict(max_new_tokens=9, do_sample=True, seed=7)
    wavs, fs = m.generate_custom_voice(["hello there", "a much longer sentence here", "x"], speaker=["alice", "bob", "alice"],
                                       language=["english", "auto", "chinese"], instruct=[None, "speak slowly", ""], **kw)
    assert fs == 24000 and len(wavs) == 3
    for w in wavs:
        assert w.dtype == np.float32 and w.ndim == 1 and w.shape[0] % 1920 == 0 and w.shape[0] <= 8 * 1920
        assert np.isfinite(w).all() and np.abs(w).max() <= 1.0
    wavs2, _ = m.generate_custom_voice(["hello there", "a much longer sentence here", "x"], speaker=["alice", "bob", "alice"],
                                       language=["english", "auto", "chinese"], instruct=[None, "speak slowly", ""], **kw)
    assert all(np.array_equal(a, b) for a, b in zip(wavs, wavs2))  # per-request state lives in the engine, seeded
    # batch rows are independent: row 0 alone reproduces row 0 of the batch
    solo, _ = m.generate_custom_voice("hello there", speaker="alice", language="english", **kw)
    assert np.array_equal(solo[0], wavs[0])


def test_batcher_packets_equal_one_shot():
    import qwen3_tts_b200 as q
    from qwen3_tts_b200.scheduler import ContinuousBatcher
    cfg, core, m = _build()
    ids = [_proc(text=f"<|im_start|>assistant\n{t}<|im_end|>\n<|im_start|>assistant\n")["input_ids"] for t in ("abc def", "ghi")]
    emb, trail, pad = core.build_prefill(ids, None, None, None, ["english", "english"], ["alice", "bob"], False)
    sp = q.SamplingParams(max_new_tokens=14, suppress_eos=True, seed=3)
    one = core.engine.generate(emb, trail, pad, sp)
    cb = ContinuousBatcher(core.engine, pad, sp, n_slots=len(emb), packet_frames=4)
    for b in range(len(emb)):
        cb.submit(emb[b], trail[b], key=b)
    parts = [[] for _ in emb]
    for new, _ in cb.packets():
        for b, p in new.items():
            parts[b].append(p)
    for b in range(len(emb)):
        assert torch.equal(torch.cat(parts[b]), one[b]) and one[b].shape == (13, 16)


def test_stream_synthesize_full_prefix_equals_one_shot_decode():
    """Packetised audio: with the whole prefix as left context the concatenated packets equal the one-shot causal
    decode bit for bit (decoder causality, SURVEY F9); with the reference's 25-frame context the first packets
    (<= 25 frames of history) are identical too."""
    import qwen3_tts_b200 as q
    from qwen3_tts_b200 import synthetic
    from qwen3_tts_b200.pipeline import TTSEngine
    cfg = synthetic.cfg_tiny()
    ccfg = q.CodecConfig(codebook_size=2048, codebook_dim=64, hidden_size=64, latent_dim=64, num_heads=4, num_kv_heads=4,
                         head_dim=16, sliding_window=6, intermediate_size=96, num_layers=2, decoder_dim=256)
    eng = TTSEngine(cfg, synthetic.random_tts_weights(cfg, device=DEV, seed=0), ccfg,
                    synthetic.random_codec_weights(ccfg, device=DEV, seed=0), device=DEV, max_batch=4, max_ctx=128, codec_max_frames=64)
    H = cfg.talker.hidden_size
    g = torch.Generator().manual_seed(1)
    embs = [(torch.randn(n, H, generator=g) * 0.5).bfloat16() for n in (5, 8)]
    trail = [torch.zeros(0, H, dtype=torch.bfloat16)] * 2
    pad = (torch.randn(H, generator=g) * 0.1).bfloat16()
    sp = q.SamplingParams(max_new_tokens=11, suppress_eos=True, seed=5)
    wavs, codes = eng.synthesize(embs, trail, pad, sp)
    for lc in ("stateful", None, 25):  # stateful codec stream (default), whole-prefix re-decode, the reference's 25-frame context
        parts = [[] for _ in embs]
        for pkt in eng.stream_synthesize(embs, trail, pad, sp, packet_frames=4, left_context=lc):
            for b, w in enumerate(pkt):
                parts[b].append(w)
        for b in range(2):
            assert np.array_equal(np.concatenate(parts[b]), wavs[b])
    eng.close()
