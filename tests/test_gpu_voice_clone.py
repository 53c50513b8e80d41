"""Checkpoint loading and voice cloning from raw audio, end to end on the GPU (BASELINE config 5 in miniature)."""
import numpy as np
import pytest
import torch

from tests.test_gpu_e2e import DEV, _build, _proc

pytestmark = pytest.mark.gpu


def test_voice_clone_from_raw_audio_end_to_end(tmp_path):
    """BASELINE config 5 in miniature: Base checkpoint -> create_voice_clone_prompt(raw 24 kHz audio + transcript)
    (codec encoder for ref_code, speaker encoder for the x-vector) -> generate_voice_clone (ICL prefill, AR decode, codec
    decode, proportional cut).  Shapes, determinism and the x-vector-only variant; no audio-quality claim (random weights)."""
    from tests.helpers import write_tiny_checkpoint
    from qwen3_tts_b200.model import Qwen3TTSModel
    write_tiny_checkpoint(str(tmp_path), device=DEV, seed=0, model_type="base", spk_enc_dim=256)   # x-vector width == talker hidden
    m = Qwen3TTSModel.from_pretrained(str(tmp_path), device_map=DEV, processor=_proc, max_batch=8, max_ctx=256, codec_max_frames=128)
    assert m.model.tts_model_type == "base" and m.model.speaker_encoder is not None
    g = np.random.default_rng(0)
    ref = (np.clip(g.standard_normal(9000).astype(np.float32) * 0.1, -1, 1), 24000)
    items = m.create_voice_clone_prompt([ref, ref], ref_text=["reference words", None], x_vector_only_mode=[False, True])
    assert tuple(items[0].ref_code.shape) == (5, 16) and items[1].ref_code is None
    assert tuple(items[0].ref_spk_embedding.shape) == (256,) and torch.equal(items[0].ref_spk_embedding, items[1].ref_spk_embedding)
    kw = dict(max_new_tokens=7, do_sample=True, seed=3)
    wavs, fs = m.generate_voice_clone(["hello there", "second"], language="english", voice_clone_prompt=items, **kw)
    assert fs == 24000 and len(wavs) == 2
    for w in wavs:
        assert w.dtype == np.float32 and 0 < w.shape[0] <= 6 * 1920 + 1920 and np.isfinite(w).all()
    again, _ = m.generate_voice_clone(["hello there", "second"], language="english", voice_clone_prompt=items, **kw)
    assert all(np.array_equal(a, b) for a, b in zip(wavs, again))
    one, _ = m.generate_voice_clone("hello there", language="english", ref_audio=ref, ref_text="reference words", **kw)
    assert np.array_equal(one[0], wavs[0])


def test_from_pretrained_equals_direct_construction(tmp_path):
    """A checkpoint directory in the reference's on-disk format (config.json, safetensors, speech_tokenizer/,
    generation_config.json) loaded through Qwen3TTSModel.from_pretrained produces the same waveforms as the model
    built directly from the same tensors; the loaded tokenizer also encodes."""
    from tests.helpers import write_tiny_checkpoint
    from qwen3_tts_b200.model import Qwen3TTSModel
    write_tiny_checkpoint(str(tmp_path), device=DEV, seed=0)
    m2 = Qwen3TTSModel.from_pretrained(str(tmp_path), device_map=DEV, processor=_proc, max_batch=8, max_ctx=256,
                                       codec_max_frames=128)
    cfg, core, m = _build()
    kw = dict(max_new_tokens=9, do_sample=True, top_k=50, top_p=1.0, temperature=0.9, repetition_penalty=1.05,
              subtalker_dosample=True, subtalker_top_k=50, subtalker_top_p=1.0, subtalker_temperature=0.9, seed=7)
    args = (["hello there", "x"],)
    a, _ = m.generate_custom_voice(*args, speaker=["alice", "bob"], language=["english", "auto"], **kw)
    b, fs = m2.generate_custom_voice(*args, speaker=["alice", "bob"], language=["english", "auto"], **kw)
    assert fs == 24000 and all(np.array_equal(x, y) for x, y in zip(a, b))
    assert m2.generate_defaults["top_k"] == 40 and m2.get_supported_speakers() == ["alice", "bob"]
    codes = m2.model.speech_tokenizer.encode(np.zeros(6000, np.float32), sr=24000).audio_codes
    assert tuple(codes[0].shape) == (4, 16) and codes[0].dtype == torch.long
