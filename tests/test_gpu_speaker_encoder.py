"""GPU parity of the speaker x-vector path (csrc/speaker_encoder.cu through the C ABI) against the CPU oracle
(oracle/speaker_encoder.py, itself bit-identical to the reference's Qwen3TTSSpeakerEncoder / mel_spectrogram)."""
import os

import numpy as np
import pytest
import torch

from oracle import speaker_encoder as S

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RTOL = 1e-3   # max |gpu - oracle| / max |oracle| (fp32 both; direct DFT vs FFT, different summation orders)


def _pkg_cfg(c):
    from qwen3_tts_b200.config import SpeakerEncoderConfig
    return SpeakerEncoderConfig(**{k: getattr(c, k) for k in S.SpkEncCfg.__dataclass_fields__})


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-20))


@pytest.mark.parametrize("which,T", [("tiny", 6000), ("tiny", 1500), ("default", 24000)])
def test_mel_and_embedding_match_oracle(which, T):
    from qwen3_tts_b200.speaker_encoder import SpeakerEncoder
    cfg = S.cfg_tiny_spk() if which == "tiny" else S.SpkEncCfg()
    W = S.random_weights(cfg, seed=1)
    enc = SpeakerEncoder(_pkg_cfg(cfg), W, device=DEV)
    g = torch.Generator().manual_seed(T)
    wav = (torch.randn(2, T, generator=g) * 0.1).clamp(-1, 1)
    mel_ref = S.mel_spectrogram(wav, num_mels=cfg.mel_dim)
    mel = enc.mel(wav.to(DEV)).cpu()
    assert mel.shape == mel_ref.shape and _rel(mel, mel_ref) < RTOL
    emb_ref = S.speaker_encoder(W, cfg, mel_ref.transpose(1, 2))
    emb = enc.forward(mel_ref.transpose(1, 2).to(DEV)).cpu()        # same mel in: isolates the ECAPA part
    assert emb.shape == emb_ref.shape == (2, cfg.enc_dim) and _rel(emb, emb_ref) < RTOL
    e2e = enc.embed_waveform(wav.to(DEV)).cpu()                     # waveform in: both stages
    assert _rel(e2e, emb_ref) < 5 * RTOL and enc.last_launches() > 0


def test_golden_vectors():
    from qwen3_tts_b200.speaker_encoder import SpeakerEncoder
    z = np.load(os.path.join(GOLD, "speaker_micro.npz"))
    cfg = S.cfg_tiny_spk()
    W = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("W::")}
    enc = SpeakerEncoder(_pkg_cfg(cfg), W, device=DEV)
    wav = torch.from_numpy(z["wav"])
    assert _rel(enc.mel(wav.to(DEV)).cpu(), torch.from_numpy(z["mel"])) < RTOL
    assert _rel(enc.embed_waveform(wav.to(DEV)).cpu(), torch.from_numpy(z["emb"])) < 5 * RTOL
