"""Pin the oracle against the reference's OWN modules.

The reference ships no tests or golden vectors (SURVEY §4).  oracle/make_golden.py (`reference`) ran the reference's
modules on these tests' seeded weights and inputs and recorded what they returned in tests/golden/reference_checks.*
(large outputs as a fixed, seeded sample of columns / positions, argmax rows in full); the oracle is held to those
recordings here, so the pin holds on every machine.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import talker as T
from oracle.make_golden import _sig

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
Z = np.load(os.path.join(GOLD, "reference_checks.npz"))
META = json.load(open(os.path.join(GOLD, "reference_checks.json")))


def test_talker_and_code_predictor_teacher_forced():
    cfg = T.cfg_tiny()
    cfg.talker.rope_theta = 1e6
    cfg.cp.rope_theta = 1e4
    W = T.random_weights(cfg, seed=1)
    torch.manual_seed(0)
    lens, H = [5, 9, 7], cfg.talker.hidden_size
    embs = [torch.randn(l, H) * 0.5 for l in lens]
    trail = [torch.randn(n, H) * 0.1 for n in (2, 1, 4)]
    pad = torch.randn(H) * 0.1
    sp = T.SamplingCfg(do_sample=False, subtalker_dosample=False, max_new_tokens=6, suppress_eos=True)
    r = T.generate(W, cfg, embs, trail, pad, sp, record_logits=True)
    assert r.codes[0].shape[0] == 5
    codes = torch.stack(r.codes)  # (B,N,16): the codes the reference was driven with
    assert (codes.numpy() == Z["tf_codes"]).all()
    tl, cl = np.stack(r.record["talker_logits"]), np.stack(r.record["cp_logits"])
    ct, cc = Z["tf_talker_cols"], Z["tf_cp_cols"]
    assert np.abs(tl[0][..., ct] - Z["tf_talker"][0]).max() < 2e-5                 # prefill
    assert np.abs(tl[1:][..., ct] - Z["tf_talker"][1:]).max() < 3e-5               # decode steps
    assert np.abs(cl[..., cc] - Z["tf_cp"]).max() < 2e-5
    assert (tl.argmax(-1) == Z["tf_talker_argmax"]).all() and (cl.argmax(-1) == Z["tf_cp_argmax"]).all()
    G = cfg.num_code_groups
    for step in range(codes.shape[1]):
        for j in range(G - 1):
            assert (np.argmax(cl[step * (G - 1) + j], -1) == codes[:, step, j + 1].numpy()).all()


def test_leaf_ops_match_reference():
    torch.manual_seed(0)
    x = torch.randn(2, 5, 64)
    w = torch.randn(64)
    assert torch.equal(T.rms_norm(x, w, 1e-6), torch.from_numpy(Z["leaf_rms"]))
    assert torch.equal(T.rms_norm(x.bfloat16(), w.bfloat16(), 1e-6).float(), torch.from_numpy(Z["leaf_rms_bf16"]))
    assert torch.equal(T.rotate_half(x), torch.from_numpy(Z["leaf_rotate_half"]))


def _codec(cfg, name, seed=3):
    from oracle import codec as C
    W = C.random_weights(cfg, seed=seed)
    assert _sig((k, v.shape) for k, v in W.items()) == META[f"codec_{name}_sig"]   # same names and shapes as the reference
    return W


def test_codec_decoder_tiny_matches_reference():
    from oracle import codec as C
    cfg = C.cfg_tiny_codec()
    W = _codec(cfg, "tiny")
    g = torch.Generator().manual_seed(5)
    codes = torch.randint(0, cfg.codebook_size, (2, 16, 13), generator=g)
    out = C.decoder_forward(W, cfg, codes)
    assert out.shape == tuple(Z["codec_tiny_shape"]) == (2, 1, 13 * 1920)
    assert np.abs(out.numpy()[..., Z["codec_tiny_pos"]] - Z["codec_tiny"]).max() < 2e-5
    assert abs(float(out.abs().max()) - float(Z["codec_tiny_absmax"])) < 2e-5
    assert out.abs().max() > 0.05  # not a degenerate all-zero / all-clamped signal
    # chunked decode with several chunks + wrapper semantics (pad -1, trim)
    codes_long = torch.randint(0, cfg.codebook_size, (2, 16, 40), generator=g)
    out_c = C.chunked_decode(W, cfg, codes_long, chunk_size=16, left_context_size=5)
    assert np.abs(out_c.numpy()[..., Z["codec_chunked_pos"]] - Z["codec_chunked"]).max() < 2e-5


def test_codec_decoder_default_shapes_names():
    """Full default config: parameter names/shapes line up with the reference (195.08 M params)."""
    from oracle import codec as C
    cfg = C.CodecCfg()
    W = _codec(cfg, "default")
    assert sum(v.numel() for v in W.values()) == META["codec_default_numel"]
    torch.manual_seed(0)
    codes = torch.randint(0, cfg.codebook_size, (1, 16, 3))
    assert (codes.numpy() == Z["codec_default_codes"]).all()
    out = C.decoder_forward(W, cfg, codes)
    assert (out - torch.from_numpy(Z["codec_default"])).abs().max() < 5e-5


@pytest.mark.parametrize("which", ["tiny", "default"])
def test_speaker_encoder_and_mel_match_reference(which):
    """ECAPA-TDNN x-vector (modeling_qwen3_tts.py:300-393) and the log-mel front end (:396-448).  The mel FILTERBANK is
    librosa's (absent): the reference function was run with oracle.speaker_encoder's restatement patched in, so STFT,
    magnitude, projection and log are pinned; the filterbank itself stays 'parity unpinned'."""
    from oracle import speaker_encoder as S
    cfg = S.cfg_tiny_spk() if which == "tiny" else S.SpkEncCfg()
    W = S.random_weights(cfg, seed=1)
    assert _sig((k, v.shape) for k, v in W.items()) == META[f"spk_{which}_sig"]  # every reference parameter has a counterpart
    torch.manual_seed(0)
    mels = torch.randn(2, 57, cfg.mel_dim)
    assert (torch.from_numpy(Z[f"spk_{which}_emb"]) - S.speaker_encoder(W, cfg, mels)).abs().max() < 1e-5
    y = (torch.randn(2, 9000) * 0.1).clamp(-1, 1)
    assert (torch.from_numpy(Z[f"spk_{which}_mel"]) - S.mel_spectrogram(y, num_mels=cfg.mel_dim)).abs().max() < 1e-5
    fb = S.slaney_mel_filterbank(24000, 1024, 128, 0, 12000)
    assert fb.shape == (128, 513) and (fb >= 0).all() and (fb.sum(1) > 0).all()
