"""Oracle against the committed golden vectors (minted from the reference's own modules by oracle/make_golden.py).
Runs everywhere, including the GPU box where /root/reference does not exist."""
import os

import numpy as np
import torch

from oracle import codec as OC, talker as OT
from oracle.make_golden import micro_codec_cfg, micro_tts_cfg

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _weights(z):
    return {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("W::")}


def test_talker_and_code_predictor_against_golden_logits():
    z = np.load(os.path.join(GOLD, "talker_micro.npz"))
    cfg = micro_tts_cfg()
    W = OT.random_weights(cfg, seed=11, with_text=False)  # the weights the golden logits were minted with
    embs = [torch.from_numpy(z["emb0"]), torch.from_numpy(z["emb1"])]
    trail = [torch.from_numpy(z["trail0"]), torch.from_numpy(z["trail1"])]
    codes = z["codes"]
    N = codes.shape[1]
    sp = OT.SamplingCfg(do_sample=False, subtalker_dosample=False, max_new_tokens=N + 1, suppress_eos=True)
    r = OT.generate(W, cfg, embs, trail, torch.from_numpy(z["pad"]), sp, record_logits=True, forced_codes=codes)
    tl = np.stack(r.record["talker_logits"])
    cl = np.stack(r.record["cp_logits"])
    assert tl.shape == z["talker_logits"].shape and cl.shape == z["cp_logits"].shape
    assert np.abs(tl - z["talker_logits"]).max() < 5e-5
    assert np.abs(cl - z["cp_logits"]).max() < 5e-5
    assert all((c.numpy() == codes[b]).all() for b, c in enumerate(r.codes))


def test_codec_decoder_against_golden_wav():
    z = np.load(os.path.join(GOLD, "codec_micro.npz"))
    cfg = micro_codec_cfg()
    W = _weights(z)
    codes = torch.from_numpy(z["codes"])
    wav = OC.decoder_forward(W, cfg, codes)
    assert wav.shape == z["wav"].shape == (2, 1, 9 * 1920)
    assert np.abs(wav.numpy() - z["wav"]).max() < 5e-5
    wav_c = OC.chunked_decode(W, cfg, codes, chunk_size=4, left_context_size=2)
    assert np.abs(wav_c.numpy() - z["wav_chunked"]).max() < 5e-5
    # self-consistency the reference guarantees by construction (SURVEY §8c): causality and length
    pre = OC.decoder_forward(W, cfg, codes[..., :5])
    assert torch.allclose(pre, wav[..., :5 * 1920], atol=1e-5)
    outs = OC.decode(W, cfg, torch.cat([codes.transpose(1, 2), -torch.ones(2, 3, 16, dtype=torch.long)], 1))
    assert [o.numel() for o in outs] == [9 * 1920] * 2


def test_speaker_encoder_against_golden():
    """x-vector path (voice cloning, SURVEY §8f-3): log-mel front end and ECAPA-TDNN against vectors minted from the
    reference's own modules."""
    from oracle import speaker_encoder as OS
    z = np.load(os.path.join(GOLD, "speaker_micro.npz"))
    cfg = OS.cfg_tiny_spk()
    W = _weights(z)
    wav = torch.from_numpy(z["wav"])
    mel = OS.mel_spectrogram(wav, num_mels=cfg.mel_dim)
    assert mel.shape == z["mel"].shape and np.abs(mel.numpy() - z["mel"]).max() < 1e-4
    emb = OS.speaker_encoder(W, cfg, torch.from_numpy(z["mel"]).transpose(1, 2))
    assert np.abs(emb.numpy() - z["emb"]).max() < 1e-5
    assert np.abs(OS.extract_speaker_embedding(W, cfg, wav[0]).numpy() - z["emb"][0]).max() < 1e-4


def test_streaming_decoder_spec_equals_full_forward():
    """oracle/codec.py::StreamingDecoder (the per-layer history a stateful codec decoder must carry, SURVEY §8f-2):
    ragged packets concatenated == one causal forward over all frames, incl. the sliding-window KV trim (window 6 < 23
    frames) and a batch of two rows."""
    cfg = OC.cfg_tiny_codec()
    W = OC.random_weights(cfg, seed=4)
    g = torch.Generator().manual_seed(0)
    codes = torch.randint(0, cfg.codebook_size, (2, 16, 23), generator=g)
    full = OC.decoder_forward(W, cfg, codes)
    sd = OC.StreamingDecoder(W, cfg, batch=2)
    outs, s = [], 0
    for n in (4, 4, 1, 7, 2, 5):
        outs.append(sd.push(codes[..., s:s + n]))
        s += n
    out = torch.cat(outs, -1)
    assert out.shape == full.shape and (out - full).abs().max() < 2e-5
    # unlike the reference's chunked_decode, which drifts from the full forward after its first chunk (SURVEY F9)
    ch = OC.chunked_decode(W, cfg, codes, chunk_size=8, left_context_size=2)
    assert (ch - full).abs().max() > 1e-3


def test_oracle_rows_are_independent_and_padding_invariant():
    """SURVEY §8e: utterances never interact (batching is left-padding + masking, modeling_qwen3_tts.py:2239-2254).
    Greedy codes of a row must not depend on what else is in the batch, nor on how far it is left-padded — the property
    that makes the data-parallel split (and the engine's unpadded per-row prefill) exact."""
    cfg = OT.cfg_tiny()
    W = OT.random_weights(cfg, seed=2, with_text=False)
    g = torch.Generator().manual_seed(3)
    H = cfg.talker.hidden_size
    embs = [torch.randn(n, H, generator=g) * 0.5 for n in (4, 11, 7)]
    trail = [torch.randn(n, H, generator=g) * 0.1 for n in (0, 3, 1)]
    pad = torch.randn(H, generator=g) * 0.1
    sp = OT.SamplingCfg(do_sample=False, subtalker_dosample=False, max_new_tokens=6, suppress_eos=True)
    full = OT.generate(W, cfg, embs, trail, pad, sp).codes
    for i in range(3):
        solo = OT.generate(W, cfg, [embs[i]], [trail[i]], pad, sp).codes[0]
        assert torch.equal(solo, full[i]), i
    rev = OT.generate(W, cfg, embs[::-1], trail[::-1], pad, sp).codes[::-1]
    assert all(torch.equal(a, b) for a, b in zip(rev, full))
