"""GPU parity of the wgmma tap-GEMM codec decoder against the CPU oracle (through the C ABI)."""
import numpy as np
import pytest
import torch

from oracle import codec as OC

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _small_cfg():
    # every channel count a multiple of 16 down to the last block (engine requirement)
    return OC.CodecCfg(codebook_size=64, codebook_dim=64, hidden_size=64, latent_dim=64, num_heads=4, num_kv_heads=4,
                       head_dim=16, sliding_window=6, intermediate_size=96, num_layers=2, num_quantizers=16,
                       upsample_rates=(8, 5, 4, 3), upsampling_ratios=(2, 2), decoder_dim=256)


def _pkg_cfg(c):
    import qwen3_tts_b200 as q
    return q.CodecConfig(**{k: getattr(c, k) for k in q.CodecConfig.__dataclass_fields__})


def _bf16_round(W):
    Wb = {k: v.to(torch.bfloat16) for k, v in W.items()}
    return Wb, {k: v.float() for k, v in Wb.items()}


def _snr_db(ref, out):
    ref, out = ref.double(), out.double()
    return float(10 * torch.log10(ref.pow(2).sum() / (ref - out).pow(2).sum().clamp(min=1e-30)))


def _run(cfg, B, T, seed, stage_check=True):
    from qwen3_tts_b200.codec import CodecDecoder
    Wb, Wf = _bf16_round(OC.random_weights(cfg, seed=seed))
    g = torch.Generator().manual_seed(seed + 1)
    codes = torch.randint(0, cfg.codebook_size, (B, cfg.num_quantizers, T), generator=g)
    ref = OC.decoder_forward(Wf, cfg, codes)
    dec = CodecDecoder(_pkg_cfg(cfg), Wb, device=DEV, max_frames=max(T, 64))
    out = dec.forward(codes.to(DEV)).cpu()
    dec.close()
    return ref, out


@pytest.mark.parametrize("B,T", [(1, 5), (2, 13), (3, 40)])
def test_small_codec_matches_oracle(B, T):
    cfg = _small_cfg()
    ref, out = _run(cfg, B, T, seed=3)
    assert out.shape == ref.shape == (B, 1, T * 1920)
    assert torch.isfinite(out).all()
    # tolerance: bf16 activations through ~45 layers vs the fp32 oracle on the same bf16 weights.
    # The oracle run in bf16 on CPU sits at ~30-35 dB against its own fp32 run (see DESIGN.md §Tolerance).
    snr = _snr_db(ref, out)
    assert snr > 25.0, f"SNR {snr:.1f} dB"
    assert (ref - out).abs().max() < 0.08


def test_codec_causality_and_batch_independence():
    """decode(prefix) == full[:prefix] (the decoder is strictly causal, SURVEY F9) and rows are independent."""
    from qwen3_tts_b200.codec import CodecDecoder
    cfg = _small_cfg()
    Wb, _ = _bf16_round(OC.random_weights(cfg, seed=5))
    dec = CodecDecoder(_pkg_cfg(cfg), Wb, device=DEV, max_frames=64)
    g = torch.Generator().manual_seed(1)
    codes = torch.randint(0, cfg.codebook_size, (2, 16, 24), generator=g).to(DEV)
    full = dec.forward(codes).clone()
    pre = dec.forward(codes[..., :9]).clone()
    assert torch.equal(pre, full[..., :9 * 1920])
    solo = dec.forward(codes[1:2]).clone()
    assert torch.equal(solo, full[1:2])
    # wrapper semantics: -1 padding, trim to T_i*1920, chunked decode with left context (…v2.py:886-896,993-1024)
    ac = codes.transpose(1, 2).clone()
    ac[1, 15:] = -1
    outs = dec.decode(ac)
    assert [o.numel() for o in outs] == [24 * 1920, 15 * 1920]
    dec.close()


def test_full_size_codec_default_config():
    """Reference default config (195 M params, 1536 -> 96 channels), 2 x 12 frames."""
    cfg = OC.CodecCfg()
    ref, out = _run(cfg, 2, 12, seed=7)
    snr = _snr_db(ref, out)
    assert torch.isfinite(out).all()
    assert snr > 22.0, f"SNR {snr:.1f} dB"


def test_chunked_decode_beyond_300_frames_matches_oracle_chunking():
    """> 300 frames: the reference decodes in 300-frame chunks with 25 frames of left context, which is NOT a full
    causal forward (SURVEY F9); the engine replicates the chunking exactly (…v2.py:886-896)."""
    from qwen3_tts_b200.codec import CodecDecoder
    cfg = _small_cfg()
    Wb, Wf = _bf16_round(OC.random_weights(cfg, seed=9))
    g = torch.Generator().manual_seed(4)
    codes = torch.randint(0, cfg.codebook_size, (1, 16, 330), generator=g)
    ref = OC.chunked_decode(Wf, cfg, codes)
    dec = CodecDecoder(_pkg_cfg(cfg), Wb, device=DEV, max_frames=512)
    out = dec.chunked_decode(codes.to(DEV)).cpu()
    assert out.shape == ref.shape == (1, 1, 330 * 1920)
    assert _snr_db(ref, out) > 25.0
    # and it differs from the un-chunked forward after the first chunk, exactly like the reference
    full = dec.forward(codes.to(DEV)).cpu()
    assert torch.equal(full[..., :300 * 1920], out[..., :300 * 1920])
    assert not torch.equal(full[..., 300 * 1920:], out[..., 300 * 1920:])
    dec.close()
