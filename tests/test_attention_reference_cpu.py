"""The fp64 attention references of tests/attention_ref.py (used by tests/test_gpu_attention.py) against the oracle:
oracle/talker.py's rms_norm, rope_cos_sin / apply_rope and eager_attention, and the sliding-window attention of
oracle/codec.py (mask 0 <= q - k < window), on the same bf16 inputs.  This ties the GPU test's reference to the model's
definition, as the tap-GEMM test's reference is tied to it."""
import math

import numpy as np
import torch

from oracle import codec as OC
from oracle import talker as OT
from tests import attention_ref as A


def t2n(t):
    return t.double().numpy()


def test_rbf_is_round_to_nearest_even_bf16():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1 << 16, generator=g) * torch.exp(torch.randn(1 << 16, generator=g) * 4)
    halfway = (x.view(torch.int32) & ~0xFFFF | 0x8000).view(torch.float32)   # exact ties: even rounding decides
    for v in (x, halfway):
        assert np.array_equal(A.rbf(v.double().numpy()), t2n(v.bfloat16()))
        assert np.array_equal(A.bf16_bits(A.rbf(v.numpy())), v.bfloat16().view(torch.int16).numpy())


def test_rope_tables_are_the_oracle_half_tables():
    for d, theta in ((128, 1e6), (64, 10000.0), (16, 10000.0)):
        cos, sin = OT.rope_cos_sin(torch.arange(600)[None], d, theta, torch.bfloat16)
        c, s = A.rope_tables(600, d, theta)
        assert np.array_equal(c, t2n(cos[0, :, :d // 2])) and np.array_equal(s, t2n(sin[0, :, :d // 2]))
        assert torch.equal(cos[..., :d // 2], cos[..., d // 2:]) and torch.equal(sin[..., :d // 2], sin[..., d // 2:])


def test_norm_rope_matches_oracle():
    """RMSNorm then RoPE on bf16: bit-exact except the counted near-boundary elements."""
    g = torch.Generator().manual_seed(1)
    n, eps = 512, 1e-6
    x = (torch.randn(n, 128, generator=g) * torch.exp(torch.randn(n, 1, generator=g))).bfloat16()
    w = (torch.randn(128, generator=g) * 0.3 + 1).bfloat16()
    pos = torch.randint(0, 2048, (1, n), generator=g)
    cos, sin = OT.rope_cos_sin(pos, 128, 1e6, torch.bfloat16)
    y = OT.rms_norm(x, w, eps)
    ref, _ = OT.apply_rope(y[None, None], y[None, None], cos, sin)
    c, s = A.rope_tables(2048, 128, 1e6)
    mine, amb = A.norm_rope(t2n(x), t2n(w), c[pos[0].numpy()], s[pos[0].numpy()], eps)
    diff = A.bf16_bits(mine) != ref[0, 0].view(torch.int16).numpy()
    assert not (diff & ~amb).any(), f"{int((diff & ~amb).sum())} elements differ away from a rounding boundary"
    assert amb.mean() < 0.01, f"near-boundary share {amb.mean():.4f}"
    # with the oracle's fp32 rsqrt the only differences are near-boundary ones; some boundary elements do match
    assert diff.sum() <= amb.sum()


def test_rope_rotate_matches_oracle_apply_rope():
    """The codec's RoPE without norm: bit-exact for every element (two rounded products, fp32 sum, bf16)."""
    g = torch.Generator().manual_seed(2)
    for d in (16, 64, 128):
        q = (torch.randn(1, 1, 300, d, generator=g) * 3).bfloat16()
        pos = torch.arange(300)[None] * 7
        cos, sin = OT.rope_cos_sin(pos, d, 10000.0, torch.bfloat16)
        ref, _ = OT.apply_rope(q, q, cos, sin)
        c, s = A.rope_tables(2100, d, 10000.0)
        mine = A.rope_rotate(t2n(q[0, 0]), c[pos[0].numpy()], s[pos[0].numpy()])
        assert np.array_equal(A.bf16_bits(mine), ref[0, 0].view(torch.int16).numpy())


def test_attend_matches_oracle_eager_attention():
    """Single-query GQA (the frame-step phase) and causal prefix attention (the prefill) in fp64."""
    g = torch.Generator().manual_seed(3)
    nh, nkv, n = 16, 8, 300
    q = torch.randn(1, nh, 1, 128, generator=g, dtype=torch.float64)
    k = torch.randn(1, nkv, n, 128, generator=g, dtype=torch.float64)
    v = torch.randn(1, nkv, n, 128, generator=g, dtype=torch.float64)
    scale = 1 / math.sqrt(128)
    ref = OT.eager_attention(q, k, v, None, scale, nh // nkv)[0, 0]
    for h in range(nh):
        o, p, L, s = A.attend(q[0, h, 0].numpy(), k[0, h // 2].numpy(), v[0, h // 2].numpy(), scale)
        assert np.allclose(o, ref[h].numpy(), rtol=0, atol=1e-6)  # the oracle softmax is fp32
    # causal: query i sees keys 0..i (the prefill's mask), as a -inf additive mask
    qs = torch.randn(1, nh, n, 128, generator=g, dtype=torch.float64)
    mask = torch.full((n, n), -math.inf, dtype=torch.float64).triu(1)[None, None]
    ref = OT.eager_attention(qs, k, v, mask, scale, nh // nkv)[0]
    for i in (0, 31, 32, 33, 63, 64, 299):
        for h in (0, 5):
            o, *_ = A.attend(qs[0, h, i].numpy(), k[0, h // 2, :i + 1].numpy(), v[0, h // 2, :i + 1].numpy(), scale)
            assert np.allclose(o, ref[i, h].numpy(), rtol=0, atol=1e-6)  # the oracle softmax is fp32


def test_codec_attention_matches_oracle(monkeypatch):
    """oracle/codec.py's pre_transformer: its rotated q / k equal rope_rotate bit for bit, its visible keys are exactly
    0 <= t - k < window, and its bf16 probabilities equal codec_attention's except where codec_bound allows a one-step
    difference (near a bf16 rounding boundary)."""
    cfg = OC.cfg_tiny_codec()
    W = OC.random_weights(cfg, seed=4, dtype=torch.bfloat16)
    T = 40
    x = (torch.randn(1, T, cfg.latent_dim, generator=torch.Generator().manual_seed(5))).bfloat16()
    seen = {"rope": [], "softmax": []}
    rope, softmax = OC.apply_rope, OC.F.softmax

    def rec_rope(q, k, cos, sin):
        out = rope(q, k, cos, sin)
        seen["rope"].append((q, k, cos, sin) + out)
        return out

    def rec_softmax(w, *a, **kw):
        out = softmax(w, *a, **kw)
        seen["softmax"].append(out)
        return out
    monkeypatch.setattr(OC, "apply_rope", rec_rope)
    monkeypatch.setattr(OC.F, "softmax", rec_softmax)
    OC.pre_transformer(W, cfg, x)
    assert len(seen["rope"]) == cfg.num_layers == len(seen["softmax"])
    hd, win = cfg.head_dim, cfg.sliding_window
    c, s = A.rope_tables(T, hd, cfg.rope_theta)
    for (q_in, k_in, _, _, q, k), probs in zip(seen["rope"], seen["softmax"]):
        pr_oracle = t2n(probs.to(torch.bfloat16))[0]
        for h in range(cfg.num_heads):
            for src, dst in ((q_in, q), (k_in, k)):
                assert np.array_equal(A.bf16_bits(A.rope_rotate(t2n(src[0, h]), c, s)),
                                      dst[0, h].view(torch.int16).numpy())
            qn, kn = t2n(q[0, h]), t2n(k[0, h])
            vis = np.zeros((T, T), bool)
            for t in range(T):
                r0 = max(0, t - win + 1)
                vis[t, r0:t + 1] = True
                _, bound, pr, _ = A.codec_bound(qn[t], kn[r0:t + 1], np.eye(t + 1 - r0), hd)
                # V = identity: the output is the probability vector itself, so the bound is per probability
                assert (np.abs(pr_oracle[h, t, r0:t + 1] - pr) <= bound).all()
            assert np.array_equal(pr_oracle[h] > 0, vis), "visible key set differs from 0 <= t - k < window"
