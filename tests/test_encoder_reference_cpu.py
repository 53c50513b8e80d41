"""The fp64 encoder references (tests/encoder_ref.py) against the CPU oracle, at float64: each reference restates, with
the kernels' own views and padding, a piece of oracle/mimi_encoder.py or oracle/speaker_encoder.py, so a kernel that
matches the reference computes the oracle's layer."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import mimi_encoder as ME
from oracle import speaker_encoder as SE
from tests import encoder_ref as R

TOL = 1e-12


def rng(seed):
    return np.random.default_rng(seed)


def close(a, b, tol=TOL):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    err = np.abs(a - b).max() / max(1.0, np.abs(b).max())
    assert err < tol, err


@pytest.mark.parametrize("k,stride,dil,T,pad", [(7, 1, 1, 23, 0), (8, 4, 1, 37, 0), (10, 5, 1, 3, 0), (4, 2, 1, 9, 1),
                                                (4, 2, 1, 1, 1), (3, 1, 2, 11, 0), (3, 2, 3, 17, 1), (1, 1, 1, 5, 0)])
def test_ref_conv_matches_mimi_conv1d(k, stride, dil, T, pad):
    """Causal MimiConv1d: left pad k_eff - stride, right "extra padding" to a stride multiple, zero or replicate: the
    kernel's view is pad_left = k_eff - stride and Tout = ceil(Tin / stride)."""
    g = rng(k * 100 + T)
    B, Cin, Cout = 2, 3, 5
    x = g.standard_normal((B, Cin, T))
    w = g.standard_normal((Cout, Cin, k))
    b = g.standard_normal(Cout)
    mode = "replicate" if pad else "constant"
    want = ME.mimi_conv1d(torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b), stride, dil, mode).numpy()
    keff = (k - 1) * dil + 1
    Tout = math.ceil(T / stride)
    assert want.shape[-1] == Tout
    got = R.ref_conv(x, w, Cin, Cout, T, Tout, k, stride, dil, keff - stride, R.PAD_REPLICATE if pad else R.PAD_ZERO, bias=b)
    close(got["y"], want)


@pytest.mark.parametrize("k,dil,T", [(5, 1, 7), (3, 2, 3), (3, 3, 4), (3, 4, 5), (1, 1, 1), (3, 2, 40)])
def test_ref_conv_matches_conv_same_reflect(k, dil, T):
    """nn.Conv1d(padding="same", padding_mode="reflect") with dilation, down to the smallest legal T = pad + 1."""
    g = rng(k * 10 + dil + T)
    B, Cin, Cout = 2, 4, 3
    x, w, b = g.standard_normal((B, Cin, T)), g.standard_normal((Cout, Cin, k)), g.standard_normal(Cout)
    want = SE._conv_same_reflect(torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b), dil).numpy()
    got = R.ref_conv(x, w, Cin, Cout, T, T, k, 1, dil, dil * (k - 1) // 2, R.PAD_REFLECT, bias=b)
    close(got["y"], want)


def test_ref_conv_epilogue_and_views():
    """x2 added before the input activation, channel offsets, bias, output activation, scale and residual."""
    g = rng(7)
    B, Cin, Cout, T = 2, 3, 4, 9
    x, x2 = g.standard_normal((B, 6, 12)), g.standard_normal((B, 5, 12))
    w, b, sc = g.standard_normal((Cout, Cin, 3)), g.standard_normal(Cout), g.standard_normal(Cout)
    res = g.standard_normal((B, 7, T))
    X = torch.from_numpy(x[:, 2:5, :T] + x2[:, 1:4, :T])
    for act_in, fin in ((R.IN_ELU, F.elu), (R.IN_TANH, torch.tanh), (R.IN_NONE, lambda v: v)):
        for act_out, fout in ((R.OUT_GELU, F.gelu), (R.OUT_SIGMOID, torch.sigmoid), (R.OUT_RELU, F.relu)):
            h = fout(ME.mimi_conv1d(fin(X), torch.from_numpy(w), torch.from_numpy(b)))
            want = torch.from_numpy(res[:, 3:7]) + torch.from_numpy(sc)[None, :, None] * h
            got = R.ref_conv(x.astype(np.float32), w, Cin, Cout, T, T, 3, 1, 1, 2, R.PAD_ZERO, act_in, act_out, b, sc,
                             res, x_off=2, x2=x2.astype(np.float32), x2_off=1, y_off=3)
            xf = x.astype(np.float32)[:, 2:5, :T] + x2.astype(np.float32)[:, 1:4, :T]
            h = fout(ME.mimi_conv1d(fin(torch.from_numpy(xf.astype(np.float64))), torch.from_numpy(w), torch.from_numpy(b)))
            want = torch.from_numpy(res[:, 3:7]) + torch.from_numpy(sc)[None, :, None] * h
            close(got["y"], want.numpy())


def tiny_enc():
    cfg = ME.cfg_tiny_encoder()
    return cfg, {k: v.double() for k, v in ME.random_weights(cfg, seed=3).items()}


def test_ref_layernorm_rope_swa_match_encoder_transformer():
    """One layer of oracle.mimi_encoder.encoder_transformer rebuilt from ref_layernorm_ct, ref_conv (1x1), ref_rope_ct
    with the oracle's rope_tables and ref_swa_ct over swa_keys, at T past the sliding window.  The oracle's softmax
    computes in fp32, so this one comparison is at fp32 accuracy."""
    cfg, W = tiny_enc()
    W = {k: v.float() for k, v in W.items()}
    cfg.num_layers = 1
    B, T, C, nh, hd = 2, 11, cfg.hidden_size, cfg.num_heads, cfg.head_dim
    g = rng(11)
    x = g.standard_normal((B, C, T))
    x = x.astype(np.float32)
    want = ME.encoder_transformer(W, cfg, torch.from_numpy(x).transpose(1, 2)).transpose(1, 2).numpy()
    p = "encoder_transformer.layers.0."
    n = lambda k: W[p + k].double().numpy()  # noqa: E731
    h = R.ref_layernorm_ct(x, n("input_layernorm.weight"), n("input_layernorm.bias"), cfg.norm_eps)
    wqkv = np.concatenate([n("self_attn.q_proj.weight"), n("self_attn.k_proj.weight"), n("self_attn.v_proj.weight")])
    qkv = R.ref_conv(h, wqkv[:, :, None], C, 3 * C, T, T, 1)["y"]
    cos, sin = (t.double().numpy() for t in ME.rope_tables(cfg, T))   # [T][hd/2]
    half = hd // 2
    for third in (0, 1):
        for hh in range(nh):
            base = third * C + hh * hd
            x1, x2 = qkv[:, base:base + half, :], qkv[:, base + half:base + hd, :]
            y1, y2, _, _ = R.ref_rope_ct(x1, x2, cos.T[None], sin.T[None])
            qkv[:, base:base + half, :], qkv[:, base + half:base + hd, :] = y1, y2
    att = np.zeros((B, C, T))
    for b in range(B):
        for hh in range(nh):
            for t in range(T):
                js = R.swa_keys(t, cfg.sliding_window)
                q = qkv[b, hh * hd:(hh + 1) * hd, t]
                K = qkv[b, C + hh * hd:C + (hh + 1) * hd, js]
                V = qkv[b, 2 * C + hh * hd:2 * C + (hh + 1) * hd, js]
                att[b, hh * hd:(hh + 1) * hd, t] = R.ref_swa_ct(q, K, V, 1 / math.sqrt(hd))[0]
    x = R.ref_conv(att, n("self_attn.o_proj.weight")[:, :, None], C, C, T, T, 1, scale=n("self_attn_layer_scale.scale"), res=x)["y"]
    h = R.ref_layernorm_ct(x, n("post_attention_layernorm.weight"), n("post_attention_layernorm.bias"), cfg.norm_eps)
    f = R.ref_conv(h, n("mlp.fc1.weight")[:, :, None], C, cfg.intermediate_size, T, T, 1, act_out=R.OUT_GELU)["y"]
    x = R.ref_conv(f, n("mlp.fc2.weight")[:, :, None], cfg.intermediate_size, C, T, T, 1, scale=n("mlp_layer_scale.scale"), res=x)["y"]
    close(x, want, 1e-5)


def test_ref_rvq_level_chain_matches_rvq_encode():
    """ref_rvq_level over E2 = |e|^2, chained with exact_argmin and r -= e, gives oracle.mimi_encoder.rvq_encode's codes."""
    cfg, W = tiny_enc()
    B, T, n_q = 2, 7, 6
    emb = torch.from_numpy(rng(5).standard_normal((B, cfg.hidden_size, T)))
    want = ME.rvq_encode(W, cfg, emb, n_q).numpy()
    got = []
    for which, n in (("semantic", cfg.num_semantic_quantizers), ("acoustic", n_q - cfg.num_semantic_quantizers)):
        pfx = f"quantizer.{which}_residual_vector_quantizer."
        r = np.einsum("dc,bct->btd", W[pfx + "input_proj.weight"][:, :, 0].numpy(), emb.numpy())
        for qi in range(n):
            E = ME.codebook_embed(W, pfx + f"layers.{qi}.codebook.").numpy()
            dist, _ = R.ref_rvq_level(r, E, (E * E).sum(1))
            c = R.exact_argmin(dist)
            got.append(c)
            r = r - E[c]
    assert np.array_equal(np.stack(got, 1), want)


def test_ref_melspec_matches_mel_spectrogram():
    """ref_melspec over fp64 Hann window, exact twiddles and the oracle's filterbank equals oracle mel_spectrogram."""
    n_fft, hop, M = 64, 16, 12
    for T in ((n_fft - hop) // 2 + 1 + 40, 203):
        wav = rng(T).standard_normal((2, T))
        fb = SE.slaney_mel_filterbank(24000, n_fft, M, 0, 12000).astype(np.float64)
        want = SE.mel_spectrogram(torch.from_numpy(wav), n_fft, M, 24000, hop, n_fft, 0, 12000, torch.from_numpy(fb)).numpy()
        j = np.arange(n_fft)
        win = 0.5 - 0.5 * np.cos(2 * np.pi * j / n_fft)
        frames = want.shape[-1]
        # ref_melspec rounds the windowed samples to fp32 (the kernel stores them so): compare at fp32 accuracy
        got, _ = R.ref_melspec(wav, win, np.cos(2 * np.pi * j / n_fft), np.sin(2 * np.pi * j / n_fft), fb.T, n_fft, hop, frames)
        close(got, want, 1e-6)


def test_ref_asp_matches_oracle_asp():
    """ref_asp_cat's [x; mean; std] and ref_asp_pool over the attention logits reproduce oracle _asp."""
    cfg = SE.cfg_tiny_spk()
    W = {k: v.double() for k, v in SE.random_weights(cfg, seed=2).items()}
    C, T = cfg.enc_channels[-1], 13
    x = rng(9).standard_normal((2, C, T))
    want = SE._asp(W, "asp", torch.from_numpy(x))[..., 0].numpy()
    m, sd, _, _ = R.ref_asp_cat(x)
    cat = np.concatenate([x, np.repeat(m[..., None], T, -1), np.repeat(sd[..., None], T, -1)], 1)
    h = R.ref_conv(cat, W["asp.tdnn.conv.weight"].numpy(), 3 * C, cfg.enc_attention_channels, T, T, 1,
                   act_out=R.OUT_RELU, bias=W["asp.tdnn.conv.bias"].numpy())["y"]
    att = R.ref_conv(h, W["asp.conv.weight"].numpy(), cfg.enc_attention_channels, C, T, T, 1, act_in=R.IN_TANH,
                     bias=W["asp.conv.bias"].numpy())["y"]
    pm, psd, _, _ = R.ref_asp_pool(x, att)
    close(np.concatenate([pm, psd], 1), want)


def test_ref_mean_t_and_se_apply_match_se_block():
    cfg = SE.cfg_tiny_spk()
    W = {k: v.double() for k, v in SE.random_weights(cfg, seed=4).items()}
    C = cfg.enc_channels[1]
    x = rng(1).standard_normal((2, C, 9))
    res = rng(2).standard_normal((2, C, 9))
    want = (SE._se(W, "blocks.1.se_block", torch.from_numpy(x)) + torch.from_numpy(res)).numpy()
    m = R.ref_mean_t(x)[..., None]
    s1 = R.ref_conv(m, W["blocks.1.se_block.conv1.weight"].numpy(), C, cfg.enc_se_channels, 1, 1, 1, act_out=R.OUT_RELU,
                    bias=W["blocks.1.se_block.conv1.bias"].numpy())["y"]
    gate = R.ref_conv(s1, W["blocks.1.se_block.conv2.weight"].numpy(), cfg.enc_se_channels, C, 1, 1, 1,
                      act_out=R.OUT_SIGMOID, bias=W["blocks.1.se_block.conv2.bias"].numpy())["y"][..., 0]
    close(R.ref_se_apply(x, gate, res), want)


def test_reflect_has_no_edge_repetition():
    assert list(R.reflect(np.arange(-3, 8), 5)) == [3, 2, 1, 0, 1, 2, 3, 4, 3, 2, 1]
