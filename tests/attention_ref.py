"""fp64 references of the three attention paths (frame-step attention phase, prefill pair, codec sliding window), with
the kernels' own bf16 rounding points.  tests/test_attention_reference_cpu.py ties them to oracle/talker.py and
oracle/codec.py; tests/test_gpu_attention.py compares the kernels with them.  Arrays are numpy float64 holding bf16 (or
fp32) values unless stated otherwise."""
import numpy as np
import torch

HD = 128
U24, U8 = 2.0 ** -24, 2.0 ** -8     # fp32 and bf16 unit roundoff


def rbf(x):
    """Round to the nearest bf16 value, ties to even (fp64 in, fp64 out; no subnormal or overflow handling needed)."""
    x = np.asarray(x, np.float64)
    m, e = np.frexp(x)
    q = np.ldexp(1.0, e - 8)
    return np.where(x == 0, x, np.round(x / q) * q)


def rf32(x):
    return np.asarray(x, np.float32).astype(np.float64)


def bf16_bits(x):
    """int16 bit patterns of bf16 values."""
    return (np.asarray(x, np.float32).view(np.uint32) >> 16).astype(np.uint16).view(np.int16)


def from_bits(b):
    return (np.asarray(b, np.int16).view(np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def rope_rotate(y, cos, sin):
    """Rotate-half RoPE of bf16 vectors y [..., d] with bf16 tables [..., d/2]: two rounded bf16 products, their fp32
    sum, then bf16 (the kernels' and the oracle's order)."""
    h = y.shape[-1] // 2
    y1, y2 = y[..., :h], y[..., h:]
    a = rf32(rf32(rbf(y1 * cos)) + rf32(rbf(-y2 * sin)))
    b = rf32(rf32(rbf(y2 * cos)) + rf32(rbf(y1 * sin)))
    return np.concatenate([rbf(a), rbf(b)], axis=-1)


# relative error of the kernels' inv = rsqrtf(fp32 warp sum / d + eps) against the fp64 value: rsqrtf's 2 ulp, half the
# relative error of a fp32 sum of d squares (d - 1 adds), the division, the eps add and the product x * inv
def norm_delta(d=HD):
    return (2 + 1 + 1 + 1) * 2.0 ** -23 + 0.5 * (d - 1) * U24


def norm_rope(x, w, cos, sin, eps):
    """RMSNorm + RoPE of bf16 vectors x [..., d]: rbf(rbf(x * inv) * w), then rope_rotate.  Returns (out, amb): amb marks
    the output elements whose value depends on a first rounding rbf(x * inv) whose fp64 argument lies within the kernel's
    inv error (norm_delta) of a bf16 rounding boundary; such an element may come out of the kernel differently."""
    d = x.shape[-1]
    inv = 1.0 / np.sqrt((x * x).mean(-1, keepdims=True) + eps)
    t = x * inv
    dl = norm_delta(d) * np.abs(t)
    y = rbf(rbf(t) * w)
    amb_in = rbf(t - dl) != rbf(t + dl)
    h = d // 2
    amb_pair = amb_in[..., :h] | amb_in[..., h:]
    return rope_rotate(y, cos, sin), np.concatenate([amb_pair, amb_pair], axis=-1)


def rope_tables(npos, d, theta):
    """bf16 cos / sin tables [npos][d/2] of oracle.talker.rope_cos_sin (its second half repeats the first)."""
    from oracle.talker import rope_cos_sin
    cos, sin = rope_cos_sin(torch.arange(npos)[None], d, theta, torch.bfloat16)
    return cos[0, :, :d // 2].double().numpy(), sin[0, :, :d // 2].double().numpy()


# ================================================================================================ softmax attention
def attend(q, K, V, scale):
    """fp64 single-query attention: q [d], K, V [n][d].  Returns (o, p, L, s): output, unnormalised weights
    exp(s - max s), their sum and the scores."""
    s = (K @ q) * scale
    p = np.exp(s - s.max())
    L = p.sum()
    return (p @ V) / L, p, L, s


def exp_err(x):
    """__expf's documented maximum error at argument x, relative: 2 + floor(1.173 |x|) ulp."""
    return (2 + np.floor(1.173 * np.abs(x))) * 2.0 ** -23


def online_bound(q, K, V, s, p, L, o, scale, chain, adds, amb_q=None):
    """Per-element bound |kernel - o| for an fp32 online softmax over the rows of K, V whose output is rounded to bf16.
    chain: most rescalings (corr factors and combine weights) any term goes through; adds: longest fp32 sum.
    Score errors: the fp32 dot product (128 terms) and the scale; q elements marked amb_q may be one bf16 ulp off."""
    ds = scale * (128 * U24 * (np.abs(K) @ np.abs(q)) + 4 * U24 * np.abs(K @ q))
    R = float(s.max() - s.min())
    eps = ds.max() * 2 + exp_err(R) * (chain + 1) + 2 * (chain + 1) * U24
    absdev = (p @ np.abs(V - o[None, :])) / L
    mag = (p @ np.abs(V)) / L
    pre = 2.2 * eps * absdev + 2.2 * adds * U24 * (mag + np.abs(o))
    if amb_q is not None and amb_q.any():
        # a q element one bf16 ulp off shifts every score by ulp * k_d * scale; to first order the output moves by
        # ulp * scale * sum_i p_i k_id (v_i - o) / L (a shift common to all scores cancels), doubled for the second order
        ulp = np.where(amb_q, 2.0 ** (np.floor(np.log2(np.maximum(np.abs(q), 1e-30))) - 7), 0.0)
        d = np.flatnonzero(amb_q)
        G = (K[:, d] * p[:, None]).T @ (V - o[None, :]) / L
        pre = pre + 2 * scale * (ulp[d] @ np.abs(G))
    return pre + U8 * (np.abs(o) + pre) + 1e-30


def drop_one(p, L, V, O):
    """Outputs with key k removed, closed form (O - p_k v_k) / (L - p_k), for every k: [n][d]."""
    return (O[None, :] - p[:, None] * V) / (L - p)[:, None]


def sensitivity(p, L, V, o, bound):
    """Smallest over keys of the largest |change| / (2 * bound) over output elements when that key is removed: > 1
    means the check would catch a kernel that drops (or, by symmetry, duplicates) any single key."""
    if len(p) < 2:
        return np.inf
    O = o * L
    dv = np.abs(drop_one(p, L, V, O) - o[None, :]) / (2 * bound[None, :])
    return float(dv.max(axis=1).min())


# ================================================================================================ codec
def codec_attention(q, K, V, hd):
    """The codec's sliding-window attention of one query over its visible keys K, V [n][hd]: fp32 dot products rounded to
    bf16, times the scale in bf16, fp64 softmax, probabilities rounded to bf16 (the eager reference's .to(q.dtype)), fp64
    weighted sum.  Returns (o, pr, s, e, amb_s): output, bf16 probabilities, bf16 scores, exp(s - max), and the scores
    whose fp64 dot product lies within the fp32 summation error of a bf16 boundary."""
    d = K @ q
    err = hd * U24 * (np.abs(K) @ np.abs(q))
    scale = hd ** -0.5
    s = rbf(rbf(d) * scale)
    amb_s = rbf(rbf(d - err) * scale) != rbf(rbf(d + err) * scale)
    e = np.exp(s - s.max())
    pr = rbf(e / e.sum())
    return pr @ V, pr, s, e, amb_s


def codec_bound(q, K, V, hd):
    """(o, bound, pr, n_amb): reference output and per-element bound for the codec kernel.  A probability may come out
    one bf16 step off where its fp64 value lies within the kernel's error (__expf, the fp32 sum and reciprocal, or an
    ambiguous score) of a rounding boundary; the fp32 sum of p * v and the bf16 output rounding are added."""
    o, pr, s, e, amb_s = codec_attention(q, K, V, hd)
    n = len(s)
    ulp_s = 2.0 ** (np.floor(np.log2(np.maximum(np.abs(s), 1e-30))) - 7)
    es = np.where(amb_s, np.expm1(ulp_s), 0.0)
    rel = exp_err(s - s.max()) + es + (n + 4) * U24 + (e * (exp_err(s - s.max()) + es)).sum() / e.sum()
    x = e / e.sum()
    lo, hi = rbf(x * (1 - rel)), rbf(x * (1 + rel))
    dp = np.maximum(np.abs(lo - pr), np.abs(hi - pr))
    pre = dp @ np.abs(V) + 1.1 * n * U24 * (pr @ np.abs(V))
    return o, pre + U8 * (np.abs(o) + pre) + 1e-30, pr, int((lo != hi).sum())


def codec_sensitivity(q, K, V, hd, bound):
    """sensitivity() for the codec: the reference with key k removed, probabilities re-rounded, for every k."""
    if len(K) < 2:
        return np.inf
    o, pr, s, e, _ = codec_attention(q, K, V, hd)
    P = rbf(e[None, :] / (e.sum() - e)[:, None])
    np.fill_diagonal(P, 0.0)
    dv = np.abs(P @ V - o[None, :]) / (2 * bound[None, :])
    return float(dv.max(axis=1).min())
