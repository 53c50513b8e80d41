"""fp64 references of the fp32 encoder kernels (csrc/conv_f32.cu, csrc/codec_encoder_kernels.cuh,
csrc/speaker_kernels.cuh), with padding, views and epilogues exactly as the kernels define them, and the per-element
error bounds of their fp32 evaluation.  tests/test_encoder_reference_cpu.py ties them to oracle/mimi_encoder.py and
oracle/speaker_encoder.py; tests/test_gpu_encoder_kernels.py compares the kernels with them.  Arrays are numpy; inputs
may be float32, results are float64."""
import math

import numpy as np

from tests import attention_ref as A

U = 2.0 ** -24                      # fp32 unit roundoff
PAD_ZERO, PAD_REPLICATE, PAD_REFLECT = 0, 1, 2
IN_NONE, IN_ELU, IN_TANH = 0, 1, 2
OUT_NONE, OUT_GELU, OUT_RELU, OUT_SIGMOID = 0, 1, 2, 3
# maximum errors of the CUDA math library with default (non-fast-math) flags, CUDA C Programming Guide, "Mathematical
# Functions", single precision: expm1f 1 ulp, tanhf 2 ulp, erff 2 ulp, expf 2 ulp, logf 1 ulp; sqrtf and the division
# are IEEE (correctly rounded).  One ulp of a float32 value y is at most 2^-23 |y|.
ULP_IN = {IN_NONE: 0, IN_ELU: 1, IN_TANH: 2}
LIPSCHITZ_OUT = {OUT_NONE: 1.0, OUT_RELU: 1.0, OUT_GELU: 1.13, OUT_SIGMOID: 0.25}


def reflect(i, T):
    """torch "reflect" padding index (no edge repetition), valid while the pad is < T."""
    i = np.abs(i)
    return np.where(i >= T, 2 * (T - 1) - i, i)


def tap_index(Tout, k, stride, dil, pad_left, Tin, pad):
    """Input column of output t and tap j [Tout][k], and whether it is inside [0, Tin) after padding."""
    ti = np.arange(Tout)[:, None] * stride + np.arange(k)[None, :] * dil - pad_left
    if pad == PAD_REPLICATE:
        ti = np.clip(ti, 0, Tin - 1)
    elif pad == PAD_REFLECT:
        ti = reflect(ti, Tin)
    ok = (ti >= 0) & (ti < Tin)
    return np.where(ok, ti, 0), ok


def act_in_f64(v, act):
    if act == IN_ELU:
        return np.where(v > 0, v, np.expm1(np.minimum(v, 0)))
    if act == IN_TANH:
        return np.tanh(v)
    return v


def act_out_f64(v, act):
    if act == OUT_GELU:
        from scipy.special import erf
        return 0.5 * v * (1.0 + erf(v * 0.7071067811865476))
    if act == OUT_RELU:
        return np.maximum(v, 0.0)
    if act == OUT_SIGMOID:
        return 1.0 / (1.0 + np.exp(-v))
    return v


def conv_input(x, Cin, Tin, x_off=0, x2=None, x2_off=0, act_in=IN_NONE):
    """X = act_in(x (+ x2)) over the view: [B][Cin][Tin] float64 (the sum x + x2 rounded to fp32 first, as loaded)."""
    v = np.asarray(x)[:, x_off:x_off + Cin, :Tin]
    if x2 is not None:
        v = (v.astype(np.float32) + np.asarray(x2)[:, x2_off:x2_off + Cin, :Tin].astype(np.float32))
    return act_in_f64(v.astype(np.float64), act_in)


def ref_conv(x, w, Cin, Cout, Tin, Tout, k, stride=1, dil=1, pad_left=0, pad=PAD_ZERO, act_in=IN_NONE,
             act_out=OUT_NONE, bias=None, scale=None, res=None, x_off=0, x2=None, x2_off=0, y_off=0):
    """conv_f32 (conv_f32.cuh) in float64.  x (and x2): [B][>= x_off + Cin][>= Tin], only columns [0, Tin) exist;
    w [Cout][Cin][k]; res [B][>= y_off + Cout][>= Tout] in y's view.  Returns dict: y (the output), pre (bias + sum,
    before the output activation), sab = sum |w * X| and X, the gathered input [B][Cin][Tout][k] (zero where padded)."""
    X = conv_input(x, Cin, Tin, x_off, x2, x2_off, act_in)
    ti, ok = tap_index(Tout, k, stride, dil, pad_left, Tin, pad)
    Xg = X[:, :, ti] * ok
    w = np.asarray(w, np.float64)
    pre = np.einsum("bctj,ocj->bot", Xg, w, optimize=True)
    sab = np.einsum("bctj,ocj->bot", np.abs(Xg), np.abs(w), optimize=True)
    if bias is not None:
        pre = pre + np.asarray(bias, np.float64)[None, :, None]
    y = act_out_f64(pre, act_out)
    if scale is not None:
        y = np.asarray(scale, np.float64)[None, :, None] * y
    if res is not None:
        y = np.asarray(res, np.float64)[:, y_off:y_off + Cout, :Tout] + y
    return {"y": y, "pre": pre, "sab": sab, "X": Xg}


def conv_bound(r, Cin, k, act_in, act_out, bias=None, scale=None, res=None, has_x2=False):
    """Per-element bound on |kernel - r["y"]| for the fp32 kernel: the FMA chain (Cin*k + 1 roundings, the bias add
    included) on sum |w*X| + |bias|; the input's load error (the x + x2 rounding and the activation's ulps) weighted by
    |w|, which is sum |w*X| times the relative error; the output activation's Lipschitz constant times that plus its own
    evaluation error; then the scale and residual roundings."""
    pre, sab = r["pre"], r["sab"]
    babs = 0.0 if bias is None else np.abs(np.asarray(bias, np.float64))[None, :, None]
    e_in = ULP_IN[act_in] * 2.0 ** -23 + (U if has_x2 else 0.0)
    E = (Cin * k + 1) * U * (sab + babs) + e_in * sab * (1 + e_in)
    z = act_out_f64(pre, act_out)
    if act_out == OUT_GELU:
        # 0.5 v (1 + erff(v c)): erff 2 ulp of |erf| <= 1, the argument product, the 1 + erf sum and the final product
        own = np.abs(pre) * 2.0 ** -21 + np.abs(z) * 2.0 ** -23
    elif act_out == OUT_SIGMOID:
        # 1 / (1 + expf(-v)): expf 2 ulp, the sum and the IEEE division
        own = np.abs(z) * 2.0 ** -21
    else:
        own = 0.0
    b = LIPSCHITZ_OUT[act_out] * E + own
    if scale is not None:
        s = np.abs(np.asarray(scale, np.float64))[None, :, None]
        b = s * b + U * s * (np.abs(z) + b)
    yabs = np.abs(r["y"])
    if res is not None:
        b = b + U * (yabs + b)
    return b * (1 + 2.0 ** -20) + 2.0 ** -140


def conv_drop_sensitivity(r, w, bound, act_out, scale=None):
    """Smallest over taps (ci, j) of the largest |change| / (2 * bound) when that single term is removed from the sum,
    evaluated at every (b, t) of the output channel with the tap's largest weight (a lower bound on the largest change
    over all elements): > 1 means a kernel that drops or duplicates any one tap fails the bound somewhere.  Taps that
    read only padding (a short input's right extra padding) have no term and are skipped."""
    w = np.asarray(w, np.float64)
    Xg, pre = r["X"], r["pre"]
    Cout, Cin, k = w.shape
    co = np.abs(w).argmax(axis=0)                                     # [Cin][k]
    wsel = np.take_along_axis(w, co[None], 0)[0]                      # [Cin][k]
    term = Xg * wsel[None, :, None, :]                                # [B][Cin][Tout][k]
    p = pre[:, co, :].transpose(0, 1, 3, 2)                           # [B][Cin][Tout][k] pre of channel co[ci][j]
    bd = bound[:, co, :].transpose(0, 1, 3, 2)
    d = np.abs(act_out_f64(p, act_out) - act_out_f64(p - term, act_out))
    if scale is not None:
        d = d * np.abs(np.asarray(scale, np.float64))[co][None, :, None, :]
    ratio = (d / (2 * bd)).max(axis=(0, 2))                           # [Cin][k]
    reads = np.abs(Xg).max(axis=(0, 2)) > 0                            # taps that read only padding carry no term
    return float(ratio[reads].min()) if reads.any() else math.inf


# ================================================================================================ LayerNorm
def ref_layernorm_ct(x, w, b, eps):
    """LayerNorm over channels of x [B][C][T] (float64): (x - mean) / sqrt(var + eps) * w + b, biased variance."""
    x = np.asarray(x, np.float64)
    m = x.mean(axis=1, keepdims=True)
    v = ((x - m) ** 2).mean(axis=1, keepdims=True)
    return (x - m) / np.sqrt(v + eps) * np.asarray(w, np.float64)[None, :, None] + np.asarray(b, np.float64)[None, :, None]


def layernorm_bound(x, w, b, eps):
    """Per-element bound for layernorm_ct_kernel: fp32 mean of C terms summed in 8 strided partial sums of C/8 terms and
    a sum of the 8 partials, the division; the same for the variance of the rounded deviations (fmaf) and the division;
    + eps, rsqrtf 2 ulp; then (x - mean) * rstd * w + b, four roundings."""
    x = np.asarray(x, np.float64)
    C = x.shape[1]
    n = math.ceil(C / 8) + 8 + 1
    A_ = np.abs(x).mean(axis=1, keepdims=True)
    m = x.mean(axis=1, keepdims=True)
    d = x - m
    dm = n * U * A_ * (1 + 1e-6)
    dd = dm + U * (np.abs(d) + dm)                                     # per-element error of the deviation
    var = (d ** 2).mean(axis=1, keepdims=True)
    dvar = ((2 * np.abs(d) + dd) * dd).mean(axis=1, keepdims=True) + n * U * ((np.abs(d) + dd) ** 2).mean(axis=1, keepdims=True)
    dvar = dvar + U * (var + dvar) * 2                                 # / C and + eps
    rstd = 1.0 / np.sqrt(var + eps)
    rel_r = 0.5 * dvar / (var + eps) * (1 + dvar / (var + eps)) + 2 * 2.0 ** -23
    wa = np.abs(np.asarray(w, np.float64))[None, :, None]
    core = (np.abs(d) * rel_r + dd * (1 + rel_r)) * rstd               # |(x - mean) * rstd| error before roundings
    y = d * rstd * np.asarray(w, np.float64)[None, :, None] + np.asarray(b, np.float64)[None, :, None]
    ya = np.abs(d) * rstd * wa
    return (wa * core + 3 * U * (ya + wa * core) + U * (np.abs(y) + wa * core)) * 1.01 + 2.0 ** -140


# ================================================================================================ RoPE / attention
def ref_rope_ct(x1, x2, c, s):
    """Rotate-half pair (i, i + hd/2) by fp32 tables: (x1 c - x2 s, x2 c + x1 s) in float64, and the bound
    2 * 2^-24 (|x1 c| + |x2 s|) (resp. |x2 c| + |x1 s|) of the kernel's two products and one sum, either product of which
    nvcc may contract into an FMA."""
    x1, x2, c, s = (np.asarray(v, np.float64) for v in (x1, x2, c, s))
    y1, y2 = x1 * c - x2 * s, x2 * c + x1 * s
    return y1, y2, 2 * U * (np.abs(x1 * c) + np.abs(x2 * s)), 2 * U * (np.abs(x2 * c) + np.abs(x1 * s))


def swa_keys(P, window):
    """Absolute key positions query position P attends to: max(P - window + 1, 0) .. P (ascending, the walk order)."""
    return np.arange(max(P - window + 1, 0), P + 1)


def ref_swa_ct(q, K, V, scale):
    """One query of swa_ct over its visible keys K, V [n][hd] (fp32 values, float64 arithmetic): attention_ref.attend
    without any bf16 rounding.  Returns (o, p, L, s)."""
    return A.attend(np.asarray(q, np.float64), np.asarray(K, np.float64), np.asarray(V, np.float64), scale)


def swa_bound(q, K, V, s, p, L, o, scale):
    """Per-element bound for swa_ct's fp32 online softmax of one query, built like attention_ref.online_bound with an
    fp32 output: the fp32 dot product over hd terms and the scale on every score; __expf's error (attention_ref.exp_err)
    on each term's own exponential and on every rescaling it passes through (one per rise of the running maximum in the
    ascending walk, __expf(0) = 1 exactly otherwise) with the rounding of its argument; one fp32 fma rounding of each
    accumulator per key; 1 / l and the final product.  The rescalings telescope, so a term's exponent carries the
    score error of two scores only."""
    q, K, V = (np.asarray(v, np.float64) for v in (q, K, V))
    hd, n = len(q), len(K)
    ds = scale * (hd * U * (np.abs(K) @ np.abs(q))) + 2 * U * np.abs(s)
    run = np.maximum.accumulate(s)
    rises = np.diff(run)[np.diff(run) > 0]
    R = float(s.max() - s.min())
    eps = (2 * ds.max() + U * (R + rises.sum()) + A.exp_err(R) + sum(A.exp_err(r) for r in rises)
           + 2 * (len(rises) + 1) * U)
    absdev = (p @ np.abs(V - o[None, :])) / L
    mag = (p @ np.abs(V)) / L
    pre = 2.2 * eps * absdev + 2.2 * n * U * (mag + np.abs(o))
    return pre + 2 * U * (np.abs(o) + pre) + 1e-37


# ================================================================================================ RVQ
def ref_rvq_level(r, E, E2):
    """Distances of one RVQ level as the kernel defines them, in float64: E2[c] - 2 r . e_c over the E2 values the kernel
    receives.  r [..][D], E [K][D].  Returns (dist [..][K], bound [..][K]): bound covers the fp32 dot product over D
    terms (2 D 2^-24 sum |r e|) and the rounding of the difference."""
    r, E, E2 = (np.asarray(v, np.float64) for v in (r, E, E2))
    D = E.shape[1]
    dot = r @ E.T
    dist = E2 - 2 * dot
    return dist, 2 * D * U * (np.abs(r) @ np.abs(E).T) * (1 + 1e-6) + U * (np.abs(dist) + np.abs(E2)) + 2.0 ** -140


def exact_argmin(dist):
    """argmin along the last axis, ties -> lowest index (np.argmin's rule)."""
    return np.argmin(dist, axis=-1)


# ================================================================================================ speaker
def ref_melspec(wav, window, twc, tws, fbT, n_fft, hop, frames):
    """melspec_kernel in float64 over the tables it receives: reflect-pad (n_fft - hop)/2, windowed frame, DFT with
    twiddle (k n mod n_fft), |X| = sqrt(re^2 + im^2 + 1e-9), mel = fbT^T |X|, log(max(mel, 1e-5)).  wav [B][T].
    Returns (out [B][n_mels][frames], bound)."""
    wav, window, twc, tws, fbT = (np.asarray(v, np.float64) for v in (wav, window, twc, tws, fbT))
    T = wav.shape[1]
    pad = (n_fft - hop) // 2
    idx = reflect(np.arange(frames)[:, None] * hop + np.arange(n_fft)[None, :] - pad, T)
    xw = wav[:, idx] * window[None, None, :]                           # [B][F][N]
    xw = xw.astype(np.float32).astype(np.float64)                      # the kernel stores fp32(y * window)
    nb = n_fft // 2 + 1
    tw = (np.arange(nb)[:, None] * np.arange(n_fft)[None, :]) % n_fft
    Cm, Sm = twc[tw], tws[tw]                                          # [nb][N]
    re, im = xw @ Cm.T, -(xw @ Sm.T)
    dre = (n_fft + 1) * U * (np.abs(xw) @ np.abs(Cm).T)
    dim_ = (n_fft + 1) * U * (np.abs(xw) @ np.abs(Sm).T)
    mag = np.sqrt(re * re + im * im + 1e-9)
    dmag = (np.abs(re) * dre + np.abs(im) * dim_) / mag + (dre ** 2 + dim_ ** 2) / mag + 4 * U * mag
    mel = mag @ fbT                                                    # [B][F][M]
    dmel = dmag @ np.abs(fbT) + (nb + 1) * U * (mag + dmag) @ np.abs(fbT)
    lo, hi = np.maximum(mel - dmel, 1e-5), np.maximum(mel + dmel, 1e-5)
    out = np.log(np.maximum(mel, 1e-5))
    bound = np.maximum(np.log(hi) - out, out - np.log(lo)) * 1.01 + 2 * 2.0 ** -23 * np.abs(out) + 1e-5 * U
    return out.transpose(0, 2, 1), bound.transpose(0, 2, 1)


def ref_mean_t(x):
    return np.asarray(x, np.float64).mean(axis=-1)


def ref_se_apply(h, gate, res):
    """h [B][C][T] * gate [B][C] + res [B][C][T]."""
    return np.asarray(h, np.float64) * np.asarray(gate, np.float64)[:, :, None] + np.asarray(res, np.float64)


def _weighted_stats(x, p, eps):
    m = (p * x).sum(-1)
    v = (p * (x - m[..., None]) ** 2).sum(-1)
    return m, np.sqrt(np.maximum(v, eps)), v


def _sd_bound(v, dv, eps):
    """|sqrt(max(v', eps)) - sqrt(max(v, eps))| for |v' - v| <= dv, plus sqrtf's rounding."""
    lo = np.maximum(v - dv, eps)
    sd = np.sqrt(np.maximum(v, eps))
    return np.minimum(np.sqrt(dv), dv / (2 * np.sqrt(lo))) + U * (sd + np.sqrt(dv))


def ref_asp_cat(x, eps=1e-12):
    """asp_cat: mean / std over time with uniform weights fp32(1 / T) (the oracle's fp32 mask weights, and the kernel's),
    clamped variance.  x [B][C][T] -> (mean, std, bounds).  The kernel sums in ceil(T/32) lane sums and a 5-level warp
    sum."""
    x = np.asarray(x, np.float64)
    T = x.shape[-1]
    p = np.full(T, float(np.float32(1.0) / np.float32(T)))
    m, sd, v = _weighted_stats(x, p, eps)
    n = math.ceil(T / 32) + 5 + 3
    ax = (p * np.abs(x)).sum(-1)
    dm = n * U * ax
    d = np.abs(x - m[..., None])
    dd = dm[..., None] + U * (d + dm[..., None])
    dv = (p * (2 * d + dd) * dd).sum(-1) + n * U * (p * (d + dd) ** 2).sum(-1)
    return m, sd, dm * 1.01 + 1e-37, _sd_bound(v, dv * 1.01, eps) + 1e-37


def ref_asp_pool(x, att, eps=1e-12):
    """asp_pool: softmax over time of att, weighted mean / std of x.  Returns (mean, std, bounds).  Each weight
    expf(a - max) / z carries the subtraction's rounding amplified by |a - max|, expf's 2 ulp, z's fp32 sum of T terms
    and the division; the sums then add their own fp32 error."""
    x, att = np.asarray(x, np.float64), np.asarray(att, np.float64)
    T = x.shape[-1]
    a = att - att.max(-1, keepdims=True)
    e = np.exp(a)
    p = e / e.sum(-1, keepdims=True)
    m, sd, v = _weighted_stats(x, p, eps)
    n = math.ceil(T / 32) + 5 + 3
    ep = (np.abs(a).max(-1) * U + 2 * 2.0 ** -23) * 2 + n * U + 2 * U    # relative error of every weight
    ax = (p * np.abs(x)).sum(-1)
    dm = ep * ax + n * U * ax * (1 + ep)
    d = np.abs(x - m[..., None])
    dd = dm[..., None] + U * (d + dm[..., None])
    dv = (p * (2 * d + dd) * dd).sum(-1) * (1 + ep) + (ep + n * U * (1 + ep)) * (p * (d + dd) ** 2).sum(-1)
    return m, sd, dm * 1.01 + 1e-37, _sd_bound(v, dv * 1.01, eps) + 1e-37
