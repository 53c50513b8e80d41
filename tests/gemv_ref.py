"""fp64 reference of the frame-step kernel's GEMV phase (csrc/ar_gemv.cuh: gemv_phase) with the kernel's own bf16
rounding points.  tests/test_gemv_reference_cpu.py ties it to oracle/talker.py; tests/test_gpu_gemv.py compares the
kernel with it.

    normed input   xn = rbf(rbf(x * rsqrt(mean x^2 + eps)) * w)
    STORE          rbf(s)              BIAS    rbf(s + b)          RESID   rbf(r + rbf(s))
    LOGITS         float(rbf(s))       SWIGLU  rbf(rbf(silu(rbf(g))) * rbf(u)), gate / up rows in the blk8 layout

where s = sum_k W[n][k] xn[c][k] exactly.  Outputs are returned as an interval [lo, hi] per element: the epilogue of
every accumulator value within s -+ delta (delta = 0 for exact data; K 2^-22 sum|w x| for an fp32 sum in any order),
with SWIGLU's __expf error of 2 + floor(1.173 |g|) ulp (plus the fp32 add and divide around it) on top.  Arrays are
torch float64 (any device) in, numpy float64 out."""
import numpy as np
import torch

from tests.attention_ref import rbf

EPI_STORE, EPI_BIAS, EPI_RESID, EPI_SWIGLU, EPI_LOGITS = range(5)
U24 = 2.0 ** -24


def normed_input(x, w, eps):
    """x [nc][K], w [K] (bf16 values, float64): the staged operand rbf(rbf(x * inv) * w), and inv (fp64)."""
    x = np.asarray(x, np.float64)
    inv = 1.0 / np.sqrt((x * x).mean(-1, keepdims=True) + eps)
    return rbf(rbf(x * inv) * np.asarray(w, np.float64)), inv


def normed_boundary_mask(x, w, eps):
    """Elements of the normed input whose value may round either way under the kernel's fp32 sum of squares and
    rsqrtf (2 ulp): rbf(x * inv) or the product with w lies within that relative error of a bf16 rounding boundary."""
    x = np.asarray(x, np.float64)
    K = x.shape[-1]
    xn, inv = normed_input(x, w, eps)
    rel = (K + 4) * U24 + 2 * 2.0 ** -23   # fp32 sum of squares + mean + eps, rsqrtf, the fp32 product x * inv
    t = x * inv
    near = _near_boundary(t, rel)
    near |= _near_boundary(rbf(t) * np.asarray(w, np.float64), 0.0)  # the bf16 product is one correctly rounded op
    return near


def _near_boundary(v, rel):
    """v within a relative `rel` (or exactly at, for rel = 0) of a bf16 rounding midpoint."""
    v = np.asarray(v, np.float64)
    lo, hi = rbf(v * (1 - rel)), rbf(v * (1 + rel))
    at_tie = rbf(np.nextafter(v, np.inf)) != rbf(np.nextafter(v, -np.inf))
    return (lo != hi) | at_tie


def gate_up_blk8(gate, up):
    """The engine's interleave (AREngine._gate_up_blk8): [I][K] gate and up -> [2I][K], 16-row tiles of 8 gate rows
    then the same 8 up rows."""
    I, K = gate.shape
    return torch.stack([gate.view(I // 8, 8, K), up.view(I // 8, 8, K)], 1).reshape(2 * I, K)


def accumulate(W, xn):
    """s [nc][N] = xn @ W^T in fp64, and sum_k |W x| per output."""
    W = torch.as_tensor(W, dtype=torch.float64)
    xn = torch.as_tensor(xn, dtype=torch.float64, device=W.device)
    s = xn @ W.T
    a = xn.abs() @ W.abs().T
    return s.cpu().numpy(), a.cpu().numpy()


def swap_k_halves(x):
    """The wrong K permutation: the two 4-element halves of every 8-k group exchanged."""
    x = torch.as_tensor(x)
    K = x.shape[-1]
    return x.reshape(*x.shape[:-1], K // 8, 2, 4).flip(-2).reshape(x.shape)


def epilogue(s, abs_sum, epi, K, exact, bias=None, resid=None):
    """[lo, hi] of the kernel's output for accumulators s [nc][N] (N = rows of the GEMV; SWIGLU: N/2 outputs)."""
    d = 0.0 if exact else K * 2.0 ** -22 * abs_sum
    a_lo, a_hi = s - d, s + d
    if epi == EPI_STORE or epi == EPI_LOGITS:
        return rbf(a_lo), rbf(a_hi)
    if epi == EPI_BIAS:
        b = np.asarray(bias, np.float64)[None, :]
        t_lo, t_hi = a_lo + b, a_hi + b
        if not exact:  # the fp32 add in front of the bf16 conversion
            t_lo, t_hi = t_lo - np.abs(t_lo) * U24, t_hi + np.abs(t_hi) * U24
        return rbf(t_lo), rbf(t_hi)
    if epi == EPI_RESID:
        r = np.asarray(resid, np.float64)
        return rbf(r + rbf(a_lo)), rbf(r + rbf(a_hi))
    assert epi == EPI_SWIGLU
    nc, N = s.shape
    g_idx = (np.arange(N // 2) // 8) * 16 + np.arange(N // 2) % 8
    g_lo, g_hi = rbf(a_lo[:, g_idx]), rbf(a_hi[:, g_idx])
    u_lo, u_hi = rbf(a_lo[:, g_idx + 8]), rbf(a_hi[:, g_idx + 8])
    sl_lo, sl_hi = _silu_range(g_lo, g_hi)
    c = [rbf(p * q) for p in (sl_lo, sl_hi) for q in (u_lo, u_hi)]
    return np.minimum.reduce(c), np.maximum.reduce(c)


SILU_MIN_BF16 = (-1.28125, -1.2734375)   # the bf16 values around silu's minimum at g = -1.2785


def _silu_range(g_lo, g_hi):
    """rbf(silu(g)) over the bf16 gate values in [g_lo, g_hi] (the kernel: gt / (1 + __expf(-gt)) in fp32).  silu is
    monotone on either side of its minimum, so the ends of the range and the bf16 values around the minimum suffice."""
    lo = np.full(g_lo.shape, np.inf)
    hi = np.full(g_lo.shape, -np.inf)
    for g, use in [(g_lo, True), (g_hi, True)] + [(np.full(g_lo.shape, m), (g_lo < m) & (m < g_hi)) for m in SILU_MIN_BF16]:
        e = np.exp(-g)
        eps = (2 + np.floor(1.173 * np.abs(g))) * 2.0 ** -23 + 4 * U24
        v1, v2 = g / (1.0 + e * (1 - eps)), g / (1.0 + e * (1 + eps))
        v1, v2 = v1 - np.abs(v1) * 2 * U24, v2 + np.abs(v2) * 2 * U24
        # fp32 range: exp(-g) overflows to inf below g = -ln(FLT_MAX) = -88.72 and the quotient is -0
        v1 = np.where(g < -88.6, np.where(g < -88.8, -0.0, np.minimum(v1, 0.0)), v1)
        v2 = np.where(g < -88.8, -0.0, v2)
        vl, vh = rbf(np.minimum(v1, v2)), rbf(np.maximum(v1, v2))
        lo = np.where(use, np.minimum(lo, vl), lo)
        hi = np.where(use, np.maximum(hi, vh), hi)
    return lo, hi


def gemv(W, x, epi, norm_w=None, eps=0.0, bias=None, resid=None, exact=True, x_kernel=None, drop=None, swap_halves=False,
         swap_gate_up=False):
    """The phase dst = epi(sum_k W[n][k] xin[c][k]) on bf16 values: W [N][K] (torch float64, any device), x [nc][K].

    Returns (lo, hi, xn): the output interval per element ([nc][N], [nc][N/2] for SWIGLU) and the normed input.
    x_kernel: the kernel's own staged operand (its save_normed copy) to accumulate over instead of the reference's.
    Mutations for the sensitivity checks: drop = (tile, k-block) left out of the sum; swap_halves = the wrong K
    permutation; swap_gate_up = gate and up rows exchanged."""
    W = torch.as_tensor(W, dtype=torch.float64)
    x = np.asarray(torch.as_tensor(x, dtype=torch.float64).cpu())
    K = W.shape[1]
    if norm_w is not None:
        xn, _ = normed_input(x, np.asarray(torch.as_tensor(norm_w, dtype=torch.float64).cpu()), eps)
    else:
        xn = x
    xin = xn if x_kernel is None else np.asarray(x_kernel, np.float64)
    Wm = W
    if drop is not None:
        tile, kb = drop
        Wm = W.clone()
        Wm[tile * 16:(tile + 1) * 16, kb * 32:(kb + 1) * 32] = 0
    xt = torch.as_tensor(xin, dtype=torch.float64)
    if swap_halves:
        xt = swap_k_halves(xt)
    if swap_gate_up:
        N = Wm.shape[0]
        perm = torch.arange(N).view(N // 16, 2, 8).flip(1).reshape(N)
        Wm = Wm[perm.to(Wm.device)]
    s, a = accumulate(Wm, xt)
    lo, hi = epilogue(s, a, epi, K, exact, bias=None if bias is None else np.asarray(torch.as_tensor(bias).double().cpu()),
                      resid=resid)
    return lo, hi, xn
