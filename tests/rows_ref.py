"""fp64 references of the row-wise kernels of the codec decoder (csrc/codec_kernels.cuh), the prefill
(csrc/ar_prefill.cuh) and the streaming codec encoder (csrc/codec_encoder_kernels.cuh), with the kernels' own bf16
rounding points, and numpy restatements of their copy and index kernels.  tests/test_rows_reference_cpu.py ties them to
oracle/codec.py, oracle/talker.py and oracle/mimi_encoder.py; tests/test_gpu_row_kernels.py compares the kernels with
them.  Where a kernel rounds to bf16 after an fp32 computation whose error is bounded, the reference returns the
admissible set at that rounding point (its two ends, lo <= hi) instead of one value.  Arrays are numpy float64 holding
bf16 or fp32 values unless stated otherwise."""
import numpy as np

from tests.attention_ref import rbf

U = 2.0 ** -24          # fp32 unit roundoff
HIST = 6                # rows of history in front of a ConvNeXt / final conv input (k = 7)


def bf16_ulp(v):
    """Spacing of bf16 values at |v| (the larger spacing at a power of two)."""
    v = np.abs(np.asarray(v, np.float64))
    e = np.frexp(np.where(v == 0, 1.0, v))[1]
    return np.ldexp(1.0, e - 8)


def granularity(v):
    """The largest power of two every bf16 value v is a multiple of (inf for zero)."""
    v = np.abs(np.asarray(v, np.float64))
    return np.where(v == 0, np.inf, np.ldexp(1.0, np.frexp(np.where(v == 0, 1.0, v))[1] - 8))


def bf16_interval(y, bound):
    """Every bf16 value the kernel may produce from an fp32 value within `bound` of y: [rbf(y - bound), rbf(y + bound)]."""
    return rbf(y - bound), rbf(y + bound)


# ================================================================================================ RVQ gather
def rvq_gather(codes, table, count=None, reverse=False):
    """e [B][T][2D] of rvq_gather_kernel: e[..., :D] = table[0][c0]; e[..., D:] = the sequential bf16 sum over k >= 1 of
    table[k][c_k], acc = rbf(fp32(acc + v)) (torch's bf16 add); frames t >= count[b] are zero.  codes [B][K][T] int,
    table [K][bins][D].  reverse: the sum over k = K-1 .. 1 instead (a plausible slip the check must catch)."""
    codes = np.asarray(codes)
    B, K, T = codes.shape
    D = table.shape[2]
    tab = np.asarray(table, np.float32)
    e = np.zeros((B, T, 2 * D), np.float32)
    for b in range(B):
        n = T if count is None else count[b]
        for t in range(n):
            e[b, t, :D] = tab[0, codes[b, 0, t]]
            ks = list(range(1, K))
            if reverse:
                ks = ks[::-1]
            acc = None
            for k in ks:
                v = tab[k, codes[b, k, t]]
                acc = v if acc is None else rbf(acc + v).astype(np.float32)
            if acc is not None:
                e[b, t, D:] = acc
    return e.astype(np.float64)


# ================================================================================================ RMSNorm
def rms_delta(C):
    """Relative error of the kernels' t = fp32(x * inv) against x * inv64: half the relative error of an fp32 sum of C
    positive squares (C / 32 per lane + a 5-level warp tree, plus the products), the division, + eps and rsqrtf's
    2 ulp; then the product x * inv itself."""
    return 0.5 * (C / 32 + 5 + 1 + 2) * U + 2 * 2.0 ** -23 + U


def rmsnorm(x, w, eps):
    """rmsnorm_rows_kernel / pf_rmsnorm_kernel: y = bf16(r * w), r = bf16(x * inv), inv = rsqrt(mean x^2 + eps).  r * w
    of two bf16 values is exact in fp32, so y is determined by r; r is one of the bf16 roundings of x * inv64 * (1 -+
    delta).  Returns (lo, hi): the kernel's y must equal one of them (they differ only where r is ambiguous)."""
    x = np.asarray(x, np.float64)
    w = np.asarray(w, np.float64)
    inv = 1.0 / np.sqrt((x * x).mean(-1, keepdims=True) + eps)
    t = x * inv
    d = rms_delta(x.shape[-1]) * np.abs(t)
    return rbf(rbf(t - d) * w), rbf(rbf(t + d) * w)


# ================================================================================================ dwconv + LayerNorm
def dwconv(x, w, bias, T, hist, x_bs_rows, B, drop=None):
    """Exact (fp64) depthwise causal conv k = 7 of dwconv_ln_kernel: x [B][x_bs_rows][C] (row hist + t is time step t),
    w [C][7], bias [C]; tap j of step t reads row hist + t - 6 + j and is skipped where t - 6 + j < -hist.  Returns
    (acc [B][T][C], abs_sum = |bias| + sum |w x|).  drop: a tap index left out (a plausible slip)."""
    x = np.asarray(x, np.float64).reshape(B, x_bs_rows, -1)
    C = x.shape[2]
    acc = np.broadcast_to(np.asarray(bias, np.float64), (B, T, C)).copy()
    asum = np.abs(acc)
    for j in range(7):
        ts = np.arange(max(0, 6 - j - hist), T)
        if j == drop or not len(ts):
            continue
        p = w[:, j][None, None, :] * x[:, hist + ts - 6 + j, :]
        acc[:, ts] += p
        asum[:, ts] += np.abs(p)
    return acc, asum


def layernorm(pre, lnw, lnb, eps=1e-6):
    """LayerNorm over the last axis, biased variance (F.layer_norm)."""
    m = pre.mean(-1, keepdims=True)
    d = pre - m
    v = (d * d).mean(-1, keepdims=True)
    return d / np.sqrt(v + eps) * lnw + lnb


def ln_bound(pre, lnw, lnb, eps=1e-6, dpre=None, threads=256):
    """Per-element bound of dwconv_ln_kernel's fp32 LayerNorm of the C values pre (bf16, each within dpre of the value
    the kernel holds): two-pass mean and variance, each a block reduction (C / threads terms per thread, a 5-level warp
    tree, the 8 warp partials in order) and a division; + eps, rsqrtf 2 ulp; then (x - mean) * inv * w + b, four
    roundings.  The bound does not depend on the rows' offset from zero."""
    C = pre.shape[-1]
    n = -(-C // threads) + 5 + threads // 32 + 1
    dp = np.zeros_like(pre) if dpre is None else dpre
    m = pre.mean(-1, keepdims=True)
    d = pre - m
    A_ = np.abs(pre).mean(-1, keepdims=True) + dp.mean(-1, keepdims=True)
    # the sum of the mean is exact in fp32 when every partial sum is a multiple of the values' common bf16 granularity
    # below 2^24 of it (rows far from zero: their values share an exponent); only the division rounds then
    exact = C * A_ < 2.0 ** 24 * np.minimum(granularity(pre), granularity(pre - dp)).min(-1, keepdims=True)
    dm = np.where(exact, U * (np.abs(m) + dp.mean(-1, keepdims=True)), n * U * A_) + dp.mean(-1, keepdims=True)
    dd = dm + dp + U * (np.abs(d) + dm + dp)                        # error of each deviation sh[c] - mean
    var = (d * d).mean(-1, keepdims=True)
    dvar = ((2 * np.abs(d) + dd) * dd).mean(-1, keepdims=True) + (n + 1) * U * ((np.abs(d) + dd) ** 2).mean(-1, keepdims=True)
    dvar = dvar + 2 * U * (var + dvar)                              # / C and + eps
    rstd = 1.0 / np.sqrt(var + eps)
    rel_r = 0.5 * dvar / (var + eps) * (1 + dvar / (var + eps)) + 2 * 2.0 ** -23
    wa = np.abs(lnw)
    core = (np.abs(d) * rel_r + dd * (1 + rel_r)) * rstd
    y = d * rstd * lnw + lnb
    ya = np.abs(d) * rstd * wa
    return (wa * core + 3 * U * (ya + wa * core) + U * (np.abs(y) + wa * core)) * 1.01 + 2.0 ** -140


def dwconv_ln(x, w, bias, lnw, lnb, T, hist, x_bs_rows, B, exact=True, drop=None):
    """dwconv_ln_kernel: pre = bf16(fp32 conv), y = bf16(LayerNorm(pre)).  Returns (y64, bound, lo, hi, n_ambiguous): the
    fp64 LayerNorm of the bf16-rounded exact pre, its fp32 bound, and the admissible bf16 interval of every output.  exact: the conv sum is exact
    in fp32 (grid inputs), so pre is known; otherwise a pre whose fp32 sum ((7 + 1) 2^-24 sum |w x|) may round either
    way widens the bound by one bf16 ulp of that channel, propagated through the mean and the variance."""
    acc, asum = dwconv(x, w, bias, T, hist, x_bs_rows, B, drop)
    pre = rbf(acc)
    if exact:
        dpre = np.zeros_like(pre)
    else:
        e = 8 * U * asum
        amb = rbf(acc - e) != rbf(acc + e)
        dpre = np.where(amb, bf16_ulp(acc + e), 0.0)
    y = layernorm(pre, lnw, lnb)
    bound = ln_bound(pre, lnw, lnb, dpre=dpre)
    lo, hi = bf16_interval(y, bound)
    return y, bound, lo, hi, int((dpre > 0).sum())


# ================================================================================================ final conv
def final_conv(x, w, bias, T, hist, x_bs_rows, B, drop=None):
    """Exact (fp64) final causal conv k = 7, C -> 1 of final_conv_kernel: x [B][x_bs_rows][C], w [7][C]; tap j of sample
    t reads row hist + t - 6 + j, skipped where t - 6 + j < -hist.  Returns (acc [B][T], abs_sum)."""
    x = np.asarray(x, np.float64).reshape(B, x_bs_rows, -1)
    acc = np.full((B, T), float(bias))
    asum = np.full((B, T), abs(float(bias)))
    for j in range(7):
        ts = np.arange(max(0, 6 - j - hist), T)
        if j == drop or not len(ts):
            continue
        xs = x[:, hist + ts - 6 + j, :]
        acc[:, ts] += xs @ w[j]
        asum[:, ts] += np.abs(xs) @ np.abs(w[j])
    return acc, asum


def clamp1(v):
    return np.minimum(1.0, np.maximum(-1.0, v))


def final_conv_out(acc, asum, C, exact):
    """The admissible clamp(bf16(acc)) interval: exact sums round once; otherwise the fp32 chain of 7 C + 1 terms,
    (7 C + 1) 2^-24 (|bias| + sum |w x|)."""
    e = 0.0 if exact else (7 * C + 1) * U * asum
    lo, hi = bf16_interval(acc, e)
    return clamp1(lo), clamp1(hi)


# ================================================================================================ history roll / reset / copy
def roll(buf, hist, factor, counts):
    """roll_history_kernel on one buffer buf [B][bs_rows][C] (any dtype, copied bit for bit): a row b with T = factor *
    counts[b] > 0 moves rows [T, T + hist) to [0, hist)."""
    out = buf.copy()
    for b, c in enumerate(counts):
        T = factor * c
        if T:
            out[b, :hist] = out[b, T:T + hist].copy()
    return out


def reset(buf, hist, flags):
    """reset_history_kernel / enc_reset_kernel on one buffer: rows [0, hist) of the batch rows with a nonzero flag are
    zero (buf [B][rows][C] for the decoder, [B][C][ld] with the history along the last axis for the encoder: pass
    axis-moved views)."""
    out = buf.copy()
    for b, f in enumerate(flags):
        if f:
            out[b, :hist] = 0
    return out


def copy_rows(dst, src, hist, src_rows, dst_rows):
    """copy_rows_kernel on one buffer pair: dst[dst_rows[i]][0:hist] = src[src_rows[i]][0:hist]."""
    out = dst.copy()
    for s, d in zip(src_rows, dst_rows):
        out[d, :hist] = src[s, :hist]
    return out


# ================================================================================================ prefill index
def pf_index(lens, slots, p0, trailing_len, V, state, seen, src, dst, stride, cap, H, prefix_kv, kc, vc, lh):
    """pf_index_kernel.  state: dict of int arrays [MAXB] (finished, n_valid, n_gen, c0, len0, trailing_len); seen
    [MAXB][V] uint8; src [n][stride][H], dst [MAXB][cap][H] (int16 bits); prefix_kv[r]: None or int16 [2][lh][p0][HD]
    (K then V); kc / vc [MAXB][lh][kcap][HD].  Returns (tok_seq, tok_pos, state, seen, dst, kc, vc)."""
    start = np.concatenate([[0], np.cumsum(lens)]).astype(int)
    tok_seq = np.concatenate([np.full(l, s) for l, s in zip(lens, slots)]).astype(np.int32)
    tok_pos = np.concatenate([p + np.arange(l) for l, p in zip(lens, p0)]).astype(np.int32)
    st = {k: v.copy() for k, v in state.items()}
    seen, dst, kc, vc = seen.copy(), dst.copy(), kc.copy(), vc.copy()
    for r, b in enumerate(slots):
        st["finished"][b] = st["n_valid"][b] = st["n_gen"][b] = st["c0"][b] = 0
        st["len0"][b] = p0[r] + start[r + 1] - start[r]
        st["trailing_len"][b] = trailing_len[r]
        seen[b] = 0
        tl = trailing_len[r]
        dst[b].reshape(-1)[:tl * H] = src[r].reshape(-1)[:tl * H]
        if prefix_kv[r] is not None:
            kc[b, :, :p0[r]] = prefix_kv[r][0]
            vc[b, :, :p0[r]] = prefix_kv[r][1]
    return tok_seq, tok_pos, st, seen, dst, kc, vc


def pf_gather_last(lens, slots, x, h_last):
    """pf_gather_last_kernel: h_last[slots[r]] = x[(last packed row of r)]."""
    out = h_last.copy()
    ends = np.cumsum(lens)
    for r, b in enumerate(slots):
        out[b] = x[ends[r] - 1]
    return out


def release(state, slots):
    """release_state_kernel: a listed slot that is not finished becomes finished with n_valid = 0x3fffffff."""
    st = {k: v.copy() for k, v in state.items()}
    for b in slots:
        if not st["finished"][b]:
            st["finished"][b] = 1
            st["n_valid"][b] = 0x3FFFFFFF
    return st


# ================================================================================================ streaming encoder
def load_wav(src, dst, n, counts, factor):
    """load_wav_kernel: dst[b][t] = src[b][t] for t < factor * counts[b], 0 for the rest of [0, n); dst past n unchanged."""
    out = dst.copy()
    for b, c in enumerate(counts):
        v = min(factor * c, n)
        out[b, :v] = src[b, :v]
        out[b, v:n] = 0
    return out


def seed_replicate(h, hist, pos, counts):
    """seed_replicate_kernel on h [B][C][ld]: a row at position 0 with frames gets hist copies of column hist."""
    out = h.copy()
    for b in range(h.shape[0]):
        if pos[b] == 0 and counts[b] != 0:
            out[b, :, :hist] = out[b, :, hist:hist + 1]
    return out


def code_frames(count, ds):
    """12.5 Hz frames a segment of `count` 25 Hz frames yields: ceil(count / ds)."""
    return -(-count // ds)


def mask_codes(codes, counts, ds):
    """mask_codes_kernel on codes [B][nq][T]: -1 at frames t >= ceil(counts[b] / ds)."""
    out = codes.copy()
    for b, c in enumerate(counts):
        out[b, :, code_frames(c, ds):] = -1
    return out
