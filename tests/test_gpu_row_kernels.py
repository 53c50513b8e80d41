"""Direct checks of the row-wise kernels that run on every request, call by call, against the fp64 references and numpy
restatements of tests/rows_ref.py, at their rounding, view, count and history edges:
- the codec decoder's rvq_gather, rmsnorm_rows, dwconv_ln, final_conv, roll_history, reset_history and copy_rows
  (csrc/codec_kernels.cuh);
- the prefill's pf_rmsnorm, pf_index, pf_prefix_index, pf_gather_last, release_state and bf16_to_f32 (csrc/ar_prefill.cuh);
- the streaming codec encoder's load_wav, seed_replicate, mask_codes and enc_reset (csrc/codec_encoder_kernels.cuh).
They run through tests/csrc/rows_shim.cu, which compiles the kernels from the shipped headers under the library's flags
and launches each with its engine's geometry.

Acceptance rules.
- rvq_gather: bit for bit against the numpy replay of acc = rbf(fp32(acc + v)) over k = 1 .. K-1, which is torch's bf16
  sequential sum.  Planted absorption and cancellation sums make the order visible: each such case asserts that the
  reversed order gives different bits.  Frames past a row's count are exactly zero.
- rmsnorm_rows / pf_rmsnorm: r * w of two bf16 values is exact in fp32, so the output is bf16(r * w) with r one of the
  bf16 roundings of x * inv64 * (1 -+ delta), delta covering the kernel's fp32 sum of squares, the division, + eps and
  rsqrtf's 2 ulp.  Every element must be one of the (at most two) admissible values; the ambiguous elements are counted
  and must stay a small fraction.  Rows where eps dominates must fail the check with eps doubled.
- dwconv_ln: grid inputs (small integers x 2^-4) make the conv sum exact, so the pre-LayerNorm bf16 value is known and
  the output must lie in the bf16 interval of the fp64 LayerNorm -+ the two-pass fp32 bound (rows_ref.ln_bound); each
  grid case asserts that dropping any single tap moves some output beyond twice that bound.  Random inputs widen the
  bound by one bf16 ulp of every channel whose conv rounding is ambiguous.  A family of rows offset from zero by 0, 32,
  128 and 512 standard deviations is held to the same offset-independent bound.  The history view equals the one-shot
  over the same rows bit for bit, and a zeroed history equals hist = 0 bit for bit.
- final_conv: grid inputs bit for bit; random inputs in the bf16 interval of the fp32 chain bound (7 C + 1) 2^-24
  (|bias| + sum |w x|), then the clamp.  Samples at or past count * up are exactly zero.
- roll / reset / copy, pf_index / pf_prefix_index / pf_gather_last / release_state / bf16_to_f32 and the encoder's
  load_wav / seed_replicate / mask_codes / enc_reset: bit for bit against the numpy restatements, on random bit patterns
  (NaN payloads included).
- Guards: outputs start as a NaN sentinel (or random bits); every row, column, slot or state field outside a launch's
  view must come back bit-unchanged.
STATS collects the ambiguous-rounding counts, the smallest sensitivity and the case counts, printed at the end.
"""
import ctypes as C
import math
import os
import subprocess
import zlib

import numpy as np
import pytest
import torch

from tests import rows_ref as R
from tests.attention_ref import rbf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM_SRC = os.path.join(ROOT, "tests", "csrc", "rows_shim.cu")
SENT16 = np.int16(0x7FC1)          # bf16 NaN with a payload
SENT32 = np.uint32(0x7FC00ABC)
STATS = {"exact": 0, "bounded": 0, "min_sensitivity": math.inf, "rms_ambiguous": 0, "rms_elements": 0,
         "conv_ambiguous": 0, "offset_ratio": []}
FIELDS = ("finished", "n_valid", "n_gen", "c0", "len0", "trailing_len")
pytestmark = pytest.mark.gpu


# ================================================================================================ shim
@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    """tests/csrc/rows_shim.cu compiled for sm_90a with the library's flags; it links against nothing."""
    from qwen3_tts_b200 import build
    out = str(tmp_path_factory.mktemp("rows_shim") / "librows_shim.so")
    cmd = [build._nvcc()] + build.NVCC_FLAGS + ["-shared", "-I", build.CSRC, SHIM_SRC, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"shim build failed:\n{r.stdout}\n{r.stderr}"
    L = C.CDLL(out)
    vp, i32, f32 = C.c_void_p, C.c_int, C.c_float
    pp, pi = C.POINTER(C.c_void_p), C.POINTER(C.c_int)
    sig = {
        "rows_shim_state": [i32, pi],
        "rows_shim_rvq_gather": [vp, vp, vp, i32, i32, i32, i32, i32, vp, vp],
        "rows_shim_rmsnorm_rows": [vp, vp, vp, i32, i32, f32, vp],
        "rows_shim_pf_rmsnorm": [vp, vp, vp, i32, i32, f32, vp],
        "rows_shim_dwconv_ln": [vp] * 6 + [i32] * 5 + [vp],
        "rows_shim_final_conv": [vp] * 4 + [i32] * 5 + [vp, i32, vp],
        "rows_shim_roll": [pp, pi, pi, pi, pi, i32, vp, i32, vp],
        "rows_shim_reset": [pp, pi, pi, pi, pi, i32, vp, i32, vp],
        "rows_shim_copy": [pp, pp, pi, pi, pi, pi, i32, vp, i32, i32, vp],
        "rows_shim_pf_index": [i32, pi, pi, pi, pi, vp, vp, i32, i32, i32, pp, vp, vp, i32, i32, vp, i32, vp, vp, vp],
        "rows_shim_pf_prefix_index": [i32, vp, vp, vp],
        "rows_shim_pf_gather_last": [i32, pi, pi, vp, vp, i32, vp],
        "rows_shim_release": [i32, pi, vp],
        "rows_shim_bf16_to_f32": [vp, vp, i32, vp],
        "rows_shim_load_wav": [vp, i32, vp, i32, i32, vp, i32, i32, vp],
        "rows_shim_seed_replicate": [vp, i32, i32, i32, vp, i32, vp],
        "rows_shim_mask_codes": [vp, i32, i32, vp, i32, i32, vp],
        "rows_shim_enc_reset": [pp, pi, pi, pi, pi, i32, vp, i32, vp],
    }
    for name, args in sig.items():
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = args
    L.rows_shim_layout.restype = i32
    L.rows_shim_layout.argtypes = [C.c_char_p]
    L.maxb, L.hd = L.rows_shim_layout(b"maxb"), L.rows_shim_layout(b"hd")
    L.roll_max = L.rows_shim_layout(b"roll_max")
    yield L
    print("\nrow kernel STATS:", STATS)


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def rng_for(name):
    return np.random.default_rng(zlib.crc32(name.encode()))


def ok(rc, what):
    assert rc == 0, f"{what}: launch failed ({rc})"


def ints(a):
    a = [int(v) for v in a]
    return (C.c_int * max(1, len(a)))(*a)


def ptrs(ts):
    return (C.c_void_p * max(1, len(ts)))(*[None if t is None else t.data_ptr() for t in ts])


def bf_dev(a):
    """bf16 device tensor of bf16-exact float64 values."""
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(torch.bfloat16).cuda()


def f32_dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def i32_dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.int32)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu()


def bf_host(t):
    return host(t).to(torch.float64).numpy()


def bits16(t):
    return host(t).view(torch.int16).numpy()


def bf_bits(a):
    return (np.asarray(a, np.float32).view(np.uint32) >> 16).astype(np.uint16).view(np.int16)


def sentinel_bf(n):
    return torch.full((n,), int(SENT16), dtype=torch.int16).cuda().view(torch.bfloat16)


def rand_bits16(g, shape):
    return torch.from_numpy(g.integers(-32768, 32768, shape, dtype=np.int64).astype(np.int16)).cuda()


def rp_dev(pos, counts):
    return i32_dev(list(pos) + list(counts))


def check_sensitivity(what, sens):
    STATS["min_sensitivity"] = min(STATS["min_sensitivity"], sens)
    assert sens > 1.0, f"{what}: the slip moves no output element beyond twice the bound ({sens:.3f})"


def grid(g, shape, lo=-8, hi=8):
    """Small integers x 2^-4, never zero."""
    v = g.integers(lo, hi, shape).astype(np.float64)
    v[v == 0] = 1
    return v / 16


def in_interval(what, got, lo, hi):
    bad = ~((got >= lo) & (got <= hi))
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {got.size} outside the admissible set, first at "
                           f"{np.argwhere(bad)[0]}: got {got[bad][0]!r}, admissible [{lo[bad][0]!r}, {hi[bad][0]!r}]")


# ================================================================================================ rvq_gather
def run_rvq(lib, codes, table, count=None):
    B, K, T = codes.shape
    D = table.shape[2]
    tab, cd = bf_dev(table), i32_dev(codes)
    rp = None if count is None else rp_dev([0] * B, count)
    guard = 2 * D + 5
    e = sentinel_bf(B * T * 2 * D + guard)
    ok(lib.rows_shim_rvq_gather(cd.data_ptr(), tab.data_ptr(), e.data_ptr(), B, K, T, D, table.shape[1],
                                None if rp is None else rp.data_ptr(), stream()), "rvq_gather")
    b = bits16(e)
    assert (b[B * T * 2 * D:] == SENT16).all(), "rvq_gather wrote past its output"
    return b[:B * T * 2 * D].reshape(B, T, 2 * D)


@pytest.mark.parametrize("K,D,bins,count", [(16, 256, 2048, None), (1, 256, 2048, None), (2, 256, 2048, None),
                                            (16, 96, 64, (0, 3, 7)), (16, 200, 2048, None), (16, 256, 2048, (7, 0))])
def test_rvq_gather(lib, K, D, bins, count):
    g = rng_for(f"rvq{K}{D}{bins}{count}")
    B = 2 if count is None or len(count) == 2 else 3
    T = 7
    table = rbf(g.standard_normal((K, bins, D)) * np.exp2(g.integers(-6, 6, (K, bins, 1))))
    codes = g.integers(0, bins, (B, K, T))
    codes[0, :, 1] = 0
    codes[B - 1, :, 2] = bins - 1
    planted = K >= 3
    if planted:  # frame (0, 0): absorption in half the dims (1 + many 2^-9), cancellation in the other half
        for k in range(K):
            table[k, 1, :D // 2] = 1.0 if k <= 1 else 2.0 ** -9
            table[k, 1, D // 2:] = {1: 2.0 ** 10, 2: -2.0 ** 10}.get(k, 1.5 * 2.0 ** -k)
        codes[0, :, 0] = 1
    got = run_rvq(lib, codes, table, count)
    want = bf_bits(R.rvq_gather(codes, table, count))
    assert np.array_equal(got, want), f"rvq_gather: {int((got != want).sum())} elements differ"
    if planted:
        rev = bf_bits(R.rvq_gather(codes, table, count, reverse=True))
        n0 = T if count is None else count[0]
        if n0 > 0:
            assert (rev[0, 0, D:] != want[0, 0, D:]).any(), "the planted sums do not depend on the order"
            assert (rev[0, 0, D:D + D // 2] != want[0, 0, D:D + D // 2]).any()
            assert (rev[0, 0, D + D // 2:] != want[0, 0, D + D // 2:]).any()
    if K == 1:
        assert (got[..., D:] == 0).all()
    if count is not None:
        for b, c in enumerate(count):
            assert (got[b, c:] == 0).all()
    STATS["exact"] += 1


# ================================================================================================ RMSNorm
def rms_rows(g, rows, C):
    x = rbf(g.standard_normal((rows, C)) * np.exp2(g.integers(-3, 4, (rows, 1))))
    x[1] = 0.0                                                   # all-zero row
    x[2] = rbf(g.standard_normal(C) * 2.0 ** -14)                # eps dominates the mean square
    x[3] = 0.0
    x[3, C // 3] = 96.0                                          # single spike
    x[4] = rbf(g.standard_normal(C) * 2.0 ** -9)                 # eps comparable to the mean square
    return x


@pytest.mark.parametrize("kind,C,rows,eps", [("rows", 1024, 13, 1e-5), ("rows", 2048, 17, 1e-6), ("rows", 40, 9, 1e-5),
                                             ("rows", 1000, 8, 1e-5), ("pf", 1024, 13, 1e-6), ("pf", 2048, 21, 1e-6),
                                             ("pf", 264, 11, 1e-5), ("pf", 2048, 1, 1e-6)])
def test_rmsnorm(lib, kind, C, rows, eps):
    g = rng_for(f"rms{kind}{C}{rows}")
    x = rms_rows(g, max(rows, 5), C)[:rows] if rows >= 5 else rbf(g.standard_normal((rows, C)))
    w = rbf(g.standard_normal(C) * 2)
    xd, wd = bf_dev(x), bf_dev(w)
    guard = 3 * C
    y = sentinel_bf(rows * C + guard)
    fn = lib.rows_shim_rmsnorm_rows if kind == "rows" else lib.rows_shim_pf_rmsnorm
    ok(fn(xd.data_ptr(), wd.data_ptr(), y.data_ptr(), rows, C, eps, stream()), kind)
    assert (bits16(y)[rows * C:] == SENT16).all(), f"{kind}: rows past the count written"
    got = bf_host(y)[:rows * C].reshape(rows, C)
    lo, hi = R.rmsnorm(x, w, eps)
    bad = (got != lo) & (got != hi)
    assert not bad.any(), f"{kind}: {int(bad.sum())} elements outside the admissible set, first {np.argwhere(bad)[0]}"
    amb = int((lo != hi).sum())
    STATS["rms_ambiguous"] += amb
    STATS["rms_elements"] += x.size
    assert amb <= 0.02 * x.size, f"{kind}: {amb} ambiguous elements of {x.size}: the check is nearly vacuous"
    if rows >= 5:
        assert (got[1] == 0).all() and (got[3][np.arange(C) != C // 3] == 0).all()
        for r in (2, 4):   # eps matters here: doubling it must break the check
            lo2, hi2 = R.rmsnorm(x[r:r + 1], w, 2 * eps)
            assert ((got[r] != lo2[0]) & (got[r] != hi2[0])).any(), f"{kind}: row {r} also passes with eps doubled"
        # a wrong divisor (C + 8) must break the check on an ordinary row
        inv = 1.0 / np.sqrt((x[0] ** 2).sum() / (C + 8) + eps)
        assert (rbf(rbf(x[0] * inv) * w) != got[0]).any()
    STATS["exact"] += 1


# ================================================================================================ dwconv + LayerNorm
def run_dw(lib, xfull, w, bias, lnw, lnb, B, T, C, x_bs_rows, hist):
    xd = bf_dev(xfull)
    wd, bd, lwd, lbd = f32_dev(w), f32_dev(bias), f32_dev(lnw), f32_dev(lnb)
    guard = 2 * C
    y = sentinel_bf(B * T * C + guard)
    ok(lib.rows_shim_dwconv_ln(xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), lwd.data_ptr(), lbd.data_ptr(), y.data_ptr(),
                               B, T, C, x_bs_rows, hist, stream()), "dwconv_ln")
    assert (bits16(y)[B * T * C:] == SENT16).all(), "dwconv_ln wrote past its output"
    return bf_host(y)[:B * T * C].reshape(B, T, C)


def dw_inputs(g, B, T, C, hist, cap, kind, offset=0.0):
    rows = hist + cap
    if kind == "grid":   # conv outputs of spread about 0.36, centred at offset x that spread
        x = grid(g, (B, rows, C))
        w, bias = grid(g, (C, 7)), grid(g, C) + np.round(offset * 0.36 * 16) / 16
    else:
        x = rbf(g.standard_normal((B, rows, C)))
        w = g.standard_normal((C, 7)).astype(np.float32).astype(np.float64) / math.sqrt(7)
        bias = (g.standard_normal(C) * 0.1 + offset).astype(np.float32).astype(np.float64)
    lnw = (1 + 0.2 * g.standard_normal(C)).astype(np.float32).astype(np.float64)
    lnb = (0.2 * g.standard_normal(C)).astype(np.float32).astype(np.float64)
    x[:, hist + T:] = np.nan                 # rows past the view: reading one shows
    return x, w, bias, lnw, lnb


def check_dw(what, got, x, w, bias, lnw, lnb, B, T, hist, rows, exact):
    y, bound, lo, hi, namb = R.dwconv_ln(x, w, bias, lnw, lnb, T, hist, rows, B, exact=exact)
    in_interval(what, got, lo, hi)
    STATS["conv_ambiguous"] += namb
    STATS["exact" if exact else "bounded"] += 1
    return y, bound


@pytest.mark.parametrize("C,T,hist,kind", [(1024, 9, 0, "grid"), (1024, 4, 6, "grid"), (96, 9, 0, "grid"),
                                           (300, 7, 0, "grid"), (1024, 9, 0, "rand"), (1024, 5, 6, "rand"),
                                           (200, 8, 0, "rand"), (1536, 3, 6, "rand")])
def test_dwconv_ln(lib, C, T, hist, kind):
    g = rng_for(f"dw{C}{T}{hist}{kind}")
    B = 3
    cap = T + 2
    x, w, bias, lnw, lnb = dw_inputs(g, B, T, C, hist, cap, kind)
    rows = hist + cap
    got = run_dw(lib, x, w, bias, lnw, lnb, B, T, C, rows, hist)
    y, bound = check_dw(f"dwconv_ln C={C} T={T} hist={hist}", got, x, w, bias, lnw, lnb, B, T, hist, rows, kind == "grid")
    if kind == "grid":
        for j in range(7):
            yd, *_ = R.dwconv_ln(x, w, bias, lnw, lnb, T, hist, rows, B, drop=j)
            check_sensitivity(f"dwconv_ln drop tap {j}", float(np.nanmax(np.abs(yd - y) / (2 * bound))))


def test_dwconv_ln_history_views(lib):
    """The hist = 6 view equals the one-shot over history + new rows bit for bit; a zeroed history equals hist = 0."""
    g = rng_for("dwviews")
    B, T, C = 2, 5, 1024
    x, w, bias, lnw, lnb = dw_inputs(g, B, T, C, 6, T, "rand")
    one = run_dw(lib, x, w, bias, lnw, lnb, B, 6 + T, C, 6 + T, 0)
    view = run_dw(lib, x, w, bias, lnw, lnb, B, T, C, 6 + T, 6)
    assert np.array_equal(bf_bits(view), bf_bits(one[:, 6:]))
    xz = x.copy()
    xz[:, :6] = 0.0
    zero_hist = run_dw(lib, xz, w, bias, lnw, lnb, B, T, C, 6 + T, 6)
    no_hist = run_dw(lib, np.ascontiguousarray(x[:, 6:]), w, bias, lnw, lnb, B, T, C, T, 0)
    assert np.array_equal(bf_bits(zero_hist), bf_bits(no_hist))
    STATS["exact"] += 2


@pytest.mark.parametrize("offset", [0.0, 32.0, 128.0, 512.0])
def test_dwconv_ln_mean_offset(lib, offset):
    """Rows whose conv outputs sit `offset` standard deviations from zero: the LayerNorm must hold the same two-pass
    bound as centred rows (a one-pass q / C - mean^2 variance loses about log2(offset^2) bits of it)."""
    g = rng_for(f"dwoff{offset}")
    B, T, C = 4, 8, 1024
    x, w, bias, lnw, lnb = dw_inputs(g, B, T, C, 0, T, "grid", offset=offset)
    got = run_dw(lib, x, w, bias, lnw, lnb, B, T, C, T, 0)
    acc, _ = R.dwconv(x, w, bias, T, 0, T, B)
    pre = rbf(acc)
    ratio = np.abs(pre.mean(-1)) / pre.std(-1)
    assert np.all(np.abs(ratio - offset) <= 0.3 * offset + 0.5), ratio
    STATS["offset_ratio"].append(round(float(ratio.mean()), 1))
    check_dw(f"dwconv_ln offset {offset}", got, x, w, bias, lnw, lnb, B, T, 0, T, True)


# ================================================================================================ final conv
def run_fc(lib, xfull, w, bias, B, T, C, x_bs_rows, hist, count=None, up=1):
    xd, wd, bd = bf_dev(xfull), f32_dev(w), f32_dev([bias])
    rp = None if count is None else rp_dev([0] * B, count)
    guard = 37
    wav = torch.from_numpy(np.full(B * T + guard, SENT32, np.uint32).view(np.float32)).cuda()
    ok(lib.rows_shim_final_conv(xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), wav.data_ptr(), B, T, C, x_bs_rows, hist,
                                None if rp is None else rp.data_ptr(), up, stream()), "final_conv")
    out = host(wav).numpy()
    assert (out[B * T:].view(np.uint32) == SENT32).all(), "final_conv wrote past its output"
    return out[:B * T].astype(np.float64).reshape(B, T)


@pytest.mark.parametrize("C,T,hist,kind,count,up", [(96, 11, 0, "grid", None, 1), (96, 9, 6, "grid", None, 1),
                                                    (16, 12, 0, "grid", (0, 2, 4), 3), (96, 40, 6, "rand", None, 1),
                                                    (16, 33, 0, "rand", (11, 5), 3), (96, 10, 6, "rand", (1, 0, 3), 2)])
def test_final_conv(lib, C, T, hist, kind, count, up):
    g = rng_for(f"fc{C}{T}{hist}{kind}{count}")
    B = 2 if count is None else len(count)
    rows = hist + T + 2
    if kind == "grid":
        x, w, bias = grid(g, (B, rows, C)) / 4, grid(g, (7, C)) / 4, 0.25
    else:
        x = rbf(g.standard_normal((B, rows, C)) * 0.3)
        w = (g.standard_normal((7, C)) * 0.3 / math.sqrt(C)).astype(np.float32).astype(np.float64) * 4
        bias = float(np.float32(0.05))
    x[:, hist + T:] = np.nan
    got = run_fc(lib, x, w, bias, B, T, C, rows, hist, count, up)
    acc, asum = R.final_conv(x, w, bias, T, hist, rows, B)
    lo, hi = R.final_conv_out(acc, asum, C, kind == "grid")
    if count is not None:
        for b, c in enumerate(count):
            lo[b, c * up:] = hi[b, c * up:] = 0.0
            tail = got[b, c * up:]
            assert (tail == 0).all() and not np.signbit(tail).any()
    in_interval(f"final_conv {kind}", got, lo, hi)
    if kind == "grid":
        for j in range(7):
            accd, _ = R.final_conv(x, w, bias, T, hist, rows, B, drop=j)
            live = np.ones_like(acc, bool) if count is None else (np.arange(T)[None, :] < np.array(count)[:, None] * up)
            moved = (R.clamp1(rbf(accd)) != got) & live
            assert moved.any(), f"final_conv: dropping tap {j} changes no output"
    STATS["exact" if kind == "grid" else "bounded"] += 1


def test_final_conv_clamp_edges(lib):
    """Values beyond -+1, exactly -+1, and fp32 sums that round to -+1 in bf16 (ties to even) before the clamp."""
    B, C, hist = 1, 16, 0
    pairs = [(1.0078125, 0), (1.0, 0), (-1.0, 0), (1.5, 0), (-3.0, 0), (1 - 2 ** -8, 2 ** -9), (-(1 - 2 ** -8), -2 ** -9),
             (1 - 2 ** -8, 2 ** -9 - 2 ** -12), (1 - 2 ** -8, 2 ** -10), (0.5, 0.25), (1.0, 2 ** -8), (-1.0, -2 ** -7)]
    T = len(pairs)
    x = np.zeros((B, T, C))
    x[0, :, 0] = [p[0] for p in pairs]
    x[0, :, 1] = [p[1] for p in pairs]
    x[0, :, 2:] = rbf(rng_for("clamp").standard_normal((T, C - 2)))
    w = np.zeros((7, C))
    w[6, 0] = w[6, 1] = 1.0
    got = run_fc(lib, x, w, 0.0, B, T, C, T, hist)
    want = R.clamp1(rbf(x[0, :, 0] + x[0, :, 1]))
    assert np.array_equal(got[0], want), (got[0], want)
    assert list(want[[5, 6, 7, 8]]) == [1.0, -1.0, 1 - 2 ** -8, 1 - 2 ** -8]
    STATS["exact"] += 1


def test_final_conv_grid_stride(lib):
    """B * T beyond the 1184 x 256 grid: the grid-stride loop's second pass, bit for bit on grid inputs."""
    g = rng_for("fcstride")
    B, T, C = 2, 160000, 16
    rows = T + 6
    x = grid(g, (B, rows, C)) / 4
    w = grid(g, (7, C)) / 4
    got = run_fc(lib, x, w, 0.125, B, T, C, rows, 6)
    acc, _ = R.final_conv(x, w, 0.125, T, 6, rows, B)
    assert B * T > 1184 * 256
    assert np.array_equal(got, R.clamp1(rbf(acc)))
    STATS["exact"] += 1


# ================================================================================================ roll / reset / copy
def hist_entries(g, n, B):
    ents = []
    for i in range(n):
        hist = int(g.integers(1, 9))
        factor = int(g.choice([1, 2, 4, 8]))
        C = int(g.choice([16, 32, 48, 112, 256, 1024, 2048]))
        bs_rows = hist + factor * 9 + int(g.integers(0, 3))
        ents.append(dict(hist=hist, factor=factor, C=C, bs_rows=bs_rows, buf=rand_bits16(g, (B, bs_rows, C))))
    return ents


def table_args(ents):
    return (ptrs([e["buf"] for e in ents]), ints([e["hist"] for e in ents]), ints([e["factor"] for e in ents]),
            ints([e["C"] for e in ents]), ints([e["bs_rows"] for e in ents]), len(ents))


@pytest.mark.parametrize("n,B", [(5, 6), (48, 1), (48, 32)])
def test_roll_and_reset(lib, n, B):
    g = rng_for(f"roll{n}{B}")
    assert n <= lib.roll_max
    ents = hist_entries(g, n, B)
    before = [host(e["buf"]).numpy().copy() for e in ents]
    # counts: 0 (untouched), 1 (T < hist for most entries: the overlapping move) and up to 9 (T >= hist)
    counts = ([0, 1, 9, 2, 5, 3] * 6)[:B] if B > 1 else [1]
    rp = rp_dev([7] * B, counts)
    ok(lib.rows_shim_roll(*table_args(ents), rp.data_ptr(), B, stream()), "roll")
    for e, b0 in zip(ents, before):
        want = R.roll(b0, e["hist"], e["factor"], counts)
        assert np.array_equal(host(e["buf"]).numpy(), want), f"roll hist={e['hist']} factor={e['factor']} C={e['C']}"
    flags = ([1, 0, 3, 0, 0, 1] * 6)[:B] if B > 1 else [1]
    rolled = [host(e["buf"]).numpy().copy() for e in ents]
    rp2 = rp_dev([0] * B, flags)
    ok(lib.rows_shim_reset(*table_args(ents), rp2.data_ptr(), B, stream()), "reset")
    for e, b0 in zip(ents, rolled):
        want = R.reset(b0, e["hist"], flags)
        got = host(e["buf"]).numpy()
        assert np.array_equal(got, want), f"reset hist={e['hist']} C={e['C']}"
        # the slip "reset zeroes hist - 1 rows" must fail
        assert not np.array_equal(R.reset(b0, e["hist"] - 1, flags), got) or not any(flags)
    STATS["exact"] += 2


def test_copy_rows(lib):
    g = rng_for("copy")
    Bs, Bd, n = 5, 7, 6
    src_rows, dst_rows = [3, 0, 4, 1], [6, 1, 2, 4]
    srcs, dsts, hists, Cs, sbs, dbs = [], [], [], [], [], []
    for i in range(n):
        hist, Cc = int(g.integers(1, 9)), int(g.choice([16, 64, 1024]))
        s_rows, d_rows = hist + int(g.integers(0, 20)), hist + int(g.integers(0, 20))
        srcs.append(rand_bits16(g, (Bs, s_rows, Cc)))
        dsts.append(rand_bits16(g, (Bd, d_rows, Cc)))
        hists.append(hist); Cs.append(Cc); sbs.append(s_rows); dbs.append(d_rows)
    before = [host(d).numpy().copy() for d in dsts]
    rows = i32_dev(src_rows + [0] * (Bd - len(src_rows)) + dst_rows + [0] * (Bd - len(dst_rows)))
    ok(lib.rows_shim_copy(ptrs(dsts), ptrs(srcs), ints(hists), ints(Cs), ints(dbs), ints(sbs), n, rows.data_ptr(), Bd,
                          len(src_rows), stream()), "copy_rows")
    for i in range(n):
        want = R.copy_rows(before[i], host(srcs[i]).numpy(), hists[i], src_rows, dst_rows)
        assert np.array_equal(host(dsts[i]).numpy(), want), f"copy_rows entry {i}"
    STATS["exact"] += 1


# ================================================================================================ prefill index kernels
def get_state(lib):
    a = (C.c_int * (6 * lib.maxb))()
    ok(lib.rows_shim_state(0, a), "state")
    v = np.frombuffer(a, np.int32).reshape(6, lib.maxb)
    return {f: v[i].copy() for i, f in enumerate(FIELDS)}


def set_state(lib, st):
    a = (C.c_int * (6 * lib.maxb))(*np.concatenate([st[f] for f in FIELDS]).tolist())
    ok(lib.rows_shim_state(1, a), "state")


def random_state(g, maxb):
    return {f: g.integers(-5, 1 << 20, maxb).astype(np.int32) for f in FIELDS}


@pytest.mark.parametrize("n", [1, 3, 17, 32])
def test_pf_index(lib, n):
    g = rng_for(f"pfidx{n}")
    MAXB, HD = lib.maxb, lib.hd
    V, H, stride, cap, lh, kcap = 3072, 64, 9, 8, 3, 24
    slots = g.permutation(MAXB)[:n].tolist()
    lens = g.integers(1, 300, n)
    lens[0] = 1
    lens[n // 2] = 256 if n > 2 else lens[n // 2]
    p0 = [int(g.integers(1, kcap - 4)) if (r % 2 == 1 or n == 1) else 0 for r in range(n)]
    trailing = [cap if r % 3 == 0 else (0 if r % 3 == 1 else int(g.integers(1, cap))) for r in range(n)]
    st0 = random_state(g, MAXB)
    set_state(lib, st0)
    seen = torch.from_numpy(g.integers(0, 256, (MAXB, V)).astype(np.uint8)).cuda()
    src = rand_bits16(g, (n, stride, H))
    dst = rand_bits16(g, (MAXB, cap, H))
    kc, vc = rand_bits16(g, (MAXB, lh, kcap, HD)), rand_bits16(g, (MAXB, lh, kcap, HD))
    pkv = [rand_bits16(g, (2, lh, p, HD)) if p else None for p in p0]
    ntok = int(lens.sum())
    seq = i32_dev(np.full(ntok + 300, -7))
    pos = i32_dev(np.full(ntok + 300, -7))
    b_seen, b_dst, b_kc, b_vc = (host(t).numpy().copy() for t in (seen, dst, kc, vc))
    ok(lib.rows_shim_pf_index(n, ints(lens), ints(slots), ints(p0), ints(trailing), src.data_ptr(), dst.data_ptr(), stride,
                              cap, H, ptrs(pkv), kc.data_ptr(), vc.data_ptr(), lh, kcap, seen.data_ptr(), V,
                              seq.data_ptr(), pos.data_ptr(), stream()), "pf_index")
    want = R.pf_index(lens, slots, p0, trailing, V, st0, b_seen, host(src).numpy(), b_dst, stride, cap, H,
                      [None if p is None else host(p).numpy() for p in pkv], b_kc, b_vc, lh)
    w_seq, w_pos, w_st, w_seen, w_dst, w_kc, w_vc = want
    gs, gp = host(seq).numpy(), host(pos).numpy()
    assert np.array_equal(gs[:ntok], w_seq) and np.array_equal(gp[:ntok], w_pos)
    assert (gs[ntok:] == -7).all() and (gp[ntok:] == -7).all(), "token index written past ntok"
    got_st = get_state(lib)
    for f in FIELDS:
        assert np.array_equal(got_st[f], w_st[f]), f"DevState.{f}"
    assert np.array_equal(host(seen).numpy(), w_seen)
    assert np.array_equal(host(dst).numpy(), w_dst)
    assert np.array_equal(host(kc).numpy(), w_kc) and np.array_equal(host(vc).numpy(), w_vc)
    # a tok_pos off by one, or a prefix copied one position short, would not match
    assert not np.array_equal(w_pos + 1, gp[:ntok])
    if any(p0):
        r = next(i for i, p in enumerate(p0) if p)
        short = list(p0)
        short[r] -= 1
        w2 = R.pf_index(lens, slots, short, trailing, V, st0, b_seen, host(src).numpy(), b_dst, stride, cap, H,
                        [None if p is None else host(p).numpy()[:, :, :q] for p, q in zip(pkv, short)], b_kc, b_vc, lh)
        assert not np.array_equal(w2[5], w_kc)
    STATS["exact"] += 1


@pytest.mark.parametrize("n", [1, 255, 256, 257, 1000])
def test_pf_prefix_index(lib, n):
    seq, pos = i32_dev(np.full(n + 300, -7)), i32_dev(np.full(n + 300, -7))
    ok(lib.rows_shim_pf_prefix_index(n, seq.data_ptr(), pos.data_ptr(), stream()), "pf_prefix_index")
    gs, gp = host(seq).numpy(), host(pos).numpy()
    assert (gs[:n] == 0).all() and np.array_equal(gp[:n], np.arange(n)) and (gs[n:] == -7).all() and (gp[n:] == -7).all()
    STATS["exact"] += 1


@pytest.mark.parametrize("n,H", [(1, 2048), (5, 64), (32, 1024)])
def test_pf_gather_last(lib, n, H):
    g = rng_for(f"gl{n}{H}")
    slots = g.permutation(lib.maxb)[:n].tolist()
    lens = g.integers(1, 40, n)
    x = rand_bits16(g, (int(lens.sum()), H))
    h_last = rand_bits16(g, (lib.maxb, H))
    before = host(h_last).numpy().copy()
    ok(lib.rows_shim_pf_gather_last(n, ints(lens), ints(slots), x.data_ptr(), h_last.data_ptr(), H, stream()), "gather_last")
    assert np.array_equal(host(h_last).numpy(), R.pf_gather_last(lens, slots, host(x).numpy(), before))
    STATS["exact"] += 1


@pytest.mark.parametrize("n", [1, 7, 32])
def test_release_state(lib, n):
    g = rng_for(f"rel{n}")
    st0 = random_state(g, lib.maxb)
    st0["finished"][:] = 0
    slots = g.permutation(lib.maxb)[:n].tolist()
    st0["finished"][slots[0]] = 1          # already finished: left as it is
    set_state(lib, st0)
    ok(lib.rows_shim_release(n, ints(slots), stream()), "release")
    got = get_state(lib)
    want = R.release(st0, slots)
    for f in FIELDS:
        assert np.array_equal(got[f], want[f]), f"DevState.{f}"
    assert got["n_valid"][slots[0]] == st0["n_valid"][slots[0]]
    STATS["exact"] += 1


@pytest.mark.parametrize("n", [1, 255, 257, 65536])
def test_bf16_to_f32(lib, n):
    g = rng_for(f"b2f{n}")
    src = np.arange(65536, dtype=np.int64).astype(np.uint16).view(np.int16)[:n] if n == 65536 else \
        g.integers(-32768, 32768, n).astype(np.int16)
    s = torch.from_numpy(src.copy()).cuda()
    out = torch.from_numpy(np.full(n + 100, SENT32, np.uint32).view(np.float32)).cuda()
    ok(lib.rows_shim_bf16_to_f32(s.data_ptr(), out.data_ptr(), n, stream()), "bf16_to_f32")
    got = host(out).numpy().view(np.uint32)
    assert np.array_equal(got[:n], src.view(np.uint16).astype(np.uint32) << 16) and (got[n:] == SENT32).all()
    STATS["exact"] += 1


# ================================================================================================ streaming encoder helpers
def test_load_wav(lib):
    g = rng_for("wav")
    B, n, factor, src_ld, dst_ld = 4, 3000, 960, 3100, 3300
    counts = [0, 1, 3, 2]                       # none, partial, full (3 * 960 < n: zeros after), partial
    src = g.standard_normal((B, src_ld)).astype(np.float32)
    dst0 = np.full((B, dst_ld), SENT32, np.uint32).view(np.float32)
    s, d = f32_dev(src), f32_dev(dst0)
    rp = rp_dev([5, 0, 9, 0], counts)
    ok(lib.rows_shim_load_wav(s.data_ptr(), src_ld, d.data_ptr(), dst_ld, n, rp.data_ptr(), B, factor, stream()), "load_wav")
    got = host(d).numpy()
    assert np.array_equal(got.view(np.uint32), R.load_wav(src, dst0, n, counts, factor).view(np.uint32))
    STATS["exact"] += 1


@pytest.mark.parametrize("C,hist", [(300, 2), (512, 5)])
def test_seed_replicate(lib, C, hist):
    g = rng_for(f"seed{C}{hist}")
    B, ld = 5, hist + 11
    pos, counts = [0, 0, 5, 0, 3], [3, 0, 2, 1, 0]     # only rows 0 and 3 are at position 0 with frames
    h0 = g.standard_normal((B, C, ld)).astype(np.float32)
    h = f32_dev(h0)
    rp = rp_dev(pos, counts)
    ok(lib.rows_shim_seed_replicate(h.data_ptr(), C, hist, ld, rp.data_ptr(), B, stream()), "seed_replicate")
    assert np.array_equal(host(h).numpy(), R.seed_replicate(h0, hist, pos, counts))
    STATS["exact"] += 1


def test_mask_codes(lib):
    g = rng_for("mask")
    B, nq, T, ds = 5, 16, 4, 2
    counts = [0, 1, 3, 7, 8]                  # ceil: 0, 1, 2, 4, 4 frames kept
    codes0 = g.integers(0, 2048, (B, nq, T)).astype(np.int32)
    cd = i32_dev(codes0)
    rp = rp_dev([0] * B, counts)
    ok(lib.rows_shim_mask_codes(cd.data_ptr(), nq, T, rp.data_ptr(), B, ds, stream()), "mask_codes")
    got = host(cd).numpy()
    assert np.array_equal(got, R.mask_codes(codes0, counts, ds))
    assert (got[2, :, :2] >= 0).all() and (got[2, :, 2:] == -1).all()   # count 3 keeps ceil(3 / 2) = 2 frames
    STATS["exact"] += 1


def test_enc_reset(lib):
    g = rng_for("encreset")
    B = 4
    flags = [1, 0, 2, 0]
    ents = [(int(g.integers(1, 70)), int(g.choice([8, 64, 300]))) for _ in range(5)]
    bufs, hs, Cs, lds = [], [], [], []
    for hist, Cc in ents:
        ld = hist + 13
        bufs.append(torch.from_numpy(g.standard_normal((B, Cc, ld)).astype(np.float32)).cuda())
        hs.append(hist); Cs.append(Cc); lds.append(ld)
    before = [host(b).numpy().copy() for b in bufs]
    rp = rp_dev([0] * B, flags)
    ok(lib.rows_shim_enc_reset(ptrs(bufs), ints(hs), ints([1] * len(bufs)), ints(Cs), ints(lds), len(bufs), rp.data_ptr(), B,
                               stream()), "enc_reset")
    for b, b0, hist in zip(bufs, before, hs):
        want = np.moveaxis(R.reset(np.moveaxis(b0, 2, 1), hist, flags), 1, 2)
        assert np.array_equal(host(b).numpy(), want)
    STATS["exact"] += 1
