"""Direct checks of the wgmma tap-GEMM (csrc/gemm_sm90.cu, tap_gemm_kernel<BN, ACT>) against a plain fp64 computation of
the same operation, call by call, at its tile, tap, view and epilogue edges.

The kernel is driven through tests/csrc/tap_gemm_shim.cu, a small C wrapper linked against the shipped
libqwen3tts_b200.so, so what runs is the binary the engines load.  The fp64 reference `ref_tap_gemm` is shared by the
CPU tests (it must reproduce the oracle's Conv1d / ConvTranspose1d / Linear / SwiGLU layers from the package's own
weight packers) and the GPU tests (the kernel must agree with it).

Acceptance rule for what the kernel writes (bf16):
- out_raw (before the activation): every element lies between the epilogue chain, with the kernel's rounding points,
  evaluated on float32 bounds of the accumulator: s - eps and s + eps, s the exact sum, eps = ntaps*Kp*2^-22*sum|a*w|.
  On the "grid" inputs (small integers times powers of two) every partial sum is exactly representable in fp32, so the
  accumulator is exact in any summation order and eps = 0: the check is then bit-exact.
- out_act next to out_raw: the activation of the kernel's own out_raw value, within one bf16 ulp.
- out_act alone: within one ulp of the activation of some bf16 value of the out_raw interval.
- every in-range element is written and finite, and every guard element around the outputs is untouched.
"""
import ctypes as C
import math
import os
import subprocess
from dataclasses import dataclass, replace

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM_SRC = os.path.join(ROOT, "tests", "csrc", "tap_gemm_shim.cu")

ACT_NONE, ACT_SNAKE, ACT_GELU, ACT_SWIGLU_PAIR, ACT_SWIGLU_BLK8 = 0, 1, 2, 3, 4
GATED = (ACT_SWIGLU_PAIR, ACT_SWIGLU_BLK8)
SENTINEL = 0x7FAB            # a bf16 NaN: outputs are filled with it before a launch
RESID_GUARD = 1.0e30         # residual elements outside the view: reading one makes the output fail loudly
A_GUARD = 1024.0             # A elements outside the [a_rows][K] view (row pitch gap, batch gap)
STATS = {"grid": 0.0, "normal": 0.0}   # largest fraction of out_raw elements whose two bounds differ, per input kind


def kpad(k):
    return (k + 63) // 64 * 64


# ================================================================================================ fp64 reference
def ref_tap_gemm(a, w, K, Kp, shifts, T, a_row0=0, a_rows=None):
    """C[b][m][n] = sum_tap sum_{k<K} A[b][a_row0 + m + shift_tap][k] * W[n][tap*Kp + k] in float64, reading zero for
    rows outside [0, a_rows) of the same batch.  a: [B][>= a_rows][>= K], w: [N][ntaps*Kp], any float dtype, any device.
    Returns (C, sum |a*w|), both [B][T][N] float64."""
    a_rows = a.shape[1] if a_rows is None else a_rows
    a = a[:, :a_rows, :K].double()
    B, N = a.shape[0], w.shape[0]
    out = torch.zeros(B, T, N, dtype=torch.float64, device=a.device)
    sab = torch.zeros_like(out)
    rows = torch.arange(T, device=a.device) + a_row0
    for tap, sh in enumerate(shifts):
        r = rows + sh
        ok = (r >= 0) & (r < a_rows)
        x = torch.zeros(B, T, K, dtype=torch.float64, device=a.device)
        x[:, ok] = a[:, r[ok]]
        wt = w[:, tap * Kp: tap * Kp + K].double().t()
        out += x @ wt
        sab += x.abs() @ wt.abs()
    return out, sab


def f32_bounds(s, eps):
    """float32 lo <= s - eps and hi >= s + eps (float64 in, float32 out)."""
    lo, hi = (s - eps).float(), (s + eps).float()
    lo = torch.where(lo.double() > s - eps, torch.nextafter(lo, torch.full_like(lo, -math.inf)), lo)
    hi = torch.where(hi.double() < s + eps, torch.nextafter(hi, torch.full_like(hi, math.inf)), hi)
    return lo, hi


def epilogue_chain(acc, bias=None, scale=None, resid=None):
    """The kernel's pre-activation chain on a float32 accumulator: bf16(acc + bias) -> bf16(x * scale) ->
    bf16(x + resid), every step a float32 operation rounded to bf16.  Returns float32 holding bf16 values."""
    x = acc + bias if bias is not None else acc
    x = x.bfloat16().float()
    if scale is not None:
        x = (x * scale).bfloat16().float()
    if resid is not None:
        x = (x + resid.float()).bfloat16().float()
    return x


def bf16_ulp(y):
    """Spacing of bf16 values at |y| (float64), subnormals included."""
    _, e = torch.frexp(y)
    e = torch.where(y == 0, torch.full_like(e, -126), torch.clamp(e - 1, min=-126))
    return torch.pow(2.0, (e - 7).double())


def bf16_key(x):
    """Order-preserving integer key of bf16 values (-0 and +0 share key 0)."""
    b = x.contiguous().view(torch.int16).to(torch.int32) & 0xFFFF
    return torch.where(b >= 0x8000, -(b & 0x7FFF), b)


def key_bf16(k):
    b = torch.where(k < 0, (-k) | 0x8000, k)
    return torch.where(b >= 0x8000, b - 0x10000, b).to(torch.int16).view(torch.bfloat16)


def bf16_between(lo, hi, n):
    """The first n bf16 values from lo up to hi (bf16 tensors, lo <= hi) along a new last axis, padded by repeating hi."""
    k = torch.minimum(bf16_key(lo)[..., None] + torch.arange(n, device=lo.device, dtype=torch.int32), bf16_key(hi)[..., None])
    return key_bf16(k).double()


def act_lipschitz(act, ea=None, ib=None):
    """Bound on |d act / dx|: SnakeBeta 1 + ib*ea, GELU 1.13."""
    return 1.0 + ib.double() * ea.double() if act == ACT_SNAKE else 1.13


def act_ref(x, act, ea=None, ib=None):
    """fp64 activation of bf16 values x and the distance from it a correct kernel may land: one bf16 ulp plus the
    float32 evaluation error, which matters only where the result nearly cancels.  SnakeBeta takes the kernel's float32
    product x*ea as the sine argument: at |x*ea| ~ 1e3 its rounding moves the argument by ~6e-5, which is the kernel's
    intended result, not its error; the reduced-range sine after that is good to 2^-21."""
    if act == ACT_SNAKE:
        arg = (x.float() * ea.float()).double()
        s = torch.sin(arg)
        y = x + ib.double() * s * s
        return y, bf16_ulp(y) + ib.double() * 2.0 ** -19 + x.abs() * 2.0 ** -22
    if act == ACT_GELU:
        y = 0.5 * x * (1.0 + torch.erf(x * 0.7071067811865476))
        return y, bf16_ulp(y) + x.abs() * 2.0 ** -22   # erff near -1: 2 ulp of 1.0
    raise ValueError(act)


SILU_ARGMIN = -1.2784645427610738


def swiglu_hull(glo, ghi, ulo, uhi):
    """Lowest and highest bf16(bf16(silu(g)) * u) over bf16 g in [glo, ghi] and u in [ulo, uhi] (float64 tensors).
    silu's extremes over the interval are at its ends or at its one minimum; the product's at the corners, and bf16
    rounding is monotone.  silu is evaluated in float32 with __expf (relative error below (4 + 1.5|g|) 2^-24; d has 4x
    margin), so its bf16 rounding may land on either neighbour; for g < -88.7 __expf overflows and silu comes out as
    -0, where the exact value is below 3e-37."""
    g = torch.stack([glo, ghi, torch.clamp(torch.full_like(glo, SILU_ARGMIN), glo, ghi)], -1)
    s = g * torch.sigmoid(g)
    d = (16.0 + 8.0 * g.abs()) * 2.0 ** -24
    slo, shi = torch.minimum(s * (1 - d), s * (1 + d)), torch.maximum(s * (1 - d), s * (1 + d))
    tiny = s.abs() < 2.0 ** -100
    slo, shi = torch.where(tiny, slo.clamp(max=0), slo), torch.where(tiny, shi.clamp(min=0), shi)
    rb = lambda v: v.float().bfloat16().double()  # noqa: E731
    slo, shi = rb(slo.amin(-1)), rb(shi.amax(-1))
    y = rb(torch.stack([slo * ulo, slo * uhi, shi * ulo, shi * uhi], -1))
    return y.amin(-1), y.amax(-1)


def gate_up_split(c, act):
    """Columns of a gated GEMM output [..., N] -> (gate, up) [..., N/2] in the order the kernel writes them."""
    if act == ACT_SWIGLU_PAIR:
        return c[..., 0::2], c[..., 1::2]
    v = c.reshape(*c.shape[:-1], c.shape[-1] // 16, 2, 8)
    return v[..., 0, :].flatten(-2), v[..., 1, :].flatten(-2)


# ================================================================================================ shim
@pytest.fixture(scope="session")
def shim(tmp_path_factory):
    """tests/csrc/tap_gemm_shim.cu compiled for sm_90a and linked against the freshly built library."""
    from qwen3_tts_b200 import _lib, build
    build.build()
    _lib.load()
    out = str(tmp_path_factory.mktemp("tap_gemm_shim") / "libtap_gemm_shim.so")
    cmd = [build._nvcc()] + build.NVCC_FLAGS + ["-shared", "-I", build.CSRC, SHIM_SRC, "-o", out, build.LIB_PATH,
                                                 "-Xlinker", "-rpath", "-Xlinker", build.LIB_DIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"shim build failed:\n{r.stdout}\n{r.stderr}"
    lib = C.CDLL(out)
    vp, i32, i64 = C.c_void_p, C.c_int, C.c_longlong
    lib.tap_gemm_shim_init.restype = i32
    lib.tap_gemm_shim_run.restype = i32
    lib.tap_gemm_shim_run.argtypes = [vp, i32, i32, i32, i64, i64, vp, i32, i32, i32, C.POINTER(i32), i32, vp, vp, vp, vp, vp,
                                      i32, i32, vp, vp, i32, i32, i64, i64, i64, vp]
    lib.path = out
    return lib


def last_error():
    from qwen3_tts_b200 import _lib
    return _lib.load().q3_last_error().decode()


def ptr(t, off=0):
    return None if t is None else t.data_ptr() + off


def shim_run(shim, a, B, T, K, lda, a_bs, w, N, Kp, shifts, bn, bias=None, scale=None, resid=None, ea=None, ib=None,
             cmod=None, act=ACT_NONE, out_raw=None, out_act=None, a_rows=0, a_row0=0, raw_bs=0, act_bs=0, resid_bs=0,
             ntaps=None):
    sh = (C.c_int * max(1, len(shifts)))(*shifts)
    return shim.tap_gemm_shim_run(a, B, T, K, lda, a_bs, w, N, Kp, len(shifts) if ntaps is None else ntaps, sh, bn, bias,
                                  scale, resid, ea, ib, N if cmod is None else cmod, act, out_raw, out_act, a_rows, a_row0,
                                  raw_bs, act_bs, resid_bs, C.c_void_p(torch.cuda.current_stream().cuda_stream))


# ================================================================================================ one checked launch
@dataclass(frozen=True)
class Case:
    T: int
    K: int
    N: int
    B: int = 1
    shifts: tuple = (0,)
    Kp: int = 0               # 0: kpad(K)
    bias: bool = True
    scale: bool = False
    resid: str = ""           # "" | "sep" (its own tensor) | "inplace" (the out_raw tensor)
    act: int = ACT_NONE
    raw: bool = True
    cmod: int = 0             # 0: N
    hist: int = 0             # history rows in front of the T rows of A (a_row0; a_rows = hist + T)
    pad: int = 0              # spare rows per batch in A and in every output / residual view
    lda_pad: int = 0          # A row pitch beyond K
    data: str = "grid"        # "grid": exact fp32 accumulation; "normal": random bf16
    big: float = 1.0          # gain on the gate rows (SwiGLU) or on exp(alpha) (SnakeBeta)


def make_inputs(c: Case, dev, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    nt = len(c.shifts)
    Kp = c.Kp or kpad(c.K)
    a_rows, lda = c.hist + c.T, c.K + c.lda_pad
    a_bs = (a_rows + c.pad) * lda
    if c.data == "grid":   # a = i/16, w = j/2^(4+e), |i|,|j| <= 15: products on a 2^-(8+e) grid
        e = max(0, math.ceil(math.log2(math.sqrt(nt * c.K))))
        av = torch.randint(-15, 16, (c.B, a_rows, c.K), generator=g).double() / 16
        wv = torch.randint(-15, 16, (c.N, nt, c.K), generator=g).double() / 2.0 ** (4 + e)
        q = 8 + e
    else:
        av = torch.randn(c.B, a_rows, c.K, generator=g).double()
        wv = torch.randn(c.N, nt, c.K, generator=g).double() / math.sqrt(nt * c.K)
        q = None
    if c.B > 1:   # large values at the end of every batch: a tap reading across the batch boundary shows
        av[:, -min(a_rows, 48):] *= 64
    if c.act in GATED and c.big != 1:
        gate_rows = torch.arange(c.N) % 2 == 0 if c.act == ACT_SWIGLU_PAIR else torch.arange(c.N) % 16 < 8
        wv[gate_rows] *= c.big
    A = torch.full((c.B * a_bs + lda,), A_GUARD, dtype=torch.bfloat16)
    A[:c.B * a_bs].view(c.B, a_rows + c.pad, lda)[:, :a_rows, :c.K] = av.bfloat16()
    W = torch.randn(c.N, nt, Kp, generator=g).bfloat16()   # columns K..Kp-1 meet A's zero fill: any value must do
    W[:, :, :c.K] = wv.bfloat16()
    cm = c.cmod or c.N
    inp = dict(A=A.to(dev), a_bs=a_bs, lda=lda, a_rows=a_rows, Kp=Kp, W=W.reshape(c.N, nt * Kp).to(dev), q=q, cmod=cm)
    inp["bias"] = (torch.randn(cm, generator=g) * 0.5).to(dev) if c.bias else None
    inp["scale"] = (torch.randn(cm, generator=g) * 0.3).to(dev) if c.scale else None   # LayerScale of both signs
    if c.act == ACT_SNAKE:
        inp["ea"] = (torch.exp(torch.rand(cm, generator=g) * 2 - 1) * c.big).to(dev)
        inp["ib"] = (1.0 / (torch.exp(torch.rand(cm, generator=g) * 2 - 1) + 1e-9)).to(dev)
    else:
        inp["ea"] = inp["ib"] = None
    inp["resid_vals"] = torch.randn(c.B, c.T, c.N, generator=g).bfloat16().to(dev) if c.resid else None
    return inp


def sentinel_buffer(elems, dev):
    return torch.full((elems,), SENTINEL, dtype=torch.int16, device=dev).view(torch.bfloat16)


def view_rows(buf, B, bs, T, width):
    """The [B][T][width] view of a flat per-batch buffer with batch stride bs (elements)."""
    return buf[:B * bs].view(B, bs)[:, :T * width].view(B, T, width)


def guard_untouched(buf, B, bs, T, width):
    bits = buf.view(torch.int16).clone()
    view_rows(bits.view(torch.bfloat16), B, bs, T, width).view(torch.int16).fill_(SENTINEL)   # mask the view
    return bool((bits == SENTINEL).all())


def launch_case(shim, c: Case, bn, inp, dev, A=None):
    """Allocate sentinel-filled outputs with guard rows, run the kernel once; returns the output buffers."""
    N, T, B = c.N, c.T, c.B
    Na = N // 2 if c.act in GATED else N
    raw_bs, act_bs = (T + c.pad) * N, (T + c.pad) * Na
    out = dict(raw_bs=raw_bs, act_bs=act_bs, Na=Na)
    raw = sentinel_buffer(B * raw_bs + 2 * N, dev) if (c.raw or c.resid == "inplace") else None
    act = sentinel_buffer(B * act_bs + 2 * Na, dev) if c.act != ACT_NONE else None
    resid, resid_bs = None, 0
    if c.resid == "sep":
        resid_bs = (T + c.pad) * N
        resid = torch.full((B * resid_bs + 2 * N,), RESID_GUARD, dtype=torch.bfloat16, device=dev)
        view_rows(resid, B, resid_bs, T, N).copy_(inp["resid_vals"])
    elif c.resid == "inplace":
        resid, resid_bs = raw, raw_bs
        view_rows(raw, B, raw_bs, T, N).copy_(inp["resid_vals"])
    rc = shim_run(shim, ptr(inp["A"] if A is None else A), B, T, c.K, inp["lda"], inp["a_bs"], ptr(inp["W"]), N, inp["Kp"],
                  c.shifts, bn, bias=ptr(inp["bias"]), scale=ptr(inp["scale"]), resid=ptr(resid), ea=ptr(inp["ea"]),
                  ib=ptr(inp["ib"]), cmod=inp["cmod"], act=c.act, out_raw=ptr(raw) if c.raw else None, out_act=ptr(act),
                  a_rows=inp["a_rows"], a_row0=c.hist, raw_bs=raw_bs if c.pad else 0, act_bs=act_bs if c.pad else 0,
                  resid_bs=resid_bs if c.pad else 0)
    assert rc == 0, last_error()
    torch.cuda.synchronize()
    out.update(raw=raw if c.raw else None, act=act)
    return out


def check_case(c: Case, inp, out, what=""):
    """Compare one launch's outputs with the fp64 reference; returns the fraction of out_raw elements whose bounds
    differ (0 when there is no out_raw)."""
    N, T, B, dev = c.N, c.T, c.B, inp["W"].device
    A3 = inp["A"][:B * inp["a_bs"]].view(B, inp["a_rows"] + c.pad, inp["lda"])
    s, sab = ref_tap_gemm(A3, inp["W"], c.K, inp["Kp"], c.shifts, T, a_row0=c.hist, a_rows=inp["a_rows"])
    eps = len(c.shifts) * inp["Kp"] * 2.0 ** -22 * sab
    if inp["q"] is not None:   # every partial sum on the 2^-q grid and below 2^24 of it: fp32 holds it exactly
        eps = torch.where(sab * 2.0 ** inp["q"] < 2.0 ** 24, torch.zeros_like(eps), eps)
    lo, hi = f32_bounds(s, eps)
    ch = torch.arange(N, device=dev) % inp["cmod"]
    bias = inp["bias"][ch] if inp["bias"] is not None else None
    scale = inp["scale"][ch] if inp["scale"] is not None else None
    rv = inp["resid_vals"]
    ca, cb = epilogue_chain(lo, bias, scale, rv), epilogue_chain(hi, bias, scale, rv)
    rlo, rhi = torch.minimum(ca, cb).double(), torch.maximum(ca, cb).double()   # the chain is monotone in acc
    wide = 0.0
    if c.raw:
        buf = out["raw"]
        got = view_rows(buf, B, out["raw_bs"], T, N).double()
        assert bool(torch.isfinite(got).all()), f"{what}: out_raw has non-finite or unwritten elements"
        assert guard_untouched(buf, B, out["raw_bs"], T, N), f"{what}: out_raw written outside its view"
        bad = (got < rlo) | (got > rhi)
        if bool(bad.any()):
            i = tuple(int(v) for v in bad.nonzero()[0])
            raise AssertionError(f"{what}: {int(bad.sum())} out_raw elements outside the reference interval; first "
                                 f"[b,m,n]={list(i)}: got {float(got[i])}, want [{float(rlo[i])}, {float(rhi[i])}] "
                                 f"(exact sum {float(s[i])})")
        wide = float((rlo != rhi).double().mean())
        STATS[c.data] = max(STATS[c.data], wide)
    if c.act == ACT_NONE:
        return wide
    Na, buf = out["Na"], out["act"]
    got = view_rows(buf, B, out["act_bs"], T, Na).double()
    assert bool(torch.isfinite(got).all()), f"{what}: out_act has non-finite or unwritten elements"
    assert guard_untouched(buf, B, out["act_bs"], T, Na), f"{what}: out_act written outside its view"
    if c.act in GATED:
        (glo, ulo), (ghi, uhi) = gate_up_split(rlo, c.act), gate_up_split(rhi, c.act)
        ylo, yhi = swiglu_hull(glo, ghi, ulo, uhi)
        bad = (got < ylo - bf16_ulp(ylo)) | (got > yhi + bf16_ulp(yhi))
        ref_desc = lambda i: f"[{float(ylo[i])}, {float(yhi[i])}]"  # noqa: E731
    else:
        ea = inp["ea"][ch][:, None] if inp["ea"] is not None else None
        ib = inp["ib"][ch][:, None] if inp["ib"] is not None else None
        if c.raw:   # the activation of the kernel's own out_raw value
            x = view_rows(out["raw"], B, out["raw_bs"], T, N).double()[..., None]
            y, tol = act_ref(x, c.act, ea, ib)
            bad = ~((got[..., None] - y).abs() <= tol).any(-1)
        else:   # every bf16 value of a narrow interval; a wide one (a nearly cancelling sum) by the slope bound
            nc = 16
            x = bf16_between(rlo.bfloat16(), rhi.bfloat16(), nc)
            y, tol = act_ref(x, c.act, ea, ib)
            ok = ((got[..., None] - y).abs() <= tol).any(-1)
            ends = torch.stack([rlo, rhi], -1)
            ye, tole = act_ref(ends, c.act, ea, ib)
            slope = act_lipschitz(c.act, ea, ib)
            ok_wide = ((got[..., None] - ye).abs() - tole).amin(-1) <= (slope * (rhi - rlo)[..., None] / 2).squeeze(-1)
            wide_iv = bf16_key(rhi.bfloat16()) - bf16_key(rlo.bfloat16()) >= nc
            bad = ~torch.where(wide_iv, ok_wide, ok)
        ref_desc = lambda i: f"{y[i].tolist()} (x {x[i].tolist()})"  # noqa: E731
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} out_act elements off the reference; first [b,m,n]={list(i)}: "
                             f"got {float(got[i])}, want {ref_desc(i)}")
    return wide


def run_case(shim, c: Case, bn, seed=0, what=""):
    dev = "cuda"
    inp = make_inputs(c, dev, seed)
    out = launch_case(shim, c, bn, inp, dev)
    return check_case(c, inp, out, what=f"{what} {c} bn={bn}")


# ================================================================================================ CPU tests
def test_shim_builds_and_links_against_the_shipped_library(shim):
    """The shim cross-compiles for sm_90a and calls the library's gemm_* symbols; it carries no copy of its own."""
    from qwen3_tts_b200 import build
    dyn = subprocess.run(["readelf", "-d", shim.path], capture_output=True, text=True).stdout
    assert os.path.basename(build.LIB_PATH) in dyn, dyn
    syms = subprocess.run(["nm", "-D", shim.path], capture_output=True, text=True).stdout.splitlines()
    defined = [ln.split()[-1] for ln in syms if len(ln.split()) == 3 and ln.split()[1] in "TtDdBbRr"]
    undefined = [ln.split()[-1] for ln in syms if len(ln.split()) == 2 and ln.split()[0] == "U"]
    assert {"tap_gemm_shim_init", "tap_gemm_shim_run"} <= set(defined)
    assert not [s for s in defined if "gemm_" in s.replace("tap_gemm_shim", "") or "q3_" in s], defined
    for s in ("gemm_init", "gemm_make_plan_v", "gemm_launch"):
        assert any(s in u for u in undefined), (s, undefined)


@pytest.mark.parametrize("k", [3, 7])
@pytest.mark.parametrize("dil", [1, 3, 9])
def test_conv_packer_and_reference_match_oracle_conv1d(k, dil):
    from oracle import codec as OC
    from qwen3_tts_b200.codec import CodecDecoder
    g = torch.Generator().manual_seed(k * 10 + dil)
    B, Ci, Co, T = 2, 40, 48, 57
    x, w, b = torch.randn(B, Ci, T, generator=g), torch.randn(Co, Ci, k, generator=g), torch.randn(Co, generator=g)
    W = CodecDecoder._conv_w(w)
    assert W.shape == (Co, k * kpad(Ci))
    got, _ = ref_tap_gemm(x.transpose(1, 2), W, Ci, kpad(Ci), [-(k - 1 - j) * dil for j in range(k)], T)
    want = OC.causal_conv1d(x.double(), w.double(), b.double(), dilation=dil).transpose(1, 2)
    torch.testing.assert_close(got + b.double(), want, rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("r", [2, 3, 5, 8])
@pytest.mark.parametrize("taps", [2, 1])
def test_conv_transpose_packer_and_reference_match_oracle(r, taps):
    """ConvTranspose1d(k=taps*r, stride r) as a GEMM over the input frames: shifts {0, -1}, N = r*Cout, channel n % Cout."""
    from oracle import codec as OC
    from qwen3_tts_b200.codec import CodecDecoder
    g = torch.Generator().manual_seed(r * 10 + taps)
    B, Ci, Co, T = 2, 72, 32, 19
    x, w, b = torch.randn(B, Ci, T, generator=g), torch.randn(Ci, Co, taps * r, generator=g), torch.randn(Co, generator=g)
    W = CodecDecoder._convT_w(w, r)
    assert W.shape == (r * Co, taps * kpad(Ci))
    got, _ = ref_tap_gemm(x.transpose(1, 2), W, Ci, kpad(Ci), [0, -1][:taps], T)
    got = got + b.double()[torch.arange(r * Co) % Co]
    want = OC.causal_conv_transpose1d(x.double(), w.double(), b.double(), r).transpose(1, 2)
    torch.testing.assert_close(got.reshape(B, T * r, Co), want, rtol=1e-10, atol=1e-10)


def test_linear_packer_and_reference_match_oracle_linear():
    from qwen3_tts_b200.codec import CodecDecoder
    g = torch.Generator().manual_seed(1)
    x, w = torch.randn(3, 21, 100, generator=g).double(), torch.randn(80, 100, generator=g)
    W = CodecDecoder._lin_w(w)
    assert W.shape == (80, 128) and bool((W[:, 100:] == 0).all())
    got, sab = ref_tap_gemm(x, W, 100, 128, [0], 21)
    torch.testing.assert_close(got, x @ w.double().t(), rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(sab, x.abs() @ w.double().abs().t(), rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("layout", ["pair", "blk8"])
def test_gate_up_packers_match_swiglu(layout):
    """The codec's PAIR and the talker's BLK8 gate/up interleaves, read back the way the kernel's gated epilogues read
    their columns, give silu(x gate^T) * (x up^T)."""
    from qwen3_tts_b200.codec import CodecDecoder
    from qwen3_tts_b200.engine import AREngine
    g = torch.Generator().manual_seed(2)
    I, K = 48, 72
    x = torch.randn(2, 11, K, generator=g).double()
    gate, up = torch.randn(I, K, generator=g).double(), torch.randn(I, K, generator=g).double()
    if layout == "pair":
        W, act = CodecDecoder._lin_w(CodecDecoder._gate_up_pair(gate, up)), ACT_SWIGLU_PAIR
    else:
        W, act = AREngine._gate_up_blk8(gate, up), ACT_SWIGLU_BLK8
    c, _ = ref_tap_gemm(x, W, K, W.shape[1], [0], 11)
    gg, uu = gate_up_split(c, act)
    want = torch.nn.functional.silu(x @ gate.t()) * (x @ up.t())
    torch.testing.assert_close(torch.nn.functional.silu(gg) * uu, want, rtol=1e-10, atol=1e-10)


def test_reference_helpers():
    """bf16 enumeration, ulp and directed float32 bounds behave at signs, zero and powers of two."""
    v = torch.tensor([-2.0, -1.0, -0.0, 0.0, 1.0, 1.0078125, 2.0], dtype=torch.bfloat16)
    assert bool((key_bf16(bf16_key(v)).float() == v.float()).all())
    assert bf16_key(v).tolist() == sorted(bf16_key(v).tolist())
    c = bf16_between(torch.tensor([-1.0], dtype=torch.bfloat16), torch.tensor([-0.9921875], dtype=torch.bfloat16), 4)
    assert c.tolist() == [[-1.0, -0.99609375, -0.9921875, -0.9921875]]
    lo, hi = swiglu_hull(*(torch.tensor([v], dtype=torch.float64) for v in (-3.0, 2.0, 1.0, 1.0)))
    assert float(lo) < -0.278 < float(hi) and abs(float(hi) - 1.7615942) < 0.01   # silu's minimum inside [-3, 2]
    assert bf16_ulp(torch.tensor([1.0, 1.99, 2.0, -0.75, 0.0], dtype=torch.float64)).tolist() == \
        [2 ** -7, 2 ** -7, 2 ** -6, 2 ** -8, 2 ** -133]
    s = torch.tensor([1.0 + 2 ** -30, -3.0], dtype=torch.float64)
    lo, hi = f32_bounds(s, torch.zeros_like(s))
    assert bool((lo.double() <= s).all() and (hi.double() >= s).all()) and float(hi[0] - lo[0]) == 2 ** -23


# ================================================================================================ GPU tests
@pytest.fixture(scope="module")
def gemm(shim):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    assert shim.tap_gemm_shim_init() == 0, last_error()
    yield shim
    print(f"\ntap-GEMM out_raw elements whose reference interval spans more than one bf16 value, largest fraction per "
          f"launch: grid inputs {STATS['grid']:.4f}, normal inputs {STATS['normal']:.4f}")


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


BNS = [64, 128]


@pytest.mark.gpu
@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("T", [1, 127, 128, 129, 300])
def test_tile_edges(gemm, bn, T):
    """Partial M and N tiles at both widths (N < bn included) and K < Kp, the last K block zero-filled by TMA."""
    for N in (16, 48, 64, 80, 144, 288):
        for K in (8, 40, 96, 192, 1000):
            run_case(gemm, Case(T=T, K=K, N=N), bn, seed=T + N + K)


@pytest.mark.gpu
@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("nkb", [1, 2, 5, 6, 7, 13, 112])
def test_ring_depth_and_persistent_walk(gemm, bn, nkb):
    """k-block counts that are and are not multiples of the 6-stage ring, on grids where CTAs walk 1, 2 and 4 tiles."""
    ntaps, K, Kp = {1: (1, 40, 64), 2: (1, 104, 128), 5: (1, 296, 320), 6: (3, 96, 128), 7: (7, 56, 64),
                    13: (1, 808, 832), 112: (7, 1000, 1024)}[nkb]
    assert ntaps * Kp // 64 == nkb
    sms = sm_count()
    for tiles in (1, sms - 1, sms, sms + 1, 3 * sms + 5):
        B = 2 if tiles % 2 == 0 else 1
        ntiles = 2
        mt = tiles // (B * ntiles) if tiles % (B * ntiles) == 0 else None
        if mt is None:
            B, ntiles, mt = 1, 1, tiles
        N = bn * ntiles - 16          # last N tile partial
        T = 128 * mt - 37 if mt > 1 else 91
        shifts = tuple(-(ntaps - 1 - j) for j in range(ntaps))
        c = Case(T=T, K=K, N=N, B=B, shifts=shifts, Kp=Kp)
        assert B * ntiles * ((T + 127) // 128) == tiles
        run_case(gemm, c, bn, seed=nkb * 1000 + tiles, what=f"tiles={tiles}")


@pytest.mark.gpu
@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("ntaps", [2, 3, 7])
@pytest.mark.parametrize("dil", [1, 3, 9])
def test_taps_batches_and_history_views(gemm, bn, ntaps, dil):
    """B = 3 with large values at the end of every batch, history prefixes that the taps reach into and past, padded
    batch strides with guard rows, a wider A pitch, and a forward-reaching tap that runs off the end of the rows."""
    shifts = tuple(-(ntaps - 1 - j) * dil for j in range(ntaps))
    for hist in (0, 2, 6, 54):
        c = Case(T=150, K=72, N=80, B=3, shifts=shifts, hist=hist, pad=5, lda_pad=8 if hist % 4 == 2 else 0,
                 scale=True, resid="sep", act=ACT_SNAKE)
        run_case(gemm, c, bn, seed=hist + ntaps * 7 + dil)
    run_case(gemm, Case(T=131, K=40, N=48, B=3, shifts=(-dil, 0, 2), hist=1), bn, seed=5)


def codec_sites(Cd=64, Cl=96, Hh=128, I=160, C=192, T=150):
    """Every tap-GEMM launch of codec_engine.cu (one-shot and streaming) with its epilogue, at small shapes."""
    Co = C // 2
    sites = {
        "rvq.proj": Case(T=T, K=Cd, N=Cd, bias=False),
        "pre_conv": Case(T=T, K=Cd, N=Cl, shifts=(-2, -1, 0)),
        "tr.in": Case(T=T, K=Cl, N=Hh),
        "tr.qkv": Case(T=T, K=Hh, N=3 * Hh, bias=False),
        "tr.o": Case(T=T, K=Hh, N=Hh, bias=False, scale=True, resid="sep"),
        "tr.gate_up": Case(T=T, K=Hh, N=2 * I, bias=False, act=ACT_SWIGLU_PAIR, raw=False),
        "tr.down": Case(T=T, K=I, N=Hh, bias=False, scale=True, resid="sep"),
        "tr.out": Case(T=T, K=Hh, N=Cl),
        "up.ct": Case(T=T, K=Cl, N=2 * Cl, cmod=Cl),
        "up.pw1": Case(T=T, K=Cl, N=4 * Cl, act=ACT_GELU, raw=False),
        "up.pw2": Case(T=T, K=4 * Cl, N=Cl, scale=True, resid="sep"),
        "dec.in": Case(T=T, K=Cl, N=C, shifts=tuple(range(-6, 1)), act=ACT_SNAKE, raw=False),
        "dec.c1": Case(T=T, K=Co, N=Co, shifts=tuple(-(6 - j) * 9 for j in range(7)), act=ACT_SNAKE, raw=False, big=128),
        "dec.c2": Case(T=T, K=Co, N=Co, resid="sep", act=ACT_SNAKE, big=128),
        "dec.c2.inplace": Case(T=T, K=Co, N=Co, resid="inplace", act=ACT_SNAKE, big=128),   # the residual stream in place
        # streaming: history-prefixed inputs and outputs inside larger per-row buffers
        "s.rvq.proj": Case(T=T, K=Cd, N=Cd, bias=False, pad=7),
        "s.pre_conv": Case(T=T, K=Cd, N=Cl, shifts=(-2, -1, 0), hist=2, pad=3),
        "s.up.ct": Case(T=T, K=Cl, N=2 * Cl, cmod=Cl, pad=6),
        "s.up.pw2": Case(T=T, K=4 * Cl, N=Cl, scale=True, resid="sep", pad=6),
        "s.dec.in": Case(T=T, K=Cl, N=C, shifts=tuple(range(-6, 1)), act=ACT_SNAKE, raw=False, hist=6, pad=1),
        "s.dec.c1": Case(T=T, K=Co, N=Co, shifts=tuple(-(6 - j) * 9 for j in range(7)), act=ACT_SNAKE, raw=False,
                         hist=54, pad=54, big=128),
        "s.dec.c2": Case(T=T, K=Co, N=Co, resid="sep", act=ACT_SNAKE, pad=9),
        "s.dec.c2.inplace": Case(T=T, K=Co, N=Co, resid="inplace", act=ACT_SNAKE, pad=9),
        # SwiGLU gates out to +-100 (exp overflow must give 0, not NaN), with a gate/up bias
        "gate_up.pair.big": Case(T=T, K=Hh, N=2 * I, act=ACT_SWIGLU_PAIR, raw=False, big=64),
        "gate_up.blk8.big": Case(T=T, K=Hh, N=2 * I, act=ACT_SWIGLU_BLK8, raw=False, big=64),
    }
    for r in (2, 3, 5, 8):   # ConvTranspose1d(2r, r) of a decoder block: cmod = Cout < N
        sites[f"dec.ct.r{r}"] = Case(T=T, K=C, N=r * Co, cmod=Co, shifts=(0, -1), act=ACT_SNAKE, big=128)
        sites[f"s.dec.ct.r{r}"] = Case(T=T, K=C, N=r * Co, cmod=Co, shifts=(0, -1), act=ACT_SNAKE, hist=1, pad=2)
    return sites


def prefill_sites(ntok, H, nh, nkv, hd, I):
    """The four launches of ar_engine.cu::prefill_rows; o and down update the residual stream in place."""
    return {
        "pf.qkv": Case(T=ntok, K=H, N=(nh + 2 * nkv) * hd, bias=False),
        "pf.o": Case(T=ntok, K=nh * hd, N=H, bias=False, resid="inplace"),
        "pf.gate_up": Case(T=ntok, K=H, N=2 * I, bias=False, act=ACT_SWIGLU_BLK8, raw=False),
        "pf.down": Case(T=ntok, K=I, N=H, bias=False, resid="inplace"),
    }


EPILOGUE_SITES = {**codec_sites(), **prefill_sites(200, 256, 4, 2, 64, 192),
                  "cp.proj": Case(T=300, K=256, N=128)}


@pytest.mark.gpu
@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("site", sorted(EPILOGUE_SITES))
def test_epilogues_of_every_call_site(gemm, bn, site):
    c = EPILOGUE_SITES[site]
    run_case(gemm, c, bn, seed=len(site), what=site)
    if c.data == "grid" and c.K >= 64:   # the same launch on unstructured data, under the eps interval
        run_case(gemm, replace(c, data="normal"), bn, seed=len(site) + 1, what=site)


def production_cases():
    from oracle import codec as OC
    from oracle import talker as OT
    cc = OC.CodecCfg()
    frames, B = 12, 2
    Tc = frames * math.prod(cc.upsampling_ratios) * math.prod(cc.upsample_rates[:-1])
    r = cc.upsample_rates[-1]
    Ci = cc.decoder_dim >> (len(cc.upsample_rates) - 1)
    Co = Ci // 2
    cases = {"codec.ct": Case(T=Tc, K=Ci, N=r * Co, B=B, cmod=Co, shifts=(0, -1), act=ACT_SNAKE),
             "codec.c1": Case(T=Tc * r, K=Co, N=Co, B=B, shifts=tuple(-(6 - j) * 9 for j in range(7)), act=ACT_SNAKE,
                              raw=False),
             "codec.c2": Case(T=Tc * r, K=Co, N=Co, B=B, resid="sep", act=ACT_SNAKE)}
    t = OT.cfg_1p7b()
    tk = t.talker
    for ntok in (9, 488):
        for k, v in prefill_sites(ntok, tk.hidden_size, tk.num_heads, tk.num_kv_heads, tk.head_dim,
                                  tk.intermediate_size).items():
            cases[f"{k}.{ntok}"] = v
    cases["cp.proj_table"] = Case(T=(t.num_code_groups - 1) * t.cp.vocab_size, K=tk.hidden_size, N=t.cp.hidden_size)
    return cases


PRODUCTION = production_cases()


@pytest.mark.gpu
@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("name", sorted(PRODUCTION))
@pytest.mark.parametrize("data", ["grid", "normal"])
def test_production_shapes(gemm, bn, name, data):
    c = replace(PRODUCTION[name], data=data)
    wide = run_case(gemm, c, bn, seed=len(name), what=name)
    if c.raw:
        print(f"{name} bn={bn} {data}: out_raw interval spans >1 bf16 value in {wide:.4f} of elements")


def raw_bits(out):
    return [None if t is None else t.view(torch.int16).clone() for t in (out["raw"], out["act"])]


def same_bits(x, y):
    return all((a is None and b is None) or torch.equal(a, b) for a, b in zip(x, y))


INVARIANT_CASES = {
    "conv7.snake.B3": Case(T=300, K=96, N=96, B=3, shifts=tuple(range(-6, 1)), act=ACT_SNAKE, resid="sep", pad=3,
                           data="normal"),
    "convT.r5": Case(T=257, K=192, N=480, B=3, cmod=96, shifts=(0, -1), act=ACT_SNAKE, data="normal"),
    "linear.scale_resid": Case(T=200, K=1000, N=144, B=3, scale=True, resid="sep", data="normal"),
    "blk8": Case(T=129, K=256, N=320, B=3, act=ACT_SWIGLU_BLK8, raw=False, data="normal"),
    "pair": Case(T=129, K=256, N=320, B=3, act=ACT_SWIGLU_PAIR, raw=False, data="normal"),
    "gelu": Case(T=129, K=2048, N=384, B=3, act=ACT_GELU, raw=False, data="normal"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(INVARIANT_CASES))
def test_bit_invariants(gemm, name):
    """Each output element's k order does not depend on the tile width, the batch count or the launch: bn = 64 equals
    bn = 128, a B = 3 launch equals three B = 1 launches, and a repeated launch is identical, all bit for bit."""
    c = INVARIANT_CASES[name]
    inp = make_inputs(c, "cuda", seed=11)
    res = {bn: raw_bits(launch_case(gemm, c, bn, inp, "cuda")) for bn in BNS}
    assert same_bits(res[64], res[128]), f"{name}: bn=64 and bn=128 outputs differ"
    assert same_bits(res[64], raw_bits(launch_case(gemm, c, 64, inp, "cuda"))), f"{name}: repeated launch differs"
    one = replace(c, B=1)
    for bn in BNS:
        full = launch_case(gemm, c, bn, inp, "cuda")
        for b in range(c.B):
            inp1 = dict(inp, resid_vals=inp["resid_vals"][b:b + 1] if inp["resid_vals"] is not None else None)
            part = launch_case(gemm, one, bn, inp1, "cuda", A=inp["A"][b * inp["a_bs"]:])
            for key, bs, w in (("raw", full["raw_bs"], c.N), ("act", full["act_bs"], full["Na"])):
                if full[key] is not None:
                    x = view_rows(full[key], c.B, bs, c.T, w)[b].view(torch.int16)
                    y = view_rows(part[key], 1, bs, c.T, w)[0].view(torch.int16)
                    assert torch.equal(x, y), f"{name}: batch {b} of a B={c.B} launch differs from a B=1 launch (bn={bn})"
    check_case(c, inp, full, what=name)


@pytest.mark.gpu
def test_host_side_rejections_launch_nothing(gemm):
    """Each argument check of gemm_make_plan_v / gemm_launch returns non-zero with a message, and writes nothing."""
    dev = "cuda"
    T, K, N = 64, 64, 64
    a = torch.randn(T, K + 8, device=dev).bfloat16()
    w = torch.randn(N, 9 * 64, device=dev).bfloat16()
    f = torch.randn(2 * N + 8, device=dev)
    out = sentinel_buffer(T * N, dev)
    half = sentinel_buffer(T * N // 2, dev)
    base = dict(a=ptr(a), B=1, T=T, K=K, lda=K, a_bs=T * K, w=ptr(w), N=N, Kp=64, shifts=(0,), bn=64, out_raw=ptr(out))
    bad = {
        "bn=96": dict(bn=96),
        "bn=0": dict(bn=0),
        "N % 16": dict(N=40),
        "Kp < K": dict(K=100, Kp=64),
        "Kp % 64": dict(K=80, Kp=96),
        "ntaps=0": dict(shifts=(), ntaps=0),
        "ntaps=9": dict(shifts=(0,) * 9),
        "bias off by 4 B": dict(bias=ptr(f, 4)),
        "cmod % 16": dict(bias=ptr(f), cmod=40),
        "swiglu + resid": dict(act=ACT_SWIGLU_PAIR, out_raw=None, out_act=ptr(half), resid=ptr(out)),
        "swiglu + out_raw": dict(act=ACT_SWIGLU_BLK8, out_act=ptr(half)),
        "swiglu + scale": dict(act=ACT_SWIGLU_PAIR, out_raw=None, out_act=ptr(half), scale=ptr(f)),
        "A pitch": dict(lda=K + 4, a_bs=T * (K + 4)),
        "activation 7": dict(act=7, out_act=ptr(half)),
    }
    for name, kw in bad.items():
        args = dict(base, **kw)
        if "ntaps" not in args:
            args["ntaps"] = None
        rc = shim_run(gemm, args.pop("a"), args.pop("B"), args.pop("T"), args.pop("K"), args.pop("lda"), args.pop("a_bs"),
                      args.pop("w"), args.pop("N"), args.pop("Kp"), args.pop("shifts"), args.pop("bn"), **args)
        torch.cuda.synchronize()
        assert rc != 0, f"{name}: accepted"
        assert last_error(), f"{name}: no error message"
        assert bool((out.view(torch.int16) == SENTINEL).all() and (half.view(torch.int16) == SENTINEL).all()), \
            f"{name}: rejected, but something was written"
    # and the base call itself is valid
    assert shim_run(gemm, base["a"], 1, T, K, K, T * K, base["w"], N, 64, (0,), 64, out_raw=ptr(out)) == 0, last_error()
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out.float()).all())

