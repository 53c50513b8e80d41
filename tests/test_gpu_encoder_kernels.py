"""Direct checks of the fp32 encoder kernels against an fp64 reference (tests/encoder_ref.py), call by call, at their
tile, padding, view, window and tie edges:
- conv_f32 (csrc/conv_f32.cu), the one Conv1d / Linear kernel of the codec and speaker encoders, through the library's
  own conv_f32_launch;
- the codec encoder's layernorm_ct, rope_ct, swa_ct<64>, rvq_encode and enc_roll (csrc/codec_encoder_kernels.cuh);
- the speaker encoder's melspec, mean_t, se_apply, copy_ch, asp_cat and asp_pool (csrc/speaker_kernels.cuh).
They run through tests/csrc/encoder_shim.cu, linked against the freshly built libqwen3tts_b200.so for the convolution and
compiling the header kernels from the shipped source under the library's flags, each with its engine's launch geometry.

Acceptance rules.
- Grid cases are checked bit for bit.  conv_f32: inputs are small integers x 2^-4 (distinct along every input row, so a
  wrong padding index or a shifted tap changes a value), weights small integers x 2^-4, power-of-two scales, act_in
  NONE and act_out NONE / RELU: every partial sum is a multiple of 2^-8 below 2^16, exact in fp32 in any order, so the
  output must equal the fp64 reference exactly.  Each grid case asserts that removing any single (ci, j) term changes
  some output.  swa_ct: zero queries (every p = __expf(0) = 1) and sparse integer V, so the output must be exactly
  fp32(acc * fp32(1 / l)); each case asserts that dropping any key changes a bit.  rvq_encode: integer centroids and
  residuals with E2 passed exactly, so every distance is exact and the code must be the exact argmin with the lowest
  index winning every tie, ties planted across one thread's slots and passes, lanes, warps and a higher warp holding a
  lower index.  mean_t, se_apply and copy_ch: grid inputs, bit-exact.
- General cases (random fp32) are held to per-element bounds derived from the kernels' fp32 evaluation (encoder_ref):
  conv: FMA chain (Cin k + 1) 2^-24 sum|w X|, the input activation's error (expm1f 1 ulp, tanhf 2 ulp, CUDA C
  Programming Guide, default flags) weighted by |w|, the output activation's Lipschitz constant (GELU 1.13, sigmoid
  0.25) times that plus its own error (erff / expf 2 ulp, IEEE division), and the scale / residual roundings; each case
  asserts that dropping any single tap moves some element by more than twice the bound.  layernorm: two-pass fp32
  mean / variance, rsqrtf 2 ulp and the affine step.  swa: attention_ref.online_bound's construction for an fp32
  output, with the drop-one-key sensitivity asserted.  rope: 2 2^-24 (|x1 c| + |x2 s|) (nvcc may contract either
  product into an FMA), V copies exact.  rvq: the kernel's codes replayed level by level (r -= e reproduced in numpy
  float32); each pick lies within the fp32 distance bound of the fp64 minimum, so it is the fp64 argmin wherever the
  gap exceeds the bound.  melspec: the two n_fft-term FMA chains through sqrt, the mel sum and log; a zero filterbank
  row gives exactly logf(1e-5f).  asp_cat / asp_pool: fp32 weighted sums, expf and the clamped sqrt.
- Invariants the streaming encoder relies on (DESIGN.md §4.4), bit for bit on random inputs: a conv computed one-shot,
  through a history-prefixed view and split in two segments agree; a LayerNorm column does not depend on T, its
  offset or the row pitch; rope + swa + enc_roll streamed in segments (one shorter than the history, one row reset, a
  ragged row) equal the one-shot, and so do the rolled history columns.
- Guards: outputs are pre-filled with a NaN sentinel, and every element outside a launch's view stays bit-unchanged;
  input channels and columns outside the view hold NaN / 1e30, so reading one shows.  No NaN reaches a checked output.
- Limit: the largest conv tile that fits 96 KB runs; one that needs more is refused with an error naming the shared
  memory, and nothing is launched.
STATS collects the near-boundary counts, the smallest sensitivity and the case counts, printed at the end.
"""
import ctypes as C
import math
import os
import subprocess
import zlib
from dataclasses import dataclass, replace

import numpy as np
import pytest
import torch

from tests import attention_ref as A
from tests import encoder_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM_SRC = os.path.join(ROOT, "tests", "csrc", "encoder_shim.cu")
SENT_BITS = np.uint32(0x7FC00ABC)   # NaN with a payload: outputs before a launch, and guard elements
COL_GUARD = np.float32(1e30)        # input columns past the view
STATS = {"grid": 0, "general": 0, "min_sensitivity": math.inf, "rvq_near_boundary": 0, "rvq_ties": 0,
         "mel_zero_row": 0, "padding_only_taps": 0}
pytestmark = pytest.mark.gpu


# ================================================================================================ shim
@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    """tests/csrc/encoder_shim.cu compiled for sm_90a and linked against the freshly built library."""
    from qwen3_tts_b200 import _lib, build
    build.build()
    _lib.load()
    out = str(tmp_path_factory.mktemp("encoder_shim") / "libencoder_shim.so")
    cmd = [build._nvcc()] + build.NVCC_FLAGS + ["-shared", "-I", build.CSRC, SHIM_SRC, "-o", out, build.LIB_PATH,
                                                 "-Xlinker", "-rpath", "-Xlinker", build.LIB_DIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"shim build failed:\n{r.stdout}\n{r.stderr}"
    L = C.CDLL(out)
    vp, i32, f32, i64 = C.c_void_p, C.c_int, C.c_float, C.c_longlong
    pp, pi = C.POINTER(C.c_void_p), C.POINTER(C.c_int)
    sig = {
        "enc_shim_init": [],
        "enc_shim_conv": [vp] * 7 + [i32] * 20 + [vp],
        "enc_shim_layernorm": [vp, i32, vp, vp, vp, i32, i32, i32, f32, i32, vp],
        "enc_shim_rope": [vp, vp, vp, i32, i32, i32, i32, vp, i32, vp, i64, i32, vp],
        "enc_shim_swa": [vp, vp, i64, i32, i32, vp, i32, i32, i32, i32, i32, f32, vp, i32, vp],
        "enc_shim_rvq": [vp, vp, pp, pp, pp, vp, i32, i32, i32, i32, i32, i32, vp],
        "enc_shim_roll": [pp, pi, pi, pi, pi, i32, vp, i32, vp],
        "enc_shim_melspec": [vp, i32, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp],
        "enc_shim_mean_t": [vp, i32, i32, i32, i32, vp, i32, vp],
        "enc_shim_se_apply": [vp, vp, vp, i32, i32, vp, i32, i32, i32, i32, i32, vp],
        "enc_shim_copy_ch": [vp, i32, i32, vp, i32, i32, i32, i32, i32, vp],
        "enc_shim_asp_cat": [vp, vp, i32, i32, f32, i32, vp],
        "enc_shim_asp_pool": [vp, vp, vp, i32, i32, f32, i32, vp],
    }
    for name, args in sig.items():
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = args
    L.path = out
    assert L.enc_shim_init() == 0, last_error()
    yield L
    print("\nencoder kernel STATS:", STATS)


def last_error():
    from qwen3_tts_b200 import _lib
    return _lib.load().q3_last_error().decode()


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def dev(a, dtype=np.float32):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype))).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def ptr(t, off=0):
    """Device pointer of tensor t, `off` elements in (None for None).  The caller holds t until the launch has run: a
    temporary freed while the arguments are evaluated may hand its memory to the next argument's tensor."""
    return None if t is None else t.data_ptr() + off * t.element_size()


def sentinel(shape):
    return np.full(shape, SENT_BITS, np.uint32).view(np.float32)


def bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


def rng_for(name):
    return np.random.default_rng(zlib.crc32(name.encode()))


def ok(rc, what):
    assert rc == 0, f"{what}: launch failed ({rc}) {last_error() if rc == 1 else ''}"


def check_sensitivity(what, sens):
    STATS["min_sensitivity"] = min(STATS["min_sensitivity"], sens)
    assert sens > 1.0, f"{what}: dropping a term moves no output element by more than twice the bound ({sens:.3f})"


def check_untouched(what, got, before, region):
    """Every element of `got` outside the boolean `region` is bit-identical to `before`."""
    bad = (bits(got) != bits(before)) & ~region
    assert not bad.any(), f"{what}: {int(bad.sum())} elements outside the view written, first at {np.argwhere(bad)[0]}"


# ================================================================================================ conv_f32
@dataclass(frozen=True)
class Conv:
    name: str
    Cin: int
    Cout: int
    Tout: int
    k: int
    stride: int = 1
    dil: int = 1
    B: int = 1
    pad: str = "zero"          # "zero" / "replicate" (causal, right extra padding) or "reflect" ("same", stride 1)
    Tin: int = 0               # causal: (Tout - 1) * stride < Tin <= Tout * stride (0: Tout * stride); reflect: Tout
    act_in: int = R.IN_NONE
    act_out: int = R.OUT_NONE
    bias: bool = True
    scale: bool = False
    res: str = ""              # "" / "sep" (own tensor) / "alias" (res is y, the in-place h += ls * o)
    x2: bool = False
    x_off: int = 0
    y_off: int = 0
    xT_pad: int = 0            # xT = Tin + xT_pad
    yT_pad: int = 0            # yT = Tout + yT_pad

    @property
    def keff(self):
        return (self.k - 1) * self.dil + 1

    @property
    def pad_left(self):
        return self.dil * (self.k - 1) // 2 if self.pad == "reflect" else self.keff - self.stride

    @property
    def tin(self):
        if self.pad == "reflect":
            return self.Tout
        return self.Tin or self.Tout * self.stride

    @property
    def padmode(self):
        return {"zero": R.PAD_ZERO, "replicate": R.PAD_REPLICATE, "reflect": R.PAD_REFLECT}[self.pad]


def grid_vals(shape, seed):
    """Small integers x 2^-4, distinct along the last axis (for rows up to 211 long) and never zero."""
    B, Cn, T = shape
    v = (np.arange(T)[None, None, :] * 37 + np.arange(Cn)[None, :, None] * 11 + np.arange(B)[:, None, None] * 5 + seed) % 211
    v = v - 105
    v[v == 0] = 106
    return (v / 16.0).astype(np.float32)


def conv_inputs(c: Conv, kind, g):
    B, Tin, Tout = c.B, c.tin, c.Tout
    xC, xT, yC, yT = c.x_off + c.Cin + 2, Tin + c.xT_pad, c.y_off + c.Cout + 1, Tout + c.yT_pad
    if kind == "grid":
        x = grid_vals((B, c.Cin, Tin), 3)
        w = (g.integers(1, 5, (c.Cout, c.Cin, c.k)) * g.choice([-1, 1], (c.Cout, c.Cin, c.k)) / 16.0).astype(np.float32)
        bias = (g.integers(-64, 65, c.Cout) / 256.0).astype(np.float32)
        scale = (2.0 ** g.integers(-1, 2, c.Cout) * g.choice([-1, 1], c.Cout)).astype(np.float32)
        res = grid_vals((B, c.Cout, Tout), 7)
        x2 = grid_vals((B, c.Cin, Tin), 9) if c.x2 else None
    else:
        # magnitudes kept away from zero, so that every single term is visible above the bound; GELU cases biased
        # into its steep half
        away = lambda *sh: (g.uniform(0.5, 1.5, sh) * g.choice([-1, 1], sh)).astype(np.float32)  # noqa: E731
        x = away(B, c.Cin, Tin)
        w = (away(c.Cout, c.Cin, c.k) / math.sqrt(c.Cin * c.k)).astype(np.float32)
        bias = (g.standard_normal(c.Cout) * 0.3 + (2.0 if c.act_out == R.OUT_GELU else 0.0)).astype(np.float32)
        scale = (g.standard_normal(c.Cout) * 0.2).astype(np.float32)
        res = g.standard_normal((B, c.Cout, Tout)).astype(np.float32)
        x2 = g.standard_normal((B, c.Cin, Tin)).astype(np.float32) if c.x2 else None
    # input buffers: the view's channels / columns hold the data; channels outside it NaN, columns past Tin 1e30
    xb = np.full((B, xC, xT), np.nan, np.float32)
    xb[:, c.x_off:c.x_off + c.Cin, :] = COL_GUARD
    xb[:, c.x_off:c.x_off + c.Cin, :Tin] = x
    x2b = None
    if c.x2:
        x2b = np.full((B, xC, xT), np.nan, np.float32)
        x2b[:, 1:1 + c.Cin, :] = COL_GUARD
        x2b[:, 1:1 + c.Cin, :Tin] = x2
    yb = sentinel((B, yC, yT))
    resb = None
    if c.res == "alias":
        yb[:, c.y_off:c.y_off + c.Cout, :Tout] = res
    elif c.res == "sep":
        resb = np.full((B, yC, yT), COL_GUARD, np.float32)
        resb[:, c.y_off:c.y_off + c.Cout, :Tout] = res
    return dict(x=x, xb=xb, x2=x2, x2b=x2b, w=w, bias=bias if c.bias else None, scale=scale if c.scale else None,
                res=res if c.res else None, resb=resb, yb=yb, xC=xC, xT=xT, yC=yC, yT=yT)


def conv_run(lib, c: Conv, I, xb=None, pad_left=None, Tin=None, xT=None):
    """One conv_f32_launch on device copies of the buffers; returns (rc, y buffer after the launch)."""
    d = {k: (dev(I[k]) if I[k] is not None else None) for k in ("xb", "x2b", "w", "bias", "scale", "resb", "yb")}
    if xb is not None:
        d["xb"] = dev(xb)
    res = d["yb"] if c.res == "alias" else d["resb"]
    rc = lib.enc_shim_conv(ptr(d["xb"]), ptr(d["x2b"]), ptr(d["w"]), ptr(d["bias"]), ptr(d["scale"]), ptr(res), ptr(d["yb"]),
                           I["xC"], c.x_off, I["xC"], 1, I["yC"], c.y_off, c.Cin, c.Cout, c.tin if Tin is None else Tin,
                           c.Tout, c.k, c.stride, c.dil, c.pad_left if pad_left is None else pad_left, c.padmode, c.act_in,
                           c.act_out, c.B, I["xT"] if xT is None else xT, I["yT"], stream())
    return rc, host(d["yb"])


def conv_ref(c: Conv, I):
    return R.ref_conv(I["x"], I["w"], c.Cin, c.Cout, c.tin, c.Tout, c.k, c.stride, c.dil, c.pad_left, c.padmode, c.act_in,
                      c.act_out, I["bias"], I["scale"], I["res"], x2=I["x2"])


def check_conv(lib, c: Conv, kind, assert_sensitivity=True):
    what = f"conv {c.name} [{kind}]"
    I = conv_inputs(c, kind, rng_for(what))
    rc, yb = conv_run(lib, c, I)
    ok(rc, what)
    region = np.zeros(yb.shape, bool)
    region[:, c.y_off:c.y_off + c.Cout, :c.Tout] = True
    check_untouched(what, yb, I["yb"], region)
    y = yb[:, c.y_off:c.y_off + c.Cout, :c.Tout]
    assert np.isfinite(y).all(), f"{what}: non-finite output"
    r = conv_ref(c, I)
    if kind == "grid":
        assert r["sab"].max() < 2.0 ** 16, f"{what}: grid sums not exact in fp32"
        want = r["y"].astype(np.float32)
        assert np.array_equal(want.astype(np.float64), r["y"]), f"{what}: grid reference not representable"
        bad = bits(y) != bits(want)
        assert not bad.any(), (f"{what}: {int(bad.sum())} elements differ, first at {np.argwhere(bad)[0]}: "
                               f"{y[tuple(np.argwhere(bad)[0])]} vs {want[tuple(np.argwhere(bad)[0])]}")
        # every tap (ci, j) that reads a real input column somewhere must change some output when removed
        reads = np.abs(r["X"]).max(axis=(0, 2)) > 0                     # [Cin][k]
        STATS["padding_only_taps"] += int((~reads).sum())
        sens = R.conv_drop_sensitivity(r, I["w"], np.full(r["y"].shape, 2.0 ** -12), R.OUT_NONE, I["scale"])
        check_sensitivity(what, sens)
        STATS["grid"] += 1
    else:
        bound = R.conv_bound(r, c.Cin, c.k, c.act_in, c.act_out, I["bias"], I["scale"], I["res"], c.x2)
        err = np.abs(y - r["y"])
        bad = err > bound
        assert not bad.any(), (f"{what}: {int(bad.sum())} elements outside the bound, worst ratio "
                               f"{float((err / bound).max()):.3f} at {np.unravel_index(np.argmax(err / bound), err.shape)}")
        sens = R.conv_drop_sensitivity(r, I["w"], bound, c.act_out, I["scale"])
        if assert_sensitivity:
            check_sensitivity(what, sens)
        else:
            STATS["min_sensitivity_real_general"] = min(STATS.get("min_sensitivity_real_general", math.inf), sens)
        STATS["general"] += 1


def sweep_cases():
    """Every value of each axis at least once, combined so that tile edges meet padding, stride and dilation."""
    couts, touts, cins = (1, 63, 64, 65, 130), (1, 63, 64, 65, 200), (1, 7, 8, 9, 24)
    ks, strides, dils, bs = (1, 2, 3, 7, 16), (1, 2, 4, 8), (1, 2, 4), (1, 3)
    out = []
    for i in range(25):
        k, s, d = ks[i % 5], strides[(i // 5 + i) % 4], dils[(i * 2) % 3]
        pad = ("zero", "replicate", "reflect")[i % 3]
        if pad == "reflect":
            s = 1
        elif (k - 1) * d + 1 < s:
            k = s                                                          # the causal convs have k_eff >= stride
        Tout = touts[(i * 3) % 5]
        c = Conv(f"sweep{i}", cins[(i + i // 5) % 5], couts[(i * 7) % 5], Tout, k, s, d, bs[i % 2], pad,
                 x_off=i % 3, y_off=(i * 5) % 3, xT_pad=(i % 4) * 3, yT_pad=(i % 3) * 5,
                 scale=i % 2 == 0, res=("", "sep", "alias")[i % 3], x2=i % 5 == 1)
        if pad == "reflect":
            need = max(c.pad_left, d * (k - 1) - c.pad_left) + 1           # smallest legal length: pad + 1
            c = replace(c, Tout=max(Tout, need))
        elif s > 1 and i % 2:
            c = replace(c, Tin=(c.Tout - 1) * s + 1)                       # right extra padding of stride - 1 columns
        out.append(c)
    out.append(Conv("reflect_min_T", 9, 65, 5, 3, 1, 4, 3, "reflect"))         # T = dil * (k - 1) / 2 + 1
    out.append(Conv("reflect_min_T_k16", 8, 64, 16, 16, 1, 1, 1, "reflect"))
    out.append(Conv("causal_dil_stride", 24, 130, 65, 7, 4, 2, 3, "replicate", x2=True, res="alias", scale=True))
    out.append(Conv("k16_s8_d4", 9, 63, 64, 16, 8, 4, 1, "zero", Tin=64 * 8 - 7))
    return out


def real_layers():
    """Every distinct conv shape of the default EncoderConfig and SpeakerEncoderConfig, with its own epilogue."""
    from qwen3_tts_b200.config import EncoderConfig, SpeakerEncoderConfig
    g, out = EncoderConfig(), []
    c, T = g.num_filters, 64 * 8
    out.append(Conv("enc.conv0", 1, c, T, g.kernel_size))
    for i, r in enumerate(g.ratios):
        out.append(Conv(f"enc.res{i}.a", c, c // g.compress, T, g.residual_kernel_size, act_in=R.IN_ELU))
        out.append(Conv(f"enc.res{i}.b", c // g.compress, c, T, 1, act_in=R.IN_ELU, res="sep"))
        T = T // r if T >= r * 8 else 8
        out.append(Conv(f"enc.down{i}", c, 2 * c, T, 2 * r, r, act_in=R.IN_ELU))
        c *= 2
    H, T = g.hidden_size, 67
    out.append(Conv("enc.conv_last", c, H, T, g.last_kernel_size, act_in=R.IN_ELU))
    out.append(Conv("tr.qkv", H, 3 * H, T, 1, bias=False))
    out.append(Conv("tr.o", H, H, T, 1, bias=False, scale=True, res="alias"))
    out.append(Conv("tr.fc1", H, g.intermediate_size, T, 1, bias=False, act_out=R.OUT_GELU))
    out.append(Conv("tr.fc2", g.intermediate_size, H, T, 1, bias=False, scale=True, res="alias"))
    out.append(Conv("down", H, H, 34, 2 * g.downsample_stride, g.downsample_stride, pad="replicate", bias=False))
    out.append(Conv("rvq.proj", H, g.codebook_dim, 34, 1, bias=False))
    s = SpeakerEncoderConfig()
    ch, L = s.enc_channels, 70
    out.append(Conv("spk.blocks.0", s.mel_dim, ch[0], L, s.enc_kernel_sizes[0], dil=s.enc_dilations[0], pad="reflect",
                    act_out=R.OUT_RELU))
    Cs = ch[1] // s.enc_res2net_scale
    out.append(Conv("spk.tdnn1", ch[0], ch[1], L, 1, pad="reflect", act_out=R.OUT_RELU, y_off=0))
    for i in range(1, len(ch) - 1):
        out.append(Conv(f"spk.res2net{i}", Cs, Cs, L, s.enc_kernel_sizes[i], dil=s.enc_dilations[i], pad="reflect",
                        act_out=R.OUT_RELU, x2=True, x_off=Cs, y_off=2 * Cs))
    out.append(Conv("spk.se1", ch[1], s.enc_se_channels, 1, 1, pad="reflect", act_out=R.OUT_RELU))
    out.append(Conv("spk.se2", s.enc_se_channels, ch[1], 1, 1, pad="reflect", act_out=R.OUT_SIGMOID))
    out.append(Conv("spk.mfa", ch[-1], ch[-1], L, s.enc_kernel_sizes[-1], pad="reflect", act_out=R.OUT_RELU))
    out.append(Conv("spk.asp.tdnn", 3 * ch[-1], s.enc_attention_channels, 40, 1, pad="reflect", act_out=R.OUT_RELU))
    out.append(Conv("spk.asp.conv", s.enc_attention_channels, ch[-1], 40, 1, pad="reflect", act_in=R.IN_TANH))
    out.append(Conv("spk.fc", 2 * ch[-1], s.enc_dim, 1, 1, pad="reflect"))
    return out


def grid_form(c: Conv):
    """The case with its activations stripped to what grid inputs keep exact (act_out RELU stays)."""
    return replace(c, act_in=R.IN_NONE, act_out=c.act_out if c.act_out in (R.OUT_NONE, R.OUT_RELU) else R.OUT_NONE)


def general_form(c: Conv, i):
    """The case with an input and an output activation, alternating ELU / TANH and GELU / SIGMOID."""
    return replace(c, act_in=(R.IN_ELU, R.IN_TANH)[i % 2], act_out=(R.OUT_GELU, R.OUT_SIGMOID, R.OUT_NONE)[i % 3])


SWEEP = sweep_cases()


@pytest.mark.parametrize("c", SWEEP, ids=lambda c: c.name)
def test_conv_grid_sweep(lib, c):
    check_conv(lib, grid_form(c), "grid")
    if c.act_out == R.OUT_NONE:
        check_conv(lib, replace(grid_form(c), act_out=R.OUT_RELU, name=c.name + "+relu"), "grid")


@pytest.mark.parametrize("i", range(len(SWEEP)), ids=lambda i: SWEEP[i].name)
def test_conv_general_sweep(lib, i):
    check_conv(lib, general_form(SWEEP[i], i), "general")


@pytest.mark.parametrize("c", real_layers(), ids=lambda c: c.name)
def test_conv_real_layers(lib, c):
    """Every layer shape of the default configs: grid form bit-exact with the drop-one-term check, then its own
    epilogue on random inputs within the bound.  With Cin k in the thousands the worst-case FMA-chain bound exceeds a
    single term, so the general form's sensitivity is reported (STATS) rather than asserted."""
    check_conv(lib, grid_form(replace(c, B=2 if c.Cin * c.Cout < 2 ** 20 else 1)), "grid")
    check_conv(lib, c, "general", assert_sensitivity=c.Cin * c.k <= 384)


@pytest.mark.parametrize("k,stride,dil,pad", [(7, 1, 1, "zero"), (3, 1, 1, "zero"), (8, 4, 1, "zero"), (12, 6, 1, "zero"),
                                              (4, 2, 1, "replicate"), (3, 1, 2, "zero"), (5, 2, 3, "replicate")])
def test_conv_column_shift_invariance(lib, k, stride, dil, pad):
    """One-shot, through a history-prefixed view as EncRunner::conv builds it (x moved back by pad_left columns,
    pad_left 0, Tin + hist, xT = ld), and split in two segments at T1 output columns (a multiple of neither 64 nor the
    stride; the second segment's history is the first one's last input columns, the first's zero or seeded with column
    0 as seed_replicate_kernel does): all three bit-identical, on random inputs with ELU in and GELU out."""
    c = Conv(f"shift k{k} s{stride} d{dil} {pad}", 9, 65, 131, k, stride, dil, 2, pad, act_in=R.IN_ELU,
             act_out=R.OUT_GELU)
    what = c.name
    I = conv_inputs(c, "general", rng_for(what))
    rc, yb = conv_run(lib, c, I)
    ok(rc, what)
    one = yb[:, :c.Cout, :c.Tout]
    hist = c.pad_left
    Tin = c.tin

    def hist_buf(x, first):
        """[B][xC][hist + n] with `first` as the history columns."""
        hb = np.full((c.B, I["xC"], hist + x.shape[-1]), np.nan, np.float32)
        hb[:, :c.Cin, :hist] = first
        hb[:, :c.Cin, hist:] = x
        return hb

    seed = np.repeat(I["x"][:, :, :1], hist, -1) if pad == "replicate" else 0.0
    hb = hist_buf(I["x"], seed)
    rc, yb2 = conv_run(lib, c, I, xb=hb, pad_left=0, Tin=Tin + hist, xT=hist + Tin)
    ok(rc, what + " history view")
    assert np.array_equal(bits(yb2[:, :c.Cout, :c.Tout]), bits(one)), f"{what}: history-prefixed view differs from one-shot"
    T1 = 37 if 37 % stride else 39
    assert T1 % 64 and (stride == 1 or T1 % stride) and T1 * stride >= hist
    x1, x2 = I["x"][:, :, :T1 * stride], I["x"][:, :, T1 * stride:]
    c1 = replace(c, Tout=T1)
    I1 = dict(I, xT=hist + T1 * stride)
    rc, ya = conv_run(lib, c1, I1, xb=hist_buf(x1, seed), pad_left=0, Tin=T1 * stride + hist, xT=hist + T1 * stride)
    ok(rc, what + " segment 1")
    c2 = replace(c, Tout=c.Tout - T1)
    I2 = dict(I, xT=hist + x2.shape[-1])
    rc, yc = conv_run(lib, c2, I2, xb=hist_buf(x2, x1[:, :, x1.shape[-1] - hist:] if hist else 0.0), pad_left=0,
                      Tin=x2.shape[-1] + hist, xT=hist + x2.shape[-1])
    ok(rc, what + " segment 2")
    seg = np.concatenate([ya[:, :c.Cout, :T1], yc[:, :c.Cout, :c.Tout - T1]], -1)
    bad = bits(seg) != bits(one)
    assert not bad.any(), f"{what}: split at {T1} differs from one-shot at {np.argwhere(bad)[0]}"


def test_conv_shared_memory_limit(lib):
    """smem = (8 * XW + 64 * 8 * k) * 4 bytes, XW = 63 stride + (k - 1) dil + 1: k = 46 at stride 1 is the largest
    tile within 96 KB and runs bit-exact; k = 47 is refused before any launch."""
    c = Conv("smem_k46", 9, 65, 70, 46, 1, 1, 1, "zero")
    assert (8 * (63 + 45 + 1) + 512 * 46) * 4 <= 96 * 1024 < (8 * (63 + 46 + 1) + 512 * 47) * 4
    check_conv(lib, c, "grid")
    c = replace(c, k=47, name="smem_k47")
    I = conv_inputs(c, "grid", rng_for(c.name))
    rc, yb = conv_run(lib, c, I)
    assert rc == 1, "a tile over 96 KB of shared memory must be refused"
    assert "shared memory" in last_error(), last_error()
    check_untouched(c.name, yb, I["yb"], np.zeros(yb.shape, bool))


# ================================================================================================ layernorm_ct
@pytest.mark.parametrize("C_", [8, 9, 64, 512])
@pytest.mark.parametrize("T", [1, 31, 32, 33, 100])
def test_layernorm_against_reference(lib, C_, T):
    what = f"layernorm C{C_} T{T}"
    g = rng_for(what)
    B, ldx, ldy = 2, T + 3, T + 7
    x = (g.standard_normal((B, C_, T)) * 2 + g.standard_normal((B, 1, T)) * 3).astype(np.float32)
    w = (1 + 0.3 * g.standard_normal(C_)).astype(np.float32)
    b = (0.2 * g.standard_normal(C_)).astype(np.float32)
    xb = np.full((B, C_, ldx), np.nan, np.float32)
    xb[:, :, :T] = x
    yb0 = sentinel((B, C_ + 1, ldy))
    d_x, d_w, d_b, d_y = dev(xb), dev(w), dev(b), dev(yb0)
    ok(lib.enc_shim_layernorm(ptr(d_x), ldx, ptr(d_w), ptr(d_b), ptr(d_y), ldy, C_, T, 1e-5, B, stream()), what)
    yb = host(d_y)
    region = np.zeros(yb.shape, bool)
    region[:, :C_, :T] = True
    # batch rows are C * ldy apart: the (C + 1)-th channel of the buffer is the next row's first, so compare flat
    flat = yb.reshape(-1)[:B * C_ * ldy].reshape(B, C_, ldy)
    reg = np.zeros(flat.shape, bool)
    reg[:, :, :T] = True
    check_untouched(what, flat, yb0.reshape(-1)[:B * C_ * ldy].reshape(B, C_, ldy), reg)
    check_untouched(what, yb.reshape(-1)[B * C_ * ldy:], yb0.reshape(-1)[B * C_ * ldy:], np.zeros(B * ldy, bool))
    y = flat[:, :, :T]
    want = R.ref_layernorm_ct(x, w, b, 1e-5)
    bound = R.layernorm_bound(x, w, b, 1e-5)
    err = np.abs(y - want)
    assert np.isfinite(y).all() and (err <= bound).all(), f"{what}: worst ratio {float((err / bound).max()):.3f}"
    STATS["general"] += 1
    # the same columns inside a wider launch at a column offset and another pitch: bit-identical
    T2, off, ld2 = T + 40, 17, T + 60
    xb2 = (g.standard_normal((B, C_, ld2)) * 3).astype(np.float32)
    xb2[:, :, off:off + T] = x
    d_x2, d_y2 = dev(xb2), dev(np.zeros((B, C_, ld2), np.float32))
    ok(lib.enc_shim_layernorm(ptr(d_x2), ld2, ptr(d_w), ptr(d_b), ptr(d_y2), ld2, C_, T2 + off, 1e-5, B, stream()), what)
    y2 = host(d_y2)[:, :, off:off + T]
    assert np.array_equal(bits(y2), bits(y)), f"{what}: a column's output depends on its surroundings"


# ================================================================================================ rope_ct / swa_ct
def rope_tables(npos, hd):
    """fp32 cos / sin [npos][hd/2] as MimiRotaryEmbedding computes them (oracle.mimi_encoder.rope_tables)."""
    from oracle.mimi_encoder import MimiEncCfg, rope_tables as rt
    c, s = rt(MimiEncCfg(head_dim=hd), npos)
    return c.numpy(), s.numpy()


def onehot(pos, d):
    v = np.zeros(d, np.float32)
    h1 = pos % d
    v[h1] += 1
    v[(h1 + 1 + (pos // d) % (d - 1)) % d] += 2
    return v


def swa_launch(lib, qkv, kvbuf, kv_bs, kv_ld, kv_hist, C_, T, nh, hd, window, rp, B):
    out0 = sentinel((B, C_ + 1, T))
    d_out = dev(out0)
    ok(lib.enc_shim_swa(ptr(qkv), ptr(kvbuf), kv_bs, kv_ld, kv_hist, ptr(d_out), C_, T, nh, hd, window,
                        1.0 / math.sqrt(hd), ptr(rp), B, stream()), "swa")
    return host(d_out), out0


@pytest.mark.parametrize("hd", [16, 64])
@pytest.mark.parametrize("window", [1, 2, 6, 250])
@pytest.mark.parametrize("kind", ["grid", "general"])
def test_swa_against_reference(lib, hd, window, kind):
    """Window buffer view with per-row positions: row 0 reset (position 0), row 1 at a position below window - 1, row 2
    far past the window, row 3 ragged (count < T); T = 130 crosses the 128-thread block boundary."""
    what = f"swa hd{hd} w{window} {kind}"
    g = rng_for(what)
    nh, B, T = 2, 4, 130
    C_ = nh * hd
    hist = window - 1
    pos = [0, min(3, max(window - 2, 0)), 400, 7]
    cnt = [T, T, T, 61]
    ld = hist + T + 5
    # absolute-position keys / values: key at position P of row b is the same whichever view holds it
    P_max = max(pos) + T
    if kind == "grid":
        Kall = np.zeros((B, nh, P_max, hd), np.float32)
        Vall = np.stack([[[onehot(p + 131 * h + 7 * b, hd) for p in range(P_max)] for h in range(nh)] for b in range(B)])
        Q = np.zeros((B, nh, T, hd), np.float32)
    else:
        Kall = g.standard_normal((B, nh, P_max, hd)).astype(np.float32)
        Vall = g.standard_normal((B, nh, P_max, hd)).astype(np.float32)
        Q = (g.standard_normal((B, nh, T, hd)) * 0.6).astype(np.float32)
    qkv = np.full((B, 3 * C_, T), np.nan, np.float32)
    kv = np.full((B, 2 * C_, ld), np.nan, np.float32)
    for b in range(B):
        for h in range(nh):
            qkv[b, h * hd:(h + 1) * hd, :] = Q[b, h].T
            for col in range(ld):
                P = pos[b] - hist + col
                if 0 <= P < P_max and col < hist + cnt[b]:
                    kv[b, h * hd:(h + 1) * hd, col] = Kall[b, h, P]
                    kv[b, C_ + h * hd:C_ + (h + 1) * hd, col] = Vall[b, h, P]
    rp = dev(np.array(pos + cnt, np.int32), np.int32)
    out, out0 = swa_launch(lib, dev(qkv), dev(kv), 2 * C_ * ld, ld, hist, C_, T, nh, hd, window, rp, B)
    flat = out.reshape(-1)[:B * C_ * T].reshape(B, C_, T)
    check_untouched(what, out.reshape(-1)[B * C_ * T:], out0.reshape(-1)[B * C_ * T:], np.zeros(out0.size - B * C_ * T, bool))
    for b in range(B):
        for h in range(nh):
            for t in range(cnt[b]):
                js = R.swa_keys(pos[b] + t, window)
                got = flat[b, h * hd:(h + 1) * hd, t]
                assert np.isfinite(got).all(), f"{what}: NaN at b{b} h{h} t{t}"
                K, V, q = Kall[b, h, js], Vall[b, h, js], Q[b, h, t]
                o, p, L, s = R.ref_swa_ct(q, K, V, 1.0 / math.sqrt(hd))
                if kind == "grid":
                    acc = V.astype(np.float64).sum(0).astype(np.float32)
                    want = acc * (np.float32(1) / np.float32(len(js)))
                    assert np.array_equal(bits(got), bits(want)), f"{what}: b{b} h{h} t{t} differs"
                    if len(js) > 1:
                        drop = [(acc - V[i]) * (np.float32(1) / np.float32(len(js) - 1)) for i in range(len(js))]
                        assert all((bits(d_) != bits(want)).any() for d_ in drop), f"{what}: a dropped key is invisible"
                else:
                    bound = R.swa_bound(q, K, V, s, p, L, o, 1.0 / math.sqrt(hd))
                    err = np.abs(got - o)
                    assert (err <= bound).all(), f"{what}: b{b} h{h} t{t} worst ratio {float((err / bound).max()):.3f}"
                    if t % 17 == 0:
                        check_sensitivity(what, A.sensitivity(p, L, V.astype(np.float64), o, bound))
    STATS[kind] += 1


@pytest.mark.parametrize("hd", [16, 64])
def test_rope_against_reference(lib, hd):
    """Rotated q / k within 2 2^-24 (|x1 c| + |x2 s|); v copied exactly; in place (one-shot) and into a window buffer
    (stream) at per-row positions, rows past their count untouched."""
    what = f"rope hd{hd}"
    g = rng_for(what)
    nh, B, T = 3, 2, 133
    C_, half = nh * hd, hd // 2
    pos, cnt = [0, 57], [T, 90]
    cosT, sinT = rope_tables(max(pos) + T, hd)
    qkv = (g.standard_normal((B, 3 * C_, T)) * 2).astype(np.float32)
    d_cos, d_sin = dev(cosT), dev(sinT)
    for stream_view in (False, True):
        d_qkv = dev(qkv)
        ld = T + 11
        kv0 = sentinel((B, 2 * C_, ld))
        d_kv = dev(kv0) if stream_view else None
        rp = dev(np.array(pos + cnt, np.int32), np.int32) if stream_view else None
        ok(lib.enc_shim_rope(ptr(d_qkv), ptr(d_cos), ptr(d_sin), C_, T, nh, hd, ptr(rp), B, ptr(d_kv, 4),
                             2 * C_ * ld if stream_view else 0, ld if stream_view else 0, stream()), what)
        out = host(d_qkv)
        kv = host(d_kv) if stream_view else None
        for b in range(B):
            n = cnt[b] if stream_view else T
            P = (pos[b] if stream_view else 0) + np.arange(n)
            for which in (0, 1):
                for h in range(nh):
                    base = which * C_ + h * hd
                    x1, x2 = qkv[b, base:base + half, :n], qkv[b, base + half:base + hd, :n]
                    y1, y2, e1, e2 = R.ref_rope_ct(x1, x2, cosT[P].T, sinT[P].T)
                    if which == 1 and stream_view:
                        g1, g2 = kv[b, h * hd:h * hd + half, 4:4 + n], kv[b, h * hd + half:(h + 1) * hd, 4:4 + n]
                        assert np.array_equal(bits(out[b, base:base + hd]), bits(qkv[b, base:base + hd])), \
                            f"{what}: stream rope wrote the k third of qkv"
                    else:
                        g1, g2 = out[b, base:base + half, :n], out[b, base + half:base + hd, :n]
                    assert (np.abs(g1 - y1) <= e1).all() and (np.abs(g2 - y2) <= e2).all(), f"{what}: b{b} {which} h{h}"
            if stream_view:
                v = kv[b, C_:2 * C_, 4:4 + n]
                assert np.array_equal(bits(v), bits(qkv[b, 2 * C_:3 * C_, :n])), f"{what}: v copy"
                reg = np.zeros(kv[b].shape, bool)
                reg[:, 4:4 + n] = True
                check_untouched(what + " window buffer", kv[b], kv0[b], reg)
                assert np.array_equal(bits(out[b, :, n:]), bits(qkv[b, :, n:])), f"{what}: columns past the count written"
            else:
                assert np.array_equal(bits(out[b, 2 * C_:]), bits(qkv[b, 2 * C_:])), f"{what}: one-shot wrote v"
        STATS["general"] += 1


def roll(lib, bufs, rp, B):
    n = len(bufs)
    ptrs = (C.c_void_p * n)(*[ptr(t) for t, *_ in bufs])
    ints = lambda i: (C.c_int * n)(*[b[i] for b in bufs])  # noqa: E731
    ok(lib.enc_shim_roll(ptrs, ints(1), ints(2), ints(3), ints(4), n, ptr(rp), B, stream()), "enc_roll")


@pytest.mark.parametrize("hd,window,segs", [(16, 6, (3, 1, 5, 2, 8, 4)), (64, 250, (100, 3, 1, 120, 60)),
                                            (64, 2, (1, 1, 3, 7)), (16, 1, (4, 2, 5))])
def test_stream_equals_one_shot(lib, hd, window, segs):
    """rope_ct + swa_ct over a clip one-shot (kv = the qkv thirds, no history, rp = nullptr) and streamed in segments
    through a [B][2C][window - 1 + cap] window buffer with rp, enc_roll_kernel between segments (a segment shorter
    than the history moves overlapping columns): every streamed output column and every rolled history column equals
    the one-shot, bit for bit.  Row 1 is ragged (its counts run behind row 0's)."""
    what = f"stream hd{hd} w{window} {segs}"
    g = rng_for(what)
    nh, B = 2, 2
    C_ = nh * hd
    T = sum(segs)
    hist, cap = window - 1, max(segs)
    cosT, sinT = rope_tables(T + 1, hd)
    d_cos, d_sin = dev(cosT), dev(sinT)
    qkv = (g.standard_normal((B, 3 * C_, T)) * 1.5).astype(np.float32)
    d1 = dev(qkv)
    ok(lib.enc_shim_rope(ptr(d1), ptr(d_cos), ptr(d_sin), C_, T, nh, hd, None, B, None, 0, 0, stream()), what)
    rot = host(d1)
    one, _ = swa_launch(lib, d1, d1[:, C_:], 3 * C_ * T, T, 0, C_, T, nh, hd, window, None, B)
    one = one.reshape(-1)[:B * C_ * T].reshape(B, C_, T)
    ld = hist + cap
    d_kv = dev(np.zeros((B, 2 * C_, ld), np.float32))
    done = [0, 0]
    for si, n in enumerate(segs):
        cnt = [n, max(0, min(n, T - done[1]) - (1 if si % 2 else 0))]    # row 1 ragged: one short every other packet
        seg = np.zeros((B, 3 * C_, n), np.float32)
        for b in range(B):
            seg[b, :, :cnt[b]] = qkv[b, :, done[b]:done[b] + cnt[b]]
        rp = dev(np.array(done + cnt, np.int32), np.int32)
        d_seg = dev(seg)
        ok(lib.enc_shim_rope(ptr(d_seg), ptr(d_cos), ptr(d_sin), C_, n, nh, hd, ptr(rp), B, ptr(d_kv, hist), 2 * C_ * ld, ld,
                             stream()), what)
        out, out0 = swa_launch(lib, d_seg, d_kv, 2 * C_ * ld, ld, hist, C_, n, nh, hd, window, rp, B)
        check_untouched(what, out.reshape(-1)[B * C_ * n:], out0.reshape(-1)[B * C_ * n:], np.zeros(out0.size - B * C_ * n, bool))
        out = out.reshape(-1)[:B * C_ * n].reshape(B, C_, n)
        for b in range(B):
            c0, k = done[b], cnt[b]
            assert np.array_equal(bits(out[b, :, :k]), bits(one[b, :, c0:c0 + k])), \
                f"{what}: segment {si} row {b} differs from one-shot"
        roll(lib, [(d_kv, hist, 1, 2 * C_, ld)], rp, B)
        kv = host(d_kv)
        for b in range(B):
            done[b] += cnt[b]
            for r in range(hist):
                P = done[b] - hist + r
                col = kv[b, :, r]
                want = np.concatenate([rot[b, C_:3 * C_, P]]) if P >= 0 else np.zeros(2 * C_, np.float32)
                assert np.array_equal(bits(col), bits(want)), f"{what}: segment {si} row {b} history column {r}"
    STATS["general"] += 1


# ================================================================================================ rvq_encode
def rvq_run(lib, r_sem, r_ac, books, nq, nsem, T, B, guard=3):
    """books: list of (E [K][D] fp32, E2 [K] fp32).  The codes buffer is [B][nq][T] plus `guard` sentinel elements."""
    K, D = books[0][0].shape
    E = [dev(e) for e, _ in books]
    ET = [dev(np.ascontiguousarray(e.T)) for e, _ in books]
    E2 = [dev(e2) for _, e2 in books]
    tab = lambda ts: (C.c_void_p * nq)(*[ptr(t) for t in ts])  # noqa: E731
    codes0 = np.full(B * nq * T + guard, -7, np.int32)
    d_codes = dev(codes0, np.int32)
    d_rs, d_ra = dev(r_sem), dev(r_ac)
    ok(lib.enc_shim_rvq(ptr(d_rs), ptr(d_ra), tab(E), tab(ET), tab(E2), ptr(d_codes), D, K, T, nq, nsem, B, stream()), "rvq")
    codes = host(d_codes)
    assert (codes[B * nq * T:] == -7).all(), "rvq: codes written past [B][nq][T]"
    return codes[:B * nq * T].reshape(B, nq, T)


RVQ_SHAPES = [(1, 1, 1, 1), (255, 7, 2, 1), (256, 256, 16, 1), (257, 257, 4, 4), (1023, 1, 2, 1), (1024, 7, 4, 4),
              (1025, 256, 2, 1), (2048, 1024, 16, 1), (2048, 257, 4, 4)]


@pytest.mark.parametrize("K,D,nq,nsem", RVQ_SHAPES)
def test_rvq_grid_ties(lib, K, D, nq, nsem):
    """Integer centroids and residuals, exact E2: the code is the exact argmin, lowest index on every tie.  Per frame the
    winner is planted at an index and duplicated at indices chosen to fall in the same thread's later slot (+256 i),
    its next pass (+1024), another lane (+1), another warp (+32), or a lower index in a higher warp."""
    what = f"rvq grid K{K} D{D} nq{nq}/{nsem}"
    g = rng_for(what)
    B, T = 2, 7
    r0 = {s: g.integers(-6, 7, (B, D, T)).astype(np.float32) for s in ("sem", "ac")}
    books = [g.integers(-6, 7, (K, D)).astype(np.float32) for _ in range(nq)]
    # plant per level and frame: a centroid near the current residual (r - d, d sparse in {-1, 0, 1}) at the indices of
    # one tie pattern
    patterns = [(0, 256, 512, 768), (5, 1029), (40, 41), (64, 96), (230, 261), (3, 3 + 2048), (700, 1724, 711)]
    used = [set() for _ in range(nq)]
    cur = np.zeros((B, T, D), np.float32)
    for q in range(nq):
        if q == 0 or q == nsem:
            cur = (r0["sem"] if q < nsem else r0["ac"]).transpose(0, 2, 1).copy()
        E = books[q]
        for b in range(B):
            for t in range(T):
                idx = [i for i in patterns[(b * T + t + q) % len(patterns)] if i < K]
                if not idx or any(i in used[q] for i in idx):
                    continue
                row = cur[b, t] - g.integers(-1, 2, D).astype(np.float32) * (g.random(D) < 0.2)
                for i in idx:
                    E[i] = row
                    used[q].add(i)
        dist, _ = R.ref_rvq_level(cur, E, (E.astype(np.float64) ** 2).sum(1))
        pick = R.exact_argmin(dist)
        STATS["rvq_ties"] += int(((dist == dist.min(-1, keepdims=True)).sum(-1) > 1).sum())
        cur = cur - E[pick]
    books = [(e, (e.astype(np.float64) ** 2).sum(1).astype(np.float32)) for e in books]
    assert all(np.array_equal(e2.astype(np.float64), (e.astype(np.float64) ** 2).sum(1)) for e, e2 in books)
    codes = rvq_run(lib, r0["sem"], r0["ac"], books, nq, nsem, T, B)
    cur = np.zeros((B, T, D), np.float64)
    for q in range(nq):
        if q == 0 or q == nsem:
            cur = (r0["sem"] if q < nsem else r0["ac"]).transpose(0, 2, 1).astype(np.float64)
        E, E2 = books[q]
        dist, _ = R.ref_rvq_level(cur, E, E2)
        want = R.exact_argmin(dist)
        assert np.array_equal(codes[:, q, :], want), f"{what}: level {q} codes {codes[:, q, :]} vs {want}"
        cur = cur - E[want]
    STATS["grid"] += 1


@pytest.mark.parametrize("K,D,nq,nsem", RVQ_SHAPES)
def test_rvq_general(lib, K, D, nq, nsem):
    """Random fp32 codebooks: replay the kernel's codes level by level with the fp32 residual r -= e; each pick lies
    within the fp32 distance bound of the fp64 minimum."""
    what = f"rvq general K{K} D{D} nq{nq}/{nsem}"
    g = rng_for(what)
    B, T = 2, 9
    r0 = {s: g.standard_normal((B, D, T)).astype(np.float32) for s in ("sem", "ac")}
    books = []
    for q in range(nq):
        E = (g.standard_normal((K, D)) * 0.8 / (1 + q) ** 0.5).astype(np.float32)
        books.append((E, (E.astype(np.float64) ** 2).sum(1).astype(np.float32)))
    codes = rvq_run(lib, r0["sem"], r0["ac"], books, nq, nsem, T, B)
    cur = None
    for q in range(nq):
        if q == 0 or q == nsem:
            cur = (r0["sem"] if q < nsem else r0["ac"]).transpose(0, 2, 1).copy()
        E, E2 = books[q]
        dist, bd = R.ref_rvq_level(cur, E, E2)
        k = codes[:, q, :]
        assert ((k >= 0) & (k < K)).all(), f"{what}: level {q} code out of range"
        best = dist.argmin(-1)
        dk = np.take_along_axis(dist, k[..., None], -1)[..., 0]
        gap = dk - dist.min(-1)
        allow = np.take_along_axis(bd, k[..., None], -1)[..., 0] + np.take_along_axis(bd, best[..., None], -1)[..., 0]
        assert (gap <= allow).all(), f"{what}: level {q} pick beyond the fp32 bound of the minimum"
        near = ((dist - dist.min(-1, keepdims=True)) <= bd + np.take_along_axis(bd, best[..., None], -1)).sum(-1) > 1
        STATS["rvq_near_boundary"] += int(near.sum())
        cur = cur - E[k]                                                   # the kernel's fp32 r -= e
    STATS["general"] += 1


# ================================================================================================ speaker kernels
@pytest.mark.parametrize("n_fft,hop,T", [(64, 16, 24 + 1), (64, 12, 203), (1024, 256, 384 + 1), (1024, 256, 3001),
                                         (4096, 1000, 4100)])
def test_melspec_against_reference(lib, n_fft, hop, T):
    """First and last frames reflect on both sides; T = (n_fft - hop)/2 + 1 is the shortest legal input; hop does not
    divide T; n_fft = 4096 needs the 96 KB attribute.  Filterbank row 1 is zero: exactly logf(1e-5f)."""
    from oracle.speaker_encoder import slaney_mel_filterbank
    what = f"melspec n{n_fft} h{hop} T{T}"
    g = rng_for(what)
    B, M = 2, 24
    pad = (n_fft - hop) // 2
    assert pad < T
    frames = 1 + (T + 2 * pad - n_fft) // hop
    wav = (g.standard_normal((B, T)) * 0.3).astype(np.float32)
    j = np.arange(n_fft)
    win = (0.5 - 0.5 * np.cos(2 * np.pi * j / n_fft)).astype(np.float32)
    twc, tws = np.cos(2 * np.pi * j / n_fft).astype(np.float32), np.sin(2 * np.pi * j / n_fft).astype(np.float32)
    fb = slaney_mel_filterbank(24000, n_fft, M, 0, 12000)
    fb[1] = 0
    fbT = np.ascontiguousarray(fb.T)
    out0 = sentinel((B, M, frames + 1))
    d_out = dev(out0)
    d_in = [dev(a) for a in (wav, win, twc, tws, fbT)]   # held until the launch has run
    ok(lib.enc_shim_melspec(ptr(d_in[0]), T, ptr(d_in[1]), ptr(d_in[2]), ptr(d_in[3]), ptr(d_in[4]), ptr(d_out), n_fft, hop,
                            M, frames, B, stream()), what)
    out = host(d_out).reshape(-1)
    check_untouched(what, out[B * M * frames:], out0.reshape(-1)[B * M * frames:], np.zeros(out.size - B * M * frames, bool))
    got = out[:B * M * frames].reshape(B, M, frames)
    want, bound = R.ref_melspec(wav, win, twc, tws, fbT, n_fft, hop, frames)
    err = np.abs(got - want)
    assert np.isfinite(got).all() and (err <= bound).all(), f"{what}: worst ratio {float((err / bound).max()):.3f}"
    z = got[:, 1, :]
    floor = np.float32(np.log(np.float64(np.float32(1e-5))))
    assert np.array_equal(bits(z), bits(np.full_like(z, z.flat[0]))), f"{what}: zero row not constant"
    assert abs(float(z.flat[0]) - float(floor)) <= abs(float(np.spacing(floor))), f"{what}: zero row {z.flat[0]} vs {floor}"
    STATS["mel_zero_row"] += z.size
    STATS["general"] += 1


@pytest.mark.parametrize("T", [1, 31, 32, 33, 257])
def test_asp_against_reference(lib, T):
    """asp_cat and asp_pool: rows of random values, a constant row (std clamps to sqrtf(1e-12f)), attention logits
    spread over +-80 and all equal."""
    what = f"asp T{T}"
    g = rng_for(what)
    B, C_ = 2, 5
    x = (g.standard_normal((B, C_, T)) * 2 + 1).astype(np.float32)
    x[:, 1, :] = 0.5
    att = (g.standard_normal((B, C_, T)) * 3).astype(np.float32)
    att[:, 2, :] = np.linspace(-80, 80, T).astype(np.float32)[None] if T > 1 else 80.0
    att[:, 3, :] = 1.25
    d_x = dev(x)
    cat0 = sentinel((B, 3 * C_ + 1, T))
    d_cat = dev(cat0)
    ok(lib.enc_shim_asp_cat(ptr(d_x), ptr(d_cat), C_, T, 1e-12, B, stream()), what)
    cat = host(d_cat).reshape(-1)
    n = B * 3 * C_ * T
    check_untouched(what, cat[n:], cat0.reshape(-1)[n:], np.zeros(cat.size - n, bool))
    cat = cat[:n].reshape(B, 3 * C_, T)
    m, sd, dm, dsd = R.ref_asp_cat(x)
    assert np.array_equal(bits(cat[:, :C_]), bits(x)), f"{what}: x copy"
    for t in range(T):
        assert (np.abs(cat[:, C_:2 * C_, t] - m) <= dm).all(), f"{what}: mean"
        assert (np.abs(cat[:, 2 * C_:, t] - sd) <= dsd).all(), f"{what}: std"
    assert np.array_equal(bits(cat[:, 2 * C_ + 1, :]), bits(np.full((B, T), np.sqrt(np.float32(1e-12)), np.float32))), \
        f"{what}: constant row std is not sqrtf(1e-12f)"
    pool0 = sentinel((B * 2 * C_ + 2,))
    d_pool = dev(pool0)
    d_att = dev(att)
    ok(lib.enc_shim_asp_pool(ptr(d_x), ptr(d_att), ptr(d_pool), C_, T, 1e-12, B, stream()), what)
    pool = host(d_pool)
    check_untouched(what, pool[B * 2 * C_:], pool0[B * 2 * C_:], np.zeros(2, bool))
    pool = pool[:B * 2 * C_].reshape(B, 2, C_)
    pm, psd, pdm, pdsd = R.ref_asp_pool(x, att)
    assert np.isfinite(pool).all()
    assert (np.abs(pool[:, 0] - pm) <= pdm).all(), f"{what}: pooled mean {np.abs(pool[:, 0] - pm) / pdm}"
    assert (np.abs(pool[:, 1] - psd) <= pdsd).all(), f"{what}: pooled std {np.abs(pool[:, 1] - psd) / pdsd}"
    STATS["general"] += 1


@pytest.mark.parametrize("T", [1, 127, 128, 129, 300])
def test_mean_se_copy_grid(lib, T):
    """mean_t, se_apply and copy_ch on channel-offset views with guard channels, grid inputs: bit-exact."""
    what = f"mean/se/copy T{T}"
    B, C_, xC, off = 2, 6, 11, 3
    x = grid_vals((B, xC, T), 1)
    x[:, :off] = np.nan
    x[:, off + C_:] = np.nan
    d_x = dev(x)
    m0 = sentinel((B * C_ + 2,))
    d_m = dev(m0)
    ok(lib.enc_shim_mean_t(ptr(d_x), xC, off, C_, T, ptr(d_m), B, stream()), what)
    m = host(d_m)
    check_untouched(what, m[B * C_:], m0[B * C_:], np.zeros(2, bool))
    want = (x[:, off:off + C_].astype(np.float64).sum(-1).astype(np.float32) / np.float32(T)).reshape(-1)
    assert np.array_equal(bits(m[:B * C_]), bits(want)), f"{what}: mean_t"
    h = grid_vals((B, C_, T), 4)
    gate = (np.arange(B * C_).reshape(B, C_) % 7 - 3).astype(np.float32) / 8
    y0 = sentinel((B, xC, T))
    d_y = dev(y0)
    d_h, d_g = dev(h), dev(gate)
    ok(lib.enc_shim_se_apply(ptr(d_h), ptr(d_g), ptr(d_x), xC, off, ptr(d_y), xC, 2, C_, T, B, stream()), what)
    y = host(d_y)
    reg = np.zeros(y.shape, bool)
    reg[:, 2:2 + C_] = True
    check_untouched(what + " se_apply", y, y0, reg)
    want = R.ref_se_apply(h, gate, x[:, off:off + C_])
    assert np.array_equal(bits(y[:, 2:2 + C_]), bits(want.astype(np.float32))), f"{what}: se_apply"
    ok(lib.enc_shim_copy_ch(ptr(d_x), xC, off, ptr(d_y), xC, 5, C_ - 1, T, B, stream()), what)
    y2 = host(d_y)
    reg = np.zeros(y.shape, bool)
    reg[:, 5:5 + C_ - 1] = True
    check_untouched(what + " copy_ch", y2, y, reg)
    assert np.array_equal(bits(y2[:, 5:5 + C_ - 1]), bits(x[:, off:off + C_ - 1])), f"{what}: copy_ch"
    STATS["grid"] += 1
