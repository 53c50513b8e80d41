"""The row-kernel references (tests/rows_ref.py) against the CPU oracle: each restates, with the kernels' own views and
rounding points, a piece of oracle/codec.py, oracle/talker.py or oracle/mimi_encoder.py, so a kernel that matches the
reference computes the oracle's operation.

The same file holds the coverage guard: every __global__ kernel under qwen3-tts_b200/csrc/ is launched by name from some
test shim under tests/csrc/ (comments do not count), or is reached through a host launcher that a shim calls, listed in
LAUNCHED_VIA.  A new kernel therefore lands with a direct test, or with an edit to that map."""
import glob
import math
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import codec as OC
from oracle import mimi_encoder as ME
from oracle import talker as OT
from tests import rows_ref as R
from tests.attention_ref import rbf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-12


def bf16_t(a):
    return torch.from_numpy(np.asarray(a, np.float32)).to(torch.bfloat16)


def f64(t):
    return t.to(torch.float64).numpy()


def close(a, b, tol=TOL):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    err = np.abs(a - b).max() / max(1.0, np.abs(b).max())
    assert err < tol, err


# ================================================================================================ references vs oracle
@pytest.mark.parametrize("K,D,bins", [(16, 8, 32), (1, 4, 8), (2, 16, 2048)])
def test_rvq_gather_matches_oracle_rvq_decode(K, D, bins):
    """The embedding sums of oracle.codec.rvq_decode in bf16, before output_proj, bit for bit: output_proj is set to
    select [first; rest] into disjoint halves, so the oracle's output is (table[0][c0], the bf16 sum of the rest)."""
    g = np.random.default_rng(K * 1000 + D)
    B, T = 2, 5
    tab = rbf(g.standard_normal((K, bins, D)) * np.exp(g.uniform(-4, 4, (K, 1, 1))))
    codes = g.integers(0, bins, (B, K, T))
    codes[0, :, 0] = 0
    codes[1, :, 1] = bins - 1
    W = {}
    eye = torch.eye(D, dtype=torch.float64)
    for pfx, ks, sel in (("quantizer.rvq_first", [0], 0), ("quantizer.rvq_rest", range(1, K), 1)):
        for i, k in enumerate(ks):
            W[f"{pfx}.vq.layers.{i}._codebook.embedding_sum"] = bf16_t(tab[k])
            W[f"{pfx}.vq.layers.{i}._codebook.cluster_usage"] = torch.ones(bins, dtype=torch.bfloat16)
        proj = torch.zeros(2 * D, D, 1, dtype=torch.float64)
        proj[sel * D:(sel + 1) * D, :, 0] = eye
        W[f"{pfx}.output_proj.weight"] = proj.to(torch.bfloat16)
    cfg = OC.CodecCfg(codebook_size=bins, codebook_dim=2 * D, num_quantizers=K)
    want = f64(OC.rvq_decode(W, cfg, torch.from_numpy(codes)).transpose(1, 2))
    got = R.rvq_gather(codes, tab)
    if K == 1:
        want[..., D:] = 0.0   # no second quantizer: the oracle adds nothing, the kernel writes zeros
    assert np.array_equal(got, want)


@pytest.mark.parametrize("C,eps,scale", [(1024, 1e-5, 1.0), (2048, 1e-6, 3.0), (40, 1e-5, 1e-3)])
def test_rmsnorm_matches_oracle_rms_norm(C, eps, scale):
    """oracle.talker.rms_norm in bf16 (fp32 mean square, rsqrt, bf16, times w) lies in the reference's admissible set."""
    g = np.random.default_rng(C)
    x = rbf(g.standard_normal((9, C)) * scale)
    x[3] = 0.0
    w = rbf(g.standard_normal(C))
    want = f64(OT.rms_norm(bf16_t(x), bf16_t(w), eps))
    lo, hi = R.rmsnorm(x, w, eps)
    assert ((want == lo) | (want == hi)).all()
    assert (want[3] == 0).all()


@pytest.mark.parametrize("C,T", [(16, 9), (96, 4), (1024, 3)])
def test_dwconv_ln_matches_oracle_convnext_front(C, T):
    """dwconv + LayerNorm at fp64 equals the first two steps of oracle.codec.convnext_block (causal depthwise conv k = 7,
    then F.layer_norm eps 1e-6) with hist = 0 and the kernel's [B][T][C] layout."""
    g = np.random.default_rng(C + T)
    B = 2
    x = g.standard_normal((B, T, C))
    w, bias = g.standard_normal((C, 7)), g.standard_normal(C)
    lnw, lnb = g.standard_normal(C), g.standard_normal(C)
    h = OC.causal_conv1d(torch.from_numpy(x).transpose(1, 2), torch.from_numpy(w)[:, None, :], torch.from_numpy(bias), groups=C)
    want = F.layer_norm(h.transpose(1, 2), (C,), torch.from_numpy(lnw), torch.from_numpy(lnb), eps=1e-6).numpy()
    acc, _ = R.dwconv(x, w, bias, T, 0, T, B)
    close(acc, h.transpose(1, 2).numpy())
    close(R.layernorm(acc, lnw, lnb), want)


def test_dwconv_history_view_is_the_causal_padding():
    """hist = 6 rows of zero history in front of the rows gives the hist = 0 result (the skipped taps read zeros)."""
    g = np.random.default_rng(7)
    B, T, C = 2, 4, 8
    x = g.standard_normal((B, T, C))
    w, bias = g.standard_normal((C, 7)), g.standard_normal(C)
    xh = np.concatenate([np.zeros((B, R.HIST, C)), x, np.zeros((B, 3, C))], axis=1)
    close(R.dwconv(xh, w, bias, T, R.HIST, R.HIST + T + 3, B)[0], R.dwconv(x, w, bias, T, 0, T, B)[0])


@pytest.mark.parametrize("C,T", [(16, 11), (96, 3)])
def test_final_conv_matches_oracle_decoder_tail(C, T):
    """The last conv of oracle.codec.decoder_forward (causal, k = 7, C -> 1) and its clamp, with w [7][C]."""
    g = np.random.default_rng(C * T)
    B = 2
    x = g.standard_normal((B, T, C)) * 0.5
    w = g.standard_normal((1, C, 7)) * 0.5
    bias = 0.1
    y = OC.causal_conv1d(torch.from_numpy(x).transpose(1, 2), torch.from_numpy(w), torch.tensor([bias], dtype=torch.float64))
    want = y.clamp(min=-1, max=1)[:, 0].numpy()
    acc, _ = R.final_conv(x, w[0].T, bias, T, 0, T, B)
    close(acc, y[:, 0].numpy())
    close(R.clamp1(acc), want)
    assert (np.abs(y.numpy()) > 1).any() and (np.abs(y.numpy()) < 1).any()


def test_seed_replicate_is_the_one_shot_replicate_padding():
    """The downsample's one-shot replicate padding (MimiConv1d, left pad k_eff - stride = 2) clamps negative indices to
    column 0; the seeded history equals those padded columns, and the conv over the seeded buffer equals the one-shot."""
    g = np.random.default_rng(3)
    B, C, T, hist = 2, 4, 6, 2
    x = g.standard_normal((B, C, T))
    buf = np.concatenate([g.standard_normal((B, C, hist)), x], axis=2)
    seeded = R.seed_replicate(buf, hist, pos=[0, 0], counts=[T, T])
    padded = F.pad(torch.from_numpy(x), (hist, 0), mode="replicate").numpy()
    assert np.array_equal(seeded, padded)
    w = torch.from_numpy(g.standard_normal((C, C, 4)))
    want = ME.mimi_conv1d(torch.from_numpy(x), w, None, stride=2, pad_mode="replicate")
    got = F.conv1d(torch.from_numpy(seeded), w, None, stride=2)
    close(got.numpy(), want.numpy())
    # a row mid-stream or without frames keeps its history
    kept = R.seed_replicate(buf, hist, pos=[5, 0], counts=[T, 0])
    assert np.array_equal(kept, buf)


@pytest.mark.parametrize("count", range(1, 10))
def test_mask_covers_ceil_count_over_ds_frames(count):
    """The downsample (k = 4, stride 2) yields ceil(count / 2) frames from count 25 Hz frames: the codes the mask keeps."""
    x = torch.zeros(1, 1, count, dtype=torch.float64)
    n = ME.mimi_conv1d(x, torch.zeros(1, 1, 4, dtype=torch.float64), None, stride=2, pad_mode="replicate").shape[-1]
    assert n == R.code_frames(count, 2) == math.ceil(count / 2)
    codes = np.zeros((1, 2, 5), np.int32)
    m = R.mask_codes(codes, [count], 2)
    assert (m[0, :, :min(n, 5)] == 0).all() and (m[0, :, n:] == -1).all()


def test_roll_is_a_memmove():
    """roll on an overlapping move (T < hist) equals moving rows [T, T + hist) as a block."""
    buf = np.arange(2 * 10 * 3).reshape(2, 10, 3)
    out = R.roll(buf, 6, 1, [2, 0])
    assert np.array_equal(out[0, :6], buf[0, 2:8]) and np.array_equal(out[0, 6:], buf[0, 6:])
    assert np.array_equal(out[1], buf[1])


# ================================================================================================ coverage guard
CSRC = os.path.join(ROOT, "qwen3-tts_b200", "csrc")
SHIMS = os.path.join(ROOT, "tests", "csrc")
# kernels a shim reaches only through the library's own host launcher, which the shim calls by name
LAUNCHED_VIA = {
    "tap_gemm_kernel": "gemm_launch",            # tests/csrc/tap_gemm_shim.cu
    "conv_f32_kernel": "conv_f32_launch",        # tests/csrc/encoder_shim.cu
    "q3_step_kernel": "kStepKernels",            # tests/csrc/gemv_shim.cu: the engine's table of instantiations
}
_GLOBAL = re.compile(r"__global__\s+(?:void\s+)?(?:__launch_bounds__\s*\([^)]*\)\s*)?(?:void\s+)?(\w+)\s*\(")


def _strip_comments(src):
    return re.sub(r"//[^\n]*|/\*.*?\*/", "", src, flags=re.S)


def kernels():
    out = {}
    for f in sorted(glob.glob(os.path.join(CSRC, "*.cu*"))):
        for m in _GLOBAL.finditer(_strip_comments(open(f).read())):
            out[m.group(1)] = os.path.basename(f)
    return out


def shim_code():
    return "\n".join(_strip_comments(open(f).read()) for f in sorted(glob.glob(os.path.join(SHIMS, "*.cu"))))


def uncovered(names, code):
    return sorted(k for k in names if not re.search(r"\b%s\b" % re.escape(LAUNCHED_VIA.get(k, k)), code))


def test_every_kernel_has_a_direct_test():
    ks = kernels()
    assert len(ks) >= 30 and "dwconv_ln_kernel" in ks and "q3_step_kernel" in ks
    missing = uncovered(ks, shim_code())
    assert not missing, f"kernels no test shim under tests/csrc launches: {[(k, ks[k]) for k in missing]}"
    assert set(LAUNCHED_VIA) <= set(ks), "LAUNCHED_VIA names a kernel that no longer exists"


def test_coverage_guard_catches_a_new_kernel():
    """A kernel added to csrc/ with no shim entry fails the guard; a mention in a shim comment does not count."""
    src = "template <int N>\n__global__ void __launch_bounds__(256) brand_new_kernel(int* p) {}\n"
    names = set(kernels()) | {m.group(1) for m in _GLOBAL.finditer(src)}
    assert "brand_new_kernel" in names
    code = shim_code()
    assert uncovered(names, code) == ["brand_new_kernel"]
    assert uncovered(names, _strip_comments(code + "\n// brand_new_kernel is tested elsewhere\n")) == ["brand_new_kernel"]
    assert uncovered(names, _strip_comments(code + "\nbrand_new_kernel<<<1, 1>>>(p);\n")) == []
