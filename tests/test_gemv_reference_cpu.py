"""CPU pin of tests/gemv_ref.py: the fp64 GEMV reference reproduces the oracle's own layer pieces (oracle/talker.py) on
bf16 inputs: rms_norm followed by F.linear, the MLP of decoder_layer with gate / up packed by AREngine._gate_up_blk8,
and the residual adds.  On grid inputs (small integers; normed rows of +-c) every partial sum is exact, so the two
must agree bit for bit; on random inputs they agree except where the oracle's own fp32 accumulation order or
rsqrt may round the other way, which is counted and bounded."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import talker as OT
from qwen3_tts_b200.engine import AREngine
from tests import gemv_ref as R

EPS = 1e-6


def grid(g, *shape, lo=-2, hi=2):
    return torch.randint(lo, hi + 1, shape, generator=g).bfloat16()


def pm_rows(g, nc, K, c=3.0):
    """Rows of +-c: the normed input is exactly +-1 before the norm weight."""
    return (torch.randint(0, 2, (nc, K), generator=g) * 2 - 1).bfloat16() * c


def f64(t):
    return t.double().numpy()


def test_blk8_interleave_is_the_engines():
    g = torch.Generator().manual_seed(0)
    gate, up = grid(g, 48, 64), grid(g, 48, 64)
    assert torch.equal(R.gate_up_blk8(gate, up), AREngine._gate_up_blk8(gate, up))


def test_normed_linear_matches_the_oracle_on_grid_inputs():
    g = torch.Generator().manual_seed(1)
    for nc, K, N in [(1, 64, 32), (7, 256, 48), (16, 2048, 64)]:
        x, w, W = pm_rows(g, nc, K), grid(g, K, lo=-3, hi=3), grid(g, N, K)
        want = F.linear(OT.rms_norm(x, w, EPS), W)
        xn, _ = R.normed_input(f64(x), f64(w), EPS)
        assert np.array_equal(xn, f64(OT.rms_norm(x, w, EPS))) and np.array_equal(np.abs(xn), np.abs(f64(w))[None].repeat(nc, 0))
        lo, hi, _ = R.gemv(W.double(), f64(x), R.EPI_STORE, norm_w=f64(w), eps=EPS)
        assert np.array_equal(lo, hi) and np.array_equal(lo, f64(want)), (nc, K, N)
        lo, hi, _ = R.gemv(W.double(), f64(x), R.EPI_LOGITS, norm_w=f64(w), eps=EPS)
        assert np.array_equal(lo, f64(want.float()))


def test_mlp_and_residuals_match_the_oracle_on_grid_inputs():
    g = torch.Generator().manual_seed(2)
    nc, H, I = 5, 256, 128
    x, ln2 = pm_rows(g, nc, H), grid(g, H, lo=1, hi=2)
    Wg, Wu, Wd, Wo = grid(g, I, H), grid(g, I, H), grid(g, H, I, lo=-1, hi=1), grid(g, H, H, lo=-1, hi=1)
    attn, res = grid(g, nc, H, lo=-3, hi=3), grid(g, nc, H, lo=-40, hi=40)
    # o projection + residual: res + F.linear(attn, Wo)
    want = res + F.linear(attn, Wo)
    lo, hi, _ = R.gemv(Wo.double(), f64(attn), R.EPI_RESID, resid=f64(res))
    assert np.array_equal(lo, hi) and np.array_equal(lo, f64(want))
    # SwiGLU: F.silu(F.linear(h, Wg)) * F.linear(h, Wu) with h = rms_norm(x, ln2), through the blk8 interleave
    h = OT.rms_norm(x, ln2, EPS)
    act = F.silu(F.linear(h, Wg)) * F.linear(h, Wu)
    lo, hi, _ = R.gemv(AREngine._gate_up_blk8(Wg, Wu).double(), f64(x), R.EPI_SWIGLU, norm_w=f64(ln2), eps=EPS)
    a = f64(act)
    assert ((lo <= a) & (a <= hi)).all()
    assert (lo == hi).mean() > 0.99 and np.array_equal(a[lo == hi], lo[lo == hi])
    # down projection + residual on the oracle's activations
    want = res + F.linear(act, Wd)
    lo, hi, _ = R.gemv(Wd.double(), f64(act), R.EPI_RESID, resid=f64(res))
    assert np.array_equal(lo, hi) and np.array_equal(lo, f64(want))
    # BIAS: F.linear(x, W, b)
    b = grid(g, H, lo=-9, hi=9)
    lo, hi, _ = R.gemv(Wo.double(), f64(attn), R.EPI_BIAS, bias=b)
    assert np.array_equal(lo, hi) and np.array_equal(lo, f64(F.linear(attn, Wo, b)))


def test_decoder_layer_mlp_matches_on_random_inputs_up_to_near_boundary_elements():
    """Random bf16 data: the oracle's bf16 F.linear rounds its own fp32 sum once, so its outputs lie in the reference's
    interval for an fp32 accumulation; elements where the normed input may round either way are counted."""
    g = torch.Generator().manual_seed(3)
    nc, H, I = 4, 512, 256
    x = torch.randn(nc, H, generator=g).bfloat16()
    ln = (1 + 0.1 * torch.randn(H, generator=g)).bfloat16()
    Wg, Wu = (0.05 * torch.randn(I, H, generator=g)).bfloat16(), (0.05 * torch.randn(I, H, generator=g)).bfloat16()
    h = OT.rms_norm(x, ln, EPS)
    xn, _ = R.normed_input(f64(x), f64(ln), EPS)
    near = R.normed_boundary_mask(f64(x), f64(ln), EPS)
    diff = xn != f64(h)
    assert not (diff & ~near).any(), "normed input differs away from a rounding boundary"
    assert near.mean() < 0.05
    act = F.silu(F.linear(h, Wg)) * F.linear(h, Wu)
    lo, hi, _ = R.gemv(AREngine._gate_up_blk8(Wg, Wu).double(), f64(x), R.EPI_SWIGLU, norm_w=f64(ln), eps=EPS, exact=False,
                       x_kernel=f64(h))
    a = f64(act)
    assert ((lo <= a) & (a <= hi)).all()
    print(f"random MLP: {int(near.sum())} of {near.size} normed elements near a rounding boundary, "
          f"{int(diff.sum())} differ; {float((lo != hi).mean()):.3f} of the outputs have a two-valued interval")


def test_mutations_change_the_reference_on_grid_data():
    g = torch.Generator().manual_seed(4)
    nc, K, N = 3, 96, 32
    x, W = grid(g, nc, K, lo=-3, hi=3), grid(g, N, K)
    base, _, _ = R.gemv(W.double(), f64(x), R.EPI_STORE)
    assert not np.array_equal(base, R.gemv(W.double(), f64(x), R.EPI_STORE, drop=(1, 2))[0])
    assert not np.array_equal(base, R.gemv(W.double(), f64(x), R.EPI_STORE, swap_halves=True)[0])
    sw, _, _ = R.gemv(W.double(), f64(x), R.EPI_SWIGLU)
    assert not np.array_equal(sw, R.gemv(W.double(), f64(x), R.EPI_SWIGLU, swap_gate_up=True)[0])
