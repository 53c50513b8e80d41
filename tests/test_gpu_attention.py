"""Direct checks of the three attention paths against an fp64 reference (tests/attention_ref.py) at their split, window
and position edges:
- the frame-step kernel's attention phase (csrc/ar_attention.cuh): q/k RMSNorm + RoPE, K/V append, single-query GQA
  over a 60-row shared-memory K/V window and global loads, cross-CTA split-K with a last-arriver combine;
- the prefill pair pf_qkv_post_kernel + pf_attention_kernel (csrc/ar_prefill.cuh);
- the codec's rope_append_kernel + swa_stream_kernel (csrc/codec_kernels.cuh), one-shot and stream views.
They run through tests/csrc/attention_shim.cu, which compiles its own copy of the kernels from the shipped source under
the library's flags; the phase kernel calls attn_prefetch, a CTA-wide sync and attn_phase, as q3_step_kernel does around
its grid barrier.  The instantiations inside the library are covered end to end by test_gpu_ar.py and the codec tests.

Acceptance rule.
- Grid cases are checked bit for bit.  Their queries are zero, so every kept score is equal and every p is
  __expf(0) = 1; the sums are small integers and V rows are sparse integer vectors (two non-zero dims per key, chosen
  from the key's position and region), so O and L are exact in fp32.  The output must equal the reference rounding of
  O / L (frame-step: fp32 O / L, then bf16; prefill: O * fp32(1 / L), then bf16; codec: bf16(fp32(1 / L)) * O, then
  bf16) through every split count, window side, unit-per-CTA mapping and view.  Each grid case asserts that dropping
  any single key changes some output bit, so a missing, duplicated or misplaced key fails exactly.
- General cases (random scores) are held to a per-element bound (attention_ref.online_bound / codec_bound) built from
  the fp32 dot product, __expf's documented error of 2 + floor(1.173 |x|) ulp on every rescaling a term passes through
  (online softmax, half-warp and split combine), fp32 summation of the terms, and the bf16 output rounding; for the codec
  a bf16 probability may be one step off where its value lies within that error of a rounding boundary.  Each case
  asserts its own sensitivity: removing any single key, (O - p_k v_k) / (L - p_k), moves some output element by more
  than twice the bound.
- New K rows match the reference bit for bit, except elements whose fp64 value x * inv lies within the rsqrtf + fp32
  warp-sum error of a bf16 rounding boundary (counted and reported).  V rows are copies and match exactly, and the
  codec's rotated q / k (no norm) match a numpy restatement bit for bit.
- Sentinels: every cache row at or past a row's context, other layers' and rows' regions, not-yet-valid codec history
  rows and the split buffer start as NaN, and outputs have guard rows.  Regions a kernel must not write stay
  bit-unchanged, and no NaN reaches an output.
- State: launches run back to back (layers 0..L-1, then the next frame) with no host reset; split_cnt is zero after
  every launch, and the same inputs give bit-identical outputs on a repeated launch and across grid sizes that give
  the same split count.
"""
import ctypes as C
import dataclasses
import math
import os
import subprocess
import zlib

import numpy as np
import pytest
import torch

from tests import attention_ref as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM_SRC = os.path.join(ROOT, "tests", "csrc", "attention_shim.cu")
HD = A.HD
NAN = np.int16(0x7FC0)    # bf16 NaN: cache rows a kernel must neither read nor write
SENT = np.int16(0x7FAB)   # bf16 NaN with a payload: output rows before the launch, and guard rows
EPS = 1e-6
QK = 0.265    # product of the q and k norm weight scales: a key sharing the query's input vector scores ~ +3
STATS = {"k_near_boundary": 0, "k_elements": 0, "codec_p_near_boundary": 0, "min_sensitivity": math.inf}
pytestmark = pytest.mark.gpu


# ================================================================================================ shim
@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    """tests/csrc/attention_shim.cu compiled for sm_90a with the library's flags; it links against nothing."""
    from qwen3_tts_b200 import build
    out = str(tmp_path_factory.mktemp("attention_shim") / "libattention_shim.so")
    cmd = [build._nvcc()] + build.NVCC_FLAGS + ["-shared", "-I", build.CSRC, SHIM_SRC, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"shim build failed:\n{r.stdout}\n{r.stderr}"
    lib = C.CDLL(out)
    vp, i32, f32 = C.c_void_p, C.c_int, C.c_float
    lib.attn_shim_layout.restype = C.c_longlong
    lib.attn_shim_layout.argtypes = [C.c_char_p]
    lib.attn_shim_phase.restype = i32
    lib.attn_shim_phase.argtypes = ([i32, i32, C.POINTER(i32), i32, vp, vp, i32, i32, i32, i32, i32, f32] + [vp] * 8
                                    + [i32] * 5 + [vp])
    lib.attn_shim_prefill.restype = i32
    lib.attn_shim_prefill.argtypes = [vp, vp, i32, vp, vp, i32, i32, vp, vp, f32, vp, vp, vp, vp, i32, i32, i32, vp]
    lib.attn_shim_codec.restype = i32
    lib.attn_shim_codec.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, vp, i32, i32, vp, i32, vp]
    lib.lay = {n: lib.attn_shim_layout(n.encode()) for n in ("sizeof", "split_cnt", "split_cnt_len", "att_smem", "kvwin",
                                                              "maxsplit", "rmax", "maxb", "hd")}
    return lib


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def bits(x):
    return A.bf16_bits(x)


def vals(b):
    return A.from_bits(b)


def rng_for(name):
    return np.random.default_rng(zlib.crc32(name.encode()))


def randn_bf16(rng, *shape, scale=1.0):
    return A.rbf(rng.standard_normal(shape).astype(np.float32) * np.float32(scale))


def onehot(t, region, d):
    """Sparse integer V row of key position t in region `region`: 1 at one dim and 2 at another, the pair distinct for
    every t < 2048 (so a key read from the wrong position or region changes the sums)."""
    v = np.zeros(d)
    h1 = (t + 17 * region) % d
    h2 = (h1 + 1 + (t // d) % (d - 1)) % d
    v[h1] += 1.0
    v[h2] += 2.0
    return v


def check_sensitivity(what, sens):
    STATS["min_sensitivity"] = min(STATS["min_sensitivity"], sens)
    assert sens > 1.0, f"{what}: dropping a key moves no output element by more than twice the bound ({sens:.3f})"


def check_k_rows(what, got_bits, ref, amb):
    """New K rows: bit-exact except near-boundary elements (counted)."""
    rb = bits(ref)
    bad = (got_bits != rb) & ~amb
    assert not bad.any(), f"{what}: {int(bad.sum())} K elements differ from the reference away from a rounding boundary"
    STATS["k_near_boundary"] += int(amb.sum())
    STATS["k_elements"] += amb.size


def grid_check(what, out_bits, V, round_out):
    """Grid case: out == round_out(O, n) bit for bit, and dropping any key changes some output bit."""
    n = V.shape[0]
    O = V.sum(0)
    ref = round_out(O, n)
    assert np.array_equal(out_bits, bits(ref)), (
        f"{what}: grid output differs from the exact reference at {np.flatnonzero(out_bits != bits(ref))[:8]}")
    if n >= 2:
        drop = round_out(O[None, :] - V, n - 1)
        assert (drop != ref[None, :]).any(axis=1).all(), f"{what}: some key's removal is invisible in bf16"


def frame_round(O, n):      # ar_attention.cuh: f2bf(O / L)
    return A.rbf(A.rf32(O / n))


def prefill_round(O, n):    # ar_prefill.cuh: pack_bf16(o * (1.f / l))
    return A.rbf(A.rf32(O * A.rf32(1.0 / n)))


def codec_round(O, n):      # codec: p = rbf(1 * (1.f / sum)), out = bf16(sum p * v)
    return A.rbf(A.rf32(A.rbf(A.rf32(1.0 / n)) * O))


# ================================================================================================ frame-step phase
@dataclasses.dataclass
class PhaseCase:
    name: str
    nh: int
    nkv: int
    B: int
    len0: tuple = ()
    max_len0: int = 0
    grid: int = 132
    steps: tuple = ((0, 0),)   # SEQ_DECODE: (layer, frame); SEQ_CP: (layer, nq, ctx_end)
    cap: int = 0
    layers: int = 2
    seqmode: int = 1           # 1 SEQ_DECODE (talker stack), 0 SEQ_CP (code-predictor stack)
    w: float = 0.3             # scale of the q norm weights (score spread) in general cases

    @property
    def stack(self):
        return 0 if self.seqmode == 1 else 1


def step_queries(c, step):
    """[(col, row b, pos, ctx_end)] of one launch, and the launch's (layer, frame, nq, ctx_end, nsplit)."""
    if c.seqmode == 1:
        layer, frame = step
        out = []
        for b in range(c.B):
            ce = max(1, min(c.len0[b] + frame + 1, c.cap))
            out.append((b, b, ce - 1, ce))
        cmax = c.max_len0 + frame + 1
        nsplit = max(1, min(-(-cmax // 128), c.grid // (c.B * c.nkv), 16))
        return out, (layer, frame, 1, 0, nsplit)
    layer, nq, ce = step
    out = [(b + j * c.B, b, ce - nq + j, ce) for j in range(nq) for b in range(c.B)]
    return out, (layer, 0, nq, ce, 1)


class PhaseWorld:
    """Device buffers of one case: NaN-filled K/V caches (rows written as the steps need them), split buffer, state."""

    def __init__(self, lib, c, kind, seed_name=None):
        self.lib, self.c, self.kind = lib, c, kind
        self.rng = rng_for(seed_name or f"{c.name}/{kind}")
        rng = self.rng
        self.R = c.nh // c.nkv
        shape = (c.B, c.layers, c.nkv, c.cap, HD)
        self.kc = np.full(shape, NAN, np.int16)
        self.vc = np.full(shape, NAN, np.int16)
        # cached rows every (row, layer) needs before its first step
        for b in range(c.B):
            for layer in range(c.layers):
                first = [step_queries(c, s) for s in c.steps if s[0] == layer]
                if not first:
                    continue
                qs, _ = first[0]
                lo = min(p for col, bb, p, ce in qs if bb == b)
                for kvh in range(c.nkv):
                    reg = (b * c.layers + layer) * c.nkv + kvh
                    self.kc[b, layer, kvh, :lo] = bits(randn_bf16(rng, lo, HD))
                    if kind == "grid":
                        self.vc[b, layer, kvh, :lo] = bits(np.stack([onehot(t, reg, HD) for t in range(lo)]) if lo else
                                                           np.zeros((0, HD)))
                    else:
                        self.vc[b, layer, kvh, :lo] = bits(randn_bf16(rng, lo, HD))
        self.cos, self.sin = A.rope_tables(c.cap, HD, 1e6)
        wq = c.w if kind == "general" else 0.5
        self.qn = A.rbf(wq * (1 + 0.05 * rng.standard_normal(HD)))
        self.kn = A.rbf(QK / wq * (1 + 0.05 * rng.standard_normal(HD)))
        self.d_kc, self.d_vc = dev(self.kc), dev(self.vc)
        self.d_cos, self.d_sin = dev(bits(self.cos)), dev(bits(self.sin))
        self.d_qn, self.d_kn = dev(bits(self.qn)), dev(bits(self.kn))
        lay = lib.lay
        self.d_state = torch.zeros(lay["sizeof"], dtype=torch.uint8, device="cuda")
        nsb = c.B * c.nkv * lay["maxsplit"] * lay["rmax"] * 130
        self.d_split = torch.full((nsb,), float("nan"), dtype=torch.float32, device="cuda")

    def make_qkv(self, qs):
        """qkv columns of one launch: q heads, k heads, v heads per column (bf16 values)."""
        c, rng = self.c, self.rng
        ncols = max(col for col, *_ in qs) + 1
        qkv = np.zeros((ncols, (c.nh + 2 * c.nkv) * HD))
        for col, b, pos, ce in qs:
            layer = self.layer
            for kvh in range(c.nkv):
                reg = (b * c.layers + layer) * c.nkv + kvh
                qo, ko, vo = (kvh * self.R) * HD, (c.nh + kvh) * HD, (c.nh + c.nkv + kvh) * HD
                if self.kind == "grid":
                    qkv[col, ko:ko + HD] = randn_bf16(rng, HD)
                    qkv[col, vo:vo + HD] = onehot(pos, reg, HD)
                else:
                    qkv[col, qo:qo + self.R * HD] = randn_bf16(rng, self.R * HD)
                    # the new key shares head 0's input vector: its score is ~ +3, so it carries a large weight
                    qkv[col, ko:ko + HD] = qkv[col, qo:qo + HD]
                    qkv[col, vo:vo + HD] = randn_bf16(rng, HD)
        return qkv

    def run(self, step, grid=None, qkv=None):
        """One launch; checks everything it may and may not write.  Returns (attn bits, qkv) of the launch."""
        c, lib = self.c, self.lib
        qs, (layer, frame, nq, ce_cp, nsplit) = step_queries(c, step)
        self.layer = layer
        if qkv is None:
            qkv = self.make_qkv(qs)
        ncols = qkv.shape[0]
        what = f"{c.name}/{self.kind} layer {layer} step {step} grid {grid or c.grid} nsplit {nsplit}"
        d_qkv = dev(bits(qkv))
        attn = np.full((ncols + 2, c.nh * HD), SENT, np.int16)
        d_attn = dev(attn)
        kc0, vc0 = host(self.d_kc), host(self.d_vc)
        rc = lib.attn_shim_phase(grid or c.grid, c.B, (C.c_int * c.B)(*[int(x) for x in (c.len0 or [0] * c.B)]),
                                 c.max_len0, self.d_state.data_ptr(), self.d_split.data_ptr(), c.stack, c.nh, c.nkv,
                                 c.layers, c.cap, EPS, d_qkv.data_ptr(), d_attn.data_ptr() + c.nh * HD * 2,
                                 self.d_kc.data_ptr(), self.d_vc.data_ptr(), self.d_cos.data_ptr(),
                                 self.d_sin.data_ptr(), self.d_qn.data_ptr(), self.d_kn.data_ptr(), layer, c.seqmode,
                                 nq, ce_cp, frame, stream())
        assert rc == 0, f"{what}: launch failed ({rc})"
        kc, vc, out = host(self.d_kc), host(self.d_vc), host(d_attn)
        st = host(self.d_state).view(np.uint32)
        o = self.lib.lay["split_cnt"] // 4
        assert not st[o:o + self.lib.lay["split_cnt_len"]].any(), f"{what}: split_cnt not reset"
        assert np.array_equal(host(d_qkv), bits(qkv)), f"{what}: qkv was written"
        # ---- new K / V rows, and nothing else of the caches
        exp_k, exp_v = kc0.copy(), vc0.copy()
        for col, b, pos, ce in qs:
            for kvh in range(c.nkv):
                ko, vo = (c.nh + kvh) * HD, (c.nh + c.nkv + kvh) * HD
                kref, amb = A.norm_rope(qkv[col, ko:ko + HD], self.kn, self.cos[pos], self.sin[pos], EPS)
                check_k_rows(f"{what} row {b} pos {pos} kvh {kvh}", kc[b, layer, kvh, pos], kref, amb)
                assert np.array_equal(vc[b, layer, kvh, pos], bits(qkv[col, vo:vo + HD])), f"{what}: V row {pos}"
                exp_k[b, layer, kvh, pos] = kc[b, layer, kvh, pos]
                exp_v[b, layer, kvh, pos] = bits(qkv[col, vo:vo + HD])
        assert np.array_equal(kc, exp_k), f"{what}: K cache written outside the new rows"
        assert np.array_equal(vc, exp_v), f"{what}: V cache written outside the new rows"
        # ---- outputs: guard rows and unused columns untouched, written columns finite and right
        cols = {col for col, *_ in qs}
        for r in range(ncols + 2):
            if r - 1 in cols:
                assert not (out[r] == SENT).any(), f"{what}: column {r - 1} not (fully) written"
                assert np.isfinite(vals(out[r])).all(), f"{what}: NaN / inf in column {r - 1}"
            else:
                assert (out[r] == SENT).all(), f"{what}: guard / unused row {r - 1} written"
        scale = 1.0 / math.sqrt(HD)
        for col, b, pos, ce in qs:
            SL = -(-ce // nsplit)
            chain = 2 * -(-SL // 32) + 2
            for h in range(c.nh):
                kvh = h // self.R
                K = vals(kc[b, layer, kvh, :pos + 1])
                V = vals(vc[b, layer, kvh, :pos + 1])
                got = out[col + 1, h * HD:(h + 1) * HD]
                hw = f"{what} col {col} head {h} pos {pos}"
                if self.kind == "grid":
                    grid_check(hw, got, V, frame_round)
                    continue
                q, amb_q = A.norm_rope(qkv[col, h * HD:(h + 1) * HD], self.qn, self.cos[pos], self.sin[pos], EPS)
                o, p, L, s = A.attend(q, K, V, scale)
                bound = A.online_bound(q, K, V, s, p, L, o, scale, chain, chain + 32 + nsplit, amb_q)
                err = np.abs(vals(got) - o)
                assert (err <= bound).all(), f"{hw}: |kernel - ref| {err.max():.3g} > bound at {np.argmax(err - bound)}"
                check_sensitivity(hw, A.sensitivity(p, L, V, o, bound))
        return out, qkv


def _ctx_cap(c):
    if c.cap:
        return c
    if c.seqmode == 1:
        top = max(c.len0) + max(f for _, f in c.steps) + 2
    else:
        top = max(ce for _, _, ce in c.steps) + 1
    return dataclasses.replace(c, cap=top + 3)


T17 = dict(nh=16, nkv=8)    # 1.7B talker / code predictor: 16 q heads over 8 kv heads
TINY = dict(nh=4, nkv=2)
PHASE_CASES = [_ctx_cap(c) for c in [
    # production geometries at grid 132
    PhaseCase("1p7b_b1_6split", **T17, B=1, len0=(700,), max_len0=700, w=0.2),
    PhaseCase("1p7b_b8_ragged_2split", **T17, B=8, len0=(250, 3, 0, 120, 59, 1, 200, 260), max_len0=260),
    PhaseCase("1p7b_b32_two_units_per_cta", **T17, B=32, len0=tuple(1 + (53 * i) % 230 for i in range(32)),
              max_len0=230),
    PhaseCase("tiny_b3", **TINY, B=3, len0=(40, 77, 130), max_len0=130),
    PhaseCase("r1", nh=8, nkv=8, B=2, len0=(90, 300), max_len0=300),
    # split counts 1, 2, 3, 15, 16 and grids 1, 7, 133
    PhaseCase("tiny_16split", **TINY, B=1, len0=(1999,), max_len0=1999, w=0.15),
    PhaseCase("tiny_15split", **TINY, B=1, len0=(1850,), max_len0=1850, w=0.15),
    PhaseCase("1p7b_16split_grid133", **T17, B=1, len0=(1930,), max_len0=1930, grid=133, w=0.15),
    PhaseCase("tiny_grid7_3split", **TINY, B=1, len0=(400,), max_len0=400, grid=7),
    PhaseCase("tiny_grid1_units_loop", **TINY, B=4, len0=(58, 59, 60, 150), max_len0=150, grid=1),
    PhaseCase("tiny_2split", **TINY, B=2, len0=(200, 129), max_len0=200),
    # split lengths 59, 60, 61 (3 splits) and a row longer than max_len0 + frame + 1 (one split of 134 rows)
    PhaseCase("split_len_59_60_61_134", **TINY, B=4, len0=(176, 179, 182, 399), max_len0=300),
    # clamp: len0 + frame + 1 > cap (context cap), and <= 0 (context 1, empty second split)
    PhaseCase("clamp", **TINY, B=3, len0=(130, -4, 50), max_len0=130, steps=((0, 1),), cap=128),
]]
CP_CASES = [_ctx_cap(c) for c in [
    PhaseCase(f"cp_b{B}", **T17, B=B, seqmode=0, steps=((0, 2, 2),) + tuple((0, 1, ce) for ce in range(3, 17)))
    for B in (16, 5)] + [PhaseCase("cp_nq1_ctx1", **T17, B=3, seqmode=0, steps=((1, 1, 1),))]]


@pytest.mark.parametrize("kind", ["grid", "general"])
@pytest.mark.parametrize("case", PHASE_CASES, ids=lambda c: c.name)
def test_phase_against_reference(shim, case, kind):
    W = PhaseWorld(shim, case, kind)
    for step in case.steps:
        W.run(step)


@pytest.mark.parametrize("kind", ["grid", "general"])
@pytest.mark.parametrize("case", CP_CASES, ids=lambda c: c.name)
def test_phase_code_predictor(shim, case, kind):
    """SEQ_CP: the two-token pass 0 (nq = 2, qstride = B) then one token per pass at ctx_end 3..16, on one cache."""
    W = PhaseWorld(shim, case, kind)
    for step in case.steps:
        W.run(step)


def test_phase_state_across_launches(shim):
    """Layers 0..L-1 of frame f, then of frame f+1, back to back on one state and split buffer; then the same inputs
    again (fresh caches) at the same and at another grid size with the same split count: bit-identical outputs."""
    c = _ctx_cap(PhaseCase("state", **TINY, B=3, len0=(300, 5, 61), max_len0=300, layers=3,
                           steps=tuple((layer, f) for f in (4, 5) for layer in range(3))))
    runs = []
    for grid in (132, 132, 140):
        W = PhaseWorld(shim, c, "general", seed_name="state")
        nsplit = {step_queries(dataclasses.replace(c, grid=grid), s)[1][4] for s in c.steps}
        assert nsplit == {3}
        outs, qkv_prev = [], []
        for i, step in enumerate(c.steps):
            qkv = runs[0][1][i] if runs else None
            out, q = W.run(step, grid=grid, qkv=qkv)
            outs.append(out)
            qkv_prev.append(q)
        runs.append((outs, qkv_prev, host(W.d_kc), host(W.d_vc)))
    for r in runs[1:]:
        for a, b in zip(runs[0][0], r[0]):
            assert np.array_equal(a, b), "outputs differ between identical launches"
        assert np.array_equal(runs[0][2], r[2]) and np.array_equal(runs[0][3], r[3]), "caches differ"


# ================================================================================================ prefill pair
def prefill_world(lib, name, prompts, nslots, nh, nkv, layers, kind, cap=None):
    rng = rng_for(name)
    cap = cap or max(n for _, n in prompts) + 8
    shape = (nslots, layers, nkv, cap, HD)
    d_kc = dev(np.full(shape, NAN, np.int16))
    d_vc = dev(np.full(shape, NAN, np.int16))
    cos, sin = A.rope_tables(cap, HD, 1e6)
    wq = 0.3 if kind == "general" else 0.5
    qn = A.rbf(wq * (1 + 0.05 * rng.standard_normal(HD)))
    kn = A.rbf(QK / wq * (1 + 0.05 * rng.standard_normal(HD)))
    return dict(rng=rng, cap=cap, d_kc=d_kc, d_vc=d_vc, cos=cos, sin=sin, qn=qn, kn=kn, d_cos=dev(bits(cos)),
                d_sin=dev(bits(sin)), d_qn=dev(bits(qn)), d_kn=dev(bits(kn)), nh=nh, nkv=nkv, layers=layers,
                nslots=nslots, kind=kind)


def prefill_layer(lib, P, prompts, layer, what, qkv=None, check_attn=True):
    """prefill of the packed prompts [(slot, len)] at one layer; checks q in place, the cache and the attention."""
    nh, nkv, rng = P["nh"], P["nkv"], P["rng"]
    R = nh // nkv
    seq = np.array([s for s, n in prompts for _ in range(n)], np.int32)
    pos = np.array([p for s, n in prompts for p in range(n)], np.int32)
    ntok = len(seq)
    W = (nh + 2 * nkv) * HD
    if qkv is None:
        qkv = np.zeros((ntok, W))
        for i in range(ntok):
            for kvh in range(nkv):
                reg = (seq[i] * P["layers"] + layer) * nkv + kvh
                ko, vo = (nh + kvh) * HD, (nh + nkv + kvh) * HD
                qkv[i, ko:ko + HD] = randn_bf16(rng, HD)
                if P["kind"] == "grid":
                    qkv[i, vo:vo + HD] = onehot(int(pos[i]), reg, HD)
                else:
                    qkv[i, vo:vo + HD] = randn_bf16(rng, HD)
            if P["kind"] != "grid":
                qkv[i, :nh * HD] = randn_bf16(rng, nh * HD)
    d_qkv = dev(bits(qkv))
    d_attn = dev(np.full((ntok + 2, nh * HD), SENT, np.int16))
    kc0, vc0 = host(P["d_kc"]), host(P["d_vc"])
    d_seq, d_pos = dev(seq), dev(pos)
    rc = lib.attn_shim_prefill(d_qkv.data_ptr(), d_attn.data_ptr() + nh * HD * 2, ntok, d_seq.data_ptr(),
                               d_pos.data_ptr(), nh, nkv, P["d_qn"].data_ptr(), P["d_kn"].data_ptr(), EPS,
                               P["d_cos"].data_ptr(), P["d_sin"].data_ptr(), P["d_kc"].data_ptr(), P["d_vc"].data_ptr(),
                               layer, P["layers"], P["cap"], stream())
    assert rc == 0, f"{what}: launch failed"
    q_out, out, kc, vc = host(d_qkv), host(d_attn), host(P["d_kc"]), host(P["d_vc"])
    exp_k, exp_v = kc0.copy(), vc0.copy()
    for i in range(ntok):
        s, p = int(seq[i]), int(pos[i])
        for h in range(nh):
            qref, amb = A.norm_rope(qkv[i, h * HD:(h + 1) * HD], P["qn"], P["cos"][p], P["sin"][p], EPS)
            check_k_rows(f"{what} q tok {i} head {h}", q_out[i, h * HD:(h + 1) * HD], qref, amb)
        for kvh in range(nkv):
            ko, vo = (nh + kvh) * HD, (nh + nkv + kvh) * HD
            kref, amb = A.norm_rope(qkv[i, ko:ko + HD], P["kn"], P["cos"][p], P["sin"][p], EPS)
            check_k_rows(f"{what} K tok {i} kvh {kvh}", kc[s, layer, kvh, p], kref, amb)
            exp_k[s, layer, kvh, p] = kc[s, layer, kvh, p]
            exp_v[s, layer, kvh, p] = bits(qkv[i, vo:vo + HD])
    assert np.array_equal(q_out[:, nh * HD:], bits(qkv[:, nh * HD:])), f"{what}: k / v heads of qkv written"
    assert np.array_equal(kc, exp_k), f"{what}: K cache differs outside / at the new rows"
    assert np.array_equal(vc, exp_v), f"{what}: V cache differs outside / at the new rows"
    assert (out[0] == SENT).all() and (out[-1] == SENT).all(), f"{what}: guard rows written"
    if not check_attn:
        return qkv, kc
    assert np.isfinite(vals(out[1:-1])).all(), f"{what}: NaN / inf / unwritten attention output"
    scale = 1.0 / math.sqrt(HD)
    for i in range(ntok):
        s, p = int(seq[i]), int(pos[i])
        nb = p // 32 + 1
        for h in range(nh):
            kvh = h // R
            K, V = vals(kc[s, layer, kvh, :p + 1]), vals(vc[s, layer, kvh, :p + 1])
            got = out[i + 1, h * HD:(h + 1) * HD]
            hw = f"{what} tok {i} (slot {s} pos {p}) head {h}"
            if P["kind"] == "grid":
                grid_check(hw, got, V, prefill_round)
                continue
            q = vals(q_out[i, h * HD:(h + 1) * HD])
            o, pr, L, sc = A.attend(q, K, V, scale)
            bound = A.online_bound(q, K, V, sc, pr, L, o, scale, nb + 2, p + 1 + 32 + nb)
            err = np.abs(vals(got) - o)
            assert (err <= bound).all(), f"{hw}: |kernel - ref| {err.max():.3g} > bound"
            check_sensitivity(hw, A.sensitivity(pr, L, V, o, bound))
    return qkv, kc


PROMPTS = [(5, 1), (0, 34), (9, 65), (2, 500)]   # positions 0, 31, 32, 33, 63, 64, ~500; slots not contiguous


@pytest.mark.parametrize("kind", ["grid", "general"])
def test_prefill_against_reference(shim, kind):
    P = prefill_world(shim, f"prefill/{kind}", PROMPTS, 12, 4, 2, 2, kind)
    for layer in range(2):
        prefill_layer(shim, P, PROMPTS, layer, f"prefill/{kind} layer {layer}")


@pytest.mark.parametrize("kind", ["grid", "general"])
def test_prefill_decode_handoff(shim, kind):
    """K/V written by the prefill for positions < len are read by the decode phase at ctx = len + 1 through both the
    shared-memory window and global loads (one split of len + 1 > 60 rows); and the prefill and the decode phase write
    the same K bits for the same qkv vector and position."""
    prompts = [(0, 100), (2, 61)]
    P = prefill_world(shim, f"handoff/{kind}", prompts, 3, 4, 2, 2, kind, cap=112)
    for layer in range(2):
        prefill_layer(shim, P, prompts, layer, f"handoff/{kind} prefill layer {layer}")
    c = PhaseCase("handoff", **TINY, B=3, len0=(100, 0, 61), max_len0=100, grid=6, cap=112,
                  steps=((0, 0), (1, 0)))
    W = PhaseWorld(shim, c, kind, seed_name=f"handoff/{kind}/decode")
    W.kc, W.vc = host(P["d_kc"]), host(P["d_vc"])
    W.d_kc, W.d_vc = P["d_kc"], P["d_vc"]
    W.qn, W.kn, W.d_qn, W.d_kn = P["qn"], P["kn"], P["d_qn"], P["d_kn"]
    for step in c.steps:
        _, qkv = W.run(step)
        layer = step[0]
        # the same k vector through the prefill at the decode token's position, into a fresh cache
        Q = prefill_world(shim, f"handoff/{kind}/k", [(0, 101)], 1, 4, 2, 2, kind, cap=112)
        Q.update(qn=P["qn"], kn=P["kn"], d_qn=P["d_qn"], d_kn=P["d_kn"])
        one = qkv[:1].copy()
        tok_seq = np.zeros(1, np.int32)
        tok_pos = np.full(1, 100, np.int32)
        d_one = dev(bits(one))
        d_attn = dev(np.full((3, 4 * HD), SENT, np.int16))
        d_seq, d_pos = dev(tok_seq), dev(tok_pos)
        rc = shim.attn_shim_prefill(d_one.data_ptr(), d_attn.data_ptr() + 4 * HD * 2, 1, d_seq.data_ptr(),
                                    d_pos.data_ptr(), 4, 2, Q["d_qn"].data_ptr(), Q["d_kn"].data_ptr(), EPS,
                                    Q["d_cos"].data_ptr(), Q["d_sin"].data_ptr(), Q["d_kc"].data_ptr(),
                                    Q["d_vc"].data_ptr(), layer, 2, 112, stream())
        assert rc == 0
        kq, kd = host(Q["d_kc"]), host(W.d_kc)
        assert np.array_equal(kq[0, layer, :, 100], kd[0, layer, :, 100]), "prefill and decode K rows differ"


# ================================================================================================ codec
@dataclasses.dataclass
class CodecCase:
    name: str
    B: int
    n: int
    nh: int
    hd: int
    window: int
    rows: tuple = ()     # stream view: (position, count) per batch row; () = one-shot


CODEC_CASES = [
    CodecCase("default_w72_oneshot", B=2, n=150, nh=16, hd=64, window=72),
    CodecCase("w96_oneshot", B=1, n=130, nh=4, hd=64, window=96),
    CodecCase("w33_oneshot", B=2, n=80, nh=4, hd=64, window=33),
    CodecCase("w6_hd16_oneshot", B=2, n=20, nh=4, hd=16, window=6),
    CodecCase("default_w72_stream", B=3, n=8, nh=16, hd=64, window=72, rows=((0, 8), (5, 3), (200, 0))),
    CodecCase("w96_stream", B=3, n=8, nh=4, hd=64, window=96, rows=((200, 8), (5, 8), (70, 5))),
    CodecCase("w6_hd16_stream", B=3, n=8, nh=4, hd=16, window=6, rows=((0, 5), (5, 8), (200, 0))),
]
CODEC_FRAMES = 512


def run_codec(lib, c, kind):
    rng = rng_for(f"codec/{c.name}/{kind}")
    nh, hd, B, n = c.nh, c.hd, c.B, c.n
    cos, sin = A.rope_tables(CODEC_FRAMES, hd, 10000.0)
    qkv = randn_bf16(rng, B, n, 3 * nh * hd)
    # q scaled so that scores spread ~ 0.4: every key keeps a weight that its removal shows
    qkv[:, :, :nh * hd] = 0.0 if kind == "grid" else randn_bf16(rng, B, n, nh * hd, scale=0.4)
    stream_view = bool(c.rows)
    pos0 = [r[0] for r in c.rows] if stream_view else [0] * B
    cnt = [r[1] for r in c.rows] if stream_view else [n] * B
    hist = c.window - 1 if stream_view else 0
    rows = hist + n
    # V heads: grid rows are sparse integer vectors of the key's absolute position
    for b in range(B):
        for t in range(n):
            for h in range(nh):
                o = (2 * nh + h) * hd
                if kind == "grid":
                    qkv[b, t, o:o + hd] = onehot(pos0[b] + t, b * nh + h, hd)
    # stream window buffer: history rows of absolute position >= 0 hold K (already rotated) and V, others NaN
    kvb = np.full((B, rows, 2 * nh * hd), NAN, np.int16)
    if stream_view:
        for b in range(B):
            for r in range(hist):
                ap = pos0[b] - hist + r
                if ap < 0:
                    continue
                kvb[b, r, :nh * hd] = bits(randn_bf16(rng, nh * hd))
                vrow = (np.concatenate([onehot(ap, b * nh + h, hd) for h in range(nh)]) if kind == "grid"
                        else randn_bf16(rng, nh * hd))
                kvb[b, r, nh * hd:] = bits(vrow)
    rp = np.array(pos0 + cnt, np.int32)
    d_qkv = dev(bits(qkv))
    d_kv = dev(kvb)
    d_out = dev(np.full((B * n + 2, nh * hd), SENT, np.int16))
    d_rp, d_cos, d_sin = dev(rp), dev(bits(cos)), dev(bits(sin))
    rc = lib.attn_shim_codec(d_qkv.data_ptr(), d_cos.data_ptr(), d_sin.data_ptr(),
                             d_kv.data_ptr() if stream_view else None, B, n, nh, hd,
                             d_rp.data_ptr() if stream_view else None, hist, rows, d_out.data_ptr() + nh * hd * 2,
                             c.window, stream())
    assert rc == 0, f"{c.name}: launch failed"
    q_out, kv_out, out = host(d_qkv), host(d_kv), host(d_out)
    what = f"codec {c.name}/{kind}"
    # ---- RoPE of q, k: bit-exact restatement; v heads untouched; frames past a row's count untouched
    exp_q = bits(qkv)
    for b in range(B):
        for t in range(cnt[b]):
            p = pos0[b] + t
            for h in range(2 * nh):
                exp_q[b, t, h * hd:(h + 1) * hd] = bits(A.rope_rotate(qkv[b, t, h * hd:(h + 1) * hd], cos[p], sin[p]))
    assert np.array_equal(q_out, exp_q), f"{what}: rotated q / k differ from the restatement (or a frame past the count)"
    exp_kv = kvb.copy()
    if stream_view:
        for b in range(B):
            for t in range(cnt[b]):
                exp_kv[b, hist + t, :nh * hd] = exp_q[b, t, nh * hd:2 * nh * hd]
                exp_kv[b, hist + t, nh * hd:] = exp_q[b, t, 2 * nh * hd:]
    assert np.array_equal(kv_out, exp_kv), f"{what}: window buffer differs (appended rows, history, or past the count)"
    # ---- attention
    assert (out[0] == SENT).all() and (out[-1] == SENT).all(), f"{what}: guard rows written"
    for b in range(B):
        if stream_view:
            K_all = vals(kv_out[b, :, :nh * hd])
            V_all = vals(kv_out[b, :, nh * hd:])
        else:
            K_all = vals(q_out[b, :, nh * hd:2 * nh * hd])
            V_all = vals(q_out[b, :, 2 * nh * hd:])
        for t in range(n):
            row = out[1 + b * n + t]
            if t >= cnt[b]:
                assert (row == SENT).all(), f"{what}: row {b} frame {t} past its count was written"
                continue
            assert np.isfinite(vals(row)).all(), f"{what}: NaN / unwritten output at row {b} frame {t}"
            r1 = hist + t
            r0 = max(r1 - c.window + 1, hist - pos0[b], 0)
            for h in range(nh):
                q = vals(q_out[b, t, h * hd:(h + 1) * hd])
                K = K_all[r0:r1 + 1, h * hd:(h + 1) * hd]
                V = V_all[r0:r1 + 1, h * hd:(h + 1) * hd]
                got = row[h * hd:(h + 1) * hd]
                hw = f"{what} row {b} frame {t} head {h} keys {r1 - r0 + 1}"
                if kind == "grid":
                    grid_check(hw, got, V, codec_round)
                    continue
                o, bound, pr, namb = A.codec_bound(q, K, V, hd)
                STATS["codec_p_near_boundary"] += namb
                err = np.abs(vals(got) - o)
                assert (err <= bound).all(), f"{hw}: |kernel - ref| {err.max():.3g} > bound"
                check_sensitivity(hw, A.codec_sensitivity(q, K, V, hd, bound))


@pytest.mark.parametrize("kind", ["grid", "general"])
@pytest.mark.parametrize("case", CODEC_CASES, ids=lambda c: c.name)
def test_codec_against_reference(shim, case, kind):
    run_codec(shim, case, kind)


@pytest.mark.parametrize("window", [0, -1, 97])
def test_codec_rejects_unsupported_window(window):
    """q3_codec_create refuses a window outside [1, 96]: below 1 a query would see no key (a division by a zero sum)
    and a stream would keep -1 history rows; above 96 the kernel's three key slots per lane do not reach."""
    from qwen3_tts_b200 import CodecConfig
    from qwen3_tts_b200.codec import CodecDecoder
    cfg = CodecConfig(codebook_size=64, codebook_dim=32, hidden_size=64, latent_dim=64, num_heads=4, num_kv_heads=4,
                      head_dim=16, sliding_window=window, intermediate_size=96, num_layers=1, decoder_dim=256)
    with pytest.raises(RuntimeError, match="sliding_window"):
        CodecDecoder(cfg, {}, device="cuda:0", max_frames=16, max_batch=1)


def test_report_stats():
    """Counts of the checks above that needed a tolerance (printed with -s)."""
    print("attention checks:", STATS)
