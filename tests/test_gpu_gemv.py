"""Direct checks of the frame-step kernel's GEMV phase (csrc/ar_gemv.cuh: gemv_phase inside q3_step_kernel<NT, VAR>)
against the fp64 reference of tests/gemv_ref.py, at its tile, split, batch-class, input-path, ring and epilogue edges.

The phases run through tests/csrc/gemv_shim.cu: the production kernel and the engine's own host plan (tile assignment,
shared-memory plan, run table), launched cooperatively as the engine does, on programs of GEMV phases built from plain
arrays.  Every output buffer is surrounded by bf16 NaN sentinels (rows >= nc, rows >= N when dst_ld > N, save_normed
rows of unmasked columns, hid_out rows outside [0, hid_stride)) that must stay untouched.

Acceptance rule.
- Grid inputs: weights and inputs are small integers, or for normed phases rows of +-c, so that bf16(x * inv) = +-1
  even with rsqrtf's 2-ulp error and the normed operand is exactly +-w.  Every partial sum is then exact in fp32 in any
  order and under tensor-core truncation, and every output must equal the reference exactly (SWIGLU: except where
  __expf's error of 2 + floor(1.173 |g|) ulp straddles a bf16 rounding boundary; such outputs are counted, and may
  take either neighbour).
- General inputs (random bf16): each output must be the epilogue of some accumulator value within
  s -+ K 2^-22 sum|w x| (SWIGLU also allows the __expf error).  Saved normed inputs match bit for bit, except elements
  within the rsqrtf and sum-of-squares bound of a bf16 rounding boundary, which are counted and reported; the output
  bound is then taken over the kernel's own saved operand.
- Sensitivity: every grid case also asserts that the reference differs from the kernel's output when one k-block of
  one tile is dropped, when the two 4-element halves of each lane's 8-k group are swapped (the K permutation), and for
  SWIGLU when gate and up are exchanged, so the data could catch those errors.
A Python restatement of cta_tiles / run_geom records which geometric properties each case reaches;
test_zz_every_property_was_hit asserts that every property was reached.
"""
import ctypes as C
import os
import subprocess
import time
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from qwen3_tts_b200 import synthetic
from qwen3_tts_b200.engine import AREngine
from tests import gemv_ref as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM_SRC = os.path.join(ROOT, "tests", "csrc", "gemv_shim.cu")
SENT16 = 0x7FC1                       # bf16 NaN sentinel
SENT32 = 0x7FC00001                   # fp32 NaN sentinel (LOGITS)
EPS = 1e-6
DEV = "cuda"
NWARPS, NTHREADS = 8, 256

PROPS = ["idle_cta", "tr_edge", "multi_round", "partial_round_3", "partial_round_5", "kb_lt_sb", "general_path",
         "empty_warp", "run_two_tiles", "nct_lt_nt", "nc2b", "staged_normed", "staged_tma", "unstaged", "unstaged_wrap",
         "ring_sb2", "ring_sb1", "ring_r2", "epi_store", "epi_bias", "epi_resid", "epi_swiglu", "epi_logits",
         "resid_loaded", "nt1", "nt2", "nt4", "chain", "mode1", "var1_capture", "general_inputs", "production_full_piece"]
HIT = {p: 0 for p in PROPS}
STATS = {"cases": 0, "launches": 0, "outputs": 0, "swiglu_two_valued": 0, "normed_near_boundary": 0,
         "normed_differs": 0, "general_two_valued": 0}
T0 = [None]


# ================================================================================================ shim
@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    """tests/csrc/gemv_shim.cu compiled for sm_90a with the library's flags; it links against nothing."""
    from qwen3_tts_b200 import build
    T0[0] = time.time()
    out = str(tmp_path_factory.mktemp("gemv_shim") / "libgemv_shim.so")
    cmd = [build._nvcc()] + build.NVCC_FLAGS + ["-shared", "-I", build.CSRC, SHIM_SRC, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"shim build failed:\n{r.stdout}\n{r.stderr}"
    L = C.CDLL(out)
    vp, i32, pi, pv = C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_void_p)
    L.gemv_shim_last_error.restype = C.c_char_p
    L.gemv_shim_layout.restype = C.c_longlong
    L.gemv_shim_layout.argtypes = [C.c_char_p]
    L.gemv_shim_pack.restype = i32
    L.gemv_shim_pack.argtypes = [vp, vp, i32, i32, vp]
    L.gemv_shim_plan.restype = i32
    L.gemv_shim_plan.argtypes = [i32, pi, pi, pi, pi, i32, i32, i32, pi, pi]
    L.gemv_shim_run.restype = i32
    L.gemv_shim_run.argtypes = ([i32, pv, pi, pi, pv, pi, pv, C.POINTER(C.c_float), pv, pi, pi, pi, pv, pv]
                                + [i32] * 6 + [C.c_uint32, pi, vp, i32, i32, vp, C.c_longlong, vp, C.c_longlong, vp,
                                               C.c_longlong, vp, vp])
    L.path = out
    L.lay = {n: L.gemv_shim_layout(n.encode()) for n in ("sizeof_state", "bar_count", "error", "step", "finished",
                                                         "sizeof_phase", "max_phases", "max_batch", "max_dyn_smem")}
    L.sms = torch.cuda.get_device_properties(0).multi_processor_count
    # caller-owned device scratch: program, run table, run offsets, state
    L.prog = torch.zeros(L.lay["max_phases"] * L.lay["sizeof_phase"], dtype=torch.uint8, device=DEV)
    L.runs = torch.zeros(1 << 23, dtype=torch.uint8, device=DEV)
    L.off = torch.zeros((L.sms * NWARPS + 1) * 4 + 64, dtype=torch.uint8, device=DEV)
    L.state = torch.zeros(L.lay["sizeof_state"], dtype=torch.uint8, device=DEV)
    return L


def err(L):
    return L.gemv_shim_last_error().decode()


# ================================================================================================ buffers and phases
class Buf:
    """[rows][ld] tensor between one guard row on each side, filled with the NaN sentinel."""

    def __init__(self, rows, ld, f32=False, data=None):
        self.rows, self.ld, self.f32 = rows, ld, f32
        if f32:
            self.t = torch.full((rows + 2, ld), SENT32, dtype=torch.int32, device=DEV).view(torch.float32)
        else:
            self.t = torch.full((rows + 2, ld), SENT16, dtype=torch.int16, device=DEV).view(torch.bfloat16)
        if data is not None:
            self.t[1:1 + data.shape[0], :data.shape[1]] = data.to(self.t.dtype)

    @property
    def ptr(self):
        return self.t.data_ptr() + self.ld * self.t.element_size()

    def snap(self):
        return self.t.clone()


def bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


@dataclass
class Ph:
    """One GEMV phase: weight [N][K] (bf16, and packed), input / output buffers by name."""
    N: int
    K: int
    epi: int
    src: str
    dst: str
    ncmode: int = 0
    norm: object = None         # bf16 [K] tensor
    bias: object = None         # bf16 [N] tensor
    save: str = None
    W: object = None            # bf16 [N][K]
    Wp: object = None           # packed
    exact: bool = True


def rnd_int(g, shape, lo, hi):
    return torch.randint(lo, hi + 1, shape, generator=g).bfloat16()


def make_weight(g, N, K, grid=True, swiglu=False):
    if grid:
        W = rnd_int(g, (N, K), -2, 2)
    else:
        W = (torch.randn(N, K, generator=g) * 0.05).bfloat16()
    if swiglu:   # gate / up through the engine's interleave
        W = AREngine._gate_up_blk8(W[:N // 2], W[N // 2:])
    return W.to(DEV)


def pack(L, W):
    N, K = W.shape
    Wp = torch.empty(N * K // 8, 4, dtype=torch.int32, device=DEV)
    assert L.gemv_shim_pack(W.data_ptr(), Wp.data_ptr(), N, K, None) == 0, err(L)
    return Wp


def grid_input(g, nc, K, normed, c=3.0):
    if normed:
        return ((torch.randint(0, 2, (nc, K), generator=g) * 2 - 1) * c).bfloat16()
    return rnd_int(g, (nc, K), -3, 3)


def rand_input(g, nc, K):
    return torch.randn(nc, K, generator=g).bfloat16()


def norm_weight(g, K, grid=True):
    if grid:
        v = torch.randint(1, 3, (K,), generator=g) * (torch.randint(0, 2, (K,), generator=g) * 2 - 1)
        return v.bfloat16().to(DEV)
    return (1 + 0.2 * torch.randn(K, generator=g)).bfloat16().to(DEV)


def out_rows(p):
    return p.N // 2 if p.epi == R.EPI_SWIGLU else p.N


def nc_of(p, B):
    return B if p.ncmode == 0 else 2 * B


# ================================================================================================ launch
def run(L, phases, bufs, B, nt, grid=None, var=0, mode=0, max_iters=1, admit=0xFFFFFFFF, frame0=None, hid=None,
        hid_stride=0, cap=0, step0=0, expect_ok=True):
    n = len(phases)
    grid = grid or L.sms
    arr = lambda T, v: (T * n)(*v)  # noqa: E731
    ptrs = lambda v: (C.c_void_p * n)(*v)  # noqa: E731
    st = torch.zeros(L.lay["sizeof_state"], dtype=torch.uint8)
    st.view(torch.int32)[L.lay["step"] // 4] = step0
    L.state.copy_(st.to(DEV))
    f0 = (C.c_int * 32)(*((frame0 or []) + [0] * (32 - len(frame0 or []))))
    torch.cuda.synchronize()
    rc = L.gemv_shim_run(
        n, ptrs([p.Wp.data_ptr() for p in phases]), arr(C.c_int, [p.N for p in phases]), arr(C.c_int, [p.K for p in phases]),
        ptrs([bufs[p.src].ptr for p in phases]), arr(C.c_int, [bufs[p.src].ld for p in phases]),
        ptrs([p.norm.data_ptr() if p.norm is not None else None for p in phases]), arr(C.c_float, [EPS] * n),
        ptrs([bufs[p.dst].ptr for p in phases]), arr(C.c_int, [bufs[p.dst].ld for p in phases]),
        arr(C.c_int, [p.epi for p in phases]), arr(C.c_int, [p.ncmode for p in phases]),
        ptrs([p.bias.data_ptr() if p.bias is not None else None for p in phases]),
        ptrs([bufs[p.save].ptr if p.save else None for p in phases]),
        grid, B, nt, var, mode, max_iters, admit, f0, hid.ptr if hid is not None else None, hid_stride, cap,
        L.prog.data_ptr(), L.prog.numel(), L.runs.data_ptr(), L.runs.numel(), L.off.data_ptr(), L.off.numel(),
        L.state.data_ptr(), None)
    if not expect_ok:
        return rc
    assert rc == 0, err(L)
    torch.cuda.synchronize()
    STATS["launches"] += 1
    stv = L.state.cpu().view(torch.int32)
    assert int(stv[L.lay["error"] // 4]) == 0
    return int(stv[L.lay["step"] // 4])


def plan(L, phases, B, nt, cap=0):
    n = len(phases)
    staged, out = (C.c_int * n)(), (C.c_int * 4)()
    rc = L.gemv_shim_plan(n, (C.c_int * n)(*[p.N for p in phases]), (C.c_int * n)(*[p.K for p in phases]),
                          (C.c_int * n)(*[int(p.norm is not None) for p in phases]),
                          (C.c_int * n)(*[p.ncmode for p in phases]), B, nt, cap, staged, out)
    assert rc == 0, err(L)
    return list(staged), dict(sb=out[0], r=out[1], total=out[2], x=out[3])


# ================================================================================================ geometry restatement
def geometry(p, B, nt, grid, staged, sb):
    """Which properties the phase reaches: a restatement of cta_tiles / run_geom and the consumer's piece walk."""
    hit = set()
    n_tiles, KB = p.N // 16, p.K // 32
    tq, tr = divmod(n_tiles, grid)
    nc = nc_of(p, B)
    PB = 2 if nt == 4 else 4
    if tq == 0:
        hit.add("idle_cta")
    if tr:
        hit.add("tr_edge")
    if KB < sb:
        hit.add("kb_lt_sb")
    if (nc + 7) // 8 < nt:
        hit.add("nct_lt_nt")
    all_full = True
    rsh = 3 if p.epi == R.EPI_SWIGLU else 4
    for ntc in {tq, tq + 1} if tr else {tq}:
        if ntc == 0:
            continue
        if ntc > 8:
            hit.add("multi_round")
        rounds = (ntc + 7) // 8
        for rd in range(rounds):
            TB = min(8, ntc - 8 * rd)
            if rd == rounds - 1 and rd > 0 and TB in (3, 5):
                hit.add(f"partial_round_{TB}")
            tbl = max(0, (TB - 1).bit_length())
            if p.epi == R.EPI_RESID and (nc << (rsh + tbl)) > 2 * NTHREADS:
                hit.add("resid_loaded")
            units = TB * KB
            upw = (units + 7) >> 3
            for w in range(NWARPS):
                u0 = min(units, w * upw)
                u1 = min(units, u0 + upw)
                if u1 <= u0:
                    hit.add("empty_warp")
                    continue
                if (u1 - 1) // KB != u0 // KB:
                    hit.add("run_two_tiles")
                u, kbi = u0, u0 % KB
                while u < u1:
                    nb = min(sb, u1 - u)
                    full = nb == sb and nb in (PB, 2) and kbi + nb <= KB
                    if not full:
                        all_full = False
                        hit.add("general_path")
                    if not staged and u + nb < u1 and kbi + nb >= KB:
                        hit.add("unstaged_wrap")
                    kbi = (kbi + nb) % KB
                    u += nb
    return hit, all_full


def record(p, B, nt, grid, staged, pl):
    hit, all_full = geometry(p, B, nt, grid, staged, pl["sb"])
    hit.add(f"nt{nt}")
    hit.add(["epi_store", "epi_bias", "epi_resid", "epi_swiglu", "epi_logits"][p.epi])
    if p.ncmode == 1:
        hit.add("nc2b")
    hit.add("unstaged" if not staged else "staged_normed" if p.norm is not None else "staged_tma")
    if pl["sb"] == 2:
        hit.add("ring_sb2")
    if pl["sb"] == 1:
        hit.add("ring_sb1")
    if pl["r"] == 2:
        hit.add("ring_r2")
    for h in hit:
        HIT[h] += 1
    return all_full


# ================================================================================================ checks
def check_phase(p, B, before, after, bufs, admit=0xFFFFFFFF, grid_data=True, sens=True):
    """The phase's output against the reference; guards of dst (and save) untouched."""
    nc, rows, K = nc_of(p, B), out_rows(p), p.K
    x = before[p.src][1:1 + nc, :K].double()
    resid = before[p.dst][1:1 + nc, :rows].double().cpu().numpy() if p.epi == R.EPI_RESID else None
    xk = None
    if p.save:
        mask = np.array([(admit >> c) & 1 for c in range(nc)], bool)
        sv = after[p.save][1:1 + nc, :K].double().cpu().numpy()
        xn, _ = R.normed_input(x.cpu().numpy(), p.norm.double().cpu().numpy(), EPS)
        near = R.normed_boundary_mask(x.cpu().numpy(), p.norm.double().cpu().numpy(), EPS)
        d = (sv != xn)[mask]
        assert not (d & ~near[mask]).any(), "saved normed input differs away from a rounding boundary"
        if grid_data:
            assert not d.any()
        STATS["normed_near_boundary"] += int(near[mask].sum())
        STATS["normed_differs"] += int(d.sum())
        sg = bits(after[p.save]).clone()
        sg[1:1 + nc][torch.from_numpy(mask).to(DEV), :K] = SENT16
        assert (sg == SENT16).all(), "save_normed written outside the admitted columns"
        if not grid_data and mask.all():
            xk = sv
    lo, hi, _ = R.gemv(p.W.double(), x, p.epi, norm_w=None if p.norm is None else p.norm.double(), eps=EPS,
                       bias=p.bias, resid=resid, exact=grid_data, x_kernel=xk)
    out = after[p.dst][1:1 + nc, :rows].double().cpu().numpy()
    ok = (lo <= out) & (out <= hi)
    assert ok.all(), f"phase N={p.N} K={p.K} epi={p.epi}: {int((~ok).sum())} outputs outside the reference, first at " \
                     f"{np.argwhere(~ok)[0]}: {out[~ok][0]} not in [{lo[~ok][0]}, {hi[~ok][0]}]"
    two = int((lo != hi).sum())
    if grid_data:
        if p.epi == R.EPI_SWIGLU:
            STATS["swiglu_two_valued"] += two
            assert two <= max(2, out.size // 1000)
        else:
            assert two == 0
    else:
        STATS["general_two_valued"] += two
        HIT["general_inputs"] += 1
    STATS["outputs"] += out.size
    g = bits(after[p.dst]).clone()
    g[1:1 + nc, :rows] = bits(before[p.dst])[1:1 + nc, :rows]
    assert torch.equal(g, bits(before[p.dst])), "dst written outside [nc][rows]"
    if grid_data and sens:
        n_tiles, KB = p.N // 16, p.K // 32
        nrm = None if p.norm is None else p.norm.double()
        kw = dict(norm_w=nrm, eps=EPS, bias=p.bias, resid=resid)
        muts = [dict(drop=(n_tiles - 1, KB - 1)), dict(swap_halves=True)]
        if p.epi == R.EPI_SWIGLU:
            muts.append(dict(swap_gate_up=True))
        for m in muts:
            ml, mh, _ = R.gemv(p.W.double(), x, p.epi, **kw, **m)
            assert not np.array_equal(ml, out), f"the data cannot see the mutation {m}"


def fresh(bufs, inits):
    for k, v in inits.items():
        bufs[k].t.copy_(v)


def snap(bufs):
    return {k: b.snap() for k, b in bufs.items()}


def single_phase_case(L, g, N, K, epi, normed, B, nt, grid=None, ncmode=0, grid_data=True, save=False, cap=0,
                      src_pad=16, dst_pad=16, admit=0xFFFFFFFF, var=0):
    """Build, plan, launch and check one phase; returns (phase, bufs, after, plan)."""
    nc = B if ncmode == 0 else 2 * B
    p = Ph(N, K, epi, "x", "y", ncmode=ncmode, exact=grid_data)
    p.W = make_weight(g, N, K, grid_data, swiglu=epi == R.EPI_SWIGLU)
    p.Wp = pack(L, p.W)
    if normed:
        p.norm = norm_weight(g, K, grid_data)
    if epi == R.EPI_BIAS:
        p.bias = rnd_int(g, (N,), -9, 9).to(DEV) if grid_data else (torch.randn(N, generator=g) * 0.1).bfloat16().to(DEV)
    x = (grid_input(g, nc, K, normed) if grid_data else rand_input(g, nc, K)).to(DEV)
    rows = out_rows(p)
    bufs = {"x": Buf(nc, K + src_pad, data=x), "y": Buf(nc, rows + dst_pad, f32=epi == R.EPI_LOGITS)}
    if epi == R.EPI_RESID:
        r = rnd_int(g, (nc, rows), -40, 40) if grid_data else torch.randn(nc, rows, generator=g).bfloat16()
        bufs["y"].t[1:1 + nc, :rows] = r.to(DEV)
    if save:
        p.save = "s"
        bufs["s"] = Buf(nc, K)
    staged, pl = plan(L, [p], B, nt, cap)
    record(p, B, nt, grid or L.sms, staged[0], pl)
    before = snap(bufs)
    run(L, [p], bufs, B, nt, grid=grid, cap=cap, admit=admit, var=var)
    after = snap(bufs)
    check_phase(p, B, before, after, bufs, admit=admit, grid_data=grid_data)
    STATS["cases"] += 1
    return p, bufs, before, after, pl, staged[0]


# ================================================================================================ 1. geometry
GEOM_KB = [1, 2, 3, 5, 7, 8, 9, 33, 64]


def geom_cases(S):
    out = []
    for grid in (1, 2, 7, S - 1, S):
        tiles = sorted({max(1, grid - 1), grid, grid + 1, 11 * grid, 13 * grid + 1})
        kbs = GEOM_KB if grid <= 7 else [1, 3, 8, 9]
        for nt_ in tiles:
            for kb in kbs:
                if nt_ * 16 * kb * 32 > (1 << 25):   # keep each weight under 64 MB
                    continue
                out.append((grid, nt_, kb))
    return out


def test_geometry_grid_tiles_and_k_blocks(lib):
    g = torch.Generator().manual_seed(10)
    cases = geom_cases(lib.sms)
    for i, (grid, n_tiles, kb) in enumerate(cases):
        B = 1 if i % 2 == 0 else 3
        single_phase_case(lib, g, n_tiles * 16, kb * 32, R.EPI_STORE, False, B, 1, grid=grid)
    print(f"geometry: {len(cases)} cases")


# ================================================================================================ 2. batch classes
def test_batch_classes_and_column_counts(lib):
    g = torch.Generator().manual_seed(11)
    N, K = 16 * 37, 32 * 24
    W = make_weight(g, N, K)
    Wp = pack(lib, W)
    X = grid_input(g, 32, K, False).to(DEV)
    ref_cols = None
    n = 0
    for nt in (1, 2, 4):
        for nc in (1, 7, 8, 9, 16, 17, 31, 32):
            if nc > 8 * nt:
                continue
            for ncmode in ((0, 1) if nc % 2 == 0 else (0,)):
                B = nc if ncmode == 0 else nc // 2
                p = Ph(N, K, R.EPI_STORE, "x", "y", ncmode=ncmode, W=W, Wp=Wp)
                bufs = {"x": Buf(nc, K + 8, data=X[:nc]), "y": Buf(nc, N + 8)}
                staged, pl = plan(lib, [p], B, nt)
                record(p, B, nt, lib.sms, staged[0], pl)
                before = snap(bufs)
                run(lib, [p], bufs, B, nt)
                after = snap(bufs)
                check_phase(p, B, before, after, bufs)
                out = after["y"][1:1 + nc, :N]
                if ref_cols is None:
                    ref_cols = torch.zeros(32, N, dtype=torch.bfloat16, device=DEV)
                    ref_cols.view(torch.int16).fill_(SENT16)
                known = bits(ref_cols[:nc]) != SENT16
                assert torch.equal(bits(out)[known], bits(ref_cols[:nc])[known]), "columns differ across batch classes"
                ref_cols[:nc] = out
                n += 1
                STATS["cases"] += 1
    print(f"batch classes: {n} cases")


# ================================================================================================ 3. input paths + 4. epilogues
def test_input_paths(lib):
    g = torch.Generator().manual_seed(12)
    for B, nt, K, normed, want_staged in [(4, 1, 512, True, 1), (8, 1, 1024, True, 1), (5, 1, 768, False, 1),
                                          (16, 2, 2080, False, 0), (1, 1, 6144, False, 0), (12, 2, 6144, False, 0),
                                          (32, 4, 2048, True, 1), (32, 4, 4096, False, 0)]:
        *_, staged = single_phase_case(lib, g, 16 * 40, K, R.EPI_STORE, normed, B, nt, save=normed)
        assert staged == want_staged, (B, nt, K, staged)
    # un-staged runs that cross a tile boundary (3 tiles per CTA): the B-fragment prefetch wraps to k-block 0
    for B, nt, K, grid in [(16, 2, 2080, 3), (1, 1, 6144, 2)]:
        *_, staged = single_phase_case(lib, g, 16 * 3 * grid, K, R.EPI_STORE, False, B, nt, grid=grid)
        assert staged == 0
    # two normed staged phases in one launch: the TMA x barrier's parity flips over consecutive un-normed phases
    ps = []
    bufs = {}
    for i in range(4):
        K = 256 + 64 * i
        p = Ph(16 * 20, K, R.EPI_STORE, f"x{i}", f"y{i}")
        p.W = make_weight(g, p.N, K)
        p.Wp = pack(lib, p.W)
        if i % 2 == 0:
            p.norm = norm_weight(g, K)
        bufs[f"x{i}"] = Buf(3, K, data=grid_input(g, 3, K, p.norm is not None).to(DEV))
        bufs[f"y{i}"] = Buf(3, p.N)
        ps.append(p)
    before = snap(bufs)
    run(lib, ps, bufs, 3, 1)
    after = snap(bufs)
    for p in ps:
        check_phase(p, 3, before, after, bufs)


@pytest.mark.parametrize("epi", [R.EPI_STORE, R.EPI_BIAS, R.EPI_RESID, R.EPI_SWIGLU, R.EPI_LOGITS])
def test_epilogues_on_grid_and_general_inputs(lib, epi):
    g = torch.Generator().manual_seed(20 + epi)
    for grid_data in (True, False):
        for B, nt, N, K, normed, grid in [(1, 1, 16 * 300, 1024, True, None), (8, 1, 16 * 64, 512, False, 7),
                                          (13, 2, 16 * 200, 2048, True, None), (32, 4, 16 * 48, 3072, False, 5),
                                          (16, 2, 16 * 24, 2080, False, 3)]:
            if epi == R.EPI_BIAS and normed:
                normed = False
            single_phase_case(lib, g, N, K, epi, normed, B, nt, grid=grid, grid_data=grid_data,
                              save=normed and not grid_data)


# ================================================================================================ 5. ring fallbacks
def test_ring_fallbacks_are_bit_identical(lib):
    g = torch.Generator().manual_seed(30)
    for B, nt, N, K, normed, epi in [(2, 1, 16 * 90, 1024, True, R.EPI_SWIGLU), (16, 2, 16 * 70, 2080, False, R.EPI_RESID),
                                     (32, 4, 16 * 50, 2048, True, R.EPI_STORE)]:
        p, bufs, before, after, pl0, _ = single_phase_case(lib, g, N, K, epi, normed, B, nt)
        default = after["y"]
        found = {}
        cap = lib.lay["max_dyn_smem"]
        while cap > 20 * 1024 and len(found) < 3:
            cap -= 1024
            try:
                st, pl = plan(lib, [p], B, nt, cap)
            except AssertionError:
                break
            for key, ok in (("sb2", pl["sb"] == 2), ("sb1", pl["sb"] == 1), ("r2", pl["r"] == 2)):
                if ok and key not in found:
                    found[key] = cap
        assert {"sb2", "sb1", "r2"} <= set(found), found
        for key, c in found.items():
            st, pl = plan(lib, [p], B, nt, c)
            record(p, B, nt, lib.sms, st[0], pl)
            fresh(bufs, before)
            run(lib, [p], bufs, B, nt, cap=c)
            assert torch.equal(bits(bufs["y"].t), bits(default)), f"ring fallback {key} (cap {c}) differs"
            STATS["cases"] += 1


# ================================================================================================ 6. programs
def layer_chain(L, g, B, nt, H=512, A=1024, I=2080, V=1024):
    bufs = {"h": Buf(B, H, data=grid_input(g, B, H, True).to(DEV)), "qkv": Buf(B, 2 * A + 8),
            "attn": Buf(B, A, data=grid_input(g, B, A, False).to(DEV)), "act": Buf(B, I), "logits": Buf(B, V + 8, f32=True),
            "s1": Buf(B, H), "s2": Buf(B, H), "s3": Buf(B, H)}
    spec = [(2 * A, H, R.EPI_STORE, "h", "qkv", True, "s1"), (H, A, R.EPI_RESID, "attn", "h", False, None),
            (2 * I, H, R.EPI_SWIGLU, "h", "act", True, "s2"), (H, I, R.EPI_RESID, "act", "h", False, None),
            (V, H, R.EPI_LOGITS, "h", "logits", True, "s3")]
    ps = []
    for N, K, epi, src, dst, normed, save in spec:
        p = Ph(N, K, epi, src, dst, save=save, exact=False)
        p.W = make_weight(g, N, K, True, swiglu=epi == R.EPI_SWIGLU)
        p.W = (p.W.float() * (0.25 if K > 1024 else 1.0)).bfloat16()   # keep the chain's sums in a sane range
        p.Wp = pack(L, p.W)
        if normed:
            p.norm = norm_weight(g, K)
        ps.append(p)
    return ps, bufs


def test_layer_chain_in_one_launch_equals_one_launch_per_phase(lib):
    g = torch.Generator().manual_seed(40)
    B, nt = 16, 2
    ps, bufs = layer_chain(lib, g, B, nt)
    st, pl = plan(lib, ps, B, nt)
    assert st == [1, 1, 1, 0, 1], st
    init = snap(bufs)
    run(lib, ps, bufs, B, nt)
    chain = snap(bufs)
    fresh(bufs, init)
    for p in ps:
        before = snap(bufs)
        run(lib, [p], bufs, B, nt)
        after = snap(bufs)
        # the chain's later inputs are no longer grid data: the general bound over the kernel's own saved operand
        check_phase(p, B, before, after, bufs, grid_data=p is ps[0])
    for k in bufs:
        assert torch.equal(bits(bufs[k].t), bits(chain[k])), f"buffer {k}: one launch differs from one launch per phase"
    HIT["chain"] += 1
    STATS["cases"] += 1


def test_mode1_applies_the_program_max_iters_times(lib):
    g = torch.Generator().manual_seed(41)
    B, nt = 3, 1
    p = Ph(16 * 150, 768, R.EPI_RESID, "x", "y")
    p.W = make_weight(g, p.N, p.K)
    p.Wp = pack(lib, p.W)
    bufs = {"x": Buf(B, p.K, data=grid_input(g, B, p.K, False).to(DEV)), "y": Buf(B, p.N)}
    bufs["y"].t[1:1 + B, :p.N] = rnd_int(g, (B, p.N), -40, 40).to(DEV)
    init = snap(bufs)
    step = run(lib, [p], bufs, B, nt, mode=1, max_iters=3, step0=5)
    assert step == 8, "DevState.step must advance by max_iters"
    looped = snap(bufs)
    fresh(bufs, init)
    for _ in range(3):
        before = snap(bufs)
        run(lib, [p], bufs, B, nt)
        after = snap(bufs)
        check_phase(p, B, before, after, bufs, sens=False)
    assert torch.equal(bits(bufs["y"].t), bits(looped["y"]))
    # the same launch repeated gives identical bits
    fresh(bufs, init)
    run(lib, [p], bufs, B, nt, mode=1, max_iters=3)
    assert torch.equal(bits(bufs["y"].t), bits(looped["y"]))
    HIT["mode1"] += 1
    STATS["cases"] += 1


# ================================================================================================ 7. VAR = 1
def test_saved_and_captured_hidden_states(lib):
    g = torch.Generator().manual_seed(50)
    B, nt, K, N = 6, 1, 1024, 16 * 64
    p = Ph(N, K, R.EPI_LOGITS, "x", "y", save="s")
    p.W = make_weight(g, N, K)
    p.Wp = pack(lib, p.W)
    p.norm = norm_weight(g, K)
    x = grid_input(g, B, K, True).to(DEV)
    mk = lambda: {"x": Buf(B, K, data=x), "y": Buf(B, N + 8, f32=True), "s": Buf(B, K)}  # noqa: E731
    # mode 0, admit_mask a subset: only those columns are saved; VAR 0 and VAR 1 write identical dst bits
    outs = []
    for var in (0, 1):
        bufs = mk()
        hs = 2
        hid = Buf(B * hs, K)
        before = snap(bufs)
        run(lib, [p], bufs, B, nt, var=var, admit=0b101001, hid=hid if var else None, hid_stride=hs if var else 0,
            frame0=[0, 0, 0, -1, 0, 0])
        after = snap(bufs)
        check_phase(p, B, before, after, bufs, admit=0b101001)
        outs.append(after["y"])
        if var:   # mode 0: step 0 - frame0[col], captured only for admitted columns inside [0, hid_stride)
            want = torch.full_like(bits(hid.t), SENT16)
            for c in range(B):
                st_ = 0 - [0, 0, 0, -1, 0, 0][c]
                if (0b101001 >> c) & 1 and 0 <= st_ < hs:
                    want[1 + c * hs + st_] = bits(after["s"])[1 + c]
            assert torch.equal(bits(hid.t), want), "hidden capture of mode 0 wrong or out of range"
    assert torch.equal(bits(outs[0]), bits(outs[1])), "VAR 0 and VAR 1 write different dst bits"
    # mode 1 with per-column frame0: step index = frame + 1 - frame0[col], rows outside [0, hid_stride) untouched
    hs, frame0 = 3, [0, -2, 2, 1, 3, -1]
    bufs = mk()
    hid = Buf(B * hs, K)
    run(lib, [p], bufs, B, nt, var=1, mode=1, max_iters=3, hid=hid, hid_stride=hs, frame0=frame0)
    saved = bits(bufs["s"].t)
    want = torch.full_like(bits(hid.t), SENT16)
    n_cap = 0
    for c in range(B):
        for f in range(3):
            s = f + 1 - frame0[c]
            if 0 <= s < hs:
                want[1 + c * hs + s] = saved[1 + c]
                n_cap += 1
    assert n_cap >= 6 and torch.equal(bits(hid.t), want), "hidden capture of mode 1 wrong or out of range"
    HIT["var1_capture"] += 1
    STATS["cases"] += 1


# ================================================================================================ 8. production shapes
def production_phases(cfg, B):
    t, c = cfg.talker, cfg.cp
    joint = 2 * B <= 32
    cols = 2 * B if joint else B
    nt_frame = 1 if cols <= 8 else 2 if cols <= 16 else 4
    nt_head = 1 if B <= 8 else 2 if B <= 16 else 4
    frame = []
    for s, stack_nc in ((c, 1 if joint else 0), (t, 0)):
        qkv = (s.num_heads + 2 * s.num_kv_heads) * 128
        for ncm in sorted({stack_nc, 0}):
            frame += [(qkv, s.hidden_size, R.EPI_STORE, True, ncm), (s.hidden_size, s.num_heads * 128, R.EPI_RESID, False, ncm),
                      (2 * s.intermediate_size, s.hidden_size, R.EPI_SWIGLU, True, ncm),
                      (s.hidden_size, s.intermediate_size, R.EPI_RESID, False, ncm)]
    frame += [(c.vocab_size, c.hidden_size, R.EPI_LOGITS, True, 0), (t.vocab_size, t.hidden_size, R.EPI_LOGITS, True, 0)]
    return nt_frame, frame, nt_head, [(t.vocab_size, t.hidden_size, R.EPI_LOGITS, True, 0)]


@pytest.mark.parametrize("model", ["1p7b", "0p6b"])
def test_production_shapes(lib, model):
    cfg = synthetic.cfg_1p7b() if model == "1p7b" else synthetic.cfg_0p6b()
    g = torch.Generator().manual_seed(60)
    n = 0
    for B in (1, 8, 32):
        nt_frame, frame, nt_head, head = production_phases(cfg, B)
        for nt, spec in ((nt_frame, frame), (nt_head, head)):
            ps, bufs = [], {}
            for i, (N, K, epi, normed, ncm) in enumerate(spec):
                nc = B if ncm == 0 else 2 * B
                p = Ph(N, K, epi, f"x{i}", f"y{i}", ncmode=ncm, save=f"s{i}" if epi == R.EPI_LOGITS else None)
                p.W = make_weight(g, N, K, swiglu=epi == R.EPI_SWIGLU)
                p.Wp = pack(lib, p.W)
                if normed:
                    p.norm = norm_weight(g, K)
                bufs[p.src] = Buf(nc, K, data=grid_input(g, nc, K, normed).to(DEV))
                bufs[p.dst] = Buf(nc, out_rows(p), f32=epi == R.EPI_LOGITS)
                if epi == R.EPI_RESID:
                    bufs[p.dst].t[1:1 + nc, :N] = rnd_int(g, (nc, N), -40, 40).to(DEV)
                if p.save:
                    bufs[p.save] = Buf(nc, K)
                ps.append(p)
            st, pl = plan(lib, ps, B, nt)
            for p, s in zip(ps, st):
                assert record(p, B, nt, lib.sms, s, pl), f"production phase {p.N}x{p.K} takes the general path"
            before = snap(bufs)
            run(lib, ps, bufs, B, nt)
            after = snap(bufs)
            for p in ps:
                check_phase(p, B, before, after, bufs)
                n += 1
            del ps, bufs, before, after
    HIT["production_full_piece"] += n
    STATS["cases"] += n
    print(f"production {model}: {n} phases checked")


# ================================================================================================ 9. refusals
def test_refusals_launch_nothing(lib):
    g = torch.Generator().manual_seed(70)
    B, nt = 4, 1

    def base(N=160, K=256, normed=False):
        p = Ph(N, K, R.EPI_STORE, "x", "y")
        p.W = make_weight(g, N, K)
        p.Wp = pack(lib, p.W)
        if normed:
            p.norm = norm_weight(g, K)
        return p, {"x": Buf(2 * B, K + 8, data=grid_input(g, 2 * B, K, normed).to(DEV)), "y": Buf(2 * B, N + 8)}

    def refused(why, p, bufs, **kw):
        before = snap(bufs)
        rc = run(lib, [p], bufs, kw.pop("B", B), kw.pop("nt", nt), expect_ok=False, **kw)
        torch.cuda.synchronize()
        assert rc == 1, f"{why}: accepted"
        msg = err(lib)
        assert all(torch.equal(bits(bufs[k].t), bits(before[k])) for k in bufs), f"{why}: something was written"
        return msg

    p, bufs = base()
    assert "grid" in refused("grid above the SM count", p, bufs, grid=lib.sms + 1)
    p2 = Ph(p.N, p.K, p.epi, "x", "y", ncmode=1, W=p.W, Wp=p.Wp)
    assert "nt < ceil(nc/8)" in refused("nt below ceil(nc/8)", p2, bufs, B=5, nt=1)
    p3 = Ph(152, p.K, p.epi, "x", "y", W=p.W, Wp=p.Wp)
    assert "multiple of 16" in refused("N % 16", p3, bufs)
    p4 = Ph(p.N, 240, p.epi, "x", "y", W=p.W, Wp=p.Wp)
    assert "multiple of 32" in refused("K % 32", p4, bufs)
    pn, bn = base(K=2080, normed=False)
    pn.norm = norm_weight(g, 2080)
    assert "2048" in refused("normed K > 2048", pn, bn)
    bufs["x"].ld = p.K + 4   # rows no longer 16-byte aligned
    assert "src" in refused("unaligned source rows", p, bufs)
    bufs["x"].ld = p.K + 8
    bad = Ph(p.N, p.K, p.epi, "x", "y", W=p.W, Wp=p.Wp.view(torch.uint8).flatten()[8:])
    assert "aligned" in refused("unaligned weight pointer", bad, bufs)
    pb, bb = base(N=16 * 64, K=2048, normed=True)
    assert "shared" in refused("a plan that does not fit", pb, bb, cap=40 * 1024)
    STATS["cases"] += 8


# ================================================================================================ coverage
def test_zz_every_property_was_hit(lib):
    wall = time.time() - T0[0] if T0[0] else float("nan")
    print("gemv coverage: " + ", ".join(f"{k}={v}" for k, v in HIT.items()))
    print("gemv stats: " + ", ".join(f"{k}={v}" for k, v in STATS.items()) + f", wall {wall:.1f} s")
    missing = [k for k, v in HIT.items() if v == 0]
    assert not missing, f"properties never reached: {missing}"
