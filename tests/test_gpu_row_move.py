"""The parked-row kernel (row_move_kernel, ar_prefill.cuh) directly, through tests/csrc/park_shim.cu: a park gathers
exactly a row's K/V positions [0, pos) into the registered-prefix layout, every span and the row's DevState fields,
then marks the row finished as a release does; a resume scatters them back and touches nothing else — at one block and
at a grid that strides over every piece, and for a row that had already finished."""
import ctypes as C
import os
import subprocess

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM_SRC = os.path.join(ROOT, "tests", "csrc", "park_shim.cu")
HD = 128


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    """tests/csrc/park_shim.cu compiled for sm_90a with the library's flags; it links against nothing."""
    from qwen3_tts_b200 import build
    out = str(tmp_path_factory.mktemp("park_shim") / "libpark_shim.so")
    cmd = [build._nvcc()] + build.NVCC_FLAGS + ["-shared", "-I", build.CSRC, SHIM_SRC, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"shim build failed:\n{r.stdout}\n{r.stderr}"
    L = C.CDLL(out)
    L.park_shim_state.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int)]
    L.park_shim_row_move.argtypes = [C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    return L


def _state(L, slot, vals=None):
    n = L.park_shim_row_ints()
    buf = (C.c_int * n)(*(vals or [0] * n))
    assert L.park_shim_state(int(vals is not None), slot, buf) == 0
    return list(buf)


def _move(L, resume, slots, recs, kc, vc, kv, lh, pos, slot, ints, grid):
    n = len(slots)
    sp = (C.c_void_p * n)(*[t.data_ptr() for t in slots])
    rp = (C.c_void_p * n)(*[t.data_ptr() for t in recs])
    ch = (C.c_int * n)(*[t.numel() // 16 for t in slots])
    rc = L.park_shim_row_move(resume, sp, rp, ch, kc.data_ptr(), vc.data_ptr(), kv.data_ptr(), lh, kc.shape[2], pos, slot,
                              ints.data_ptr(), grid, None)
    assert rc == 0
    torch.cuda.synchronize()


@pytest.mark.parametrize("grid", [1, 37])
@pytest.mark.parametrize("finished", [0, 1])
def test_park_then_resume_moves_exactly_the_row(shim, grid, finished):
    L = shim
    nr, ns = L.park_shim_row_ints(), L.park_shim_row_spans()
    g = torch.Generator(device=DEV).manual_seed(grid + 10 * finished)
    seqs, lh, cap, pos, slot = 5, 6, 40, 27, 3
    kc = torch.randn(seqs, lh, cap, HD, generator=g, device=DEV).bfloat16()
    vc = torch.randn(seqs, lh, cap, HD, generator=g, device=DEV).bfloat16()
    kv = torch.full((2, lh, pos, HD), float("nan"), device=DEV).bfloat16()
    sizes = [3, 5, 0, 7, 11, 2][:ns]   # 16-byte chunks of each span; an empty span (no trailing text) included
    slots = [torch.randint(0, 256, (16 * n,), generator=g, device=DEV, dtype=torch.uint8) for n in sizes]
    recs = [torch.zeros(16 * n, dtype=torch.uint8, device=DEV) for n in sizes]
    ints = torch.zeros(nr, dtype=torch.int32, device=DEV)
    vals = [int(v) for v in torch.randint(1, 1 << 20, (nr,), generator=g, device=DEV)]
    vals[1] = finished
    _state(L, slot, vals)
    other = [int(v) for v in torch.randint(1, 1 << 20, (nr,), generator=g, device=DEV)]
    _state(L, slot + 1, other)
    kc0, vc0 = kc.clone(), vc.clone()

    _move(L, 0, slots, recs, kc, vc, kv, lh, pos, slot, ints, grid)      # park
    assert torch.equal(kv[0], kc[slot, :, :pos]) and torch.equal(kv[1], vc[slot, :, :pos])
    assert all(torch.equal(r, s) for r, s in zip(recs, slots))
    assert ints.tolist() == vals
    after = list(vals)
    if not finished:
        after[1], after[2] = 1, 0x3fffffff        # finished as release_state_kernel leaves it
    assert _state(L, slot) == after and _state(L, slot + 1) == other
    assert torch.equal(kc, kc0) and torch.equal(vc, vc0)

    saved = [s.clone() for s in slots]
    for s in slots:
        s.zero_()
    kc[slot].zero_()
    vc[slot].zero_()
    _state(L, slot, [0] * nr)
    _move(L, 1, slots, recs, kc, vc, kv, lh, pos, slot, ints, grid)      # resume
    assert torch.equal(kc[slot, :, :pos], kc0[slot, :, :pos]) and torch.equal(vc[slot, :, :pos], vc0[slot, :, :pos])
    assert not kc[slot, :, pos:].any() and not vc[slot, :, pos:].any()  # past the row's positions: untouched
    others = [b for b in range(seqs) if b != slot]
    assert torch.equal(kc[others], kc0[others]) and torch.equal(vc[others], vc0[others])
    assert all(torch.equal(s, v) for s, v in zip(slots, saved))
    assert _state(L, slot) == vals and _state(L, slot + 1) == other
