"""The streaming limiter's kernels run directly (tests/csrc/limit_shim.cu) on rows, histories and counters chosen here,
against the numpy restatement (tests/limiter_ref.py), bit for bit: whole clips ended in one launch (random, planted
peaks, silence, 0 … 1700 samples across the 256-output tile edges) with rows that have no work beside them; rows
resumed mid-clip from a history at its deepest read, with their next history half; save / load records."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import audio_shims
from tests import limiter_ref as LR

pytestmark = pytest.mark.gpu
HIST = audio_shims.LIMIT_HIST
DEV = "cuda:0"


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return audio_shims.load(tmp_path_factory, "limit_shim")


def _arr(t, xs):
    return (t * len(xs))(*xs)


class Rows:
    """Device state of `rows` limiter rows (double-buffered history) and one launch helper."""

    def __init__(self, rows, cap=8192):
        self.rows, self.cap = rows, cap
        self.hist = torch.zeros(2, rows, HIST, device=DEV)
        self.out = torch.zeros(rows, cap, device=DEV)

    def launch(self, lib, jobs, x, cur=None):
        """jobs: {row: (n_in, count, end, gain)}, other rows idle; the output counts follow the host formulas.
        Returns {row: its outputs}."""
        n_in, out0, fields, gains, nouts = [], [], [], [], {}
        for r in range(self.rows):
            n0, c, end, g = jobs.get(r, (0, 0, False, 1.0))
            e0 = LR.emitted(n0)
            nout = ((n0 + c) if end else LR.emitted(n0 + c)) - e0 if (c or end) else 0
            n_in.append(n0)
            out0.append(e0)
            fields += [c, nout, int(end), 0 if cur is None else cur[r]]
            gains.append(float(g))
            if r in jobs:
                nouts[r] = nout
        xd = torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(DEV)
        self.out.zero_()
        rc = lib.limit_shim_step(self.rows, _arr(C.c_longlong, n_in), _arr(C.c_longlong, out0), _arr(C.c_int, fields),
                                 _arr(C.c_float, gains), xd.data_ptr(), xd.shape[1], self.hist.data_ptr(),
                                 self.out.data_ptr(), self.cap)
        assert rc == 0
        o = self.out.cpu().numpy()
        return {r: o[r, :k].copy() for r, k in nouts.items()}


def _clip(g, n, kind):
    if kind == "noise":
        return g.uniform(-1, 1, n).astype(np.float32)
    if kind == "peaks":
        x = (g.uniform(-1, 1, n) * 0.3).astype(np.float32)
        for p in g.integers(0, max(n, 1), 6)[: n // 50 + 1]:
            if n:
                x[p] = np.float32(g.choice([-1, 1]) * g.uniform(0.9, 1.0))
        return x
    return np.zeros(n, np.float32)


def test_clips_ended_in_one_launch_equal_the_reference_bit_for_bit(lib):
    g = np.random.default_rng(0)
    lens = (0, 1, 119, 120, 255, 256, 257, 511, 1438, 1439, 1700)
    combos = [(n, kind, vol) for n in lens for kind, vol in (("noise", 6.0), ("peaks", 12.0), ("silence", 3.0),
                                                                ("noise", -20.0))]
    R, L = len(combos) + 2, max(lens)
    x = np.zeros((R, L), np.float32)
    jobs, clips = {}, {}
    for i, (n, kind, vol) in enumerate(combos):
        r = i + 1                    # rows 0 and R - 1 have no work
        clips[r] = _clip(g, n, kind)
        x[r, :n] = clips[r]
        jobs[r] = (0, n, True, LR.gain(vol))
    st = Rows(R)
    idle = torch.randn(2, HIST, device=DEV)
    st.hist[:, 0] = idle
    got = st.launch(lib, jobs, x)
    for i, (n, kind, vol) in enumerate(combos):
        want = LR.limit(clips[i + 1], LR.gain(vol))
        assert got[i + 1].shape == (n,) and np.array_equal(got[i + 1], want), (n, kind, vol)
    assert torch.equal(st.hist[:, 0], idle)


@pytest.mark.parametrize("cur", [0, 1])
def test_rows_resumed_mid_clip_equal_the_reference_and_write_the_next_history(lib, cur):
    g = np.random.default_rng(1 + cur)
    N = 9000
    n0s = [119, 120, 1438, 1537, 3000]          # a history at its deepest read, and short ones
    counts = [256 * 3, 1, 257, 2000, 4000]
    R = len(n0s)
    clips = [_clip(g, N, "peaks" if r % 2 else "noise") for r in range(R)]
    st = Rows(R)
    x = np.zeros((R, max(counts)), np.float32)
    jobs = {}
    for r, (n0, c) in enumerate(zip(n0s, counts)):
        h = np.zeros(HIST, np.float32)
        k = min(n0, HIST)
        h[HIST - k:] = clips[r][n0 - k:n0]
        st.hist[cur, r] = torch.from_numpy(h)
        x[r, :c] = clips[r][n0:n0 + c]
        jobs[r] = (n0, c, False, LR.gain(9.0))
    got = st.launch(lib, jobs, x, cur=[cur] * R)
    for r, (n0, c) in enumerate(zip(n0s, counts)):
        y = LR.limit(clips[r], LR.gain(9.0))
        assert np.array_equal(got[r], y[LR.emitted(n0):LR.emitted(n0 + c)]), r
        n1 = n0 + c
        want = np.zeros(HIST, np.float32)
        k = min(n1, HIST)
        want[HIST - k:] = clips[r][n1 - k:n1]
        assert np.array_equal(st.hist[cur ^ 1, r].cpu().numpy(), want), r


def test_move_kernel_saves_and_loads_records(lib):
    R = 4
    st = Rows(R)
    st.hist.copy_(torch.randn(2, R, HIST, device=DEV))
    rows, n_in, cur, gains = [2, 0], [123456789012, 5000], [1, 0], [2.5, 0.125]
    fields = [0, 0, 0, cur[0], 0, 0, 0, cur[1]]
    rec = torch.zeros(2, 6160, dtype=torch.uint8, device=DEV)
    assert lib.limit_shim_move(2, _arr(C.c_int, rows), _arr(C.c_longlong, n_in), _arr(C.c_int, fields),
                               _arr(C.c_float, gains), st.hist.data_ptr(), R, rec.data_ptr(), 0) == 0
    rc = rec.cpu().numpy()
    for i, r in enumerate(rows):
        assert rc[i, :4].view(np.float32)[0] == gains[i] and rc[i, 4:8].view(np.int32)[0] == 0
        assert rc[i, 8:16].view(np.int64)[0] == n_in[i]
        assert np.array_equal(rc[i, 16:].view(np.float32), st.hist[cur[i], r].cpu().numpy())
    before = st.hist.clone()
    fields2 = [0, 0, 0, 0, 0, 0, 0, 1]
    assert lib.limit_shim_move(2, _arr(C.c_int, [3, 1]), _arr(C.c_longlong, [0, 0]), _arr(C.c_int, fields2),
                               _arr(C.c_float, [1.0, 1.0]), st.hist.data_ptr(), R, rec.data_ptr(), 1) == 0
    assert torch.equal(st.hist[0, 3], before[cur[0], 2]) and torch.equal(st.hist[1, 1], before[cur[1], 0])
    for keep in ((1, 3), (0, 1), (0, 0), (1, 0), (0, 2), (1, 2)):
        assert torch.equal(st.hist[keep], before[keep]), keep
