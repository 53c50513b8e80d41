"""The streaming time-stretch's kernels run directly (tests/csrc/stretch_shim.cu) on rows, histories, tails and counters
chosen here, against the fp64 / fp32 reference (tests/stretch_ref.py): on grid inputs (small integers x 2^-4, so every
correlation is exact in fp32) every chosen offset and every output bit for bit, for hops 240 … 960 and clips of
0 … 1201 samples ended in one launch with their zero-padded end frames, many rows and hops in one launch; rows resumed
mid-clip from a history at its deepest read, with their next history, tail and frame position; on random inputs each
offset justified by the fp32 summation bound (the reference follows the kernel after a near-tie); save / load
records."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import audio_shims
from tests import stretch_ref as S

pytestmark = pytest.mark.gpu
HIST = audio_shims.STRETCH_HIST
DEV = "cuda:0"
HOPS = (240, 360, 479, 481, 600, 960)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return audio_shims.load(tmp_path_factory, "stretch_shim")


def _arr(t, xs):
    return (t * len(xs))(*xs)


class Rows:
    """Device state of `rows` stretch rows (history, tail, last frame position) and one launch helper."""

    def __init__(self, rows, cap=16384):
        self.rows, self.cap = rows, cap
        self.hist = torch.zeros(rows, HIST, device=DEV)
        self.tail = torch.zeros(rows, 480, device=DEV)
        self.plast = torch.zeros(rows, dtype=torch.int64, device=DEV)
        self.w = torch.from_numpy(S.window32()).to(DEV)
        self.out = torch.zeros(rows, cap, device=DEV)

    def launch(self, lib, jobs, x):
        """jobs: [(row, n_in, count, end, ha)]; the frame and output counts follow the host formulas.  Returns
        {row: its outputs}."""
        n_in, f0, fields, nouts = [], [], [], {}
        for row, n0, c, end, ha in jobs:
            n = n0 + c
            a = S.frames_done(n0, ha)
            upto = S.total(n, ha) if end else S.emitted(n, ha)
            f1 = -(-upto // 480) if end else S.frames_done(n, ha)
            n_in.append(n0)
            f0.append(a)
            fields += [row, c, f1 - a, upto - 480 * a, int(end), ha]
            nouts[row] = upto - 480 * a
        xd = torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(DEV)
        self.out.zero_()
        rc = lib.stretch_shim_wsola(len(jobs), _arr(C.c_longlong, n_in), _arr(C.c_longlong, f0), _arr(C.c_int, fields),
                                    self.w.data_ptr(), xd.data_ptr(), xd.shape[1], self.hist.data_ptr(),
                                    self.tail.data_ptr(), self.plast.data_ptr(), self.out.data_ptr(), self.cap)
        assert rc == 0
        o = self.out.cpu().numpy()
        return {row: o[row, :k].copy() for row, k in nouts.items()}


def _grid(g, n):
    return (g.integers(-8, 9, n) / 16).astype(np.float32)


def test_grid_clips_ended_in_one_launch_equal_the_reference_bit_for_bit(lib):
    g = np.random.default_rng(0)
    lens = (0, 1, 479, 960, 1199, 1200, 1201, 4999)
    combos = [(ha, n) for ha in HOPS for n in lens]
    R, L = len(combos), max(lens)
    x = np.zeros((R, L), np.float32)
    clips = []
    for r, (ha, n) in enumerate(combos):
        clip = _grid(g, n)
        if r % 3 == 0:
            clip[n // 2:] = 0          # silence inside the clip: exact ties, broken to the smallest |d|, then negative
        clips.append(clip)
        x[r, :n] = clip
    st = Rows(R)
    got = st.launch(lib, [(r, 0, n, True, ha) for r, (ha, n) in enumerate(combos)], x)
    for r, (ha, n) in enumerate(combos):
        want, _, _ = S.stretch(clips[r], ha)
        assert got[r].shape == (S.total(n, ha),) and np.array_equal(got[r], want), (ha, n)


def test_grid_rows_resumed_mid_clip_equal_the_reference_and_leave_the_next_state(lib):
    g = np.random.default_rng(1)
    L, c = 9000, 2500
    clips = [_grid(g, L) for _ in HOPS]
    st = Rows(len(HOPS) + 1)
    x = np.zeros((len(HOPS) + 1, c), np.float32)
    jobs, n0s = [], []
    for r, ha in enumerate(HOPS):
        # just before a frame completes: the next frame's reads reach furthest back into the history
        n0 = S.READY + 3 * ha - 1
        f, pk, tail, hist = S.state_after(clips[r], n0, ha)
        st.hist[r] = torch.from_numpy(hist)
        st.tail[r] = torch.from_numpy(tail)
        st.plast[r] = pk
        x[r] = clips[r][n0:n0 + c]
        jobs.append((r, n0, c, False, ha))
        n0s.append(n0)
    idle = torch.randn(HIST, device=DEV)
    st.hist[len(HOPS)] = idle
    got = st.launch(lib, jobs, x)
    w = S.window32()
    for r, ha in enumerate(HOPS):
        n0, n1 = n0s[r], n0s[r] + c
        y, p, _ = S.stretch(clips[r], ha)
        assert np.array_equal(got[r], y[S.emitted(n0, ha):S.emitted(n1, ha)]), ha
        f1 = S.frames_done(n1, ha)
        assert int(st.plast[r]) == p[f1 - 1]
        assert np.array_equal(st.tail[r].cpu().numpy(), w[480:] * clips[r][p[f1 - 1] + 480:p[f1 - 1] + 960])
        assert np.array_equal(st.hist[r].cpu().numpy(), clips[r][n1 - HIST:n1])
    assert torch.equal(st.hist[len(HOPS)], idle)          # a row without a job is untouched


@pytest.mark.parametrize("ha", [240, 481, 960])
def test_random_inputs_choose_offsets_within_the_fp32_bound(lib, ha):
    g = np.random.default_rng(ha)
    n = 1200 + 40 * ha
    clip = g.uniform(-1, 1, n).astype(np.float32)
    clip[n // 2: n // 2 + 3000] *= np.float32(1e-3)          # a quiet stretch: small correlations beside large ones
    st = Rows(1)
    got, deltas, n0 = [], {}, 0
    for c in [1200] + [ha] * 40:                              # one frame per launch: read its position back
        x = clip[n0:n0 + c][None]
        out = st.launch(lib, [(0, n0, c, False, ha)], x)
        n0 += c
        k = S.frames_done(n0, ha) - 1
        deltas[k] = int(st.plast[0]) - k * ha if k > 0 else 0
        got.append(out[0])
    y, p, stats = S.stretch(clip, ha, follow=deltas)
    near = 0
    for k in range(1, len(deltas)):
        cc, bound = stats[k]
        b, d = S.best(cc), deltas[k]
        if b != d:
            assert cc[b + 240] - cc[d + 240] <= bound[b + 240] + bound[d + 240], (k, b, d)
        top2 = np.sort(cc)[-2:]
        near += top2[1] - top2[0] <= 2 * bound.max()
    assert near <= len(deltas) // 4, near
    got = np.concatenate(got)
    assert np.array_equal(got, y[:got.shape[0]])


def test_move_kernel_saves_and_loads_records(lib):
    R = 4
    st = Rows(R)
    st.hist.copy_(torch.randn(R, HIST, device=DEV))
    st.tail.copy_(torch.randn(R, 480, device=DEV))
    st.plast.copy_(torch.tensor([11, 22, 33, 44], device=DEV))
    rows, n_in, f0, ha = [2, 0], [123456789012, 5000], [3, 8], [600, 240]
    fields = [rows[0], 0, 0, 0, 0, ha[0], rows[1], 0, 0, 0, 0, ha[1]]
    rec = torch.zeros(2, 10144, dtype=torch.uint8, device=DEV)
    assert lib.stretch_shim_move(2, _arr(C.c_longlong, n_in), _arr(C.c_longlong, f0), _arr(C.c_int, fields),
                                 st.hist.data_ptr(), st.tail.data_ptr(), st.plast.data_ptr(), rec.data_ptr(), 0) == 0
    rc = rec.cpu().numpy()
    for i, r in enumerate(rows):
        assert rc[i, :8].view(np.int32).tolist() == [ha[i], 0]
        assert rc[i, 8:32].view(np.int64).tolist() == [n_in[i], f0[i], int(st.plast[r])]
        assert np.array_equal(rc[i, 32:32 + 1920].view(np.float32), st.tail[r].cpu().numpy())
        assert np.array_equal(rc[i, 32 + 1920:].view(np.float32), st.hist[r].cpu().numpy())
    before = (st.hist.clone(), st.tail.clone(), st.plast.clone())
    fields2 = [3, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0]
    assert lib.stretch_shim_move(2, _arr(C.c_longlong, [0, 0]), _arr(C.c_longlong, [0, 0]), _arr(C.c_int, fields2),
                                 st.hist.data_ptr(), st.tail.data_ptr(), st.plast.data_ptr(), rec.data_ptr(), 1) == 0
    for src, dst in ((2, 3), (0, 1)):
        assert torch.equal(st.hist[dst], before[0][src]) and torch.equal(st.tail[dst], before[1][src])
        assert int(st.plast[dst]) == int(before[2][src])
    for keep in (0, 2):
        assert torch.equal(st.hist[keep], before[0][keep]) and int(st.plast[keep]) == int(before[2][keep])
