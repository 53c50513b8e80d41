"""The streaming resampler's kernels run directly (tests/csrc/resample_shim.cu) on rows, histories and counters chosen
here, against an fp64 reference: outputs read from the history at its deepest and from the new inputs, an end's zero
padding past the clip, several filters and encodings in one launch, the s16 clamp and round-half-even ties, the next
history half (zeros after an end, untouched for an idle row), and save / load records."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import audio_shims
from tests.test_gpu_resample import _s16, _ulaw

pytestmark = pytest.mark.gpu
HIST = audio_shims.RESAMPLE_HIST
DEV = "cuda:0"


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return audio_shims.load(tmp_path_factory, "resample_shim")


def _arr(t, xs):
    return (t * len(xs))(*xs)


def _ref(h, up, down, hl, x, n_tot, j):
    """fp64 y[j] of the clip x (indexed from 0, x = 0 at and past n_tot)."""
    c = hl + j * down
    return sum(float(x[m]) * float(h[c - m * up]) for m in range(max(0, -(-(c - 2 * hl) // up)), min(c // up, n_tot - 1) + 1))


def test_poly_kernel_rows_against_fp64(lib):
    g = np.random.default_rng(0)
    filters = [(3, 2, 12), (1, 3, 30), (1, 1, 0)]            # (up, down, hl): 16 -> 24 kHz, 24 -> 8 kHz, a copy
    taps = [torch.from_numpy(g.uniform(-0.4, 0.4, 2 * hl + 1).astype(np.float32)).to(DEV) for _, _, hl in filters]
    taps[2] = torch.ones(1, device=DEV)
    # rows: (filter, encoding, inputs before, new inputs, end).  Row 0 starts at its deepest history read (the first
    # output not yet emitted reads floor(2*hl/up) inputs back); row 1 ends with no input (zero padding only); row 2 is a
    # fresh clip ended in the same launch; row 3 encodes s16 past the clamp; row 4 is ulaw; row 5 is idle.
    rows = [(1, 0, 1000, 300, 0), (0, 0, 777, 0, 1), (1, 0, 0, 50, 1), (0, 1, 400, 257, 0), (1, 2, 130, 64, 0), (0, 0, 90, 0, 0)]
    R, L = len(rows), 400
    clips = [g.uniform(-3 if r == 3 else -1, 3 if r == 3 else 1, n0 + c).astype(np.float32) for r, (_, _, n0, c, _) in enumerate(rows)]
    hist = np.zeros((2, R, HIST), np.float32)
    x = np.zeros((R, L), np.float32)
    n_in, out0, fields, cur = [], [], [], [r % 2 for r in range(R)]
    for r, (fi, enc, n0, c, end) in enumerate(rows):
        up, down, hl = filters[fi]
        for k in range(HIST):       # the history: the clip's last HIST inputs before this launch
            m = n0 - HIST + k
            hist[cur[r], r, k] = clips[r][m] if m >= 0 else 0.0
        x[r, :c] = clips[r][n0:]
        e0 = max(0, (n0 * up - 1 - hl) // down + 1)
        e1 = -(-(n0 + c) * up // down) if end else max(0, ((n0 + c) * up - 1 - hl) // down + 1)
        n_in.append(n0)
        out0.append(e0)
        fields += [c, e1 - e0, end, fi, enc, cur[r]]
    hd = torch.from_numpy(hist).to(DEV)
    xd = torch.from_numpy(x).to(DEV)
    cap = 4 * 1024
    out = torch.zeros(R, cap, dtype=torch.uint8, device=DEV)
    rc = lib.resample_shim_poly(len(filters), _arr(C.c_void_p, [t.data_ptr() for t in taps]), _arr(C.c_int, [f[0] for f in filters]),
                                _arr(C.c_int, [f[1] for f in filters]), _arr(C.c_int, [f[2] for f in filters]), R,
                                _arr(C.c_longlong, n_in), _arr(C.c_longlong, out0), _arr(C.c_int, fields), xd.data_ptr(), L,
                                hd.data_ptr(), out.data_ptr(), cap)
    assert rc == 0
    o, hn = out.cpu().numpy(), hd.cpu().numpy()
    for r, (fi, enc, n0, c, end) in enumerate(rows):
        up, down, hl = filters[fi]
        h = taps[fi].cpu().numpy()
        nout = fields[6 * r + 1]
        want = np.array([_ref(h, up, down, hl, clips[r], n0 + c, out0[r] + t) for t in range(nout)])
        ntap = max(1, -(-(2 * hl + 1) // up))
        bound = ntap * 2.0 ** -24 * np.abs(h).sum() * np.abs(clips[r]).max() * 2   # a sequential fp32 sum's error
        if enc == 0:
            y = o[r, :4 * nout].view(np.float32)
            assert np.abs(y - want).max(initial=0) <= bound, (r, np.abs(y - want).max(initial=0), bound)
        else:
            # the encodings of the fp64 value moved by the sum's error bound either way: the kernel's must be one of them
            lo, hi = _s16((want - bound).astype(np.float32)), _s16((want + bound).astype(np.float32))
            if enc == 1:
                got = o[r, :2 * nout].view(np.int16)
                assert ((lo <= got) & (got <= hi)).all(), r
            else:
                got = o[r, :nout]
                assert ((got == _ulaw(lo)) | (got == _ulaw(hi))).all(), r
        if enc == 1:
            assert (o[r, :2 * nout].view(np.int16) == 32767).any() and (o[r, :2 * nout].view(np.int16) == -32768).any()
        # the next history half
        nh = hn[1 - cur[r], r]
        if c == 0 and not end:
            assert np.array_equal(nh, hist[1 - cur[r], r])            # an idle row is untouched
        elif end:
            assert not nh.any()
        else:
            n1 = n0 + c
            assert np.array_equal(nh, np.array([clips[r][n1 - HIST + k] if n1 - HIST + k >= 0 else 0 for k in range(HIST)], np.float32))
        assert np.array_equal(hn[cur[r], r], hist[cur[r], r])            # the current half is only read


def test_s16_round_half_even_and_clamp_through_the_copy_filter(lib):
    vals = np.array([0.5, 1.5, 2.5, -0.5, -1.5, 32766.5, 32767.5, -32768.5, 40000, -40000, 3.49, -3.51], np.float64) / 32768
    x = torch.from_numpy(vals.astype(np.float32)).to(DEV)[None]
    taps = torch.ones(1, device=DEV)
    n = len(vals)
    hist = torch.zeros(2, 1, HIST, device=DEV)
    out = torch.zeros(1, 4 * n, dtype=torch.uint8, device=DEV)
    rc = lib.resample_shim_poly(1, _arr(C.c_void_p, [taps.data_ptr()]), _arr(C.c_int, [1]), _arr(C.c_int, [1]), _arr(C.c_int, [0]), 1,
                                _arr(C.c_longlong, [0]), _arr(C.c_longlong, [0]), _arr(C.c_int, [n, n, 1, 0, 1, 0]), x.data_ptr(), n,
                                hist.data_ptr(), out.data_ptr(), 4 * n)
    assert rc == 0
    got = out.cpu().numpy()[0, :2 * n].view(np.int16)
    assert got.tolist() == [0, 2, 2, 0, -2, 32766, 32767, -32768, 32767, -32768, 3, -4]


def test_move_kernel_saves_and_loads_records(lib):
    R = 4
    hist = torch.randn(2, R, HIST, device=DEV)
    rows, n_in, cur = [2, 0], [12345678901, 7], [1, 0]
    fields = [0, 0, 0, 3, 2, cur[0], 0, 0, 0, 1, 0, cur[1]]
    rec = torch.zeros(2, 528, dtype=torch.uint8, device=DEV)
    assert lib.resample_shim_move(2, _arr(C.c_int, rows), _arr(C.c_longlong, n_in), _arr(C.c_int, fields), hist.data_ptr(), R,
                                  rec.data_ptr(), 0) == 0
    rc = rec.cpu().numpy()
    h = hist.cpu().numpy()
    for i, r in enumerate(rows):
        assert rc[i, :8].view(np.int32).tolist() == [fields[6 * i + 3], fields[6 * i + 4]]
        assert rc[i, 8:16].view(np.int64)[0] == n_in[i]
        assert np.array_equal(rc[i, 16:].view(np.float32), h[cur[i], r])
    before = hist.clone()
    # load record 0 into row 3's half 0 and record 1 into row 1's half 1: nothing else changes
    fields2 = [0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1]
    assert lib.resample_shim_move(2, _arr(C.c_int, [3, 1]), _arr(C.c_longlong, [0, 0]), _arr(C.c_int, fields2), hist.data_ptr(), R,
                                  rec.data_ptr(), 1) == 0
    want = before.clone()
    want[0, 3] = before[cur[0], 2]
    want[1, 1] = before[cur[1], 0]
    assert torch.equal(hist, want)
