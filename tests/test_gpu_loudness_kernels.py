"""The streaming loudness normaliser's kernels run directly (tests/csrc/loud_shim.cu) on rows, records and counters
chosen here, against the fp64 definition (tests/loudness_ref.py): pushes of 1, 2399, 2400 and 2401 samples and segments
that complete exactly at a push boundary, several rows per launch; all-silent input; input below -70 LUFS followed by
speech-like bursts; both ends of the +-30 dB clamp; save / load records.  Through the library: an end in the middle of
a segment, the block cap refused before any launch, and a reset of one row leaving the others bit-identical.

Each kernel output equals the numpy float32 apply of the gains A_s the kernel measured (read from the row's record
after segment-aligned pushes), bit for bit, and the A_s agree with the fp64 definition within A_TOL_DB wherever every
block is more than 0.01 LU from both gates.  A_TOL_DB bounds what fp32 K-weighting through the chunked scan costs: on
12 random noise and speech-like clips of 6 s at -60 to -5 LUFS and targets -40 to -10, the largest error was 4.1e-6 dB
(NVIDIA H100 80GB HBM3), so the bound leaves a margin of about 250."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from tests import loudness_ref as LR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_HDR = {k: int(v) for k, v in re.findall(r"#define (Q3_LOUD_\w+) (\d+)\b",
                                          open(os.path.join(ROOT, "include", "qwen3tts_b200.h")).read())}
ROW_BYTES, MAX_BLOCKS = _HDR["Q3_LOUD_ROW_BYTES"], _HDR["Q3_LOUD_MAX_BLOCKS"]
A_TOL_DB = 1e-3
SEG = LR.SEG


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    from qwen3_tts_b200 import build as b
    out = str(tmp_path_factory.mktemp("loud_shim") / "libloud_shim.so")
    r = subprocess.run([b._nvcc()] + b.NVCC_FLAGS + ["-shared", "-I", b.CSRC,
                        os.path.join(ROOT, "tests", "csrc", "loud_shim.cu"), "-o", out], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lib = C.CDLL(out)
    pl, pi, pd, vp = C.POINTER(C.c_longlong), C.POINTER(C.c_int), C.POINTER(C.c_double), C.c_void_p
    lib.loud_shim_step.argtypes = [C.c_int, pl, pi, pi, pd, C.POINTER(C.c_float), vp, C.c_longlong, vp, vp, C.c_longlong]
    lib.loud_shim_move.argtypes = [C.c_int, pi, pl, pd, vp, vp, C.c_int]
    return lib


def _arr(t, xs):
    return (t * len(xs))(*xs)


SOS = _arr(C.c_float, LR.sos(24000).astype(np.float32).ravel())


class Rows:
    """Records of `rows` rows on the device, their host counters, and one launch helper."""

    def __init__(self, rows, cap=32768):
        self.rows, self.cap = rows, cap
        self.st = torch.zeros(rows, ROW_BYTES, dtype=torch.uint8, device=DEV)
        self.out = torch.zeros(rows, cap, device=DEV)
        self.n = [0] * rows

    def launch(self, lib, pushes, target):
        """pushes {row: fp32 samples}; every row's target `target` (or {row: target}).  Returns {row: outputs}."""
        rows = sorted(pushes)
        L = max(len(pushes[r]) for r in rows)
        x = np.zeros((self.rows, L), np.float32)
        for r in rows:
            x[r, :len(pushes[r])] = pushes[r]
        xd = torch.from_numpy(x).to(DEV)
        tg = [target[r] if isinstance(target, dict) else target for r in rows]
        rc = lib.loud_shim_step(len(rows), _arr(C.c_longlong, [self.n[r] for r in rows]), _arr(C.c_int, rows),
                                _arr(C.c_int, [len(pushes[r]) for r in rows]), _arr(C.c_double, tg), SOS,
                                xd.data_ptr(), L, self.st.data_ptr(), self.out.data_ptr(), self.cap)
        assert rc == 0
        o = self.out.cpu().numpy()
        for r in rows:
            self.n[r] += len(pushes[r])
        return {r: o[r, :len(pushes[r])].copy() for r in rows}

    def a1(self, r):
        return self.st[r, 16:20].cpu().numpy().view(np.float32)[0]


def _gpu_gains(lib, x, target):
    """The kernel's A_s of a whole clip, pushed segment by segment (A_s is then the record's A_{k-1})."""
    st = Rows(1)
    A = []
    for s in range(len(x) // SEG):
        st.launch(lib, {0: x[s * SEG:(s + 1) * SEG]}, target)
        A.append(st.a1(0))
    return np.array(A, np.float32)


def _check_gains(A, x, target):
    """A against the fp64 definition within A_TOL_DB where every block is clear of both gates; the largest error."""
    ref, _, margin = LR.measure(x, target)
    assert A.shape == ref.shape
    ok = margin > 0.01
    err = np.abs(20 * np.log10(A.astype(np.float64) / ref.astype(np.float64)))[ok]
    assert ok.sum() >= len(ok) // 2, "too few segments clear of the gates to compare"
    assert err.max(initial=0) <= A_TOL_DB, (err.max(), np.argmax(err))
    return err.max(initial=0)


def _speech(g, n, level):
    """Speech-like bursts: noise under a 3 Hz on/off envelope with a syllable rate wobble, scaled by `level`."""
    t = np.arange(n) / 24000
    env = np.clip(np.sin(2 * np.pi * 3.1 * t + 2 * np.sin(2 * np.pi * 0.7 * t)), 0, None) ** 2
    return (level * env * g.standard_normal(n)).astype(np.float32)


def _at(x, lufs):
    return (x * 10 ** ((lufs - LR.integrated(x)) / 20)).astype(np.float32)


@pytest.mark.parametrize("sizes", [[1], [2399], [2400], [2401], [1, 2399, 2400, 2401, 4800, 7], [1200, 1200, 3600]])
def test_pushes_of_any_size_apply_the_measured_gains_bit_for_bit(lib, sizes):
    g = np.random.default_rng(sum(sizes))
    N = 24000 * 3 + 1234
    clips = [_at(_speech(g, N, 1.0), -30.0), _at(g.standard_normal(N).astype(np.float32), -20.0)]
    targets = {0: -16.0, 1: -23.0}
    st = Rows(2)
    got = {0: [], 1: []}
    pos = [0, 0]
    k = 0
    while min(pos) < N:
        pushes = {}
        for r in (0, 1):
            c = min(sizes[(k + r) % len(sizes)], N - pos[r])
            if c:
                pushes[r] = clips[r][pos[r]:pos[r] + c]
                pos[r] += c
        for r, y in st.launch(lib, pushes, targets).items():
            got[r].append(y)
        k += 1
    for r in (0, 1):
        A = _gpu_gains(lib, clips[r], targets[r])
        assert np.array_equal(np.concatenate(got[r]), LR.apply(clips[r], A)), r
        _check_gains(A, clips[r], targets[r])


def test_silence_keeps_unity_gain_and_quiet_input_then_bursts_follow_the_definition(lib):
    g = np.random.default_rng(5)
    z = np.zeros(24000 * 2 + 10, np.float32)
    assert np.all(_gpu_gains(lib, z, -16.0) == 1)
    quiet = (g.standard_normal(24000) * 10 ** (-80 / 20)).astype(np.float32)   # about -80 LUFS
    x = np.concatenate([quiet, _at(_speech(g, 24000 * 4, 1.0), -24.0)])
    A = _gpu_gains(lib, x, -16.0)
    assert np.all(A[:10] == 1)                                            # every block so far is below -70 LUFS
    assert A[-1] > 2.0
    _check_gains(A, x, -16.0)


@pytest.mark.parametrize("level,target,want_db", [(-65.0, -10.0, 30.0), (-2.0, -40.0, -30.0)])
def test_the_gain_is_clamped_at_30_db(lib, level, target, want_db):
    g = np.random.default_rng(11)
    x = _at((g.standard_normal(24000 * 2) * 0.1).astype(np.float32), level)
    A = _gpu_gains(lib, x, target)
    assert np.all(A[3:] == np.float32(10 ** (want_db / 20)))
    _check_gains(A, x, target)


def test_move_kernel_saves_and_loads_records(lib):
    R = 4
    st = Rows(R)
    st.st.copy_(torch.randint(0, 256, st.st.shape, dtype=torch.uint8, device=DEV))
    rows, n_in, tg = [2, 0], [123456789, 5000], [-16.0, -23.5]
    rec = torch.zeros(2, ROW_BYTES, dtype=torch.uint8, device=DEV)
    assert lib.loud_shim_move(2, _arr(C.c_int, rows), _arr(C.c_longlong, n_in), _arr(C.c_double, tg),
                              st.st.data_ptr(), rec.data_ptr(), 0) == 0
    rc, sv = rec.cpu().numpy(), st.st.cpu().numpy()
    for i, r in enumerate(rows):
        assert rc[i, :8].view(np.float64)[0] == tg[i] and rc[i, 8:16].view(np.int64)[0] == n_in[i]
        assert np.array_equal(rc[i, 16:], sv[r, 16:])
    before = st.st.clone()
    assert lib.loud_shim_move(2, _arr(C.c_int, [3, 1]), _arr(C.c_longlong, [0, 0]), _arr(C.c_double, [0.0, 0.0]),
                              st.st.data_ptr(), rec.data_ptr(), 1) == 0
    assert torch.equal(st.st[3], rec[0]) and torch.equal(st.st[1], rec[1])
    assert torch.equal(st.st[0], before[0]) and torch.equal(st.st[2], before[2])


# ------------------------------------------------------------------------------------------------- through the library
def test_an_end_mid_segment_emits_nothing_more_and_the_next_clip_starts_fresh():
    from qwen3_tts_b200.audio import Loudness
    g = np.random.default_rng(3)
    a, b = _at(_speech(g, 3500 + 2400 * 5, 1.0), -20.0)[:3500], _at(_speech(g, 24000 * 2, 1.0), -28.0)
    ld = Loudness(DEV, 2, 4096)
    try:
        ld.reset([0, 1], -16.0)
        y = ld.push({0: a[:3000]})[0]
        y = np.concatenate([y, ld.push({0: a[3000:]}, end=[0])[0]])
        assert y.shape == (3500,) and np.array_equal(y, ld.oneshot(a, -16.0))
        assert ld.push({}, end=[0])[0].shape == (0,)
        y2 = np.concatenate([ld.push({0: b[i:i + 4096]})[0] for i in range(0, len(b), 4096)])
        assert np.array_equal(y2, ld.oneshot(b, -16.0))
    finally:
        ld.close()


def test_the_block_cap_is_refused_before_any_launch():
    from qwen3_tts_b200.audio import Loudness
    cap = MAX_BLOCKS * SEG
    ld = Loudness(DEV, 2, 256)
    try:
        ld.reset([0, 1], -16.0)
        ld.push({0: np.full(10, 0.1, np.float32), 1: np.full(10, 0.1, np.float32)})
        rec = ld.save([0, 1])
        rec[0, 8:16] = torch.tensor([cap - 100], dtype=torch.int64).view(torch.uint8).to(DEV)
        ld.load([0, 1], rec)
        before = ld.save([0, 1])
        with pytest.raises(RuntimeError, match="segments"):
            ld.push({0: np.full(101, 0.1, np.float32), 1: np.full(5, 0.1, np.float32)})
        assert torch.equal(ld.save([0, 1]), before)              # nothing moved, not even the other row
        assert ld.push({0: np.full(100, 0.1, np.float32)})[0].shape == (100,)
        with pytest.raises(RuntimeError, match="segments"):
            ld.push({0: np.full(1, 0.1, np.float32)})
        ld.push({}, end=[0])
        assert ld.push({0: np.full(1, 0.1, np.float32)})[0].shape == (1,)
    finally:
        ld.close()


def test_a_reset_of_one_row_leaves_the_others_bit_identical():
    from qwen3_tts_b200.audio import Loudness
    g = np.random.default_rng(9)
    clips = [_at(_speech(g, 24000 * 2, 1.0), lv) for lv in (-18.0, -30.0, -25.0)]

    def run(reset_mid):
        ld = Loudness(DEV, 3, 3000)
        try:
            ld.reset([0, 1, 2], -16.0)
            out = {r: [] for r in range(3)}
            for i in range(0, 48000, 3000):
                if reset_mid and i == 24000:
                    ld.reset([1], -20.0)
                for r, y in ld.push({r: c[i:i + 3000] for r, c in enumerate(clips)}).items():
                    out[r].append(y)
            return {r: np.concatenate(v) for r, v in out.items()}, ld.save([0, 2]).cpu()
        finally:
            ld.close()

    a, ra = run(False)
    b, rb = run(True)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2]) and torch.equal(ra, rb)
    assert not np.array_equal(a[1], b[1])
