"""fp64 / fp32 reference of the WSOLA time-stretch (DESIGN §4.7, audio.TimeStretch, csrc/stretch_kernels.cuh).

Frames of N = 960 samples at analysis hop Ha, synthesis hop 480, search tolerance 240: frame k sits at
p_k = k*Ha + d_k (d_0 = 0), where d_k maximises C_k(d) = sum_{n<480} x[p_{k-1} + 480 + n] * x[k*Ha + d + n] over
|d| <= 240, ties to the smallest |d| and then to the negative d.  The correlations are computed here in fp64 (the kernel
sums in fp32; `c_bound` is the gap between the two); the output is the kernel's fp32 arithmetic exactly:
y[m] = x[m] for m < 480, y[k*480 + i] = fl(fl(w[i]*x[p_k + i]) + fl(w[i+480]*x[p_{k-1} + i + 480])), and a clip of n
samples has ceil(n*480/Ha) of them, with x = 0 past n."""
import numpy as np

N, HS, DELTA = 960, 480, 240
READY = N + DELTA          # frame k is done once input k*Ha + READY - 1 has arrived


def window32() -> np.ndarray:
    return (np.sin(np.pi * np.arange(N) / N) ** 2).astype(np.float32)


def hop(speed: float) -> int:
    return int(np.floor(speed * HS + 0.5))


def frames_done(n: int, ha: int) -> int:
    return 0 if n < READY else (n - READY) // ha + 1


def emitted(n: int, ha: int) -> int:
    return HS * frames_done(n, ha)


def total(n: int, ha: int) -> int:
    return -(-n * HS // ha)


def best(c: np.ndarray) -> int:
    """The chosen offset among candidates d = -240 .. 240 with correlations c[d + 240]: the key (C, -|d|, -d)."""
    d = np.arange(-DELTA, DELTA + 1)
    order = np.lexsort((d, np.abs(d), -c))   # last key primary: largest C, then smallest |d|, then smallest d
    return int(d[order[0]])


def correlations(xp: np.ndarray, p_prev: int, ak: int) -> np.ndarray:
    """C(d) for d = -240 .. 240 in fp64."""
    ref = xp[p_prev + HS: p_prev + N].astype(np.float64)
    cand = np.lib.stride_tricks.sliding_window_view(xp[ak - DELTA: ak + DELTA + HS].astype(np.float64), HS)
    return cand @ ref


def c_bound(xp: np.ndarray, p_prev: int, ak: int) -> np.ndarray:
    """An upper bound of |C_fp32(d) - C(d)| for the kernel's sequential fp32 sum of 480 products."""
    ref = np.abs(xp[p_prev + HS: p_prev + N].astype(np.float64))
    cand = np.lib.stride_tricks.sliding_window_view(np.abs(xp[ak - DELTA: ak + DELTA + HS].astype(np.float64)), HS)
    u = 2.0 ** -24
    return (HS * u / (1 - HS * u)) * (cand @ ref)


def stretch(x: np.ndarray, ha: int, follow=None, w: np.ndarray = None):
    """The whole clip x (fp32) at hop ha.  `follow`: {k: d} offsets to take instead of the fp64 choice (the kernel's
    choice after a near-tie).  Returns (y fp32 [total(n, ha)], positions p_k, [(C fp64, bound) per frame k >= 1])."""
    x = np.asarray(x, np.float32)
    w = window32() if w is None else w
    n = x.shape[0]
    M = total(n, ha)
    K = -(-M // HS)
    xp = np.zeros(max(n, (K + 1) * ha + READY + HS), np.float32)
    xp[:n] = x
    y = np.zeros(K * HS, np.float32)
    p = [0]
    stats = [None]
    if K == 0:
        return y, p, stats
    y[:HS] = xp[:HS]
    tail = w[HS:] * xp[HS:N]
    for k in range(1, K):
        ak = k * ha
        c = correlations(xp, p[-1], ak)
        stats.append((c, c_bound(xp, p[-1], ak)))
        d = best(c) if follow is None or k not in follow else int(follow[k])
        pk = ak + d
        y[k * HS:(k + 1) * HS] = w[:HS] * xp[pk: pk + HS] + tail
        tail = w[HS:] * xp[pk + HS: pk + N]
        p.append(pk)
    return y[:M], p, stats


def state_after(x: np.ndarray, n0: int, ha: int, w: np.ndarray = None):
    """A row's state after the first n0 samples of x without an end: (frames done, p of the last frame, its windowed
    second half fp32 [480], the last 2048 inputs fp32 with zeros before sample 0)."""
    w = window32() if w is None else w
    f = frames_done(n0, ha)
    hist = np.zeros(2048, np.float32)
    lo = max(0, n0 - 2048)
    hist[2048 - (n0 - lo):] = x[lo:n0]
    if f == 0:
        return 0, 0, np.zeros(HS, np.float32), hist
    _, p, _ = stretch(x[:n0], ha, w=w)
    pk = p[f - 1]
    xs = np.zeros(pk + N, np.float32)
    m = min(len(x), pk + N)
    xs[:m] = x[:m]
    return f, pk, w[HS:] * xs[pk + HS: pk + N], hist
