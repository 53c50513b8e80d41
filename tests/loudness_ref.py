"""fp64 restatement of the streaming loudness normaliser (csrc/loud.cu, audio.Loudness, DESIGN §4.9), and a standard
BS.1770 integrated-loudness meter to read outputs with.

gains(x, T) is the definition in fp64: scipy sosfilt with the fp64 K-weighting over the complete 100 ms segments,
z_s, the blocks of up to four segments, the -70 LUFS and relative gates and the clamped gain law, each A_s rounded to
fp32.  apply(x, A) is the output's fp32 arithmetic in numpy float32, bit for bit the kernel's given the same A."""
import numpy as np
from scipy.signal import sosfilt

SEG = 2400
F32 = np.float32


def sos(fs: float) -> np.ndarray:
    """BS.1770-4 K-weighting at fs (libebur128's bilinear design), fp64 (2, 6): shelf, then high-pass."""
    def sec(f0, q):
        k = np.tan(np.pi * f0 / fs)
        a0 = 1 + k / q + k * k
        return k, a0, [1.0, 2 * (k * k - 1) / a0, (1 - k / q + k * k) / a0]
    k, a0, a = sec(1681.974450955533, 0.7071752369554196)
    q = 0.7071752369554196
    vh = 10 ** (3.999843853973347 / 20)
    vb = vh ** 0.4996667741545416
    shelf = [(vh + vb * k / q + k * k) / a0, 2 * (k * k - vh) / a0, (vh - vb * k / q + k * k) / a0] + a
    _, _, a = sec(38.13547087602444, 0.5003270373238773)
    return np.array([shelf, [1.0, -2.0, 1.0] + a])


def lufs(ms):
    with np.errstate(divide="ignore"):
        return -0.691 + 10 * np.log10(ms)


def measure(x, target):
    """The definition of one whole clip x: (A, ms, margin), A[s] the fp32 gain when segment s completes, ms the block
    mean squares and margin[s] the least distance in LU of any block j <= s from the -70 gate and the relative gate of
    segment s (inf where no gate applies)."""
    x = np.asarray(x, np.float64)
    S = x.shape[0] // SEG
    y = sosfilt(sos(24000), x[:S * SEG]) if S else np.zeros(0)
    z = (y.reshape(S, SEG) ** 2).sum(axis=1) if S else np.zeros(0)
    ms = np.array([z[max(0, j - 3):j + 1].sum() / (SEG * min(j + 1, 4)) for j in range(S)])
    l = lufs(ms)
    A, margin, prev = np.zeros(S, F32), np.full(S, np.inf), F32(1)
    for s in range(S):
        ls, m = l[:s + 1], ms[:s + 1]
        ja = ls > -70
        margin[s] = np.min(np.abs(ls + 70))
        if not ja.any():
            A[s] = prev
            continue
        gr = lufs(m[ja].mean()) - 10
        j = ja & (ls > gr)
        margin[s] = min(margin[s], np.min(np.abs(ls - gr)))
        d = np.clip(target - lufs(m[j].mean()), -30, 30)
        A[s] = prev = F32(10 ** (d / 20))
    return A, ms, margin


def gains(x, target) -> np.ndarray:
    return measure(x, target)[0]


def apply(x, A) -> np.ndarray:
    """y[n] = x[n] * (A_{k-2} + (A_{k-1} - A_{k-2}) * fp32((i+1)/2400)), n = 2400k + i, in numpy float32, with
    A_{-1} = A_{-2} = 1; A holds at least the gains of the segments before the last one x reaches."""
    x = np.asarray(x, F32)
    n = x.shape[0]
    Ax = np.concatenate([np.ones(2, F32), np.asarray(A, F32)])
    k = np.arange(n) // SEG
    i = np.arange(n) % SEG
    r = (i + 1).astype(F32) / F32(SEG)                  # IEEE fp32 division: correctly rounded
    aa, ab = Ax[k + 1], Ax[k]
    g = ab + (aa - ab) * r
    return (x * g).astype(F32)


def integrated(x, fs: int = 24000) -> float:
    """The standard BS.1770-4 integrated loudness of x at fs: 400 ms blocks every 100 ms (complete blocks only), the
    -70 LUFS absolute and -10 LU relative gates.  -inf when every block is gated out."""
    x = np.asarray(x, np.float64)
    y = sosfilt(sos(fs), x)
    blk, hop = int(round(0.4 * fs)), int(round(0.1 * fs))
    if y.shape[0] < blk:
        return -np.inf
    c = np.concatenate([[0.0], np.cumsum(y * y)])
    st = np.arange(0, y.shape[0] - blk + 1, hop)
    ms = (c[st + blk] - c[st]) / blk
    l = lufs(ms)
    ja = l > -70
    if not ja.any():
        return -np.inf
    gr = lufs(ms[ja].mean()) - 10
    return float(lufs(ms[ja & (l > gr)].mean()))
