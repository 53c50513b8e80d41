"""numpy restatement of the streaming look-ahead limiter (csrc/limit.cu, audio.Limiter, DESIGN §4.8).

Every operation is an fp32 numpy operation, elementwise and in the definition's order, so the result is the kernel's
bit for bit:
    u = g*x,  a = 1 where |u| <= c else c/|u|,  b[m] = min a[m .. m+L-1],
    s[n] = min(a[n], (b[n] + b[n-1] + ... + b[n-L+1]) * inv),
    G[n] = min over m in [max(0, n-W), n] of s[m] + fp32(n-m)*delta,  y = u*G,
with x = 0 before the clip and past its end."""
import numpy as np

L, W = 120, 1200
DELAY = L - 1
REACH = W + 2 * L - 2                  # inputs the first pending output reads back
C = np.float32(10 ** (-1 / 20))
DELTA = np.float32(1 / 1200)
INV = np.float32(1 / 120)
F32 = np.float32


def gain(volume: float) -> np.float32:
    return np.float32(10.0 ** (volume / 20))


def emitted(n: int) -> int:
    return max(0, n - DELAY)


def limit(x, g) -> np.ndarray:
    """y of a whole clip x (float32) at gain g (fp32)."""
    x = np.asarray(x, np.float32)
    n = x.shape[0]
    g = np.float32(g)
    pre = W + L - 1                                        # positions -pre .. n + L - 2 are staged
    xs = np.concatenate([np.zeros(pre, F32), x, np.zeros(L, F32)])
    u = xs * g
    m = np.abs(u)
    with np.errstate(divide="ignore"):
        a = np.where(m <= C, F32(1), C / np.where(m <= C, F32(1), m)).astype(F32)
    # b[j] for staged positions j = 0 .. len - L
    nb = a.shape[0] - L + 1
    b = a[:nb].copy()
    for q in range(1, L):
        b = np.minimum(b, a[q:q + nb])
    # s at positions -W .. n-1: staged index p = pos + pre; b index p - k for k = 0 .. L-1
    pos = np.arange(-W, n)
    p = pos + pre
    acc = b[p].copy()
    for k in range(1, L):
        acc = (acc + b[p - k]).astype(F32)
    s = np.minimum(a[p], (acc * INV).astype(F32))
    s = np.where(pos < 0, F32(np.inf), s).astype(F32)
    # G[n] for n = 0 .. n-1: s index of position n - d is n - d + W
    G = s[W:W + n].copy()
    for d in range(1, W + 1):
        G = np.minimum(G, (s[W - d:W - d + n] + F32(d) * DELTA).astype(F32))
    return (u[pre:pre + n] * G).astype(F32)
