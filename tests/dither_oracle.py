"""The dithered PCM encoder's definition (DESIGN.md §4 "Dither") restated in numpy float64 -- tests only.

Vectorised over (segment, channel): every segment runs its error-feedback loop over the 32 warm-up frames and its
1024 own frames in lock step, one frame position at a time.  numpy rounds every product and sum on its own (no FMA),
and the feedback sums oldest tap first, as the definition says.
"""
import numpy as np

SEGMENT = 1024
WARMUP = 32
GOLDEN = 0x9E3779B97F4A7C15
MASK64 = (1 << 64) - 1


def splitmix64_int(x: int) -> int:
    """The splitmix64 finaliser on a Python int (the reference the vectorised hash is checked against)."""
    z = x & MASK64
    z ^= z >> 30
    z = (z * 0xBF58476D1CE4E5B9) & MASK64
    z ^= z >> 27
    z = (z * 0x94D049BB133111EB) & MASK64
    z ^= z >> 31
    return z


def splitmix64(x: np.ndarray) -> np.ndarray:
    z = np.asarray(x, dtype=np.uint64).copy()
    with np.errstate(over="ignore"):
        z ^= z >> np.uint64(30)
        z *= np.uint64(0xBF58476D1CE4E5B9)
        z ^= z >> np.uint64(27)
        z *= np.uint64(0x94D049BB133111EB)
        z ^= z >> np.uint64(31)
    return z


def tpdf(seed: int, n: np.ndarray, c) -> np.ndarray:
    """d[n, c] in LSB: (a - b) / 2^24 of z = splitmix64(seed + (2n + c + 1) * golden), exact in float64."""
    i1 = (2 * np.asarray(n, dtype=np.int64) + np.asarray(c, dtype=np.int64) + 1).astype(np.uint64)
    with np.errstate(over="ignore"):
        z = splitmix64(np.uint64(seed & MASK64) + i1 * np.uint64(GOLDEN))
    a = (z >> np.uint64(40)).astype(np.int64)
    b = ((z >> np.uint64(16)) & np.uint64(0xFFFFFF)).astype(np.int64)
    return (a - b).astype(np.float64) / 16777216.0


def plain(x: np.ndarray, top: float) -> np.ndarray:
    """The plain encoder's sample: rint(x * top) clipped, NaN -> the lower bound (fmax returns the number)."""
    q = np.rint(np.asarray(x, dtype=np.float32).astype(np.float64) * top)
    q = np.where(np.isnan(q), -top - 1.0, q)
    return np.clip(q, -top - 1.0, top)


def quantize(x: np.ndarray, bits: int, h=(), seed: int = 0, return_error: bool = False):
    """(N, 2) float32 -> the dithered integers, (N, 2) int32 (and with return_error, eps (N, 2) float64: q - v)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    N = x.shape[0]
    top = float(2 ** (bits - 1) - 1)
    h = np.asarray(h, dtype=np.float64)
    K = len(h)
    nseg = max(1, -(-N // SEGMENT))
    # lanes: (segment, channel)
    seg = np.repeat(np.arange(nseg, dtype=np.int64), 2)
    ch = np.tile(np.arange(2, dtype=np.int64), nseg)
    flat = x.reshape(-1)
    out = np.zeros(2 * N, dtype=np.int64)
    eps_out = np.zeros(2 * N, dtype=np.float64) if return_error else None
    hist = [np.zeros(2 * nseg) for _ in range(K)]  # hist[k] = eps[n - 1 - k]
    for j in range(WARMUP + SEGMENT):
        n = seg * SEGMENT - WARMUP + j
        live = (n >= 0) & (n < N)
        idx = np.where(live, 2 * n + ch, 0)
        xv = np.where(live, flat[idx], np.float32(0.0))
        u = xv.astype(np.float64) * top
        fb = np.zeros(2 * nseg)
        for k in range(K - 1, -1, -1):
            fb = fb + h[k] * hist[k]
        v = u - fb
        q = np.rint(v + tpdf(seed, n, ch))
        finite = np.isfinite(q)
        with np.errstate(invalid="ignore"):
            e = np.where(finite, q - v, 0.0)
        e = np.where(n >= 0, e, 0.0)  # before frame 0 there is nothing: segment 0 starts from a zero history
        if K:
            hist = [e] + hist[:-1]
        write = live & (j >= WARMUP)
        y = np.where(finite, np.clip(np.where(finite, q, 0.0), -top - 1.0, top), plain(xv, top))
        out[idx[write]] = y[write].astype(np.int64)
        if return_error:
            eps_out[idx[write]] = e[write]
    res = out.reshape(N, 2).astype(np.int32)
    return (res, eps_out.reshape(N, 2)) if return_error else res


def encode(x: np.ndarray, bits: int, h=(), seed: int = 0) -> np.ndarray:
    """The bytes mgb_pcm_encode_dithered writes: int16 (N, 2), or packed little-endian 24-bit uint8 (N, 6)."""
    q = quantize(x, bits, h, seed)
    if bits == 16:
        return q.astype(np.int16)
    b = q.astype("<i4").view(np.uint8).reshape(-1, 2, 4)[:, :, :3]
    return np.ascontiguousarray(b).reshape(-1, 6)
