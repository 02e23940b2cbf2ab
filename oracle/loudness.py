"""Float64 restatement of the loudness meter (matchering_b200.loudness, mgb_loudness) for the tests.

ITU-R BS.1770-4 K-weighting and gating, EBU Tech 3342 loudness range with libebur128's percentile rule, and the
true peak as the maximum of |upfirdn(h, x, up=L)|.  Written from the definition with numpy and scipy only: every
coefficient is derived here again, not taken from the package.  Any length runs in bounded memory: the filters
carry their state (`zi`) across chunks, the sub-block energies are added chunk by chunk, and the interpolator runs
over overlapping chunks.
"""
from __future__ import annotations

import math

import numpy as np
from scipy import signal

LUFS_OFFSET = -0.691


def k_weighting(fs: int):
    """(shelf_b, shelf_a, highpass_b, highpass_a) for any rate, from the analog prototypes."""
    def section(f0, q):
        k = math.tan(math.pi * f0 / fs)
        a0 = 1.0 + k / q + k * k
        return k, a0, np.array([1.0, 2.0 * (k * k - 1.0) / a0, (1.0 - k / q + k * k) / a0])
    q = 0.7071752369554196
    k, a0, shelf_a = section(1681.974450955533, q)
    vh = 10.0 ** (3.999843853973347 / 20.0)
    vb = vh ** 0.4996667741545416
    shelf_b = np.array([vh + vb * k / q + k * k, 2.0 * (k * k - vh), vh - vb * k / q + k * k]) / a0
    _, _, hp_a = section(38.13547087602444, 0.5003270373238773)
    return shelf_b, shelf_a, np.array([1.0, -2.0, 1.0]), hp_a


def true_peak_filter(fs: int):
    """(L, h): oversampling factor and the 12 L + 1 taps sinc((m - 6L)/L) * kaiser(12L + 1, 8)."""
    L = 4 if fs < 96000 else (2 if fs < 192000 else 1)
    m = np.arange(12 * L + 1)
    return L, np.sinc((m - 6 * L) / L) * np.kaiser(12 * L + 1, 8.0)


def lufs(mean_square):
    with np.errstate(divide="ignore"):
        return LUFS_OFFSET + 10.0 * np.log10(mean_square)


def sub_block_energies(x: np.ndarray, fs: int, chunk: int = 1 << 20) -> np.ndarray:
    """e_b = sum over sub-block b of yL^2 + yR^2 (y = K-weighted), complete sub-blocks only."""
    sb, sa, hb, ha = k_weighting(fs)
    B = (fs + 5) // 10
    N = len(x)
    nb = N // B
    e = np.zeros(nb)
    zi = np.zeros((2, 2, 2))  # [section][channel][state]: lfilter from rest at n = 0
    for a in range(0, N, chunk):
        seg = np.asarray(x[a:a + chunk], dtype=np.float64)
        sq = np.zeros(len(seg))
        for c in range(2):
            y, zi[0, c] = signal.lfilter(sb, sa, seg[:, c], zi=zi[0, c])
            y, zi[1, c] = signal.lfilter(hb, ha, y, zi=zi[1, c])
            sq += y * y
        end = min(a + len(seg), nb * B)
        if end <= a:
            continue
        first = a // B
        starts = np.concatenate([[0], np.arange((first + 1) * B - a, end - a, B)]).astype(np.int64)
        sums = np.add.reduceat(sq[:end - a], starts)
        e[first:first + len(sums)] += sums
    return e


def true_peak(x: np.ndarray, fs: int, chunk: int = 1 << 20) -> np.ndarray:
    """max |upfirdn(h, x_channel, up=L)| per channel (zero outside the signal), over overlapping chunks of centres:
    the output at (n + 6) L + phase interpolates around frame n, n = -6 .. N + 5."""
    L, h = true_peak_filter(fs)
    N = len(x)
    tp = np.zeros(2)
    for c0 in range(-6, N + 6, chunk):
        c1 = min(c0 + chunk, N + 6)
        lo, hi = c0 - 6, c1 + 6
        seg = np.zeros((hi - lo, 2))
        seg[max(lo, 0) - lo:min(hi, N) - lo] = x[max(lo, 0):min(hi, N)]
        for c in range(2):
            y = signal.upfirdn(h, seg[:, c], up=L)[12 * L:(c1 - c0 + 12) * L]
            tp[c] = max(tp[c], float(np.abs(y).max()))
    return tp


def measure(x, fs: int, chunk: int = 1 << 20) -> dict:
    """The meter's result for (N, 2) samples at rate fs."""
    x = np.asarray(x)
    assert x.ndim == 2 and x.shape[1] == 2
    B = (fs + 5) // 10
    e = sub_block_energies(x, fs, chunk)
    nb = len(e)
    z = np.lib.stride_tricks.sliding_window_view(e, 4).sum(axis=1) / (4 * B) if nb >= 4 else np.zeros(0)
    s = np.lib.stride_tricks.sliding_window_view(e, 30).sum(axis=1) / (30 * B) if nb >= 30 else np.zeros(0)
    lm, ls = lufs(z), lufs(s)

    integrated = -math.inf
    j_abs = lm > -70.0
    if j_abs.any():
        gate = float(lufs(z[j_abs].mean())) - 10.0
        j_rel = j_abs & (lm > gate)
        if j_rel.any():
            integrated = float(lufs(z[j_rel].mean()))

    lra = 0.0
    k_abs = ls > -70.0
    if k_abs.any():
        gate = float(lufs(s[k_abs].mean())) - 20.0
        v = np.sort(ls[k_abs & (ls > gate)])
        n = len(v)
        if n:
            lra = float(v[int(math.floor(0.95 * (n - 1) + 0.5))] - v[int(math.floor(0.10 * (n - 1) + 0.5))])

    peak = np.zeros(2)
    for a in range(0, len(x), chunk):
        peak = np.maximum(peak, np.abs(np.asarray(x[a:a + chunk], dtype=np.float64)).max(axis=0))
    return dict(integrated=integrated, loudness_range=lra,
                momentary_max=float(lm.max()) if len(lm) else -math.inf,
                short_term_max=float(ls.max()) if len(ls) else -math.inf,
                sample_peak=peak, true_peak=true_peak(x, fs, chunk),
                momentary_count=len(z), short_term_count=len(s))
