"""Float64 restatement of the limiter's true-peak mode (Config(true_peak=True)) for the tests.

The detector d[n] = max(u[n], u[n-1]), u[-1] = 0, where u[n] is the largest |y_c[n, ph]| over both channels and the
phases ph = 0 .. L-1 of upfirdn(h, x_c, up=L) at output (n + 6) L + ph, with the loudness meter's interpolator
(oracle/loudness.py, true_peak_filter).  The limiter is oracle/port.py's `limit` with d in place of max(|L|, |R|), and the
normalised output takes its coefficient from max(d).  Any length runs in bounded memory: the interpolator runs over
overlapping chunks, as oracle/loudness.true_peak does.
"""
from __future__ import annotations

import numpy as np
from scipy import signal

import loudness
import port


def oversampling(fs: int) -> int:
    return loudness.true_peak_filter(fs)[0]


def interpolated(x: np.ndarray, fs: int) -> np.ndarray:
    """y[c, n, ph] for a short (N, 2) signal: the interpolated value at n + ph/L, zeros outside the signal."""
    L, h = loudness.true_peak_filter(fs)
    x = np.asarray(x, dtype=np.float64)
    N = len(x)
    y = np.stack([signal.upfirdn(h, x[:, c], up=L)[6 * L:(N + 6) * L] for c in range(2)])
    return y.reshape(2, N, L)


def true_peak_detector(x: np.ndarray, fs: int, chunk: int = 1 << 20) -> np.ndarray:
    """d[n] for an (N, 2) signal of any length."""
    L, h = loudness.true_peak_filter(fs)
    N = len(x)
    d = np.empty(N)
    prev = 0.0  # u[-1]
    for a in range(0, N, chunk):
        b = min(a + chunk, N)
        lo, hi = a - 6, b + 6  # u[a .. b-1] reads x[a - 6 .. b + 5]
        seg = np.zeros((hi - lo, 2))
        seg[max(lo, 0) - lo:min(hi, N) - lo] = x[max(lo, 0):min(hi, N)]
        u = np.zeros(b - a)
        for c in range(2):
            y = signal.upfirdn(h, seg[:, c], up=L)[12 * L:(b - a + 12) * L].reshape(b - a, L)
            u = np.maximum(u, np.abs(y).max(axis=1))
        d[a:b] = np.maximum(u, np.concatenate([[prev], u[:-1]]))
        prev = u[-1]
    return d


def limit(x: np.ndarray, cfg, trace: dict | None = None) -> np.ndarray:
    """limiter/hyrax.py:78-99 with the rectifier r = max(d, thr) / thr."""
    cfg_o = port.config_from(cfg)
    thr = cfg_o.threshold
    x = np.asarray(x, dtype=np.float64)
    d = true_peak_detector(x, cfg_o.internal_sample_rate)
    r = np.maximum(d, thr) / thr
    if np.all(np.isclose(r, 1.0)):
        return x
    g = 1.0 - 1.0 / r
    k = port.limiter_coefficients(cfg_o)
    a_env = port.centred_max(g, k["reach"])
    g_att = port.one_pole_forward_backward(a_env, k["c"])
    h_env = port.trailing_max(a_env, k["hold"])
    hold_out = signal.lfilter(k["bh"], k["ah"], h_env)
    rel_out = signal.lfilter(k["br"], k["ar"], np.maximum(h_env, hold_out))
    g_rel = np.maximum(hold_out, rel_out)
    gain = 1.0 - np.maximum(np.maximum(g, g_att), g_rel)
    if trace is not None:
        trace.update(d=d, g=g, g_att=g_att, g_rel=g_rel, gain=gain)
    return x * gain[:, None]


def main(target: np.ndarray, reference: np.ndarray, cfg):
    """stages.main's (limited, normalised) outputs in true-peak mode: port.main up to the corrected result, then the
    limiter above times the final amplitude coefficient, and the result over max(eps, max(d) / thr)."""
    cfg_o = port.config_from(cfg)
    trace = {}
    _, result, _ = port.main(np.asarray(target, dtype=np.float64), np.asarray(reference, dtype=np.float64), cfg_o,
                             need_default=False, need_no_limiter=True, trace=trace)
    limited = limit(result, cfg_o) * trace["final_coef"]
    peak = float(true_peak_detector(result, cfg_o.internal_sample_rate).max())
    normalized = result / max(cfg_o.min_value, peak / cfg_o.threshold)
    return limited, normalized, trace
