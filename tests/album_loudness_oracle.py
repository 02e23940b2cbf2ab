"""Float64 restatement of album loudness (mg.album_loudness / mgb_album_loudness, album_loudness_target /
mgb_album_finalize_to_loudness) for the tests.

measure_album: every track K-weighted from rest and cut into its own sub-blocks and windows (oracle/loudness.py), the
gates and the loudness-range percentiles over the union of all tracks' windows, the maxima and peaks over the tracks.
search_album: tests/loudness_target_oracle.py's search rule line for line, with one drive x for every track and the
album's integrated loudness of y_t(x) = limited(s_t, x) in place of a single track's.
"""
from __future__ import annotations

import math

import numpy as np

import loudness
import loudness_target_oracle as lto
import port


def _windows(y: np.ndarray, fs: int):
    """(momentary, short-term) mean squares of one track, complete windows only."""
    B = (fs + 5) // 10
    e = loudness.sub_block_energies(np.asarray(y), fs)
    nb = len(e)
    z = np.lib.stride_tricks.sliding_window_view(e, 4).sum(axis=1) / (4 * B) if nb >= 4 else np.zeros(0)
    s = np.lib.stride_tricks.sliding_window_view(e, 30).sum(axis=1) / (30 * B) if nb >= 30 else np.zeros(0)
    return z, s


def measure_album(ys, fs: int) -> dict:
    """The album meter of the tracks ys ((N_t, 2) each) at rate fs, in loudness.measure's fields."""
    parts = [_windows(y, fs) for y in ys]
    z = np.concatenate([p[0] for p in parts])
    s = np.concatenate([p[1] for p in parts])
    lm, ls = loudness.lufs(z), loudness.lufs(s)

    integrated = -math.inf
    j_abs = lm > -70.0
    if j_abs.any():
        gate = float(loudness.lufs(z[j_abs].mean())) - 10.0
        j_rel = j_abs & (lm > gate)
        if j_rel.any():
            integrated = float(loudness.lufs(z[j_rel].mean()))

    lra = 0.0
    k_abs = ls > -70.0
    if k_abs.any():
        gate = float(loudness.lufs(s[k_abs].mean())) - 20.0
        v = np.sort(ls[k_abs & (ls > gate)])
        n = len(v)
        if n:
            lra = float(v[int(math.floor(0.95 * (n - 1) + 0.5))] - v[int(math.floor(0.10 * (n - 1) + 0.5))])

    peak, tp = np.zeros(2), np.zeros(2)
    for y in ys:
        peak = np.maximum(peak, np.abs(np.asarray(y, dtype=np.float64)).max(axis=0))
        tp = np.maximum(tp, loudness.true_peak(np.asarray(y, dtype=np.float64), fs))
    return dict(integrated=integrated, loudness_range=lra,
                momentary_max=float(lm.max()) if len(lm) else -math.inf,
                short_term_max=float(ls.max()) if len(ls) else -math.inf,
                sample_peak=peak, true_peak=tp, momentary_count=len(z), short_term_count=len(s))


def integrated_album(ys, fs: int) -> float:
    return float(measure_album(ys, fs)["integrated"])


def search_album(ss, cfg, target: float, max_gain_db: float = lto.MAX_GAIN_DB) -> dict:
    """The album search over the tracks ss (float64 (N_t, 2) each, s_t = result_t * gain).  -> lto.search's dict, with
    `outputs` (one per track) in place of `output`."""
    fs = port.config_from(cfg).internal_sample_rate
    measure = lambda ys: integrated_album(ys, fs)
    T, X = float(target), float(max_gain_db)
    I_s = measure(ss)
    undefined = not math.isfinite(I_s)
    x = 0.0 if undefined else min(T - I_s, X)
    lo = hi = None  # (x, f): largest drive below the target, smallest above
    trace = []
    status = 0
    for k in range(1, lto.MAX_PASSES + 1):
        ys = [lto.limited(s, x, cfg) for s in ss]
        I = measure(ys)
        f = I - T
        trace.append((x, I))
        if undefined or not math.isfinite(I):
            status = lto.UNDEFINED
        elif abs(f) <= lto.TOLERANCE:
            status = lto.REACHED
        elif f < 0.0 and x >= X:
            status = lto.UNREACHABLE
        else:
            if f < 0.0 and (lo is None or x > lo[0]):
                lo = (x, f)
            if f > 0.0 and (hi is None or x < hi[0]):
                hi = (x, f)
            if lo is not None and hi is not None and hi[0] - lo[0] < 1e-3:
                status = lto.BRACKET
            elif k >= lto.MAX_PASSES:
                status = lto.PASSES
        if status:
            return dict(gain_db=x, integrated=I, input_integrated=I_s, trace=trace, passes=k, status=status, outputs=ys)
        m = 1.0
        if k >= 2:
            xp, Ip = trace[-2]
            dx = x - xp
            ms = (f - (Ip - T)) / dx if dx != 0.0 else 0.0
            if ms > 0.0 and math.isfinite(ms):
                m = ms
        c = x - f / m
        if lo is not None and hi is None:
            c = max(c, lo[0] - lo[1])
        if hi is not None and lo is None:
            c = min(c, hi[0] - hi[1])
        if lo is not None and hi is not None and not (lo[0] < c < hi[0]):
            c = 0.5 * (lo[0] + hi[0])
        x = min(c, X)
    raise AssertionError("unreachable")
