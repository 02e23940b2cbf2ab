"""Float64 restatement of loudness targets (Config(loudness_target=T), mgb_limit_to_loudness, mgb_finalize_to_loudness)
for the tests.

y(x) = limit(s * 10^(x/20)) with oracle/port.py's limiter (tests/true_peak_oracle.py's in true-peak mode), no final
amplitude coefficient; I(.) = oracle/loudness.py's integrated loudness.  `search` is the device's rule line for line
(matchering_b200/csrc/loudness_target.cuh): deterministic given the measured loudness values.
"""
from __future__ import annotations

import math

import numpy as np

import loudness
import port
import true_peak_oracle as tpo

MAX_PASSES = 8
TOLERANCE = 0.01  # LU
MAX_GAIN_DB = 24.0  # matchering_b200.loudness.LOUDNESS_TARGET_MAX_GAIN_DB
REACHED, UNREACHABLE, BRACKET, PASSES, UNDEFINED = 1, 2, 3, 4, 5


def integrated(y: np.ndarray, fs: int) -> float:
    return float(loudness.measure(y, fs)["integrated"])


def limited(s: np.ndarray, x: float, cfg) -> np.ndarray:
    """y(x): the limiter (in cfg's peak mode) over s * 10^(x/20)."""
    cfg_o = port.config_from(cfg)
    v = np.asarray(s, dtype=np.float64) * 10.0 ** (x / 20.0)
    return tpo.limit(v, cfg) if getattr(cfg, "true_peak", False) else port.limit(v, cfg_o)


def search(s: np.ndarray, cfg, target: float, max_gain_db: float = MAX_GAIN_DB, measure=None) -> dict:
    """The search over s (float64 (N, 2)).  `measure(y)` -> integrated loudness (default: the oracle meter at cfg's
    rate).  -> dict(gain_db, integrated, input_integrated, trace=[(x, I)], passes, status, output)"""
    fs = port.config_from(cfg).internal_sample_rate
    measure = measure or (lambda y: integrated(y, fs))
    T, X = float(target), float(max_gain_db)
    I_s = measure(s)
    undefined = not math.isfinite(I_s)
    x = 0.0 if undefined else min(T - I_s, X)
    lo = hi = None  # (x, f): largest drive below the target, smallest above
    trace = []
    status = 0
    for k in range(1, MAX_PASSES + 1):
        y = limited(s, x, cfg)
        I = measure(y)
        f = I - T
        trace.append((x, I))
        if undefined or not math.isfinite(I):
            status = UNDEFINED
        elif abs(f) <= TOLERANCE:
            status = REACHED
        elif f < 0.0 and x >= X:
            status = UNREACHABLE
        else:
            if f < 0.0 and (lo is None or x > lo[0]):
                lo = (x, f)
            if f > 0.0 and (hi is None or x < hi[0]):
                hi = (x, f)
            if lo is not None and hi is not None and hi[0] - lo[0] < 1e-3:
                status = BRACKET
            elif k >= MAX_PASSES:
                status = PASSES
        if status:
            return dict(gain_db=x, integrated=I, input_integrated=I_s, trace=trace, passes=k, status=status, output=y)
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


def main(target: np.ndarray, reference: np.ndarray, cfg, loudness_target: float, max_gain_db: float = MAX_GAIN_DB) -> dict:
    """stages.main's limited output at the target: port.main up to the corrected result (s = result * gain), then the
    search over s.  The dict also holds the trace of port.main under 'main'."""
    tr = {}
    _, result, _ = port.main(np.asarray(target, dtype=np.float64), np.asarray(reference, dtype=np.float64),
                             port.config_from(cfg), need_default=False, need_no_limiter=True, trace=tr)
    out = search(result, cfg, loudness_target, max_gain_db)
    out["main"] = tr
    out["s"] = result
    return out
