"""Float64 restatement of linked versions (stages.main_versions, mgb_version_match_frequencies / mgb_finalize_versions;
DESIGN.md section 4 "Linked versions") for the tests, on top of oracle/port.py.

The main x_0 runs stages 1-3 as port.main runs them.  Every target x_v (the main included) then goes through the main's
chain: s_v = ms_to_lr(h * (c0 mid_v), h * (c0 side_v)) * G, with the main's FIRs h, c0 and correction gain G.  One
detector D = max over v of the limiter's detector of s_v drives port's limiter steps once; its gain e multiplies every
s_v.
"""
from __future__ import annotations

import contextlib

import numpy as np
from scipy import signal

import loudness_target_oracle
import port
import true_peak_oracle


def chain(x: np.ndarray, trace: dict) -> np.ndarray:
    """s = the main's FIRs, c0 and correction gain applied to x."""
    mid, side = port.mid_side(np.asarray(x, np.float64))
    c0 = trace["c0"]
    r_mid = port.convolve_same(mid * c0, trace["firs"]["mid"])
    r_side = port.convolve_same(side * c0, trace["firs"]["side"])
    return np.stack([r_mid + r_side, r_mid - r_side], axis=1) * float(np.prod(trace["correction"]))


def detector(s: np.ndarray, cfg, true_peak: bool) -> np.ndarray:
    if true_peak:
        return true_peak_oracle.true_peak_detector(s, port.config_from(cfg).internal_sample_rate)
    return np.abs(s).max(axis=1)


def envelope(D: np.ndarray, cfg) -> np.ndarray:
    """port.limit's gain with its rectifier fed D (ones where its early-out applies)."""
    cfg_o = port.config_from(cfg)
    thr = cfg_o.threshold
    r = np.maximum(D, thr) / thr
    if np.all(np.isclose(r, 1.0)):
        return np.ones_like(D)
    g = 1.0 - 1.0 / r
    k = port.limiter_coefficients(cfg_o)
    a_env = port.centred_max(g, k["reach"])
    g_att = port.one_pole_forward_backward(a_env, k["c"])
    h_env = port.trailing_max(a_env, k["hold"])
    hold_out = signal.lfilter(k["bh"], k["ah"], h_env)
    rel_out = signal.lfilter(k["br"], k["ar"], np.maximum(h_env, hold_out))
    return 1.0 - np.maximum(np.maximum(g, g_att), np.maximum(hold_out, rel_out))


@contextlib.contextmanager
def _linked_limiter(D: np.ndarray):
    """loudness_target_oracle's y(x) with the limiter reading D * 10^(x/20) instead of s's own detector."""
    plain = loudness_target_oracle.limited

    def limited(s, x, cfg):
        k = 10.0 ** (x / 20.0)
        return np.asarray(s, np.float64) * k * envelope(D * k, cfg)[:, None]

    loudness_target_oracle.limited = limited
    try:
        yield
    finally:
        loudness_target_oracle.limited = plain


def main_versions(targets: list, reference: np.ndarray, cfg, need_default=True, need_no_limiter=False,
                  need_no_limiter_normalized=False, loudness_target: float | None = None, trace: dict | None = None):
    """-> one (limited, plain, normalized) per target (targets[0] is the main), None where not requested.  With
    loudness_target the limited outputs are y_v(x*) = s_v 10^(x*/20) e(x*) from the main's search; the search's dict
    goes into trace['search']."""
    true_peak = bool(getattr(cfg, "true_peak", False))
    cfg_o = port.config_from(cfg)
    tr = {}
    port.main(np.asarray(targets[0], np.float64), np.asarray(reference, np.float64), cfg_o, need_default=False,
              need_no_limiter=True, trace=tr)
    ss = [chain(x, tr) for x in targets]
    D = np.max(np.stack([detector(s, cfg, true_peak) for s in ss]), axis=0)
    limited = [None] * len(ss)
    if need_default and loudness_target is not None:
        with _linked_limiter(D):
            found = loudness_target_oracle.search(ss[0], cfg, loudness_target)
        k = 10.0 ** (found["gain_db"] / 20.0)
        e = envelope(D * k, cfg)
        limited = [s * k * e[:, None] for s in ss]
        tr["search"] = found
    elif need_default:
        e = envelope(D, cfg)
        limited = [s * e[:, None] * tr["final_coef"] for s in ss]
    coef = max(cfg_o.min_value, float(D.max()) / cfg_o.threshold)
    outs = [(lim, s if need_no_limiter else None, s / coef if need_no_limiter_normalized else None)
            for lim, s in zip(limited, ss)]
    if trace is not None:
        trace.update(tr, s=ss, D=D)
    return outs
