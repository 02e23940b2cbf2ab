"""Float64 restatement of a native-rate job (Config(native_rate=True), stages.main_native,
mgb_match_frequencies_native; DESIGN.md section 4 "Native-rate masters") for the tests, on top of oracle/port.py.

Stage 1 and the smoothed matching curve come from the analysis copy (the target resampled to R) exactly as port.main
computes them; the curve is then carried to the native FIR of F' points at R', and the FIR, the RMS correction with
R' pieces and the limiter run on the native target under the derived Config.  The analysis copy is an input: the tests
feed the one the device made, so the resampler's own parity stays out of the comparison.
"""
from __future__ import annotations

import copy
import math

import numpy as np
from scipy import signal

import port

EDGE = 0.9  # f_e = EDGE * R/2


def native_fft_size(R: int, F: int, rate: int) -> int:
    return int(F * 2 ** math.floor(math.log2(rate / R) + 0.5))


def native_cfg(cfg, rate: int):
    """port.OracleConfig at `rate`: F', and max_piece_size the same length in seconds."""
    c = copy.copy(port.config_from(cfg))
    R = c.internal_sample_rate
    c.fft_size = native_fft_size(R, c.fft_size, rate)
    c.max_piece_size = c.max_piece_size / R * rate
    c.internal_sample_rate = rate
    return c


def transplant(s: np.ndarray, R: int, F: int, rate: int) -> np.ndarray:
    """s (F/2 + 1 values at k R/F) -> s' (F'/2 + 1 values at j R'/F'): linear interpolation up to f_e, then a crossfade
    in log gain from g_e = s(f_e) to g_inf = min(g_e, 1) at R/2, then g_inf."""
    Fn = native_fft_size(R, F, rate)
    f = np.arange(Fn // 2 + 1) * (rate / Fn)
    f_e = EDGE * R / 2
    bins = np.arange(len(s), dtype=np.float64)
    g_e = float(np.interp(f_e * F / R, bins, s))
    g_inf = min(g_e, 1.0)
    out = np.interp(f * F / R, bins, s)
    for j in np.nonzero(f > f_e)[0]:
        t = min((f[j] - f_e) / (R / 2 - f_e), 1.0)
        out[j] = math.exp((1 - t) * math.log(g_e) + t * math.log(g_inf)) if g_e > 1.0 else g_e
    return out


def fir_from_curve(s_native: np.ndarray) -> np.ndarray:
    """match_frequencies.py:98-99 at the curve's own length."""
    h = np.fft.irfft(s_native)
    return np.fft.ifftshift(h) * signal.windows.hann(len(h))


def main(native_target: np.ndarray, analysis: np.ndarray, reference, cfg, rate: int, need_default=True,
         need_no_limiter=False, need_no_limiter_normalized=False, trace: dict | None = None, profile=None):
    """-> (limited, no limiter, normalised) at `rate`.  reference: (N, 2) samples, or None with `profile` =
    (avg_mid, avg_side, final_coef, match_rms) of the normalised reference (what a reference profile records)."""
    cfg_o = port.config_from(cfg)
    R, F = cfg_o.internal_sample_rate, cfg_o.fft_size
    ta = port.analyze(np.asarray(analysis, dtype=np.float64), cfg_o)
    if profile is None:
        ref, final_coef = port.normalize(np.asarray(reference, dtype=np.float64), cfg_o.threshold, cfg_o.min_value, False)
        ra = port.analyze(ref, cfg_o)
        match_r = ra["match_rms"]
        avg_r = {name: port.average_spectrum(ra[name], ra["piece"], ra["mask"], F) for name in ("mid", "side")}
    else:
        avg_r = {"mid": profile[0], "side": profile[1]}
        final_coef, match_r = profile[2], profile[3]
    c0 = match_r / max(cfg_o.min_value, ta["match_rms"])
    curves, firs = {}, {}
    for name in ("mid", "side"):
        at = port.average_spectrum(ta[name] * c0, ta["piece"], ta["mask"], F)
        s = port.smooth_matching_curve(avg_r[name] / np.maximum(cfg_o.min_value, at), cfg_o)
        curves[name] = transplant(s, R, F, rate)
        firs[name] = fir_from_curve(curves[name])
    nc = native_cfg(cfg_o, rate)
    mid, side = port.mid_side(np.asarray(native_target, dtype=np.float64))
    r_mid = port.convolve_same(mid * c0, firs["mid"])
    r_side = port.convolve_same(side * c0, firs["side"])
    result = np.stack([r_mid + r_side, r_mid - r_side], axis=1)
    divisions, piece = port.piece_layout(len(mid), nc.max_piece_size)
    for _ in range(nc.rms_correction_steps):
        rm = port.piece_rms(np.clip(r_mid, -1.0, 1.0), piece, divisions)
        _, match, _ = port.loudest_mask_and_match_rms(rm)
        c = match_r / max(nc.min_value, match)
        r_mid = r_mid * c
        result = result * c
    if trace is not None:
        trace.update(c0=c0, curves=curves, firs=firs, final_coef=final_coef, pre_limiter=result, native_cfg=nc)
    out_norm = port.normalize(result, nc.threshold, nc.min_value, True)[0] if need_no_limiter_normalized else None
    out = port.limit(result, nc) * final_coef if need_default else None
    return out, (result if need_no_limiter else None), out_norm
