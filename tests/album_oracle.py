"""Float64 restatement of album mastering (stages.main_album, mgb_album_match; DESIGN.md section 4 "Album mastering")
for the tests, on top of oracle/port.py.

An album is K stereo targets at the internal rate and one reference.  Every track keeps its own piece layout; the level
statistics, the target spectra and every RMS-correction step pool the pieces of all tracks, each piece counting once;
one FIR and one gain then apply to every track, and the limiter and the normalisation run per track.
"""
from __future__ import annotations

import math

import numpy as np

import port
import true_peak_oracle


def pooled_match(rmses: list) -> tuple:
    """The loud mask of every track and the match RMS over the union of their pieces (match_levels.py:62-71)."""
    allr = np.concatenate(rmses)
    avg = math.sqrt(float(allr @ allr) / allr.shape[0])
    masks = [r >= avg for r in rmses]
    sel = allr[allr >= avg]
    return masks, math.sqrt(float(sel @ sel) / sel.shape[0])


def album_spectrum(values: list, pieces: list, masks: list, F: int) -> np.ndarray:
    """Mean |rfft| / F over every boxcar frame of every loud piece of every track (match_frequencies.py:30-42 cut per
    track)."""
    total, count = 0.0, 0
    for v, piece, mask in zip(values, pieces, masks):
        frames = piece // F
        u = v[: piece * mask.shape[0]].reshape(mask.shape[0], piece)[mask][:, : frames * F].reshape(-1, F)
        total = total + (np.abs(np.fft.rfft(u, axis=-1)) / F).sum(axis=0)
        count += u.shape[0]
    return total / count


def main_album(targets: list, reference: np.ndarray, cfg, need_default=True, need_no_limiter=False,
               need_no_limiter_normalized=False, trace: dict | None = None):
    """-> one (limited, plain, normalized) per track, None where not requested.  Config(true_peak=True) limits and
    normalises on the true-peak detector (tests/true_peak_oracle.py)."""
    true_peak = bool(getattr(cfg, "true_peak", False))
    cfg = port.config_from(cfg)
    F = cfg.fft_size
    reference, final_coef = port.normalize(np.asarray(reference, np.float64), cfg.threshold, cfg.min_value, False)
    ra = port.analyze(reference, cfg)
    tas = [port.analyze(np.asarray(t, np.float64), cfg) for t in targets]
    masks, match = pooled_match([ta["rmses"] for ta in tas])
    c0 = ra["match_rms"] / max(cfg.min_value, match)
    firs = {}
    for name in ("mid", "side"):
        at = album_spectrum([ta[name] * c0 for ta in tas], [ta["piece"] for ta in tas], masks, F)
        ar = port.average_spectrum(ra[name], ra["piece"], ra["mask"], F)
        firs[name] = port.design_fir(at, ar, cfg)
    r_mids = [port.convolve_same(ta["mid"] * c0, firs["mid"]) for ta in tas]
    r_sides = [port.convolve_same(ta["side"] * c0, firs["side"]) for ta in tas]
    gain, coefs = 1.0, []
    for _ in range(cfg.rms_correction_steps):
        rms = [port.piece_rms(np.clip(m * gain, -1.0, 1.0), ta["piece"], ta["divisions"]) for m, ta in zip(r_mids, tas)]
        _, m = pooled_match(rms)
        c = ra["match_rms"] / max(cfg.min_value, m)
        coefs.append(c)
        gain *= c
    outs = []
    for r_mid, r_side in zip(r_mids, r_sides):
        result = np.stack([r_mid + r_side, r_mid - r_side], axis=1) * gain
        limited = normalized = None
        if true_peak:
            if need_default:
                limited = true_peak_oracle.limit(result, cfg) * final_coef
            if need_no_limiter_normalized:
                peak = float(true_peak_oracle.true_peak_detector(result, cfg.internal_sample_rate).max())
                normalized = result / max(cfg.min_value, peak / cfg.threshold)
        else:
            if need_default:
                limited = port.limit(result, cfg) * final_coef
            if need_no_limiter_normalized:
                normalized, _ = port.normalize(result, cfg.threshold, cfg.min_value, True)
        outs.append((limited, result if need_no_limiter else None, normalized))
    if trace is not None:
        trace.update(c0=c0, firs=firs, masks=masks, match=match, correction=coefs, gain=gain, final_coef=final_coef)
    return outs
