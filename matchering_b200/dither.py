"""Dither for 16- and 24-bit results: the shaping filter, designed on the host, and the device parameters.

The quantiser itself is `mgb_pcm_encode_dithered` (csrc/dither.cuh): TPDF dither, optionally noise-shaped by error
feedback with the taps h_1 .. h_K, so that the quantisation error y - x * top is that TPDF-plus-rounding noise (0.25
LSB^2, white) filtered by NTF(z) = 1 - sum_k h_k z^-k.  DESIGN.md §4 "Dither" states the definition.

`shaping_filter(sample_rate)` is a Gerzon-Craven minimum-phase design whose |NTF| follows the threshold of hearing
(Terhardt's approximation): the noise moves out of the ear's most sensitive band, at 2-5 kHz, to where it is heard
least.  Its taps are computed in float64 numpy and cached per rate.
"""
from __future__ import annotations

import functools

import numpy as np

from . import _native

KINDS = (None, "tpdf", "shaped")
SHAPED_TAPS = 12
_GRID = 8192  # M: points of the design grid over [0, sr/2]
_RANGE_DB = 30.0  # the threshold curve is clamped to at most min + 30 dB


def hearing_threshold_db(f_hz) -> np.ndarray:
    """Terhardt's threshold in quiet, dB SPL, at f_hz (clamped below at 20 Hz)."""
    f = np.maximum(np.asarray(f_hz, dtype=np.float64) / 1000.0, 0.02)
    return 3.64 * f ** -0.8 - 6.5 * np.exp(-0.6 * (f - 3.3) ** 2) + 1e-3 * f ** 4


def _design_curve(sample_rate: int):
    """The design grid f_j = j (sr/2) / M, j = 0 .. M, and the threshold on it, clamped to at most min + 30 dB."""
    f = np.arange(_GRID + 1) * (sample_rate / 2.0) / _GRID
    a = hearing_threshold_db(f)
    return f, np.minimum(a, a.min() + _RANGE_DB)


@functools.lru_cache(maxsize=None)
def _shaping_filter(sample_rate: int, taps: int) -> tuple:
    _, a = _design_curve(sample_rate)
    # real cepstrum of the log-magnitude (zero log-mean), folded to causal: the minimum-phase response of |NTF| = 10^(A/20)
    c = np.fft.irfft(a * (np.log(10.0) / 20.0))
    c[0] = 0.0
    folded = np.zeros_like(c)
    folded[1:_GRID] = 2.0 * c[1:_GRID]
    folded[_GRID] = c[_GRID]
    ntf = np.fft.irfft(np.exp(np.fft.rfft(folded)))
    return tuple(float(v) for v in -ntf[1:taps + 1] / ntf[0])


def shaping_filter(sample_rate: int, taps: int = SHAPED_TAPS) -> np.ndarray:
    """The error-feedback taps h_1 .. h_taps (float64) of the shaped dither at `sample_rate`: NTF(z) = 1 - sum h_k z^-k,
    monic and minimum phase before truncation.  Cached per (rate, taps)."""
    if not 1 <= int(taps) <= _native.MGB_MAX_DITHER_TAPS:
        raise ValueError(f"taps must be in [1, {_native.MGB_MAX_DITHER_TAPS}]")
    return np.array(_shaping_filter(int(sample_rate), int(taps)))


def weighted_noise_db(h, sample_rate: int, top_hz: float = 20000.0) -> float:
    """Noise power of the shaped error weighted by 10^(-A/10) (A: the design's clamped threshold) over
    0 .. min(top_hz, sr/2), against flat TPDF's, in dB."""
    f, a = _design_curve(sample_rate)
    keep = f <= top_hz
    w = 10.0 ** (-a[keep] / 10.0)
    ntf = np.fft.rfft(np.concatenate([[1.0], -np.asarray(h, dtype=np.float64)]), 2 * _GRID)[keep]
    return float(10.0 * np.log10(np.sum(w * np.abs(ntf) ** 2) / np.sum(w)))


def check_kind(dither) -> None:
    if dither not in KINDS:
        raise ValueError(f"dither must be one of {KINDS}, not {dither!r}")


def params(dither: str, sample_rate: int, seed: int = 0) -> _native.DitherParams:
    """The C parameters of a dither kind ("tpdf" or "shaped") at a rate."""
    check_kind(dither)
    if dither is None:
        raise ValueError("no dither to describe")
    p = _native.DitherParams()
    p.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    h = shaping_filter(sample_rate) if dither == "shaped" else np.zeros(0)
    p.taps = len(h)
    for k, v in enumerate(h):
        p.h[k] = float(v)
    return p
