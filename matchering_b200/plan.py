"""Config-only tables for the device pipeline (the "plan", like an FFT plan).

Everything here depends on `Config` alone -- never on audio data -- and is computed once per
Config on the host in float64, then uploaded.  Data-dependent arithmetic all runs in the CUDA
kernels (matchering_b200/csrc).  What is tabulated, and the reference code it serves:

* the two not-a-knot cubic splines of ``__smooth_exponentially``
  (matchering/stage_helpers/match_frequencies.py:45-75, scipy ``interp1d(kind="cubic")``):
  the knots are Config-only, so the tridiagonal system of the spline moments is LU-factorised
  here (Thomas factors) and the evaluation points are reduced to an interval index plus four
  weights; the kernel only does the right-hand side, two substitution sweeps and a 4-term dot;
* the LOWESS bookkeeping (matchering/dsp.py:103-106; statsmodels ``_smoothers_lowess``): which
  abscissae get a local regression, each neighbourhood's left edge, and which pair of regression
  points brackets every skipped abscissa (the ``delta`` interpolation);
* the symmetric Hann window (match_frequencies.py:99) and the limiter constants
  (matchering/limiter/hyrax.py:44-72, matchering/utils.py:50-55).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
from scipy import signal as _signal

SUPPORTED_FFT_SIZES = (512, 1024, 2048, 4096, 8192, 16384)
OPERATOR_MAX_FFT_SIZE = 8192  # above: no Config-only smoothing matrix (its row bands would be 80 MB), direct chain per track
NATIVE_EDGE = 0.9  # native-rate jobs: the analysis curve is trusted up to 0.9 * R/2, below the resampler's roll-off


class UnsupportedConfig(NotImplementedError):
    """A Config the reference accepts but this build has no kernel for (fails loudly)."""


# ------------------------------------------------------------------------------------------------
# splines
# ------------------------------------------------------------------------------------------------
def spline_factor(knots: np.ndarray):
    """Thomas factors of the not-a-knot moment system on `knots` (n >= 4).

    Unknowns are the interior second derivatives M_1..M_{n-2}; the two not-a-knot conditions
    (third derivative continuous across knots 1 and n-2) eliminate M_0 and M_{n-1}:
        M_0     = e0*M_1     + e1*M_2
        M_{n-1} = e2*M_{n-2} + e3*M_{n-3}
    Returns hinv [n-1], lu [3, n-2] (sub/den, 1/den, sup/den) and end [4] = (e0, e1, e2, e3).
    Row i (1-based interior index) of the system is
        h_{i-1} M_{i-1} + 2 (h_{i-1}+h_i) M_i + h_i M_{i+1} = 6 ((y_{i+1}-y_i)/h_i - (y_i-y_{i-1})/h_{i-1}).
    """
    x = np.asarray(knots, dtype=np.float64)
    n = len(x)
    if n < 4:
        raise ValueError("not-a-knot cubic needs at least 4 knots")
    h = np.diff(x)
    m = n - 2
    a = h[:-1].copy()                  # sub-diagonal   (row i uses h_{i-1})
    b = 2.0 * (h[:-1] + h[1:])         # diagonal
    c = h[1:].copy()                   # super-diagonal (row i uses h_i)
    e0 = 1.0 + h[0] / h[1]
    e1 = -h[0] / h[1]
    e2 = 1.0 + h[-1] / h[-2]
    e3 = -h[-1] / h[-2]
    # fold M_0 into row 1 and M_{n-1} into row n-2
    b[0] += a[0] * e0
    c[0] += a[0] * e1
    a[0] = 0.0
    b[-1] += c[-1] * e2
    a[-1] += c[-1] * e3
    c[-1] = 0.0
    fa = np.zeros(m)
    invden = np.zeros(m)
    cp = np.zeros(m)
    den = b[0]
    invden[0] = 1.0 / den
    cp[0] = c[0] / den
    for i in range(1, m):
        den = b[i] - a[i] * cp[i - 1]
        invden[i] = 1.0 / den
        fa[i] = a[i] / den
        cp[i] = c[i] / den
    return 1.0 / h, np.stack([fa, invden, cp]), np.array([e0, e1, e2, e3])


def spline_eval_table(knots: np.ndarray, points: np.ndarray):
    """Interval index and the weights of (y_i, y_{i+1}, M_i, M_{i+1}) for each evaluation point.

    S(x) = A y_i + B y_{i+1} + ((A^3 - A) M_i + (B^3 - B) M_{i+1}) h^2 / 6,
    A = (x_{i+1} - x)/h, B = (x - x_i)/h.  Points outside the knot range use the end interval
    (cubic extrapolation, what BSpline / interp1d(fill_value="extrapolate") do).
    """
    x = np.asarray(knots, dtype=np.float64)
    p = np.asarray(points, dtype=np.float64)
    idx = np.clip(np.searchsorted(x, p, side="right") - 1, 0, len(x) - 2).astype(np.int32)
    h = x[idx + 1] - x[idx]
    A = (x[idx + 1] - p) / h
    B = (p - x[idx]) / h
    w = np.stack([A, B, (A ** 3 - A) * h * h / 6.0, (B ** 3 - B) * h * h / 6.0], axis=1)
    return idx, np.ascontiguousarray(w)


# ------------------------------------------------------------------------------------------------
# LOWESS bookkeeping
# ------------------------------------------------------------------------------------------------
def lowess_tables(n: int, frac: float, delta: float):
    """One LOWESS pass (it = 0) on x = linspace(0, 1, n) as a Config-only linear operator.

    With no robustness iterations every fitted value is a fixed linear combination of the k
    ordinates in its neighbourhood: the tricube weights, the weighted mean and variance of the
    abscissae (statsmodels calculate_weights / calculate_y_fit) depend on x only.  So the host
    tabulates, per regression point f (the points statsmodels' update_indices visits):
        fit_idx[f], fit_left[f]   position and left edge of the neighbourhood [left, left+k)
        rows[row_idx[f]]          the k coefficients, fit = rows . y[left : left+k]
    (on the uniform grid all interior rows coincide, so rows are stored once) and, per abscissa j,
        seg[j]    index of the last regression point <= j
        alpha[j]  weight of the NEXT regression point in the `delta` interpolation (0 at a
                  regression point): y_fit[j] = alpha*fit[seg+1] + (1-alpha)*fit[seg].
    """
    x = np.linspace(0, 1, n)
    k = int(frac * n + 1e-10)
    if not 2 <= k <= n:
        raise UnsupportedConfig(f"lowess_frac={frac} gives a neighbourhood of {k} points (need 2..{n})")
    fit_idx, lefts = [], []
    i, left, right = 0, 0, k
    while True:
        while right < n and (x[i] - x[left]) > (x[right] - x[i]):  # update_neighborhood
            left += 1
            right += 1
        fit_idx.append(i)
        lefts.append(left)
        last_fit = i                                               # update_indices
        cut = x[last_fit] + delta
        kk = last_fit
        for kk in range(last_fit + 1, n):
            if x[kk] > cut:
                break
        i = max(kk - 1, last_fit + 1)
        if last_fit >= n - 1:
            break
    fit_idx = np.asarray(fit_idx, dtype=np.int32)
    lefts = np.asarray(lefts, dtype=np.int32)
    rows, row_idx = [], np.zeros(len(fit_idx), dtype=np.int32)
    for f, (i, left) in enumerate(zip(fit_idx, lefts)):
        xs = x[left:left + k]
        dist = np.abs(xs - x[i])
        radius = max(dist[0], dist[-1])
        w = dist / radius
        w = 1.0 - w * w * w
        w = w * w * w
        w[dist >= radius] = 0.0
        sw = w.sum()
        if sw <= 0.0 or np.count_nonzero(w) == 1:      # regression "not ok": fit = y[i]
            row = np.zeros(k)
            row[i - left] = 1.0
        else:
            w = w / sw
            xbar = np.sum(w * xs)
            sqdev = np.sum(w * (xs - xbar) ** 2)
            row = w * (1.0 + (x[i] - xbar) * (xs - xbar) / sqdev)
        if rows and np.abs(row - rows[-1]).max() <= 4e-16 * np.abs(row).max():
            row_idx[f] = len(rows) - 1                  # same operator as the previous point
        else:
            rows.append(row)
            row_idx[f] = len(rows) - 1
    seg = (np.searchsorted(fit_idx, np.arange(n), side="right") - 1).astype(np.int32)
    alpha = np.zeros(n)
    for j in range(n):
        fa = fit_idx[seg[j]]
        if fa != j:
            fb = fit_idx[seg[j] + 1]
            alpha[j] = (x[j] - x[fa]) / (x[fb] - x[fa])
    return dict(lw_fit_idx=fit_idx, lw_fit_left=lefts, lw_seg=seg, lw_alpha=alpha, lw_rows=np.stack(rows),
                lw_row_idx=row_idx), k


# ------------------------------------------------------------------------------------------------
# the smoothing operator's band
# ------------------------------------------------------------------------------------------------
def band_operator(dense: np.ndarray, relative_floor: float = 1e-18):
    """Row bands of the dense smoothing operator S (mgb_plan_build_operator): spline -> LOWESS -> spline
    has finite reach (a 307-point LOWESS window on the log grid, spline influence decaying 0.27^n), so
    each row is non-negligible only on a contiguous stretch of columns.  Entries outside the stretch
    are below `relative_floor` * max|S| (2e-15 of the largest matching-curve value in the worst case,
    less than the float64 rounding of the row sums themselves).
    -> (values float64 [total], rows int32 [n][4] = (offset into values, even; first column; count; 0))"""
    n = dense.shape[0]
    keep = np.abs(dense) > relative_floor * np.abs(dense).max()
    any_ = keep.any(axis=1)
    lo = np.where(any_, keep.argmax(axis=1), 0).astype(np.int64)
    hi = np.where(any_, n - keep[:, ::-1].argmax(axis=1), 0).astype(np.int64)
    width = hi - lo
    start = np.zeros(n + 1, dtype=np.int64)
    np.cumsum((width + 1) // 2 * 2, out=start[1:])   # every row starts on a 16-byte boundary
    values = np.zeros(max(2, int(start[-1])), dtype=np.float64)
    for r in range(n):
        values[start[r]:start[r] + width[r]] = dense[r, lo[r]:hi[r]]
    rows = np.stack([start[:-1], lo, width, np.zeros(n, dtype=np.int64)], axis=1).astype(np.int32)
    return values, np.ascontiguousarray(rows)


# ------------------------------------------------------------------------------------------------
# limiter constants
# ------------------------------------------------------------------------------------------------
@dataclass
class LimiterConstants:
    threshold: float
    reach: int
    hold: int
    warmup: int
    attack_c: float
    hold_b: np.ndarray
    hold_a: np.ndarray
    release_b: np.ndarray
    release_a: np.ndarray
    true_peak: int = 0  # mgb_limiter_params.true_peak: 0 (sample peaks) or the detector's oversampling factor L


MAX_FILTER_ORDER = 2   # MGB_MAX_FILTER_ORDER


def limiter_constants(config) -> LimiterConstants:
    sr = config.internal_sample_rate
    lim = config.limiter
    attack = int(sr * lim.attack * 1e-3)   # utils.ms_to_samples, utils.py:50-51
    hold = int(sr * lim.hold * 1e-3)
    if attack < 1:
        raise UnsupportedConfig("limiter attack shorter than one sample")
    if hold < 3:
        # hyrax.py:38-40 slices with [:-0] when (hold-1)//2 == 0 and returns an empty array
        raise UnsupportedConfig("limiter hold shorter than 3 samples breaks the reference itself")
    if lim.hold_filter_order > MAX_FILTER_ORDER or lim.release_filter_order > MAX_FILTER_ORDER:
        raise UnsupportedConfig(
            f"hold / release filter orders above {MAX_FILTER_ORDER} have no kernel: at the limiter's cut-offs scipy's "
            "transfer-function form (what the reference runs) is ill-conditioned from order 3 on -- its own rounding "
            "noise exceeds the parity bound, order 4 release is unstable -- so there is no reference result to match")
    reach = (attack + 1 if not attack & 1 else attack) - 1  # make_odd(attack) - 1, utils.py:54-55
    c = math.exp(lim.attack_filter_coefficient / attack)
    if not 0.0 < c < 1.0:
        raise UnsupportedConfig("attack_filter_coefficient must be negative (a decaying one-pole)")
    warmup = int(math.ceil(math.log(1e-8) / math.log(c)))
    warmup = max(32, (warmup + 31) // 32 * 32)  # (the halo kernel's warm-up; wider windows take the wide-window path)
    bh, ah = _signal.butter(lim.hold_filter_order, lim.hold_filter_coefficient, fs=sr)
    br, ar = _signal.butter(lim.release_filter_order, lim.release_filter_coefficient / lim.release, fs=sr)
    # Config(true_peak=True): the meter's oversampling at this rate (loudness_constants)
    tp = (4 if sr < 96000 else (2 if sr < 192000 else 1)) if getattr(config, "true_peak", False) else 0
    return LimiterConstants(config.threshold, reach, hold, warmup, c, bh, ah, br, ar, tp)


# ------------------------------------------------------------------------------------------------
# loudness meter constants (ITU-R BS.1770-4), depending on the sample rate only
# ------------------------------------------------------------------------------------------------
@dataclass
class LoudnessConstants:
    sample_rate: int
    block: int          # sub-block of 100 ms: (fs + 5) // 10 frames
    oversample: int     # true-peak oversampling factor
    shelf_b: np.ndarray
    shelf_a: np.ndarray
    highpass_b: np.ndarray
    highpass_a: np.ndarray
    tp_taps: np.ndarray  # 12 * oversample + 1 interpolator taps


LOUDNESS_MIN_RATE, LOUDNESS_MAX_RATE = 8000, 384000


def _k_weighting_section(fs: int, f0: float, q: float):
    k = math.tan(math.pi * f0 / fs)
    a0 = 1.0 + k / q + k * k
    return k, a0, np.array([1.0, 2.0 * (k * k - 1.0) / a0, (1.0 - k / q + k * k) / a0])


def loudness_constants(fs: int) -> LoudnessConstants:
    """K-weighting sections for any rate from their analog prototypes (as libebur128 and pyloudnorm derive them;
    at 48 kHz they reproduce BS.1770's published coefficients) and the true-peak interpolator."""
    fs = int(fs)
    if not LOUDNESS_MIN_RATE <= fs <= LOUDNESS_MAX_RATE:
        raise ValueError(f"loudness: sample rate {fs} outside [{LOUDNESS_MIN_RATE}, {LOUDNESS_MAX_RATE}]")
    # high-shelf (the head's acoustic effect)
    gain_db, f0, q = 3.999843853973347, 1681.974450955533, 0.7071752369554196
    k, a0, shelf_a = _k_weighting_section(fs, f0, q)
    vh = 10.0 ** (gain_db / 20.0)
    vb = vh ** 0.4996667741545416
    shelf_b = np.array([vh + vb * k / q + k * k, 2.0 * (k * k - vh), vh - vb * k / q + k * k]) / a0
    # high-pass (RLB weighting)
    _, _, highpass_a = _k_weighting_section(fs, 38.13547087602444, 0.5003270373238773)
    highpass_b = np.array([1.0, -2.0, 1.0])
    os_ = 4 if fs < 96000 else (2 if fs < 192000 else 1)
    m = np.arange(12 * os_ + 1)
    taps = np.sinc((m - 6 * os_) / os_) * np.kaiser(12 * os_ + 1, 8.0)
    return LoudnessConstants(fs, (fs + 5) // 10, os_, shelf_b, shelf_a, highpass_b, highpass_a, taps)


# ------------------------------------------------------------------------------------------------
# the plan
# ------------------------------------------------------------------------------------------------
@dataclass
class PlanTables:
    sample_rate: int
    fft_size: int
    n_lin: int
    n_log: int
    rms_correction_steps: int
    lowess_k: int
    lowess_it: int
    max_piece_size: float
    threshold: float
    min_value: float
    limiter: LimiterConstants
    arrays: dict = field(default_factory=dict)  # name -> numpy array, names = mgb_plan fields without d_


def config_key(config) -> tuple:
    lim = config.limiter
    return (config.internal_sample_rate, config.fft_size, config.lin_log_oversampling,
            config.rms_correction_steps, float(config.max_piece_size), config.threshold, config.min_value,
            config.lowess_frac, config.lowess_it, config.lowess_delta, lim.attack, lim.hold, lim.release,
            lim.attack_filter_coefficient, lim.hold_filter_order, lim.hold_filter_coefficient,
            lim.release_filter_order, lim.release_filter_coefficient, bool(getattr(config, "true_peak", False)))


def build_tables(config) -> PlanTables:
    F = config.fft_size
    if F not in SUPPORTED_FFT_SIZES:
        raise UnsupportedConfig(f"fft_size={F}: kernels exist for {SUPPORTED_FFT_SIZES}")
    if config.lowess_it > 8:
        raise UnsupportedConfig("lowess_it > 8")
    if config.rms_correction_steps > 16:
        raise UnsupportedConfig("rms_correction_steps > 16")
    sr = config.internal_sample_rate
    half = F // 2
    # match_frequencies.py:46-58
    grid_lin = sr * 0.5 * np.linspace(0, 1, half + 1)
    grid_log = sr * 0.5 * np.logspace(np.log10(4 / F), 0, half * config.lin_log_oversampling + 1)
    n_lin, n_log = len(grid_lin), len(grid_log)
    arrays = {}
    hinv, lu, end = spline_factor(grid_lin)
    idx, w = spline_eval_table(grid_lin, grid_log)
    arrays.update(sa_hinv=hinv, sa_lu=lu, sa_end=end, sa_eval_idx=idx, sa_eval_w=w)
    hinv, lu, end = spline_factor(grid_log)
    idx, w = spline_eval_table(grid_log, grid_lin)
    arrays.update(sb_hinv=hinv, sb_lu=lu, sb_end=end, sb_eval_idx=idx, sb_eval_w=w)
    lw, k = lowess_tables(n_log, config.lowess_frac, config.lowess_delta)
    arrays.update(lw)
    arrays["hann"] = _signal.windows.hann(F)
    for name, arr in arrays.items():
        want = np.int32 if arr.dtype.kind == "i" else np.float64
        arrays[name] = np.ascontiguousarray(arr, dtype=want)
    return PlanTables(sr, F, n_lin, n_log, config.rms_correction_steps, k, int(config.lowess_it), float(config.max_piece_size),
                      config.threshold, config.min_value, limiter_constants(config), arrays)


# ------------------------------------------------------------------------------------------------
# native-rate jobs (Config(native_rate=True); DESIGN.md section 4 "Native-rate masters")
# ------------------------------------------------------------------------------------------------
def native_fft_size(config, rate: int) -> int:
    """F' = F * 2^round(log2(R'/R)): the native FIR keeps the analysis FIR's length in seconds to within a factor of
    sqrt(2), and so its frequency resolution.  UnsupportedConfig where no kernel exists for it."""
    R, F = config.internal_sample_rate, config.fft_size
    size = F * 2.0 ** math.floor(math.log2(rate / R) + 0.5)
    if size not in SUPPORTED_FFT_SIZES:
        raise UnsupportedConfig(f"a {rate} Hz target at internal_sample_rate={R}, fft_size={F} needs a native FIR of "
                                f"{size:.0f} points: kernels exist for {SUPPORTED_FFT_SIZES}")
    return int(size)


def native_config(config, rate: int):
    """The Config stages 2-4 of a native-rate job run under: `config` at `rate`, every seconds-valued field the same
    length in seconds, fft_size = native_fft_size."""
    import copy
    R = config.internal_sample_rate
    out = copy.copy(config)
    out.fft_size = native_fft_size(config, rate)
    out.internal_sample_rate = int(rate)
    for name in ("max_piece_size", "preview_size", "preview_analysis_step", "preview_fade_size"):
        setattr(out, name, getattr(config, name) / R * rate)
    return out


def native_check_length(config, rate: int, frames: int) -> None:
    """A native target must give the native FIR what the analysis FIR needs at R: more frames than F' and pieces
    (match_levels.py:47-59 at R') of at least F' frames.  ValueError otherwise, before anything runs."""
    nc = native_config(config, rate)
    F = nc.fft_size
    piece = int(frames / (int(frames / nc.max_piece_size) + 1))
    if frames <= F or piece < F:
        raise ValueError(f"a target of {frames} frames at {rate} Hz is too short for the native FIR of {F} points "
                         f"(pieces of {piece} frames)")


def native_tables(config, rate: int) -> dict:
    """mgb_plan::d_native_idx / d_native_w of the native plan at `rate`: for j = 0 .. F'/2 at f_j = j R'/F', the
    analysis curve's bin i and weight w of s'[j] = s[i] + w (s[i+1] - s[i]) at position f_j F/R while f_j <= f_e, and
    above f_e (idx -1) the crossfade position t = (f_j - f_e) / (R/2 - f_e), held at 1 from R/2 on.  Entry F'/2 + 1
    is the edge f_e itself."""
    R, F = config.internal_sample_rate, config.fft_size
    Fn = native_fft_size(config, rate)
    hb = Fn // 2 + 1
    f_e = NATIVE_EDGE * R / 2
    f = np.append(np.arange(hb) * (rate / Fn), f_e)
    inside = f <= f_e
    pos = f * (F / R)
    i = np.minimum(np.floor(pos), F // 2 - 1)
    idx = np.where(inside, i, -1).astype(np.int32)
    w = np.where(inside, pos - i, np.minimum((f - f_e) / (R / 2 - f_e), 1.0))
    return {"native_idx": np.ascontiguousarray(idx), "native_w": np.ascontiguousarray(w, dtype=np.float64)}
