"""Config / LimiterConfig with the reference's constructor signature, attribute names, unit
conversions and validation (matchering/defaults.py:25-155).  Invalid values raise AssertionError
like the reference's bare asserts do."""
from __future__ import annotations

import math

from .log import debug


def _require(condition: bool, what: str) -> None:
    if not condition:
        raise AssertionError(what)


class LimiterConfig:
    def __init__(self, attack: float = 1, hold: float = 1, release: float = 3000,
                 attack_filter_coefficient: float = -2, hold_filter_order: int = 1,
                 hold_filter_coefficient: float = 7, release_filter_order: int = 1,
                 release_filter_coefficient: float = 800):
        for name, value in (("attack", attack), ("hold", hold), ("release", release)):
            _require(value > 0, f"limiter {name} must be positive (milliseconds)")
        for name, value in (("hold_filter_order", hold_filter_order),
                            ("release_filter_order", release_filter_order)):
            _require(isinstance(value, int) and value > 0, f"limiter {name} must be a positive int")
        self.attack = attack
        self.hold = hold
        self.release = release
        self.attack_filter_coefficient = attack_filter_coefficient
        self.hold_filter_order = hold_filter_order
        self.hold_filter_coefficient = hold_filter_coefficient
        self.release_filter_order = release_filter_order
        self.release_filter_coefficient = release_filter_coefficient


class Config:
    def __init__(self, internal_sample_rate: int = 44100, max_length: float = 15 * 60,
                 max_piece_size: float = 15, threshold: float = (2 ** 15 - 61) / 2 ** 15,
                 min_value: float = 1e-6, fft_size: int = 4096, lin_log_oversampling: int = 4,
                 rms_correction_steps: int = 4, clipping_samples_threshold: int = 8,
                 limited_samples_threshold: int = 128, allow_equality: bool = False,
                 lowess_frac: float = 0.0375, lowess_it: int = 0, lowess_delta: float = 0.001,
                 preview_size: float = 30, preview_analysis_step: float = 5, preview_fade_size: float = 1,
                 preview_fade_coefficient: float = 8, temp_folder: str = None,
                 limiter: LimiterConfig = None, true_peak: bool = False, loudness_target: float = None,
                 native_rate: bool = False):
        sr = internal_sample_rate
        _require(isinstance(sr, int) and sr > 0, "internal_sample_rate must be a positive int")
        if sr != 44100:
            debug("Using an internal sample rate other than 44100 has not been tested properly! "
                  "Use it at your own risk!")
        frame_seconds = fft_size / sr
        _require(max_length > 0 and max_length > frame_seconds, "max_length must exceed one FFT frame")
        _require(min_value < threshold < 1, "threshold must lie in (min_value, 1)")
        _require(0 < min_value < 0.1, "min_value must lie in (0, 0.1)")
        _require(max_piece_size > 0 and frame_seconds < max_piece_size < max_length,
                 "max_piece_size must lie between one FFT frame and max_length")
        _require(fft_size > 1 and math.log2(fft_size).is_integer(), "fft_size must be a power of two")
        _require(isinstance(lin_log_oversampling, int) and lin_log_oversampling > 0,
                 "lin_log_oversampling must be a positive int")
        _require(isinstance(rms_correction_steps, int) and rms_correction_steps >= 0,
                 "rms_correction_steps must be a non-negative int")
        _require(isinstance(clipping_samples_threshold, int) and isinstance(limited_samples_threshold, int),
                 "sample-count thresholds must be ints")
        _require(clipping_samples_threshold >= 0 and limited_samples_threshold > 0
                 and limited_samples_threshold > clipping_samples_threshold,
                 "need 0 <= clipping_samples_threshold < limited_samples_threshold")
        _require(isinstance(allow_equality, bool), "allow_equality must be a bool")
        _require(lowess_frac > 0 and lowess_delta >= 0 and isinstance(lowess_it, int) and lowess_it >= 0,
                 "bad LOWESS parameters")
        _require(preview_size > 5 and preview_analysis_step > 1 and preview_fade_size > 0
                 and preview_fade_coefficient >= 2, "bad preview parameters")
        _require(temp_folder is None or isinstance(temp_folder, str), "temp_folder must be a str")
        if limiter is None:
            limiter = _DEFAULT_LIMITER
        _require(isinstance(limiter, LimiterConfig), "limiter must be a LimiterConfig")
        _require(isinstance(true_peak, bool), "true_peak must be a bool")
        _require(isinstance(native_rate, bool), "native_rate must be a bool")
        _require(loudness_target is None or (isinstance(loudness_target, (int, float)) and not isinstance(loudness_target, bool)
                                             and math.isfinite(loudness_target) and -70 < loudness_target < 0),
                 "loudness_target must be None or a finite LUFS value in (-70, 0)")

        self.internal_sample_rate = sr
        self.max_length = max_length
        self.threshold = threshold
        self.min_value = min_value
        self.max_piece_size = max_piece_size * sr  # kept in samples, as the reference does
        self.fft_size = fft_size
        self.lin_log_oversampling = lin_log_oversampling
        self.rms_correction_steps = rms_correction_steps
        self.clipping_samples_threshold = clipping_samples_threshold
        self.limited_samples_threshold = limited_samples_threshold
        self.allow_equality = allow_equality
        self.lowess_frac = lowess_frac
        self.lowess_it = lowess_it
        self.lowess_delta = lowess_delta
        self.preview_size = preview_size * sr
        self.preview_analysis_step = preview_analysis_step * sr
        self.preview_fade_size = preview_fade_size * sr
        self.preview_fade_coefficient = preview_fade_coefficient
        self.temp_folder = temp_folder
        self.limiter = limiter
        # True: the limiter, its early-out and the normalised output hold `threshold` on the true peak (the signal
        # between samples, through the loudness meter's interpolator) instead of the sample peak
        self.true_peak = true_peak
        # LUFS: the limited outputs are driven into the limiter until they read this integrated loudness (a search on
        # the device; final_amplitude_coefficient is not applied there).  None: the reference's level, as before
        self.loudness_target = None if loudness_target is None else float(loudness_target)
        # True: mg.process masters a target whose file rate differs from internal_sample_rate at that rate.  The match
        # is still analysed on a copy resampled to internal_sample_rate; the FIR, the corrections, the limiter and every
        # result then run on the target's own samples.  False: the reference's behaviour, every result at the internal rate
        self.native_rate = native_rate


_DEFAULT_LIMITER = LimiterConfig()  # shared default instance, like the reference's default argument
