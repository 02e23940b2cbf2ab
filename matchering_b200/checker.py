"""mg.check (reference: matchering/checker.py:30-142): input validation in front of the hot path, for arrays
that are on the host (device_io.check_on_device is the same for signals already on the device); resampling
runs on the device either way."""
import numpy as np

from .defaults import Config
from .log import Code, ModuleError, debug, info, warning
from .utils import time_str


def _resample(array, old_rate: int, new_rate: int):
    """matchering/checker.py:42: resampy.resample(array, old_rate, new_rate, axis=0) -- here the device kernel
    (csrc/resample.cu) with resampy's kaiser_best table rebuilt from its documented parameters."""
    from .resample import resample
    return resample(array, int(old_rate), int(new_rate))


def _count_max_peaks(array):
    peak = np.abs(array).max()
    hits = np.count_nonzero(np.isclose(np.abs(array), peak))
    return peak, hits


def peak_warning(peak: float, hits: int, config: Config):
    """matchering/checker.py:75-87: nothing unless more than `clipping_samples_threshold` samples sit at
    the peak; then CLIPPING when the peak is (close to) full scale, else LIMITER when there are more
    than `limited_samples_threshold` of them.  -> the warning Code or None (shared by the host and the
    device route)."""
    if hits > config.clipping_samples_threshold:
        if np.isclose(peak, 1.0):
            return Code.WARNING_TARGET_IS_CLIPPING
        if hits > config.limited_samples_threshold:
            return Code.WARNING_TARGET_LIMITER_IS_APPLIED
    return None


def check(array: np.ndarray, sample_rate: int, config: Config, name: str, native: bool = False):
    """matchering/checker.py:90-137, in the reference's order: length at the SOURCE rate (minimum
    scaled by the rate ratio, :99), channels, resampling, then (target only) clipping / limiter.
    native (the target of a Config(native_rate=True) job): -> (array, sample_rate, the stereo signal at its own
    rate), and a resampled target is only its analysis copy, which is logged, not warned about."""
    name = name.upper()
    is_target = name == "TARGET"
    frames, channels = array.shape[0], array.shape[1]
    debug(f"{name} audio length: {frames} samples ({time_str(frames, sample_rate)})")
    if frames > config.max_length * sample_rate:
        raise ModuleError(Code.ERROR_TARGET_LENGTH_IS_EXCEEDED if is_target
                          else Code.ERROR_REFERENCE_LENGTH_LENGTH_IS_EXCEEDED)
    if frames < config.fft_size * sample_rate // config.internal_sample_rate:
        raise ModuleError(Code.ERROR_TARGET_LENGTH_IS_TOO_SMALL if is_target
                          else Code.ERROR_REFERENCE_LENGTH_LENGTH_TOO_SMALL)
    if channels == 1:
        info(Code.INFO_TARGET_IS_MONO if is_target else Code.INFO_REFERENCE_IS_MONO)
        array = np.repeat(array, 2, axis=1)
    elif channels != 2:
        raise ModuleError(Code.ERROR_TARGET_NUM_OF_CHANNELS_IS_EXCEEDED if is_target
                          else Code.ERROR_REFERENCE_NUM_OF_CHANNELS_IS_EXCEEDED)
    source = array
    if sample_rate != config.internal_sample_rate:
        debug(f"Resampling {name} audio from {sample_rate} Hz to {config.internal_sample_rate} Hz...")
        array = _resample(array, sample_rate, config.internal_sample_rate)
        if native:
            debug(resampled_for_analysis(sample_rate, config))
        else:
            (warning if is_target else info)(
                Code.WARNING_TARGET_IS_RESAMPLED if is_target else Code.INFO_REFERENCE_IS_RESAMPLED)
        sample_rate = config.internal_sample_rate
    if is_target:
        code = peak_warning(*_count_max_peaks(array), config)
        if code is not None:
            warning(code)
    return (array, sample_rate, source) if native else (array, sample_rate)


def resampled_for_analysis(rate: int, config: Config) -> str:
    return (f"Only the TARGET's analysis copy was resampled to {config.internal_sample_rate} Hz: "
            f"the TARGET is mastered at its own {rate} Hz")


def check_equality(target: np.ndarray, reference: np.ndarray) -> None:
    if target.shape == reference.shape and np.allclose(target, reference):
        raise ModuleError(Code.ERROR_TARGET_EQUALS_REFERENCE)
