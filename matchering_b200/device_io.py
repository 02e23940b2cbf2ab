"""File boundary on the device (SURVEY.md section 8f, items 1, 2 and 4): when a WAV file holds 16/24-bit PCM
(at any sample rate), its raw samples go to the GPU as they are, are decoded there (mgb_pcm_decode),
resampled to the internal rate there if need be (mgb_resample), checked there (mgb_check_peaks /
mgb_check_equality, the reductions of matchering/checker.py) and never exist as a float array on the
host.  Anything else (other formats, more than two channels) takes the reference's host route through
loader/checker.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _native, wavio
from .checker import peak_warning, resampled_for_analysis
from .defaults import Config
from .engine import _require_cuda, _stream_ptr
from .log import Code, ModuleError, debug, info, warning
from .results import real_soundfile
from .utils import time_str


def load_to_device(file: str, file_type: str, config: Config):
    """-> float32 CUDA tensor (frames, channels) decoded on the device, or None when the file is not
    eligible for the device route (the caller then uses loader.load + checker.check)."""
    if real_soundfile() is not None or not file.lower().endswith(".wav"):
        return None
    from .engine import HostIO
    _require_cuda()
    try:
        got = wavio.read_pcm(file, HostIO.get().pool.array)  # into pinned memory: the upload below is one DMA
    except OSError:
        return None
    if got is None:
        return None
    raw, rate, channels, bits = got
    if channels > 2:
        return None
    debug(f"Loading the {file_type.upper()} file: '{file}'... ({bits}-bit PCM, decoded on the device)")
    lib = _native.load()
    device = torch.device("cuda", torch.cuda.current_device())
    d_raw = torch.from_numpy(raw).to(device)
    frames = raw.shape[0]
    out = torch.empty((frames, channels), dtype=torch.float32, device=device)
    _native.check(lib, lib.mgb_pcm_decode(d_raw.data_ptr(), bits, out.data_ptr(), frames * channels, _stream_ptr(device)))
    debug(f"The {file_type.upper()} file is loaded")
    return out, rate


def check_on_device(audio: torch.Tensor, config: Config, name: str, sample_rate: int = None, native: bool = False):
    """matchering/checker.py:90-137 for a signal that is already on the device, in the reference's order: length
    limits at the SOURCE rate, mono -> stereo, resampling to the internal rate (csrc/resample.cu), and (target
    only) the clipping / limiter detection.  native (the target of a Config(native_rate=True) job): -> (audio, the
    stereo signal at its own rate), as checker.check."""
    name = name.upper()
    is_target = name == "TARGET"
    frames, channels = audio.shape
    sr = config.internal_sample_rate
    sample_rate = sr if sample_rate is None else int(sample_rate)
    debug(f"{name} audio length: {frames} samples ({time_str(frames, sample_rate)})")
    if frames > config.max_length * sample_rate:
        raise ModuleError(Code.ERROR_TARGET_LENGTH_IS_EXCEEDED if is_target
                          else Code.ERROR_REFERENCE_LENGTH_LENGTH_IS_EXCEEDED)
    if frames < config.fft_size * sample_rate // sr:
        raise ModuleError(Code.ERROR_TARGET_LENGTH_IS_TOO_SMALL if is_target
                          else Code.ERROR_REFERENCE_LENGTH_LENGTH_TOO_SMALL)
    if channels == 1:
        info(Code.INFO_TARGET_IS_MONO if is_target else Code.INFO_REFERENCE_IS_MONO)
        audio = audio.repeat(1, 2).contiguous()
    source = audio
    if sample_rate != sr:
        from .resample import resample_on_device
        debug(f"Resampling {name} audio from {sample_rate} Hz to {sr} Hz...")
        audio = resample_on_device(audio, sample_rate, sr)
        frames = audio.shape[0]
        if native:
            debug(resampled_for_analysis(sample_rate, config))
        else:
            (warning if is_target else info)(Code.WARNING_TARGET_IS_RESAMPLED if is_target else Code.INFO_REFERENCE_IS_RESAMPLED)
    if is_target:
        lib = _native.load()
        scratch = torch.zeros(16, dtype=torch.uint8, device=audio.device)
        _native.check(lib, lib.mgb_check_peaks(audio.data_ptr(), frames, scratch.data_ptr(), _stream_ptr(audio.device)))
        host = scratch.cpu().numpy()
        peak = float(host[:4].view(np.float32)[0])
        hits = int(host[8:16].view(np.uint64)[0])
        code = peak_warning(peak, hits, config)  # matchering/checker.py:75-87
        if code is not None:
            warning(code)
    return (audio, source) if native else audio


def check_equality_on_device(target: torch.Tensor, reference: torch.Tensor) -> None:
    """matchering/checker.py:140-142."""
    if target.shape != reference.shape:
        return
    lib = _native.load()
    scratch = torch.zeros(8, dtype=torch.uint8, device=target.device)
    _native.check(lib, lib.mgb_check_equality(target.data_ptr(), reference.data_ptr(), target.shape[0], scratch.data_ptr(),
                                              _stream_ptr(target.device)))
    if int(scratch.cpu().numpy().view(np.uint64)[0]) == 0:
        raise ModuleError(Code.ERROR_TARGET_EQUALS_REFERENCE)
