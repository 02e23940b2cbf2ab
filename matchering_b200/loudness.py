"""Loudness meter on the device: ITU-R BS.1770-4 integrated loudness, EBU Tech 3342 loudness range, maximum
momentary and short-term loudness, sample peak and true peak of a stereo track (mgb_loudness).

    m = mg.loudness("master.wav")         # at the file's own rate, no resampling
    m = mg.loudness(array, 44100)         # (N, 2) float32 / float64 numpy
    m = mg.loudness(cuda_tensor, 44100)   # (N, 2) float32 CUDA tensor: the samples stay on the device
    m.integrated, m.loudness_range, m.true_peak

Both channels are weighted 1.  Mono and multichannel input raise ValueError: BS.1770 weighs surround channels
differently, and it reads dual mono 3 LU above the same signal as mono, so duplicating a mono channel would
mislead.  The true peak is read through a 12-zero-crossing Kaiser-windowed sinc interpolator at 4x oversampling
below 96 kHz (2x below 192 kHz, none above): it is never below the sample peak, and its parity with other meters'
true peak is not pinned (DESIGN.md section 7).
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np

from . import _native, plan as _plan


@dataclass(frozen=True)
class Loudness:
    """One track's meter.  Loudness in LUFS, range in LU, peaks in dBFS / dBTP; -inf where undefined (a track
    shorter than one 400 ms or 3 s window, or silence)."""
    integrated: float
    loudness_range: float
    momentary_max: float
    short_term_max: float
    sample_peak: float            # max over both channels
    true_peak: float              # max over both channels
    true_peak_per_channel: tuple  # (left, right)

    @classmethod
    def from_result(cls, r: _native.LoudnessResult) -> "Loudness":
        db = lambda v: 20.0 * math.log10(v) if v > 0.0 else -math.inf
        tp = (db(r.true_peak[0]), db(r.true_peak[1]))
        return cls(float(r.integrated), float(r.loudness_range), float(r.momentary_max), float(r.short_term_max),
                   db(max(r.sample_peak[0], r.sample_peak[1])), max(tp), tp)


# the largest drive a loudness target may apply on top of the correction gain (Config(loudness_target=...)), dB
LOUDNESS_TARGET_MAX_GAIN_DB = 24.0

_TARGET_STATUS = {_native.MGB_LOUDNESS_REACHED: "reached", _native.MGB_LOUDNESS_UNREACHABLE: "unreachable",
                  _native.MGB_LOUDNESS_BRACKET: "bracket", _native.MGB_LOUDNESS_PASSES: "passes",
                  _native.MGB_LOUDNESS_UNDEFINED: "undefined"}


@dataclass(frozen=True)
class LoudnessTarget:
    """How a loudness-targeted limiter run ended (Config(loudness_target=...)).  gain_db is the drive into the limiter on
    top of the correction gain, integrated the loudness measured on the samples written; status is "reached" (within
    0.01 LU), "unreachable" (still too quiet at the largest drive), "bracket" (the loudness jumps across the target within
    1e-3 dB), "passes" (the pass limit came first) or "undefined" (silence, or shorter than one 400 ms window)."""
    target: float
    gain_db: float
    integrated: float
    input_integrated: float
    passes: int
    status: str
    trace: tuple  # ((gain_db, integrated), ...) per pass

    @classmethod
    def from_report(cls, target: float, r: _native.LoudnessTargetReport) -> "LoudnessTarget":
        n = int(r.passes)
        return cls(float(target), float(r.gain_db), float(r.integrated), float(r.input_integrated), n,
                   _TARGET_STATUS.get(int(r.status), f"status {int(r.status)}"),
                   tuple((float(r.trace_gain_db[k]), float(r.trace_integrated[k])) for k in range(n)))


def target_params(target_lufs: float) -> _native.LoudnessTargetParams:
    t = _native.LoudnessTargetParams()
    t.target_lufs, t.max_gain_db = float(target_lufs), LOUDNESS_TARGET_MAX_GAIN_DB
    return t


def debug_target(t: LoudnessTarget) -> None:
    from .log import debug
    debug(f"Loudness target {t.target:.2f} LUFS: drive {t.gain_db:+.4f} dB, measured {t.integrated:.4f} LUFS "
          f"after {t.passes} pass(es), {t.status}")


class DeviceMeter:
    """The C parameters of one rate, with their filter tables on one device (cached per device and rate)."""

    def __init__(self, sample_rate: int, device):
        import torch
        from .engine import _stream_ptr
        self.lib = _native.load()
        self.device = device
        self.params = _native.LoudnessParams.from_constants(_plan.loudness_constants(sample_rate))
        self.tables = torch.empty(int(self.lib.mgb_loudness_tables_bytes()), dtype=torch.uint8, device=device)
        self.params.d_tables = self.tables.data_ptr()
        with torch.cuda.device(device):
            _native.check(self.lib, self.lib.mgb_loudness_fill_tables(C.byref(self.params), self.tables.data_ptr(),
                                                                     _stream_ptr(device)))

    def measure(self, x) -> Loudness:
        """x: (N, 2) float32 CUDA tensor on this meter's device."""
        import torch
        from .engine import _stream_ptr
        frames = int(x.shape[0])
        ws_bytes = int(self.lib.mgb_loudness_workspace_bytes(C.byref(self.params), frames))
        with torch.cuda.device(self.device):
            ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=self.device)
            out = torch.empty(C.sizeof(_native.LoudnessResult), dtype=torch.uint8, device=self.device)
            _native.check(self.lib, self.lib.mgb_loudness(C.byref(self.params), x.data_ptr(), frames, ws.data_ptr(),
                                                         ws_bytes, out.data_ptr(), _stream_ptr(self.device)))
            raw = out.cpu().numpy().tobytes()
        return Loudness.from_result(_native.LoudnessResult.from_buffer_copy(raw))

    def measure_album(self, xs: list) -> "AlbumLoudness":
        """xs: (N_t, 2) float32 CUDA tensors on this meter's device, one per track (mgb_album_loudness)."""
        import torch
        from .engine import _stream_ptr
        n = len(xs)
        frames = (C.c_int64 * n)(*(int(x.shape[0]) for x in xs))
        ptrs = (C.c_void_p * n)(*(x.data_ptr() for x in xs))
        ws_bytes = int(self.lib.mgb_album_loudness_workspace_bytes(C.byref(self.params), n, frames))
        size = C.sizeof(_native.LoudnessResult)
        with torch.cuda.device(self.device):
            ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=self.device)
            out = torch.empty((n + 1) * size, dtype=torch.uint8, device=self.device)  # the album, then each track
            _native.check(self.lib, self.lib.mgb_album_loudness(C.byref(self.params), n, ptrs, frames, ws.data_ptr(),
                                                               ws_bytes, out.data_ptr(), out.data_ptr() + size,
                                                               _stream_ptr(self.device)))
            raw = out.cpu().numpy().tobytes()
        results = [Loudness.from_result(_native.LoudnessResult.from_buffer_copy(raw[k * size:(k + 1) * size]))
                   for k in range(n + 1)]
        return AlbumLoudness(results[0], tuple(results[1:]))


@dataclass(frozen=True)
class AlbumLoudness:
    """An album's meter (mg.album_loudness): `album` meters the tracks as one programme (the gates and the loudness
    range over the union of every track's windows, the maxima over the tracks), `tracks` each track on its own."""
    album: Loudness
    tracks: tuple


_METERS: dict = {}


def device_meter(sample_rate: int, device=None) -> DeviceMeter:
    import torch
    from .engine import _require_cuda
    _require_cuda()
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    key = (device.index, int(sample_rate))
    meter = _METERS.get(key)
    if meter is None:
        meter = _METERS[key] = DeviceMeter(int(sample_rate), device)
    return meter


def _check_shape(shape) -> None:
    if len(shape) != 2 or shape[1] != 2:
        raise ValueError(f"loudness: stereo (N, 2) samples only, not shape {tuple(shape)} (BS.1770 weighs other "
                         "channel layouts differently, and reads dual mono 3 LU above mono)")
    if shape[0] < 1:
        raise ValueError("loudness: no samples")


def loudness(audio, sample_rate: int | None = None) -> Loudness:
    """Meter `audio`: a file path (loaded as mg.load loads it, metered at its own rate), an (N, 2) float32 or
    float64 numpy array, or an (N, 2) float32 CUDA tensor.  `sample_rate` is required for arrays and tensors.
    The meter reads float32, as the pipeline's outputs are: float64 samples are rounded to float32 first."""
    import torch
    if isinstance(audio, (str, bytes)) or hasattr(audio, "__fspath__"):
        import os
        from .loader import load
        path = os.fsdecode(os.fspath(audio))
        audio, rate = load(path, "target", os.path.dirname(os.path.abspath(path)))
        if sample_rate is not None and int(sample_rate) != int(rate):
            raise ValueError(f"loudness: the file's rate is {rate} Hz, not {sample_rate}")
        sample_rate = rate
    if sample_rate is None:
        raise ValueError("loudness: sample_rate is required for arrays and tensors")
    sample_rate = int(sample_rate)
    if isinstance(audio, torch.Tensor):
        _check_shape(audio.shape)
        if not audio.is_cuda or audio.dtype != torch.float32:
            raise ValueError("loudness: tensors must be float32 on a CUDA device (numpy arrays may be float64)")
        meter = device_meter(sample_rate, audio.device)
        return meter.measure(audio.contiguous())
    a = np.asarray(audio)
    _check_shape(a.shape)
    if a.dtype not in (np.float32, np.float64):
        raise ValueError(f"loudness: float32 or float64 samples, not {a.dtype}")
    meter = device_meter(sample_rate)
    from .engine import to_device_f32
    return meter.measure(to_device_f32(a, meter.device))


def _album_audio(audio, sample_rate):
    """One album track -> ((N, 2) float32 CUDA tensor or float numpy array, its rate or None)."""
    import torch
    if isinstance(audio, (str, bytes)) or hasattr(audio, "__fspath__"):
        import os
        from .loader import load
        path = os.fsdecode(os.fspath(audio))
        audio, rate = load(path, "target", os.path.dirname(os.path.abspath(path)))
        if sample_rate is not None and int(sample_rate) != int(rate):
            raise ValueError(f"album_loudness: '{path}' is at {rate} Hz, not {sample_rate}")
        _check_shape(np.shape(audio))
        return audio, int(rate)
    if isinstance(audio, torch.Tensor):
        _check_shape(audio.shape)
        if not audio.is_cuda or audio.dtype != torch.float32:
            raise ValueError("album_loudness: tensors must be float32 on a CUDA device (numpy arrays may be float64)")
        return audio, None
    a = np.asarray(audio)
    _check_shape(a.shape)
    if a.dtype not in (np.float32, np.float64):
        raise ValueError(f"album_loudness: float32 or float64 samples, not {a.dtype}")
    return a, None


def album_loudness(tracks, sample_rate: int | None = None) -> AlbumLoudness:
    """Meter an album as one programme: `tracks` is a list of file paths, (N, 2) numpy arrays or (N, 2) float32 CUDA
    tensors, all at one rate (`sample_rate` is required unless every track is a file).  The album's integrated loudness
    and loudness range gate the union of every track's 400 ms and 3 s windows, each window counting once and none
    straddling two tracks (libebur128's ebur128_loudness_global_multiple); its maxima and peaks are the tracks' maxima.
    -> AlbumLoudness(album, tracks), the second each track's own meter, as mg.loudness reads it."""
    import torch
    tracks = list(tracks)
    if not tracks:
        raise ValueError("album_loudness: an album needs at least one track")
    if len(tracks) > _native.MGB_MAX_ALBUM_TRACKS:
        raise ValueError(f"album_loudness: {len(tracks)} tracks, at most {_native.MGB_MAX_ALBUM_TRACKS}")
    loaded = [_album_audio(t, sample_rate) for t in tracks]
    rates = {r for _, r in loaded if r is not None}
    if sample_rate is not None:
        rates.add(int(sample_rate))
    if len(rates) > 1:
        raise ValueError(f"album_loudness: the tracks are at different rates {sorted(rates)}")
    if not rates:
        raise ValueError("album_loudness: sample_rate is required for arrays and tensors")
    rate = rates.pop()
    devices = {a.device for a, _ in loaded if isinstance(a, torch.Tensor)}
    if len(devices) > 1:
        raise ValueError("album_loudness: the tensors are on different devices")
    meter = device_meter(rate, devices.pop() if devices else None)
    from .engine import to_device_f32
    xs = [a.contiguous() if isinstance(a, torch.Tensor) else to_device_f32(a, meter.device) for a, _ in loaded]
    return meter.measure_album(xs)
