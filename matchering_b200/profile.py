"""Reference profiles: analyse a reference once, master any number of targets against it.

Everything the later stages take from the reference -- its peak and final amplitude coefficient
(match_levels.py normalize_reference), the match RMS of the normalised reference and its number of loud
pieces (analyze_levels), and its two average spectra over the loud pieces (match_frequencies.py:30-42,93-94
__average_fft) -- depends only on the reference and on five Config fields.  `analyze_reference` computes those
on the device (mgb_analyze_reference) and returns them as a `ReferenceProfile`, which `stages.main`,
`mg.process`, `MasteringPipeline` and `master_many` accept wherever they accept a reference.  A job mastered
against a profile computes the same level statistics and FIR, bit for bit, as the job mastered against the
reference's samples, and then runs the same kernels on the same data: its outputs differ from the paired job's only
as much as two device runs of the paired job differ from each other (stage 3's float64 atomic sums).

A profile fits any Config with the same fingerprint (internal_sample_rate, fft_size, max_piece_size, threshold,
min_value); the limiter, LOWESS, lin_log_oversampling and rms_correction_steps may differ.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native

FORMAT = "matchering_b200.reference_profile"
# the Config fields a profile depends on, as mgb_reference_profile names them
FINGERPRINT = ("sample_rate", "fft_size", "n_lin", "max_piece_size", "threshold", "min_value")
_HEADER_FIELDS = [name for name, _ in _native.ReferenceProfileHeader._fields_ if name != "reserved"]
_INT_FIELDS = {"version", "sample_rate", "fft_size", "n_lin", "reference_frames", "reference_piece",
               "reference_divisions", "reference_loud_pieces"}


def config_fingerprint(config) -> dict:
    """The fingerprint fields of a Config, with the values mgb_plan holds."""
    return dict(sample_rate=int(config.internal_sample_rate), fft_size=int(config.fft_size),
                n_lin=int(config.fft_size) // 2 + 1, max_piece_size=float(config.max_piece_size),
                threshold=float(config.threshold), min_value=float(config.min_value))


class ReferenceProfile:
    """The reference side of a mastering job: a header (fingerprint, geometry, scalars) and the spectra
    [2, n_lin] (mid, side) of the normalised reference.  Immutable; the device copy is made on first use and
    kept per device."""

    def __init__(self, header: dict, spectra: np.ndarray):
        spectra = np.ascontiguousarray(spectra)
        if spectra.dtype != np.float64 or spectra.shape != (2, int(header["n_lin"])):
            raise ValueError(f"reference profile: spectra must be float64 [2, {header['n_lin']}], "
                             f"not {spectra.dtype} {list(spectra.shape)}")
        if int(header["version"]) != _native.MGB_REFERENCE_PROFILE_VERSION:
            raise ValueError(f"reference profile: version {header['version']}, this library reads "
                             f"{_native.MGB_REFERENCE_PROFILE_VERSION}")
        self._header = {k: (int(header[k]) if k in _INT_FIELDS else float(header[k])) for k in _HEADER_FIELDS}
        spectra.setflags(write=False)
        self._spectra = spectra
        self._device_blobs = {}

    # -- read-only attributes ---------------------------------------------------------------------
    version = property(lambda self: self._header["version"])
    sample_rate = property(lambda self: self._header["sample_rate"])
    fft_size = property(lambda self: self._header["fft_size"])
    n_lin = property(lambda self: self._header["n_lin"])
    max_piece_size = property(lambda self: self._header["max_piece_size"])
    threshold = property(lambda self: self._header["threshold"])
    min_value = property(lambda self: self._header["min_value"])
    frames = property(lambda self: self._header["reference_frames"])
    piece = property(lambda self: self._header["reference_piece"])
    divisions = property(lambda self: self._header["reference_divisions"])
    loud_pieces = property(lambda self: self._header["reference_loud_pieces"])
    peak = property(lambda self: self._header["reference_peak"])
    final_amplitude_coef = property(lambda self: self._header["final_amplitude_coef"])
    match_rms = property(lambda self: self._header["reference_match_rms"])
    spectra = property(lambda self: self._spectra)

    def fingerprint(self) -> dict:
        return {k: self._header[k] for k in FINGERPRINT}

    def check_config(self, config) -> None:
        """ValueError naming the first fingerprint field in which `config` differs from the profile's Config."""
        want = config_fingerprint(config)
        for k in FINGERPRINT:
            if want[k] != self._header[k]:
                raise ValueError(f"reference profile: {k} {self._header[k]!r} differs from the Config's {want[k]!r}")

    def header_struct(self) -> _native.ReferenceProfileHeader:
        h = _native.ReferenceProfileHeader()
        for k in _HEADER_FIELDS:
            setattr(h, k, self._header[k])
        return h

    def to_bytes(self) -> bytes:
        """The device blob's bytes: mgb_reference_profile, then spectra[2][n_lin]."""
        return bytes(self.header_struct()) + self._spectra.tobytes()

    def device_blob(self, device):
        """The profile in device memory on `device` (uploaded once per device)."""
        import torch
        device = torch.device(device)
        blob = self._device_blobs.get(device.index)
        if blob is None:
            host = torch.frombuffer(bytearray(self.to_bytes()), dtype=torch.uint8)
            blob = self._device_blobs[device.index] = host.to(device)
        return blob

    def checked_blob(self, plan):
        """The device blob for `plan`'s device after the library's own fingerprint check against the plan."""
        h = self.header_struct()
        _native.check(plan.lib, plan.lib.mgb_reference_profile_check(C.byref(plan.struct), C.byref(h)))
        return self.device_blob(plan.device)

    # -- files --------------------------------------------------------------------------------------
    def save(self, path) -> None:
        """An .npz with a format tag, the header fields and the spectra (no pickled objects)."""
        fields = {k: np.array(v, dtype=np.int64 if k in _INT_FIELDS else np.float64) for k, v in self._header.items()}
        with open(path, "wb") as f:
            np.savez(f, format=np.array(FORMAT), spectra=self._spectra, **fields)

    @classmethod
    def load(cls, path) -> "ReferenceProfile":
        try:
            with np.load(path, allow_pickle=False) as z:
                data = {k: z[k] for k in z.files}
        except Exception as e:  # a truncated or corrupt archive, or not an archive at all
            raise ValueError(f"reference profile: cannot read {path}: {e}") from e
        if "format" not in data or data["format"].shape != () or str(data["format"]) != FORMAT:
            raise ValueError(f"reference profile: {path} is not a {FORMAT} file")
        header = {}
        for k in _HEADER_FIELDS:
            v = data.get(k)
            want = np.int64 if k in _INT_FIELDS else np.float64
            if v is None or v.shape != () or v.dtype != want:
                raise ValueError(f"reference profile: field {k} missing or not a {np.dtype(want)} scalar")
            header[k] = v.item()
        spectra = data.get("spectra")
        if spectra is None:
            raise ValueError("reference profile: spectra missing")
        return cls(header, spectra)

    def __repr__(self) -> str:
        return (f"ReferenceProfile({self.frames} frames, {self.divisions} pieces of {self.piece}, {self.loud_pieces} loud, "
                f"fft_size {self.fft_size}, {self.sample_rate} Hz)")


def analyze_reference(reference, config=None) -> ReferenceProfile:
    """Analyse `reference` once.  `reference` is a file path (loaded and checked like mg.process loads its
    reference) or an (N, 2) numpy array / torch tensor at config.internal_sample_rate."""
    import torch

    from .defaults import Config
    from .engine import get_plan, to_device_f32, _stream_ptr
    if config is None:
        config = Config()
    if isinstance(reference, (str, bytes)) or hasattr(reference, "__fspath__"):
        import os

        from .core import _load_and_check
        from .log import Code, ModuleError
        path = os.fspath(reference)
        temp_folder = config.temp_folder if config.temp_folder else os.path.dirname(os.path.abspath(path))
        reference, rate = _load_and_check(path, "reference", temp_folder, config)
        if rate != config.internal_sample_rate or reference.shape[1] != 2 or reference.shape[0] <= config.fft_size:
            raise ModuleError(Code.ERROR_VALIDATION)
    if reference.ndim != 2 or reference.shape[1] != 2:
        raise ValueError("reference must be a (frames, 2) stereo array")
    plan = get_plan(config)
    lib, device = plan.lib, plan.device
    frames = int(reference.shape[0])
    with torch.cuda.device(device):
        d_ref = to_device_f32(reference, device)
        ws_bytes = int(lib.mgb_reference_workspace_bytes(C.byref(plan.struct), frames))
        if ws_bytes < 0:  # (the reference is too short, or has too many pieces)
            raise ValueError(lib.mgb_last_error_string().decode("utf-8", "replace"))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        blob = torch.empty(int(lib.mgb_reference_profile_bytes(C.byref(plan.struct))), dtype=torch.uint8, device=device)
        _native.check(lib, lib.mgb_analyze_reference(C.byref(plan.struct), d_ref.data_ptr(), frames, ws.data_ptr(), ws_bytes,
                                                     blob.data_ptr(), _stream_ptr(device)))
        raw = blob.cpu().numpy().tobytes()
    profile = profile_from_bytes(raw)
    profile._device_blobs[device.index] = blob
    return profile


def profile_from_bytes(raw: bytes) -> ReferenceProfile:
    """A profile from the bytes of a device blob (mgb_reference_profile, then the spectra)."""
    size = C.sizeof(_native.ReferenceProfileHeader)
    h = _native.ReferenceProfileHeader.from_buffer_copy(raw[:size])
    spectra = np.frombuffer(raw[size:size + 16 * h.n_lin], dtype=np.float64).reshape(2, h.n_lin).copy()
    return ReferenceProfile({k: getattr(h, k) for k in _HEADER_FIELDS}, spectra)
