"""GPU drop-in for matchering/limiter/hyrax.py:78-99 `limit(array, config)`."""
from __future__ import annotations

import ctypes as C

import torch

from .. import _native
from ..defaults import Config
import numpy as np

from ..engine import HostIO, _require_cuda, _stream_ptr, host_array_ok, limiter_params, to_device_f32, to_host_like
from ..log import debug
from ..plan import limiter_constants


def limit(array, config: Config):
    """Returns the limited (N, 2) array; like the reference, returns `array` ITSELF (same object)
    when no frame exceeds the threshold (hyrax.py:83-85).  With Config(loudness_target=T) the input is driven into the
    limiter until the output reads T LUFS (a new array, always)."""
    _require_cuda()
    lib = _native.load()
    params = limiter_params(limiter_constants(config))
    device = torch.device("cuda", torch.cuda.current_device())
    debug("The limiter is started. Preparing the gain envelope...")
    if config.loudness_target is not None:
        out, _ = limit_to_loudness(array, config)
        return out
    if host_array_ok(array):
        return _limit_host(array, params, device, lib)
    with torch.cuda.device(device):
        x = to_device_f32(array, device)
        frames = x.shape[0]
        if frames <= 6:
            raise ValueError("The length of the input vector x must be greater than padlen, which is 6.")
        ws_bytes = int(lib.mgb_limiter_workspace_bytes(C.byref(params), frames))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        out = torch.empty_like(x)
        engaged = torch.zeros(1, dtype=torch.int32, device=device)
        _native.check(lib, lib.mgb_limit(C.byref(params), x.data_ptr(), out.data_ptr(), frames, ws.data_ptr(),
                                         ws_bytes, engaged.data_ptr(), _stream_ptr(device)))
        if int(engaged.item()) == 0:
            debug("The limiter is not needed!")
            return array
        return to_host_like(out, array)


_LIMIT_BUFFERS: dict = {}


def _limit_host(array: np.ndarray, params, device, lib):
    """numpy in, numpy out through mgb_limit_host (one native call; the library's worker threads narrow
    and upload the pageable array, the result lands in pooled pinned memory)."""
    frames = array.shape[0]
    if frames <= 6:
        raise ValueError("The length of the input vector x must be greater than padlen, which is 6.")
    io = HostIO.get()
    with torch.cuda.device(device):
        # (the workspace depends on the orders and, on the wide-window path, on the windows: key on its size)
        ws_bytes = int(lib.mgb_limiter_workspace_bytes(C.byref(params), frames))
        key = (device.index, frames, ws_bytes)
        bufs = _LIMIT_BUFFERS.get(key)
        if bufs is None:
            _LIMIT_BUFFERS.clear()  # one size cached: an hour of audio is 1.3 GB per buffer
            bufs = _LIMIT_BUFFERS[key] = dict(
                x=torch.empty((frames, 2), dtype=torch.float32, device=device),
                y=torch.empty((frames, 2), dtype=torch.float32, device=device),
                wide=torch.empty((frames, 2), dtype=torch.float64, device=device) if array.dtype == np.float64 else None,
                ws=torch.empty(ws_bytes, dtype=torch.uint8, device=device), ws_bytes=ws_bytes,
                engaged=torch.zeros(1, dtype=torch.int32, device=device))
        if bufs["wide"] is None and array.dtype == np.float64:
            bufs["wide"] = torch.empty((frames, 2), dtype=torch.float64, device=device)
        out = io.pool.array(array.shape, array.dtype)
        engaged = C.c_int32(0)
        width = array.dtype.itemsize
        with io.lock:
            status = lib.mgb_limit_host(
                io.handle, C.byref(params), array.ctypes.data, width, out.ctypes.data, width, frames, bufs["x"].data_ptr(),
                bufs["y"].data_ptr(), bufs["wide"].data_ptr() if bufs["wide"] is not None else None, bufs["ws"].data_ptr(),
                bufs["ws_bytes"], bufs["engaged"].data_ptr(), C.byref(engaged), _stream_ptr(device))
        _native.check(lib, status)
    if engaged.value == 0:
        debug("The limiter is not needed!")
        return array
    return out


def limit_to_loudness(array, config: Config):
    """limit() at Config.loudness_target (mgb_limit_to_loudness).  -> (output in the caller's array type, LoudnessTarget)"""
    from ..loudness import LoudnessTarget, debug_target, device_meter, target_params
    _require_cuda()
    lib = _native.load()
    params = limiter_params(limiter_constants(config))
    device = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
        x = to_device_f32(array, device)
        frames = x.shape[0]
        if frames <= 6:
            raise ValueError("The length of the input vector x must be greater than padlen, which is 6.")
        meter = device_meter(config.internal_sample_rate, device)
        ws_bytes = int(lib.mgb_limiter_workspace_bytes(C.byref(params), frames)) + int(
            lib.mgb_loudness_target_workspace_bytes(C.byref(meter.params), frames))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        out = torch.empty_like(x)
        report = torch.empty(C.sizeof(_native.LoudnessTargetReport), dtype=torch.uint8, device=device)
        _native.check(lib, lib.mgb_limit_to_loudness(C.byref(params), C.byref(meter.params),
                                                     C.byref(target_params(config.loudness_target)), x.data_ptr(),
                                                     out.data_ptr(), frames, ws.data_ptr(), ws_bytes, report.data_ptr(),
                                                     _stream_ptr(device)))
        t = LoudnessTarget.from_report(config.loudness_target,
                                       _native.LoudnessTargetReport.from_buffer_copy(report.cpu().numpy().tobytes()))
        debug_target(t)
        return to_host_like(out, array), t
