"""Device-side session objects: PyTorch is the memory manager and stream provider, the compute
is libmatchering_b200 (hand-written sm_90a kernels behind the C ABI).

DevicePlan   Config-only tables on one GPU (cached per device + Config).
TrackSession the buffers of one mastering job of fixed sizes; calls the four stage entry points
             that mirror matchering/stages.py's private functions.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _native, plan as _plan
from .log import debug

_PLAN_CACHE: dict = {}


def _require_cuda() -> None:
    if not torch.cuda.is_available():
        raise RuntimeError("matchering_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")


def _stream_ptr(device) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


class DevicePlan:
    def __init__(self, config, device: torch.device):
        self.lib = _native.load()
        self.device = device
        self.tables = _plan.build_tables(config)
        t = self.tables
        s = _native.Plan()
        s.sample_rate, s.fft_size, s.n_lin, s.n_log = t.sample_rate, t.fft_size, t.n_lin, t.n_log
        s.rms_correction_steps, s.lowess_k = t.rms_correction_steps, t.lowess_k
        s.lowess_nfit = len(t.arrays["lw_fit_idx"])
        s.lowess_nrows = len(t.arrays["lw_rows"])
        s.lowess_it = t.lowess_it
        s.max_piece_size, s.threshold, s.min_value = t.max_piece_size, t.threshold, t.min_value
        s.limiter = limiter_params(t.limiter)
        self._keep = {}
        for name, arr in t.arrays.items():
            dev = torch.from_numpy(arr).to(device)
            self._keep[name] = dev
            setattr(s, "d_" + name, dev.data_ptr())
        sizes = (C.c_int64 * 5)()
        _native.check(self.lib, self.lib.mgb_plan_twiddle_bytes(t.fft_size, sizes))
        for name, nbytes in zip(("tw_f32_F", "tw_f32_2F", "tw_f64_F", "tw_f64_2F", "limiter_tables"), sizes):
            buf = torch.zeros(int(nbytes), dtype=torch.uint8, device=device)
            self._keep[name] = buf
            setattr(s, "d_" + name, buf.data_ptr())
        self.struct = s
        with torch.cuda.device(device):
            _native.check(self.lib, self.lib.mgb_plan_fill_twiddles(C.byref(s), _stream_ptr(device)))
            if t.lowess_it > 0 or t.fft_size > _plan.OPERATOR_MAX_FFT_SIZE:
                return  # robustness iterations make the smoothing non-linear in the data: direct chain per track
            # the smoothing chain as one Config-only matrix, built on the device from the direct kernels
            ws_bytes = int(self.lib.mgb_plan_operator_workspace_bytes(C.byref(s)))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
            op = torch.empty((t.n_lin, t.n_lin), dtype=torch.float64, device=device)
            _native.check(self.lib, self.lib.mgb_plan_build_operator(C.byref(s), op.data_ptr(), ws.data_ptr(), ws_bytes,
                                                                    _stream_ptr(device)))
            torch.cuda.current_stream(device).synchronize()
            # S is banded: keep each row's band only (4.8 MB instead of 33.6 MB at the default Config)
            values, rows = _plan.band_operator(op.cpu().numpy())
            del ws, op
            self._keep["smooth_op"] = torch.from_numpy(values).to(device)
            self._keep["smooth_op_rows"] = torch.from_numpy(rows).to(device)
            s.d_smooth_op = self._keep["smooth_op"].data_ptr()
            s.d_smooth_op_rows = self._keep["smooth_op_rows"].data_ptr()

    def layout(self, target_frames: int, reference_frames: int) -> _native.TrackLayout:
        L = _native.TrackLayout()
        _native.check(self.lib, self.lib.mgb_track_layout_init(C.byref(self.struct), target_frames,
                                                              reference_frames, C.byref(L)))
        return L


def limiter_params(lc: _plan.LimiterConstants) -> _native.LimiterParams:
    return _native.LimiterParams.from_constants(lc)


def get_plan(config, device=None) -> DevicePlan:
    _require_cuda()
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    key = (device.index, _plan.config_key(config))
    plan = _PLAN_CACHE.get(key)
    if plan is None:
        plan = _PLAN_CACHE[key] = DevicePlan(config, device)
    return plan


def to_device_f32(array, device) -> torch.Tensor:
    """(N, 2) samples -> contiguous float32 CUDA tensor.  float64 host arrays (what the reference's
    loader hands to stages.main) are copied as they are and narrowed on the device by the library's
    own conversion kernel."""
    if isinstance(array, torch.Tensor):
        t = array.to(device)
        if t.dtype == torch.float32:
            return t.contiguous()
        t = t.to(torch.float64).contiguous()
    else:
        a = np.ascontiguousarray(array)
        if a.dtype == np.float32:
            return torch.from_numpy(a).to(device)
        t = torch.from_numpy(a.astype(np.float64, copy=False)).to(device)
    out = torch.empty(t.shape, dtype=torch.float32, device=device)
    lib = _native.load()
    _native.check(lib, lib.mgb_convert_f64_to_f32(t.data_ptr(), out.data_ptr(), t.numel(), _stream_ptr(device)))
    return out


def to_host_like(t: torch.Tensor, like):
    """Give a float32 CUDA result back in the caller's currency: torch in -> torch out (float32,
    on the device); numpy in -> numpy out with the input's dtype (float64 for the reference's)."""
    if isinstance(like, torch.Tensor):
        return t
    want = np.asarray(like).dtype
    if want == np.float32:
        return t.cpu().numpy()
    wide = torch.empty(t.shape, dtype=torch.float64, device=t.device)
    lib = _native.load()
    _native.check(lib, lib.mgb_convert_f32_to_f64(t.data_ptr(), wide.data_ptr(), t.numel(), _stream_ptr(t.device)))
    return wide.cpu().numpy()


class TrackSession:
    """Buffers for one (plan, target length, reference length) and the stage calls over them."""

    def __init__(self, plan: DevicePlan, target_frames: int, reference_frames: int):
        self.plan = plan
        self.lib = plan.lib
        self.device = plan.device
        self.layout = plan.layout(target_frames, reference_frames)
        self.workspace = torch.empty(int(self.layout.workspace_bytes), dtype=torch.uint8, device=self.device)
        self.state = torch.zeros(C.sizeof(_native.TrackState), dtype=torch.uint8, device=self.device)
        self.result = torch.empty((target_frames, 2), dtype=torch.float32, device=self.device)

    # -- the four stages of matchering/stages.py ------------------------------------------------
    def _args(self):
        return C.byref(self.plan.struct), C.byref(self.layout)

    def match_levels(self, target: torch.Tensor, reference: torch.Tensor) -> None:
        p, l = self._args()
        _native.check(self.lib, self.lib.mgb_match_levels(p, l, target.data_ptr(), reference.data_ptr(),
                                                         self.workspace.data_ptr(), self.state.data_ptr(),
                                                         _stream_ptr(self.device)))

    def match_frequencies(self, target: torch.Tensor, fir_out: torch.Tensor | None = None) -> None:
        p, l = self._args()
        _native.check(self.lib, self.lib.mgb_match_frequencies(
            p, l, target.data_ptr(), self.result.data_ptr(), fir_out.data_ptr() if fir_out is not None else None,
            self.workspace.data_ptr(), self.state.data_ptr(), _stream_ptr(self.device)))

    def correct_levels(self) -> None:
        p, l = self._args()
        _native.check(self.lib, self.lib.mgb_correct_levels(p, l, self.workspace.data_ptr(), self.state.data_ptr(),
                                                           _stream_ptr(self.device)))

    def finalize(self, need_default: bool, need_no_limiter: bool, need_no_limiter_normalized: bool):
        p, l = self._args()
        n = self.layout.target_frames
        mk = lambda need: torch.empty((n, 2), dtype=torch.float32, device=self.device) if need else None
        limited, plain, normalized = mk(need_default), mk(need_no_limiter), mk(need_no_limiter_normalized)
        ptr = lambda t: t.data_ptr() if t is not None else None
        _native.check(self.lib, self.lib.mgb_finalize(p, l, self.result.data_ptr(), ptr(limited), ptr(plain),
                                                     ptr(normalized), self.workspace.data_ptr(),
                                                     self.state.data_ptr(), _stream_ptr(self.device)))
        return limited, plain, normalized

    def read_state(self) -> _native.TrackState:
        """One device->host read of the job's scalars (synchronises)."""
        raw = self.state.cpu().numpy().tobytes()
        return _native.TrackState.from_buffer_copy(raw)


# ------------------------------------------------------------------------------------------------
# host arrays in, host arrays out (the reference's seam: pageable float64 numpy, core.py:77-86)
# ------------------------------------------------------------------------------------------------
class PinnedBlock:
    """A block of pinned host memory from `PinnedPool`, seen by numpy through __array_interface__:
    np.asarray(block) (and every view of it) keeps the block alive, and the memory goes back to the
    pool -- not to the OS -- when the last of them is dropped.  A result array therefore costs no page
    faults and no cudaHostAlloc after the first call of its size, and the device can DMA float64
    results straight into it."""

    def __init__(self, pool, ptr: int, capacity: int, shape, dtype):
        self._pool, self._ptr, self._capacity = pool, ptr, capacity
        self.__array_interface__ = {"shape": tuple(shape), "typestr": np.dtype(dtype).str, "data": (ptr, False),
                                    "version": 3}

    def __del__(self):
        pool, self._pool = self._pool, None
        if pool is not None:
            try:
                pool.release(self._ptr, self._capacity)
            except Exception:  # interpreter shutdown: the library may already be gone
                pass


class PinnedPool:
    GRANULE = 2 << 20

    def __init__(self, lib, keep_bytes: int):
        import threading
        self.lib, self.keep_bytes = lib, keep_bytes
        self.free: dict = {}
        self.cached = 0
        self._lock = threading.Lock()  # arrays are dropped (and blocks released) from whatever thread holds the last reference

    def array(self, shape, dtype) -> np.ndarray:
        nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        capacity = max(self.GRANULE, (nbytes + self.GRANULE - 1) // self.GRANULE * self.GRANULE)
        with self._lock:
            stack = self.free.get(capacity)
            ptr = stack.pop() if stack else None
            if ptr is not None:
                self.cached -= capacity
        if ptr is None:
            ptr = self.lib.mgb_host_alloc(capacity)
            if not ptr:
                self.trim(0)
                ptr = self.lib.mgb_host_alloc(capacity)
            if not ptr:
                raise MemoryError(f"cannot pin {capacity} bytes of host memory for a result array")
        return np.asarray(PinnedBlock(self, ptr, capacity, shape, dtype))

    def release(self, ptr: int, capacity: int) -> None:
        with self._lock:
            keep = self.cached + capacity <= self.keep_bytes
            if keep:
                self.free.setdefault(capacity, []).append(ptr)
                self.cached += capacity
        if not keep:
            self.lib.mgb_host_free(ptr)

    def trim(self, keep_bytes: int) -> None:
        drop = []
        with self._lock:
            for capacity, stack in self.free.items():
                while stack and self.cached > keep_bytes:
                    drop.append(stack.pop())
                    self.cached -= capacity
        for ptr in drop:
            self.lib.mgb_host_free(ptr)


class HostIO:
    """The library's host transport (mgb_host_io: worker threads + pinned staging ring) and the pool of
    pinned result arrays; one per process."""
    _instance = None

    def __init__(self):
        import os
        self.lib = _native.load()
        handle = C.c_void_p()
        threads = int(os.environ.get("MGB_HOST_THREADS", "0"))
        chunk = int(os.environ.get("MGB_HOST_CHUNK", "0"))  # samples per ring chunk, chunks in the ring (tuning)
        ring = int(os.environ.get("MGB_HOST_RING", "0"))
        _native.check(self.lib, self.lib.mgb_host_io_create(threads, chunk, ring, C.byref(handle)))
        self.handle = handle
        import threading
        self.lock = threading.Lock()  # one transfer at a time per mgb_host_io (ctypes drops the GIL during a call)
        self.pool = PinnedPool(self.lib, int(float(os.environ.get("MGB_PINNED_CACHE_GB", "4")) * (1 << 30)))

    @classmethod
    def get(cls) -> "HostIO":
        if cls._instance is None:
            _require_cuda()
            cls._instance = HostIO()
        return cls._instance

    @property
    def threads(self) -> int:
        return int(self.lib.mgb_host_io_threads(self.handle))


def host_array_ok(a) -> bool:
    """numpy arrays the host transport takes as they are: (frames, 2), float32/float64, C-contiguous."""
    return (isinstance(a, np.ndarray) and a.ndim == 2 and a.shape[1] == 2 and a.dtype in (np.float32, np.float64)
            and a.flags["C_CONTIGUOUS"])


_SESSION_CACHE: dict = {}
_SESSION_CACHE_MAX = 2


def host_session(plan: DevicePlan, target_frames: int, reference_frames: int) -> "TrackSession":
    """TrackSession with the device staging of the single-call host entry, cached per (plan, sizes):
    mastering the next track of the same length allocates nothing."""
    key = (id(plan), target_frames, reference_frames)
    sess = _SESSION_CACHE.pop(key, None)
    if sess is None:
        sess = TrackSession(plan, target_frames, reference_frames)
        dev = plan.device
        sess.d_target = torch.empty((target_frames, 2), dtype=torch.float32, device=dev)
        sess.d_reference = torch.empty((reference_frames, 2), dtype=torch.float32, device=dev)
        sess.d_out = torch.empty((target_frames, 2), dtype=torch.float32, device=dev)
        sess.d_wide = torch.empty((target_frames, 2), dtype=torch.float64, device=dev)
        b = _native.HostBuffers()
        b.d_target_lr, b.d_reference_lr = sess.d_target.data_ptr(), sess.d_reference.data_ptr()
        b.d_result_lr, b.d_out_lr, b.d_wide = sess.result.data_ptr(), sess.d_out.data_ptr(), sess.d_wide.data_ptr()
        b.d_workspace, b.d_state = sess.workspace.data_ptr(), sess.state.data_ptr()
        sess.host_buffers = b
    _SESSION_CACHE[key] = sess  # most recently used last
    while len(_SESSION_CACHE) > _SESSION_CACHE_MAX:
        _SESSION_CACHE.pop(next(iter(_SESSION_CACHE)))
    return sess


def stages_main_host(plan: DevicePlan, target: np.ndarray, reference: np.ndarray, need_default: bool,
                     need_no_limiter: bool, need_no_limiter_normalized: bool):
    """stages.main on host numpy arrays through mgb_stages_main_host: one native call, results in pinned
    arrays of the target's dtype.  -> ((limited, plain, normalized), TrackState)"""
    io = HostIO.get()
    if reference.dtype != target.dtype:
        reference = reference.astype(target.dtype)
    sess = host_session(plan, target.shape[0], reference.shape[0])
    width = target.dtype.itemsize
    outs = [io.pool.array(target.shape, target.dtype) if need else None
            for need in (need_default, need_no_limiter, need_no_limiter_normalized)]
    state = _native.TrackState()
    ptr = lambda a: a.ctypes.data if a is not None else None
    with io.lock:
        status = io.lib.mgb_stages_main_host(
            io.handle, C.byref(plan.struct), C.byref(sess.layout), target.ctypes.data, reference.ctypes.data, width,
            ptr(outs[0]), ptr(outs[1]), ptr(outs[2]), width, C.byref(sess.host_buffers), C.byref(state),
            _stream_ptr(plan.device))
    _native.check(io.lib, status)
    return tuple(outs), state


def encode_pcm(t: torch.Tensor, bits: int):
    """float32 CUDA (frames, 2) -> host numpy PCM: int16 (frames, 2) or packed 24-bit uint8 (frames, 6),
    quantised on the device (lrint(x * (2^(bits-1) - 1)), clipped: libsndfile's float -> int write) and
    copied into pooled pinned memory."""
    lib = _native.load()
    frames = t.shape[0]
    if bits == 16:
        out = torch.empty((frames, 2), dtype=torch.int16, device=t.device)
    elif bits == 24:
        out = torch.empty((frames, 6), dtype=torch.uint8, device=t.device)
    else:
        raise ValueError("PCM width must be 16 or 24")
    _native.check(lib, lib.mgb_pcm_encode(t.data_ptr(), bits, out.data_ptr(), frames * 2, _stream_ptr(t.device)))
    host = HostIO.get().pool.array(tuple(out.shape), np.int16 if bits == 16 else np.uint8)
    torch.from_numpy(host).copy_(out)
    return host
