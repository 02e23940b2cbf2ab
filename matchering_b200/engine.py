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
    """`native_tables` (plan.native_tables): the plan of a native-rate job's stages 2-4, which designs no curve of its
    own -- it carries the analysis plan's over -- and so builds no smoothing operator."""

    def __init__(self, config, device: torch.device, native_tables: dict | None = None):
        self.lib = _native.load()
        self.device = device
        self.tables = _plan.build_tables(config)
        t = self.tables
        if native_tables is not None:
            t.arrays.update(native_tables)
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
            if t.lowess_it > 0 or t.fft_size > _plan.OPERATOR_MAX_FFT_SIZE or native_tables is not None:
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

    def layout_profiled(self, target_frames: int) -> _native.TrackLayout:
        """Layout of a job whose reference comes from a ReferenceProfile (no reference pieces)."""
        L = _native.TrackLayout()
        _native.check(self.lib, self.lib.mgb_track_layout_init_profiled(C.byref(self.struct), target_frames, C.byref(L)))
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


def get_native_plan(config, rate: int, device=None) -> DevicePlan:
    """The plan of stages 2-4 of a native-rate job at `rate` (plan.native_config), with the tables that carry the
    analysis curve of `config`'s plan over to its FIR; cached per device, Config and rate."""
    _require_cuda()
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    key = (device.index, _plan.config_key(config), "native", int(rate))
    plan = _PLAN_CACHE.get(key)
    if plan is None:
        plan = _PLAN_CACHE[key] = DevicePlan(_plan.native_config(config, rate), device, _plan.native_tables(config, rate))
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
    """Buffers for one (plan, target length, reference length) and the stage calls over them;
    reference_frames None: the reference comes from a profile (match_levels_profiled)."""

    def __init__(self, plan: DevicePlan, target_frames: int, reference_frames: int | None):
        self.plan = plan
        self.lib = plan.lib
        self.device = plan.device
        self.layout = (plan.layout_profiled(target_frames) if reference_frames is None
                       else plan.layout(target_frames, reference_frames))
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

    def match_levels_profiled(self, target: torch.Tensor, d_profile: torch.Tensor) -> None:
        p, l = self._args()
        _native.check(self.lib, self.lib.mgb_match_levels_profiled(p, l, target.data_ptr(), d_profile.data_ptr(),
                                                                  self.workspace.data_ptr(), self.state.data_ptr(),
                                                                  _stream_ptr(self.device)))

    def match_frequencies(self, target: torch.Tensor, fir_out: torch.Tensor | None = None) -> None:
        p, l = self._args()
        _native.check(self.lib, self.lib.mgb_match_frequencies(
            p, l, target.data_ptr(), self.result.data_ptr(), fir_out.data_ptr() if fir_out is not None else None,
            self.workspace.data_ptr(), self.state.data_ptr(), _stream_ptr(self.device)))

    def design_frequencies(self, fir_out: torch.Tensor | None = None) -> None:
        """Stage 2's FIR design without its convolution (mgb_design_frequencies): what a native-rate job takes from
        its analysis session."""
        p, l = self._args()
        _native.check(self.lib, self.lib.mgb_design_frequencies(
            p, l, fir_out.data_ptr() if fir_out is not None else None, self.workspace.data_ptr(), self.state.data_ptr(),
            _stream_ptr(self.device)))

    def match_frequencies_native(self, analysis: "TrackSession", target: torch.Tensor,
                                 fir_out: torch.Tensor | None = None) -> None:
        """Stage 2 of a native-rate job in this session (a native plan's, profiled layout): the FIR carried over from
        `analysis`, which has run match_levels and design_frequencies, then the convolution of `target` at this rate."""
        p, l = analysis._args()
        np_, nl = self._args()
        _native.check(self.lib, self.lib.mgb_match_frequencies_native(
            p, l, analysis.workspace.data_ptr(), analysis.state.data_ptr(), np_, nl, target.data_ptr(),
            self.result.data_ptr(), fir_out.data_ptr() if fir_out is not None else None, self.workspace.data_ptr(),
            self.state.data_ptr(), _stream_ptr(self.device)))

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

    def finalize_to_loudness(self, target_lufs: float, need_no_limiter: bool, need_no_limiter_normalized: bool):
        """finalize with the limited output searched to `target_lufs` (mgb_finalize_to_loudness); the other two
        outputs as mgb_finalize writes them.  -> (limited, plain, normalized, the device report)"""
        from .loudness import device_meter, target_params
        limited, plain, normalized = self.finalize(False, need_no_limiter, need_no_limiter_normalized)
        n = self.layout.target_frames
        meter = device_meter(self.plan.tables.sample_rate, self.device)
        search_bytes = int(self.lib.mgb_loudness_target_workspace_bytes(C.byref(meter.params), n))
        search = torch.empty(search_bytes, dtype=torch.uint8, device=self.device)
        report = torch.empty(C.sizeof(_native.LoudnessTargetReport), dtype=torch.uint8, device=self.device)
        limited = torch.empty((n, 2), dtype=torch.float32, device=self.device)
        p, l = self._args()
        _native.check(self.lib, self.lib.mgb_finalize_to_loudness(
            p, l, C.byref(meter.params), C.byref(target_params(target_lufs)), self.result.data_ptr(), limited.data_ptr(),
            self.workspace.data_ptr(), search.data_ptr(), search_bytes, self.state.data_ptr(), report.data_ptr(),
            _stream_ptr(self.device)))
        return limited, plain, normalized, report

    def read_state(self) -> _native.TrackState:
        """One device->host read of the job's scalars (synchronises)."""
        raw = self.state.cpu().numpy().tobytes()
        return _native.TrackState.from_buffer_copy(raw)


def album_match(sessions: list, targets: list, d_profile: torch.Tensor, fir_out: torch.Tensor | None = None) -> None:
    """Stages 1-3 of an album (mgb_album_match): one TrackSession per track, each a profiled session of the same plan,
    and its target on the device.  Leaves every session where correct_levels leaves a single job."""
    plan = sessions[0].plan
    n = len(sessions)
    table = (_native.AlbumTrack * n)()
    for entry, session, target in zip(table, sessions, targets):
        entry.layout = C.pointer(session.layout)
        entry.d_target_lr, entry.d_result_lr = target.data_ptr(), session.result.data_ptr()
        entry.d_workspace, entry.d_state = session.workspace.data_ptr(), session.state.data_ptr()
    layouts = (_native.TrackLayout * n)(*(s.layout for s in sessions))
    ws_bytes = int(plan.lib.mgb_album_workspace_bytes(C.byref(plan.struct), n, layouts))
    if ws_bytes < 0:
        raise ValueError(plan.lib.mgb_last_error_string().decode("utf-8", "replace"))
    album_ws = torch.empty(ws_bytes, dtype=torch.uint8, device=plan.device)
    _native.check(plan.lib, plan.lib.mgb_album_match(
        C.byref(plan.struct), n, table, d_profile.data_ptr(), fir_out.data_ptr() if fir_out is not None else None,
        album_ws.data_ptr(), ws_bytes, _stream_ptr(plan.device)))


def album_finalize_to_loudness(sessions: list, target_lufs: float, need_no_limiter: bool = False,
                               need_no_limiter_normalized: bool = False):
    """Stage 4 of an album after album_match, with ONE limiter drive for every track searched until the album reads
    `target_lufs` (mgb_album_finalize_to_loudness); the other two outputs as mgb_finalize writes them.
    -> ([(limited, plain, normalized) per track], the album's device report)"""
    from .loudness import device_meter, target_params
    plan = sessions[0].plan
    n = len(sessions)
    outs = [s.finalize(False, need_no_limiter, need_no_limiter_normalized) for s in sessions]
    limited = [torch.empty((int(s.layout.target_frames), 2), dtype=torch.float32, device=plan.device) for s in sessions]
    table = (_native.AlbumTrack * n)()
    for entry, session in zip(table, sessions):
        entry.layout = C.pointer(session.layout)
        entry.d_target_lr, entry.d_result_lr = None, session.result.data_ptr()
        entry.d_workspace, entry.d_state = session.workspace.data_ptr(), session.state.data_ptr()
    out_ptrs = (C.c_void_p * n)(*(t.data_ptr() for t in limited))
    layouts = (_native.TrackLayout * n)(*(s.layout for s in sessions))
    meter = device_meter(plan.tables.sample_rate, plan.device)
    search_bytes = int(plan.lib.mgb_album_loudness_target_workspace_bytes(C.byref(meter.params), n, layouts))
    if search_bytes < 0:
        raise ValueError(plan.lib.mgb_last_error_string().decode("utf-8", "replace"))
    search = torch.empty(search_bytes, dtype=torch.uint8, device=plan.device)
    report = torch.empty(C.sizeof(_native.LoudnessTargetReport), dtype=torch.uint8, device=plan.device)
    _native.check(plan.lib, plan.lib.mgb_album_finalize_to_loudness(
        C.byref(plan.struct), n, table, out_ptrs, C.byref(meter.params), C.byref(target_params(target_lufs)),
        search.data_ptr(), search_bytes, report.data_ptr(), _stream_ptr(plan.device)))
    return [(lim, plain, normalized) for lim, (_, plain, normalized) in zip(limited, outs)], report


def versions_match(main: TrackSession, sessions: list, targets: list) -> None:
    """Stage 2 of each version with the main's FIR (mgb_version_match_frequencies), after the main's correct_levels: one
    profiled TrackSession per version, of the main's frame count, and its target on the device."""
    n = len(sessions)
    table = (_native.VersionTrack * n)()
    for entry, session, target in zip(table, sessions, targets):
        entry.layout = C.pointer(session.layout)
        entry.d_target_lr, entry.d_result_lr = target.data_ptr(), session.result.data_ptr()
        entry.d_workspace, entry.d_state = session.workspace.data_ptr(), session.state.data_ptr()
    p, l = main._args()
    _native.check(main.lib, main.lib.mgb_version_match_frequencies(p, l, main.workspace.data_ptr(), main.state.data_ptr(), n,
                                                                    table, _stream_ptr(main.device)))


def versions_finalize(main: TrackSession, results: list, need_default: bool, need_no_limiter: bool,
                      need_no_limiter_normalized: bool, loudness_target: float | None = None):
    """Stage 4 of the main (results[0], its own result) and its versions with one detector and one gain envelope
    (mgb_finalize_versions; with loudness_target the limited outputs at the main's searched drive,
    mgb_finalize_versions_to_loudness).  -> ([(limited, plain, normalized) per entry], the device report or None)"""
    lib, dev = main.lib, main.device
    n, count = main.layout.target_frames, len(results)
    p, l = main._args()
    vbytes = int(lib.mgb_versions_workspace_bytes(p, l))
    if vbytes < 0:
        raise ValueError(lib.mgb_last_error_string().decode("utf-8", "replace"))
    vws = torch.empty(vbytes, dtype=torch.uint8, device=dev)
    mk = lambda need: torch.empty((n, 2), dtype=torch.float32, device=dev) if need else None
    targeted = need_default and loudness_target is not None
    outs = [(mk(need_default), mk(need_no_limiter), mk(need_no_limiter_normalized)) for _ in results]
    ptr = lambda t: t.data_ptr() if t is not None else None
    table = (_native.VersionEntry * count)()
    for entry, result, (lim, plain, norm) in zip(table, results, outs):
        entry.d_result_lr = result.data_ptr()
        entry.d_out_limited = None if targeted else ptr(lim)
        entry.d_out_no_limiter, entry.d_out_normalized = ptr(plain), ptr(norm)
    report = None
    if any(t is not None for entry in outs for t in entry) and (not targeted or need_no_limiter or need_no_limiter_normalized):
        _native.check(lib, lib.mgb_finalize_versions(p, l, count, table, main.workspace.data_ptr(), main.state.data_ptr(),
                                                     vws.data_ptr(), vbytes, _stream_ptr(dev)))
    if targeted:
        from .loudness import device_meter, target_params
        for entry, (lim, _, _) in zip(table, outs):
            entry.d_out_limited, entry.d_out_no_limiter, entry.d_out_normalized = lim.data_ptr(), None, None
        meter = device_meter(main.plan.tables.sample_rate, dev)
        search_bytes = int(lib.mgb_loudness_target_workspace_bytes(C.byref(meter.params), n))
        search = torch.empty(search_bytes, dtype=torch.uint8, device=dev)
        report = torch.empty(C.sizeof(_native.LoudnessTargetReport), dtype=torch.uint8, device=dev)
        _native.check(lib, lib.mgb_finalize_versions_to_loudness(
            p, l, C.byref(meter.params), C.byref(target_params(loudness_target)), count, table, main.workspace.data_ptr(),
            main.state.data_ptr(), vws.data_ptr(), vbytes, search.data_ptr(), search_bytes, report.data_ptr(),
            _stream_ptr(dev)))
    return outs, report


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
        sess.d_reference = (None if reference_frames is None
                            else torch.empty((reference_frames, 2), dtype=torch.float32, device=dev))
        sess.d_out = torch.empty((target_frames, 2), dtype=torch.float32, device=dev)
        sess.d_wide = torch.empty((target_frames, 2), dtype=torch.float64, device=dev)
        b = _native.HostBuffers()
        b.d_target_lr = sess.d_target.data_ptr()
        b.d_reference_lr = sess.d_reference.data_ptr() if sess.d_reference is not None else None
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


def stages_main_host_profiled(plan: DevicePlan, target: np.ndarray, profile, need_default: bool, need_no_limiter: bool,
                              need_no_limiter_normalized: bool):
    """stages_main_host with the reference from a ReferenceProfile (mgb_stages_main_host_profiled): only the
    target is uploaded.  -> ((limited, plain, normalized), TrackState)"""
    io = HostIO.get()
    d_profile = profile.checked_blob(plan)
    sess = host_session(plan, target.shape[0], None)
    width = target.dtype.itemsize
    outs = [io.pool.array(target.shape, target.dtype) if need else None
            for need in (need_default, need_no_limiter, need_no_limiter_normalized)]
    state = _native.TrackState()
    ptr = lambda a: a.ctypes.data if a is not None else None
    with io.lock:
        status = io.lib.mgb_stages_main_host_profiled(
            io.handle, C.byref(plan.struct), C.byref(sess.layout), target.ctypes.data, width, d_profile.data_ptr(),
            ptr(outs[0]), ptr(outs[1]), ptr(outs[2]), width, C.byref(sess.host_buffers), C.byref(state),
            _stream_ptr(plan.device))
    _native.check(io.lib, status)
    return tuple(outs), state


def encode_pcm(t: torch.Tensor, bits: int, dither: _native.DitherParams | None = None):
    """float32 CUDA (frames, 2) -> host numpy PCM: int16 (frames, 2) or packed 24-bit uint8 (frames, 6),
    quantised on the device (lrint(x * (2^(bits-1) - 1)), clipped: libsndfile's float -> int write) and
    copied into pooled pinned memory.  With `dither` (dither.params) the dithered encoder quantises instead
    (mgb_pcm_encode_dithered)."""
    lib = _native.load()
    frames = t.shape[0]
    if bits == 16:
        out = torch.empty((frames, 2), dtype=torch.int16, device=t.device)
    elif bits == 24:
        out = torch.empty((frames, 6), dtype=torch.uint8, device=t.device)
    else:
        raise ValueError("PCM width must be 16 or 24")
    if dither is None:
        _native.check(lib, lib.mgb_pcm_encode(t.data_ptr(), bits, out.data_ptr(), frames * 2, _stream_ptr(t.device)))
    else:
        t = t.contiguous()
        if t.data_ptr() % 16:  # (the dithered encoder takes 16-byte aligned buffers)
            t = t.clone()
        _native.check(lib, lib.mgb_pcm_encode_dithered(C.byref(dither), t.data_ptr(), frames, bits, out.data_ptr(),
                                                       _stream_ptr(t.device)))
    host = HostIO.get().pool.array(tuple(out.shape), np.int16 if bits == 16 else np.uint8)
    torch.from_numpy(host).copy_(out)
    return host
