"""Drive the emulator build of the kernels (tests/emul) with numpy buffers -- tests only."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "emul")):
    if p not in sys.path:
        sys.path.insert(0, p)

from matchering_b200 import _native, plan as plan_mod  # noqa: E402

_LIB = None


def emul_lib():
    """The emulator library; with MGB_EMUL_BUILD=racecheck, its ThreadSanitizer build (which needs libtsan
    preloaded into the process: tests/test_emul_racecheck.py runs the emulator tests that way)."""
    global _LIB
    if _LIB is None:
        import build_emul
        racecheck = os.environ.get("MGB_EMUL_BUILD", "") == "racecheck"
        _LIB = _native.bind(C.CDLL(build_emul.build(racecheck=racecheck)))
    return _LIB


def ptr(a: np.ndarray):
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


def aligned(shape, dtype, align=256):
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    raw = np.zeros(n + align, dtype=np.uint8)
    off = (-raw.ctypes.data) % align
    return raw[off:off + n].view(dtype).reshape(shape)


def aligned_copy(a, dtype=None):
    a = np.asarray(a)
    out = aligned(a.shape, dtype or a.dtype)
    out[...] = a
    return out


def limiter_params(lc: plan_mod.LimiterConstants) -> _native.LimiterParams:
    return _native.LimiterParams.from_constants(lc)


class EmulPlan:
    """mgb_plan over numpy memory (device pointers == host pointers in the emulator)."""

    def __init__(self, config, operator=False):
        self.lib = emul_lib()
        self.tables = plan_mod.build_tables(config)
        t = self.tables
        self.keep = {}
        s = _native.Plan()
        s.sample_rate, s.fft_size, s.n_lin, s.n_log = t.sample_rate, t.fft_size, t.n_lin, t.n_log
        s.rms_correction_steps, s.lowess_k = t.rms_correction_steps, t.lowess_k
        s.lowess_nfit = len(t.arrays["lw_fit_idx"])
        s.lowess_nrows = len(t.arrays["lw_rows"])
        s.lowess_it = t.lowess_it
        s.max_piece_size, s.threshold, s.min_value = t.max_piece_size, t.threshold, t.min_value
        s.limiter = limiter_params(t.limiter)
        for name, arr in t.arrays.items():
            buf = aligned_copy(arr)
            self.keep[name] = buf
            setattr(s, "d_" + name, buf.ctypes.data)
        sizes = (C.c_int64 * 5)()
        _native.check(self.lib, self.lib.mgb_plan_twiddle_bytes(t.fft_size, sizes))
        for name, nbytes in zip(("tw_f32_F", "tw_f32_2F", "tw_f64_F", "tw_f64_2F", "limiter_tables"), sizes):
            buf = aligned((nbytes,), np.uint8)
            self.keep[name] = buf
            setattr(s, "d_" + name, buf.ctypes.data)
        self.struct = s
        _native.check(self.lib, self.lib.mgb_plan_fill_twiddles(C.byref(s), None))
        if operator:
            ws_bytes = int(self.lib.mgb_plan_operator_workspace_bytes(C.byref(s)))
            ws = aligned((ws_bytes,), np.uint8)
            op = aligned((t.n_lin, t.n_lin), np.float64)
            _native.check(self.lib, self.lib.mgb_plan_build_operator(C.byref(s), ptr(op), ptr(ws), ws_bytes, None))
            values, rows = plan_mod.band_operator(np.array(op))
            self.keep["smooth_op"], self.keep["smooth_op_rows"] = aligned_copy(values), aligned_copy(rows)
            s.d_smooth_op = self.keep["smooth_op"].ctypes.data
            s.d_smooth_op_rows = self.keep["smooth_op_rows"].ctypes.data

    def layout(self, target_frames, reference_frames):
        L = _native.TrackLayout()
        _native.check(self.lib, self.lib.mgb_track_layout_init(C.byref(self.struct), target_frames, reference_frames,
                                                              C.byref(L)))
        return L


_PLANS = {}


def get_emul_plan(config, operator=False):
    key = (plan_mod.config_key(config), operator)
    if key not in _PLANS:
        _PLANS[key] = EmulPlan(config, operator)
    return _PLANS[key]


def run_pipeline(config, target_f32, reference_f32, need=(True, True, True), tma=1, operator=False):
    """All four stages through the emulator; returns (outputs, state, fir[2,F])."""
    lib = emul_lib()
    lib.mgb_set_option(b"tma", tma)
    ep = get_emul_plan(config, operator)
    T, R = len(target_f32), len(reference_f32)
    L = ep.layout(T, R)
    ws = aligned((L.workspace_bytes,), np.uint8)
    tgt = aligned_copy(target_f32, np.float32)
    ref = aligned_copy(reference_f32, np.float32)
    result = aligned((T, 2), np.float32)
    fir = aligned((2, config.fft_size), np.float64)
    state = _native.TrackState()
    P, LL = C.byref(ep.struct), C.byref(L)
    _native.check(lib, lib.mgb_match_levels(P, LL, ptr(tgt), ptr(ref), ptr(ws), C.byref(state), None))
    _native.check(lib, lib.mgb_match_frequencies(P, LL, ptr(tgt), ptr(result), ptr(fir), ptr(ws), C.byref(state), None))
    _native.check(lib, lib.mgb_correct_levels(P, LL, ptr(ws), C.byref(state), None))
    outs = [aligned((T, 2), np.float32) if n else None for n in need]
    _native.check(lib, lib.mgb_finalize(P, LL, ptr(result), *(ptr(o) if o is not None else None for o in outs),
                                        ptr(ws), C.byref(state), None))
    return outs, state, fir, result, L
