"""ctypes binding of libmatchering_b200.so (include/matchering_b200.h).

The product has exactly one compute path: the nvcc-built CUDA library next to this file.  If it
is missing or fails to load, importing the GPU entry points raises -- there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(PKG_DIR, "libmatchering_b200.so")

MGB_OK = 0
MGB_ERR_INVALID = -1
MGB_ERR_UNSUPPORTED = -2
MGB_ERR_WORKSPACE = -3
MGB_ERR_CUDA = -4
MGB_MAX_CORRECTION_STEPS = 16


MGB_MAX_FILTER_ORDER = 2


class LimiterParams(C.Structure):
    _fields_ = [
        ("threshold", C.c_double),
        ("reach", C.c_int32),
        ("hold", C.c_int32),
        ("warmup", C.c_int32),
        ("hold_order", C.c_int32),
        ("release_order", C.c_int32),
        ("reserved", C.c_int32),
        ("attack_c", C.c_double),
        ("hold_b", C.c_double * (MGB_MAX_FILTER_ORDER + 1)), ("hold_a", C.c_double * (MGB_MAX_FILTER_ORDER + 1)),
        ("release_b", C.c_double * (MGB_MAX_FILTER_ORDER + 1)), ("release_a", C.c_double * (MGB_MAX_FILTER_ORDER + 1)),
    ]

    @classmethod
    def from_constants(cls, lc) -> "LimiterParams":
        """plan.LimiterConstants -> the C struct (coefficients zero-padded above the filter's order)."""
        p = cls()
        p.threshold = lc.threshold
        p.reach, p.hold, p.warmup = lc.reach, lc.hold, lc.warmup
        p.attack_c = lc.attack_c
        p.hold_order, p.release_order = len(lc.hold_a) - 1, len(lc.release_a) - 1
        for name in ("hold_b", "hold_a", "release_b", "release_a"):
            dst = getattr(p, name)
            for i, v in enumerate(getattr(lc, name)):
                dst[i] = float(v)
        return p


class Plan(C.Structure):
    _fields_ = [
        ("sample_rate", C.c_int32),
        ("fft_size", C.c_int32),
        ("n_lin", C.c_int32), ("n_log", C.c_int32),
        ("rms_correction_steps", C.c_int32),
        ("lowess_k", C.c_int32),
        ("lowess_nfit", C.c_int32),
        ("lowess_nrows", C.c_int32),
        ("lowess_it", C.c_int32),
        ("reserved0", C.c_int32),
        ("max_piece_size", C.c_double),
        ("threshold", C.c_double),
        ("min_value", C.c_double),
        ("limiter", LimiterParams),
        ("d_sa_hinv", C.c_void_p), ("d_sa_lu", C.c_void_p), ("d_sa_end", C.c_void_p),
        ("d_sa_eval_idx", C.c_void_p), ("d_sa_eval_w", C.c_void_p),
        ("d_sb_hinv", C.c_void_p), ("d_sb_lu", C.c_void_p), ("d_sb_end", C.c_void_p),
        ("d_sb_eval_idx", C.c_void_p), ("d_sb_eval_w", C.c_void_p),
        ("d_lw_fit_idx", C.c_void_p), ("d_lw_fit_left", C.c_void_p), ("d_lw_seg", C.c_void_p),
        ("d_lw_alpha", C.c_void_p), ("d_lw_rows", C.c_void_p), ("d_lw_row_idx", C.c_void_p),
        ("d_hann", C.c_void_p),
        ("d_tw_f32_F", C.c_void_p), ("d_tw_f32_2F", C.c_void_p),
        ("d_tw_f64_F", C.c_void_p), ("d_tw_f64_2F", C.c_void_p),
        ("d_limiter_tables", C.c_void_p),
        ("d_smooth_op", C.c_void_p), ("d_smooth_op_rows", C.c_void_p),
    ]


class TrackState(C.Structure):
    _fields_ = [
        ("reference_peak", C.c_double),
        ("final_amplitude_coef", C.c_double),
        ("target_match_rms", C.c_double),
        ("reference_match_rms", C.c_double),
        ("rms_coefficient", C.c_double),
        ("gain", C.c_double),
        ("correction", C.c_double * MGB_MAX_CORRECTION_STEPS),
        ("result_peak", C.c_double),
        ("normalize_coef", C.c_double),
        ("conv_peak_bits", C.c_float),
        ("target_loud_pieces", C.c_int32),
        ("reference_loud_pieces", C.c_int32),
        ("limiter_engaged", C.c_int32),
        ("steps_done", C.c_int32),
        ("fir_peak_mid_bits", C.c_float),
        ("fir_peak_side_bits", C.c_float),
        ("conv_precise", C.c_int32),
    ]


class HostBuffers(C.Structure):
    _fields_ = [
        ("d_target_lr", C.c_void_p), ("d_reference_lr", C.c_void_p), ("d_result_lr", C.c_void_p),
        ("d_out_lr", C.c_void_p), ("d_wide", C.c_void_p), ("d_workspace", C.c_void_p), ("d_state", C.c_void_p),
    ]


class TrackLayout(C.Structure):
    _fields_ = [
        ("target_frames", C.c_int64), ("reference_frames", C.c_int64),
        ("target_piece", C.c_int64), ("reference_piece", C.c_int64),
        ("target_divisions", C.c_int32), ("reference_divisions", C.c_int32),
        ("target_slots", C.c_int32), ("reference_slots", C.c_int32),
        ("workspace_bytes", C.c_int64),
    ]


# name -> (restype, argtypes): every symbol include/matchering_b200.h declares
PROTOTYPES = {
    "mgb_version": (C.c_int, []),
    "mgb_last_error_string": (C.c_char_p, []),
    "mgb_set_option": (C.c_int, [C.c_char_p, C.c_int]),
    "mgb_launch_count": (C.c_longlong, []),
    "mgb_profile_enable": (C.c_int, [C.c_int]),
    "mgb_profile_collect": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(C.c_float), C.c_int]),
    "mgb_plan_twiddle_bytes": (C.c_int, [C.c_int32, C.POINTER(C.c_int64)]),
    "mgb_plan_fill_twiddles": (C.c_int, [C.POINTER(Plan), C.c_void_p]),
    "mgb_plan_operator_workspace_bytes": (C.c_int64, [C.POINTER(Plan)]),
    "mgb_plan_build_operator": (C.c_int, [C.POINTER(Plan), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "mgb_track_layout_init": (C.c_int, [C.POINTER(Plan), C.c_int64, C.c_int64, C.POINTER(TrackLayout)]),
    "mgb_match_levels": (C.c_int, [C.POINTER(Plan), C.POINTER(TrackLayout), C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p]),
    "mgb_match_frequencies": (C.c_int, [C.POINTER(Plan), C.POINTER(TrackLayout), C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p]),
    "mgb_correct_levels": (C.c_int, [C.POINTER(Plan), C.POINTER(TrackLayout), C.c_void_p, C.c_void_p, C.c_void_p]),
    "mgb_finalize": (C.c_int, [C.POINTER(Plan), C.POINTER(TrackLayout), C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mgb_limiter_workspace_bytes": (C.c_int64, [C.POINTER(LimiterParams), C.c_int64]),
    "mgb_limit": (C.c_int, [C.POINTER(LimiterParams), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                            C.c_void_p, C.c_void_p]),
    "mgb_process_host": (C.c_int, [C.POINTER(Plan), C.POINTER(TrackLayout), C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mgb_host_io_create": (C.c_int, [C.c_int32, C.c_int64, C.c_int32, C.POINTER(C.c_void_p)]),
    "mgb_host_io_destroy": (C.c_int, [C.c_void_p]),
    "mgb_host_io_threads": (C.c_int, [C.c_void_p]),
    "mgb_host_download_through_ring": (C.c_int, [C.c_int64]),
    "mgb_host_alloc": (C.c_void_p, [C.c_int64]),
    "mgb_host_free": (None, [C.c_void_p]),
    "mgb_host_upload": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p]),
    "mgb_host_download": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]),
    "mgb_stages_main_host": (C.c_int, [C.c_void_p, C.POINTER(Plan), C.POINTER(TrackLayout), C.c_void_p, C.c_void_p,
                                       C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                       C.POINTER(HostBuffers), C.POINTER(TrackState), C.c_void_p]),
    "mgb_limit_host": (C.c_int, [C.c_void_p, C.POINTER(LimiterParams), C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                 C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                 C.POINTER(C.c_int32), C.c_void_p]),
    "mgb_pipeline_create": (C.c_int, [C.POINTER(Plan), C.c_int64, C.c_int64, C.c_int32, C.POINTER(C.c_void_p)]),
    "mgb_pipeline_submit": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                      C.POINTER(C.c_int32)]),
    "mgb_pipeline_submit_pcm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_int32, C.c_int64,
                                          C.c_void_p, C.c_int32, C.POINTER(C.c_int32)]),
    "mgb_pipeline_wait": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(TrackState)]),
    "mgb_pipeline_streams": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]),
    "mgb_pipeline_destroy": (C.c_int, [C.c_void_p]),
    "mgb_convert_f64_to_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "mgb_convert_f32_to_f64": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "mgb_pcm_decode": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p]),
    "mgb_pcm_encode": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p]),
    "mgb_check_peaks": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "mgb_window_energy": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]),
    "mgb_preview_piece": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_double, C.c_int64, C.c_void_p]),
    "mgb_check_equality": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "mgb_resample_frames": (C.c_int64, [C.c_int64, C.c_int32, C.c_int32]),
    "mgb_resample": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32,
                               C.c_int32, C.c_void_p]),
    "mgb_test_limiter_gains": (C.c_int, [C.POINTER(LimiterParams), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                         C.c_void_p, C.c_void_p]),
    "mgb_test_fft": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                               C.c_void_p]),
    "mgb_test_design_fir": (C.c_int, [C.POINTER(Plan), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mgb_test_workspace_regions": (C.c_int, [C.POINTER(Plan), C.POINTER(TrackLayout), C.POINTER(C.c_int64)]),
}


class NativeError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"matchering_b200 native call failed ({status}): {message}")
        self.status = status


def bind(lib: C.CDLL) -> C.CDLL:
    """Attach prototypes; raises AttributeError if the library lacks a declared symbol."""
    for name, (restype, argtypes) in PROTOTYPES.items():
        fn = getattr(lib, name)
        fn.restype = restype
        fn.argtypes = argtypes
    return lib


def check(lib: C.CDLL, status: int) -> None:
    if status != MGB_OK:
        msg = lib.mgb_last_error_string()
        text = msg.decode("utf-8", "replace") if msg else ""
        if status == MGB_ERR_UNSUPPORTED:
            from .plan import UnsupportedConfig
            raise UnsupportedConfig(text)
        if status == MGB_ERR_INVALID:
            raise ValueError(text)
        raise NativeError(status, text)


_LIB = None


def load() -> C.CDLL:
    """The CUDA library, loaded once.  Fails loudly when it has not been built."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -m matchering_b200.build` "
                "(nvcc, sm_90a). matchering_b200 has no CPU fallback.")
        _LIB = bind(C.CDLL(LIB_PATH))
        if _LIB.mgb_version() < 200:
            raise ImportError("libmatchering_b200.so is older than this package")
    return _LIB
