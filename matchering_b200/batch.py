"""Batches of tracks with host buffers: `depth` tracks in flight per GPU (mgb_pipeline_*).

A single `stages.main` call is bound by its own PCIe copies (190 MB for a 3-minute track against
well under a millisecond of kernels); independent tracks overlap them: while track k computes, track
k+1 is already arriving and track k-1's result is leaving.  This is the entry point for the
"batch of tracks sharded one-per-GPU" configuration; across GPUs use one process per GPU and
`sharding.tracks_for_rank`.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _native
from .engine import get_plan
from .loudness import Loudness, LoudnessTarget, debug_target, device_meter, target_params
from .profile import ReferenceProfile


class MasteringPipeline:
    def __init__(self, config, max_target_frames: int, max_reference_frames: int, depth: int = 3, device=None,
                 loudness: bool = False, dither: str = None, dither_seed: int = 0):
        """max_reference_frames bounds the references submitted as samples; profiles have no such bound
        (a pipeline that only takes profiles may pass smallest_reference_frames(config)).
        loudness=True meters every limited output on the device (mg.loudness's meter, at the Config's rate)
        and `wait_loudness` returns it.  With Config(loudness_target=T) every limited output is driven to T LUFS
        (mgb_pipeline_enable_loudness_target; its search uses the meter, which is then always on) and
        `wait_loudness_target` returns the meter and the search's report.
        dither ("tpdf" or "shaped", as in mg.Result) dithers every `submit_pcm` result with dither_seed
        (mgb_pipeline_enable_dither); float32 submissions are unaffected."""
        self.config = config
        self.plan = get_plan(config, device)
        self.lib = self.plan.lib
        self.device = self.plan.device
        self.depth = depth
        self._handle = C.c_void_p()
        # (the meter's tables are cached per device and rate: they outlive the pipeline)
        self.target = getattr(config, "loudness_target", None)
        self._meter = (device_meter(config.internal_sample_rate, self.device)
                       if loudness or self.target is not None else None)
        self._pending = {}  # slot -> (target, reference, out) kept alive until the slot is waited on
        dither_params = None
        if dither is not None:
            from .dither import params
            dither_params = params(dither, config.internal_sample_rate, dither_seed)
        with torch.cuda.device(self.device):
            _native.check(self.lib, self.lib.mgb_pipeline_create(C.byref(self.plan.struct), max_target_frames,
                                                                 max_reference_frames, depth, C.byref(self._handle)))
            if self._meter is not None:
                status = self.lib.mgb_pipeline_enable_loudness(self._handle, C.byref(self._meter.params))
                if status == _native.MGB_OK and self.target is not None:
                    status = self.lib.mgb_pipeline_enable_loudness_target(self._handle, C.byref(target_params(self.target)))
                if status != _native.MGB_OK:
                    self.close()
                    _native.check(self.lib, status)
            if dither_params is not None:
                status = self.lib.mgb_pipeline_enable_dither(self._handle, C.byref(dither_params))
                if status != _native.MGB_OK:
                    self.close()
                    _native.check(self.lib, status)

    @staticmethod
    def _ptr(a):
        if isinstance(a, torch.Tensor):
            assert a.dtype == torch.float32 and a.is_contiguous() and not a.is_cuda
            return a.data_ptr(), a.shape[0]
        assert a.dtype == np.float32 and a.flags["C_CONTIGUOUS"]
        return a.ctypes.data, a.shape[0]

    def _profile_blob(self, profile: ReferenceProfile):
        profile.check_config(self.config)
        return profile.checked_blob(self.plan)

    def submit(self, target, reference, out) -> int:
        """target, reference, out: (frames, 2) float32 host arrays (numpy or torch, ideally pinned).
        `reference` may be a ReferenceProfile: then no reference bytes are copied.
        Returns the slot to `wait` on; `out` is valid once that wait returns."""
        tp, tn = self._ptr(target)
        op, on = self._ptr(out)
        assert on == tn
        slot = C.c_int32()
        if isinstance(reference, ReferenceProfile):
            blob = self._profile_blob(reference)
            with torch.cuda.device(self.device):
                _native.check(self.lib, self.lib.mgb_pipeline_submit_profiled(self._handle, tp, tn, blob.data_ptr(), op,
                                                                              C.byref(slot)))
            self._pending[slot.value] = (target, blob, out)
            return slot.value
        rp, rn = self._ptr(reference)
        with torch.cuda.device(self.device):
            _native.check(self.lib, self.lib.mgb_pipeline_submit(self._handle, tp, tn, rp, rn, op, C.byref(slot)))
        self._pending[slot.value] = (target, reference, out)
        return slot.value

    def submit_pcm(self, target, reference, out) -> int:
        """PCM host buffers (what audio files hold): int16 arrays of shape (frames, 2), or uint8
        arrays of shape (frames, 6) for packed little-endian 24-bit.  `out` chooses the result's
        width the same way.  A quarter to a half of the PCIe bytes of `submit`."""
        def describe(a):
            a_np = a.numpy() if isinstance(a, torch.Tensor) else a
            if a_np.dtype == np.int16 and a_np.ndim == 2 and a_np.shape[1] == 2:
                bits = 16
            elif a_np.dtype == np.uint8 and a_np.ndim == 2 and a_np.shape[1] == 6:
                bits = 24
            else:
                raise TypeError("PCM buffers are int16 (frames, 2) or uint8 (frames, 6)")
            assert a_np.flags["C_CONTIGUOUS"]
            return a_np.ctypes.data, bits, a_np.shape[0]
        tp, tb, tn = describe(target)
        op, ob, on = describe(out)
        assert on == tn
        slot = C.c_int32()
        if isinstance(reference, ReferenceProfile):
            blob = self._profile_blob(reference)
            with torch.cuda.device(self.device):
                _native.check(self.lib, self.lib.mgb_pipeline_submit_pcm_profiled(self._handle, tp, tb, tn, blob.data_ptr(),
                                                                                  op, ob, C.byref(slot)))
            self._pending[slot.value] = (target, blob, out)
            return slot.value
        rp, rb, rn = describe(reference)
        with torch.cuda.device(self.device):
            _native.check(self.lib, self.lib.mgb_pipeline_submit_pcm(self._handle, tp, tb, tn, rp, rb, rn, op, ob,
                                                                     C.byref(slot)))
        self._pending[slot.value] = (target, reference, out)
        return slot.value

    def wait(self, slot: int) -> _native.TrackState:
        st = _native.TrackState()
        _native.check(self.lib, self.lib.mgb_pipeline_wait(self._handle, slot, C.byref(st)))
        self._pending.pop(slot, None)
        return st

    def wait_loudness(self, slot: int) -> tuple:
        """wait(slot), and the meter of the slot's limited output: (TrackState, Loudness).  Needs loudness=True."""
        if self._meter is None:
            raise ValueError("this pipeline was created without loudness=True")
        st, res = _native.TrackState(), _native.LoudnessResult()
        _native.check(self.lib, self.lib.mgb_pipeline_wait_loudness(self._handle, slot, C.byref(st), C.byref(res)))
        self._pending.pop(slot, None)
        return st, Loudness.from_result(res)

    def wait_loudness_target(self, slot: int) -> tuple:
        """wait(slot), the meter of the slot's limited output and how its loudness search ended:
        (TrackState, Loudness, LoudnessTarget).  Needs a Config with loudness_target."""
        if self.target is None:
            raise ValueError("this pipeline's Config has no loudness_target")
        st, res, rep = _native.TrackState(), _native.LoudnessResult(), _native.LoudnessTargetReport()
        _native.check(self.lib, self.lib.mgb_pipeline_wait_loudness_target(self._handle, slot, C.byref(st), C.byref(res),
                                                                            C.byref(rep)))
        self._pending.pop(slot, None)
        return st, Loudness.from_result(res), LoudnessTarget.from_report(self.target, rep)

    def wait_all(self) -> None:
        for slot in list(self._pending):
            self.wait(slot)

    def streams(self):
        h, c, d = C.c_void_p(), C.c_void_p(), C.c_void_p()
        _native.check(self.lib, self.lib.mgb_pipeline_streams(self._handle, C.byref(h), C.byref(c), C.byref(d)))
        return h.value, c.value, d.value

    def close(self) -> None:
        if self._handle:
            self.wait_all()
            self.lib.mgb_pipeline_destroy(self._handle)
            self._handle = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def smallest_reference_frames(config) -> int:
    """The shortest reference a pipeline can be created for: one piece just longer than fft_size."""
    return int(config.fft_size) + 1


def master_many(pairs, config, depth: int = 3, loudness: bool = False):
    """[(target, reference), ...] float32 host arrays -> list of limited results (numpy float32).  A reference
    may be a ReferenceProfile (an album against one reference: analysed once, never copied again).
    loudness=True returns (results, meters): each result's Loudness, metered on the device.  With
    Config(loudness_target=T) every result is driven to T LUFS; how each search ended goes to the debug log."""
    pairs = list(pairs)
    if not pairs:
        return ([], []) if loudness else []
    for _, r in pairs:  # a Config the profile was not made for fails before any device work
        if isinstance(r, ReferenceProfile):
            r.check_config(config)
    max_t = max(len(t) for t, _ in pairs)
    max_r = max((len(r) for _, r in pairs if not isinstance(r, ReferenceProfile)), default=smallest_reference_frames(config))
    outs = [np.empty((len(t), 2), dtype=np.float32) for t, _ in pairs]
    meters = [None] * len(pairs)
    target = getattr(config, "loudness_target", None) is not None

    def collect(pipe, slot, k):
        if target:
            _, meters[k], t = pipe.wait_loudness_target(slot)
            debug_target(t)
        else:
            meters[k] = pipe.wait_loudness(slot)[1]

    with MasteringPipeline(config, max_t, max_r, depth, loudness=loudness) as pipe:
        in_flight = []  # (slot, track) in submission order; slots are reused round-robin
        for i, ((t, r), o) in enumerate(zip(pairs, outs)):
            if not isinstance(r, ReferenceProfile):
                r = np.ascontiguousarray(r, dtype=np.float32)
            if (loudness or target) and len(in_flight) == depth:  # collect the slot this submit reuses
                collect(pipe, *in_flight.pop(0))
            in_flight.append((pipe.submit(np.ascontiguousarray(t, dtype=np.float32), r, o), i))
        if loudness or target:
            for slot, k in in_flight:
                collect(pipe, slot, k)
        pipe.wait_all()
    return (outs, meters) if loudness else outs
