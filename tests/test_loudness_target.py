"""Loudness targets without a GPU: the float64 search (tests/loudness_target_oracle.py) on its own, and
mgb_limit_to_loudness / mgb_finalize_to_loudness on the CPU emulator against it, on poisoned workspaces, in other thread
orders and under ThreadSanitizer; the argument checks and Config's validation."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from emul_harness import aligned, aligned_copy, emul_lib, get_emul_plan, ptr, run_pipeline  # (puts oracle/ on sys.path)
import loudness
import loudness_target_oracle as lto
import port
import matchering_b200 as mg
from matchering_b200 import _native, plan
from test_loudness import emul_params

TOL = 1e-5  # the limiter's parity bound
CHUNK = 4608  # kLimiterCore
WIDE = dict(attack=50, hold_filter_order=2, release_filter_order=2)


def material(kind, n, fs=44100):
    if kind == "noise":
        return port.synth_target(n, 41, kind="plain").astype(np.float64) * 0.5
    if kind == "tonal":
        return port.synth_tonal(n, 42, fs).astype(np.float64)
    if kind == "c5":
        return port.synth_limiter_input(n, 43).astype(np.float64) * 0.3
    return port.synth_target(n, 44).astype(np.float64) * 0.4  # enveloped


def cfg_of(fs=44100, true_peak=False, **limiter):
    return mg.Config(internal_sample_rate=fs, true_peak=true_peak, limiter=mg.LimiterConfig(**limiter) if limiter else None)


def target_of(t, x=lto.MAX_GAIN_DB):
    p = _native.LoudnessTargetParams()
    p.target_lufs, p.max_gain_db = t, x
    return p


def emul_limit_to_loudness(x, cfg, target, max_gain_db=lto.MAX_GAIN_DB, pattern=None):
    """mgb_limit_to_loudness on the emulator -> (output, report)."""
    lib = emul_lib()
    params = _native.LimiterParams.from_constants(plan.limiter_constants(cfg))
    meter = emul_params(cfg.internal_sample_rate)
    n = len(x)
    nbytes = int(lib.mgb_limiter_workspace_bytes(C.byref(params), n)) + int(
        lib.mgb_loudness_target_workspace_bytes(C.byref(meter), n))
    ws = aligned((nbytes,), np.uint8)
    if pattern == "ff":
        ws[...] = 0xFF
    xi, out = aligned_copy(x, np.float32), aligned((n, 2), np.float32)
    rep = aligned((C.sizeof(_native.LoudnessTargetReport),), np.uint8)
    rep[...] = 0xFF
    _native.check(lib, lib.mgb_limit_to_loudness(C.byref(params), C.byref(meter), C.byref(target_of(target, max_gain_db)),
                                                 ptr(xi), ptr(out), n, ptr(ws), nbytes, ptr(rep), None))
    return np.array(out), _native.LoudnessTargetReport.from_buffer_copy(bytes(rep))


def emul_limit(x, cfg):
    lib = emul_lib()
    params = _native.LimiterParams.from_constants(plan.limiter_constants(cfg))
    n = len(x)
    nbytes = int(lib.mgb_limiter_workspace_bytes(C.byref(params), n))
    ws, xi, out, eng = aligned((nbytes,), np.uint8), aligned_copy(x, np.float32), aligned((n, 2), np.float32), aligned((4,), np.int32)
    _native.check(lib, lib.mgb_limit(C.byref(params), ptr(xi), ptr(out), n, ptr(ws), nbytes, ptr(eng), None))
    return np.array(out)


def assert_report_matches(rep, want):
    assert rep.passes == want["passes"] and rep.status == want["status"], (rep.passes, rep.status, want["trace"])
    for k, (x, I) in enumerate(want["trace"]):
        assert abs(rep.trace_gain_db[k] - x) < 1e-4, (k, rep.trace_gain_db[k], x)
        assert rep.trace_integrated[k] == I or abs(rep.trace_integrated[k] - I) < 1e-3, (k, rep.trace_integrated[k], I)
    assert rep.gain_db == rep.trace_gain_db[rep.passes - 1] and rep.integrated == rep.trace_integrated[rep.passes - 1]
    I_s = want["input_integrated"]
    assert rep.input_integrated == I_s or abs(rep.input_integrated - I_s) < 1e-3


# ---- the oracle on its own ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["noise", "tonal", "c5", "enveloped"])
def test_oracle_reaches_targets(kind):
    """-20 .. -6 LUFS on four materials: REACHED within 0.01 LU in at most 8 passes, or UNREACHABLE at the largest drive;
    the measured curve rises at most 1 LU per dB between the points the search visits, as its one-sided steps assume."""
    fs = 44100
    s = material(kind, 6 * fs, fs)
    cfg = cfg_of(fs)
    for target in (-20.0, -14.0, -9.0, -6.0, -3.0):
        r = lto.search(s, cfg, target)
        assert r["passes"] <= lto.MAX_PASSES
        if r["status"] == lto.REACHED:
            assert abs(r["integrated"] - target) <= lto.TOLERANCE
            assert abs(lto.integrated(r["output"], fs) - target) <= lto.TOLERANCE
        else:
            assert r["status"] == lto.UNREACHABLE and target >= -9.0, (kind, target, r["status"], r["trace"])
            assert r["gain_db"] == lto.MAX_GAIN_DB
        pts = sorted(r["trace"])
        for (x0, i0), (x1, i1) in zip(pts, pts[1:]):
            if x1 - x0 > 1e-6:
                assert (i1 - i0) / (x1 - x0) <= 1.0 + 1e-6, (kind, target, pts)


# ---- mgb_limit_to_loudness against the oracle ------------------------------------------------------------------------
CASES = [(44100, False, {}, -14.0), (48000, True, {}, -12.0), (96000, False, {}, -10.0), (96000, True, {}, -16.0),
         (44100, False, WIDE, -11.0), (44100, True, WIDE, -13.0)]


@pytest.mark.parametrize("fs,tp,limiter,target", CASES,
                         ids=["44100", "48000-tp", "96000", "96000-tp", "44100-wide", "44100-wide-tp"])
def test_limit_to_loudness_matches_oracle_emulated(fs, tp, limiter, target):
    cfg = cfg_of(fs, tp, **limiter)
    x = material("c5", 2 * fs + 333, fs)
    got, rep = emul_limit_to_loudness(x, cfg, target)
    want = lto.search(x.astype(np.float32).astype(np.float64), cfg, target)
    assert_report_matches(rep, want)
    assert rep.status == lto.REACHED
    assert float(np.abs(got - lto.limited(x.astype(np.float32).astype(np.float64), rep.gain_db, cfg)).max()) < TOL
    assert abs(lto.integrated(got.astype(np.float64), fs) - target) <= lto.TOLERANCE


# ---- edge cases -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["silence", "short"])
def test_undefined_input_gives_the_plain_limiter_emulated(kind):
    cfg = cfg_of()
    x = np.zeros((3 * CHUNK, 2)) if kind == "silence" else material("c5", 17000)  # 17000 < one 400 ms window
    got, rep = emul_limit_to_loudness(x, cfg, -14.0)
    assert rep.status == lto.UNDEFINED and rep.passes == 1 and rep.gain_db == 0.0
    assert math.isinf(rep.input_integrated) and rep.input_integrated < 0
    np.testing.assert_array_equal(got, emul_limit(x, cfg))


def test_quieter_target_takes_one_pass_through_the_bypass_emulated():
    cfg = cfg_of()
    x = material("noise", 2 * 44100)
    got, rep = emul_limit_to_loudness(x, cfg, -40.0)
    assert rep.passes == 1 and rep.status == lto.REACHED and rep.gain_db < -20
    k = 10.0 ** (rep.gain_db / 20.0)
    want = (x.astype(np.float32).astype(np.float64) * k).astype(np.float32)  # the limiter's early-out: x * pre
    np.testing.assert_array_equal(got, want)


def test_unreachable_target_ends_at_the_largest_drive_emulated():
    cfg = cfg_of()
    x = material("c5", 2 * 44100)
    got, rep = emul_limit_to_loudness(x, cfg, -1.0, max_gain_db=6.0)
    assert rep.status == lto.UNREACHABLE and rep.gain_db == 6.0
    want = lto.search(x.astype(np.float32).astype(np.float64), cfg, -1.0, 6.0)
    assert_report_matches(rep, want)
    assert float(np.abs(got - lto.limited(x.astype(np.float32).astype(np.float64), 6.0, cfg)).max()) < TOL


@pytest.mark.parametrize("n", [7, 13, CHUNK + 1, 17640, 3 * CHUNK])
def test_track_lengths_emulated(n):
    """From 7 frames (no sub-block: UNDEFINED) to three chunks (a complete window at 44.1 kHz from 17640 frames)."""
    cfg = cfg_of()
    x = material("c5", n)
    got, rep = emul_limit_to_loudness(x, cfg, -12.0)
    want = lto.search(x.astype(np.float32).astype(np.float64), cfg, -12.0)
    assert_report_matches(rep, want)
    assert float(np.abs(got - want["output"]).max()) < TOL


def test_poisoned_workspace_changes_nothing_emulated():
    for cfg in (cfg_of(), cfg_of(44100, True, **WIDE)):
        x = material("c5", 44100 + 777)
        a, ra = emul_limit_to_loudness(x, cfg, -13.0)
        b, rb = emul_limit_to_loudness(x, cfg, -13.0, pattern="ff")
        np.testing.assert_array_equal(a, b)
        assert bytes(ra) == bytes(rb)


# ---- mgb_finalize_to_loudness after stages 1-3 -------------------------------------------------------------------------
def emul_finalize_to_loudness(cfg, t, r, target, max_gain_db=lto.MAX_GAIN_DB, profile=None, search_fill=0xFF):
    """Stages 1-3 through the emulator (the reference from `profile`, a profile blob, when given), then
    mgb_finalize_to_loudness on a search workspace filled with `search_fill` -> (limited, report, state, plain output,
    result)."""
    (_, plain, _), state, _, result, L = run_pipeline(cfg, t, r, need=(False, True, False))
    lib = emul_lib()
    ep = get_emul_plan(cfg)
    meter = emul_params(cfg.internal_sample_rate)
    if profile is not None:
        L = _native.TrackLayout()
        _native.check(lib, lib.mgb_track_layout_init_profiled(C.byref(ep.struct), len(t), C.byref(L)))
    ws = aligned((L.workspace_bytes,), np.uint8)
    # a fresh job workspace: run the three stages again into it (run_pipeline keeps its own)
    tgt, ref = aligned_copy(t, np.float32), aligned_copy(r, np.float32)
    res = aligned((len(t), 2), np.float32)
    st = _native.TrackState()
    P, LL = C.byref(ep.struct), C.byref(L)
    if profile is not None:
        _native.check(lib, lib.mgb_match_levels_profiled(P, LL, ptr(tgt), ptr(profile), ptr(ws), C.byref(st), None))
    else:
        _native.check(lib, lib.mgb_match_levels(P, LL, ptr(tgt), ptr(ref), ptr(ws), C.byref(st), None))
    _native.check(lib, lib.mgb_match_frequencies(P, LL, ptr(tgt), ptr(res), None, ptr(ws), C.byref(st), None))
    _native.check(lib, lib.mgb_correct_levels(P, LL, ptr(ws), C.byref(st), None))
    nbytes = int(lib.mgb_loudness_target_workspace_bytes(C.byref(meter), len(t)))
    search = aligned((nbytes,), np.uint8)
    search[...] = search_fill
    out = aligned((len(t), 2), np.float32)
    rep = aligned((C.sizeof(_native.LoudnessTargetReport),), np.uint8)
    _native.check(lib, lib.mgb_finalize_to_loudness(P, LL, C.byref(meter), C.byref(target_of(target, max_gain_db)), ptr(res),
                                                    ptr(out), ptr(ws), ptr(search), nbytes, C.byref(st), ptr(rep), None))
    return np.array(out), _native.LoudnessTargetReport.from_buffer_copy(bytes(rep)), st, plain, res


@pytest.mark.parametrize("tp", [False, True])
def test_finalize_to_loudness_matches_oracle_emulated(tp):
    cfg = mg.Config(max_piece_size=1.0, true_peak=tp)
    n = 44100 * 3 + 123
    t, r = port.synth_target(n, 51), port.synth_reference(n - 999, 52)
    got, rep, st, plain, _ = emul_finalize_to_loudness(cfg, t, r, -12.0)
    want = lto.main(t, r, cfg, -12.0)
    assert_report_matches(rep, want)
    assert rep.status == lto.REACHED
    assert float(np.abs(got - want["output"]).max()) < TOL
    assert abs(lto.integrated(got.astype(np.float64), 44100) - -12.0) <= lto.TOLERANCE
    # the un-limited output is mgb_finalize's, untouched by the target
    _, _, _, plain_w, _ = emul_finalize_to_loudness(cfg, t, r, -20.0)
    np.testing.assert_array_equal(plain, plain_w)


def test_finalize_at_zero_drive_is_the_plain_finalize_emulated():
    """A target at the loudness of s with no room to drive (max_gain_db = 0): one pass at x = 0, which with
    final_amplitude_coef = 1 writes mgb_finalize's limited output bit for bit."""
    cfg = mg.Config(max_piece_size=1.0)
    n = 44100 * 3 + 7
    t, r = port.synth_target(n, 61), port.synth_reference(n, 62) * np.float32(1.2)  # the reference reaches the threshold
    (lim, _, _), st0, _, _, _ = run_pipeline(cfg, t, r, need=(True, False, False))
    assert st0.final_amplitude_coef == 1.0
    _, _, _, _, res = emul_finalize_to_loudness(cfg, t, r, -14.0)
    _, first, _, _, _ = emul_finalize_to_loudness(cfg, t, r, -14.0)
    got, rep, _, _, _ = emul_finalize_to_loudness(cfg, t, r, first.input_integrated, max_gain_db=0.0)
    assert rep.passes == 1 and rep.gain_db == 0.0
    assert rep.status in (lto.REACHED, lto.UNREACHABLE)
    np.testing.assert_array_equal(got, lim)


def test_quiet_reference_reaches_the_threshold_emulated():
    """A quiet reference (final_amplitude_coef < 1) no longer lowers the ceiling: a loud target's peaks reach the
    threshold, not threshold * coef."""
    cfg = mg.Config(max_piece_size=1.0)
    n = 44100 * 3 + 11
    t, r = port.synth_target(n, 71), port.synth_reference(n, 72, kind="quiet") * np.float32(0.5)
    got, rep, st, _, _ = emul_finalize_to_loudness(cfg, t, r, -8.0)
    assert st.final_amplitude_coef < 0.99
    peak = float(np.abs(got).max())
    assert peak > cfg.threshold * st.final_amplitude_coef * 1.001
    assert peak <= cfg.threshold * (1 + 1e-6)
    assert rep.status in (lto.REACHED, lto.UNREACHABLE)


def test_finalize_search_workspace_and_profile_change_nothing_emulated():
    """The same job's report and output from a zeroed and a 0xFF search workspace, and from a reference profile in
    place of the reference's samples: byte for byte."""
    from test_reference_profile import emul_profile
    cfg = mg.Config(max_piece_size=1.0, true_peak=True)
    n = 44100 * 2 + 501
    t, r = port.synth_target(n, 81), port.synth_reference(n - 777, 82)
    a, ra, _, _, _ = emul_finalize_to_loudness(cfg, t, r, -11.0, search_fill=0)
    b, rb, _, _, _ = emul_finalize_to_loudness(cfg, t, r, -11.0, search_fill=0xFF)
    blob, _ = emul_profile(cfg, r)
    c, rc, _, _, _ = emul_finalize_to_loudness(cfg, t, r, -11.0, profile=blob)
    assert ra.passes >= 1 and ra.status == lto.REACHED
    for out, rep in ((b, rb), (c, rc)):
        np.testing.assert_array_equal(out, a)
        assert bytes(rep) == bytes(ra)


def test_output_may_not_alias_the_input_emulated():
    lib = emul_lib()
    cfg = cfg_of()
    params = _native.LimiterParams.from_constants(plan.limiter_constants(cfg))
    meter = emul_params(44100)
    n = 20000
    nbytes = int(lib.mgb_limiter_workspace_bytes(C.byref(params), n)) + int(
        lib.mgb_loudness_target_workspace_bytes(C.byref(meter), n))
    ws, x = aligned((nbytes,), np.uint8), aligned((n, 2), np.float32)
    rep = aligned((C.sizeof(_native.LoudnessTargetReport),), np.uint8)
    assert lib.mgb_limit_to_loudness(C.byref(params), C.byref(meter), C.byref(target_of(-14.0)), ptr(x), ptr(x), n, ptr(ws),
                                     nbytes, ptr(rep), None) == _native.MGB_ERR_INVALID
    ep = get_emul_plan(mg.Config(max_piece_size=1.0))
    L = ep.layout(50000, 50000)
    job = aligned((L.workspace_bytes,), np.uint8)
    res = aligned((50000, 2), np.float32)
    sb = int(lib.mgb_loudness_target_workspace_bytes(C.byref(meter), 50000))
    search = aligned((sb,), np.uint8)
    st = _native.TrackState()
    assert lib.mgb_finalize_to_loudness(C.byref(ep.struct), C.byref(L), C.byref(meter), C.byref(target_of(-14.0)), ptr(res),
                                        ptr(res), ptr(job), ptr(search), sb, C.byref(st), ptr(rep),
                                        None) == _native.MGB_ERR_INVALID


# ---- the batch pipeline -----------------------------------------------------------------------------------------------
def _pcm16(x):
    return np.clip(np.rint(np.asarray(x, np.float64) * 32767.0), -32768, 32767).astype(np.int16)


def test_pipeline_reports_what_the_single_job_reports_emulated():
    """A depth-2 pipeline with metering and a target, fed paired and profiled, float32 and PCM16 jobs: every float32
    output and report is the single-job entry's (mgb_finalize_to_loudness) byte for byte, every meter is mgb_loudness of
    the slot's output, and the PCM jobs report what the float32 jobs of the same samples report.  Enabling a target
    before metering, twice, or after a submit is refused; a pipeline without a target masters as before."""
    from test_loudness import emul_meter
    from test_reference_profile import emul_profile
    lib = emul_lib()
    cfg = port.OracleConfig(fft_size=1024, max_piece_size=0.3)
    fs = cfg.internal_sample_rate
    ep = get_emul_plan(cfg)
    lengths = [20011, 19003]
    pcm_t = [_pcm16(port.synth_target(n, 90 + k) * 1.6) for k, n in enumerate(lengths)]
    targets = [(q.astype(np.float64) / 32768.0).astype(np.float32) for q in pcm_t]
    pcm_r = _pcm16(port.synth_reference(18000, 93))
    r = (pcm_r.astype(np.float64) / 32768.0).astype(np.float32)
    blob, _ = emul_profile(cfg, r)
    goal = target_of(-13.0, lto.MAX_GAIN_DB)

    def run(with_target):
        h = C.c_void_p()
        _native.check(lib, lib.mgb_pipeline_create(C.byref(ep.struct), max(lengths), len(r), 2, C.byref(h)))
        results, keep = [], []
        try:
            if with_target:
                assert lib.mgb_pipeline_enable_loudness_target(h, C.byref(goal)) == _native.MGB_ERR_INVALID  # no meter yet
            _native.check(lib, lib.mgb_pipeline_enable_loudness(h, C.byref(emul_params(fs))))
            if with_target:
                _native.check(lib, lib.mgb_pipeline_enable_loudness_target(h, C.byref(goal)))
                assert lib.mgb_pipeline_enable_loudness_target(h, C.byref(goal)) == _native.MGB_ERR_INVALID  # twice
            for k in range(len(targets)):
                for kind in ("float", "pcm"):
                    for profiled in (False, True):
                        slot = C.c_int32(-1)
                        if kind == "pcm":
                            tt, rr, o = aligned_copy(pcm_t[k]), aligned_copy(pcm_r), aligned((len(targets[k]), 2), np.int16)
                            rc = (lib.mgb_pipeline_submit_pcm_profiled(h, ptr(tt), 16, len(tt), ptr(blob), ptr(o), 16,
                                                                       C.byref(slot)) if profiled
                                  else lib.mgb_pipeline_submit_pcm(h, ptr(tt), 16, len(tt), ptr(rr), 16, len(rr), ptr(o), 16,
                                                                   C.byref(slot)))
                        else:
                            tt, rr, o = aligned_copy(targets[k]), aligned_copy(r), aligned((len(targets[k]), 2), np.float32)
                            rc = (lib.mgb_pipeline_submit_profiled(h, ptr(tt), len(tt), ptr(blob), ptr(o), C.byref(slot))
                                  if profiled else lib.mgb_pipeline_submit(h, ptr(tt), len(tt), ptr(rr), len(rr), ptr(o),
                                                                           C.byref(slot)))
                        _native.check(lib, rc)
                        st, res, rep = _native.TrackState(), _native.LoudnessResult(), _native.LoudnessTargetReport()
                        if with_target:
                            _native.check(lib, lib.mgb_pipeline_wait_loudness_target(h, slot.value, C.byref(st), C.byref(res),
                                                                                     C.byref(rep)))
                        else:
                            assert lib.mgb_pipeline_wait_loudness_target(h, slot.value, C.byref(st), C.byref(res),
                                                                         C.byref(rep)) == _native.MGB_ERR_INVALID
                            _native.check(lib, lib.mgb_pipeline_wait_loudness(h, slot.value, C.byref(st), C.byref(res)))
                        keep.append((tt, rr))
                        results.append((k, kind, profiled, np.array(o), bytes(res), bytes(rep)))
            if with_target:
                assert lib.mgb_pipeline_enable_loudness_target(h, C.byref(goal)) == _native.MGB_ERR_INVALID  # after a submit
        finally:
            lib.mgb_pipeline_destroy(h)
        return results

    targeted, plain = run(True), run(False)
    for k in range(len(targets)):
        want, want_rep, _, _, _ = emul_finalize_to_loudness(cfg, targets[k], r, -13.0)
        assert want_rep.status == lto.REACHED
        for kk, kind, profiled, o, raw, rep in targeted:
            if kk != k:
                continue
            assert rep == bytes(want_rep), (k, kind, profiled)
            if kind == "float":
                np.testing.assert_array_equal(o, want)
                assert raw == emul_meter(o, fs)
                assert abs(_native.LoudnessResult.from_buffer_copy(raw).integrated - -13.0) <= lto.TOLERANCE
                # the search's integrated-only meter and the full meter gate the same way, to the bit
                assert _native.LoudnessTargetReport.from_buffer_copy(rep).integrated == \
                    _native.LoudnessResult.from_buffer_copy(raw).integrated
        # without a target: mgb_finalize's limited output, as before
        (lim, _, _), _, _, _, _ = run_pipeline(cfg, targets[k], r, need=(True, False, False))
        for kk, kind, profiled, o, _, _ in plain:
            if kk == k and kind == "float":
                np.testing.assert_array_equal(o, lim)


# ---- argument checks and Config -------------------------------------------------------------------------------------
def test_argument_errors_emulated():
    lib = emul_lib()
    cfg = cfg_of()
    params = _native.LimiterParams.from_constants(plan.limiter_constants(cfg))
    meter = emul_params(44100)
    n = 20000
    nbytes = int(lib.mgb_limiter_workspace_bytes(C.byref(params), n)) + int(
        lib.mgb_loudness_target_workspace_bytes(C.byref(meter), n))
    ws, x, out = aligned((nbytes,), np.uint8), aligned((n, 2), np.float32), aligned((n, 2), np.float32)
    rep = aligned((C.sizeof(_native.LoudnessTargetReport),), np.uint8)

    def call(target=-14.0, gain=24.0, xp=None, size=nbytes, m=meter):
        return lib.mgb_limit_to_loudness(C.byref(params), C.byref(m), C.byref(target_of(target, gain)),
                                         xp if xp is not None else ptr(x), ptr(out), n, ptr(ws), size, ptr(rep), None)
    assert call() == _native.MGB_OK
    for bad in (float("nan"), float("inf"), 0.0, 1.0, -70.0, -90.0):
        assert call(target=bad) == _native.MGB_ERR_INVALID, bad
    for bad in (-0.5, 48.5, float("nan")):
        assert call(gain=bad) == _native.MGB_ERR_INVALID, bad
    assert call(xp=C.c_void_p(x.ctypes.data + 4)) == _native.MGB_ERR_INVALID
    assert call(size=nbytes - 1) == _native.MGB_ERR_WORKSPACE
    assert lib.mgb_loudness_target_workspace_bytes(C.byref(meter), 0) == -1
    # a meter of another rate than the plan's
    ep = get_emul_plan(mg.Config(max_piece_size=1.0))
    L = ep.layout(50000, 50000)
    m48 = emul_params(48000)
    big = aligned((max(L.workspace_bytes, nbytes),), np.uint8)
    assert lib.mgb_finalize_to_loudness(C.byref(ep.struct), C.byref(L), C.byref(m48), C.byref(target_of(-14.0)),
                                        ptr(out), ptr(out), ptr(big), ptr(ws), nbytes, ptr(big), ptr(rep),
                                        None) == _native.MGB_ERR_INVALID


def test_config_validation():
    assert mg.Config().loudness_target is None
    assert mg.Config(loudness_target=-14).loudness_target == -14.0
    for bad in (0, 3.0, float("nan"), float("-inf"), -70, "loud", True):
        with pytest.raises(AssertionError):
            mg.Config(loudness_target=bad)
    # the target is not part of the plan: a reference profile and the plan cache stay valid across targets
    assert plan.config_key(mg.Config(loudness_target=-14)) == plan.config_key(mg.Config())


# ---- the same kernels under ThreadSanitizer and in other thread orders ----------------------------------------------
HERE = "tests/test_loudness_target.py::"
RACECHECK_IDS = [HERE + "test_track_lengths_emulated[13]", HERE + f"test_track_lengths_emulated[{CHUNK + 1}]",
                 HERE + "test_dump_for_thread_orders_emulated"]


def test_dump_for_thread_orders_emulated():
    """Outputs and reports of fixed inputs (halo and wide-window, both peak modes); with MGB_TARGET_DUMP set, their
    bytes go to that file (the thread-order runs below compare them with a forward run)."""
    raws = b""
    x = material("c5", 22050 + 3 * CHUNK)
    for cfg in (cfg_of(), cfg_of(44100, True, **WIDE)):
        out, rep = emul_limit_to_loudness(x, cfg, -12.5)
        raws += out.tobytes() + bytes(rep)
    if os.environ.get("MGB_TARGET_DUMP"):
        with open(os.environ["MGB_TARGET_DUMP"], "wb") as f:
            f.write(raws)


@pytest.fixture(scope="module")
def other_runs(tmp_path_factory):
    from concurrent.futures import ThreadPoolExecutor

    import build_emul
    from test_emul_racecheck import run_group, tsan_env
    build_emul.build(racecheck=True)
    build_emul.build()
    base = tmp_path_factory.mktemp("loudness_target_racecheck")
    jobs = {}
    for k, i in enumerate(RACECHECK_IDS):
        log_dir = str(base / f"tsan_{k}")
        env = tsan_env(log_dir)
        env["MGB_EMUL_BUILD"] = "racecheck"
        jobs[("tsan", k)] = ([i], env, log_dir)
    for order in ("forward", "reverse", "seeded"):
        env = dict(os.environ, MGB_EMUL_ORDER=order, MGB_EMUL_SEED="4242", MGB_TARGET_DUMP=str(base / f"dump_{order}.bin"))
        jobs[(order, 0)] = ([RACECHECK_IDS[-1]], env, str(base / order))
    with ThreadPoolExecutor(max_workers=6) as ex:
        futures = {key: ex.submit(run_group, *job) for key, job in jobs.items()}
        done = {key: f.result() + (jobs[key][2],) for key, f in futures.items()}
    return done, base


@pytest.mark.parametrize("k", range(len(RACECHECK_IDS)))
def test_loudness_target_kernels_have_no_data_races(other_runs, k):
    from test_emul_racecheck import reports
    rc, out, _, log_dir = other_runs[0][("tsan", k)]
    n, first = reports(log_dir)
    assert n == 0, f"{n} ThreadSanitizer report(s) in {RACECHECK_IDS[k]}; the first:\n{first}"
    assert rc == 0, out


@pytest.mark.parametrize("order", ["reverse", "seeded"])
def test_loudness_target_is_bit_identical_in_other_thread_orders(other_runs, order):
    done, base = other_runs
    for o in ("forward", order):
        rc, out, _, _ = done[(o, 0)]
        assert rc == 0, out
    forward = (base / "dump_forward.bin").read_bytes()
    assert len(forward) > 0
    assert (base / f"dump_{order}.bin").read_bytes() == forward
