"""Linked versions (mgb_version_match_frequencies, mgb_finalize_versions, mgb_finalize_versions_to_loudness,
stages.main_versions, mg.process_versions) on the CPU: the float64 restatement against oracle/port.py, the emulator build
against the restatement and against the single job, argument errors and refusals."""
import ctypes as C
import os

import numpy as np
import pytest

import loudness_target_oracle as lto
import port
import versions_oracle
from emul_harness import aligned_copy, emul_lib, get_emul_plan, ptr
from matchering_b200 import _native
from test_loudness import emul_params
from test_loudness_target import target_of
from test_reference_profile import emul_profile, ebuf, profiled_layout

import matchering_b200 as mg
from matchering_b200 import stages

TOL = 1e-5  # the pipeline's parity bound
N = 44100 * 2 + 313
WIDE = dict(attack=50, hold_filter_order=2, release_filter_order=2)  # the wide-window limiter path


def cfg_of(true_peak=False, **limiter):
    return mg.Config(max_piece_size=0.5, true_peak=true_peak, limiter=mg.LimiterConfig(**limiter) if limiter else None)


def parts(n=N, seed=0):
    """a (an instrumental) and b (a vocal-like tonal part), float32"""
    a = port.synth_target(n, 80 + seed).astype(np.float64) * 0.6
    b = port.synth_tonal(n, 90 + seed).astype(np.float64) * 0.35
    return a.astype(np.float32), b.astype(np.float32)


def reference():
    return port.synth_reference(44100 + 77, 52)


# ---- the restatement -------------------------------------------------------------------------------------------------
def test_oracle_without_versions_is_port_main():
    cfg = cfg_of()
    a, b = parts()
    x, r = (a + b), reference()
    got = versions_oracle.main_versions([x], r, cfg, True, True, True)[0]
    want = port.main(x.astype(np.float64), r.astype(np.float64), cfg, True, True, True)
    for g, w in zip(got, want):
        assert float(np.abs(g - w).max()) <= 1e-12


def test_oracle_half_version_is_half_the_main():
    cfg = cfg_of()
    a, b = parts()
    x = a + b
    outs = versions_oracle.main_versions([x, 0.5 * x], reference(), cfg, True, True, True)
    for m, v in zip(*outs):
        assert float(np.abs(v - 0.5 * m).max()) <= 1e-12


def test_oracle_main_minus_instrumental_is_the_vocal_through_the_chain():
    cfg = cfg_of()
    a, b = parts()
    tr = {}
    outs = versions_oracle.main_versions([a + b, a], reference(), cfg, True, True, False, trace=tr)
    e = versions_oracle.envelope(tr["D"], cfg)
    want = versions_oracle.chain(b, tr) * e[:, None] * tr["final_coef"]
    assert float(np.abs((outs[0][0] - outs[1][0]) - want).max()) <= 1e-6  # (float64 FFT convolutions of 0.35-peak material)


# ---- emulator drivers ------------------------------------------------------------------------------------------------
def run_versions(cfg, targets, r=None, blob=None, pattern=None, lufs=None, need=(True, True, True)):
    """Stages 1-3 of targets[0] (paired with r, or profiled from blob), mgb_version_match_frequencies for the others,
    then mgb_finalize_versions (or, with lufs, the limited outputs from mgb_finalize_versions_to_loudness)
    -> ([(limited, plain, normalized) per target], main state bytes, report or None)"""
    lib, ep = emul_lib(), get_emul_plan(cfg)
    P = C.byref(ep.struct)
    T = len(targets[0])
    if blob is not None:
        L = profiled_layout(lib, ep, T)
    else:
        L = _native.TrackLayout()
        _native.check(lib, lib.mgb_track_layout_init(P, T, len(r), C.byref(L)))
    LL = C.byref(L)
    ws = ebuf(L.workspace_bytes, pattern, 3)
    tgt = aligned_copy(targets[0], np.float32)
    res = ebuf(T * 8, pattern, 4)
    st = ebuf(C.sizeof(_native.TrackState), pattern, 6)
    if blob is not None:
        _native.check(lib, lib.mgb_match_levels_profiled(P, LL, ptr(tgt), ptr(blob), ptr(ws), ptr(st), None))
    else:
        ref = aligned_copy(r, np.float32)
        _native.check(lib, lib.mgb_match_levels(P, LL, ptr(tgt), ptr(ref), ptr(ws), ptr(st), None))
    _native.check(lib, lib.mgb_match_frequencies(P, LL, ptr(tgt), ptr(res), None, ptr(ws), ptr(st), None))
    _native.check(lib, lib.mgb_correct_levels(P, LL, ptr(ws), ptr(st), None))
    V = len(targets) - 1
    keep, results = [], [res]
    if V:
        table = (_native.VersionTrack * V)()
        for k, x in enumerate(targets[1:]):
            VL = profiled_layout(lib, ep, T)
            vws, vt = ebuf(VL.workspace_bytes, pattern, 10 + k), aligned_copy(x, np.float32)
            vres, vst = ebuf(T * 8, pattern, 20 + k), ebuf(C.sizeof(_native.TrackState), pattern, 30 + k)
            table[k].layout = C.pointer(VL)
            table[k].d_target_lr, table[k].d_result_lr = vt.ctypes.data, vres.ctypes.data
            table[k].d_workspace, table[k].d_state = vws.ctypes.data, vst.ctypes.data
            keep.append((VL, vws, vt, vst))
            results.append(vres)
        _native.check(lib, lib.mgb_version_match_frequencies(P, LL, ptr(ws), ptr(st), V, table, None))
    nb = int(lib.mgb_versions_workspace_bytes(P, LL))
    assert nb > 0
    vws = ebuf(nb, pattern, 40)
    outs = [[ebuf(T * 8, pattern, 50 + 3 * k + j).view(np.float32).reshape(T, 2) if need[j] else None for j in range(3)]
            for k in range(V + 1)]
    entries = (_native.VersionEntry * (V + 1))()
    for e, rr, o in zip(entries, results, outs):
        e.d_result_lr = rr.ctypes.data
        e.d_out_limited, e.d_out_no_limiter, e.d_out_normalized = (x.ctypes.data if x is not None else None for x in o)
    report = None
    if lufs is None:
        _native.check(lib, lib.mgb_finalize_versions(P, LL, V + 1, entries, ptr(ws), ptr(st), ptr(vws), nb, None))
    else:
        for e in entries:
            e.d_out_no_limiter = e.d_out_normalized = None
        meter = emul_params(cfg.internal_sample_rate)
        sb = int(lib.mgb_loudness_target_workspace_bytes(C.byref(meter), T))
        search, rep = ebuf(sb, pattern, 41), ebuf(C.sizeof(_native.LoudnessTargetReport), pattern, 42)
        _native.check(lib, lib.mgb_finalize_versions_to_loudness(P, LL, C.byref(meter), C.byref(target_of(lufs)), V + 1,
                                                                 entries, ptr(ws), ptr(st), ptr(vws), nb, ptr(search), sb,
                                                                 ptr(rep), None))
        report = _native.LoudnessTargetReport.from_buffer_copy(bytes(rep))
    return [tuple(None if o is None else np.array(o) for o in entry) for entry in outs], bytes(st), report


def run_single(cfg, x, r=None, blob=None, lufs=None):
    """The single job on the same buffers' driver: run_versions without versions, through mgb_finalize (and
    mgb_finalize_to_loudness) -> ((limited, plain, normalized), state bytes, report or None)"""
    lib, ep = emul_lib(), get_emul_plan(cfg)
    P = C.byref(ep.struct)
    T = len(x)
    if blob is not None:
        L = profiled_layout(lib, ep, T)
    else:
        L = _native.TrackLayout()
        _native.check(lib, lib.mgb_track_layout_init(P, T, len(r), C.byref(L)))
    LL = C.byref(L)
    ws, tgt, res = ebuf(L.workspace_bytes, None, 3), aligned_copy(x, np.float32), ebuf(T * 8, None, 4)
    st = ebuf(C.sizeof(_native.TrackState), None, 6)
    if blob is not None:
        _native.check(lib, lib.mgb_match_levels_profiled(P, LL, ptr(tgt), ptr(blob), ptr(ws), ptr(st), None))
    else:
        _native.check(lib, lib.mgb_match_levels(P, LL, ptr(tgt), ptr(aligned_copy(r, np.float32)), ptr(ws), ptr(st), None))
    _native.check(lib, lib.mgb_match_frequencies(P, LL, ptr(tgt), ptr(res), None, ptr(ws), ptr(st), None))
    _native.check(lib, lib.mgb_correct_levels(P, LL, ptr(ws), ptr(st), None))
    outs = [ebuf(T * 8, None, 8 + k).view(np.float32).reshape(T, 2) for k in range(3)]
    report = None
    if lufs is None:
        _native.check(lib, lib.mgb_finalize(P, LL, ptr(res), *(ptr(o) for o in outs), ptr(ws), ptr(st), None))
    else:
        meter = emul_params(cfg.internal_sample_rate)
        sb = int(lib.mgb_loudness_target_workspace_bytes(C.byref(meter), T))
        search, rep = ebuf(sb, None, 41), ebuf(C.sizeof(_native.LoudnessTargetReport), None, 42)
        _native.check(lib, lib.mgb_finalize_to_loudness(P, LL, C.byref(meter), C.byref(target_of(lufs)), ptr(res),
                                                        ptr(outs[0]), ptr(ws), ptr(search), sb, ptr(st), ptr(rep), None))
        report = _native.LoudnessTargetReport.from_buffer_copy(bytes(rep))
    return tuple(np.array(o) for o in outs), bytes(st), report


MODES = [dict(), dict(true_peak=True), dict(**WIDE)]


# ---- the main where no version is louder: the single job bit for bit -------------------------------------------------
@pytest.mark.parametrize("mode", MODES, ids=["sample", "true-peak", "wide"])
@pytest.mark.parametrize("profiled", [False, True], ids=["paired", "profiled"])
def test_quieter_versions_leave_the_main_bit_identical(mode, profiled):
    cfg = cfg_of(**mode)
    a, b = parts()
    x, r = a + b, reference()
    blob = emul_profile(cfg, r)[0] if profiled else None
    quieter = [0.5 * x, 0.7 * x, np.zeros_like(x)]
    got, st, _ = run_versions(cfg, [x] + quieter, r, blob)
    want, st_w, _ = run_single(cfg, x, r, blob)
    for g, w in zip(got[0], want):
        assert np.array_equal(g, w)
    if not cfg.true_peak:  # (mgb_finalize in true-peak mode writes the true peak's coefficients into the state)
        assert st == st_w  # mgb_finalize_versions leaves the main's state as mgb_correct_levels left it


@pytest.mark.parametrize("tp", [False, True], ids=["sample", "true-peak"])
def test_quieter_versions_leave_the_main_at_a_loudness_target_bit_identical(tp):
    cfg = cfg_of(true_peak=tp)
    a, b = parts()
    x, r = a + b, reference()
    got, _, rep = run_versions(cfg, [x, 0.5 * x, np.zeros_like(x)], r, lufs=-14.0, need=(True, False, False))
    want, _, rep_w = run_single(cfg, x, r, lufs=-14.0)
    assert np.array_equal(got[0][0], want[0])
    assert bytes(rep) == bytes(rep_w)
    # the linked pass at the search's drive: half the main, exactly, and silence
    assert np.array_equal(got[1][0], 0.5 * got[0][0])
    assert not got[2][0].any()


@pytest.mark.parametrize("tp", [False, True], ids=["sample", "true-peak"])
def test_equal_half_and_silent_versions_are_exact(tp):
    cfg = cfg_of(true_peak=tp)
    a, b = parts()
    x = a + b
    got, _, _ = run_versions(cfg, [x, x, 0.5 * x, np.zeros_like(x)], reference())
    for j in range(3):
        assert np.array_equal(got[1][j], got[0][j])
        assert np.array_equal(got[2][j], 0.5 * got[0][j])
        assert not got[3][j].any()


# ---- versions of a + b against the restatement -----------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES, ids=["sample", "true-peak", "wide"])
def test_three_versions_match_the_restatement(mode):
    cfg = cfg_of(**mode)
    a, b = parts(seed=1)
    targets = [a + b, a, b, a + 0.5 * b]
    r = reference()
    got, _, _ = run_versions(cfg, targets, r)
    tr = {}
    want = versions_oracle.main_versions(targets, r, cfg, True, True, True, trace=tr)
    for k, (g, w) in enumerate(zip(got, want)):
        for j in range(3):
            assert float(np.abs(g[j] - w[j]).max()) < TOL, (k, j)
    # the null: main - instrumental is the vocal through the chain, under the same gain
    e = versions_oracle.envelope(tr["D"], cfg)
    vocal = versions_oracle.chain(b, tr) * e[:, None] * tr["final_coef"]
    assert float(np.abs((got[0][0].astype(np.float64) - got[1][0]) - vocal).max()) < TOL


@pytest.mark.parametrize("tp", [False, True], ids=["sample", "true-peak"])
def test_a_version_louder_than_the_main_is_held_at_the_threshold(tp):
    cfg = cfg_of(true_peak=tp)
    a, b = parts(seed=2)
    x = a + b
    loud = x.copy()
    c = len(x) // 2
    loud[c:c + 2000] *= 2.0  # a transient 6 dB above the main
    r = reference()
    got, _, _ = run_versions(cfg, [x, loud], r)
    tr = {}
    want = versions_oracle.main_versions([x, loud], r, cfg, True, True, True, trace=tr)
    thr = port.config_from(cfg).threshold * tr["final_coef"]
    for k in range(2):
        assert float(np.abs(got[k][0] - want[k][0]).max()) < TOL
        if tp:
            peak = float(versions_oracle.detector(got[k][0].astype(np.float64), cfg, True).max())
            assert 20 * np.log10(peak / thr) <= 0.2
        else:
            assert float(np.abs(got[k][0]).max()) <= thr * (1 + 1e-6)
    # the main is limited a little harder than alone: the loud version's gain is everybody's
    alone, _, _ = run_single(cfg, x, r)
    assert float(np.abs(got[0][0]).max()) <= float(np.abs(alone[0]).max())


@pytest.mark.parametrize("tp", [False, True], ids=["sample", "true-peak"])
def test_loudness_target_with_versions_matches_the_restatement(tp):
    cfg = cfg_of(true_peak=tp)
    a, b = parts(seed=3)
    targets = [a + b, a, a + 0.5 * b]
    r = reference()
    got, _, rep = run_versions(cfg, targets, r, lufs=-14.0, need=(True, False, False))
    tr = {}
    want = versions_oracle.main_versions(targets, r, cfg, True, False, False, loudness_target=-14.0, trace=tr)
    found = tr["search"]
    assert rep.passes == found["passes"] and rep.status == found["status"]
    assert abs(rep.gain_db - found["gain_db"]) <= 1e-4
    for k in range(len(targets)):
        assert float(np.abs(got[k][0] - want[k][0]).max()) < TOL, k
    assert abs(lto.integrated(got[0][0].astype(np.float64), 44100) - -14.0) <= lto.TOLERANCE


def test_poisoned_workspaces_change_nothing():
    cfg = cfg_of()
    a, b = parts(seed=4)
    targets = [a + b, a, b]
    r = reference()
    clean, st, _ = run_versions(cfg, targets, r)
    dirty, st_d, _ = run_versions(cfg, targets, r, pattern=0xFF)
    assert st == st_d
    for g, w in zip(dirty, clean):
        for j in range(3):
            assert np.array_equal(g[j], w[j])


# ---- argument errors and refusals ------------------------------------------------------------------------------------
def test_argument_errors():
    cfg = cfg_of()
    lib, ep = emul_lib(), get_emul_plan(cfg)
    P = C.byref(ep.struct)
    T = 20000
    L = profiled_layout(lib, ep, T)
    LL = C.byref(L)
    ws, st = ebuf(L.workspace_bytes, None, 1), ebuf(C.sizeof(_native.TrackState), None, 2)
    VL = profiled_layout(lib, ep, T)
    vws, vst, vt, vres = (ebuf(VL.workspace_bytes, None, 3), ebuf(C.sizeof(_native.TrackState), None, 4),
                          ebuf(T * 8, None, 5), ebuf(T * 8, None, 6))
    table = (_native.VersionTrack * 9)()
    for e in table:
        e.layout = C.pointer(VL)
        e.d_target_lr, e.d_result_lr, e.d_workspace, e.d_state = vt.ctypes.data, vres.ctypes.data, vws.ctypes.data, vst.ctypes.data
    match = lambda n, t=table: lib.mgb_version_match_frequencies(P, LL, ptr(ws), ptr(st), n, t, None)
    assert match(0) == _native.MGB_ERR_INVALID
    assert match(9) == _native.MGB_ERR_INVALID
    one = (_native.VersionTrack * 1)(table[0])
    other = profiled_layout(lib, ep, T + 1)
    one[0].layout = C.pointer(other)
    assert match(1, one) == _native.MGB_ERR_INVALID  # another frame count
    paired = _native.TrackLayout()
    _native.check(lib, lib.mgb_track_layout_init(P, T, 30000, C.byref(paired)))
    one[0].layout = C.pointer(paired)
    assert match(1, one) == _native.MGB_ERR_INVALID  # not a profiled layout of this plan
    one[0].layout = C.pointer(VL)
    one[0].d_result_lr = vt.ctypes.data
    assert match(1, one) == _native.MGB_ERR_INVALID  # the result is the target
    one[0].d_result_lr = vres.ctypes.data + 4
    assert match(1, one) == _native.MGB_ERR_INVALID  # misaligned
    one[0].d_result_lr = None
    assert match(1, one) == _native.MGB_ERR_INVALID

    nb = int(lib.mgb_versions_workspace_bytes(P, LL))
    assert nb > 0
    vw = ebuf(nb, None, 7)
    res, out, out2 = ebuf(T * 8, None, 8), ebuf(T * 8, None, 9), ebuf(T * 8, None, 10)
    entries = (_native.VersionEntry * 10)()
    for e in entries:
        e.d_result_lr = res.ctypes.data
    fin = lambda n, nbytes=nb: lib.mgb_finalize_versions(P, LL, n, entries, ptr(ws), ptr(st), ptr(vw), nbytes, None)
    assert fin(0) == _native.MGB_ERR_INVALID
    assert fin(10) == _native.MGB_ERR_INVALID
    entries[0].d_out_limited = res.ctypes.data
    assert fin(1) == _native.MGB_ERR_INVALID  # an output that is a result
    entries[0].d_out_limited = out.ctypes.data
    entries[1].d_out_normalized = out.ctypes.data
    assert fin(2) == _native.MGB_ERR_INVALID  # two outputs in one buffer
    entries[1].d_out_normalized = out2.ctypes.data + 8
    assert fin(2) == _native.MGB_ERR_INVALID  # misaligned
    entries[1].d_out_normalized = None
    assert fin(2, nb - 1) == _native.MGB_ERR_WORKSPACE
    meter = emul_params(44100)
    sb = int(lib.mgb_loudness_target_workspace_bytes(C.byref(meter), T))
    search, rep = ebuf(sb, None, 11), ebuf(C.sizeof(_native.LoudnessTargetReport), None, 12)
    loud = lambda n, ssb=sb: lib.mgb_finalize_versions_to_loudness(P, LL, C.byref(meter), C.byref(target_of(-14.0)), n, entries,
                                                                   ptr(ws), ptr(st), ptr(vw), nb, ptr(search), ssb, ptr(rep),
                                                                   None)
    assert loud(2) == _native.MGB_ERR_INVALID  # entry 1 has no limited output
    entries[1].d_out_limited = out2.ctypes.data
    entries[1].d_out_no_limiter = out.ctypes.data
    assert loud(2) == _native.MGB_ERR_INVALID  # only the limited outputs are written there
    entries[1].d_out_no_limiter = None
    assert loud(2, sb - 1) == _native.MGB_ERR_WORKSPACE


def test_refusals_before_any_device_work():
    cfg = mg.Config()
    x = np.zeros((50000, 2), np.float32)
    r = np.zeros((50000, 2), np.float32)
    with pytest.raises(ValueError, match="frames"):
        stages.main_versions_device([x, x[:-1]], r, cfg)
    with pytest.raises(ValueError, match="at most 8"):
        stages.main_versions_device([x] * 10, r, cfg)
    with pytest.raises(ValueError, match="stereo"):
        stages.main_versions_device([x, x[:, :1]], r, cfg)
    with pytest.raises(ValueError, match="main mix"):
        stages.main_versions_device([], r, cfg)


def test_process_versions_refuses_other_rates(tmp_path):
    from scipy.io import wavfile
    n = 50000
    paths = []
    for k, rate in enumerate((44100, 48000)):
        p = str(tmp_path / f"v{k}.wav")
        wavfile.write(p, rate, np.zeros((n, 2), np.int16))
        paths.append(p)
    res = [[mg.pcm24(str(tmp_path / f"o{k}.wav"))] for k in range(2)]
    with pytest.raises(ValueError, match="Hz"):
        mg.process_versions(paths, paths[0], res)
    with pytest.raises(ValueError, match="native rates"):
        mg.process_versions(paths, paths[0], res, mg.Config(native_rate=True))
    with pytest.raises(ValueError, match="at most 8"):
        mg.process_versions([paths[0]] * 10, paths[0], [res[0]] * 10)


# ---- thread orders and ThreadSanitizer -------------------------------------------------------------------------------
DUMP_ID = "tests/test_versions.py::test_dump_for_thread_orders_emulated"


def test_dump_for_thread_orders_emulated():
    """Two short versions at F = 512 in both peak modes, on the wide-window path and at -14 LUFS; with
    MGB_VERSIONS_DUMP set, every output (float32) goes to that file."""
    a, b = parts(n=44100 + 313, seed=5)
    raws = b""
    for mode, lufs in ((dict(), None), (dict(true_peak=True), None), (WIDE, None), (dict(true_peak=True), -14.0)):
        cfg = mg.Config(max_piece_size=0.25, fft_size=512, **({"true_peak": True} if mode.get("true_peak") else {}),
                        limiter=mg.LimiterConfig(**mode) if mode is WIDE else None)
        outs, st, _ = run_versions(cfg, [a + b, a, b], reference(), lufs=lufs,
                                   need=(True, False, False) if lufs else (True, True, True))
        raws += b"".join(o.tobytes() for entry in outs for o in entry if o is not None)
    if os.environ.get("MGB_VERSIONS_DUMP"):
        with open(os.environ["MGB_VERSIONS_DUMP"], "wb") as f:
            f.write(raws)


@pytest.fixture(scope="module")
def other_runs(tmp_path_factory):
    from concurrent.futures import ThreadPoolExecutor

    import build_emul
    from test_emul_racecheck import run_group, tsan_env
    build_emul.build(racecheck=True)
    build_emul.build()
    base = tmp_path_factory.mktemp("versions_racecheck")
    jobs = {}
    env = tsan_env(str(base / "tsan"))
    env["MGB_EMUL_BUILD"] = "racecheck"
    jobs["tsan"] = ([DUMP_ID], env, str(base / "tsan"))
    for order in ("forward", "reverse", "seeded"):
        env = dict(os.environ, MGB_EMUL_ORDER=order, MGB_EMUL_SEED="4242", MGB_VERSIONS_DUMP=str(base / f"dump_{order}.bin"))
        jobs[order] = ([DUMP_ID], env, str(base / order))
    with ThreadPoolExecutor(max_workers=4) as ex:
        futures = {key: ex.submit(run_group, *job) for key, job in jobs.items()}
        done = {key: f.result() + (jobs[key][2],) for key, f in futures.items()}
    return done, base


def test_versions_kernels_have_no_data_races(other_runs):
    from test_emul_racecheck import reports
    rc, out, _, log_dir = other_runs[0]["tsan"]
    n, first = reports(log_dir)
    assert n == 0, f"{n} ThreadSanitizer report(s); the first:\n{first}"
    assert rc == 0, out


@pytest.mark.parametrize("order", ["reverse", "seeded"])
def test_versions_in_other_thread_orders(other_runs, order):
    """The linked detector's maxima are order-free: the reverse order gives the same bytes.  A seeded order (a different
    order in every launch) adds stage 3's per-piece float64 atomic sums in another order, as the device does, so there
    the outputs keep the bound two device runs of one job keep."""
    done, base = other_runs
    for o in ("forward", order):
        rc, out, _, _ = done[o]
        assert rc == 0, out
    forward = (base / "dump_forward.bin").read_bytes()
    other = (base / f"dump_{order}.bin").read_bytes()
    assert len(forward) > 0 and len(other) == len(forward)
    if order == "reverse":
        assert other == forward
    else:
        a, b = np.frombuffer(forward, np.float32), np.frombuffer(other, np.float32)
        assert float(np.abs(a.astype(np.float64) - b).max()) <= 1e-6
