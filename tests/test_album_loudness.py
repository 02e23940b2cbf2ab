"""Album loudness on the CPU: the float64 restatement (tests/album_loudness_oracle.py) on its own, mgb_album_loudness and
mgb_album_finalize_to_loudness on the emulator against it and against the single-track entries, poisoned workspaces,
argument errors and Python refusals, and the new kernel under ThreadSanitizer and in other thread orders."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from emul_harness import aligned, aligned_copy, emul_lib, get_emul_plan, ptr  # (puts oracle/ on sys.path)
import album_loudness_oracle as alo
import loudness
import loudness_target_oracle as lto
import port
import matchering_b200 as mg
from matchering_b200 import _native, stages
from test_loudness import LOUD_TOL, TP_TOL_DB, emul_meter, emul_params, poison
from test_loudness_target import assert_report_matches, target_of
from test_reference_profile import ebuf, emul_profile, profiled_layout

FS = 44100
TOL = 1e-5  # the limiter's parity bound
RESULT = C.sizeof(_native.LoudnessResult)


def _noise(n, seed, gain_db=0.0):
    return (port.synth_target(n, seed).astype(np.float64) * 0.4 * 10 ** (gain_db / 20)).astype(np.float32)


# ---- the restatement --------------------------------------------------------------------------------------------------
def test_oracle_one_track_album_is_the_meter():
    y = _noise(3 * FS + 77, 1).astype(np.float64)
    got, want = alo.measure_album([y], FS), loudness.measure(y, FS)
    for k in ("integrated", "loudness_range", "momentary_max", "short_term_max", "momentary_count", "short_term_count"):
        assert got[k] == want[k], k
    assert np.array_equal(got["sample_peak"], want["sample_peak"]) and np.array_equal(got["true_peak"], want["true_peak"])


def test_oracle_two_identical_tracks_read_the_track():
    y = _noise(4 * FS + 5, 2).astype(np.float64)
    got, want = alo.measure_album([y, y], FS), loudness.measure(y, FS)
    assert abs(got["integrated"] - want["integrated"]) <= 1e-12
    assert got["momentary_count"] == 2 * want["momentary_count"]


def test_oracle_one_track_search_is_the_search():
    cfg = mg.Config()
    s = (_noise(3 * FS, 3) * 1.5).astype(np.float64)
    for target in (-20.0, -12.0, -6.0):
        a, b = alo.search_album([s], cfg, target), lto.search(s, cfg, target)
        assert a["trace"] == b["trace"] and a["status"] == b["status"] and a["passes"] == b["passes"]
        assert np.array_equal(a["outputs"][0], b["output"])


def test_oracle_album_gain_keeps_offsets_per_track_search_levels_them():
    """At a quiet target no limiter engages: every track is s_t times one gain, so the tracks keep their offsets,
    where a search per track brings each to the target."""
    cfg = mg.Config()
    ss = [(_noise(3 * FS + 11 * k, 4 + k, g)).astype(np.float64) for k, g in enumerate((0.0, -6.0, -12.0))]
    r = alo.search_album(ss, cfg, -40.0)
    assert r["status"] == lto.REACHED
    k = 10 ** (r["gain_db"] / 20)
    for s, y in zip(ss, r["outputs"]):
        assert float(np.abs(y - s * k).max()) <= 1e-12
    levels = [lto.integrated(y, FS) for y in r["outputs"]]
    inputs = [lto.integrated(s, FS) for s in ss]
    for a, b in zip(levels, inputs):
        assert abs((a - levels[0]) - (b - inputs[0])) <= 1e-9
    singles = [lto.search(s, cfg, -40.0)["integrated"] for s in ss]
    assert max(singles) - min(singles) <= 2 * lto.TOLERANCE
    assert levels[0] - levels[2] > 11.0


# ---- mgb_album_loudness on the emulator -------------------------------------------------------------------------------
def emul_album_meter(xs, fs, per_track=True, pattern=None):
    """mgb_album_loudness on the emulator -> (album result bytes, [track result bytes] or None)."""
    lib = emul_lib()
    p = emul_params(fs)
    n = len(xs)
    arrs = [aligned_copy(x, np.float32) for x in xs]
    frames = (C.c_int64 * n)(*(len(x) for x in xs))
    ptrs = (C.c_void_p * n)(*(a.ctypes.data for a in arrs))
    nb = int(lib.mgb_album_loudness_workspace_bytes(C.byref(p), n, frames))
    assert nb > 0
    ws = aligned((nb,), np.uint8)
    ws[...] = poison(nb, pattern, 3)
    out = aligned(((n + 1) * RESULT,), np.uint8)
    out[...] = poison(len(out), pattern, 4)
    _native.check(lib, lib.mgb_album_loudness(C.byref(p), n, ptrs, frames, ptr(ws), nb, ptr(out),
                                              out.ctypes.data + RESULT if per_track else None, None))
    raw = bytes(out)
    return raw[:RESULT], ([raw[(k + 1) * RESULT:(k + 2) * RESULT] for k in range(n)] if per_track else None)


def test_one_track_album_meter_is_mgb_loudness_emulated():
    x = _noise(3 * FS + 333, 5)
    album, tracks = emul_album_meter([x], FS)
    want = emul_meter(x, FS)
    assert album == want and tracks[0] == want
    assert emul_album_meter([x], FS, per_track=False)[0] == want


def _unequal():
    """one track with a few 3 s windows, one shorter than a 3 s window, one shorter than a 400 ms window"""
    return [_noise(3 * FS + 6123, 6), _noise(FS + 4545, 7, -9.0), _noise(12000, 8, 3.0)]


def test_album_meter_matches_the_restatement_emulated():
    xs = _unequal()
    album, tracks = emul_album_meter(xs, FS)
    for raw, x in zip(tracks, xs):
        assert raw == emul_meter(x, FS)  # each track's own meter, bit for bit
    assert emul_album_meter(xs, FS, per_track=False)[0] == album  # (with and without the per-track finishes)
    got = _native.LoudnessResult.from_buffer_copy(album)
    want = alo.measure_album([x.astype(np.float64) for x in xs], FS)
    for k in ("integrated", "loudness_range", "momentary_max", "short_term_max"):
        assert abs(getattr(got, k) - want[k]) <= LOUD_TOL, (k, getattr(got, k), want[k])
    assert (got.momentary_count, got.short_term_count) == (want["momentary_count"], want["short_term_count"])
    assert list(got.sample_peak) == list(want["sample_peak"])
    for g, w in zip(got.true_peak, want["true_peak"]):
        assert abs(20.0 * math.log10(g / w)) <= TP_TOL_DB, (g, w)
    # the pooled windows differ from both the concatenation and the mean of the tracks' values
    concat = loudness.measure(np.concatenate([x.astype(np.float64) for x in xs]), FS)
    assert got.momentary_count < concat["momentary_count"]


def test_silent_album_reads_minus_infinity_emulated():
    xs = [np.zeros((FS, 2), np.float32), np.zeros((2 * FS, 2), np.float32)]
    got = _native.LoudnessResult.from_buffer_copy(emul_album_meter(xs, FS)[0])
    assert got.integrated == -math.inf and got.loudness_range == 0.0


def test_album_meter_poisoned_workspace_emulated():
    xs = _unequal()
    clean = emul_album_meter(xs, FS)
    for pattern in ("ff", "random"):
        assert emul_album_meter(xs, FS, pattern=pattern) == clean


# ---- mgb_album_finalize_to_loudness on the emulator -------------------------------------------------------------------
def _ref():
    return port.synth_reference(FS + 77, 52)


_PROFILES = {}


def profile_of(cfg):
    """emul_profile of _ref() for cfg, made once per Config"""
    key = (cfg.fft_size, cfg.max_piece_size, cfg.true_peak)
    if key not in _PROFILES:
        _PROFILES[key] = emul_profile(cfg, _ref())[0]
    return _PROFILES[key]


def run_album_target(cfg, targets, blob, target, max_gain_db=lto.MAX_GAIN_DB, pattern=None, search_pattern=None):
    """mgb_album_match, then mgb_album_finalize_to_loudness -> (limited outputs, report, s_t per track as float64)."""
    lib, ep = emul_lib(), get_emul_plan(cfg)
    P = C.byref(ep.struct)
    n = len(targets)
    layouts = [profiled_layout(lib, ep, len(t)) for t in targets]
    table = (_native.AlbumTrack * n)()
    keep = []
    for k, (t, L) in enumerate(zip(targets, layouts)):
        ws = ebuf(L.workspace_bytes, pattern, 10 + k)
        tgt = aligned_copy(t, np.float32)
        res = ebuf(len(t) * 8, pattern, 20 + k)
        st = ebuf(C.sizeof(_native.TrackState), pattern, 30 + k)
        table[k].layout = C.pointer(L)
        table[k].d_target_lr, table[k].d_result_lr = tgt.ctypes.data, res.ctypes.data
        table[k].d_workspace, table[k].d_state = ws.ctypes.data, st.ctypes.data
        keep.append((L, ws, tgt, res, st))
    arr = (_native.TrackLayout * n)(*layouts)
    nb = int(lib.mgb_album_workspace_bytes(P, n, arr))
    aws = ebuf(nb, pattern, 40)
    _native.check(lib, lib.mgb_album_match(P, n, table, ptr(blob), None, ptr(aws), nb, None))
    meter = emul_params(cfg.internal_sample_rate)
    sb = int(lib.mgb_album_loudness_target_workspace_bytes(C.byref(meter), n, arr))
    assert sb > 0
    search = ebuf(sb, search_pattern if search_pattern is not None else pattern, 41)
    outs = [ebuf(len(t) * 8, pattern, 50 + k).view(np.float32).reshape(len(t), 2) for k, t in enumerate(targets)]
    optrs = (C.c_void_p * n)(*(o.ctypes.data for o in outs))
    rep = ebuf(C.sizeof(_native.LoudnessTargetReport), pattern, 60)
    _native.check(lib, lib.mgb_album_finalize_to_loudness(P, n, table, optrs, C.byref(meter),
                                                          C.byref(target_of(target, max_gain_db)), ptr(search), sb,
                                                          ptr(rep), None))
    ss = []
    for L, ws, tgt, res, st in keep:
        gain = _native.TrackState.from_buffer_copy(bytes(st)).gain
        ss.append(res.view(np.float32).reshape(-1, 2).astype(np.float64) * gain)
    return [np.array(o) for o in outs], _native.LoudnessTargetReport.from_buffer_copy(bytes(rep)), ss


def run_profiled_target(cfg, t, blob, target):
    """The profiled single job's stages 1-3, then mgb_finalize_to_loudness -> (limited, report)."""
    lib, ep = emul_lib(), get_emul_plan(cfg)
    L = profiled_layout(lib, ep, len(t))
    P, LL = C.byref(ep.struct), C.byref(L)
    ws = aligned((L.workspace_bytes,), np.uint8)
    tgt, res = aligned_copy(t, np.float32), aligned((len(t), 2), np.float32)
    st = _native.TrackState()
    _native.check(lib, lib.mgb_match_levels_profiled(P, LL, ptr(tgt), ptr(blob), ptr(ws), C.byref(st), None))
    _native.check(lib, lib.mgb_match_frequencies(P, LL, ptr(tgt), ptr(res), None, ptr(ws), C.byref(st), None))
    _native.check(lib, lib.mgb_correct_levels(P, LL, ptr(ws), C.byref(st), None))
    meter = emul_params(cfg.internal_sample_rate)
    nbytes = int(lib.mgb_loudness_target_workspace_bytes(C.byref(meter), len(t)))
    search = aligned((nbytes,), np.uint8)
    out = aligned((len(t), 2), np.float32)
    rep = aligned((C.sizeof(_native.LoudnessTargetReport),), np.uint8)
    _native.check(lib, lib.mgb_finalize_to_loudness(P, LL, C.byref(meter), C.byref(target_of(target)), ptr(res), ptr(out),
                                                    ptr(ws), ptr(search), nbytes, C.byref(st), ptr(rep), None))
    return np.array(out), _native.LoudnessTargetReport.from_buffer_copy(bytes(rep))


CFG = dict(max_piece_size=0.25, fft_size=512)


@pytest.mark.parametrize("tp", [False, True])
def test_one_track_album_target_is_the_profiled_job_emulated(tp):
    cfg = mg.Config(**CFG, true_peak=tp)
    x = port.synth_target(FS + 311, 61)
    blob = profile_of(cfg)
    outs, rep, _ = run_album_target(cfg, [x], blob, -12.0)
    want, want_rep = run_profiled_target(cfg, x, blob, -12.0)
    assert rep.status == lto.REACHED
    assert outs[0].tobytes() == want.tobytes()
    assert bytes(rep) == bytes(want_rep)


def _three():
    return [_noise(30313, 71, 0.0), _noise(40007, 72, -6.0), _noise(25000, 73, -12.0)]


@pytest.mark.parametrize("tp", [False, True])
def test_three_tracks_match_the_restatement_emulated(tp):
    cfg = mg.Config(**CFG, true_peak=tp)
    blob = profile_of(cfg)
    outs, rep, ss = run_album_target(cfg, _three(), blob, -11.0)
    want = alo.search_album(ss, cfg, -11.0)
    assert_report_matches(rep, want)
    assert rep.status == lto.REACHED
    for k, (o, s) in enumerate(zip(outs, ss)):
        err = float(np.abs(o - lto.limited(s, rep.gain_db, cfg)).max())
        assert err < TOL, (k, err)
    assert abs(alo.integrated_album([o.astype(np.float64) for o in outs], FS) - -11.0) <= lto.TOLERANCE
    # the album meter of the outputs is the search's last measurement, to the bit
    album, _ = emul_album_meter(outs, FS, per_track=False)
    assert _native.LoudnessResult.from_buffer_copy(album).integrated == rep.integrated


def test_quiet_target_keeps_the_offsets_emulated():
    cfg = mg.Config(**CFG)
    blob = profile_of(cfg)
    xs = _three()
    outs, rep, ss = run_album_target(cfg, xs, blob, -35.0)
    assert rep.status == lto.REACHED
    k = 10 ** (rep.gain_db / 20)
    for o, s in zip(outs, ss):  # no limiter engages: every track is s_t times the one drive
        assert float(np.abs(o - s * k).max()) <= 1e-6


def test_silent_album_is_undefined_after_one_pass_emulated():
    cfg = mg.Config(**CFG)
    blob = profile_of(cfg)
    xs = [np.zeros((20999, 2), np.float32), np.zeros((30000, 2), np.float32)]
    outs, rep, ss = run_album_target(cfg, xs, blob, -14.0)
    assert rep.status == lto.UNDEFINED and rep.passes == 1 and rep.gain_db == 0.0
    assert math.isinf(rep.input_integrated) and rep.input_integrated < 0
    for o, s in zip(outs, ss):
        assert float(np.abs(o - lto.limited(s, 0.0, cfg)).max()) < TOL


def test_short_tracks_are_undefined_emulated():
    """Tracks shorter than one 400 ms window add no window: the album is undefined and keeps the outputs of x = 0."""
    cfg = mg.Config(**CFG)
    blob = profile_of(cfg)
    xs = [_noise(12000, 81), _noise(15000, 82, -3.0)]
    outs, rep, ss = run_album_target(cfg, xs, blob, -14.0)
    assert rep.status == lto.UNDEFINED and rep.passes == 1 and rep.gain_db == 0.0
    for o, s in zip(outs, ss):
        assert float(np.abs(o - lto.limited(s, 0.0, cfg)).max()) < TOL


def test_unreachable_target_ends_at_the_largest_drive_emulated():
    cfg = mg.Config(**CFG)
    blob = profile_of(cfg)
    outs, rep, ss = run_album_target(cfg, _three(), blob, -1.0, max_gain_db=6.0)
    assert rep.status == lto.UNREACHABLE and rep.gain_db == 6.0
    assert_report_matches(rep, alo.search_album(ss, cfg, -1.0, 6.0))


def test_track_order_does_not_move_the_drive_emulated():
    cfg = mg.Config(**CFG)
    blob = profile_of(cfg)
    xs = _three()
    a, ra, _ = run_album_target(cfg, xs, blob, -12.0)
    b, rb, _ = run_album_target(cfg, xs[::-1], blob, -12.0)
    assert ra.status == rb.status == lto.REACHED
    assert abs(ra.gain_db - rb.gain_db) <= 1e-6
    for x, y in zip(a, b[::-1]):
        assert float(np.abs(x - y).max()) < TOL


def test_poisoned_workspaces_give_the_same_bytes_emulated():
    cfg = mg.Config(**CFG, true_peak=True)
    blob = profile_of(cfg)
    xs = _three()
    clean, rc, _ = run_album_target(cfg, xs, blob, -12.0, pattern=None, search_pattern=0)
    for pattern in ("ff", "random"):
        got, rg, _ = run_album_target(cfg, xs, blob, -12.0, pattern=pattern)
        assert bytes(rg) == bytes(rc), pattern
        for a, b in zip(got, clean):
            assert a.tobytes() == b.tobytes(), pattern


# ---- argument errors ---------------------------------------------------------------------------------------------------
def test_meter_argument_errors_emulated():
    lib = emul_lib()
    p = emul_params(FS)
    x = aligned_copy(_noise(20000, 9), np.float32)
    frames = (C.c_int64 * 2)(20000, 20000)
    ptrs = (C.c_void_p * 2)(x.ctypes.data, x.ctypes.data)
    nb = int(lib.mgb_album_loudness_workspace_bytes(C.byref(p), 2, frames))
    ws, out = aligned((nb,), np.uint8), aligned((3 * RESULT,), np.uint8)

    def call(n=2, fr=frames, pp=ptrs, size=nb, w=ptr(ws), o=ptr(out)):
        return lib.mgb_album_loudness(C.byref(p), n, pp, fr, w, size, o, None, None)
    assert call() == _native.MGB_OK
    assert call(n=0) == _native.MGB_ERR_INVALID
    assert call(n=_native.MGB_MAX_ALBUM_TRACKS + 1) == _native.MGB_ERR_INVALID
    assert call(pp=None) == _native.MGB_ERR_INVALID
    assert call(pp=(C.c_void_p * 2)(x.ctypes.data, x.ctypes.data + 4)) == _native.MGB_ERR_INVALID
    assert call(fr=(C.c_int64 * 2)(20000, 0)) == _native.MGB_ERR_INVALID
    assert call(size=nb - 1) == _native.MGB_ERR_WORKSPACE
    assert call(w=None) == _native.MGB_ERR_INVALID
    assert call(o=out.ctypes.data + 8) == _native.MGB_ERR_INVALID
    assert int(lib.mgb_album_loudness_workspace_bytes(C.byref(p), 0, frames)) == -1
    assert int(lib.mgb_album_loudness_workspace_bytes(C.byref(p), 2, None)) == -1


def test_target_argument_errors_emulated():
    cfg = mg.Config(**CFG)
    lib, ep = emul_lib(), get_emul_plan(cfg)
    P = C.byref(ep.struct)
    n = 30000
    L = profiled_layout(lib, ep, n)
    ws = ebuf(L.workspace_bytes, None)
    res, out = ebuf(n * 8, None), ebuf(n * 8, None)
    st = ebuf(C.sizeof(_native.TrackState), None)
    meter = emul_params(FS)
    arr = (_native.TrackLayout * 1)(L)
    sb = int(lib.mgb_album_loudness_target_workspace_bytes(C.byref(meter), 1, arr))
    search, rep = ebuf(sb, None), ebuf(C.sizeof(_native.LoudnessTargetReport), None)

    def call(k=1, edit=None, outp=out.ctypes.data, m=meter, target=-14.0, size=sb, plan=P, report=ptr(rep)):
        table = (_native.AlbumTrack * max(k, 1))()
        for e in table:
            e.layout = C.pointer(L)
            e.d_target_lr, e.d_result_lr, e.d_workspace, e.d_state = None, res.ctypes.data, ws.ctypes.data, st.ctypes.data
        if edit:
            edit(table[0])
        optrs = (C.c_void_p * max(k, 1))(*([outp] * max(k, 1)))
        return lib.mgb_album_finalize_to_loudness(plan, k, table, optrs, C.byref(m), C.byref(target_of(target)), ptr(search),
                                                  size, report, None)
    assert call() == _native.MGB_OK
    assert call(k=0) == _native.MGB_ERR_INVALID
    assert call(k=_native.MGB_MAX_ALBUM_TRACKS + 1) == _native.MGB_ERR_INVALID
    assert call(edit=lambda e: setattr(e, "d_workspace", ws.ctypes.data + 4)) == _native.MGB_ERR_INVALID
    assert call(edit=lambda e: setattr(e, "d_state", None)) == _native.MGB_ERR_INVALID
    assert call(outp=None) == _native.MGB_ERR_INVALID
    assert call(outp=res.ctypes.data) == _native.MGB_ERR_INVALID  # the output is the track's result
    assert call(m=emul_params(48000)) == _native.MGB_ERR_INVALID
    other = get_emul_plan(mg.Config(max_piece_size=0.25, fft_size=2048))
    foreign = profiled_layout(lib, other, n)
    assert call(edit=lambda e: setattr(e, "layout", C.pointer(foreign))) == _native.MGB_ERR_INVALID
    assert call(target=0.5) == _native.MGB_ERR_INVALID
    assert call(target=-80.0) == _native.MGB_ERR_INVALID
    assert call(size=sb - 1) == _native.MGB_ERR_WORKSPACE
    assert call(report=None) == _native.MGB_ERR_INVALID
    assert int(lib.mgb_album_loudness_target_workspace_bytes(C.byref(meter), 0, arr)) == -1
    assert int(lib.mgb_album_loudness_target_workspace_bytes(C.byref(meter), 1, None)) == -1


def test_python_refusals(tmp_path):
    x = np.zeros((50000, 2))
    for bad in (0.0, 3.0, -70.0, -80.0, float("nan"), float("inf"), True, "-14"):
        with pytest.raises(ValueError):
            stages.main_album([x], x, mg.Config(), album_loudness_target=bad)
        with pytest.raises(ValueError):
            mg.process_album(["a.wav"], "ref.wav", [[mg.pcm16("o.wav")]], album_loudness_target=bad)
    with pytest.raises(ValueError, match="album_loudness_target"):
        stages.main_album([x], x, mg.Config(loudness_target=-14))
    with pytest.raises(ValueError):
        mg.album_loudness([])
    with pytest.raises(ValueError):
        mg.album_loudness([x] * (_native.MGB_MAX_ALBUM_TRACKS + 1), 44100)
    with pytest.raises(ValueError):
        mg.album_loudness([x, np.zeros((5000, 1))], 44100)
    with pytest.raises(ValueError):
        mg.album_loudness([x])  # arrays need a rate
    import wave
    paths = []
    for rate in (44100, 48000):
        path = str(tmp_path / f"t{rate}.wav")
        with wave.open(path, "wb") as w:
            w.setnchannels(2), w.setsampwidth(2), w.setframerate(rate)
            w.writeframes(np.zeros(rate * 2, np.int16).tobytes())
        paths.append(path)
    with pytest.raises(ValueError):
        mg.album_loudness(paths)
    with pytest.raises(ValueError):
        mg.album_loudness([paths[0], x], 48000)


# ---- thread orders and ThreadSanitizer ---------------------------------------------------------------------------------
DUMP_ID = "tests/test_album_loudness.py::test_dump_for_thread_orders_emulated"


def test_dump_for_thread_orders_emulated():
    """The album meter of three unequal tracks and a three-track album target in both peak modes; with
    MGB_ALBUM_LOUDNESS_DUMP set, their results, reports and outputs go to that file."""
    album, tracks = emul_album_meter(_unequal(), FS)
    raws = album + b"".join(tracks)
    for tp in (False, True):
        cfg = mg.Config(**CFG, true_peak=tp)
        blob = profile_of(cfg)
        outs, rep, _ = run_album_target(cfg, _three(), blob, -11.0)
        raws += bytes(rep) + b"".join(o.tobytes() for o in outs)
    if os.environ.get("MGB_ALBUM_LOUDNESS_DUMP"):
        with open(os.environ["MGB_ALBUM_LOUDNESS_DUMP"], "wb") as f:
            f.write(raws)


@pytest.fixture(scope="module")
def other_runs(tmp_path_factory):
    from concurrent.futures import ThreadPoolExecutor

    import build_emul
    from test_emul_racecheck import run_group, tsan_env
    build_emul.build(racecheck=True)
    build_emul.build()
    base = tmp_path_factory.mktemp("album_loudness_racecheck")
    jobs = {}
    env = tsan_env(str(base / "tsan"))
    env["MGB_EMUL_BUILD"] = "racecheck"
    jobs["tsan"] = ([DUMP_ID], env, str(base / "tsan"))
    for order in ("forward", "reverse", "seeded"):
        env = dict(os.environ, MGB_EMUL_ORDER=order, MGB_EMUL_SEED="4242",
                   MGB_ALBUM_LOUDNESS_DUMP=str(base / f"dump_{order}.bin"))
        jobs[order] = ([DUMP_ID], env, str(base / order))
    with ThreadPoolExecutor(max_workers=4) as ex:
        futures = {key: ex.submit(run_group, *job) for key, job in jobs.items()}
        done = {key: f.result() + (jobs[key][2],) for key, f in futures.items()}
    return done, base


def test_album_loudness_has_no_data_races(other_runs):
    from test_emul_racecheck import reports
    rc, out, _, log_dir = other_runs[0]["tsan"]
    n, first = reports(log_dir)
    assert n == 0, f"{n} ThreadSanitizer report(s); the first:\n{first}"
    assert rc == 0, out


@pytest.mark.parametrize("order", ["reverse", "seeded"])
def test_album_loudness_is_bit_identical_in_other_thread_orders(other_runs, order):
    done, base = other_runs
    for o in ("forward", order):
        rc, out, _, _ = done[o]
        assert rc == 0, out
    forward = (base / "dump_forward.bin").read_bytes()
    assert len(forward) > 0
    assert (base / f"dump_{order}.bin").read_bytes() == forward
