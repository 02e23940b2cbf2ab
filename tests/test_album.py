"""Album mastering (mgb_album_match, stages.main_album, mg.process_album) on the CPU: the float64 restatement against
oracle/port.py, the emulator build against the restatement and against the profiled single job, argument errors and
refusals, and the new kernels under ThreadSanitizer and in other thread orders."""
import ctypes as C
import os

import numpy as np
import pytest

import album_oracle
import port
from emul_harness import aligned_copy, emul_lib, get_emul_plan, ptr
from matchering_b200 import _native
from test_reference_profile import assert_identical, ebuf, emul_profile, profiled_layout, run_profiled

import matchering_b200 as mg
from matchering_b200 import stages


# ---- the restatement -------------------------------------------------------------------------------------------------
def _pair(n=44100 * 3 + 17):
    return port.synth_target(n, 3), port.synth_reference(44100 * 2 + 99, 4)


def test_oracle_one_track_is_port_main():
    cfg = mg.Config(max_piece_size=0.5)
    x, r = _pair()
    got = album_oracle.main_album([x], r, cfg, True, True, True)[0]
    want = port.main(x.astype(np.float64), r.astype(np.float64), cfg, True, True, True)
    for a, b in zip(got, want):
        assert float(np.abs(a - b).max()) <= 1e-12


def test_oracle_doubled_album_is_the_single_job():
    cfg = mg.Config(max_piece_size=0.5)
    x, r = _pair()
    ta, tw = {}, {}
    album_oracle.main_album([x, x], r, cfg, trace=ta)
    port.main(x.astype(np.float64), r.astype(np.float64), cfg, trace=tw)
    assert abs(ta["c0"] - tw["c0"]) <= 1e-12 * tw["c0"]
    for name in ("mid", "side"):
        assert float(np.abs(ta["firs"][name] - tw["firs"][name]).max()) <= 1e-12


def test_oracle_album_keeps_level_relation_independent_jobs_do_not():
    cfg = mg.Config(max_piece_size=0.5)
    x, r = _pair()
    outs = album_oracle.main_album([x, 0.5 * x], r, cfg, False, True, False)
    p1, p2 = outs[0][1], outs[1][1]
    assert float(np.abs(p2 - 0.5 * p1).max()) <= 1e-12
    j1 = port.main(x.astype(np.float64), r.astype(np.float64), cfg, False, True)[1]
    j2 = port.main(0.5 * x.astype(np.float64), r.astype(np.float64), cfg, False, True)[1]
    # independent jobs bring both to the reference's level: 6 dB away from the 0.5 relation
    off_db = 20 * np.log10(np.sqrt(np.mean(j2 ** 2)) / np.sqrt(np.mean((0.5 * j1) ** 2)))
    assert off_db > 3.0


# ---- emulator driver -------------------------------------------------------------------------------------------------
def run_album(cfg, targets, blob, operator=False, pattern=None, album_pattern=None):
    """mgb_album_match then mgb_finalize per track -> ([outs per track], [states], fir)."""
    lib, ep = emul_lib(), get_emul_plan(cfg, operator)
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
    assert nb > 0
    aws = ebuf(nb, album_pattern if album_pattern is not None else pattern, 40)
    fir = ebuf(16 * cfg.fft_size, pattern, 41).view(np.float64).reshape(2, cfg.fft_size)
    _native.check(lib, lib.mgb_album_match(P, n, table, ptr(blob), ptr(fir), ptr(aws), nb, None))
    outs, states = [], []
    for k, (L, ws, tgt, res, st) in enumerate(keep):
        T = L.target_frames
        o = [ebuf(T * 8, pattern, 50 + 3 * k + j).view(np.float32).reshape(T, 2) for j in range(3)]
        _native.check(lib, lib.mgb_finalize(P, C.byref(L), ptr(res), *(ptr(x) for x in o), ptr(ws), ptr(st), None))
        outs.append(o)
        states.append(_native.TrackState.from_buffer_copy(bytes(st)))
    return outs, states, np.array(fir)


def _ref():
    return port.synth_reference(44100 + 77, 52)


# ---- one-track album == profiled job ---------------------------------------------------------------------------------
PIECE_S = {512: 0.25, 4096: 0.3, 16384: 0.45}  # pieces of 21, 3.2 (the 4F-point convolution) and 1.2 FIR lengths
ONE_TRACK = [(512, False, 4), (512, True, 4), (4096, False, 4), (4096, True, 4), (16384, False, 4), (16384, True, 4),
             (4096, False, 0), (4096, True, 1), (512, False, 1), (512, True, 0)]


@pytest.mark.parametrize("fft_size,operator,steps", ONE_TRACK)
def test_one_track_album_is_the_profiled_job_bit_for_bit(fft_size, operator, steps):
    cfg = mg.Config(max_piece_size=PIECE_S[fft_size], fft_size=fft_size, rms_correction_steps=steps)
    x = port.synth_target(int(cfg.max_piece_size * 2.6) + 211, 61)
    r = _ref() if fft_size < 16384 else port.synth_reference(2 * 44100 + 77, 52)  # (reference pieces of at least F)
    blob, _ = emul_profile(cfg, r, operator)
    outs, states, fir = run_album(cfg, [x], blob, operator)
    want = run_profiled(cfg, x, blob, operator)
    assert_identical((outs[0], states[0], fir), want, (fft_size, operator, steps))


# ---- K = 3 against the restatement -----------------------------------------------------------------------------------
def _three(cfg):
    """one track shorter than a piece, one of many pieces, one whose pieces end at a frame edge"""
    piece = int(cfg.max_piece_size)
    F = cfg.fft_size
    short = piece // 2 + 37
    edge = (piece // F) * F * 3  # three pieces of a whole number of frames
    return [port.synth_target(short, 71), port.synth_target(piece * 6 + 999, 72), port.synth_target(edge, 73)]


CONFIGS = {"f512": dict(max_piece_size=0.25, fft_size=512), "f2048": dict(max_piece_size=0.5, fft_size=2048)}


@pytest.mark.parametrize("true_peak", [False, True])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_three_tracks_match_the_restatement(name, true_peak):
    cfg = mg.Config(**CONFIGS[name], true_peak=true_peak)
    xs, r = _three(cfg), _ref()
    blob, _ = emul_profile(cfg, r)
    outs, states, fir = run_album(cfg, xs, blob)
    trace = {}
    want = album_oracle.main_album(xs, r, cfg, True, True, True, trace=trace)
    # (the analysis keeps its per-(piece, slot) spectra in float32, as a single job's does: 2e-9 from the float64 FIR)
    assert float(np.abs(fir[0] - trace["firs"]["mid"]).max()) <= 1e-8
    assert float(np.abs(fir[1] - trace["firs"]["side"]).max()) <= 1e-8
    for k, (got, w) in enumerate(zip(outs, want)):
        for j, (a, b) in enumerate(zip(got, w)):
            err = float(np.abs(a - b).max())
            assert err <= 1e-5, (name, true_peak, k, j, err)
    for st in states:  # the album's scalars in every track
        assert st.rms_coefficient == states[0].rms_coefficient and st.gain == states[0].gain
        assert abs(st.rms_coefficient - trace["c0"]) <= 1e-9 * trace["c0"]  # (the golden bound of a single job's c0)
        assert abs(st.gain - trace["gain"]) <= 1e-6 * trace["gain"]  # (measured on the float32 result)
        assert st.target_loud_pieces == sum(int(m.sum()) for m in trace["masks"])


def test_half_level_track_keeps_its_relation():
    cfg = mg.Config(max_piece_size=0.25, fft_size=512)
    x = port.synth_target(44100 + 500, 81)
    blob, _ = emul_profile(cfg, _ref())
    outs, _, _ = run_album(cfg, [x, (0.5 * x).astype(np.float32)], blob)
    p1, p2 = outs[0][1].astype(np.float64), outs[1][1].astype(np.float64)
    assert float(np.abs(p2 - 0.5 * p1).max()) <= 1e-6


def test_track_order_does_not_matter():
    cfg = mg.Config(max_piece_size=0.25, fft_size=512)
    xs, r = _three(cfg), _ref()
    blob, _ = emul_profile(cfg, r)
    a, _, fa = run_album(cfg, xs, blob)
    order = [2, 0, 1]
    b, _, fb = run_album(cfg, [xs[i] for i in order], blob)
    assert float(np.abs(fa - fb).max()) <= 1e-12
    for pos, i in enumerate(order):
        for x, y in zip(a[i], b[pos]):
            assert float(np.abs(x.astype(np.float64) - y).max()) <= 1e-6


def test_poisoned_workspaces_give_the_same_bytes():
    cfg = mg.Config(max_piece_size=0.25, fft_size=2048)
    xs, r = _three(cfg), _ref()
    blob, _ = emul_profile(cfg, r)
    clean = run_album(cfg, xs, blob, pattern=None)
    for pattern in ("ff", "random"):
        got = run_album(cfg, xs, blob, pattern=pattern, album_pattern=pattern)
        assert np.array_equal(got[2], clean[2])
        for go, co in zip(got[0], clean[0]):
            for a, b in zip(go, co):
                assert a.tobytes() == b.tobytes(), pattern
        for gs, cs in zip(got[1], clean[1]):
            assert bytes(gs) == bytes(cs), pattern


# ---- argument errors -------------------------------------------------------------------------------------------------
def test_argument_errors():
    cfg = mg.Config(max_piece_size=0.25, fft_size=512)
    lib, ep = emul_lib(), get_emul_plan(cfg)
    P = C.byref(ep.struct)
    x = port.synth_target(30000, 91)
    blob, _ = emul_profile(cfg, _ref())
    L = profiled_layout(lib, ep, len(x))
    ws = ebuf(L.workspace_bytes, None)
    tgt, res = aligned_copy(x, np.float32), ebuf(len(x) * 8, None)
    st = ebuf(C.sizeof(_native.TrackState), None)
    arr = (_native.TrackLayout * 1)(L)
    nb = int(lib.mgb_album_workspace_bytes(P, 1, arr))
    aws = ebuf(nb, None)

    def call(n=1, edit=None, profile=blob, ws_bytes=nb, album_ws=aws, table_null=False):
        table = (_native.AlbumTrack * max(n, 1))()
        for e in table:
            e.layout = C.pointer(L)
            e.d_target_lr, e.d_result_lr, e.d_workspace, e.d_state = tgt.ctypes.data, res.ctypes.data, ws.ctypes.data, st.ctypes.data
        if edit:
            edit(table[0])
        return lib.mgb_album_match(P, n, None if table_null else table, ptr(profile), None,
                                   album_ws.ctypes.data if album_ws is not None else None, ws_bytes, None)

    assert call() == _native.MGB_OK
    assert call(n=0) == _native.MGB_ERR_INVALID
    assert call(n=_native.MGB_MAX_ALBUM_TRACKS + 1) == _native.MGB_ERR_INVALID
    assert call(table_null=True) == _native.MGB_ERR_INVALID
    assert call(edit=lambda e: setattr(e, "d_target_lr", None)) == _native.MGB_ERR_INVALID
    assert call(edit=lambda e: setattr(e, "d_workspace", ws.ctypes.data + 4)) == _native.MGB_ERR_INVALID
    assert call(edit=lambda e: setattr(e, "d_state", None)) == _native.MGB_ERR_INVALID
    assert call(edit=lambda e: setattr(e, "d_result_lr", tgt.ctypes.data)) == _native.MGB_ERR_INVALID
    paired = ep.layout(len(x), 30000)
    assert call(edit=lambda e: setattr(e, "layout", C.pointer(paired))) == _native.MGB_ERR_INVALID
    other = get_emul_plan(mg.Config(max_piece_size=0.5, fft_size=512))
    foreign = profiled_layout(lib, other, len(x))  # another plan's layout of the same length
    assert call(edit=lambda e: setattr(e, "layout", C.pointer(foreign))) == _native.MGB_ERR_INVALID
    assert lib.mgb_track_layout_init_profiled(P, 512, C.byref(_native.TrackLayout())) == _native.MGB_ERR_INVALID
    assert call(ws_bytes=nb - 1) == _native.MGB_ERR_WORKSPACE
    assert call(album_ws=None) == _native.MGB_ERR_INVALID
    bad = np.array(blob)
    bad_blob = aligned_copy(bad)
    h = _native.ReferenceProfileHeader.from_buffer_copy(bytes(bad_blob[:C.sizeof(_native.ReferenceProfileHeader)]))
    h.max_piece_size = h.max_piece_size * 2
    bad_blob[:C.sizeof(h)] = np.frombuffer(bytes(h), np.uint8)
    assert call(profile=bad_blob) == _native.MGB_ERR_INVALID
    assert int(lib.mgb_album_workspace_bytes(P, 0, arr)) == -1
    assert int(lib.mgb_album_workspace_bytes(P, 1, None)) == -1


# ---- Python refusals (before any device work) ------------------------------------------------------------------------
def test_python_refusals(tmp_path):
    x = np.zeros((50000, 2))
    with pytest.raises(ValueError):
        stages.main_album([], x, mg.Config())
    with pytest.raises(ValueError):
        stages.main_album([x] * (_native.MGB_MAX_ALBUM_TRACKS + 1), x, mg.Config())
    with pytest.raises(ValueError):
        stages.main_album([x], x, mg.Config(loudness_target=-14))
    with pytest.raises(ValueError):
        mg.process_album([], "ref.wav", [])
    with pytest.raises(ValueError):
        mg.process_album(["a.wav", "b.wav"], "ref.wav", [[mg.pcm16("a_out.wav")]])
    with pytest.raises(ValueError):
        mg.process_album(["a.wav"], "ref.wav", [[mg.pcm16("a_out.wav")]], config=mg.Config(loudness_target=-14))
    with pytest.raises(ValueError):
        mg.process_album(["a.wav"] * (_native.MGB_MAX_ALBUM_TRACKS + 1), "ref.wav",
                         [[mg.pcm16("o.wav")]] * (_native.MGB_MAX_ALBUM_TRACKS + 1))
    # native_rate with a target off the internal rate: refused when the file's rate is read, before the device
    import wave
    path = str(tmp_path / "t48.wav")
    with wave.open(path, "wb") as w:
        w.setnchannels(2), w.setsampwidth(2), w.setframerate(48000)
        w.writeframes(np.zeros(48000 * 2, np.int16).tobytes())
    with pytest.raises(ValueError):
        mg.process_album([path], "ref.wav", [[mg.pcm16(str(tmp_path / "o.wav"))]], config=mg.Config(native_rate=True))


# ---- thread orders and ThreadSanitizer -------------------------------------------------------------------------------
DUMP_ID = "tests/test_album.py::test_dump_for_thread_orders_emulated"


def test_dump_for_thread_orders_emulated():
    """A small album at F = 512 and 2048 (both convolution grids, two correction steps); with MGB_ALBUM_DUMP set, its
    FIRs, states and outputs go to that file."""
    raws = b""
    for name in CONFIGS:
        cfg = mg.Config(**CONFIGS[name], rms_correction_steps=3)
        xs = _three(cfg)
        blob, _ = emul_profile(cfg, _ref())
        outs, states, fir = run_album(cfg, xs, blob)
        raws += fir.tobytes() + b"".join(bytes(s) for s in states) + b"".join(o.tobytes() for t in outs for o in t)
    if os.environ.get("MGB_ALBUM_DUMP"):
        with open(os.environ["MGB_ALBUM_DUMP"], "wb") as f:
            f.write(raws)


@pytest.fixture(scope="module")
def other_runs(tmp_path_factory):
    from concurrent.futures import ThreadPoolExecutor

    import build_emul
    from test_emul_racecheck import run_group, tsan_env
    build_emul.build(racecheck=True)
    build_emul.build()
    base = tmp_path_factory.mktemp("album_racecheck")
    jobs = {}
    env = tsan_env(str(base / "tsan"))
    env["MGB_EMUL_BUILD"] = "racecheck"
    jobs["tsan"] = ([DUMP_ID], env, str(base / "tsan"))
    for order in ("forward", "reverse", "seeded"):
        env = dict(os.environ, MGB_EMUL_ORDER=order, MGB_EMUL_SEED="4242", MGB_ALBUM_DUMP=str(base / f"dump_{order}.bin"))
        jobs[order] = ([DUMP_ID], env, str(base / order))
    with ThreadPoolExecutor(max_workers=4) as ex:
        futures = {key: ex.submit(run_group, *job) for key, job in jobs.items()}
        done = {key: f.result() + (jobs[key][2],) for key, f in futures.items()}
    return done, base


def test_album_kernels_have_no_data_races(other_runs):
    from test_emul_racecheck import reports
    rc, out, _, log_dir = other_runs[0]["tsan"]
    n, first = reports(log_dir)
    assert n == 0, f"{n} ThreadSanitizer report(s); the first:\n{first}"
    assert rc == 0, out


@pytest.mark.parametrize("order", ["reverse", "seeded"])
def test_album_is_bit_identical_in_other_thread_orders(other_runs, order):
    """The album's pooled sums visit pieces and items in a fixed order and its per-piece sums are added block after
    block in the emulator, so every thread order gives the same bytes."""
    done, base = other_runs
    for o in ("forward", order):
        rc, out, _, _ = done[o]
        assert rc == 0, out
    forward = (base / "dump_forward.bin").read_bytes()
    assert len(forward) > 0
    assert (base / f"dump_{order}.bin").read_bytes() == forward
