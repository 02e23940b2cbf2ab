"""Album loudness on the H100: test_album_gpu.py's four 3-minute C2 tracks driven to -14 LUFS as an album, in sample-peak
mode and at -1 dBTP, against the float64 search (tests/album_loudness_oracle.py); the level offsets kept at a quiet
target; a one-track album against the profiled single job with Config(loudness_target=-14); the album meter against the
restatement; mg.process_album to 24-bit WAV files at -14 LUFS; the new kernel launched."""
import ctypes as C
import math

import numpy as np
import pytest

import album_loudness_oracle as alo
import loudness_target_oracle as lto
from test_album_gpu import C2_FRAMES, GAINS_DB, REPEAT_TOL, album_material
from test_loudness import LOUD_TOL, TP_TOL_DB
from test_loudness_target_gpu import assert_report_matches

pytestmark = pytest.mark.gpu
FS = 44100


@pytest.fixture(scope="module")
def c2():
    import torch
    import matchering_b200 as mg
    from matchering_b200 import analyze_reference
    import port
    assert torch.cuda.is_available()
    r = port.synth_reference(C2_FRAMES, 1000)
    return album_material(), r, {tp: analyze_reference(r, _cfg(tp)) for tp in (False, True)}


def _cfg(tp):
    import matchering_b200 as mg
    return mg.Config(true_peak=True, threshold=10 ** (-1.0 / 20)) if tp else mg.Config()


def album_to_loudness(xs, prof, cfg, target):
    """stages 1-3 of the album and the album target on the device -> (limited numpy per track, report, s_t per track)."""
    import torch
    from matchering_b200 import _native
    from matchering_b200.engine import TrackSession, album_finalize_to_loudness, album_match, get_plan, to_device_f32
    plan = get_plan(cfg)
    with torch.cuda.device(plan.device):
        d = [to_device_f32(x, plan.device) for x in xs]
        sessions = [TrackSession(plan, int(x.shape[0]), None) for x in d]
        album_match(sessions, d, prof.checked_blob(plan))
        outs, report = album_finalize_to_loudness(sessions, target)
        rep = _native.LoudnessTargetReport.from_buffer_copy(report.cpu().numpy().tobytes())
        ss = [s.result.cpu().numpy().astype(np.float64) * s.read_state().gain for s in sessions]
        return [o[0].cpu().numpy() for o in outs], rep, ss


@pytest.mark.parametrize("tp", [False, True], ids=["sample-peak", "true-peak"])
def test_album_reaches_minus_14(c2, tp):
    import matchering_b200 as mg
    xs, _, profs = c2
    cfg = _cfg(tp)
    outs, rep, ss = album_to_loudness(xs, profs[tp], cfg, -14.0)
    assert rep.status == lto.REACHED, (rep.status, list(rep.trace_gain_db), list(rep.trace_integrated))
    m = mg.album_loudness(outs, FS)
    assert abs(m.album.integrated - -14.0) <= lto.TOLERANCE
    assert abs(m.album.integrated - rep.integrated) <= 1e-6
    want = alo.search_album(ss, cfg, -14.0)
    assert_report_matches(rep, want)
    assert abs(rep.gain_db - want["gain_db"]) <= 1e-4 and abs(rep.integrated - want["integrated"]) <= 1e-3


def test_quiet_album_keeps_the_offsets(c2):
    import matchering_b200 as mg
    xs, _, profs = c2
    outs, rep, _ = album_to_loudness(xs, profs[False], _cfg(False), -30.0)
    assert rep.status == lto.REACHED
    got = [mg.loudness(o, FS).integrated for o in outs[:len(GAINS_DB)]]
    inputs = [mg.loudness(x, FS).integrated for x in xs[:len(GAINS_DB)]]
    for k in range(1, len(GAINS_DB)):
        assert abs((got[k] - got[0]) - (inputs[k] - inputs[0])) <= 1e-3, (k, got, inputs)


def test_one_track_album_is_the_profiled_target_job(c2):
    import matchering_b200 as mg
    from matchering_b200 import stages
    xs, _, profs = c2
    got = stages.main_album([xs[0]], profs[False], mg.Config(), True, False, False, album_loudness_target=-14.0)[0][0]
    cfg = mg.Config(loudness_target=-14.0)
    want = stages.main_device(xs[0], profs[False], cfg, True, False, False)[0].cpu().numpy()
    again = stages.main_device(xs[0], profs[False], cfg, True, False, False)[0].cpu().numpy()
    bound = max(REPEAT_TOL, float(np.abs(want.astype(np.float64) - again).max()))
    assert float(np.abs(got.astype(np.float64) - want).max()) / max(1.0, float(np.abs(want).max())) <= bound


def test_album_meter_of_the_inputs_matches_the_restatement(c2):
    import matchering_b200 as mg
    xs, _, _ = c2
    m = mg.album_loudness(xs, FS)
    want = alo.measure_album([x.astype(np.float64) for x in xs], FS)
    for k in ("integrated", "loudness_range", "momentary_max", "short_term_max"):
        assert abs(getattr(m.album, k) - want[k]) <= LOUD_TOL, (k, getattr(m.album, k), want[k])
    db = 20 * math.log10(float(np.max(want["true_peak"])))
    assert abs(m.album.true_peak - db) <= TP_TOL_DB
    for t, x in zip(m.tracks, xs):
        assert t == mg.loudness(x, FS)


def test_process_album_to_minus_14(c2, tmp_path):
    import matchering_b200 as mg
    from matchering_b200 import wavio
    xs, r, _ = c2
    paths = []
    for k, x in enumerate(xs):
        p = str(tmp_path / f"t{k}.wav")
        wavio.write(p, x.astype(np.float64), FS, "PCM_24")
        paths.append(p)
    ref = str(tmp_path / "ref.wav")
    wavio.write(ref, r.astype(np.float64), FS, "PCM_24")
    outs = [str(tmp_path / f"o{k}.wav") for k in range(len(xs))]
    mg.process_album(paths, ref, [[mg.pcm24(o)] for o in outs], album_loudness_target=-14)
    m = mg.album_loudness(outs)
    assert abs(m.album.integrated - -14.0) <= lto.TOLERANCE, m.album


def test_every_new_kernel_is_launched(c2):
    import matchering_b200 as mg
    from matchering_b200 import _native, stages
    xs, _, profs = c2
    lib = _native.load()
    lib.mgb_profile_enable(1)
    try:
        stages.main_album_device(xs[:2], profs[False], mg.Config(), True, False, False, album_loudness_target=-14.0)
        names = C.create_string_buffer(1 << 16)
        ms = (C.c_float * 4096)()
        n = lib.mgb_profile_collect(names, len(names), ms, 4096)
    finally:
        lib.mgb_profile_enable(0)
    launched = set(names.value.decode().split("\n")[:n])
    assert "album_target_fanout_kernel" in launched
