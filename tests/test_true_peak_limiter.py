"""The limiter's true-peak mode without a GPU: the float64 oracle (tests/true_peak_oracle.py) against its definition and
the overshoot it leaves, and the kernels (mgb_limit, mgb_test_limiter_gains, mgb_finalize, the pipeline) on the CPU
emulator against the oracle, on poisoned workspaces, in other thread orders and under ThreadSanitizer."""
import ctypes as C
import os

import numpy as np
import pytest

from emul_harness import aligned, aligned_copy, emul_lib, get_emul_plan, ptr, run_pipeline  # (puts oracle/ on sys.path)
import loudness
import port
import true_peak_oracle as tpo
import matchering_b200 as mg
from matchering_b200 import _native, plan

TOL = 1e-5  # the limiter's parity bound
CHUNK = 4608  # kLimiterCore
RATES = {44100: 4, 48000: 4, 96000: 2, 192000: 1}


def tp_config(fs=44100, **limiter):
    return mg.Config(internal_sample_rate=fs, true_peak=True, limiter=mg.LimiterConfig(**limiter) if limiter else None)


def emul_limit(x, cfg, gains=False, pattern=None):
    """mgb_limit (or mgb_test_limiter_gains) on the emulator -> (output, engaged)."""
    lib = emul_lib()
    params = _native.LimiterParams.from_constants(plan.limiter_constants(cfg))
    n = len(x)
    nbytes = int(lib.mgb_limiter_workspace_bytes(C.byref(params), n))
    ws = aligned((nbytes,), np.uint8)
    if pattern == "ff":
        ws[...] = 0xFF
    elif pattern == "random":
        ws[...] = np.random.default_rng(n).integers(0, 256, nbytes, dtype=np.uint8)
    xi, out, engaged = aligned_copy(x, np.float32), aligned((n, 2), np.float32), aligned((4,), np.int32)
    entry = lib.mgb_test_limiter_gains if gains else lib.mgb_limit
    _native.check(lib, entry(C.byref(params), ptr(xi), ptr(out), n, ptr(ws), nbytes, ptr(engaged), None))
    return np.array(out), int(engaged[0])


def overshoot_db(y, fs, thr):
    return 20.0 * np.log10(loudness.true_peak(np.asarray(y, np.float64), fs).max() / thr)


# ---- the oracle --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fs", [44100, 96000, 192000])
def test_oracle_phase_zero_is_the_signal(fs):
    x = port.synth_limiter_input(3000, 1).astype(np.float64)
    y = tpo.interpolated(x, fs)
    assert y.shape == (2, 3000, RATES[fs])
    np.testing.assert_allclose(y[:, :, 0].T, x, rtol=0, atol=1e-15)


def test_oracle_detector_at_one_times_oversampling_is_the_sample_peak_pair():
    x = port.synth_limiter_input(5000, 2).astype(np.float64)
    u = np.abs(x).max(axis=1)
    want = np.maximum(u, np.concatenate([[0.0], u[:-1]]))
    np.testing.assert_allclose(tpo.true_peak_detector(x, 192000), want, rtol=0, atol=1e-15)


def test_oracle_detector_streams_in_chunks():
    x = port.synth_limiter_input(10007, 3).astype(np.float64)
    whole = tpo.true_peak_detector(x, 44100)
    np.testing.assert_array_equal(tpo.true_peak_detector(x, 44100, chunk=999), whole)
    # it bounds every interpolated point of the meter, within one sample of each frame
    assert whole.max() == pytest.approx(loudness.true_peak(x, 44100).max(), rel=1e-12)


@pytest.mark.parametrize("oversample", [1, 2, 4])
def test_taps_built_in_c_match_the_meters_filter(oversample):
    lib = emul_lib()
    h = np.zeros(12 * oversample + 1)
    _native.check(lib, lib.mgb_true_peak_taps(oversample, h.ctypes.data_as(C.c_void_p)))
    fs = {4: 44100, 2: 96000, 1: 192000}[oversample]
    np.testing.assert_allclose(h, loudness.true_peak_filter(fs)[1], rtol=0, atol=1e-15)
    assert lib.mgb_true_peak_taps(3, h.ctypes.data_as(C.c_void_p)) == _native.MGB_ERR_INVALID


def _material(kind, n):
    if kind == "white":
        return port.synth_target(n, 11).astype(np.float64) * 2.0
    if kind == "c5":
        return port.synth_limiter_input(n, 12).astype(np.float64)
    if kind == "pink":
        return port.synth_reference(n, 13).astype(np.float64) * 1.5
    return port.synth_tonal(n, 14).astype(np.float64) * 6.0


@pytest.mark.parametrize("kind,bound_db", [("white", 0.2), ("c5", 0.2), ("pink", 0.05), ("tonal", 0.05)])
def test_oracle_overshoot_is_small(kind, bound_db):
    """The gain follows the detector but is applied to the samples, so its own movement inside the interpolator's
    support leaks through: a small overshoot remains (DESIGN.md, section 4).  20 s at 44.1 kHz."""
    x = _material(kind, 20 * 44100)
    for attack in (0.1, 1.0, 5.0):
        cfg = tp_config(attack=attack)
        over = overshoot_db(tpo.limit(x, cfg), 44100, cfg.threshold)
        assert over <= bound_db, (kind, attack, over)
        assert overshoot_db(port.limit(x, mg.Config(limiter=mg.LimiterConfig(attack=attack))), 44100, cfg.threshold) > over


# ---- the kernels against the oracle ------------------------------------------------------------------------------------
LENGTHS = [7, 13, CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK + 1, 3 * CHUNK + 517]


@pytest.mark.parametrize("fs", list(RATES))
@pytest.mark.parametrize("n", LENGTHS)
def test_limit_matches_oracle_emulated(fs, n):
    x = port.synth_limiter_input(n, n + fs)
    cfg = tp_config(fs)
    got, engaged = emul_limit(x, cfg)
    assert engaged == 1
    assert float(np.abs(got - tpo.limit(x.astype(np.float64), cfg)).max()) < TOL


WIDE = dict(attack=50, hold_filter_order=2, release_filter_order=2)


@pytest.mark.parametrize("n", [13, CHUNK + 1, 5 * CHUNK + 7])
def test_limit_matches_oracle_on_the_wide_window_path_emulated(n):
    cfg = tp_config(44100, **WIDE)
    assert _native.LimiterParams.from_constants(plan.limiter_constants(cfg)).true_peak == 4
    x = port.synth_limiter_input(n, n)
    got, engaged = emul_limit(x, cfg)
    assert engaged == 1
    assert float(np.abs(got - tpo.limit(x.astype(np.float64), cfg)).max()) < TOL


@pytest.mark.parametrize("fs,limiter", [(44100, {}), (48000, {}), (96000, {}), (44100, dict(hold_filter_order=2)),
                                        (44100, WIDE)], ids=["44100", "48000", "96000", "44100-order2", "44100-wide"])
def test_gain_envelopes_match_oracle_emulated(fs, limiter):
    """Both gains through mgb_test_limiter_gains: (g_att, max(hold_out, release_out)).  (The halo kernel's test entry
    exists for the spans of the default limiter up to 96 kHz; at 192 kHz the outputs above are compared instead.)"""
    cfg = tp_config(fs, **limiter)
    x = port.synth_limiter_input(3 * CHUNK + 11, 7)
    got, _ = emul_limit(x, cfg, gains=True)
    trace = {}
    tpo.limit(x.astype(np.float64), cfg, trace)
    assert float(np.abs(got[:, 0] - trace["g_att"]).max()) < TOL
    assert float(np.abs(got[:, 1] - trace["g_rel"]).max()) < TOL


def _sine_between_samples(n, amplitude):
    """A sine at fs/4 sampled 45 degrees off its crests: every sample is amplitude / sqrt(2), the true peak is
    amplitude."""
    k = np.arange(n)
    s = amplitude * np.sin(0.5 * np.pi * k + 0.25 * np.pi)
    return np.ascontiguousarray(np.stack([s, s], axis=1).astype(np.float32))


def test_early_out_follows_the_true_peak_emulated():
    cfg = tp_config()
    x = _sine_between_samples(6000, 1.0)
    assert np.abs(x).max() < cfg.threshold < tpo.true_peak_detector(x.astype(np.float64), 44100).max()
    _, engaged = emul_limit(x, mg.Config())
    assert engaged == 0  # sample peaks: nothing to do
    got, engaged = emul_limit(x, cfg)
    assert engaged == 1
    assert float(np.abs(got - tpo.limit(x.astype(np.float64), cfg)).max()) < TOL
    quiet = _sine_between_samples(6000, 0.9)
    got, engaged = emul_limit(quiet, cfg)
    assert engaged == 0
    np.testing.assert_array_equal(got, quiet)
    q64 = quiet.astype(np.float64)
    assert tpo.limit(q64, cfg) is q64


def test_sample_peak_mode_is_unchanged():
    """true_peak=False is the default Config's limiter: the same parameters, bit for bit the same output."""
    for fs in (44100, 192000):
        a = _native.LimiterParams.from_constants(plan.limiter_constants(mg.Config(internal_sample_rate=fs)))
        b = _native.LimiterParams.from_constants(plan.limiter_constants(mg.Config(internal_sample_rate=fs, true_peak=False)))
        assert bytes(a) == bytes(b) and a.true_peak == 0
    x = port.synth_limiter_input(2 * CHUNK + 5, 4)
    got, _ = emul_limit(x, mg.Config(true_peak=False))
    np.testing.assert_array_equal(got, emul_limit(x, mg.Config())[0])
    assert float(np.abs(got - port.limit(x.astype(np.float64), port.OracleConfig())).max()) < TOL
    assert plan.config_key(mg.Config(true_peak=True)) != plan.config_key(mg.Config())


def test_workspace_grows_by_the_detector_plane_only_in_true_peak_mode():
    lib = emul_lib()
    for cfg in (mg.Config(), mg.Config(limiter=mg.LimiterConfig(**WIDE))):
        p = _native.LimiterParams.from_constants(plan.limiter_constants(cfg))
        base = int(lib.mgb_limiter_workspace_bytes(C.byref(p), 100000))
        p.true_peak = 4
        assert int(lib.mgb_limiter_workspace_bytes(C.byref(p), 100000)) == base + 400128
    ep, tp = get_emul_plan(mg.Config(max_piece_size=1.0)), get_emul_plan(mg.Config(max_piece_size=1.0, true_peak=True))
    assert tp.layout(100000, 50000).workspace_bytes == ep.layout(100000, 50000).workspace_bytes + 256 + 400128


def test_invalid_oversampling_is_rejected_emulated():
    lib = emul_lib()
    p = _native.LimiterParams.from_constants(plan.limiter_constants(mg.Config()))
    x, out, eng = aligned((1000, 2), np.float32), aligned((1000, 2), np.float32), aligned((4,), np.int32)
    for bad in (-1, 3, 8):
        p.true_peak = bad
        nbytes = 1 << 22
        ws = aligned((nbytes,), np.uint8)
        assert lib.mgb_limit(C.byref(p), ptr(x), ptr(out), 1000, ptr(ws), nbytes, ptr(eng), None) == _native.MGB_ERR_INVALID


@pytest.mark.parametrize("pattern", ["ff", "random"])
def test_poisoned_workspace_changes_nothing_emulated(pattern):
    for cfg, n in ((tp_config(), 3 * CHUNK + 1), (tp_config(**WIDE), 2 * CHUNK + 3)):
        x = port.synth_limiter_input(n, 9)
        np.testing.assert_array_equal(emul_limit(x, cfg, pattern=pattern)[0], emul_limit(x, cfg)[0])


# ---- the whole job: mgb_finalize -----------------------------------------------------------------------------------
def test_finalize_matches_oracle_emulated():
    """Limited and normalised outputs of a true-peak plan against the oracle; the normalised output's true peak is the
    threshold, and the state's sample-peak fields are the sample-peak plan's."""
    cfg = mg.Config(max_piece_size=1.0, true_peak=True)
    n = 44100 * 2 + 123
    t, r = port.synth_target(n, 21), port.synth_reference(n - 999, 22)
    (lim, plain, norm), st, fir, _, _ = run_pipeline(cfg, t, r)
    want_lim, want_norm, _ = tpo.main(t, r, cfg)
    assert float(np.abs(lim - want_lim).max()) < TOL
    assert float(np.abs(norm - want_norm).max()) < TOL
    assert tpo.true_peak_detector(norm.astype(np.float64), 44100).max() == pytest.approx(cfg.threshold, rel=1e-6)
    (lim0, plain0, _), st0, fir0, _, _ = run_pipeline(mg.Config(max_piece_size=1.0), t, r)
    np.testing.assert_array_equal(plain, plain0)
    np.testing.assert_array_equal(fir, fir0)
    assert st.result_peak == st0.result_peak and st.gain == st0.gain
    assert st.normalize_coef > st0.normalize_coef and st.limiter_engaged == 1


def test_finalize_dump_for_thread_orders_emulated():
    """Limited outputs of fixed inputs (halo and wide-window plans); with MGB_TRUE_PEAK_DUMP set, their bytes go to
    that file (the thread-order runs below compare them with a forward run)."""
    raws = b""
    n = 44100 + 4000
    t, r = port.synth_target(n, 31), port.synth_reference(n, 32)
    for cfg in (mg.Config(max_piece_size=0.5, true_peak=True),
                mg.Config(max_piece_size=0.5, true_peak=True, limiter=mg.LimiterConfig(**WIDE))):
        (lim, _, norm), _, _, _, _ = run_pipeline(cfg, t, r)
        want_lim, want_norm, _ = tpo.main(t, r, cfg)
        assert float(np.abs(lim - want_lim).max()) < TOL
        raws += lim.tobytes() + norm.tobytes()
    x = port.synth_limiter_input(2 * CHUNK + 9, 33)
    raws += emul_limit(x, tp_config())[0].tobytes() + emul_limit(x, tp_config(96000, **WIDE))[0].tobytes()
    if os.environ.get("MGB_TRUE_PEAK_DUMP"):
        with open(os.environ["MGB_TRUE_PEAK_DUMP"], "wb") as f:
            f.write(raws)


# ---- the pipeline ----------------------------------------------------------------------------------------------------
def _pcm16(x):
    return np.clip(np.rint(np.asarray(x, np.float64) * 32767.0), -32768, 32767).astype(np.int16)


def test_pipeline_limits_and_meters_every_kind_of_submit_emulated():
    """A depth-2 pipeline of a true-peak plan, with metering, fed paired and profiled, float32 and PCM16 jobs: every
    float32 output matches the oracle, every meter is mgb_loudness of the slot's output, and a profile made by a plan
    WITHOUT true_peak masters here with the paired job's level statistics."""
    from test_loudness import emul_meter, emul_params
    from test_reference_profile import emul_profile
    lib = emul_lib()
    cfg = port.OracleConfig(fft_size=1024, max_piece_size=0.3)
    cfg.true_peak = True
    fs = cfg.internal_sample_rate
    ep = get_emul_plan(cfg)
    assert ep.struct.limiter.true_peak == 4
    lengths = [20011, 16007, 19003]
    pcm_t = [_pcm16(port.synth_target(n, 70 + k) * 1.6) for k, n in enumerate(lengths)]
    targets = [(q.astype(np.float64) / 32768.0).astype(np.float32) for q in pcm_t]
    pcm_r = _pcm16(port.synth_reference(18000, 3))
    r = (pcm_r.astype(np.float64) / 32768.0).astype(np.float32)
    blob, _ = emul_profile(port.OracleConfig(fft_size=1024, max_piece_size=0.3), r)  # (a sample-peak plan's profile)
    h = C.c_void_p()
    _native.check(lib, lib.mgb_pipeline_create(C.byref(ep.struct), max(lengths), len(r), 2, C.byref(h)))
    results, keep = [], []
    try:
        _native.check(lib, lib.mgb_pipeline_enable_loudness(h, C.byref(emul_params(fs))))
        for k in range(len(targets)):
            for kind in ("float", "pcm"):
                for profiled in (False, True):
                    slot = C.c_int32(-1)
                    if kind == "pcm":
                        tt, rr, o = aligned_copy(pcm_t[k]), aligned_copy(pcm_r), aligned((len(targets[k]), 2), np.int16)
                        rc = (lib.mgb_pipeline_submit_pcm_profiled(h, ptr(tt), 16, len(tt), ptr(blob), ptr(o), 16, C.byref(slot))
                              if profiled else lib.mgb_pipeline_submit_pcm(h, ptr(tt), 16, len(tt), ptr(rr), 16, len(rr),
                                                                           ptr(o), 16, C.byref(slot)))
                    else:
                        tt, rr, o = aligned_copy(targets[k]), aligned_copy(r), aligned((len(targets[k]), 2), np.float32)
                        rc = (lib.mgb_pipeline_submit_profiled(h, ptr(tt), len(tt), ptr(blob), ptr(o), C.byref(slot))
                              if profiled else lib.mgb_pipeline_submit(h, ptr(tt), len(tt), ptr(rr), len(rr), ptr(o),
                                                                       C.byref(slot)))
                    _native.check(lib, rc)
                    st, res = _native.TrackState(), _native.LoudnessResult()
                    _native.check(lib, lib.mgb_pipeline_wait_loudness(h, slot.value, C.byref(st), C.byref(res)))
                    keep.append((tt, rr))
                    results.append((k, kind, profiled, np.array(o), st, bytes(res)))
    finally:
        lib.mgb_pipeline_destroy(h)
    thr = cfg.threshold
    for k, kind, profiled, o, st, raw in results:
        paired = next(s for kk, kd, p, _, s, _ in results if kk == k and kd == kind and not p)
        for f in ("target_match_rms", "reference_match_rms", "rms_coefficient", "final_amplitude_coef"):
            assert getattr(st, f) == getattr(paired, f), (k, kind, f)
        if kind == "float":
            want, _, _ = tpo.main(targets[k], r, cfg)
            assert float(np.abs(o - want).max()) < TOL, (k, profiled)
            assert raw == emul_meter(o, fs)
            met = _native.LoudnessResult.from_buffer_copy(raw)
            assert max(met.true_peak) <= thr * st.final_amplitude_coef * 10 ** (0.2 / 20)


# ---- the same kernels under ThreadSanitizer and in other thread orders ----------------------------------------------
HERE = "tests/test_true_peak_limiter.py::"
RACECHECK_IDS = [HERE + "test_limit_matches_oracle_emulated[13-44100]",
                 HERE + f"test_limit_matches_oracle_emulated[{CHUNK + 1}-96000]",
                 HERE + f"test_limit_matches_oracle_emulated[{CHUNK + 1}-192000]",
                 HERE + "test_limit_matches_oracle_on_the_wide_window_path_emulated[13]",
                 HERE + "test_gain_envelopes_match_oracle_emulated[44100]",
                 HERE + "test_finalize_dump_for_thread_orders_emulated"]


@pytest.fixture(scope="module")
def other_runs(tmp_path_factory):
    from concurrent.futures import ThreadPoolExecutor

    import build_emul
    from test_emul_racecheck import run_group, tsan_env
    build_emul.build(racecheck=True)
    build_emul.build()
    base = tmp_path_factory.mktemp("true_peak_racecheck")
    jobs = {}
    for k, i in enumerate(RACECHECK_IDS):
        log_dir = str(base / f"tsan_{k}")
        env = tsan_env(log_dir)
        env["MGB_EMUL_BUILD"] = "racecheck"
        jobs[("tsan", k)] = ([i], env, log_dir)
    for order in ("forward", "reverse", "seeded"):
        env = dict(os.environ, MGB_EMUL_ORDER=order, MGB_EMUL_SEED="4242", MGB_TRUE_PEAK_DUMP=str(base / f"dump_{order}.bin"))
        jobs[(order, 0)] = (RACECHECK_IDS, env, str(base / order))
    with ThreadPoolExecutor(max_workers=8) as ex:
        futures = {key: ex.submit(run_group, *job) for key, job in jobs.items()}
        done = {key: f.result() + (jobs[key][2],) for key, f in futures.items()}
    return done, base


@pytest.mark.parametrize("k", range(len(RACECHECK_IDS)))
def test_true_peak_kernels_have_no_data_races(other_runs, k):
    from test_emul_racecheck import reports
    rc, out, _, log_dir = other_runs[0][("tsan", k)]
    n, first = reports(log_dir)
    assert n == 0, f"{n} ThreadSanitizer report(s) in {RACECHECK_IDS[k]}; the first:\n{first}"
    assert rc == 0, out


@pytest.mark.parametrize("order", ["reverse", "seeded"])
def test_true_peak_limiter_is_bit_identical_in_other_thread_orders(other_runs, order):
    done, base = other_runs
    for o in ("forward", order):
        rc, out, _, _ = done[(o, 0)]
        assert rc == 0, out
    forward = (base / "dump_forward.bin").read_bytes()
    assert len(forward) > 0
    assert (base / f"dump_{order}.bin").read_bytes() == forward
