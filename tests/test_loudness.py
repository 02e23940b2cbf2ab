"""The loudness meter without a GPU: the constants, the float64 oracle against the EBU Tech 3341 / 3342 cases and
analytic true peaks, and the kernels (mgb_loudness, the pipeline's metering) on the CPU emulator against the oracle,
on poisoned workspaces, in other thread orders and under ThreadSanitizer."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from emul_harness import aligned, aligned_copy, emul_lib, get_emul_plan, ptr  # (puts oracle/ on sys.path)
import loudness as oracle
import port
from matchering_b200 import _native, plan

LOUD_TOL = 1e-6   # LU
TP_TOL_DB = 1e-4


# ---- constants -------------------------------------------------------------------------------------------------------
def test_constants_reproduce_bs1770_table_at_48k():
    lc = plan.loudness_constants(48000)
    assert lc.block == 4800 and lc.oversample == 4 and len(lc.tp_taps) == 49
    np.testing.assert_allclose(lc.shelf_b, [1.53512485958697, -2.69169618940638, 1.19839281085285], rtol=0, atol=1e-12)
    np.testing.assert_allclose(lc.shelf_a, [1.0, -1.69065929318241, 0.73248077421585], rtol=0, atol=1e-12)
    np.testing.assert_allclose(lc.highpass_b, [1.0, -2.0, 1.0], rtol=0, atol=0)
    np.testing.assert_allclose(lc.highpass_a, [1.0, -1.99004745483398, 0.99007225036621], rtol=0, atol=1e-12)
    # the oracle derives the same coefficients on its own
    for got, want in zip((lc.shelf_b, lc.shelf_a, lc.highpass_b, lc.highpass_a), oracle.k_weighting(48000)):
        np.testing.assert_array_equal(got, want)


def test_constants_by_rate():
    for fs, os_ in ((8000, 4), (44100, 4), (95999, 4), (96000, 2), (191999, 2), (192000, 1), (384000, 1)):
        lc = plan.loudness_constants(fs)
        assert lc.block == (fs + 5) // 10 and lc.oversample == os_ and len(lc.tp_taps) == 12 * os_ + 1
        assert lc.tp_taps[6 * os_] == 1.0  # phase 0 is the identity
    for fs in (7999, 384001):
        with pytest.raises(ValueError):
            plan.loudness_constants(fs)


# ---- the oracle against the EBU test signals ------------------------------------------------------------------------
def sine_steps(fs, steps, freq=1000.0):
    """A stereo sine at `freq` through (dBFS peak, seconds) steps, phase continuous."""
    n = [int(round(s * fs)) for _, s in steps]
    amp = np.concatenate([np.full(k, 10.0 ** (db / 20.0)) for (db, _), k in zip(steps, n)])
    x = amp * np.sin(2.0 * np.pi * freq * np.arange(len(amp)) / fs)
    return np.stack([x, x], axis=1)


EBU = [  # name, steps, {field: (expected, tolerance)}
    ("3341-1", [(-23, 20)], dict(integrated=(-23, 0.1), momentary_max=(-23, 0.1), short_term_max=(-23, 0.1))),
    ("3341-2", [(-33, 20)], dict(integrated=(-33, 0.1))),
    ("3341-3", [(-36, 10), (-23, 60), (-36, 10)], dict(integrated=(-23, 0.1))),
    ("3341-4", [(-72, 10), (-36, 10), (-23, 60), (-36, 10), (-72, 10)], dict(integrated=(-23, 0.1))),
    ("3341-5", [(-26, 20), (-20, 20.1), (-26, 20)], dict(integrated=(-23, 0.1))),
    ("3342-1", [(-20, 20), (-30, 20)], dict(loudness_range=(10, 1))),
    ("3342-2", [(-20, 20), (-15, 20)], dict(loudness_range=(5, 1))),
    ("3342-3", [(-40, 20), (-20, 20)], dict(loudness_range=(20, 1))),
    ("3342-4", [(-50, 20), (-35, 20), (-20, 20), (-35, 20), (-50, 20)], dict(loudness_range=(15, 1))),
]


@pytest.mark.parametrize("fs", [48000, 44100])
@pytest.mark.parametrize("name,steps,want", EBU, ids=[e[0] for e in EBU])
def test_oracle_passes_ebu_cases(fs, name, steps, want):
    got = oracle.measure(sine_steps(fs, steps), fs)
    for field, (value, tol) in want.items():
        assert abs(got[field] - value) <= tol, (field, got[field])


def test_oracle_true_peak_of_sines():
    """Sines of -6 dBFS analytic peak read -6 dBTP.  They fade in and out over 50 ms: an abrupt start is a step,
    and the interpolator rings over the step's edge."""
    fs = 48000
    n = np.arange(9600)
    env = np.minimum(1.0, np.minimum(n, n[::-1]) / 2400.0)
    env = np.sin(0.5 * np.pi * env) ** 2
    peak = 10.0 ** (-6.0 / 20.0)
    for div, phase_deg in ((4, 0.0), (4, 45.0), (6, 60.0), (8, 67.5)):
        x = peak * env * np.sin(2.0 * np.pi * n / div + np.deg2rad(phase_deg))
        tp = oracle.true_peak(np.stack([x, x], axis=1), fs)
        assert abs(20.0 * np.log10(tp[0]) + 6.0) <= 0.01, (div, phase_deg, tp)
    rng = np.random.default_rng(7)
    for _ in range(40):
        f, ph = rng.uniform(0.01, 0.4) * fs, rng.uniform(0, 2 * np.pi)
        x = peak * env * np.sin(2.0 * np.pi * f * n / fs + ph)
        err = 20.0 * np.log10(oracle.true_peak(np.stack([x, x], axis=1), fs)[0]) + 6.0
        assert -0.5 <= err <= 0.01, (f, ph, err)


def test_oracle_streaming_matches_one_pass():
    from scipy import signal
    rng = np.random.default_rng(3)
    x = rng.standard_normal((160007, 2)) * np.linspace(0.01, 0.5, 160007)[:, None]
    fs = 44100
    whole, chunked = oracle.measure(x, fs), oracle.measure(x, fs, chunk=1000)
    for k in ("integrated", "loudness_range", "momentary_max", "short_term_max"):
        assert abs(whole[k] - chunked[k]) <= 1e-9, k
    L, h = oracle.true_peak_filter(fs)
    direct = [np.abs(signal.upfirdn(h, x[:, c], up=L)).max() for c in range(2)]
    np.testing.assert_allclose(chunked["true_peak"], direct, rtol=1e-14)
    sb, sa, hb, ha = oracle.k_weighting(fs)
    y = signal.lfilter(hb, ha, signal.lfilter(sb, sa, x, axis=0), axis=0)
    B = (fs + 5) // 10
    e = (y[:len(y) // B * B] ** 2).sum(axis=1).reshape(-1, B).sum(axis=1)
    np.testing.assert_allclose(oracle.sub_block_energies(x, fs, chunk=777), e, rtol=1e-12)


# ---- the kernels on the emulator ------------------------------------------------------------------------------------
_TABLES = {}


def emul_params(fs):
    lib = emul_lib()
    if fs not in _TABLES:
        p = _native.LoudnessParams.from_constants(plan.loudness_constants(fs))
        tables = aligned((int(lib.mgb_loudness_tables_bytes()),), np.uint8)
        _native.check(lib, lib.mgb_loudness_fill_tables(C.byref(p), ptr(tables), None))
        p.d_tables = tables.ctypes.data
        _TABLES[fs] = (p, tables)
    return _TABLES[fs][0]


def poison(n, pattern, seed=0):
    if pattern == "ff":
        return np.full(n, 0xFF, np.uint8)
    if pattern == "random":
        return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)
    return np.zeros(n, np.uint8)


def emul_meter(x, fs, pattern=None) -> bytes:
    """mgb_loudness on the emulator -> the raw mgb_loudness_result."""
    lib = emul_lib()
    p = emul_params(fs)
    xa = aligned_copy(x, np.float32)
    n = int(lib.mgb_loudness_workspace_bytes(C.byref(p), len(x)))
    ws = aligned((n,), np.uint8)
    ws[...] = poison(n, pattern)
    res = aligned((C.sizeof(_native.LoudnessResult),), np.uint8)
    res[...] = poison(len(res), pattern, 1)
    _native.check(lib, lib.mgb_loudness(C.byref(p), ptr(xa), len(x), ptr(ws), n, ptr(res), None))
    return bytes(res)


def assert_matches_oracle(raw: bytes, x, fs):
    got = _native.LoudnessResult.from_buffer_copy(raw)
    want = oracle.measure(np.asarray(x, np.float32).astype(np.float64), fs)
    for k in ("integrated", "loudness_range", "momentary_max", "short_term_max"):
        g, w = getattr(got, k), want[k]
        if math.isinf(w):
            assert g == w, (k, g, w)
        else:
            assert abs(g - w) <= LOUD_TOL, (k, g, w)
    assert (got.momentary_count, got.short_term_count) == (want["momentary_count"], want["short_term_count"])
    assert list(got.sample_peak) == list(want["sample_peak"])
    for g, w in zip(got.true_peak, want["true_peak"]):
        if w == 0.0:
            assert g == 0.0
        else:
            assert abs(20.0 * math.log10(g / w)) <= TP_TOL_DB, (g, w)


def material(kind, n, fs, seed):
    rng = np.random.default_rng(seed)
    if kind == "silence":
        return np.zeros((n, 2), np.float32)
    if kind == "impulse":  # one full-scale sample
        x = np.zeros((n, 2), np.float32)
        x[n // 2, 1] = 1.0
        return x
    x = rng.standard_normal((n, 2))
    if kind == "bandlimited":  # 200 Hz .. 0.2 fs
        from scipy import signal
        sos = signal.butter(6, [200.0, 0.2 * fs], btype="bandpass", fs=fs, output="sos")
        x = signal.sosfilt(sos, x, axis=0)
    # level steps: -40, -10, -25 dB thirds, and a quiet stretch under the absolute gate
    gains = np.ones(n)
    cuts = [n // 4, n // 2, 3 * n // 4]
    for (a, b), db in zip(zip([0] + cuts, cuts + [n]), (-40.0, -10.0, -25.0, -80.0)):
        gains[a:b] = 10.0 ** (db / 20.0)
    return (x * gains[:, None]).astype(np.float32)


RATES = [8000, 44100, 96000, 384000]


def lengths(fs):
    B = (fs + 5) // 10
    return {"chunks-1": 3 * 4608 - 1, "chunks+1": 3 * 4608 + 1, "4B-1": 4 * B - 1, "4B": 4 * B,
            "30B": 30 * B if 30 * B <= 300000 else 7 * B + 3, "under_B": B // 2 + 7}


METER_CASES = [(fs, name, kind) for fs in RATES for name, kind in
               zip(lengths(fs), ["noise", "bandlimited", "noise", "bandlimited", "noise", "noise"])]
METER_CASES += [(fs, "4B", kind) for fs in (8000, 384000) for kind in ("silence", "impulse")]
METER_CASES += [(44100, "30B", "silence"), (44100, "30B", "impulse")]


@pytest.mark.parametrize("fs,length,kind", METER_CASES, ids=[f"{fs}-{n}-{k}" for fs, n, k in METER_CASES])
def test_meter_matches_oracle_emulated(fs, length, kind):
    n = lengths(fs)[length]
    x = material(kind, n, fs, seed=n)
    raw = emul_meter(x, fs)
    assert_matches_oracle(raw, x, fs)
    if kind == "silence":
        got = _native.LoudnessResult.from_buffer_copy(raw)
        assert got.integrated == got.momentary_max == -math.inf and got.loudness_range == 0.0
        assert list(got.true_peak) == [0.0, 0.0]


DUMP_CASES = [(44100, 3 * 4608 + 1, "noise"), (96000, 40000, "bandlimited")]


@pytest.mark.parametrize("pattern", ["ff", "random"])
def test_meter_on_poisoned_workspace_is_bit_identical_emulated(pattern):
    for fs, n, kind in DUMP_CASES:
        x = material(kind, n, fs, seed=5)
        assert emul_meter(x, fs, pattern) == emul_meter(x, fs)


def test_meter_rejects_bad_arguments_emulated():
    lib = emul_lib()
    p = emul_params(44100)
    x = aligned((1000, 2), np.float32)
    n = int(lib.mgb_loudness_workspace_bytes(C.byref(p), 1000))
    ws, res = aligned((n,), np.uint8), aligned((128,), np.uint8)
    run = lambda params, xp, frames, wsp, nbytes: lib.mgb_loudness(C.byref(params), xp, frames, wsp, nbytes, ptr(res), None)
    assert run(p, ptr(x), 1000, ptr(ws), n) == _native.MGB_OK
    assert run(p, ptr(x), 1000, ptr(ws), n - 1) == _native.MGB_ERR_INVALID
    assert run(p, ptr(x), 0, ptr(ws), n) == _native.MGB_ERR_INVALID
    assert run(p, C.c_void_p(x.ctypes.data + 4), 999, ptr(ws), n) == _native.MGB_ERR_INVALID
    for field, value in (("sample_rate", 7999), ("sample_rate", 400000), ("block", 4411), ("oversample", 2)):
        bad = _native.LoudnessParams.from_buffer_copy(bytes(p))
        setattr(bad, field, value)
        assert run(bad, ptr(x), 1000, ptr(ws), n) == _native.MGB_ERR_INVALID, field
        assert lib.mgb_loudness_fill_tables(C.byref(bad), ptr(ws), None) == _native.MGB_ERR_INVALID


def test_meter_dump_for_thread_orders_emulated():
    """Meters of fixed inputs; with MGB_LOUDNESS_DUMP set, their raw bytes go to that file (the thread-order runs
    below compare them with a forward run)."""
    raws = b""
    for fs, n, kind in DUMP_CASES:
        x = material(kind, n, fs, seed=9)
        raw = emul_meter(x, fs, "ff")
        assert_matches_oracle(raw, x, fs)
        raws += raw
    if os.environ.get("MGB_LOUDNESS_DUMP"):
        with open(os.environ["MGB_LOUDNESS_DUMP"], "wb") as f:
            f.write(raws)


def _pcm16(x):
    return np.clip(np.rint(np.asarray(x, np.float64) * 32767.0), -32768, 32767).astype(np.int16)


def test_pipeline_meters_every_kind_of_submit_emulated():
    """mgb_pipeline_* at depth 2, created with poison_alloc and metering, fed paired and profiled, float32 and PCM16
    submissions: every slot's meter is bit-identical to mgb_loudness of that slot's float32 limited output (a PCM
    submission's: the float32 submission of the same decoded samples)."""
    from test_reference_profile import emul_profile
    lib = emul_lib()
    cfg = port.OracleConfig(fft_size=1024, max_piece_size=0.3)
    fs = cfg.internal_sample_rate
    ep = get_emul_plan(cfg)
    lengths_ = [20011, 16007, 19003, 14009, 17011]
    pcm_t = [_pcm16(port.synth_target(n, 60 + k)) for k, n in enumerate(lengths_)]
    targets = [(q.astype(np.float64) / 32768.0).astype(np.float32) for q in pcm_t]  # exact in float32
    pcm_r = _pcm16(port.synth_reference(18000, 2))
    r = (pcm_r.astype(np.float64) / 32768.0).astype(np.float32)
    blob, _ = emul_profile(cfg, r)
    h = C.c_void_p()
    _native.check(lib, lib.mgb_set_option(b"poison_alloc", 1))
    try:
        _native.check(lib, lib.mgb_pipeline_create(C.byref(ep.struct), max(lengths_), len(r), 2, C.byref(h)))
        _native.check(lib, lib.mgb_pipeline_enable_loudness(h, C.byref(emul_params(fs))))
    finally:
        lib.mgb_set_option(b"poison_alloc", 0)
    # (float, paired) (pcm, profiled) (float, profiled) (pcm, paired) ...: each slot is reused by the other kinds
    jobs = [(k, kind) for k in range(len(targets)) for kind in (("float", "pcm") if k % 2 else ("float",))]
    results, keep = [], []
    try:
        assert lib.mgb_pipeline_enable_loudness(h, C.byref(emul_params(fs))) == _native.MGB_ERR_INVALID  # once only
        for j, (k, kind) in enumerate(jobs):
            slot = C.c_int32(-1)
            profiled = j % 3 == 1
            if kind == "pcm":
                tt, rr, o = aligned_copy(pcm_t[k]), aligned_copy(pcm_r), aligned((len(targets[k]), 2), np.int16)
                rc = (lib.mgb_pipeline_submit_pcm_profiled(h, ptr(tt), 16, len(tt), ptr(blob), ptr(o), 16, C.byref(slot))
                      if profiled else
                      lib.mgb_pipeline_submit_pcm(h, ptr(tt), 16, len(tt), ptr(rr), 16, len(rr), ptr(o), 16, C.byref(slot)))
            else:
                tt, rr, o = aligned_copy(targets[k]), aligned_copy(r), aligned((len(targets[k]), 2), np.float32)
                rc = (lib.mgb_pipeline_submit_profiled(h, ptr(tt), len(tt), ptr(blob), ptr(o), C.byref(slot)) if profiled
                      else lib.mgb_pipeline_submit(h, ptr(tt), len(tt), ptr(rr), len(rr), ptr(o), C.byref(slot)))
            _native.check(lib, rc)
            st, res = _native.TrackState(), _native.LoudnessResult()
            _native.check(lib, lib.mgb_pipeline_wait_loudness(h, slot.value, C.byref(st), C.byref(res)))
            keep.append((tt, rr))
            results.append((k, kind, o, bytes(res)))
    finally:
        lib.mgb_pipeline_destroy(h)
    float_out = {k: o for k, kind, o, _ in results if kind == "float"}
    seeded = os.environ.get("MGB_EMUL_ORDER") == "seeded"
    for k, kind, o, raw in results:
        want = emul_meter(float_out[k], fs)
        if kind == "float" or not seeded:
            assert raw == want, (k, kind)
        else:  # a random thread order sums stage 3's float64 atomics in another order in each job
            got, ref = _native.LoudnessResult.from_buffer_copy(raw), _native.LoudnessResult.from_buffer_copy(want)
            for f in ("integrated", "momentary_max"):
                assert getattr(got, f) == getattr(ref, f) or abs(getattr(got, f) - getattr(ref, f)) <= 1e-4, f
    # a pipeline without metering refuses the meter's wait
    h = C.c_void_p()
    _native.check(lib, lib.mgb_pipeline_create(C.byref(ep.struct), 20000, 20000, 1, C.byref(h)))
    try:
        assert lib.mgb_pipeline_wait_loudness(h, 0, None, None) == _native.MGB_ERR_INVALID
    finally:
        lib.mgb_pipeline_destroy(h)


# ---- the same kernels under ThreadSanitizer and in other thread orders ----------------------------------------------
HERE = "tests/test_loudness.py::"
RACECHECK_IDS = [HERE + "test_meter_matches_oracle_emulated[44100-chunks+1-bandlimited]",
                 HERE + "test_meter_matches_oracle_emulated[8000-4B-impulse]",
                 HERE + "test_meter_matches_oracle_emulated[96000-4B-1-noise]",
                 HERE + "test_meter_matches_oracle_emulated[384000-under_B-noise]",
                 HERE + "test_meter_dump_for_thread_orders_emulated",
                 HERE + "test_pipeline_meters_every_kind_of_submit_emulated"]


@pytest.fixture(scope="module")
def other_runs(tmp_path_factory):
    from concurrent.futures import ThreadPoolExecutor

    import build_emul
    from test_emul_racecheck import run_group, tsan_env
    build_emul.build(racecheck=True)
    build_emul.build()
    base = tmp_path_factory.mktemp("loudness_racecheck")
    jobs = {}
    for k, i in enumerate(RACECHECK_IDS):
        log_dir = str(base / f"tsan_{k}")
        env = tsan_env(log_dir)
        env["MGB_EMUL_BUILD"] = "racecheck"
        jobs[("tsan", k)] = ([i], env, log_dir)
    for order in ("forward", "reverse", "seeded"):
        env = dict(os.environ, MGB_EMUL_ORDER=order, MGB_EMUL_SEED="4242",
                   MGB_LOUDNESS_DUMP=str(base / f"dump_{order}.bin"))
        jobs[(order, 0)] = (RACECHECK_IDS, env, str(base / order))
    with ThreadPoolExecutor(max_workers=8) as ex:
        futures = {key: ex.submit(run_group, *job) for key, job in jobs.items()}
        done = {key: f.result() + (jobs[key][2],) for key, f in futures.items()}
    return done, base


@pytest.mark.parametrize("k", range(len(RACECHECK_IDS)))
def test_meter_kernels_have_no_data_races(other_runs, k):
    from test_emul_racecheck import reports
    rc, out, _, log_dir = other_runs[0][("tsan", k)]
    n, first = reports(log_dir)
    assert n == 0, f"{n} ThreadSanitizer report(s) in {RACECHECK_IDS[k]}; the first:\n{first}"
    assert rc == 0, out


@pytest.mark.parametrize("order", ["reverse", "seeded"])
def test_meter_is_bit_identical_in_other_thread_orders(other_runs, order):
    done, base = other_runs
    for o in ("forward", order):
        rc, out, _, _ = done[(o, 0)]
        assert rc == 0, out
    forward = (base / "dump_forward.bin").read_bytes()
    assert len(forward) == len(DUMP_CASES) * C.sizeof(_native.LoudnessResult)
    assert (base / f"dump_{order}.bin").read_bytes() == forward
