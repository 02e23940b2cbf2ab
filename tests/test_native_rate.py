"""Native-rate masters without a GPU: the plan's tables, the native job (mgb_design_frequencies +
mgb_match_frequencies_native + stages 3-4 on the native plan) on the CPU emulator against the float64 restatement
(tests/native_rate_oracle.py), in true-peak mode, to a loudness target and with a reference profile, on poisoned
workspaces, under ThreadSanitizer and in other thread orders; the argument checks and Config's validation."""
import ctypes as C
import math
import os

import numpy as np
import pytest
from scipy import signal

from emul_harness import EmulPlan, aligned, aligned_copy, emul_lib, get_emul_plan, ptr  # (puts oracle/ on sys.path)
import loudness_target_oracle as lto
import native_rate_oracle as nro
import port
import true_peak_oracle as tpo
import matchering_b200 as mg
from matchering_b200 import _native, plan
from test_loudness import emul_params
from test_loudness_target import target_of
from test_reference_profile import emul_profile, spectra_of, header_of

TOL = 1e-5
FIR_TOL = 1e-13


def material(n, seed, rate):
    """Enveloped noise with a little tonal colour, so that the curve is not flat."""
    x = port.synth_target(n, seed).astype(np.float64)
    t = np.arange(n) / rate
    x += 0.2 * np.sin(2 * np.pi * 997.0 * t)[:, None]
    return np.ascontiguousarray(x.astype(np.float32))


def analysis_copy(x, rate, R=44100):
    """The analysis copy of the tests: any signal at R will do (the oracle takes it as an input), here a polyphase
    resampling of the native target."""
    g = math.gcd(R, rate)
    y = signal.resample_poly(x.astype(np.float64), R // g, rate // g, axis=0)
    return np.ascontiguousarray(y.astype(np.float32))


_NATIVE_PLANS = {}


def native_emul_plan(cfg, rate):
    key = (plan.config_key(cfg), rate)
    if key not in _NATIVE_PLANS:
        ep = EmulPlan(plan.native_config(cfg, rate))
        for name, arr in plan.native_tables(cfg, rate).items():
            ep.keep[name] = aligned_copy(arr)
            setattr(ep.struct, "d_" + name, ep.keep[name].ctypes.data)
        _NATIVE_PLANS[key] = ep
    return _NATIVE_PLANS[key]


def run_native(cfg, xn, rate, xa, r=None, blob=None, need=(True, True, True), pattern=None, operator=False,
               loudness_target=None):
    """Stage 1 and the design on the analysis copy xa at R, then the native job on xn at `rate`.  pattern "ff": every
    native buffer starts as 0xFF bytes.  -> dict(outs, fir (native), state, result)"""
    lib = emul_lib()
    ep, nep = get_emul_plan(cfg, operator), native_emul_plan(cfg, rate)
    T, N = len(xa), len(xn)
    L = _native.TrackLayout()
    if blob is None:
        _native.check(lib, lib.mgb_track_layout_init(C.byref(ep.struct), T, len(r), C.byref(L)))
    else:
        _native.check(lib, lib.mgb_track_layout_init_profiled(C.byref(ep.struct), T, C.byref(L)))
    NL = _native.TrackLayout()
    _native.check(lib, lib.mgb_track_layout_init_profiled(C.byref(nep.struct), N, C.byref(NL)))
    fill = (lambda a: a.fill(0xFF)) if pattern == "ff" else (lambda a: None)
    ws = aligned((L.workspace_bytes,), np.uint8)
    nws = aligned((NL.workspace_bytes,), np.uint8)
    fill(nws)
    ta, tn = aligned_copy(xa, np.float32), aligned_copy(xn, np.float32)
    res = aligned((N, 2), np.float32)
    fill(res.view(np.uint8))
    Fn = nep.tables.fft_size
    fir = aligned((2, Fn), np.float64)
    st = _native.TrackState()
    nst_raw = aligned((C.sizeof(_native.TrackState),), np.uint8)
    fill(nst_raw)
    nst = _native.TrackState.from_address(nst_raw.ctypes.data)
    P, LL, NP, NLL = C.byref(ep.struct), C.byref(L), C.byref(nep.struct), C.byref(NL)
    if blob is None:
        ref = aligned_copy(r, np.float32)
        _native.check(lib, lib.mgb_match_levels(P, LL, ptr(ta), ptr(ref), ptr(ws), C.byref(st), None))
    else:
        _native.check(lib, lib.mgb_match_levels_profiled(P, LL, ptr(ta), ptr(blob), ptr(ws), C.byref(st), None))
    _native.check(lib, lib.mgb_design_frequencies(P, LL, None, ptr(ws), C.byref(st), None))
    _native.check(lib, lib.mgb_match_frequencies_native(P, LL, ptr(ws), C.byref(st), NP, NLL, ptr(tn), ptr(res), ptr(fir),
                                                        ptr(nws), ptr(nst_raw), None))
    _native.check(lib, lib.mgb_correct_levels(NP, NLL, ptr(nws), ptr(nst_raw), None))
    outs = [aligned((N, 2), np.float32) if k else None for k in need]
    for o in outs:
        if o is not None:
            fill(o.view(np.uint8))
    report = None
    if loudness_target is None:
        _native.check(lib, lib.mgb_finalize(NP, NLL, ptr(res), *(ptr(o) if o is not None else None for o in outs),
                                            ptr(nws), ptr(nst_raw), None))
    else:
        _native.check(lib, lib.mgb_finalize(NP, NLL, ptr(res), None, *(ptr(o) if o is not None else None for o in outs[1:]),
                                            ptr(nws), ptr(nst_raw), None))
        meter = emul_params(rate)
        nbytes = int(lib.mgb_loudness_target_workspace_bytes(C.byref(meter), N))
        search = aligned((nbytes,), np.uint8)
        search.fill(0xFF)
        rep = aligned((C.sizeof(_native.LoudnessTargetReport),), np.uint8)
        _native.check(lib, lib.mgb_finalize_to_loudness(NP, NLL, C.byref(meter), C.byref(target_of(loudness_target)),
                                                        ptr(res), ptr(outs[0]), ptr(nws), ptr(search), nbytes, ptr(nst_raw),
                                                        ptr(rep), None))
        report = _native.LoudnessTargetReport.from_buffer_copy(bytes(rep))
    off = (C.c_int64 * 16)()
    _native.check(lib, lib.mgb_test_workspace_regions(NP, NLL, off))
    return dict(outs=[None if o is None else np.array(o) for o in outs], fir=np.array(fir), result=np.array(res),
                state=_native.TrackState.from_buffer_copy(bytes(nst_raw)), report=report,
                spectra=np.array(nws[off[8]:off[10]]),  # h_mid, h_side
                curves=analysis_curves(ep, L, ws))


def analysis_curves(ep, L, ws):
    """The smoothed curves the analysis design left in its workspace (design.cu: the parity-0 block of each channel,
    at 2 n_lin; the design blocks lie right before h_mid)."""
    off = (C.c_int64 * 16)()
    _native.check(emul_lib(), emul_lib().mgb_test_workspace_regions(C.byref(ep.struct), C.byref(L), off))
    t = ep.tables
    assert t.fft_size <= 8192  # (no float64 planes behind the vectors)
    stride = (3 * t.n_lin + 4 * t.n_log + t.fft_size + 16 + 31) // 32 * 32
    design = off[8] - (64 * stride + 255) // 256 * 256
    return [np.array(ws[design + 8 * (4 * ch * stride + 2 * t.n_lin):][:8 * t.n_lin].view(np.float64)) for ch in (0, 1)]


def assert_fir_follows_curves(got, F, rate):
    """h' within 1e-13 of the restatement's transplant and FIR applied to the device's own analysis curves."""
    for ch in (0, 1):
        want = nro.fir_from_curve(nro.transplant(got["curves"][ch], 44100, F, rate))
        err = float(np.abs(got["fir"][ch] - want).max())
        assert err < FIR_TOL, (ch, err)


def case(F, rate, seconds=2.0, seed=0, extra=0):
    cfg = mg.Config(max_piece_size=1.0, fft_size=F)
    n = int(seconds * rate) + extra
    xn = material(n, 10 + seed, rate)
    xa = analysis_copy(xn, rate)
    r = port.synth_reference(int(2.3 * 44100) + 77, 20 + seed)
    return cfg, xn, xa, r


def assert_close(got, want, tol, what):
    for k, (g, w) in enumerate(zip(got, want)):
        assert (g is None) == (w is None), (what, k)
        if g is not None:
            err = float(np.abs(g.astype(np.float64) - w).max())
            assert err < tol, (what, k, err)


# ---- the plan ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F,rate,want", [(4096, 22050, 2048), (4096, 32000, 4096), (4096, 48000, 4096),
                                         (4096, 88200, 8192), (4096, 96000, 8192), (4096, 192000, 16384),
                                         (512, 48000, 512), (512, 96000, 1024), (512, 192000, 2048)])
def test_native_fft_size(F, rate, want):
    cfg = mg.Config(fft_size=F)
    assert plan.native_fft_size(cfg, rate) == want == nro.native_fft_size(44100, F, rate)
    nc = plan.native_config(cfg, rate)
    assert (nc.internal_sample_rate, nc.fft_size) == (rate, want)
    assert nc.max_piece_size / rate == cfg.max_piece_size / 44100 and nc.preview_size / rate == cfg.preview_size / 44100
    assert (cfg.internal_sample_rate, cfg.fft_size) == (44100, F)  # the Config itself is untouched


@pytest.mark.parametrize("F,rate", [(4096, 352800), (4096, 384000), (512, 22050), (16384, 96000)])
def test_unsupported_native_fft_size_is_rejected(F, rate):
    with pytest.raises(plan.UnsupportedConfig):
        plan.native_fft_size(mg.Config(fft_size=F), rate)


def test_native_tables_follow_the_definition():
    cfg = mg.Config()
    for rate in (22050, 48000, 96000, 192000):
        t = plan.native_tables(cfg, rate)
        Fn = plan.native_fft_size(cfg, rate)
        idx, w = t["native_idx"], t["native_w"]
        assert idx.dtype == np.int32 and w.dtype == np.float64 and len(idx) == len(w) == Fn // 2 + 2
        f = np.arange(Fn // 2 + 1) * rate / Fn
        inside = f <= 0.9 * 22050
        np.testing.assert_array_equal(idx[:-1] >= 0, inside)
        pos = f[inside] * 4096 / 44100
        np.testing.assert_allclose(idx[:-1][inside] + w[:-1][inside], pos, rtol=0, atol=1e-12)
        assert np.all((w[:-1] >= 0) & (w[:-1] <= 1))
        np.testing.assert_array_equal(w[:-1][f >= 22050], 1.0)
        assert idx[-1] + w[-1] == pytest.approx(0.9 * 22050 * 4096 / 44100, abs=1e-12)


def test_short_native_target_is_rejected_before_anything_runs():
    cfg = mg.Config(max_piece_size=1.0)
    plan.native_check_length(cfg, 96000, 96000)  # one piece of 96000 frames >= 8192
    with pytest.raises(ValueError, match="too short"):
        plan.native_check_length(cfg, 96000, 8192)
    with pytest.raises(ValueError, match="too short"):  # pieces of 8191 frames
        plan.native_check_length(mg.Config(max_piece_size=0.1), 96000, 2 * 8191 + 1)


def test_config_native_rate():
    assert mg.Config().native_rate is False
    assert mg.Config(native_rate=True).native_rate is True
    with pytest.raises(AssertionError):
        mg.Config(native_rate=1)
    assert plan.config_key(mg.Config(native_rate=True)) == plan.config_key(mg.Config())


def test_surface():
    from test_cabi_and_surface import header_symbols
    for name in ("mgb_design_frequencies", "mgb_match_frequencies_native"):
        assert name in header_symbols() and name in _native.PROTOTYPES
    names = [f[0] for f in _native.Plan._fields_]
    assert names[-2:] == ["d_native_idx", "d_native_w"]
    from matchering_b200 import stages
    assert callable(stages.main_native)


# ---- the split design -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("operator", [False, True])
def test_split_design_is_match_frequencies_emulated(operator):
    """mgb_design_frequencies leaves what mgb_match_frequencies's design leaves, to the bit; the convolution after it
    is the rest of mgb_match_frequencies."""
    lib = emul_lib()
    cfg = mg.Config(max_piece_size=1.0, fft_size=512)
    t, r = port.synth_target(44100 * 2 + 33, 1), port.synth_reference(44100 * 2 - 11, 2)
    ep = get_emul_plan(cfg, operator)
    L = ep.layout(len(t), len(r))
    P, LL = C.byref(ep.struct), C.byref(L)
    tgt, ref = aligned_copy(t), aligned_copy(r)
    runs = []
    for split in (False, True):
        ws = aligned((L.workspace_bytes,), np.uint8)
        st = _native.TrackState()
        fir = aligned((2, 512), np.float64)
        res = aligned((len(t), 2), np.float32)
        _native.check(lib, lib.mgb_match_levels(P, LL, ptr(tgt), ptr(ref), ptr(ws), C.byref(st), None))
        if split:
            _native.check(lib, lib.mgb_design_frequencies(P, LL, ptr(fir), ptr(ws), C.byref(st), None))
        else:
            _native.check(lib, lib.mgb_match_frequencies(P, LL, ptr(tgt), ptr(res), ptr(fir), ptr(ws), C.byref(st), None))
        runs.append((bytes(st), np.array(fir), np.array(ws)))
    off = (C.c_int64 * 16)()
    _native.check(lib, lib.mgb_test_workspace_regions(P, LL, off))
    (s0, f0, w0), (s1, f1, w1) = runs
    np.testing.assert_array_equal(f0, f1)
    a, b = _native.TrackState.from_buffer_copy(s0), _native.TrackState.from_buffer_copy(s1)
    for name, _ in _native.TrackState._fields_:
        if name not in ("conv_peak_bits", "conv_precise"):  # what the convolution measures
            va, vb = getattr(a, name), getattr(b, name)
            assert (list(va) == list(vb)) if name == "correction" else va == vb, name
    # both FIR spectra (regions 8 and 9 of mgb_test_workspace_regions: h_mid, h_side)
    np.testing.assert_array_equal(w0[off[8]:off[10]], w1[off[8]:off[10]])


# ---- against the oracle -----------------------------------------------------------------------------------------------
CASES = [(4096, rate) for rate in (22050, 32000, 48000, 88200, 96000, 192000)] + \
        [(512, rate) for rate in (32000, 48000, 88200, 96000, 192000)]


@pytest.mark.parametrize("F,rate", CASES)
def test_native_job_matches_oracle_emulated(F, rate):
    cfg, xn, xa, r = case(F, rate, extra=rate % 997)
    got = run_native(cfg, xn, rate, xa, r)
    tr = {}
    want = nro.main(xn, xa, r, cfg, rate, True, True, True, trace=tr)
    assert_fir_follows_curves(got, F, rate)
    for ch, name in enumerate(("mid", "side")):  # (the curves themselves: float32 spectra, as at R)
        err = float(np.abs(got["fir"][ch] - tr["firs"][name]).max())
        assert err < 1e-7, (name, err)
    assert_close(got["outs"], want, TOL, "outputs")
    assert got["state"].steps_done == cfg.rms_correction_steps


@pytest.mark.parametrize("n", [96000 + 8192, 2 * 96000 + 1, 2 * 96000 + 8191])
def test_lengths_around_pieces_and_frames_emulated(n):
    """Tracks just past a piece and a frame edge at 96 kHz (pieces of one second, F' = 8192)."""
    rate = 96000
    cfg = mg.Config(max_piece_size=1.0)
    xn = material(n, 31, rate)
    xa = analysis_copy(xn, rate)
    r = port.synth_reference(44100 * 2 + 5, 32)
    got = run_native(cfg, xn, rate, xa, r)
    want = nro.main(xn, xa, r, cfg, rate, True, True, True)
    assert_close(got["outs"], want, TOL, n)


def test_true_peak_mode_emulated():
    rate = 96000
    cfg, xn, xa, r = case(4096, rate, seed=3)
    cfg = mg.Config(max_piece_size=1.0, true_peak=True)
    got = run_native(cfg, xn, rate, xa, r)
    tr = {}
    nro.main(xn, xa, r, cfg, rate, False, False, False, trace=tr)
    nc = plan.native_config(cfg, rate)
    s = tr["pre_limiter"]
    limited = tpo.limit(s, nc) * tr["final_coef"]
    normalized = s / max(nc.min_value, float(tpo.true_peak_detector(s, rate).max()) / nc.threshold)
    assert_close(got["outs"], [limited, s, normalized], TOL, "true peak")


def test_loudness_target_emulated():
    rate = 48000
    cfg, xn, xa, r = case(4096, rate, seconds=3.0, seed=4)
    cfg = mg.Config(max_piece_size=1.0, loudness_target=-14.0)
    got = run_native(cfg, xn, rate, xa, r, loudness_target=-14.0)
    tr = {}
    nro.main(xn, xa, r, cfg, rate, False, False, False, trace=tr)
    want = lto.search(tr["pre_limiter"], plan.native_config(cfg, rate), -14.0)
    assert got["report"].status == want["status"] == lto.REACHED
    assert float(np.abs(got["outs"][0] - want["output"]).max()) < TOL
    assert abs(lto.integrated(got["outs"][0].astype(np.float64), rate) + 14.0) <= lto.TOLERANCE


@pytest.mark.parametrize("rate", [48000, 96000])
def test_reference_profile_emulated(rate):
    """A native job against a profile is the paired native job, output for output, and so within 1e-5 of the oracle."""
    cfg, xn, xa, r = case(4096, rate, seed=5)
    blob, _ = emul_profile(cfg, r)
    got = run_native(cfg, xn, rate, xa, blob=blob)
    paired = run_native(cfg, xn, rate, xa, r)
    for g, p in zip(got["outs"], paired["outs"]):
        np.testing.assert_array_equal(g, p)
    np.testing.assert_array_equal(got["fir"], paired["fir"])
    h = header_of(blob)
    sp = spectra_of(blob, cfg.fft_size // 2 + 1)
    want = nro.main(xn, xa, None, cfg, rate, True, True, True,
                    profile=(sp[0], sp[1], h.final_amplitude_coef, h.reference_match_rms))
    assert_close(got["outs"], want, TOL, "profile")


def test_band_limited_target_is_never_boosted_above_the_analysed_band_emulated():
    """A target low-passed at 2 kHz against bright noise: gains of tens near the top of the analysed band,
    none above 1 from R/2 on."""
    rate = 96000
    cfg = mg.Config(max_piece_size=1.0)
    n = 2 * rate + 17
    b, a = signal.butter(8, 2000, fs=rate)
    xn = np.ascontiguousarray(signal.lfilter(b, a, material(n, 41, rate).astype(np.float64), axis=0).astype(np.float32))
    xa = analysis_copy(xn, rate)
    r = port.synth_target(44100 * 2 + 3, 42, kind="plain")  # white: bright
    got = run_native(cfg, xn, rate, xa, r)
    tr = {}
    want = nro.main(xn, xa, r, cfg, rate, True, True, True, trace=tr)
    Fn = plan.native_fft_size(cfg, rate)
    f = np.arange(Fn // 2 + 1) * rate / Fn
    for ch, name in enumerate(("mid", "side")):
        s = tr["curves"][name]
        assert s[(f > 15000) & (f <= 0.9 * 22050)].max() > 10  # the analysed band's top is strongly boosted
        assert s[f >= 22050].max() <= 1.0
        dev = nro.transplant(got["curves"][ch], 44100, cfg.fft_size, rate)
        assert dev[f >= 22050].max() <= 1.0
    assert_fir_follows_curves(got, cfg.fft_size, rate)
    # the limited and normalised outputs within 1e-5; the un-limited one peaks far above full scale here (gains of
    # tens over the whole upper band), so relative to its peak -- as the ordinary job on this material
    assert_close([got["outs"][0], got["outs"][2]], [want[0], want[2]], TOL, "band-limited")
    peak = float(np.abs(want[1]).max())
    assert float(np.abs(got["outs"][1] - want[1]).max()) < TOL * max(1.0, peak)


def test_poisoned_native_workspaces_change_nothing_emulated():
    cfg, xn, xa, r = case(512, 88200, seed=6)
    clean = run_native(cfg, xn, 88200, xa, r)
    dirty = run_native(cfg, xn, 88200, xa, r, pattern="ff")
    for a, b in zip(clean["outs"], dirty["outs"]):
        np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(clean["fir"], dirty["fir"])
    assert bytes(clean["state"]) == bytes(dirty["state"])


# ---- argument checks ---------------------------------------------------------------------------------------------------
def test_argument_errors_emulated():
    lib = emul_lib()
    cfg = mg.Config(max_piece_size=1.0, fft_size=512)
    rate = 96000
    ep, nep = get_emul_plan(cfg), native_emul_plan(cfg, rate)
    t, r = port.synth_target(44100 * 2, 1), port.synth_reference(44100 * 2, 2)
    L = ep.layout(len(t), len(r))
    N = 2 * rate
    NL = _native.TrackLayout()
    _native.check(lib, lib.mgb_track_layout_init_profiled(C.byref(nep.struct), N, C.byref(NL)))
    ws, nws = aligned((L.workspace_bytes,), np.uint8), aligned((NL.workspace_bytes,), np.uint8)
    st, nst = _native.TrackState(), aligned((C.sizeof(_native.TrackState),), np.uint8)
    tn, res = aligned((N, 2), np.float32), aligned((N, 2), np.float32)

    def call(p=ep.struct, np_=nep.struct, nl=NL, layout=L, tgt=None):
        return lib.mgb_match_frequencies_native(C.byref(p), C.byref(layout), ptr(ws), C.byref(st), C.byref(np_),
                                                C.byref(nl), ptr(tn) if tgt is None else tgt, ptr(res), None, ptr(nws),
                                                ptr(nst), None)

    inv = _native.MGB_ERR_INVALID
    same = _native.Plan.from_buffer_copy(bytes(nep.struct))
    same.sample_rate = 44100
    assert call(np_=same) == inv and b"differ" in lib.mgb_last_error_string()
    wrong = _native.Plan.from_buffer_copy(bytes(nep.struct))
    wrong.sample_rate = 48000  # 48 kHz wants F' = 512, the plan has 1024
    assert call(np_=wrong) == inv and b"fft_size" in lib.mgb_last_error_string()
    bare = _native.Plan.from_buffer_copy(bytes(nep.struct))
    bare.d_native_idx = None
    assert call(np_=bare) == inv and b"tables" in lib.mgb_last_error_string()
    big = _native.Plan.from_buffer_copy(bytes(nep.struct))
    big.fft_size, big.n_lin = 32768, 16385
    assert call(np_=big) == _native.MGB_ERR_UNSUPPORTED
    paired = nep.layout(N, N)
    assert call(nl=paired) == inv and b"profiled" in lib.mgb_last_error_string()
    short = _native.TrackLayout.from_buffer_copy(bytes(NL))
    short.target_frames, short.target_piece = 1024, 1024
    assert call(nl=short) == inv
    assert call(tgt=C.c_void_p(ptr(tn).value + 4)) == inv and b"aligned" in lib.mgb_last_error_string()


# ---- the kernel under ThreadSanitizer and in other thread orders -------------------------------------------------------
HERE = "tests/test_native_rate.py::"
DUMP_ID = HERE + "test_dump_for_thread_orders_emulated"


def test_dump_for_thread_orders_emulated():
    """Two small native jobs (F' = 512 and 1024); with MGB_NATIVE_DUMP set, what the native design writes -- both FIRs,
    their spectra on the convolution grid and their peaks -- goes to that file."""
    raws = b""
    for rate in (48000, 96000):
        cfg = mg.Config(max_piece_size=0.5, fft_size=512)
        n = rate + 333
        xn = material(n, 51, rate)
        xa = analysis_copy(xn, rate)
        r = port.synth_reference(44100 + 77, 52)
        got = run_native(cfg, xn, rate, xa, r)
        st = got["state"]
        raws += got["fir"].tobytes() + got["spectra"].tobytes() + np.float32([st.fir_peak_mid_bits, st.fir_peak_side_bits]).tobytes()
    if os.environ.get("MGB_NATIVE_DUMP"):
        with open(os.environ["MGB_NATIVE_DUMP"], "wb") as f:
            f.write(raws)


@pytest.fixture(scope="module")
def other_runs(tmp_path_factory):
    from concurrent.futures import ThreadPoolExecutor

    import build_emul
    from test_emul_racecheck import run_group, tsan_env
    build_emul.build(racecheck=True)
    build_emul.build()
    base = tmp_path_factory.mktemp("native_racecheck")
    jobs = {}
    env = tsan_env(str(base / "tsan"))
    env["MGB_EMUL_BUILD"] = "racecheck"
    jobs["tsan"] = ([DUMP_ID], env, str(base / "tsan"))
    for order in ("forward", "reverse", "seeded"):
        env = dict(os.environ, MGB_EMUL_ORDER=order, MGB_EMUL_SEED="4242", MGB_NATIVE_DUMP=str(base / f"dump_{order}.bin"))
        jobs[order] = ([DUMP_ID], env, str(base / order))
    with ThreadPoolExecutor(max_workers=4) as ex:
        futures = {key: ex.submit(run_group, *job) for key, job in jobs.items()}
        done = {key: f.result() + (jobs[key][2],) for key, f in futures.items()}
    return done, base


def test_native_design_has_no_data_races(other_runs):
    from test_emul_racecheck import reports
    rc, out, _, log_dir = other_runs[0]["tsan"]
    n, first = reports(log_dir)
    assert n == 0, f"{n} ThreadSanitizer report(s); the first:\n{first}"
    assert rc == 0, out


@pytest.mark.parametrize("order", ["reverse", "seeded"])
def test_native_job_is_bit_identical_in_other_thread_orders(other_runs, order):
    done, base = other_runs
    for o in ("forward", order):
        rc, out, _, _ = done[o]
        assert rc == 0, out
    forward = (base / "dump_forward.bin").read_bytes()
    assert len(forward) > 0
    assert (base / f"dump_{order}.bin").read_bytes() == forward
