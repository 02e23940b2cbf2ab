"""Reference profiles (mgb_analyze_reference, mgb_match_levels_profiled, matchering_b200/profile.py): a job whose
reference comes from a profile must be bit-identical to the job that takes the reference's samples -- outputs, the
whole mgb_track_state and the FIR -- and the profile itself must hold what the float64 oracle computes for the
reference side.  Emulator tests run on the CPU; tests/test_reference_profile_gpu.py checks the same at full size on the
device, where stage 3's float64 atomic sums keep even a paired job from repeating bit for bit (assert_identical)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import port
from emul_harness import aligned, aligned_copy, emul_lib, get_emul_plan, ptr, run_pipeline
from matchering_b200 import _native

U = 2.0 ** -24
POISONS = ["ff", "7f", "random"]
HEADER = C.sizeof(_native.ReferenceProfileHeader)


def a256(n):
    return (n + 255) // 256 * 256


def poison(n, pattern, seed=0):
    if pattern is None:
        return np.zeros(n, np.uint8)
    if pattern == "ff":
        return np.full(n, 0xFF, np.uint8)
    if pattern == "7f":
        return np.full(n, 0x7F, np.uint8)
    return np.random.default_rng(4321 + seed).integers(0, 256, n, dtype=np.uint8)


def ebuf(nbytes, pattern, seed=0):
    a = aligned((nbytes,), np.uint8)
    a[...] = poison(nbytes, pattern, seed)
    return a


# ---- emulator drivers ------------------------------------------------------------------------------------------------
def emul_profile(cfg, r, operator=False, pattern=None):
    """mgb_analyze_reference on the emulator -> (blob uint8, reference workspace)."""
    lib, ep = emul_lib(), get_emul_plan(cfg, operator)
    R = len(r)
    nb = int(lib.mgb_reference_workspace_bytes(C.byref(ep.struct), R))
    pb = int(lib.mgb_reference_profile_bytes(C.byref(ep.struct)))
    assert nb > 0 and pb == HEADER + 16 * (cfg.fft_size // 2 + 1)
    ws, blob = ebuf(nb, pattern, 1), ebuf(pb, pattern, 2)
    ref = aligned_copy(r, np.float32)
    _native.check(lib, lib.mgb_analyze_reference(C.byref(ep.struct), ptr(ref), R, ptr(ws), nb, ptr(blob), None))
    return blob, ws


def header_of(blob):
    return _native.ReferenceProfileHeader.from_buffer_copy(bytes(blob[:HEADER]))


def spectra_of(blob, n_lin):
    return np.frombuffer(bytes(blob[HEADER:HEADER + 16 * n_lin]), np.float64).reshape(2, n_lin)


def profiled_layout(lib, ep, T):
    L = _native.TrackLayout()
    _native.check(lib, lib.mgb_track_layout_init_profiled(C.byref(ep.struct), T, C.byref(L)))
    return L


def run_profiled(cfg, t, blob, operator=False, pattern=None, clobber_profile=False):
    """The four stage calls with stage 1 from the profile; buffers filled with `pattern` first.  clobber_profile:
    the caller's profile buffer is overwritten once stage 1 has been issued (it has been copied by then)."""
    lib, ep = emul_lib(), get_emul_plan(cfg, operator)
    T = len(t)
    L = profiled_layout(lib, ep, T)
    assert (L.reference_frames, L.reference_piece, L.reference_divisions, L.reference_slots) == (0, 0, 0, 0)
    ws = ebuf(L.workspace_bytes, pattern, 3)
    tgt = aligned_copy(t, np.float32)
    result = ebuf(T * 8, pattern, 4).view(np.float32).reshape(T, 2)
    fir = ebuf(16 * cfg.fft_size, pattern, 5).view(np.float64).reshape(2, cfg.fft_size)
    state = _native.TrackState.from_buffer_copy(bytes(poison(C.sizeof(_native.TrackState), pattern, 6)))
    P, LL = C.byref(ep.struct), C.byref(L)
    _native.check(lib, lib.mgb_match_levels_profiled(P, LL, ptr(tgt), ptr(blob), ptr(ws), C.byref(state), None))
    if clobber_profile:
        blob[...] = poison(blob.nbytes, "random", 7)
    _native.check(lib, lib.mgb_match_frequencies(P, LL, ptr(tgt), ptr(result), ptr(fir), ptr(ws), C.byref(state), None))
    _native.check(lib, lib.mgb_correct_levels(P, LL, ptr(ws), C.byref(state), None))
    outs = [ebuf(T * 8, pattern, 8 + k).view(np.float32).reshape(T, 2) for k in range(3)]
    _native.check(lib, lib.mgb_finalize(P, LL, ptr(result), *(ptr(o) for o in outs), ptr(ws), C.byref(state), None))
    return outs, state, np.array(fir)


# mgb_track_state fields stages 1 and 2 write: exact whatever order the threads run in
EXACT_FIELDS = ["reference_peak", "final_amplitude_coef", "target_match_rms", "reference_match_rms", "rms_coefficient",
                "target_loud_pieces", "reference_loud_pieces", "fir_peak_mid_bits", "fir_peak_side_bits",
                "conv_precise", "conv_peak_bits"]
SEEDED = os.environ.get("MGB_EMUL_ORDER") == "seeded"
REPEAT_TOL = 1e-6  # tests/test_workspace_reuse.py: two runs of one job on the device, relative to max(1, peak)


def assert_identical(got, want, what=""):
    """Bit-identical outputs, state and FIR.  Under a random thread order (MGB_EMUL_ORDER=seeded, a different order in
    every launch) stage 3's float64 atomic sums are added in a different order in the two jobs, as on the device:
    then the stage 1-2 fields and the FIR stay exact and the outputs keep the device's repeat bound."""
    (outs, st, fir), (w_outs, w_st, w_fir) = got, want
    assert np.array_equal(fir, w_fir), (what, "fir")
    if SEEDED:
        for f in EXACT_FIELDS:
            assert getattr(st, f) == getattr(w_st, f), (what, f)
        for k, (a, b) in enumerate(zip(outs, w_outs)):
            e = float(np.abs(a.astype(np.float64) - b).max()) / max(1.0, float(np.abs(b).max()))
            assert e <= REPEAT_TOL, (what, "output", k, e)
        return
    for k, (a, b) in enumerate(zip(outs, w_outs)):
        assert np.array_equal(a, b), (what, "output", k, float(np.abs(a - b).max()))
    assert bytes(st) == bytes(w_st), (what, "state")


def paired(cfg, t, r, operator=False):
    outs, st, fir, _, L = run_pipeline(cfg, t, r, need=(True, True, True), operator=operator)
    return (outs, st, np.array(fir)), L


# ---- material ----------------------------------------------------------------------------------------------------
def _mono(n):
    mid = port.synth_target(n, 71)[:, :1]
    return np.ascontiguousarray(np.concatenate([mid, mid], axis=1))


def _quiet():
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pipeline_quiet_reference.npz"))
    return g["target"], g["reference"], float(g["max_piece_size_s"])


def _coloured():
    import test_coloured_material as tc
    t, r = tc.material("lp2k_bright", False)
    return t, r


# name -> (config arguments, target, reference, smoothing operator)
def case(name):
    T = 30000
    syn_t, syn_r = (lambda n: port.synth_target(n, 1)), (lambda n: port.synth_reference(n, 2))
    base = dict(fft_size=1024, max_piece_size=0.3)
    if name == "f512":
        return dict(fft_size=512, max_piece_size=0.2), syn_t(20011), syn_r(18007), False
    if name == "f512_operator":
        return dict(fft_size=512, max_piece_size=0.2), syn_t(20011), syn_r(18007), True
    if name == "f1024":
        return base, syn_t(T), syn_r(28000), False
    if name == "f1024_operator":
        return base, syn_t(T), syn_r(28000), True
    if name == "f2048_4F":  # pieces of more than 3F samples: the 4F-frame convolution
        return dict(fft_size=2048, max_piece_size=0.25), syn_t(30011), syn_r(26011), False
    if name == "f2048_4F_operator":
        return dict(fft_size=2048, max_piece_size=0.25), syn_t(30011), syn_r(26011), True
    if name == "f4096":
        return dict(fft_size=4096, max_piece_size=0.5), syn_t(60011), syn_r(56011), False
    if name == "f4096_operator":
        return dict(fft_size=4096, max_piece_size=0.5), syn_t(60011), syn_r(56011), True
    if name == "f16384":
        n = 16384 * 6 + 777
        return dict(fft_size=16384, max_piece_size=1.0), syn_t(n), syn_r(n - 5003), False
    if name == "lowess_it2":
        return dict(base, lowess_it=2), syn_t(T), syn_r(28000), False
    if name == "steps0":
        return dict(base, rms_correction_steps=0), syn_t(T), syn_r(28000), False
    if name == "steps1":
        return dict(base, rms_correction_steps=1), syn_t(T), syn_r(28000), False
    if name == "quiet_reference":
        t, r, piece_s = _quiet()
        return dict(max_piece_size=piece_s), t, r, False
    if name == "reference_one_piece":
        return base, syn_t(T), syn_r(9000), False
    if name == "reference_40_pieces":  # more pieces than lanes: the warps' loops over pieces go round twice
        return dict(fft_size=512, max_piece_size=0.02), syn_t(20011), syn_r(35700), False
    if name == "reference_longer":
        return base, syn_t(T), syn_r(2 * T + 17), False
    if name == "reference_shorter":
        return base, syn_t(T), syn_r(T // 2 + 5), False
    if name == "mono_target":
        return base, _mono(T), syn_r(28000), False
    if name == "lp2k_bright":  # coloured: the convolution takes convolve_precise_kernel
        t, r = _coloured()
        return dict(fft_size=4096, max_piece_size=1.0), t, r, False
    raise KeyError(name)


IDENTITY_CASES = ["f512", "f512_operator", "f1024", "f1024_operator", "f2048_4F", "f2048_4F_operator", "f4096",
                  "f4096_operator", "f16384", "lowess_it2", "steps0", "steps1", "quiet_reference", "reference_one_piece",
                  "reference_40_pieces", "reference_longer", "reference_shorter", "mono_target", "lp2k_bright"]
# the race-checked subset (ThreadSanitizer is ~20x slower)
RACECHECK_CASES = ["f512", "reference_40_pieces", "steps0"]


@pytest.mark.parametrize("name", IDENTITY_CASES)
def test_profiled_job_is_bit_identical_to_paired_emulated(name):
    kw, t, r, operator = case(name)
    cfg = port.OracleConfig(**kw)
    want, L = paired(cfg, t, r, operator)
    blob, _ = emul_profile(cfg, r, operator)
    got = run_profiled(cfg, t, blob, operator)
    assert_identical(got, want, name)
    h = header_of(blob)
    assert (h.reference_divisions, h.reference_piece, h.reference_frames) == (L.reference_divisions, L.reference_piece, len(r))
    if name == "quiet_reference":
        assert h.final_amplitude_coef < 1.0 and got[1].limiter_engaged == 0
    if name == "reference_one_piece":
        assert h.reference_divisions == 1
    if name == "reference_40_pieces":
        assert h.reference_divisions > 32
    if name == "lp2k_bright":
        assert got[1].conv_precise == 1


@pytest.mark.parametrize("name", ["f1024", "reference_40_pieces", "quiet_reference", "f4096"])
def test_profile_matches_oracle_emulated(name):
    kw, t, r, operator = case(name)
    cfg = port.OracleConfig(**kw)
    blob, ws = emul_profile(cfg, r, operator)
    h = header_of(blob)
    F, HB = cfg.fft_size, cfg.fft_size // 2 + 1
    tr = {}
    port.main(np.asarray(t, np.float64), np.asarray(r, np.float32).astype(np.float64), cfg, True, False, False, trace=tr)
    ra, coef = tr["reference"], tr["final_coef"]
    assert h.version == _native.MGB_REFERENCE_PROFILE_VERSION
    assert (h.sample_rate, h.fft_size, h.n_lin) == (cfg.internal_sample_rate, F, HB)
    assert (h.max_piece_size, h.threshold, h.min_value) == (cfg.max_piece_size, cfg.threshold, cfg.min_value)
    assert h.reference_peak == float(np.abs(np.asarray(r, np.float32)).max())
    assert (h.reference_divisions, h.reference_piece) == (ra["divisions"], ra["piece"])
    assert h.reference_loud_pieces == int(ra["mask"].sum())
    assert abs(h.final_amplitude_coef - coef) <= 1e-7 * coef
    assert abs(h.reference_match_rms - ra["match_rms"]) <= 1e-7 * ra["match_rms"]
    # the mask, from the reference workspace (spectra, sums of squares, peaks, then the mask)
    L = get_emul_plan(cfg, operator).layout(len(t), len(r))
    items = L.reference_divisions * L.reference_slots
    off = a256(items * 2 * HB * 4) + a256(items * 8) + a256((items + 1) * 4)
    assert np.array_equal(ws[off:off + ra["divisions"]].astype(bool), ra["mask"])
    # spectra: the float32-FFT bound of test_stage_parity.check_analysis, summed over the loud pieces and scaled like
    # the mean (the oracle's normalised reference is r / coef)
    from test_stage_parity import frame_sums
    D, P = ra["divisions"], ra["piece"]
    mid, side = port.mid_side(np.asarray(r, np.float32).astype(np.float64))
    fpp = P // F
    _, norm_m = frame_sums(mid, P, D, F)
    _, norm_s = frame_sums(side, P, D, F)
    slots = L.reference_slots
    bound_piece = (4 * np.log2(F) + -(-fpp // slots)) * U * (norm_m + norm_s)
    scale = coef * h.reference_loud_pieces * fpp * F
    bound = bound_piece[ra["mask"]].sum() / scale
    spectra = spectra_of(blob, HB)
    for ch, name_ch in ((0, "mid"), (1, "side")):
        want = tr["avgs"][name_ch][1]
        err = np.abs(spectra[ch] - want)
        assert np.all(err <= bound + 1e-12 * np.abs(want)), (name_ch, float(err.max()), bound)


def test_profile_reused_under_other_target_configs_emulated():
    """A profile made under the default Config serves a Config that differs in the limiter's attack and hold,
    rms_correction_steps and the LOWESS fraction: bit-identical to the paired job under that Config."""
    kw, t, r, _ = case("f1024")
    blob, _ = emul_profile(port.OracleConfig(**kw), r)
    other = port.OracleConfig(**kw, rms_correction_steps=2, lowess_frac=0.05,
                              limiter=port.OracleLimiterConfig(attack=3.0, hold=5.0))
    want, _ = paired(other, t, r)
    assert_identical(run_profiled(other, t, blob), want)


def _plan_copy(cfg, **fields):
    s = _native.Plan()
    C.pointer(s)[0] = get_emul_plan(cfg).struct
    for k, v in fields.items():
        setattr(s, k, v)
    return s


@pytest.mark.parametrize("field,value", [("sample_rate", 48000), ("fft_size", 2048), ("n_lin", 1025),
                                         ("max_piece_size", 13231.0), ("threshold", 0.99), ("min_value", 1e-7),
                                         ("version", 2)])
def test_profile_check_rejects_every_fingerprint_field(field, value):
    lib = emul_lib()
    kw, _, r, _ = case("f1024")
    cfg = port.OracleConfig(**kw)
    blob, _ = emul_profile(cfg, r)
    h = header_of(blob)
    assert lib.mgb_reference_profile_check(C.byref(get_emul_plan(cfg).struct), C.byref(h)) == _native.MGB_OK
    setattr(h, field, value)
    assert lib.mgb_reference_profile_check(C.byref(get_emul_plan(cfg).struct), C.byref(h)) == _native.MGB_ERR_INVALID
    assert field.encode() in lib.mgb_last_error_string()
    # the Python side names the field too, before any device work
    from matchering_b200.profile import ReferenceProfile
    raw = bytes(blob)
    fields = {k: getattr(h, k) for k, _ in _native.ReferenceProfileHeader._fields_ if k != "reserved"}
    fields[field] = value
    if field in ("version", "n_lin"):  # not a Config field: the profile itself is refused
        with pytest.raises(ValueError):
            ReferenceProfile(fields, spectra_of(np.frombuffer(raw, np.uint8), h.n_lin))
        return
    prof = ReferenceProfile(fields, spectra_of(np.frombuffer(raw, np.uint8), h.n_lin))
    with pytest.raises(ValueError, match=re.escape(field)):
        prof.check_config(cfg)


def test_layout_kinds_and_pointer_checks_are_enforced():
    lib = emul_lib()
    kw, t, r, _ = case("f1024")
    cfg = port.OracleConfig(**kw)
    ep = get_emul_plan(cfg)
    P = C.byref(ep.struct)
    blob, _ = emul_profile(cfg, r)
    Lp, Lq = profiled_layout(lib, ep, len(t)), ep.layout(len(t), len(r))
    ws = aligned((max(Lp.workspace_bytes, Lq.workspace_bytes) + 64,), np.uint8)
    tgt, ref = aligned_copy(t, np.float32), aligned_copy(r, np.float32)
    st = _native.TrackState()
    inv = _native.MGB_ERR_INVALID
    assert lib.mgb_match_levels_profiled(P, C.byref(Lq), ptr(tgt), ptr(blob), ptr(ws), C.byref(st), None) == inv
    assert lib.mgb_match_levels(P, C.byref(Lp), ptr(tgt), ptr(ref), ptr(ws), C.byref(st), None) == inv
    assert lib.mgb_match_levels_profiled(P, C.byref(Lp), ptr(tgt), None, ptr(ws), C.byref(st), None) == inv
    assert lib.mgb_match_levels_profiled(P, C.byref(Lp), ptr(tgt), ptr(blob) .value + 8, ptr(ws), C.byref(st), None) == inv
    assert lib.mgb_match_levels_profiled(P, C.byref(Lp), ptr(tgt), ptr(blob), ptr(ws).value + 4, C.byref(st), None) == inv
    nb = int(lib.mgb_reference_workspace_bytes(P, len(r)))
    rws = aligned((nb,), np.uint8)
    assert lib.mgb_analyze_reference(P, ptr(ref), len(r), ptr(rws), nb, None, None) == inv
    assert lib.mgb_analyze_reference(P, ptr(ref), len(r), ptr(rws), nb, ptr(blob).value + 8, None) == inv
    assert lib.mgb_analyze_reference(P, ptr(ref).value + 4, len(r), ptr(rws), nb, ptr(blob), None) == inv
    assert lib.mgb_analyze_reference(P, ptr(ref), len(r), ptr(rws), nb - 1, ptr(blob), None) == _native.MGB_ERR_WORKSPACE
    assert lib.mgb_analyze_reference(P, ptr(ref), cfg.fft_size, ptr(rws), nb, ptr(blob), None) == inv
    assert lib.mgb_reference_workspace_bytes(P, cfg.fft_size) < 0
    assert lib.mgb_reference_profile_check(P, None) == inv
    # a paired layout's workspace is the same as before profiles existed: a profiled one drops the reference regions
    # and adds the profile behind everything else
    regions = (C.c_int64 * 16)()
    _native.check(lib, lib.mgb_test_workspace_regions(P, C.byref(Lp), regions))
    assert Lp.workspace_bytes < Lq.workspace_bytes


def _profile_object(blob):
    from matchering_b200.profile import profile_from_bytes
    return profile_from_bytes(bytes(blob))


def test_save_load_round_trip_and_corrupt_files(tmp_path):
    from matchering_b200.profile import ReferenceProfile
    kw, t, r, _ = case("f1024")
    cfg = port.OracleConfig(**kw)
    blob, _ = emul_profile(cfg, r)
    prof = _profile_object(blob)
    path = tmp_path / "album.npz"
    prof.save(path)
    back = ReferenceProfile.load(path)
    assert back.to_bytes() == bytes(blob)
    assert back.spectra.dtype == np.float64 and back.spectra.shape == (2, 513) and not back.spectra.flags.writeable
    assert (back.frames, back.divisions, back.loud_pieces) == (len(r), prof.divisions, prof.loud_pieces)
    # the loaded profile drives a bit-identical job
    want, _ = paired(cfg, t, r)
    assert_identical(run_profiled(cfg, t, aligned_copy(np.frombuffer(back.to_bytes(), np.uint8))), want)
    # truncated, garbage, wrong tag, wrong version, wrong spectra shape and dtype
    raw = path.read_bytes()
    (tmp_path / "short.npz").write_bytes(raw[: len(raw) // 2])
    (tmp_path / "junk.npz").write_bytes(b"not a profile at all" * 10)
    z = dict(np.load(path, allow_pickle=False))
    bad = {"tag": dict(z, format=np.array("something else")), "version": dict(z, version=np.array(7, np.int64)),
           "shape": dict(z, spectra=z["spectra"][:, :-1]), "dtype": dict(z, spectra=z["spectra"].astype(np.float32)),
           "field_dtype": dict(z, reference_peak=np.array(1, np.int64)),
           "missing": {k: v for k, v in z.items() if k != "reference_match_rms"}}
    for name, d in bad.items():
        with open(tmp_path / f"{name}.npz", "wb") as f:
            np.savez(f, **d)
    for name in ["short", "junk", *bad]:
        with pytest.raises(ValueError):
            ReferenceProfile.load(tmp_path / f"{name}.npz")


@pytest.mark.parametrize("pattern", POISONS)
def test_profiled_job_on_poisoned_buffers_emulated(pattern):
    """Every buffer of a profiled job starts as poison (NaN / -1 / random bytes): the workspace, the result, the
    outputs, the FIR, the state; the reference's analysis workspace and the profile buffer too; and the caller's
    profile is overwritten once stage 1 is issued.  Bit-identical to the clean paired job."""
    kw, t, r, _ = case("f1024")
    cfg = port.OracleConfig(**kw)
    want, _ = paired(cfg, t, r)
    blob, _ = emul_profile(cfg, r, pattern=pattern)
    assert_identical(run_profiled(cfg, t, blob, pattern=pattern, clobber_profile=True), want, pattern)


def _pcm16(x):
    return np.clip(np.rint(np.asarray(x, np.float64) * 32767.0), -32768, 32767).astype(np.int16)


@pytest.mark.parametrize("pcm", [False, True])
def test_mixed_paired_and_profiled_batch_on_poisoned_pipeline_emulated(pcm):
    """mgb_pipeline_* created with poison_alloc, fed paired and profiled submissions in turn (slots reused by the
    other kind), float32 or PCM16: each result is the clean single-track one."""
    lib = emul_lib()
    kw, _, r, _ = case("f1024")
    cfg = port.OracleConfig(**kw)
    ep = get_emul_plan(cfg)
    lengths = [20011, 16007, 19003, 14009]
    targets = [port.synth_target(n, 40 + k) for k, n in enumerate(lengths)]
    r = r[:18000]
    if pcm:  # what mgb_pcm_decode makes of the int16 buffers: exact in float32
        targets_pcm, r_pcm = [_pcm16(x) for x in targets], _pcm16(r)
        targets = [(q.astype(np.float64) / 32768.0).astype(np.float32) for q in targets_pcm]
        r = (r_pcm.astype(np.float64) / 32768.0).astype(np.float32)
    blob, _ = emul_profile(cfg, r)
    # the shortest reference the pipeline accepts: every profiled job's workspace must still fit
    _native.check(lib, lib.mgb_set_option(b"poison_alloc", 1))
    h = C.c_void_p()
    try:
        _native.check(lib, lib.mgb_pipeline_create(C.byref(ep.struct), max(lengths), len(r), 2, C.byref(h)))
    finally:
        lib.mgb_set_option(b"poison_alloc", 0)
    keep, outs = [], []
    try:
        for k, t in enumerate(targets):
            slot = C.c_int32(-1)
            profiled = k % 2 == 0
            if pcm:
                tt, rr = aligned_copy(targets_pcm[k]), aligned_copy(r_pcm)
                o = aligned((len(t), 2), np.int16)
                if profiled:
                    rc = lib.mgb_pipeline_submit_pcm_profiled(h, ptr(tt), 16, len(t), ptr(blob), ptr(o), 16, C.byref(slot))
                else:
                    rc = lib.mgb_pipeline_submit_pcm(h, ptr(tt), 16, len(t), ptr(rr), 16, len(r), ptr(o), 16, C.byref(slot))
            else:
                tt, rr = aligned_copy(t, np.float32), aligned_copy(r, np.float32)
                o = aligned((len(t), 2), np.float32)
                if profiled:
                    rc = lib.mgb_pipeline_submit_profiled(h, ptr(tt), len(t), ptr(blob), ptr(o), C.byref(slot))
                else:
                    rc = lib.mgb_pipeline_submit(h, ptr(tt), len(t), ptr(rr), len(r), ptr(o), C.byref(slot))
            _native.check(lib, rc)
            st = _native.TrackState()
            _native.check(lib, lib.mgb_pipeline_wait(h, slot.value, C.byref(st)))
            keep.append((tt, rr))
            outs.append((o, bytes(st)))
    finally:
        lib.mgb_pipeline_destroy(h)
    for t, (o, st) in zip(targets, outs):
        (w_outs, w_st, _), _ = paired(cfg, t, r)
        want = w_outs[0]
        if pcm:  # the library's own quantiser
            want = aligned((len(t), 2), np.int16)
            _native.check(lib, lib.mgb_pcm_encode(ptr(w_outs[0]), 16, ptr(want), 2 * len(t), None))
        if SEEDED:  # see assert_identical
            limit = 1 if pcm else REPEAT_TOL * max(1.0, float(np.abs(want).max()))
            assert np.abs(o.astype(np.float64) - want).max() <= limit
            got_st = _native.TrackState.from_buffer_copy(st)
            assert all(getattr(got_st, f) == getattr(w_st, f) for f in EXACT_FIELDS)
            continue
        assert np.array_equal(o, want)
        assert st == bytes(w_st)


@pytest.fixture(scope="module")
def io():
    lib = emul_lib()
    h = C.c_void_p()
    _native.check(lib, lib.mgb_host_io_create(3, 1024, 3, C.byref(h)))
    yield h
    lib.mgb_host_io_destroy(h)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_stages_main_host_profiled_matches_staged_calls_emulated(io, dtype):
    lib = emul_lib()
    kw, t, r, _ = case("f1024")
    cfg = port.OracleConfig(**kw)
    ep = get_emul_plan(cfg)
    blob, _ = emul_profile(cfg, r)
    want, _, _ = run_profiled(cfg, t, blob)
    T = len(t)
    L = profiled_layout(lib, ep, T)
    keep = dict(t=aligned((T, 2), np.float32), res=aligned((T, 2), np.float32), out=aligned((T, 2), np.float32),
                wide=aligned((T, 2), np.float64), ws=ebuf(L.workspace_bytes, "ff"),
                st=aligned((C.sizeof(_native.TrackState),), np.uint8))
    bufs = _native.HostBuffers()
    bufs.d_target_lr, bufs.d_reference_lr, bufs.d_result_lr = ptr(keep["t"]).value, None, ptr(keep["res"]).value
    bufs.d_out_lr, bufs.d_wide = ptr(keep["out"]).value, ptr(keep["wide"]).value
    bufs.d_workspace, bufs.d_state = ptr(keep["ws"]).value, ptr(keep["st"]).value
    ht = np.ascontiguousarray(t.astype(dtype))
    outs = [np.zeros((T, 2), dtype=dtype) for _ in range(3)]
    state = _native.TrackState()
    w = ht.dtype.itemsize
    _native.check(lib, lib.mgb_stages_main_host_profiled(io, C.byref(ep.struct), C.byref(L), ht.ctypes.data, w, ptr(blob),
                                                         *(o.ctypes.data for o in outs), w, C.byref(bufs), C.byref(state),
                                                         None))
    _, st_want, _ = run_profiled(cfg, t, blob)
    assert_identical(([o.astype(np.float32) for o in outs], state, None), (want, st_want, None))


# ---- the same under ThreadSanitizer and in other thread orders -----------------------------------------------------------
HERE = "tests/test_reference_profile.py::"
RACECHECK_IDS = ([HERE + f"test_profiled_job_is_bit_identical_to_paired_emulated[{c}]" for c in RACECHECK_CASES] +
                 [HERE + "test_profiled_job_on_poisoned_buffers_emulated",
                  HERE + "test_mixed_paired_and_profiled_batch_on_poisoned_pipeline_emulated",
                  HERE + "test_stages_main_host_profiled_matches_staged_calls_emulated"])


@pytest.fixture(scope="module")
def racecheck_runs(tmp_path_factory):
    from concurrent.futures import ThreadPoolExecutor

    import build_emul
    from test_emul_racecheck import run_group, tsan_env
    build_emul.build(racecheck=True)
    build_emul.build()
    base = tmp_path_factory.mktemp("profile_racecheck")
    jobs = {}
    for k, i in enumerate(RACECHECK_IDS):
        log_dir = str(base / f"tsan_{k}")
        env = tsan_env(log_dir)
        env["MGB_EMUL_BUILD"] = "racecheck"
        jobs[("tsan", k)] = ([i], env, log_dir)
    for order in ("reverse", "seeded"):
        env = dict(os.environ, MGB_EMUL_ORDER=order, MGB_EMUL_SEED="12345")
        jobs[(order, 0)] = (RACECHECK_IDS, env, str(base / order))
    with ThreadPoolExecutor(max_workers=8) as ex:
        futures = {key: ex.submit(run_group, *job) for key, job in jobs.items()}
        return {key: f.result() + (jobs[key][2],) for key, f in futures.items()}


@pytest.mark.parametrize("k", range(len(RACECHECK_IDS)))
def test_profile_kernels_have_no_data_races(racecheck_runs, k):
    from test_emul_racecheck import reports
    rc, out, _, log_dir = racecheck_runs[("tsan", k)]
    n, first = reports(log_dir)
    assert n == 0, f"{n} ThreadSanitizer report(s) in {RACECHECK_IDS[k]}; the first:\n{first}"
    assert rc == 0, out


@pytest.mark.parametrize("order", ["reverse", "seeded"])
def test_profile_tests_pass_in_other_thread_orders(racecheck_runs, order):
    rc, out, _, _ = racecheck_runs[(order, 0)]
    assert rc == 0, out
