"""Every stage's hand-off values against the float64 oracle (oracle/port.py), for every convolution kernel.

The end-to-end tests compare only the outputs, at 1e-5.  This file reads the job's workspace after each stage call
(mgb_test_workspace_regions) and compares what one stage hands the next: the analysis partials (per piece and slot:
|rfft| sums, sum(mid^2), peaks), the loudest-piece masks and level scalars, the FIR and its spectra on the
convolution's grid, the uncorrected convolution result, the per-piece sums of every correction step and the loud
lists (kernels.cuh: kLoudMid) the later steps read.  Each tolerance comes from float32 rounding; its derivation is
written next to it.

Variants: every convolution kernel `launch_convolve_t` can pick (fft_size 512 .. 16384, the fused kernels with and
without the persistent schedule and TMA, OVS 2 and 4, the generic fallback), twiddle_chain on and off, tma and
analyze_chain on and off.  Signals (edge_track) are built so that the edges where kernels go wrong are reached, and
each test asserts that they are."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import port

LOUD_MID = 0.5        # kLoudMid
U = 2.0 ** -24        # unit roundoff of float32
STEPS = 4
OPTION_DEFAULTS = {"tma": 1, "twiddle_chain": 1, "conv_fused": 1, "conv_frame": 4, "conv_persistent": 1,
                   "analyze_chain": 1}
REGIONS = ["spec_part_t", "spec_part_r", "sumsq_part_t", "sumsq_part_r", "absmax_part_t", "absmax_part_r", "mask_t",
           "mask_r", "h_mid", "h_side", "loud_values", "piece_sums", "loud_count"]


# on the device (132 SMs: 396 analysis CTAs, 79 slots per piece at 5 pieces) 81 frames per piece leave the last
# slot three frames, and every persistent convolution walks more frames than it has CTAs
DEVICE_FPP = 81


# ---- variants --------------------------------------------------------------------------------------------------
class Variant:
    """One kernel choice: fft_size, switches, the kernel they select, and the frames per piece the signal needs."""

    def __init__(self, name, F, options, kernel, ovs, fpp, emulated=True, device_fpp=None):
        self.name, self.F, self.options, self.kernel, self.ovs, self.fpp = name, F, options, kernel, ovs, fpp
        self.emulated = emulated
        self.device_fpp = device_fpp or DEVICE_FPP

    def expected_ovs(self, piece):
        """conv_frame_ovs (convolve.cu): 4 where the 4F-point fused kernel exists, is switched on and a piece
        holds at least 3F samples; 2 otherwise."""
        o = dict(OPTION_DEFAULTS, **self.options)
        if o["conv_frame"] == 4 and o["conv_fused"] and self.F in (2048, 4096) and piece >= 3 * self.F:
            return 4
        return 2


# fpp: whole analysis frames per piece on the emulator (8 SMs there: 24 analysis CTAs, 4 slots per piece at 5
# pieces; 5 frames per piece make the last slot take two).  The 4F-frame kernels need pieces of at least
# N = 4F samples for the silent-channel frames, and 5 frames at 4096 give the persistent schedule of the
# emulator's 8 CTAs 9 frames to walk.  The 16384 and 8192 variants without chaining, and 8192 without TMA,
# cost more emulator time than they add there: they run on the device only.
VARIANTS = [
    Variant("f512_generic", 512, {}, "convolve_kernel<512>", 2, 5),
    Variant("f1024_generic", 1024, {}, "convolve_kernel<1024>", 2, 5),
    Variant("f2048_fused4", 2048, {}, "convolve_fused_kernel<2048,4,.,false>", 4, 5),
    Variant("f2048_generic_short_piece", 2048, {}, "convolve_kernel<2048>", 2, 2, device_fpp=2),
    Variant("f4096_default", 4096, {}, "convolve_fused_kernel<4096,4,chain,persistent>", 4, 5),
    Variant("f4096_no_chain", 4096, {"twiddle_chain": 0}, "convolve_fused_kernel<4096,4,nochain,persistent>", 4, 5),
    Variant("f4096_no_tma", 4096, {"tma": 0}, "convolve_fused_kernel<4096,4,chain,false>", 4, 5),
    Variant("f4096_not_persistent", 4096, {"conv_persistent": 0}, "convolve_fused_kernel<4096,4,chain,false>", 4, 5),
    Variant("f4096_no_analyze_chain", 4096, {"analyze_chain": 0}, "convolve_fused_kernel<4096,4,chain,persistent>", 4, 5),
    Variant("f4096_ovs2", 4096, {"conv_frame": 2}, "convolve_fused_kernel<4096,2,chain,false>", 2, 2),
    Variant("f4096_generic", 4096, {"conv_fused": 0}, "convolve_kernel<4096>", 2, 2),
    Variant("f8192_fused", 8192, {}, "convolve_fused_kernel<8192,2,chain,persistent>", 2, 2),
    Variant("f8192_no_chain", 8192, {"twiddle_chain": 0}, "convolve_fused_kernel<8192,2,nochain,persistent>", 2, 2,
            emulated=False),
    Variant("f8192_no_tma", 8192, {"tma": 0}, "convolve_fused_kernel<8192,2,chain,false>", 2, 2, emulated=False),
    Variant("f8192_generic", 8192, {"conv_fused": 0}, "convolve_kernel<8192>", 2, 2),
    Variant("f16384_global", 16384, {}, "convolve_global_kernel<chain>", 2, 2),
    Variant("f16384_global_no_chain", 16384, {"twiddle_chain": 0}, "convolve_global_kernel<nochain>", 2, 2,
            emulated=False),
]
BY_NAME = {v.name: v for v in VARIANTS}


# ---- signals ---------------------------------------------------------------------------------------------------
def edge_track(F, ovs, fpp, seed=3):
    """Five pieces of P = fpp*F + F/2 + 1 samples (odd: analysis frames of odd pieces start on odd samples; the
    piece's last F/2 + 1 samples come after its last whole frame) and two samples past 5P:
      piece 0  noise with some loud mid samples;
      piece 1  loud noise: its loud list overflows; its last F samples are quiet;
      piece 2  quiet noise, no loud sample; ends in a stretch with L == R (side silent);
      piece 3  digital silence;
      piece 4  starts with a stretch with L == -R (mid silent), then noise with some loud samples;
      tail     the track's largest sample (uncounted: it must count for the peak only).
    The two stretches reach into the silent piece so that each covers a whole convolution input frame (N = ovs*F
    samples from n0 - F/2), while the other channel is non-zero in that frame.  T = 5P + 2 is odd and not a
    multiple of the frame's output count.  Returns (x float32 [T, 2], info)."""
    rng = np.random.default_rng(seed)
    P = fpp * F + F // 2 + 1
    T = 5 * P + 2
    N = ovs * F
    OUT = N - F
    start = lambda k: k * OUT - F // 2
    x = np.zeros((T, 2))
    n = np.arange(T)
    # every non-quiet stretch is the reference's kind of material (compressed pink noise): the matching FIR stays
    # near flat, so the result's levels follow the input's.  Piece 1, the only loud piece, comes out at the
    # reference's level; pieces 0 and 4, at 0.3 of it, below the average piece RMS
    loud = np.tanh(3.0 * port.synth_reference(T, seed + 100)).astype(np.float64)
    x[:P] = 0.3 * loud[:P]
    x[P:2 * P] = loud[P:2 * P]
    x[2 * P - F:2 * P] = rng.uniform(-0.02, 0.02, (F, 2))
    x[2 * P:3 * P] = rng.uniform(-0.02, 0.02, (P, 2))
    # side-silent frame: the last frame that starts inside piece 2 (it ends inside piece 3: P >= N)
    ks = max(k for k in range(T // OUT + 2) if start(k) < 3 * P)
    a = start(ks)
    x[a:3 * P, 1] = x[a:3 * P, 0]
    x[3 * P:4 * P] = 0.0
    # mid-silent frame: the first frame that starts inside piece 3 and ends inside piece 4
    km = min(k for k in range(T // OUT + 2) if start(k) >= 3 * P and start(k) + N > 4 * P)
    b = start(km) + N
    x[4 * P:5 * P] = 0.3 * loud[4 * P:5 * P]
    # 256-sample bursts at piece 1's level: loud samples in pieces 0 and 4 whatever the track's length, well below
    # their lists' capacity, those of piece 0 in the frame that holds the 0|1 boundary (P mod OUT >= F/2 + 1)
    x[P - 256:P] = loud[P - 256:P]
    x[4 * P + P // 2:4 * P + P // 2 + 256] = loud[4 * P + P // 2:4 * P + P // 2 + 256]
    s = rng.uniform(-0.03, 0.03, b - 4 * P)
    x[4 * P:b, 0], x[4 * P:b, 1] = s, -s
    x[5 * P:] = [[0.999, 0.97], [-0.98, -0.96]]  # (the loud material stays below tanh(3) = 0.9951)
    info = dict(P=P, T=T, N=N, OUT=OUT, side_silent_frame=ks, mid_silent_frame=km, fpp=fpp)
    return np.ascontiguousarray(x.astype(np.float32)), info


def edge_reference(T, seed=7):
    """Heavily compressed pink noise two samples shorter than the target (its own odd length and piece layout).
    Piece 1 is the target's only loud piece, so the result's level there follows this reference's: more than a
    quarter of its mid samples reach kLoudMid (the list overflows); pieces 0 and 4, at 0.3 of its level, a few."""
    return np.tanh(3.0 * port.synth_reference(T - 2, seed)).astype(np.float32)


def max_piece_seconds(T, divisions):
    """max_piece_size (seconds at 44.1 kHz) that cuts T samples into `divisions` pieces (match_levels.py:47-59)."""
    return T / (divisions - 0.5) / 44100.0


def spiky(n, seed):
    """Quiet noise with rare large spikes (test_correction_loud_list.py): the correction gain crosses 1 / kLoudMid
    between the later steps."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, 2)) * 0.05
    x[rng.random(n) < 0.002] *= 200
    return x.astype(np.float32)


# ---- running the stages ----------------------------------------------------------------------------------------
def regions(lib, plan_struct, layout):
    out = (C.c_int64 * 16)()
    from matchering_b200 import _native
    _native.check(lib, lib.mgb_test_workspace_regions(C.byref(plan_struct), C.byref(layout), out))
    return dict(zip(REGIONS + ["loud_capacity"], list(out)[:14]))


def view(ws, off, dtype, count):
    return np.frombuffer(ws, dtype=dtype, count=count, offset=off).copy()


def unpack(snap, reg, L, F):
    """The hand-off arrays of the three workspace snapshots (after match_levels, match_frequencies, correct_levels)."""
    HB = F // 2 + 1
    Dt, Dr, St, Sr = L.target_divisions, L.reference_divisions, L.target_slots, L.reference_slots
    w0, w1, w2 = snap
    cap = reg["loud_capacity"]
    return dict(
        spec_t=view(w0, reg["spec_part_t"], np.float32, Dt * St * 2 * HB).reshape(Dt, St, 2, HB),
        spec_r=view(w0, reg["spec_part_r"], np.float32, Dr * Sr * 2 * HB).reshape(Dr, Sr, 2, HB),
        sumsq_t=view(w0, reg["sumsq_part_t"], np.float64, Dt * St).reshape(Dt, St),
        sumsq_r=view(w0, reg["sumsq_part_r"], np.float64, Dr * Sr).reshape(Dr, Sr),
        absmax_t=view(w0, reg["absmax_part_t"], np.float32, Dt * St + 1),
        absmax_r=view(w0, reg["absmax_part_r"], np.float32, Dr * Sr + 1),
        mask_t=view(w1, reg["mask_t"], np.uint8, Dt), mask_r=view(w1, reg["mask_r"], np.uint8, Dr),
        h_mid=view(w1, reg["h_mid"], np.complex64, 2 * F + 1), h_side=view(w1, reg["h_side"], np.complex64, 2 * F + 1),
        loud_values=view(w1, reg["loud_values"], np.float32, Dt * cap).reshape(Dt, cap),
        loud_count=view(w1, reg["loud_count"], np.uint32, Dt),
        sums0=view(w1, reg["piece_sums"], np.float64, 16 * Dt).reshape(16, Dt),
        sums=view(w2, reg["piece_sums"], np.float64, 16 * Dt).reshape(16, Dt),
        capacity=cap)


def set_options(lib, options):
    for k, v in options.items():
        assert lib.mgb_set_option(k.encode(), v) == 0, k


def restore_options(lib):
    for k, v in OPTION_DEFAULTS.items():
        lib.mgb_set_option(k.encode(), v)


def run_emulated(cfg, t, r, options):
    from emul_harness import aligned, aligned_copy, emul_lib, get_emul_plan, ptr
    from matchering_b200 import _native
    lib = emul_lib()
    set_options(lib, options)
    try:
        ep = get_emul_plan(cfg)
        L = ep.layout(len(t), len(r))
        ws = aligned((L.workspace_bytes,), np.uint8)
        tgt, ref = aligned_copy(t, np.float32), aligned_copy(r, np.float32)
        result = aligned((len(t), 2), np.float32)
        fir = aligned((2, cfg.fft_size), np.float64)
        state = _native.TrackState()
        P, LL = C.byref(ep.struct), C.byref(L)
        snap = []
        _native.check(lib, lib.mgb_match_levels(P, LL, ptr(tgt), ptr(ref), ptr(ws), C.byref(state), None))
        snap.append(ws.tobytes())
        _native.check(lib, lib.mgb_match_frequencies(P, LL, ptr(tgt), ptr(result), ptr(fir), ptr(ws), C.byref(state), None))
        snap.append(ws.tobytes())
        _native.check(lib, lib.mgb_correct_levels(P, LL, ptr(ws), C.byref(state), None))
        snap.append(ws.tobytes())
        reg = regions(lib, ep.struct, L)
        return dict(L=L, state=state, result=np.array(result), fir=np.array(fir), snap=snap, reg=reg, device=False)
    finally:
        restore_options(lib)


def run_device(cfg, t, r, options):
    import torch
    from matchering_b200.engine import TrackSession, get_plan, to_device_f32
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    plan = get_plan(cfg)
    set_options(plan.lib, options)
    try:
        s = TrackSession(plan, len(t), len(r))
        td, rd = to_device_f32(t, plan.device), to_device_f32(r, plan.device)
        fir = torch.empty((2, cfg.fft_size), dtype=torch.float64, device=plan.device)
        snap = []
        s.match_levels(td, rd)
        snap.append(s.workspace.cpu().numpy().tobytes())
        s.match_frequencies(td, fir)
        snap.append(s.workspace.cpu().numpy().tobytes())
        s.correct_levels()
        snap.append(s.workspace.cpu().numpy().tobytes())
        reg = regions(plan.lib, plan.struct, s.layout)
        return dict(L=s.layout, state=s.read_state(), result=s.result.cpu().numpy(), fir=fir.cpu().numpy(), snap=snap,
                    reg=reg, device=True)
    finally:
        restore_options(plan.lib)


# ---- the float64 restatement of each stage ---------------------------------------------------------------------
def frame_sums(v, piece, divisions, F):
    """Per piece: sum over its whole F-sample frames of |rfft(frame)| (unscaled) and of sqrt(F) * ||frame||_2."""
    fpp = piece // F
    u = v[: piece * divisions].reshape(divisions, piece)[:, : fpp * F].reshape(divisions, fpp, F)
    spec = np.abs(np.fft.rfft(u, axis=-1)).sum(axis=1)
    norm = (np.sqrt(F) * np.sqrt((u * u).sum(axis=-1))).sum(axis=1)
    return spec, norm


def check_analysis(name, got_spec, got_sumsq, got_absmax, x, cfg, device, report):
    F = cfg.fft_size
    x64 = x.astype(np.float64)
    a = port.analyze(x64, cfg)
    D, P = a["divisions"], a["piece"]
    # sum(mid^2) per piece (over its slots): each term is a float32-rounded mid squared (relative error <= 2u + u^2)
    # summed in float64 (relative error ~ n * 2^-53, negligible); the slot sums add in float64 too
    want = (a["mid"][: D * P].reshape(D, P) ** 2).sum(axis=1)
    got = got_sumsq.sum(axis=1)
    rel = np.abs(got - want) / np.maximum(want, 1e-300)
    report[name + "_sumsq_rel"] = float(rel.max())
    assert np.all(rel <= 2.5e-7), (name, rel)
    assert np.all((want == 0) == (got == 0))
    # peaks: max|x| is exact in float32; the tail past piece*divisions counts for the peak only
    S = got_sumsq.shape[1]
    pk = got_absmax[: D * S].reshape(D, S).max(axis=1)
    want_pk = np.abs(x[: D * P]).reshape(D, 2 * P).max(axis=1)
    assert np.array_equal(pk, want_pk), name
    tail = np.abs(x[D * P:]).max() if len(x) > D * P else np.float32(0)
    assert got_absmax[D * S] == tail, name
    # |rfft| sums, every piece (the loudness mask is applied later, in the design): a float32 radix-r FFT errs by at
    # most c * log2(F) * u * sqrt(F) * ||frame||_2 per bin (Higham, ch. 24); mid and side share one transform, so
    # ||frame|| is that of mid + side (the balance factor is a power of two); c = 4 also covers the float32 rounding
    # of mid and side, the split of the pair Z[k], Z[F-k] and the float32 sum over a slot's frames (at most
    # ceil(frames/slots) terms: one u each).  On the device |z| comes from sqrt.approx: 2^-21 relative.
    spec_m, norm_m = frame_sums(a["mid"], P, D, F)
    spec_s, norm_s = frame_sums(a["side"], P, D, F)
    norm = norm_m + norm_s
    fps = -(-(P // F) // S)
    bound = (4 * np.log2(F) + fps) * U * norm + (2.0 ** -21 * norm if device else 0.0)
    got_spec = got_spec.astype(np.float64).sum(axis=1)  # [D][2][HB]
    for ch, want_spec in ((0, spec_m), (1, spec_s)):
        err = np.abs(got_spec[:, ch, :] - want_spec).max(axis=1)
        report[f"{name}_spec{ch}_err_over_bound"] = float((err / np.maximum(bound, 1e-300)).max())
        assert np.all(err <= bound), (name, ch, err, bound)
    return a


def full_plane_piece_sums(m, divisions, piece, correction, steps):
    """Per-piece sums of steps 1..steps-1 as the reference forms them, from the result's mid = (L + R) / 2:
    clip(mid * float32(gain)) in float32, squares summed in float64 (test_correction_loud_list.py)."""
    mm = m[: divisions * piece].reshape(divisions, piece)
    out = []
    for k in range(1, steps):
        g = np.float32(np.prod(correction[:k]))
        c = np.clip(mm * g, np.float32(-1), np.float32(1)).astype(np.float64)
        out.append((c * c).sum(axis=1))
    return np.array(out)


def submultiset_within(stored, ref, tol):
    """Every stored value matches a distinct reference value within tol (greedy over both sorted lists)."""
    s, r = np.sort(stored), np.sort(ref)
    j = 0
    for v in s:
        while j < len(r) and r[j] < v - tol:
            j += 1
        if j == len(r) or r[j] > v + tol:
            return False
        j += 1
    return True


def check_pipeline(run, cfg, t, r, report, expect_ovs=None):
    """Every stage's hand-off values of one job against the oracle; returns facts about what the job reached."""
    F = cfg.fft_size
    L, st, res, dev = run["L"], run["state"], run["result"], run["device"]
    w = unpack(run["snap"], run["reg"], L, F)
    trace = {}
    port.main(t.astype(np.float64), r.astype(np.float64), cfg, False, False, False, trace=trace)
    ta, ra = trace["target"], trace["reference"]
    D, P = L.target_divisions, L.target_piece
    assert (D, P) == (ta["divisions"], ta["piece"]) and (L.reference_divisions, L.reference_piece) == (
        ra["divisions"], ra["piece"])

    # ---- analysis: the target, and the reference before its normalisation (applied in the design)
    check_analysis("target", w["spec_t"], w["sumsq_t"], w["absmax_t"], t, cfg, dev, report)
    check_analysis("reference", w["spec_r"], w["sumsq_r"], w["absmax_r"], r, cfg, dev, report)

    # ---- levels: masks exactly (the signals have no ties), scalars to 1e-7: each is a square root of float64
    # sums whose terms carry the 2u of a float32 mid squared -> u of the root, 6e-8 (the c0 ratio: 2u)
    assert np.array_equal(w["mask_t"].astype(bool), ta["mask"])
    assert np.array_equal(w["mask_r"].astype(bool), ra["mask"])
    assert st.target_loud_pieces == ta["mask"].sum() and st.reference_loud_pieces == ra["mask"].sum()
    for got, want, what in ((st.target_match_rms, ta["match_rms"], "target_match_rms"),
                            (st.reference_match_rms, ra["match_rms"], "reference_match_rms"),
                            (st.rms_coefficient, trace["c0"], "rms_coefficient"),
                            (st.final_amplitude_coef, trace["final_coef"], "final_amplitude_coef")):
        rel = abs(got - want) / abs(want)
        report[what + "_rel"] = rel
        assert rel <= 1e-7, (what, got, want)
    assert st.reference_peak == np.abs(r).max()

    # ---- design: FIR to 1e-6 of its peak (the float64 chain on float32-summed spectra: their 2^-21..2^-24
    # relative errors, amplified by the smoothing's conditioning, stay below that); spectra on the convolution's grid
    ovs = expect_ovs
    N = ovs * F
    c0 = st.rms_coefficient
    for ch, key in ((0, "mid"), (1, "side")):
        want_fir = trace["firs"][key]
        err = np.abs(run["fir"][ch] - want_fir).max() / np.abs(want_fir).max()
        report[f"fir_{key}_rel"] = float(err)
        assert err <= 1e-6, (key, err)
        # H = c0/N * rfft(fir zero-padded to N): float32 rounding of the float64 spectrum (u relative) on top of the
        # FIR's own 1e-6
        want_h = np.fft.rfft(want_fir, n=N) * (c0 / N)
        got_h = w["h_mid" if ch == 0 else "h_side"][: N // 2 + 1].astype(np.complex128)
        err = np.abs(got_h - want_h).max() / np.abs(want_h).max()
        report[f"h_{key}_rel"] = float(err)
        assert err <= 1e-6, (key, err)
        peak_bits = st.fir_peak_mid_bits if ch == 0 else st.fir_peak_side_bits
        assert abs(peak_bits - np.abs(got_h).max()) <= 4 * U * peak_bits

    # ---- convolution, before correction: L/R = r_mid +- r_side at c0
    r_mid = port.convolve_same(ta["mid"] * trace["c0"], trace["firs"]["mid"])
    r_side = port.convolve_same(ta["side"] * trace["c0"], trace["firs"]["side"])
    want = np.stack([r_mid + r_side, r_mid - r_side], axis=1)
    err = float(np.abs(res.astype(np.float64) - want).max())
    scale = max(1.0, float(np.abs(want).max()))
    report["conv_abs"] = err
    report["conv_over_scale"] = err / scale
    # float32 transforms: the error grows with the result's magnitude (relative to full scale where that exceeds 1)
    assert err <= CONV_BOUND * scale, (err, scale)
    assert st.conv_peak_bits == np.abs(res).max()

    # ---- step 0 and the loud lists, per piece, from the result's mid = (L + R) / 2 (float32, as the reference)
    m = (res[:, 0] + res[:, 1]) * np.float32(0.5)
    mp = m[: D * P].reshape(D, P)
    c = np.clip(mp, -1, 1).astype(np.float64)
    want0 = (c * c).sum(axis=1)
    # the kernel squares the transform's mid m; (L + R)/2 differs from it by the half-ulps of L and R: relative
    # 2 * 2u per term where |side| <~ |mid|, more where the side dominates -- 1e-6 leaves room for that
    rel0 = np.abs(w["sums0"][0] - want0) / np.maximum(want0, 1e-300)
    report["step0_rel"] = float(rel0.max())
    assert np.all(rel0 <= 1e-6), rel0
    assert np.all((want0 == 0) == (w["sums0"][0] == 0))
    cap = w["capacity"]
    counts = w["loud_count"].astype(np.int64)
    facts = dict(overflow=[], no_loud=[], loud=[])
    for p in range(D):
        seg = res[p * P:(p + 1) * P]
        amp = float(np.abs(seg).max()) if len(seg) else 0.0
        # window around kLoudMid where m and (L + R)/2 may fall on different sides: their half-ulps at |L|, |R|
        win = 2 * np.spacing(np.float32(max(amp, LOUD_MID)))
        a = np.abs(mp[p])
        lo, hi = int((a >= LOUD_MID + win).sum()), int((a >= LOUD_MID - win).sum())
        assert lo <= counts[p] <= hi, (p, counts[p], lo, hi)
        sure = mp[p][a >= LOUD_MID + win]
        tol = 2 * np.spacing(np.float32(max(amp, LOUD_MID)))
        if counts[p] <= cap:
            got = w["loud_values"][p, : counts[p]]
            got_sure = got[np.abs(got) >= LOUD_MID + win]
            assert len(got_sure) == len(sure), (p, len(got_sure), len(sure))
            assert np.abs(np.sort(got_sure) - np.sort(sure)).max(initial=0) <= tol, p
            (facts["no_loud"] if counts[p] == 0 else facts["loud"]).append(p)
        else:
            facts["overflow"].append(p)
            cand = mp[p][a >= LOUD_MID - win]
            assert submultiset_within(w["loud_values"][p, :cap], cand, tol), p
    report["loud_counts"] = counts.tolist()

    # ---- later steps
    steps = cfg.rms_correction_steps
    corr = np.array([st.correction[i] for i in range(steps)])
    np.testing.assert_allclose(corr, trace["correction"], rtol=1e-6, atol=0)
    report["correction_rel"] = float(np.abs(corr / np.array(trace["correction"]) - 1).max())
    assert st.steps_done == steps
    gains = np.cumprod(corr)
    assert abs(st.gain - gains[-1]) <= 4 * steps * 2.0 ** -53 * gains[-1]
    fp = full_plane_piece_sums(m, D, P, corr, steps)
    # the list path squares the transform's m, the full plane (L + R)/2: they differ by at most
    # delta = ulp(max(|L|, |R|)) (half an ulp each for L = m + s, R = m - s and their sum, halved)
    delta = np.spacing(np.abs(res).max(axis=1).astype(np.float32)).astype(np.float64)[: D * P].reshape(D, P)
    worst = 0.0
    for k in range(1, steps):
        g = float(np.prod(corr[:k]))
        got = w["sums"][k]
        cg = np.abs(np.clip(mp.astype(np.float64) * g, -1, 1))
        for p in range(D):
            list_path = counts[p] <= cap and g * LOUD_MID <= 1 - 1e-6
            if list_path:
                # g^2 * S_quiet + exact list terms: each term off the full plane's by 2 |clip(g mid)| g delta
                # + (g delta)^2, the quiet part also by float32(g)^2 / g^2 - 1 (the full plane's gain is float32)
                terms = (2 * cg[p] * g * delta[p] + (g * delta[p]) ** 2).sum()
                tol = terms / max(fp[k - 1][p], 1e-300) + abs((float(np.float32(g)) / g) ** 2 - 1) + 1e-12
            else:
                tol = 1e-12  # the same pass over the result, float64 sums in another order
            rel = abs(got[p] - fp[k - 1][p]) / max(fp[k - 1][p], 1e-300)
            worst = max(worst, rel)
            assert rel <= tol, (k, p, rel, tol, list_path)
    report["later_steps_rel"] = worst
    # the scalars __finalize needs follow from conv_peak_bits and the gain, and agree with the oracle's result
    peak = float(st.conv_peak_bits) * st.gain
    assert st.result_peak == peak
    assert st.normalize_coef == max(cfg.min_value, peak / cfg.threshold)
    want_peak = float(np.abs(trace["pre_limiter"]).max())
    assert abs(peak - want_peak) <= CONV_BOUND * gains[-1] + 1e-6 * want_peak
    engaged = not np.isclose(max(peak, cfg.threshold) / cfg.threshold, 1.0)
    assert st.limiter_engaged == int(engaged)
    facts["gains"] = gains
    return facts


# The convolution's bound, relative to max(1, max|result|): twice the emulator's measured worst over every variant
# and both signals, 8.64e-7 (fft_size 4096, the 4F-frame fused kernels), and below the 3e-6 the float32 transform
# pair would allow (about log2(4F) * 2^-24 * max|result|, with the FIR's 1e-6 on top).
CONV_BOUND = 1.75e-6


# ---- the edge track through one variant ------------------------------------------------------------------------
def edge_case(variant, device):
    F = variant.F
    fpp = variant.device_fpp if device else variant.fpp
    t, info = edge_track(F, variant.ovs, fpp)
    r = edge_reference(info["T"])
    mps = max_piece_seconds(info["T"], 5)
    return t, r, info, mps


def check_edge_variant(variant, device):
    import matchering_b200 as mg
    t, r, info, mps = edge_case(variant, device)
    P, F, T = info["P"], variant.F, info["T"]
    if device:
        cfg = mg.Config(fft_size=F, max_piece_size=mps, rms_correction_steps=STEPS)
        run = run_device(cfg, t, r, variant.options)
        cfg = port.config_from(cfg)
    else:
        cfg = port.OracleConfig(fft_size=F, max_piece_size=mps, rms_correction_steps=STEPS)
        run = run_emulated(cfg, t, r, variant.options)
    L = run["L"]
    # the layout the signal was built for
    assert (L.target_divisions, L.target_piece, L.target_frames) == (5, P, T)
    assert P % 2 == 1 and T % 2 == 1 and T % info["OUT"] != 0 and T > 5 * P
    ovs = variant.expected_ovs(P)
    assert ovs == variant.ovs, (variant.name, ovs)
    report = {}
    facts = check_pipeline(run, cfg, t, r, report, expect_ovs=ovs)
    # edges reached: several slots per piece with frames_per_piece not a multiple of them (where the geometry
    # allows: the emulator's 8 SMs and the small pieces of some variants); an overflowing and a loud-free piece;
    # loud samples on both sides of a piece boundary inside one convolution frame; the largest sample uncounted
    if (P // F) in (5, DEVICE_FPP):
        assert L.target_slots > 1 and (P // F) % L.target_slots != 0, (P // F, L.target_slots)
        report["multi_slot"] = True
    assert facts["overflow"] == [1], facts
    assert 2 in facts["no_loud"] and 3 in facts["no_loud"] and 0 in facts["loud"] and 4 in facts["loud"], facts
    res = run["result"]
    m = (res[:, 0] + res[:, 1]) * np.float32(0.5)
    OUT = info["OUT"]
    k = P // OUT  # the frame with the 0|1 boundary
    lo, hi = k * OUT, min((k + 1) * OUT, T)
    assert lo < P < hi and (np.abs(m[lo:P]) >= LOUD_MID).any() and (np.abs(m[P:hi]) >= LOUD_MID).any()
    assert np.abs(t).max() == np.abs(t[5 * P:]).max() > np.abs(t[:5 * P]).max()
    assert (np.abs(m[5 * P:]) >= LOUD_MID).any()  # loud outputs past the counted samples, kept off the lists
    # silent-channel frames are exact
    for key, sign in (("mid_silent_frame", -1), ("side_silent_frame", 1)):
        f = info[key]
        o = res[f * OUT:(f + 1) * OUT]
        assert np.array_equal(o[:, 0], sign * o[:, 1]), key
        assert np.abs(o).max() > 0, key
    return report


def check_gain_crossing(variant, device):
    """The correction gain crosses 1 / kLoudMid between the later steps: a step on the lists, the next on the result."""
    import matchering_b200 as mg
    F = variant.F
    n = 16 * 3 * F + 1 if F >= 2048 else 40001
    t, r = spiky(n, 5), port.synth_reference(n - 5000, 32)
    mps = max_piece_seconds(n, 4)
    if device:
        cfg = mg.Config(fft_size=F, max_piece_size=mps, rms_correction_steps=STEPS)
        run = run_device(cfg, t, r, variant.options)
        cfg = port.config_from(cfg)
    else:
        cfg = port.OracleConfig(fft_size=F, max_piece_size=mps, rms_correction_steps=STEPS)
        run = run_emulated(cfg, t, r, variant.options)
    ovs = variant.expected_ovs(run["L"].target_piece)
    assert ovs == variant.ovs
    report = {}
    facts = check_pipeline(run, cfg, t, r, report, expect_ovs=ovs)
    g = facts["gains"][:-1]
    assert g[0] * LOUD_MID < 1 < g[-1] * LOUD_MID, g
    return report


def _record(tag, report):
    """Measured errors, one JSON line per case, where MGB_STAGE_REPORT names a file."""
    path = os.environ.get("MGB_STAGE_REPORT")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps({"case": tag, **{k: v for k, v in report.items()}}) + "\n")


# ---- the workspace view itself ---------------------------------------------------------------------------------
def test_workspace_regions_follow_the_layout():
    from emul_harness import emul_lib, get_emul_plan
    lib = emul_lib()
    cfg = port.OracleConfig(fft_size=1024, max_piece_size=0.3)
    ep = get_emul_plan(cfg)
    L = ep.layout(40001, 35001)
    reg = regions(lib, ep.struct, L)
    offs = [reg[k] for k in REGIONS]
    assert all(o % 256 == 0 for o in offs) and offs == sorted(offs) and offs[-1] < L.workspace_bytes
    assert reg["loud_capacity"] == ((L.target_piece + 3) // 4 + 3) // 4 * 4
    assert reg["spec_part_r"] - reg["spec_part_t"] >= L.target_divisions * L.target_slots * 2 * 513 * 4
    assert reg["loud_count"] - reg["piece_sums"] >= 16 * L.target_divisions * 8


# ---- emulator --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [v.name for v in VARIANTS if v.emulated])
def test_stage_parity_emulated(name):
    report = check_edge_variant(BY_NAME[name], device=False)
    _record("emulated:" + name, report)


@pytest.mark.parametrize("name", ["f1024_generic", "f4096_default"])
def test_gain_crossing_stage_parity_emulated(name):
    _record("emulated:gain_crossing:" + name, check_gain_crossing(BY_NAME[name], device=False))


# ---- device ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", [v.name for v in VARIANTS])
def test_stage_parity_device(name):
    report = check_edge_variant(BY_NAME[name], device=True)
    _record("device:" + name, report)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["f1024_generic", "f4096_default", "f8192_fused", "f16384_global"])
def test_gain_crossing_stage_parity_device(name):
    _record("device:gain_crossing:" + name, check_gain_crossing(BY_NAME[name], device=True))
