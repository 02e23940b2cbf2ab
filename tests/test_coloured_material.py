"""The pipeline on the material matchering exists for: band-limited, upsampled, transient and bass-heavy targets,
matched to a bright reference, against the float64 oracle (oracle/port.py).

The other end-to-end tests feed white noise under a slow envelope, whose matching FIR stays within about 20x of flat.
Here the FIR raises a target's empty band by up to 10^4, and with it the float32 rounding noise of a transform that
the band holds instead of signal.  Each case asserts what makes it hard (premises), then:
  - the limited output within 1e-5 absolute of the oracle's;
  - the no-limiter outputs within 1e-5 of max(1, max|oracle output|) (a pre-limiter peak of 20 is stored in
    float32 with an ulp of 2e-6);
  - the uncorrected convolution result against the float64 convolution of the c0-scaled mid / side with the
    device's OWN FIR (design error kept out), to a bound that does not grow with the FIR's dynamic range."""
import numpy as np
import pytest
from scipy import signal

import port
from test_stage_parity import BY_NAME, restore_options, set_options

SR = 44100
SECONDS = 3.3
U = 2.0 ** -24
PRECISE_ERROR = 5e-6  # convolve.cu: kConvPreciseError


# ---- material: float64 from a seed, cast to float32 ------------------------------------------------------------
def brick_wall(x, f):
    """Every rfft bin above f Hz zeroed, in float64."""
    X = np.fft.rfft(np.asarray(x, np.float64), axis=0)
    X[np.fft.rfftfreq(len(x), 1.0 / SR) > f] = 0
    return np.fft.irfft(X, n=len(x), axis=0)


def butterworth(x, f=16000.0, order=16):
    """A steep IIR low-pass, zero phase."""
    sos = signal.butter(order, f, fs=SR, output="sos")
    return signal.sosfiltfilt(sos, np.asarray(x, np.float64), axis=0)


def bursts(n, seed):
    """Decaying noise bursts (amplitude 0.9, every 0.45 s) over a 0.01 noise floor."""
    rng = np.random.default_rng(seed)
    x = 0.01 * rng.uniform(-1, 1, (n, 2))
    period, length = int(0.45 * SR), int(0.2 * SR)
    env = np.exp(-np.arange(length) / (0.03 * SR))
    for s in range(period // 3, n - length, period):
        b = rng.uniform(-1, 1, (length, 2)) * env[:, None]
        x[s:s + length] += 0.9 * b / np.abs(b).max()
    return x


def bass_tilt(n, seed):
    """White noise tilted by -12 dB/octave above 40 Hz (flat below), peak 0.7."""
    w = np.random.default_rng(seed).uniform(-1, 1, (n, 2))
    f = np.fft.rfftfreq(n, 1.0 / SR)
    X = np.fft.rfft(w, axis=0) * (40.0 / np.maximum(f, 40.0))[:, None] ** 2
    x = np.fft.irfft(X, n=n, axis=0)
    return 0.7 * x / np.abs(x).max()


def bright(n, seed):
    """The bright modern reference: tanh(2 w / max|w|), w uniform white noise."""
    w = np.random.default_rng(seed).uniform(-1, 1, (n, 2))
    return np.tanh(2.0 * w / np.abs(w).max())


def resample_emulated(x, rate_in, rate_out):
    """mgb_resample through the emulator, with the product's Kaiser-sinc table (matchering_b200/resample.py)."""
    from emul_harness import aligned, aligned_copy, emul_lib, ptr
    from scipy.signal.windows import kaiser
    from matchering_b200 import _native
    from matchering_b200 import resample as product
    lib = emul_lib()
    bits = 2 ** product.PRECISION
    m = bits * product.NUM_ZEROS
    win = product.ROLLOFF * np.sinc(product.ROLLOFF * np.linspace(0, product.NUM_ZEROS, num=m + 1)) * kaiser(2 * m + 1, product.BETA)[m:]
    if rate_out < rate_in:
        win = (rate_out / rate_in) * win
    pairs = aligned_copy(np.stack([win, np.diff(win, append=win[-1])], axis=1))
    n_out = int(lib.mgb_resample_frames(len(x), rate_in, rate_out))
    xin, out = aligned_copy(x.astype(np.float32)), aligned((n_out, 2), np.float32)
    _native.check(lib, lib.mgb_resample(ptr(xin), len(x), rate_in, ptr(out), n_out, rate_out, ptr(pairs), len(win), bits, None))
    return np.array(out)


def upsampled(n, seed, device):
    """synth_target made at 22.05 kHz, taken to 44.1 kHz by the product's resampler (what mg.process does)."""
    x22 = port.synth_target(n // 2 + 1, seed)
    if device:
        import torch
        from matchering_b200.resample import resample_on_device
        x = resample_on_device(torch.from_numpy(x22).cuda(), 22050, SR).cpu().numpy()
    else:
        x = resample_emulated(x22, 22050, SR)
    return np.ascontiguousarray(x[:n])


TARGETS = {
    "lp2k": lambda n, d: brick_wall(port.synth_target(n, 1), 2000),
    "lp4k": lambda n, d: brick_wall(port.synth_target(n, 1), 4000),
    "lp8k": lambda n, d: brick_wall(port.synth_target(n, 1), 8000),
    "lp11k": lambda n, d: brick_wall(port.synth_target(n, 1), 11025),
    "lp16k": lambda n, d: brick_wall(port.synth_target(n, 1), 16000),
    "quiet_lp11k": lambda n, d: 0.05 * brick_wall(port.synth_target(n, 1), 11025),
    "quiet_lp4k": lambda n, d: 0.02 * brick_wall(port.synth_target(n, 1), 4000),
    "butter16k": lambda n, d: butterworth(port.synth_target(n, 1)),
    "upsampled22k": lambda n, d: upsampled(n, 1, d),
    "bursts": lambda n, d: bursts(n, 5),
    "bass": lambda n, d: bass_tilt(n, 6),
}
REFERENCES = {
    "bright": lambda n: bright(n, 2),
    "pink": lambda n: port.synth_reference(n, 2),
}
# (target, reference, premise: the oracle's c0 * max|H| * max|target| at least this, pre-limiter peak at least this)
CASES = {
    "lp2k_bright": ("lp2k", "bright", 150, 50),
    "lp4k_bright": ("lp4k", "bright", 150, 20),
    "lp8k_bright": ("lp8k", "bright", 150, 10),
    "lp11k_bright": ("lp11k", "bright", 100, 4),
    "lp16k_bright": ("lp16k", "bright", 100, 3),
    "lp16k_pink": ("lp16k", "pink", 25, 2),
    "quiet_lp11k_bright": ("quiet_lp11k", "bright", 100, 4),
    "quiet_lp4k_bright": ("quiet_lp4k", "bright", 150, 20),
    "butter16k_bright": ("butter16k", "bright", 100, 3),
    "upsampled22k_bright": ("upsampled22k", "bright", 100, 3),
    "bursts_pink": ("bursts", "pink", 50, 15),
    "bass_bright": ("bass", "bright", 100, 3),
}
KERNELS = ["f1024_generic", "f4096_default", "f4096_ovs2", "f8192_fused", "f16384_global"]
EMULATED = [("lp2k_bright", "f4096_default"), ("lp4k_bright", "f4096_default"), ("lp8k_bright", "f4096_default"),
            ("quiet_lp11k_bright", "f4096_default"), ("upsampled22k_bright", "f4096_ovs2"),
            ("butter16k_bright", "f1024_generic"), ("bursts_pink", "f4096_default"), ("bass_bright", "f8192_fused"),
            ("lp8k_bright", "f16384_global")]


def material(case, device):
    tname, rname, _, _ = CASES[case]
    n = int(SECONDS * SR)
    t = np.ascontiguousarray(np.asarray(TARGETS[tname](n, device), np.float64).astype(np.float32))
    r = np.ascontiguousarray(np.asarray(REFERENCES[rname](n - 1000), np.float64).astype(np.float32))
    return t, r


# ---- running the pipeline ---------------------------------------------------------------------------------------
def run(case, kernel, device):
    import matchering_b200 as mg
    variant = BY_NAME[kernel]
    t, r = material(case, device)
    if device:
        from matchering_b200.engine import TrackSession, get_plan, to_device_f32
        cfg = mg.Config(fft_size=variant.F, max_piece_size=1.0)
        plan = get_plan(cfg)
        set_options(plan.lib, variant.options)
        try:
            import torch
            s = TrackSession(plan, len(t), len(r))
            fir = torch.empty((2, cfg.fft_size), dtype=torch.float64, device=plan.device)
            s.match_levels(to_device_f32(t, plan.device), to_device_f32(r, plan.device))
            s.match_frequencies(to_device_f32(t, plan.device), fir)
            s.correct_levels()
            outs = [o.cpu().numpy() for o in s.finalize(True, True, True)]
            st, fir, res = s.read_state(), fir.cpu().numpy(), s.result.cpu().numpy()
            ovs = variant.expected_ovs(s.layout.target_piece)
        finally:
            restore_options(plan.lib)
        cfg = port.config_from(cfg)
    else:
        from emul_harness import emul_lib, run_pipeline
        cfg = port.OracleConfig(fft_size=variant.F, max_piece_size=1.0)
        lib = emul_lib()
        set_options(lib, variant.options)
        try:
            outs, st, fir, res, L = run_pipeline(cfg, t, r)
            ovs = variant.expected_ovs(L.target_piece)
        finally:
            restore_options(lib)
    return t, r, cfg, outs, st, np.array(fir), np.array(res), ovs


# The convolution's bound on the float64 path, relative to max(1, max|result|).  Its rounding happens in three
# places, none of which sees the FIR's dynamic range: the FIR spectra are stored in float32 (relative 2^-24 per
# component of every bin: the product errs by at most sqrt(2) u |H X| per bin, independent roundings, so the
# output's error has an rms of about sqrt(2) u rms(result) -- 6 sigma of it below 8.5 u max|result|); L and R are
# rounded to float32 once (u max|result|); the float64 transforms add 2^-53 log2(N) of the frame's level times the
# FIR's gain (at a gain of 10^4 still below 1e-11).  Together: 10 u.
PRECISE_CONV_BOUND = 10 * U


def estimate(st, N, t):
    """convolve.cu conv_precise: u sqrt(log2 N) N max(FIR peaks as applied) max|target|."""
    return U * np.sqrt(np.log2(N)) * N * max(st.fir_peak_mid_bits, st.fir_peak_side_bits) * float(np.abs(t).max())


def check(case, kernel, device):
    t, r, cfg, outs, st, fir, res, ovs = run(case, kernel, device)
    _, _, min_gain, min_pre = CASES[case]
    trace = {}
    want = port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True, trace=trace)
    N = ovs * cfg.fft_size
    report = {}
    # ---- premises: what makes the case hard
    H = max(np.abs(np.fft.rfft(trace["firs"][k], n=N)).max() for k in ("mid", "side"))
    gain = trace["c0"] * H * float(np.abs(t).max())
    pre = float(np.abs(trace["pre_limiter"]).max())
    report.update(gain=gain, pre=pre)
    assert gain >= min_gain, (case, gain)
    assert pre >= min_pre, (case, pre)
    assert st.limiter_engaged == 1
    # the float32 transforms would not do: the path is the float64 one
    est = estimate(st, N, t)
    assert est > PRECISE_ERROR and st.conv_precise == 1, (case, est, st.conv_precise)
    # ---- the uncorrected convolution against the float64 convolution with the device's own FIR
    c0 = st.rms_coefficient
    mid, side = trace["target"]["mid"], trace["target"]["side"]
    r_mid, r_side = port.convolve_same(mid * c0, fir[0]), port.convolve_same(side * c0, fir[1])
    conv = np.stack([r_mid + r_side, r_mid - r_side], axis=1)
    scale = max(1.0, float(np.abs(conv).max()))
    err = float(np.abs(res.astype(np.float64) - conv).max())
    report["conv_over_scale"] = err / scale
    assert err <= PRECISE_CONV_BOUND * scale, (case, err, scale)
    # ---- outputs
    lim = float(np.abs(outs[0].astype(np.float64) - want[0]).max())
    report["limited"] = lim
    assert lim <= 1e-5, (case, lim)
    for name, got, w in (("no_limiter", outs[1], want[1]), ("normalized", outs[2], want[2])):
        e = float(np.abs(got.astype(np.float64) - w).max()) / max(1.0, float(np.abs(w).max()))
        report[name] = e
        assert e <= 1e-5, (case, name, e)
    return report


def test_broadband_material_stays_on_the_float32_path():
    """The suite's and the benchmark's kind of material: white noise under an envelope, pink reference.  Its FIR is
    close to flat and the float32 transforms are accurate enough, so they are what runs."""
    from emul_harness import run_pipeline
    cfg = port.OracleConfig(max_piece_size=1.0)
    n = int(SECONDS * SR)
    t, r = port.synth_target(n, 1), port.synth_reference(n - 1000, 2)
    outs, st, _, _, _ = run_pipeline(cfg, t, r)
    assert st.conv_precise == 0 and estimate(st, 4 * cfg.fft_size, t) < PRECISE_ERROR / 1.5
    want = port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, False, False)[0]
    assert np.abs(outs[0] - want).max() <= 1e-5


@pytest.mark.parametrize("case,kernel", EMULATED)
def test_coloured_material_emulated(case, kernel):
    check(case, kernel, device=False)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("case", list(CASES))
def test_coloured_material_device(case, kernel):
    report = check(case, kernel, device=True)
    print(case, kernel, report)
