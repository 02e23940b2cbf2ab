"""Native-rate masters on the H100: 3-minute 48 and 96 kHz targets against the C2 reference, against the float64
restatement (tests/native_rate_oracle.py) fed the device's analysis copy; mg.process of a 96 kHz 24-bit WAV to a
loudness target in true-peak mode with shaped dither; a target already at the internal rate; repeats; every instance
of the native design kernel launched."""
import ctypes as C

import numpy as np
import pytest

import native_rate_oracle as nro
import port

pytestmark = pytest.mark.gpu
C2_REF_FRAMES = 44100 * 180 - 44100 * 7
TOL = 1e-5
FIR_TOL = 1e-7
REPEAT_TOL = 1e-6  # tests/test_workspace_reuse.py: two runs of one job on the device, relative to max(1, peak)


def material(n, seed, rate):
    x = port.synth_target(n, seed).astype(np.float64)
    x += 0.2 * np.sin(2 * np.pi * 997.0 * np.arange(n) / rate)[:, None]
    return np.ascontiguousarray(x.astype(np.float32))


def device_native_job(cfg, xn, rate, r):
    """The staged native job on the device -> (outputs, native FIRs, analysis copy) as numpy."""
    import torch
    from matchering_b200.engine import TrackSession, get_native_plan, get_plan
    from matchering_b200.resample import resample_on_device
    plan, nplan = get_plan(cfg), get_native_plan(cfg, rate)
    dev = plan.device
    d_n = torch.from_numpy(xn).to(dev)
    d_a = resample_on_device(d_n, rate, cfg.internal_sample_rate)
    d_r = torch.from_numpy(r).to(dev)
    sess = TrackSession(plan, d_a.shape[0], d_r.shape[0])
    sess.match_levels(d_a, d_r)
    sess.design_frequencies()
    nat = TrackSession(nplan, d_n.shape[0], None)
    fir = torch.empty((2, nplan.tables.fft_size), dtype=torch.float64, device=dev)
    nat.match_frequencies_native(sess, d_n, fir)
    nat.correct_levels()
    outs = nat.finalize(True, True, True)
    return [o.cpu().numpy() for o in outs], fir.cpu().numpy(), d_a.cpu().numpy()


def max_err(got, want):
    return max(float(np.abs(g.astype(np.float64) - w).max()) for g, w in zip(got, want))


@pytest.mark.parametrize("rate", [48000, 96000])
def test_three_minute_native_job_matches_oracle(rate):
    import matchering_b200 as mg
    from matchering_b200 import stages
    cfg = mg.Config()
    xn = material(rate * 180, 0, rate)
    r = port.synth_reference(C2_REF_FRAMES, 1)
    outs, fir, xa = device_native_job(cfg, xn, rate, r)
    tr = {}
    want = nro.main(xn, xa, r, cfg, rate, True, True, True, trace=tr)
    for ch, name in enumerate(("mid", "side")):
        assert float(np.abs(fir[ch] - tr["firs"][name]).max()) < FIR_TOL, name
    assert max_err(outs, want) < TOL
    # the public seam computes the same job; two device runs agree to the repeat bound
    again = stages.main_native(xn, rate, r, cfg, True, True, True)
    for a, b in zip(outs, again):
        assert a.shape == b.shape == xn.shape
        assert float(np.abs(a - b).max()) <= REPEAT_TOL * max(1.0, float(np.abs(a).max()))


def test_repeats_agree_like_the_ordinary_job():
    import matchering_b200 as mg
    from matchering_b200 import stages
    cfg = mg.Config(max_piece_size=2.0)
    rate = 96000
    xn = material(rate * 20 + 11, 3, rate)
    r = port.synth_reference(44100 * 20, 4)
    a = stages.main_native(xn, rate, r, cfg, True, True, True)
    b = stages.main_native(xn, rate, r, cfg, True, True, True)
    for x, y in zip(a, b):
        assert float(np.abs(x - y).max()) <= REPEAT_TOL * max(1.0, float(np.abs(x).max()))


def test_process_96k_24_bit_to_a_loudness_target(tmp_path):
    import matchering_b200 as mg
    from matchering_b200 import wavio
    rate, n = 96000, 96000 * 30 + 123
    x = port.synth_target(n, 5).astype(np.float64) * 0.5  # white: content up to 48 kHz
    r = port.synth_reference(44100 * 30, 6).astype(np.float64)
    tp, rp, out = str(tmp_path / "t.wav"), str(tmp_path / "r.wav"), str(tmp_path / "out.wav")
    wavio.write(tp, x, rate, "PCM_24")
    wavio.write(rp, r, 44100, "PCM_16")
    cfg = mg.Config(native_rate=True, true_peak=True, loudness_target=-14)
    mg.process(tp, rp, [mg.pcm24(out, dither="shaped")], config=cfg,
               preview_result=mg.pcm24(str(tmp_path / "pr.wav")), preview_target=mg.pcm24(str(tmp_path / "pt.wav")))
    y, sr = wavio.read(out)
    assert sr == rate and y.shape == (n, 2)
    for name in ("pr.wav", "pt.wav"):
        assert wavio.read(str(tmp_path / name))[1] == rate
    m = mg.loudness(out)
    assert abs(m.integrated + 14.0) <= 0.01, m
    assert m.true_peak <= 20 * np.log10(cfg.threshold) + 0.2, m

    def high_share(v):
        spec = np.abs(np.fft.rfft(v[:, 0] + v[:, 1])) ** 2
        f = np.fft.rfftfreq(len(v), 1 / rate)
        return spec[f > 22050].sum() / spec.sum()

    share_in, share_out = high_share(x), high_share(y)
    assert share_in > 0.3 and share_out > 0.1 * share_in, (share_in, share_out)


def test_target_at_the_internal_rate_is_unchanged(tmp_path):
    """native_rate with a target already at internal_sample_rate writes the same files, byte for byte."""
    import matchering_b200 as mg
    from matchering_b200 import wavio
    t, r = port.synth_target(44100 * 12, 7), port.synth_reference(44100 * 10, 8)
    tp, rp = str(tmp_path / "t.wav"), str(tmp_path / "r.wav")
    wavio.write(tp, t.astype(np.float64), 44100, "PCM_16")
    wavio.write(rp, r.astype(np.float64), 44100, "PCM_16")
    files = {}
    for native in (False, True):
        out = [str(tmp_path / f"{native}_{k}.wav") for k in ("a", "b", "pr")]
        mg.process(tp, rp, [mg.pcm16(out[0]), mg.Result(out[1], "FLOAT", use_limiter=False)],
                   config=mg.Config(native_rate=native, max_piece_size=2.0), preview_result=mg.pcm16(out[2]))
        files[native] = [open(p, "rb").read() for p in out]
    # (device float64 atomics can move a last bit between any two runs: compare the 16-bit files exactly, the float
    # one to the repeat bound)
    assert files[False][0] == files[True][0] and files[False][2] == files[True][2]
    a = np.frombuffer(files[False][1][-8 * 44100:], np.float32)
    b = np.frombuffer(files[True][1][-8 * 44100:], np.float32)
    assert float(np.abs(a - b).max()) <= REPEAT_TOL


def test_every_native_design_instance_launches_and_matches_oracle():
    import matchering_b200 as mg
    from matchering_b200 import _native, stages
    lib = _native.load()
    jobs = [(512, 48000), (512, 96000), (512, 192000), (4096, 48000), (4096, 96000), (4096, 192000)]
    lib.mgb_profile_enable(1)
    try:
        results = []
        for F, rate in jobs:
            cfg = mg.Config(max_piece_size=1.0, fft_size=F)
            xn = material(rate * 3 + 17, 9, rate)
            r = port.synth_reference(44100 * 3, 10)
            results.append((cfg, xn, rate, r, device_native_job(cfg, xn, rate, r)))
    finally:
        cap = 8192
        names = C.create_string_buffer(1 << 18)
        ms = (C.c_float * cap)()
        got = lib.mgb_profile_collect(names, len(names), ms, cap)
        lib.mgb_profile_enable(0)
    launched = set(names.value.decode().split("\n")[:got])
    for F in (512, 1024, 2048, 4096, 8192, 16384):
        assert f"design_native_kernel<{F}>" in launched, F
    for cfg, xn, rate, r, (outs, fir, xa) in results:
        tr = {}
        want = nro.main(xn, xa, r, cfg, rate, True, True, True, trace=tr)
        assert float(np.abs(fir[0] - tr["firs"]["mid"]).max()) < FIR_TOL, (cfg.fft_size, rate)
        assert max_err(outs, want) < TOL, (cfg.fft_size, rate)
