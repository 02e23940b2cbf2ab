"""Loudness targets on the H100: the C2 job through stages.main in both peak modes against the float64 search, the
one-hour C5 buffer through mg.limit, a 24-bit file at -14 LUFS / -1 dBTP through mg.process, and run-to-run agreement."""
import ctypes as C
import math

import numpy as np
import pytest

import loudness
import loudness_target_oracle as lto
import port

pytestmark = pytest.mark.gpu
C2_FRAMES = 44100 * 180
TOL = 1e-5


def session_to_loudness(t, r, cfg):
    """stages.main_device's four stages with the target, keeping the device report -> (limited numpy, report)."""
    import torch

    from matchering_b200 import _native
    from matchering_b200.engine import TrackSession, get_plan, to_device_f32
    plan = get_plan(cfg)
    with torch.cuda.device(plan.device):
        dt, dr = to_device_f32(t, plan.device), to_device_f32(r, plan.device)
        s = TrackSession(plan, dt.shape[0], dr.shape[0])
        s.match_levels(dt, dr)
        s.match_frequencies(dt)
        s.correct_levels()
        limited, _, _, report = s.finalize_to_loudness(cfg.loudness_target, False, False)
        rep = _native.LoudnessTargetReport.from_buffer_copy(report.cpu().numpy().tobytes())
        return limited.cpu().numpy(), rep


def assert_report_matches(rep, want):
    assert rep.passes == want["passes"] and rep.status == want["status"], (rep.passes, rep.status, want["trace"])
    for k, (x, I) in enumerate(want["trace"]):
        assert abs(rep.trace_gain_db[k] - x) < 1e-4, (k, rep.trace_gain_db[k], x)
        assert rep.trace_integrated[k] == I or abs(rep.trace_integrated[k] - I) < 1e-3, (k, rep.trace_integrated[k], I)


@pytest.mark.parametrize("target", [-16.0, -14.0, -9.0])
@pytest.mark.parametrize("tp", [False, True])
def test_c2_job_through_stages_main_against_oracle(target, tp):
    import matchering_b200 as mg
    from matchering_b200 import stages
    cfg = mg.Config(true_peak=tp, loudness_target=target)
    t, r = port.synth_target(C2_FRAMES, 0), port.synth_reference(C2_FRAMES - 44100 * 7, 1)
    got, rep = session_to_loudness(t, r, cfg)
    want = lto.main(t, r, cfg, target)
    assert_report_matches(rep, want)
    assert rep.status == lto.REACHED
    assert float(np.abs(got - lto.limited(want["s"], rep.gain_db, cfg)).max()) < TOL
    assert abs(mg.loudness(got, 44100).integrated - target) <= lto.TOLERANCE
    # stages.main on numpy takes the same device path and gives the same samples, up to the limiter's look-back
    out = stages.main(t, r, cfg)[0]
    assert float(np.abs(out - got).max()) <= 2.5e-7
    # and the output is repeatable
    got2, rep2 = session_to_loudness(t, r, cfg)
    assert abs(rep2.gain_db - rep.gain_db) < 1e-4 and rep2.passes == rep.passes
    assert float(np.abs(got2 - got).max()) < TOL


def test_c3_job_at_minus_14_lufs():
    """The C3 job (10 minutes at 96 kHz) through the device session: the report is what the meter reads of the output,
    within 0.01 LU of the target, and stages.main gives the same samples."""
    import matchering_b200 as mg
    from matchering_b200 import stages
    fs = 96000
    cfg = mg.Config(internal_sample_rate=fs, loudness_target=-14)
    t, r = port.synth_target(fs * 600, 10), port.synth_reference(fs * 590, 11)
    got, rep = session_to_loudness(t, r, cfg)
    m = mg.loudness(got, fs)
    print(f"C3: {rep.passes} passes, status {rep.status}, drive {rep.gain_db:+.4f} dB, {rep.integrated:.4f} LUFS")
    assert rep.status == lto.REACHED and rep.passes <= lto.MAX_PASSES
    assert abs(m.integrated - rep.integrated) <= 1e-6
    assert abs(m.integrated - -14.0) <= lto.TOLERANCE
    assert float(np.abs(stages.main(t, r, cfg)[0] - got).max()) <= 2.5e-7


def test_master_many_with_a_profile_reaches_the_target():
    """master_many with a target, a reference profile and loudness=True: every meter within 0.01 LU of the target; the
    pipeline's reports agree with its meters and with the single-job entry, and a target-free pipeline is unchanged."""
    import matchering_b200 as mg
    from matchering_b200.batch import MasteringPipeline, master_many
    cfg = mg.Config(loudness_target=-14, true_peak=True)
    rng = np.random.default_rng(21)
    pairs = [(port.synth_target(44100 * 20 - int(rng.integers(0, 44100)), 300 + k), port.synth_reference(44100 * 15, 400 + k))
             for k in range(4)]
    pairs[1] = (pairs[1][0], mg.analyze_reference(pairs[1][1], cfg))
    outs, meters = master_many(pairs, cfg, depth=2, loudness=True)
    for m in meters:
        assert abs(m.integrated - -14.0) <= lto.TOLERANCE
    plain = master_many(pairs, mg.Config(true_peak=True), depth=2)
    assert any(abs(mg.loudness(o, 44100).integrated - -14.0) > 0.1 for o in plain)  # (the target did something)
    max_t = max(len(t) for t, _ in pairs)
    with MasteringPipeline(cfg, max_t, 44100 * 15, depth=2) as pipe:
        for k, (t, r) in enumerate(pairs):
            o = np.empty((len(t), 2), np.float32)
            slot = pipe.submit(np.ascontiguousarray(t), r if k == 1 else np.ascontiguousarray(r), o)
            _, meter, target = pipe.wait_loudness_target(slot)
            assert target.status == "reached" and abs(target.integrated - meter.integrated) <= 1e-6
            assert abs(meter.integrated - meters[k].integrated) <= 1e-4
            if k == 0:
                _, rep = session_to_loudness(t, r, cfg)
                assert target.passes == rep.passes and abs(target.gain_db - rep.gain_db) < 1e-4
            assert float(np.abs(o - outs[k]).max()) < TOL


def test_c5_hour_through_limit():
    import torch

    import matchering_b200 as mg
    from matchering_b200.limiter.hyrax import limit_to_loudness
    cfg = mg.Config(loudness_target=-14)
    x = torch.from_numpy(port.synth_limiter_input(44100 * 3600, 0) * np.float32(0.3)).cuda()
    out, t = limit_to_loudness(x, cfg)
    m = mg.loudness(out, 44100)
    print(f"C5 hour: {t.passes} passes, status {t.status}, drive {t.gain_db:+.4f} dB, {t.integrated:.4f} LUFS")
    assert t.status == "reached" and t.passes <= lto.MAX_PASSES
    assert abs(m.integrated - t.integrated) <= 1e-6
    assert abs(m.integrated - -14.0) <= lto.TOLERANCE


def test_limit_never_returns_its_input_with_a_target():
    import matchering_b200 as mg
    from matchering_b200.limiter import limit
    x = port.synth_target(44100 * 10, 3) * np.float32(0.1)
    got = limit(x, mg.Config(loudness_target=-30))
    assert got is not x
    assert abs(mg.loudness(got, 44100).integrated - -30.0) <= lto.TOLERANCE


def test_process_to_24_bit_file_at_minus_14_lufs(tmp_path):
    import matchering_b200 as mg
    from matchering_b200 import wavio
    t, r = port.synth_target(44100 * 20, 5), port.synth_reference(44100 * 15, 6)
    tp, rp, op = str(tmp_path / "t.wav"), str(tmp_path / "r.wav"), str(tmp_path / "out.wav")
    wavio.write(tp, t.astype(np.float64), 44100, "PCM_24")
    wavio.write(rp, r.astype(np.float64), 44100, "PCM_24")
    cfg = mg.Config(loudness_target=-14, threshold=10 ** (-1 / 20), true_peak=True)
    mg.process(tp, rp, [mg.pcm24(op)], config=cfg)
    m = mg.loudness(op)
    assert abs(m.integrated - -14.0) <= 0.02
    assert m.true_peak <= -1.0 + 0.2
