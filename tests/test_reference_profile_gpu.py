"""Reference profiles on the H100 at full size: every entry point that accepts a reference accepts a profile.

On the emulator (tests/test_reference_profile.py) a profiled job is bit-identical to the paired one end to end.  On
the device, stage 3 adds per-piece sums with float64 atomics in whatever order the CTAs finish, so not even a paired
job repeats bit for bit from there on (tests/test_workspace_reuse.py bounds two runs of one job by REPEAT_TOL).  Here
the level statistics and the FIR -- everything the profile feeds -- are held bit-identical, and the outputs to the
bound a paired job keeps against itself."""
import numpy as np
import pytest

import port

pytestmark = pytest.mark.gpu
TOL = 1e-5
REPEAT_TOL = 1e-6  # tests/test_workspace_reuse.py: two runs of one job on the device, relative to max(1, peak)
C2_FRAMES = 44100 * 180
# mgb_track_state fields stages 1 and 2 write: the same bits for a profiled and a paired job
EXACT_FIELDS = ["reference_peak", "final_amplitude_coef", "target_match_rms", "reference_match_rms", "rms_coefficient",
                "target_loud_pieces", "reference_loud_pieces", "fir_peak_mid_bits", "fir_peak_side_bits",
                "conv_precise", "conv_peak_bits"]


def close(a, b):
    """Within the device's repeat bound (and bit-identical wherever the device is deterministic)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape
    return float(np.abs(a - b).max()) / max(1.0, float(np.abs(b).max())) <= REPEAT_TOL


def stage_calls(cfg, t, reference):
    """The four stage calls through TrackSession -> (state, FIR, limited output)."""
    import torch

    import matchering_b200 as mg
    from matchering_b200.engine import TrackSession, get_plan, to_device_f32
    plan = get_plan(cfg)
    d_t = to_device_f32(t, plan.device)
    profiled = isinstance(reference, mg.ReferenceProfile)
    s = TrackSession(plan, len(t), None if profiled else len(reference))
    fir = torch.zeros((2, cfg.fft_size), dtype=torch.float64, device=plan.device)
    if profiled:
        s.match_levels_profiled(d_t, reference.checked_blob(plan))
    else:
        s.match_levels(d_t, to_device_f32(reference, plan.device))
    s.match_frequencies(d_t, fir)
    s.correct_levels()
    limited = s.finalize(True, False, False)[0].cpu().numpy()
    return s.read_state(), fir.cpu().numpy(), limited


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    return torch


@pytest.fixture(scope="module")
def c2(torch_cuda):
    """The benchmark's C2 recipe: a 3-minute target and a 3-minute reference, float64 like the reference's loader."""
    import matchering_b200 as mg
    t = port.synth_target(C2_FRAMES, 0).astype(np.float64)
    r = port.synth_reference(C2_FRAMES, 1000).astype(np.float64)
    cfg = mg.Config()
    return t, r, cfg, mg.analyze_reference(r, cfg)


def test_level_statistics_and_fir_bit_identical_at_full_size(c2):
    t, r, cfg, prof = c2
    st_p, fir_p, lim_p = stage_calls(cfg, t, r)
    st_q, fir_q, lim_q = stage_calls(cfg, t, prof)
    for f in EXACT_FIELDS:
        assert getattr(st_q, f) == getattr(st_p, f), f
    assert np.array_equal(fir_q, fir_p)
    assert st_q.steps_done == st_p.steps_done and st_q.limiter_engaged == st_p.limiter_engaged
    assert close(lim_q, lim_p)
    # the paired job against itself: the same bound
    assert close(stage_calls(cfg, t, r)[2], lim_p)


def test_stages_main_numpy_and_torch(c2, torch_cuda):
    torch = torch_cuda
    from matchering_b200 import stages
    t, r, cfg, prof = c2
    want = stages.main(t, r, cfg, True, True, True)
    got = stages.main(t, prof, cfg, True, True, True)
    for a, b in zip(got, want):
        assert a.dtype == np.float64 and close(a, b)
    td, rd = torch.from_numpy(t).cuda(), torch.from_numpy(r).cuda()
    want_t = stages.main(td, rd, cfg, True, True, True)
    got_t = stages.main(td, prof, cfg, True, True, True)
    for a, b in zip(got_t, want_t):
        assert a.dtype == torch.float32 and close(a.cpu().numpy(), b.cpu().numpy())
    dev = stages.main_device(t, prof, cfg, True, False, False)[0]
    assert close(dev.cpu().numpy(), want[0])
    assert np.abs(got[0] - port.main(t, r, port.config_from(cfg))[0]).max() < TOL


def test_master_many_profile_equals_pairs_float32_and_pcm16(c2):
    from matchering_b200._native import load
    from matchering_b200.batch import MasteringPipeline, master_many
    _, r, cfg, prof = c2
    r32 = r.astype(np.float32)
    targets = [port.synth_target(C2_FRAMES - 977 * k, 50 + k) for k in range(8)]
    want = master_many([(t, r32) for t in targets], cfg)
    got = master_many([(t, prof) for t in targets], cfg)
    for a, b in zip(got, want):
        assert close(a, b)
    pcm = lambda x: np.clip(np.rint(np.asarray(x, np.float64) * 32767.0), -32768, 32767).astype(np.int16)
    r16 = pcm(r32)
    outs = {}
    lib = load()
    for poisoned in (False, True):
        lib.mgb_set_option(b"poison_alloc", 1 if poisoned else 0)
        try:
            pipe = MasteringPipeline(cfg, C2_FRAMES, C2_FRAMES, depth=3)
        finally:
            lib.mgb_set_option(b"poison_alloc", 0)
        with pipe:
            for kind in ("pair", "profile"):
                res = [np.empty((len(t), 2), np.int16) for t in targets]
                for t, o in zip(targets, res):
                    pipe.submit_pcm(pcm(t), r16 if kind == "pair" else prof, o)
                pipe.wait_all()
                outs[(poisoned, kind)] = res
    for key, res in outs.items():  # within one LSB: a repeat's last-bit differences may cross a rounding boundary
        for a, b in zip(res, outs[(False, "pair")]):
            assert np.abs(a.astype(np.int32) - b).max() <= 1, key


def test_profile_only_pipeline_is_created_for_the_smallest_reference(c2):
    from matchering_b200.batch import MasteringPipeline, smallest_reference_frames
    t, r, cfg, prof = c2
    t32 = t[: 44100 * 30].astype(np.float32)
    with MasteringPipeline(cfg, len(t32), smallest_reference_frames(cfg), depth=2) as pipe:
        out = np.empty_like(t32)
        pipe.wait(pipe.submit(t32, prof, out))
        with pytest.raises(ValueError):
            pipe.submit(t32, r.astype(np.float32), np.empty_like(t32))  # samples longer than the pipeline allows
    from matchering_b200.batch import master_many
    assert close(out, master_many([(t32, r.astype(np.float32))], cfg)[0])


def test_config_with_other_fingerprint_is_refused(c2):
    import matchering_b200 as mg
    from matchering_b200 import stages
    t, _, _, prof = c2
    for cfg in (mg.Config(fft_size=2048), mg.Config(max_piece_size=10.0), mg.Config(threshold=0.9),
                mg.Config(internal_sample_rate=48000)):
        with pytest.raises(ValueError):
            stages.main(t, prof, cfg)
    # the target side may differ: limiter, correction steps, LOWESS
    other = mg.Config(rms_correction_steps=2, lowess_frac=0.05, limiter=mg.LimiterConfig(attack=3.0, hold=5.0))
    tt = t[: 44100 * 20]
    assert close(stages.main(tt, prof, other)[0], stages.main(tt, c2[1], other)[0])


def test_process_files_with_profile_and_after_save_load(c2, tmp_path):
    import matchering_b200 as mg
    from matchering_b200 import wavio
    n = 44100 * 40
    t = port.synth_target(n, 3).astype(np.float64)
    r = port.synth_reference(n + 5000, 4).astype(np.float64)
    tp, rp = str(tmp_path / "target.wav"), str(tmp_path / "reference.wav")
    wavio.write_pcm(tp, np.clip(np.rint(t * 32767), -32768, 32767).astype(np.int16), 44100, 16)
    wavio.write_pcm(rp, np.clip(np.rint(r * 32767), -32768, 32767).astype(np.int16), 44100, 16)

    def run(reference, tag):
        res = [mg.pcm16(str(tmp_path / f"{tag}_16.wav")), mg.pcm24(str(tmp_path / f"{tag}_24.wav")),
               mg.Result(str(tmp_path / f"{tag}_plain.wav"), "PCM_24", use_limiter=False, normalize=False)]
        pt, pr = mg.pcm16(str(tmp_path / f"{tag}_pt.wav")), mg.pcm16(str(tmp_path / f"{tag}_pr.wav"))
        mg.process(tp, reference, res, preview_target=pt, preview_result=pr)
        return [wavio.read(x.file) for x in res + [pt, pr]]

    def same_files(got, want):  # same rate and shape; samples within one LSB of the file's format
        for (a, ra), (b, rb), lsb in zip(got, want, (2.0 ** -15, 2.0 ** -23, 2.0 ** -23, 2.0 ** -15, 2.0 ** -15)):
            assert ra == rb and a.shape == b.shape
            assert np.abs(a - b).max() <= lsb * 1.0001

    want = run(rp, "paired")
    prof = mg.analyze_reference(rp)
    assert prof.frames == n + 5000
    same_files(run(prof, "profile"), want)
    prof.save(tmp_path / "ref.npz")
    loaded = mg.ReferenceProfile.load(tmp_path / "ref.npz")
    assert loaded.to_bytes() == prof.to_bytes()
    same_files(run(loaded, "loaded"), want)


def test_loaded_profile_on_this_and_other_devices(c2, tmp_path, torch_cuda):
    torch = torch_cuda
    import matchering_b200 as mg
    from matchering_b200 import stages
    t, r, cfg, prof = c2
    tt = t[: 44100 * 30]
    prof.save(tmp_path / "p.npz")
    loaded = mg.ReferenceProfile.load(tmp_path / "p.npz")
    want = stage_calls(cfg, tt, r)
    got = stage_calls(cfg, tt, loaded)
    assert np.array_equal(got[1], want[1]) and close(got[2], want[2])
    for d in range(1, torch.cuda.device_count()):
        with torch.cuda.device(d):
            got = stage_calls(cfg, tt, loaded)
        assert np.array_equal(got[1], want[1]) and close(got[2], want[2])


def test_goldens_through_the_profiled_path(torch_cuda, golden):
    """The small pipeline golden and the config-3 golden (10 minutes at 96 kHz) through a profile, within the
    suite's bound -- implied by bit-identity, asserted directly."""
    torch = torch_cuda
    import matchering_b200 as mg
    from matchering_b200 import stages
    g = golden("pipeline_small.npz")
    cfg = mg.Config(max_piece_size=float(g["max_piece_size_s"]))
    prof = mg.analyze_reference(g["reference"], cfg)
    got = stages.main(g["target"], prof, cfg, True, True, True)
    for a, k in zip(got, ("limited", "no_limiter", "normalized")):
        assert np.abs(a - g[k]).max() < TOL
    g = golden("c3_pipeline_96k.npz")
    n = int(g["limited_frames"])
    t = torch.from_numpy(port.synth_target(n, int(g["target_seed"]))).cuda()
    r = torch.from_numpy(port.synth_reference(n, int(g["reference_seed"]))).cuda()
    cfg = mg.Config(internal_sample_rate=int(g["sample_rate"]))
    prof = mg.analyze_reference(r, cfg)
    del r
    limited, plain, _ = stages.main(t, prof, cfg, True, True, False)
    from test_gpu_parity import _compare_decimated
    _compare_decimated(limited, g, "limited_", TOL)
    _compare_decimated(plain, g, "no_limiter_", TOL)
