"""Parity of the CUDA path (libmatchering_b200.so on a real H100) against the oracle and the
golden vectors.  Everything goes through the C ABI, either directly or through the reference-shaped
Python surface (stages.main / limiter.limit).  Tolerance: sample-wise max-abs <= 1e-5 (north star);
the float64 FIR design is held to 1e-9."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TOL = 1e-5


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    return torch


@pytest.fixture(scope="module")
def lib(torch_cuda):
    from matchering_b200 import _native
    return _native.load()


@pytest.fixture(params=[1, 0], ids=["tma", "plain-loads"])
def tma(request, lib):
    lib.mgb_set_option(b"tma", request.param)
    yield request.param
    lib.mgb_set_option(b"tma", 1)


def test_native_library_is_the_cuda_build(lib):
    import matchering_b200._native as n
    assert n.LIB_PATH.endswith("libmatchering_b200.so") and lib.mgb_version() >= 100


@pytest.mark.parametrize("n,f64", [(512, 0), (512, 1), (1024, 0), (2048, 0), (4096, 0), (8192, 0), (16384, 0), (4096, 1), (8192, 1)])
def test_fft_matches_numpy(torch_cuda, lib, n, f64):
    torch = torch_cuda
    from matchering_b200 import _native
    rng = np.random.default_rng(n + f64)
    dt = np.complex128 if f64 else np.complex64
    x = (rng.standard_normal((5, n)) + 1j * rng.standard_normal((5, n))).astype(dt)
    p = _native.Plan()
    p.fft_size = n if n <= 8192 else n // 2
    p.n_lin, p.n_log, p.lowess_k, p.lowess_nfit = p.fft_size // 2 + 1, 10, 2, 2
    bufs = [torch.zeros(1 << 20, dtype=torch.uint8, device="cuda") for _ in range(4)]
    p.d_tw_f32_F, p.d_tw_f32_2F, p.d_tw_f64_F, p.d_tw_f64_2F = [b.data_ptr() for b in bufs]
    _native.check(lib, lib.mgb_plan_fill_twiddles(C.byref(p), None))
    tw = bufs[1] if n > 8192 else (bufs[2] if f64 else bufs[0])
    xin = torch.from_numpy(x).cuda()
    out = torch.empty_like(xin)
    for direction in (1, -1):
        _native.check(lib, lib.mgb_test_fft(n, f64, direction, xin.data_ptr(), out.data_ptr(), 5, tw.data_ptr(), None))
        torch.cuda.synchronize()
        want = np.fft.fft(x.astype(np.complex128), axis=1) if direction == 1 else np.fft.ifft(x.astype(np.complex128), axis=1) * n
        err = np.abs(out.cpu().numpy() - want).max() / np.abs(want).max()
        assert err < (1e-14 if f64 else 5e-7)


def _config(**kw):
    import matchering_b200 as mg
    return mg.Config(**kw)


def _compare(got, want, tol=TOL):
    for a, b in zip(got, want):
        if b is None:
            assert a is None
        else:
            assert a.shape == b.shape and np.abs(a - b).max() < tol


def test_pipeline_matches_golden(torch_cuda, tma, golden):
    from matchering_b200 import stages
    g = golden("pipeline_small.npz")
    cfg = _config(max_piece_size=float(g["max_piece_size_s"]))
    got = stages.main(g["target"].astype(np.float64), g["reference"].astype(np.float64), cfg, True, True, True)
    assert all(o.dtype == np.float64 for o in got)
    _compare(got, (g["limited"], g["no_limiter"], g["normalized"]))


def test_pipeline_quiet_reference_early_out(torch_cuda, golden):
    from matchering_b200 import stages
    g = golden("pipeline_quiet_reference.npz")
    cfg = _config(max_piece_size=float(g["max_piece_size_s"]))
    got = stages.main(g["target"], g["reference"], cfg, True, True, False)
    assert got[0].dtype == np.float32 and got[2] is None
    _compare(got, (g["limited"], g["no_limiter"], None))


def test_fir_and_scalars_match_golden(torch_cuda, golden):
    torch = torch_cuda
    from matchering_b200.engine import TrackSession, get_plan, to_device_f32
    g = golden("pipeline_small.npz")
    cfg = _config(max_piece_size=float(g["max_piece_size_s"]))
    plan = get_plan(cfg)
    t, r = to_device_f32(g["target"], plan.device), to_device_f32(g["reference"], plan.device)
    s = TrackSession(plan, t.shape[0], r.shape[0])
    fir = torch.zeros((2, cfg.fft_size), dtype=torch.float64, device=plan.device)
    s.match_levels(t, r)
    s.match_frequencies(t, fir)
    s.correct_levels()
    st = s.read_state()
    assert (s.layout.target_divisions, s.layout.target_piece) == (int(g["target_divisions"]), int(g["target_piece"]))
    assert abs(st.rms_coefficient - float(g["rms_coefficient"])) < 1e-9
    assert abs(st.final_amplitude_coef - float(g["final_amplitude_coefficient"])) < 1e-12
    assert abs(st.target_match_rms - float(g["target_match_rms"])) < 1e-9
    f = fir.cpu().numpy()
    assert np.abs(f[0] - g["fir_mid"]).max() < 1e-7 and np.abs(f[1] - g["fir_side"]).max() < 1e-7
    assert st.steps_done == 4 and st.limiter_engaged == 1


@pytest.mark.parametrize("fft_size,sr,seconds", [(512, 44100, 1.0), (1024, 44100, 1.5), (2048, 22050, 2.0), (4096, 96000, 1.2), (8192, 44100, 2.5)])
def test_pipeline_other_configs_against_oracle(torch_cuda, fft_size, sr, seconds):
    import port
    from matchering_b200 import stages
    cfg = _config(internal_sample_rate=sr, fft_size=fft_size, max_piece_size=0.6, rms_correction_steps=3)
    n = int(sr * seconds) + 13
    t, r = port.synth_target(n, 5), port.synth_reference(n - 4001, 6)
    got = stages.main(t, r, cfg, True, True, True)
    want = port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True)
    _compare(got, want)


def test_pipeline_fft_size_16384_against_oracle(torch_cuda):
    """fft_size 16384 (frames and design planes in global memory): two minutes, so that every CTA of the
    global-memory convolution walks several frames; pieces of a few frames with ragged tails."""
    import port
    from matchering_b200 import stages
    cfg = _config(fft_size=16384, max_piece_size=2.0)
    n = 44100 * 120 + 311  # 323 frames of 16384 outputs on 296 CTAs
    t, r = port.synth_target(n, 15), port.synth_reference(n - 7001, 16)
    got = stages.main(t, r, cfg, True, True, True)
    want = port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True)
    _compare(got, want)


@pytest.mark.parametrize("fft_size", [4096, 8192])
def test_generic_convolution_kernel_against_oracle(torch_cuda, lib, fft_size):
    """These sizes normally take the fused convolution kernel; the all-shared-memory one must agree too."""
    import port
    from matchering_b200 import stages
    cfg = _config(fft_size=fft_size, max_piece_size=1.0)
    n = 44100 * 4 + 5
    t, r = port.synth_target(n, 21), port.synth_reference(n - 999, 22)
    lib.mgb_set_option(b"conv_fused", 0)
    try:
        got = stages.main(t, r, cfg, True, True, True)
    finally:
        lib.mgb_set_option(b"conv_fused", 1)
    fused = stages.main(t, r, cfg, True, True, True)
    want = port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True)
    _compare(got, want)
    _compare(fused, want)


def test_pipeline_half_minute_against_oracle(torch_cuda, tma):
    """30 s at the default Config (3 pieces, ~320 convolution frames, ~290 limiter chunks)."""
    import port
    from matchering_b200 import stages
    cfg = _config()
    n = 44100 * 30 + 7
    t, r = port.synth_target(n, 0), port.synth_reference(n + 1001, 1)
    got = stages.main(t, r, cfg, True, True, True)
    want = port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True)
    _compare(got, want)
    assert abs(np.abs(got[0]).max() - np.abs(want[0]).max()) < 1e-6


def test_pipeline_is_reproducible_and_does_not_touch_inputs(torch_cuda):
    import port
    from matchering_b200 import stages
    cfg = _config(max_piece_size=2.0)
    t, r = port.synth_target(200000, 8), port.synth_reference(190000, 9)
    t0, r0 = t.copy(), r.copy()
    a = stages.main(t, r, cfg)[0]
    b = stages.main(t, r, cfg)[0]
    assert np.array_equal(t, t0) and np.array_equal(r, r0)
    assert np.abs(a - b).max() < 1e-6  # float64 atomics may reorder the per-piece sums' last bits


def test_limiter_matches_golden(torch_cuda, golden):
    from matchering_b200.limiter import limit
    g = golden("limiter.npz")
    got = limit(g["x"].astype(np.float64), _config())
    assert got.dtype == np.float64 and np.abs(got - g["y_44100"]).max() < 3e-7
    got96 = limit(g["x"], _config(internal_sample_rate=96000))
    assert np.abs(got96 - g["y_96000"]).max() < 3e-7


@pytest.mark.parametrize("n", [7, 100, 4607, 4608, 4609, 9217, 200001])
def test_limiter_edge_lengths(torch_cuda, n):
    import port
    from matchering_b200.limiter import limit
    x = port.synth_limiter_input(max(n, 64), seed=n)[:n]
    got = limit(x, _config())
    want = port.limit(x.astype(np.float64), port.OracleConfig())
    assert np.abs(got - want).max() < 3e-7


def test_limiter_early_out_returns_input_object(torch_cuda):
    import port
    from matchering_b200.limiter import limit
    x = (0.2 * port.synth_limiter_input(6000, 2)).astype(np.float64)
    assert limit(x, _config()) is x
    with pytest.raises(ValueError):
        limit(np.zeros((6, 2)), _config())


def test_limiter_three_minutes_against_oracle(torch_cuda):
    """1723 chunks chained by decoupled look-back; the release pole needs float64 carries."""
    import port
    from matchering_b200.limiter import limit
    x = port.synth_limiter_input(44100 * 180, seed=0)
    got = limit(x, _config())
    want = port.limit(x.astype(np.float64), port.OracleConfig())
    assert np.abs(got - want).max() < 3e-7
    assert abs(np.abs(got).max() - _config().threshold) < 1e-6


def _compare_decimated(y, g, prefix, tol):
    """y: (frames, 2) CUDA tensor; g: a golden file of oracle/make_golden_full.py (decimated output of the
    UNMODIFIED reference at full size).  -> the largest error seen anywhere."""
    import torch
    every, window = int(g[prefix + "every"]), int(g[prefix + "window"])
    assert y.shape[0] == int(g[prefix + "frames"])
    worst = float(np.abs(y[::every].cpu().numpy().astype(np.float64) - g[prefix + "rows"]).max())
    for start, want in zip(g[prefix + "window_starts"], g[prefix + "windows"]):
        got = y[int(start):int(start) + window].cpu().numpy().astype(np.float64)
        worst = max(worst, float(np.abs(got - want).max()))
    assert worst < tol, f"decimated rows / windows differ by {worst}"
    # 64 block sums of the output and of its square: every frame of the buffer takes part
    edges = g[prefix + "block_edges"]
    y64 = y.to(torch.float64)
    csum = torch.cat([torch.zeros((1, 2), dtype=torch.float64, device=y.device), torch.cumsum(y64, 0)])
    csq = torch.cat([torch.zeros((1, 2), dtype=torch.float64, device=y.device), torch.cumsum(y64 * y64, 0)])
    idx = torch.from_numpy(edges).to(y.device)
    block_sum = (csum[idx[1:]] - csum[idx[:-1]]).cpu().numpy()
    block_sq = (csq[idx[1:]] - csq[idx[:-1]]).cpu().numpy()
    frames_per_block = np.diff(edges)[:, None]
    # a per-sample error e moves a block's mean by at most e and its mean square by at most 2*peak*e
    assert np.abs(block_sum - g[prefix + "block_sum"]).max() / frames_per_block.min() < tol
    peak = float(g[prefix + "peak"])
    assert (np.abs(block_sq - g[prefix + "block_sumsq"]) / frames_per_block).max() < 2 * max(peak, 1.0) * tol
    mono = y.abs().amax(dim=1)
    assert abs(float(mono.max()) - peak) < tol
    assert abs(float(mono[int(g[prefix + "peak_at"])]) - peak) < tol
    return worst


def test_config5_limiter_one_hour_against_reference_golden(torch_cuda, golden):
    """BASELINE config 5 AT FULL SIZE: limit() on one hour of 44.1 kHz stereo (158.76 M frames, 34 454
    chunks chained by look-back) against the unmodified reference's output, decimated
    (tests/golden/c5_limiter_hour.npz: every 997th frame, 12 windows across chunk boundaries up to the
    buffer's end, 64 block sums, the peak).  Tolerance 3e-7 like the short limiter tests."""
    torch = torch_cuda
    import port
    from matchering_b200.limiter import limit
    g = golden("c5_limiter_hour.npz")
    n = int(g["frames"])
    x = port.synth_limiter_input(n, seed=int(g["seed"]))
    assert abs(float(x.astype(np.float64).sum()) - float(g["input_sum"])) < 1e-3, "synthetic input differs from the golden's"
    xd = torch.from_numpy(x).cuda()
    del x
    y = limit(xd, _config())
    worst = _compare_decimated(y, g, "", 3e-7)
    print("config-5 (1 h limiter) max-abs error vs the reference at the golden points:", worst)
    thr = _config().threshold
    assert abs(float(y.abs().max()) - thr) < 1e-6
    assert bool((y.abs() <= xd.abs() + 1e-7).all())


def test_full_size_config2_against_oracle(torch_cuda):
    """BASELINE config 2: 3-minute 44.1 kHz stereo track, full pipeline (oracle: ~9 s of CPU)."""
    import port
    from matchering_b200 import stages
    n = 44100 * 180
    t, r = port.synth_target(n, 0), port.synth_reference(n, 1)
    got = stages.main(t, r, _config(), True, True, True)
    want = port.main(t.astype(np.float64), r.astype(np.float64), port.OracleConfig(), True, True, True)
    errs = [float(np.abs(a - b).max()) for a, b in zip(got, want)]
    print("config-2 max-abs errors (limited, no-limiter, normalised):", errs)
    assert max(errs) < TOL


def test_process_files_end_to_end(torch_cuda, tmp_path):
    """BASELINE config 1 shape: mg.process on WAV files (10 s white target vs pink reference)."""
    import matchering_b200 as mg
    import port
    from matchering_b200 import wavio
    n = 441000
    t = port.synth_target(n, 0, kind="white")
    r = port.synth_reference(n, 1, kind="quiet")
    wavio.write(str(tmp_path / "t.wav"), t, 44100, "FLOAT")
    wavio.write(str(tmp_path / "r.wav"), r, 44100, "FLOAT")
    codes = []
    mg.log(info_handler=codes.append)
    try:
        mg.process(str(tmp_path / "t.wav"), str(tmp_path / "r.wav"),
                   [mg.pcm16(str(tmp_path / "o16.wav")), mg.Result(str(tmp_path / "of.wav"), "FLOAT", use_limiter=False)])
    finally:
        mg.log()
    assert codes[0] == "Loading and analysis" and codes[-1] == "The task is completed" and "Matching frequencies" in codes
    want = port.main(t.astype(np.float64), r.astype(np.float64), port.OracleConfig(), True, False, True)
    got_f, _ = wavio.read(str(tmp_path / "of.wav"))
    got_16, _ = wavio.read(str(tmp_path / "o16.wav"))
    assert np.abs(got_f - want[2]).max() < TOL
    assert np.abs(got_16 - want[0]).max() < 1.0 / 32767 + TOL


def test_batch_pipeline_matches_single_track_path(torch_cuda):
    """master_many (three tracks in flight, copies overlapped with kernels) vs stages.main."""
    import port
    from matchering_b200 import stages
    from matchering_b200.batch import master_many
    cfg = _config(max_piece_size=3.0)
    pairs = [(port.synth_target(300000 + 1111 * k, 20 + k), port.synth_reference(280000, 40 + k)) for k in range(5)]
    got = master_many(pairs, cfg, depth=3)
    for (t, r), o in zip(pairs, got):
        want = stages.main(t, r, cfg)[0]
        assert o.shape == want.shape and np.abs(o - want).max() < 1e-6


def test_pcm_batch_entry(torch_cuda):
    """int16 in / int16 out through the batch pipeline == decode, float pipeline, encode (bit-exact
    up to one LSB where the float32 result sits on a rounding boundary)."""
    import port
    from matchering_b200 import stages
    from matchering_b200.batch import MasteringPipeline
    cfg = _config(max_piece_size=3.0)
    t = port.synth_target(300000, 3)
    r = port.synth_reference(280000, 4)
    t16 = np.clip(np.rint(t * 32767.0), -32768, 32767).astype(np.int16)
    r16 = np.clip(np.rint(r * 32767.0), -32768, 32767).astype(np.int16)
    out16 = np.zeros((300000, 2), dtype=np.int16)
    with MasteringPipeline(cfg, 300000, 280000, depth=2) as pipe:
        st = pipe.wait(pipe.submit_pcm(t16, r16, out16))
    assert st.steps_done == 4
    want = stages.main(t16.astype(np.float32) / np.float32(32768.0), r16.astype(np.float32) / np.float32(32768.0), cfg)[0]
    want16 = np.clip(np.rint(want * np.float32(32767.0)), -32768, 32767).astype(np.int16)
    assert np.abs(out16.astype(np.int32) - want16.astype(np.int32)).max() <= 1
    assert (out16 != want16).mean() < 1e-3


@pytest.mark.parametrize("steps", [0, 1, 3])
def test_rms_correction_step_counts(torch_cuda, steps):
    import port
    from matchering_b200 import stages
    cfg = _config(fft_size=1024, max_piece_size=0.3, rms_correction_steps=steps)
    t, r = port.synth_target(40000, 31), port.synth_reference(35000, 32)
    _compare(stages.main(t, r, cfg, True, True, True),
             port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True))


def test_shortest_legal_tracks_and_extreme_levels(torch_cuda):
    import port
    from matchering_b200 import stages
    cfg = _config(fft_size=1024)
    t, r = port.synth_target(1500, 41), port.synth_reference(1025, 42)
    _compare(stages.main(t, r, cfg, True, True, True),
             port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True))
    cfg = _config(fft_size=1024, max_piece_size=0.4)
    t = (1e-4 * port.synth_target(30000, 51)).astype(np.float32)
    r = np.clip(1.5 * port.synth_reference(30000, 52), -1.0, 1.0).astype(np.float32)
    _compare(stages.main(t, r, cfg, True, True, True),
             port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True))


def test_unsupported_configs_fail_loudly(torch_cuda):
    from matchering_b200 import stages
    from matchering_b200.plan import UnsupportedConfig
    import matchering_b200 as mg
    x = np.zeros((20000, 2), dtype=np.float32)
    for cfg in (_config(fft_size=256), _config(fft_size=32768), _config(limiter=mg.LimiterConfig(release_filter_order=3)),
                _config(fft_size=4096, max_piece_size=0.1)):
        with pytest.raises(UnsupportedConfig):
            stages.main(x[:5000], x[:5000], cfg)


def test_direct_smoothing_path_matches_operator_path(torch_cuda, lib, golden):
    """mgb_plan.d_smooth_op == NULL makes design_kernel run spline/LOWESS/spline itself."""
    torch = torch_cuda
    import ctypes as C
    from matchering_b200 import _native
    from matchering_b200.engine import TrackSession, get_plan, to_device_f32
    g = golden("pipeline_small.npz")
    cfg = _config(max_piece_size=float(g["max_piece_size_s"]))
    plan = get_plan(cfg)
    t, r = to_device_f32(g["target"], plan.device), to_device_f32(g["reference"], plan.device)
    firs = []
    saved = plan.struct.d_smooth_op
    try:
        for op in (saved, None):
            plan.struct.d_smooth_op = op
            s = TrackSession(plan, t.shape[0], r.shape[0])
            fir = torch.zeros((2, cfg.fft_size), dtype=torch.float64, device=plan.device)
            s.match_levels(t, r)
            s.match_frequencies(t, fir)
            firs.append(fir.cpu().numpy())
    finally:
        plan.struct.d_smooth_op = saved
    assert np.abs(firs[0] - firs[1]).max() < 1e-12
    assert np.abs(firs[0][0] - g["fir_mid"]).max() < 1e-7


def test_config3_ten_minutes_96k_against_reference_golden(torch_cuda, golden):
    """BASELINE config 3 AT FULL SIZE: stages.main on 10 minutes of 96 kHz stereo (57.6 M frames, 41
    pieces x 342 STFT frames, limiter windows 193 / 96) against the unmodified reference's outputs,
    decimated (tests/golden/c3_pipeline_96k.npz).  Tolerance: the north star's 1e-5."""
    torch = torch_cuda
    import port
    from matchering_b200 import stages
    g = golden("c3_pipeline_96k.npz")
    n = int(g["limited_frames"])
    t = port.synth_target(n, int(g["target_seed"]))
    r = port.synth_reference(n, int(g["reference_seed"]))
    got_sum = float(t.astype(np.float64).sum() + r.astype(np.float64).sum())
    assert abs(got_sum - float(g["input_sum"])) < 1e-3, "synthetic inputs differ from the golden's"
    cfg = _config(internal_sample_rate=int(g["sample_rate"]))
    td, rd = torch.from_numpy(t).cuda(), torch.from_numpy(r).cuda()
    del t, r
    limited, plain, _ = stages.main(td, rd, cfg, True, True, False)
    e_lim = _compare_decimated(limited, g, "limited_", TOL)
    e_plain = _compare_decimated(plain, g, "no_limiter_", TOL)
    print("config-3 (10 min @ 96 kHz) max-abs errors vs the reference at the golden points (limited, no limiter):", e_lim, e_plain)
    assert float(limited.abs().max()) <= cfg.threshold + 1e-6


def test_config4_shape_batch_of_tracks(torch_cuda):
    """BASELINE config 4 is a batch of 64 x 3-min tracks sharded across GPUs; per GPU that is
    master_many over its share.  Eight 20-s tracks here, each against stages.main."""
    import port
    from matchering_b200 import sharding, stages
    from matchering_b200.batch import master_many
    cfg = _config()
    n = 44100 * 20
    mine = sharding.tracks_for_rank(64, 0, 8)
    assert mine == [0, 8, 16, 24, 32, 40, 48, 56]
    pairs = [(port.synth_target(n, seed), port.synth_reference(n, 1000 + seed)) for seed in mine]
    outs = master_many(pairs, cfg, depth=3)
    for (t, r), o in zip(pairs[:3], outs[:3]):
        assert np.abs(o - stages.main(t, r, cfg)[0]).max() < 1e-6
    for (t, r), o in zip(pairs, outs):
        coef = min(1.0, float(np.abs(r).max()) / cfg.threshold)  # normalize_reference's coefficient
        assert np.isfinite(o).all() and abs(float(np.abs(o).max()) - cfg.threshold * coef) < 1e-5


def test_process_pcm_files_stay_on_the_device(torch_cuda, tmp_path):
    """mg.process on 16-bit (mono target!) and 24-bit PCM WAV: decode, checks, mastering and
    quantisation all on the device; result against the oracle fed the same decoded samples."""
    import matchering_b200 as mg
    import port
    from matchering_b200 import wavio
    from matchering_b200.log import ModuleError
    n = 44100 * 6
    t = port.synth_target(n, 3)[:, :1]                       # mono
    r = port.synth_reference(n + 500, 4)
    wavio.write(str(tmp_path / "t16.wav"), t, 44100, "PCM_16")
    wavio.write(str(tmp_path / "r24.wav"), r, 44100, "PCM_24")
    seen = []
    mg.log(info_handler=seen.append, warning_handler=seen.append)
    try:
        mg.process(str(tmp_path / "t16.wav"), str(tmp_path / "r24.wav"), [mg.pcm24(str(tmp_path / "o24.wav"))],
                   config=mg.Config(max_piece_size=2.0))
    finally:
        mg.log()
    assert "The TARGET audio is mono. Converting it to stereo..." in seen
    t_dec, _ = wavio.read(str(tmp_path / "t16.wav"))
    r_dec, _ = wavio.read(str(tmp_path / "r24.wav"))
    want = port.main(np.repeat(t_dec, 2, axis=1), r_dec, port.OracleConfig(max_piece_size=2.0))[0]
    got, sr = wavio.read(str(tmp_path / "o24.wav"))
    assert sr == 44100 and np.abs(got - want).max() < TOL + 2.0 / 8388607
    # the same file twice is refused like in the reference (checker.py:140-142)
    wavio.write(str(tmp_path / "s.wav"), r, 44100, "PCM_16")
    with pytest.raises(ModuleError):
        mg.process(str(tmp_path / "s.wav"), str(tmp_path / "s.wav"), [mg.pcm16(str(tmp_path / "x.wav"))])


def test_preview_pieces_match_golden(torch_cuda, golden):
    """matchering_b200.preview_creator against the reference's create_preview (tests/golden/preview.npz)."""
    import matchering_b200 as mg
    from matchering_b200.preview_creator import preview_pieces
    g = golden("preview.npz")
    cfg = mg.Config(internal_sample_rate=int(g["sample_rate"]), preview_size=int(g["preview_size_s"]),
                    preview_analysis_step=int(g["preview_analysis_step_s"]))
    every = int(g["every"])
    index, t_piece, r_piece = preview_pieces(g["target"], g["result"], cfg)
    t_piece, r_piece = t_piece.cpu().numpy(), r_piece.cpu().numpy()
    assert index == int(g["index"])
    assert np.abs(t_piece[::every] - g["target_piece"]).max() < 2e-7
    assert np.abs(r_piece[::every] - g["result_piece"]).max() < 2e-7
    assert np.abs(t_piece[:300] - g["target_piece_head"]).max() < 2e-7
    assert np.abs(r_piece[-300:] - g["result_piece_tail"]).max() < 2e-7
    assert np.abs(t_piece).max() <= cfg.threshold  # the target piece is clipped at the threshold


def test_process_with_previews(torch_cuda, tmp_path):
    """mg.process(..., preview_target=, preview_result=): the loudest 30-s window of the result, from both signals."""
    import matchering_b200 as mg
    import port
    from matchering_b200 import wavio
    n = 44100 * 50 + 3
    t = port.synth_target(n, 5)
    r = port.synth_reference(n, 6)
    wavio.write(str(tmp_path / "t.wav"), t, 44100, "PCM_24")
    wavio.write(str(tmp_path / "r.wav"), r, 44100, "PCM_24")
    mg.process(str(tmp_path / "t.wav"), str(tmp_path / "r.wav"), [mg.pcm24(str(tmp_path / "o.wav"))],
               preview_target=mg.pcm16(str(tmp_path / "pt.wav")), preview_result=mg.Result(str(tmp_path / "pr.wav"), "FLOAT"))
    t_file, _ = wavio.read(str(tmp_path / "t.wav"))
    r_file, _ = wavio.read(str(tmp_path / "r.wav"))
    cfg = mg.Config()
    result = port.main(t_file, r_file, port.config_from(cfg), True, False, False)[0]
    index, want_t, want_r = port.preview_pieces(t_file, result, cfg)
    got_t, _ = wavio.read(str(tmp_path / "pt.wav"))
    got_r, _ = wavio.read(str(tmp_path / "pr.wav"))
    assert got_t.shape == want_t.shape == (30 * 44100, 2) and got_r.shape == want_r.shape
    assert np.abs(got_r - want_r).max() < TOL
    assert np.abs(got_t - want_t).max() < 1.6 / 32768
    assert got_r[0].tolist() == [0.0, 0.0]


@pytest.mark.parametrize("one_sided", [False, True])
def test_tonal_material_with_digital_silence(torch_cuda, one_sided):
    import port
    from matchering_b200 import stages
    cfg = _config(max_piece_size=1.5)
    n = 44100 * 8
    t = 0.5 * port.synth_tonal(n, 1)
    r = np.tanh(2.0 * port.synth_tonal(n + 500, 2)).astype(np.float32)
    if one_sided:
        t[:, 1] = 0.0
        t[:, 0] += 0.05
    got = stages.main(t, r, cfg, True, True, True)
    want = port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True)
    _compare(got, want)


def test_single_call_host_entry(torch_cuda, lib):
    """mgb_process_host: host buffers in, all three outputs and the scalars back, one call."""
    import ctypes as C
    torch = torch_cuda
    import port
    from matchering_b200 import _native, stages
    from matchering_b200.engine import TrackSession, get_plan
    cfg = _config(max_piece_size=2.0)
    n, m = 250007, 240000
    t = torch.from_numpy(port.synth_target(n, 61)).pin_memory()
    r = torch.from_numpy(port.synth_reference(m, 62)).pin_memory()
    plan = get_plan(cfg)
    s = TrackSession(plan, n, m)
    dev = plan.device
    d_t, d_r = torch.empty((n, 2), device=dev), torch.empty((m, 2), device=dev)
    d_out = torch.empty((n, 2), device=dev)
    outs = [torch.zeros((n, 2)).pin_memory() for _ in range(3)]
    state = _native.TrackState()
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    _native.check(lib, lib.mgb_process_host(C.byref(plan.struct), C.byref(s.layout), t.data_ptr(), r.data_ptr(),
                                            outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), d_t.data_ptr(),
                                            d_r.data_ptr(), s.result.data_ptr(), d_out.data_ptr(), s.workspace.data_ptr(),
                                            s.state.data_ptr(), C.byref(state), stream))
    torch.cuda.synchronize()
    want = stages.main(t.numpy(), r.numpy(), cfg, True, True, True)
    for got, ref in zip(outs, want):
        assert np.abs(got.numpy() - ref).max() < 1e-6
    assert state.steps_done == 4 and state.limiter_engaged == 1


@pytest.mark.parametrize("fft_size", [2048, 4096])
def test_both_convolution_frame_lengths_against_oracle(torch_cuda, lib, fft_size):
    """Overlap-save frames of 4 FIR lengths (default where the kernel exists) and of 2, ragged ends, piece
    boundaries inside frames."""
    import port
    from matchering_b200 import stages
    cfg = _config(fft_size=fft_size, max_piece_size=1.0)
    n = 44100 * 6 + 5
    t, r = port.synth_target(n, 31), port.synth_reference(n - 999, 32)
    want = port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True)
    got = {}
    try:
        for frame in (2, 4):
            assert lib.mgb_set_option(b"conv_frame", frame) == 0
            got[frame] = stages.main(t, r, cfg, True, True, True)
            _compare(got[frame], want)
    finally:
        lib.mgb_set_option(b"conv_frame", 4)
    assert np.abs(got[2][1] - got[4][1]).max() < 2e-6
    assert lib.mgb_set_option(b"conv_frame", 3) != 0


def test_kernel_variants_behind_switches_agree(torch_cuda, lib):
    """The convolution with one CTA per frame (conv_persistent = 0; default: one CTA per SM walks its frames, the next
    frame's bulk copy under the epilogue) and the analysis that reads every twiddle from its table (analyze_chain = 0;
    default: powers built in registers): every combination against the oracle and against each other, on a track
    long enough that every CTA of the persistent grid takes several frames."""
    import port
    from matchering_b200 import stages
    cfg = _config(max_piece_size=15.0)
    n = 44100 * 120 + 77  # 431 frames of 12288 outputs on 132 SMs: three or four per CTA
    t, r = port.synth_target(n, 41), port.synth_reference(n - 4321, 42)
    want = port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True)
    got = {}
    try:
        for persistent in (0, 1):
            for chain in (0, 1):
                assert lib.mgb_set_option(b"conv_persistent", persistent) == 0
                assert lib.mgb_set_option(b"analyze_chain", chain) == 0
                got[persistent, chain] = stages.main(t, r, cfg, True, True, True)
                _compare(got[persistent, chain], want)
    finally:
        lib.mgb_set_option(b"conv_persistent", 1)
        lib.mgb_set_option(b"analyze_chain", 1)
    for key, outs in got.items():
        for a, b in zip(outs, got[0, 0]):
            # (the per-piece sums are accumulated with atomics: even one variant is not bit-identical between runs)
            assert np.abs(a - b).max() < 2e-6, key


def test_host_seam_results_are_owned_by_the_caller(torch_cuda):
    """stages.main(numpy) returns arrays in pooled pinned memory: two live results never share memory,
    a dropped result's block is reused, and the inputs are not touched (SURVEY.md 8b ownership)."""
    import gc
    import port
    from matchering_b200 import stages
    from matchering_b200.engine import HostIO
    cfg = _config(max_piece_size=2.0)
    t, r = port.synth_target(150000, 71).astype(np.float64), port.synth_reference(140000, 72).astype(np.float64)
    t0, r0 = t.copy(), r.copy()
    a = stages.main(t, r, cfg)[0]
    a_copy = a.copy()
    b = stages.main(t * 0.5, r, cfg)[0]
    assert a.dtype == np.float64 and a.flags["WRITEABLE"] and not np.shares_memory(a, b)
    assert np.array_equal(a, a_copy) and np.array_equal(t, t0) and np.array_equal(r, r0)
    addr = a.ctypes.data
    view = a[::2]  # a view keeps the block alive after `a` is gone
    del a
    gc.collect()
    c = stages.main(t, r, cfg)[0]
    assert c.ctypes.data != addr and np.array_equal(view, a_copy[::2])
    del view, c
    gc.collect()
    pool = HostIO.get().pool
    assert pool.cached > 0
    d = stages.main(t, r, cfg)[0]
    assert np.abs(d - a_copy).max() < 1e-6
    want = port.main(t, r, cfg)[0]
    assert np.abs(d - want).max() < TOL


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_host_seam_matches_device_path(torch_cuda, dtype):
    """numpy in (one native call, worker-thread upload, pinned results) == torch in (staged calls)."""
    torch = torch_cuda
    import port
    from matchering_b200 import stages
    from matchering_b200.limiter import limit
    cfg = _config(max_piece_size=3.0)
    # several ring wraps: 1.3 M samples per signal against 1 Mi-sample chunks x 6
    t, r = port.synth_target(660000 + 123, 81), port.synth_reference(600000, 82)
    dev = stages.main(torch.from_numpy(t).cuda(), torch.from_numpy(r).cuda(), cfg, True, True, True)
    host = stages.main(t.astype(dtype), r.astype(dtype), cfg, True, True, True)
    for h, d in zip(host, dev):
        assert h.dtype == dtype and np.abs(h - d.cpu().numpy()).max() < 1e-6
    x = port.synth_limiter_input(500000, 3)
    yd = limit(torch.from_numpy(x).cuda(), cfg).cpu().numpy()
    yh = limit(x.astype(dtype), cfg)
    assert yh.dtype == dtype and np.array_equal(yh.astype(np.float32), yd)
    quiet = (0.1 * x).astype(dtype)
    assert limit(quiet, cfg) is quiet


def test_checker_rule_on_the_device(torch_cuda):
    """matchering/checker.py:75-87 through device_io.check_on_device (mgb_check_peaks): the same cases and
    expected warnings as tests/test_checker_parity.py, which pins them to the live reference."""
    torch = torch_cuda
    import matchering_b200 as mg
    from matchering_b200.device_io import check_on_device
    from matchering_b200.log import Code
    from matchering_b200.log.explanations import explain
    from test_checker_parity import CASES
    for label, array, expected in CASES:
        seen = []
        mg.log(warning_handler=seen.append)
        try:
            check_on_device(torch.from_numpy(array.astype(np.float32)).cuda(), mg.Config(), "target")
        finally:
            mg.log()
        assert seen == [explain(Code(c), False) for c in expected], label


def test_device_pcm_quantiser_is_bit_identical_to_the_host_writer(torch_cuda):
    """encode_pcm (device) == wavio.write's quantiser (host, float64 like libsndfile's double writers),
    including ties and values near full scale."""
    torch = torch_cuda
    from matchering_b200.engine import encode_pcm
    rng = np.random.default_rng(5)
    x = rng.uniform(-1.05, 1.05, (200000, 2)).astype(np.float32)
    for bits, top in ((16, 32767.0), (24, 8388607.0)):
        ties = ((rng.integers(-int(top), int(top), 4096) + 0.5) / top).astype(np.float32)
        x[:2048, 0], x[:2048, 1] = ties[:2048], ties[2048:]
        want = np.clip(np.rint(x.astype(np.float64) * top), -top - 1, top).astype(np.int64)
        got = encode_pcm(torch.from_numpy(x).cuda(), bits)
        if bits == 24:
            b = got.astype(np.int64).reshape(-1, 2, 3)
            val = b[..., 0] | (b[..., 1] << 8) | (b[..., 2] << 16)
            got = np.where(val >= 1 << 23, val - (1 << 24), val)
        assert np.array_equal(got.astype(np.int64), want)


@pytest.mark.parametrize("it", [1, 2])
def test_lowess_robustness_iterations_against_oracle(torch_cuda, it):
    """Config.lowess_it > 0: the design kernel runs spline / LOWESS with bisquare re-weighting / spline itself."""
    import port
    from matchering_b200 import stages
    cfg = _config(max_piece_size=1.0, lowess_it=it)
    n = 44100 * 4 + 5
    t, r = port.synth_target(n, 21), port.synth_reference(n - 999, 22)
    got = stages.main(t, r, cfg, True, True, True)
    want = port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True)
    _compare(got, want)
    plain = stages.main(t, r, _config(max_piece_size=1.0), False, True, False)[1]
    assert np.abs(plain - got[1]).max() > 1e-6  # not the it = 0 result


@pytest.mark.parametrize("hold_order,release_order,sr", [(2, 1, 44100), (1, 2, 44100), (2, 2, 96000)])
def test_limiter_second_order_filters_against_oracle(torch_cuda, hold_order, release_order, sr):
    """LimiterConfig.hold_filter_order / release_filter_order = 2 (legal, matchering/defaults.py:48-56): blocked
    scans over the filters' state vectors, 2x2 matrix carries across threads, warps and (by look-back) 130
    chunks; a short release so that the release filter shows in the output, and the default one."""
    import matchering_b200 as mg
    import port
    from matchering_b200.limiter import limit
    x = port.synth_limiter_input(600000, seed=hold_order * 10 + release_order)
    x[200000:330000] *= 0.05
    for release in (25.0, 3000.0):
        kw = dict(hold_filter_order=hold_order, release_filter_order=release_order, release=release)
        cfg = _config(internal_sample_rate=sr, limiter=mg.LimiterConfig(**kw))
        want = port.limit(x.astype(np.float64), port.OracleConfig(internal_sample_rate=sr, limiter=port.OracleLimiterConfig(**kw)))
        got = limit(x, cfg)
        err = float(np.abs(got - want).max())
        assert err < 1e-6, f"release={release}: max-abs {err} at frame {int(np.abs(got - want).max(axis=1).argmax())}"
    plain = limit(x, _config(internal_sample_rate=sr, limiter=mg.LimiterConfig(release=25.0)))
    second = limit(x, _config(internal_sample_rate=sr, limiter=mg.LimiterConfig(
        release=25.0, hold_filter_order=hold_order, release_filter_order=release_order)))
    assert np.abs(plain - second).max() > 1e-4


def test_pipeline_with_second_order_limiter_filters(torch_cuda):
    import matchering_b200 as mg
    import port
    from matchering_b200 import stages
    kw = dict(hold_filter_order=2, release_filter_order=2, release=40.0)
    cfg = _config(max_piece_size=1.0, limiter=mg.LimiterConfig(**kw))
    n = 44100 * 4 + 5
    t, r = port.synth_target(n, 21), port.synth_reference(n - 999, 22)
    got = stages.main(t, r, cfg, True, True, True)
    want = port.main(t.astype(np.float64), r.astype(np.float64),
                     port.OracleConfig(max_piece_size=1.0, limiter=port.OracleLimiterConfig(**kw)), True, True, True)
    _compare(got, want)


@pytest.mark.parametrize("rate_in", [48000, 22050, 96000])
def test_device_resampler_against_oracle(torch_cuda, rate_in):
    """matchering_b200.resample (mgb_resample) against the oracle's restatement of resampy.resample (kaiser_best)."""
    torch = torch_cuda
    import resample as oracle_resample
    from matchering_b200.resample import resample_on_device
    rng = np.random.default_rng(rate_in)
    x = rng.uniform(-0.9, 0.9, (rate_in * 2 + 17, 2)).astype(np.float32)
    want = oracle_resample.resample(x.astype(np.float64), rate_in, 44100)
    got = resample_on_device(torch.from_numpy(x).cuda(), rate_in, 44100).cpu().numpy()
    assert got.shape == want.shape and np.abs(got - want).max() < 2e-7


def test_process_resamples_files_on_the_device(torch_cuda, tmp_path):
    """mg.process with a 48 kHz 24-bit target and a 22.05 kHz 16-bit reference: both are resampled to the internal
    44.1 kHz on the device (the reference resamples with resampy on the host, matchering/checker.py:30-44), the
    target's resampling is announced as a warning, the reference's as an info, like in the reference."""
    import matchering_b200 as mg
    import port
    import resample as oracle_resample
    from matchering_b200 import wavio
    t48 = port.synth_target(48000 * 5, 3)
    r22 = port.synth_reference(22050 * 6, 4)
    wavio.write(str(tmp_path / "t.wav"), t48, 48000, "PCM_24")
    wavio.write(str(tmp_path / "r.wav"), r22, 22050, "PCM_16")
    warnings_seen, infos_seen = [], []
    mg.log(warning_handler=warnings_seen.append, info_handler=infos_seen.append)
    try:
        mg.process(str(tmp_path / "t.wav"), str(tmp_path / "r.wav"), [mg.Result(str(tmp_path / "o.wav"), "FLOAT", use_limiter=False)],
                   config=mg.Config(max_piece_size=2.0))
    finally:
        mg.log()
    assert any("resampl" in w.lower() for w in warnings_seen) and any("resampl" in i.lower() for i in infos_seen)
    t_dec, _ = wavio.read(str(tmp_path / "t.wav"))
    r_dec, _ = wavio.read(str(tmp_path / "r.wav"))
    t44 = oracle_resample.resample(t_dec, 48000, 44100).astype(np.float32).astype(np.float64)
    r44 = oracle_resample.resample(r_dec, 22050, 44100).astype(np.float32).astype(np.float64)
    # Result(..., use_limiter=False) keeps normalize=True: the normalised no-limiter output (results.py:26-38)
    want = port.main(t44, r44, port.OracleConfig(max_piece_size=2.0), False, False, True)[2]
    got, sr = wavio.read(str(tmp_path / "o.wav"))
    assert sr == 44100 and got.shape == want.shape and np.abs(got - want).max() < 2e-5


def test_limiter_gain_envelopes_match_golden(torch_cuda, lib, golden):
    """The limiter's two scanned envelopes on the device (mgb_test_limiter_gains) against the unmodified reference's
    private helpers: attack gain (filtfilt) and release gain (hold / release low-passes), at 44.1 and 96 kHz windows."""
    torch = torch_cuda
    import port
    from matchering_b200 import _native
    from matchering_b200.engine import limiter_params
    from matchering_b200.plan import limiter_constants
    g = golden("limiter.npz")
    x = torch.from_numpy(g["x"]).cuda()
    n = x.shape[0]

    def gains(cfg):
        params = limiter_params(limiter_constants(cfg))
        ws_bytes = int(lib.mgb_limiter_workspace_bytes(C.byref(params), n))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
        out = torch.empty((n, 2), dtype=torch.float32, device="cuda")
        flag = torch.zeros(1, dtype=torch.int32, device="cuda")
        _native.check(lib, lib.mgb_test_limiter_gains(C.byref(params), x.data_ptr(), out.data_ptr(), n, ws.data_ptr(), ws_bytes,
                                                      flag.data_ptr(), None))
        return out.cpu().numpy()

    got = gains(_config())
    assert np.abs(got[:, 0] - g["gain_attack"]).max() < 2e-7
    assert np.abs(got[:, 1] - g["gain_release"]).max() < 2e-7
    for sr in (44100, 96000):
        trace = {}
        port.limit(g["x"].astype(np.float64), port.OracleConfig(internal_sample_rate=sr), trace)
        got = gains(_config(internal_sample_rate=sr))
        assert np.abs(got[:, 0] - trace["g_att"]).max() < 2e-7
        assert np.abs(got[:, 1] - np.maximum(trace["hold_out"], trace["rel_out"])).max() < 2e-7
