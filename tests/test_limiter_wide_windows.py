"""The limiter's wide-window path (matchering_b200/csrc/limiter_wide.cuh): the Configs whose attack filter warm-up,
centred max and hold window do not fit the halo kernel's span -- slow attacks, long holds, attack coefficients close
to zero, 352.8 / 384 kHz -- against the unmodified reference (tests/golden/limiter_windows.npz, made by
oracle/make_golden_limiter_windows.py) and against oracle/port.py.  Bounds as for the halo kernel: 3e-7 on the
output, 2e-7 on the attack and release envelopes.

Which path ran: on the emulator through mgb_limiter_workspace_bytes (the wide-window path adds its planes and
attack look-back words; the halo kernel's workspace is unchanged), on the device through the launch names of
mgb_profile_collect."""
import ctypes as C
import json

import numpy as np
import pytest

import port
from emul_harness import aligned, aligned_copy, emul_lib, get_emul_plan, limiter_params, ptr, run_pipeline
from matchering_b200 import _native, plan as plan_mod

OUT_TOL, ENV_TOL = 3e-7, 2e-7
LENGTHS = [7, 100, 4607, 4608, 4609, 9217, 30011]
LIMIT_HEADER = 256 + 32768  # mgb_limiter_workspace_bytes before the look-back words (api.cu)


def golden_cases(g):
    """-> {name: (sample rate, OracleConfig, LimiterConfig keyword arguments)}.  Every case runs on the one input g["x"];
    the reference's output and envelopes are kept at every g["every"]-th frame."""
    out = {}
    for key in g.files:
        if key.startswith("cfg_"):
            sr, kw = json.loads(str(g[key]))
            out[key[4:]] = (sr, port.OracleConfig(internal_sample_rate=sr, limiter=port.OracleLimiterConfig(**kw)), kw)
    return out


CASE_NAMES = ["attack10", "attack50", "hold200", "hold1000", "attack1000", "coef01", "default384k", "orders22"]


def halo_workspace_bytes(cfg, n):
    """What mgb_limiter_workspace_bytes returns where the halo kernel serves the Config."""
    lim = cfg.limiter
    no = 1 if lim.hold_filter_order <= 1 and lim.release_filter_order <= 1 else 2
    return LIMIT_HEADER + ((n + 4607) // 4608 * 2 * no * 16 + 255) // 256 * 256


def span_too_wide(cfg):
    """limiter.cu limiter_span_too_wide, restated: the halo kernel's span over 512 threads exceeds 25 samples each."""
    lc = plan_mod.limiter_constants(cfg)
    lim = cfg.limiter
    no = 1 if lim.hold_filter_order <= 1 and lim.release_filter_order <= 1 else 2
    span = 4608 + max(lc.warmup, lc.hold + no - 1) + lc.warmup + 2 * lc.reach
    return -(-span // 512) > 25


def fast_limit(x, cfg):
    """port.limit with the window maxima of the reference's own calls (hyrax.py:32-40, scipy's maximum_filter1d),
    which cost O(n) where port's explicit windows cost O(n * window)."""
    from scipy import signal
    from scipy.ndimage import maximum_filter1d
    cfg = port.config_from(cfg)
    r, g = port.rectified_gain(x, cfg.threshold)
    if np.all(np.isclose(r, 1.0)):
        return x
    k = port.limiter_coefficients(cfg)
    w = k["attack"] + 1 if not k["attack"] & 1 else k["attack"]  # make_odd
    a_env = maximum_filter1d(g, size=2 * w - 1)
    half = (k["hold"] - 1) // 2
    h_env = maximum_filter1d(np.pad(a_env, (half, 0)), size=k["hold"])[:-half]
    g_att = port.one_pole_forward_backward(a_env, k["c"])
    hold_out = signal.lfilter(k["bh"], k["ah"], h_env)
    rel_out = signal.lfilter(k["br"], k["ar"], np.maximum(h_env, hold_out))
    gain = 1.0 - np.maximum(np.maximum(g, g_att), np.maximum(hold_out, rel_out))
    return x * gain[:, None]


# ------------------------------------------------------------------------------------------------ CPU only
def test_port_limit_matches_reference_golden(golden):
    g = golden("limiter_windows.npz")
    cases = golden_cases(g)
    assert sorted(cases) == sorted(CASE_NAMES)
    for name, (sr, cfg, _) in cases.items():
        k = int(g["every"])
        tr = {}
        got = port.limit(g["x"].astype(np.float64), cfg, tr)
        assert np.abs(got[::k] - g[f"y_{name}"]).max() <= 1e-12, name
        assert np.abs(tr["g_att"][::k] - g[f"att_{name}"]).max() < 1e-6, name
        assert np.abs(np.maximum(tr["hold_out"], tr["rel_out"])[::k] - g[f"rel_{name}"]).max() < 1e-6, name


def test_golden_cases_cover_the_windows_asked_for(golden):
    g = golden("limiter_windows.npz")
    cases = golden_cases(g)
    for name, (sr, cfg, _) in cases.items():
        lc = plan_mod.limiter_constants(cfg)
        n = len(g["x"])
        assert span_too_wide(cfg) == (name != "default384k"), name  # (384 kHz: the halo kernel's widest span)
        if name == "hold1000":
            assert lc.hold > n
        if name == "attack1000":
            assert 2 * lc.reach + 1 > n


def test_fast_oracle_equals_port():
    for kw, n in ((dict(attack=10.0), 3000), (dict(hold=200.0), 2500), (dict(attack=100.0), 1500), (dict(), 2000)):
        cfg = port.OracleConfig(limiter=port.OracleLimiterConfig(**kw))
        x = port.synth_limiter_input(n, seed=n).astype(np.float64)
        assert np.array_equal(fast_limit(x, cfg), port.limit(x, cfg)), kw


def test_plan_accepts_every_window_and_keeps_its_rejections():
    table = [(44100, dict(attack=10.0)), (44100, dict(hold=200.0)), (48000, dict(attack=10.0, hold=200.0)),
             (96000, dict(attack=5.0)), (96000, dict(hold=100.0)), (192000, dict(attack=3.0)), (192000, dict(hold=50.0)),
             (352800, dict()), (352800, dict(attack=2.0, hold=2.0)), (384000, dict()), (384000, dict(attack=5.0, hold=500.0)),
             (44100, dict(attack_filter_coefficient=-0.1)), (44100, dict(attack=1000.0, hold=5000.0))]
    for sr, kw in table:
        cfg = port.OracleConfig(internal_sample_rate=sr, limiter=port.OracleLimiterConfig(**kw))
        lc = plan_mod.limiter_constants(cfg)
        # the constants are the reference's (utils.py:50-55, hyrax.py:44-48)
        k = port.limiter_coefficients(cfg)
        assert (lc.reach, lc.hold, lc.attack_c) == (k["reach"], k["hold"], k["c"])
    for sr, kw in ((44100, dict(attack=0.01)), (44100, dict(hold=0.05)), (44100, dict(hold_filter_order=3)),
                   (44100, dict(release_filter_order=3)), (44100, dict(attack_filter_coefficient=0.0)),
                   (44100, dict(attack_filter_coefficient=0.5))):
        with pytest.raises(plan_mod.UnsupportedConfig):
            plan_mod.limiter_constants(port.OracleConfig(internal_sample_rate=sr, limiter=port.OracleLimiterConfig(**kw)))


# ------------------------------------------------------------------------------------------------ emulator
@pytest.fixture(scope="module")
def lib():
    return emul_lib()


def _limit(lib, x, cfg, gains=False, fill=None):
    """mgb_limit (or mgb_test_limiter_gains) on the emulator.  fill: None (zeroed workspace), or the byte pattern
    the workspace and output start from.  -> (out, engaged, workspace bytes)"""
    params = limiter_params(plan_mod.limiter_constants(cfg))
    n = len(x)
    ws_bytes = int(lib.mgb_limiter_workspace_bytes(C.byref(params), n))
    ws = aligned((ws_bytes,), np.uint8)
    out = aligned((n, 2), np.float32)
    if fill is not None:
        ws[:] = fill[:ws_bytes] if isinstance(fill, np.ndarray) else fill
        out.view(np.uint8).reshape(-1)[:] = 0xFF
    xin = aligned_copy(x, np.float32)
    engaged = aligned((4,), np.int32)
    fn = lib.mgb_test_limiter_gains if gains else lib.mgb_limit
    _native.check(lib, fn(C.byref(params), ptr(xin), ptr(out), n, ptr(ws), ws_bytes, ptr(engaged), None))
    return out, int(engaged[0]), ws_bytes


@pytest.mark.parametrize("name", CASE_NAMES)
def test_emulator_matches_reference_golden(lib, golden, name):
    g = golden("limiter_windows.npz")
    sr, cfg, _ = golden_cases(g)[name]
    x, k = g["x"], int(g["every"])
    out, engaged, ws_bytes = _limit(lib, x, cfg)
    assert engaged == 1
    assert np.abs(out[::k] - g[f"y_{name}"]).max() < OUT_TOL
    tr = {}
    assert np.abs(out - port.limit(x.astype(np.float64), cfg, tr)).max() < OUT_TOL
    wide = ws_bytes > halo_workspace_bytes(cfg, len(x))
    assert wide == span_too_wide(cfg)
    if wide:  # (the envelopes' test entry serves every wide-window Config, the halo kernel only its golden windows)
        env, _, _ = _limit(lib, x, cfg, gains=True)
        assert np.abs(env[::k, 0] - g[f"att_{name}"]).max() < ENV_TOL
        assert np.abs(env[::k, 1] - g[f"rel_{name}"]).max() < ENV_TOL
        assert np.abs(env[:, 0] - tr["g_att"]).max() < ENV_TOL
        assert np.abs(env[:, 1] - np.maximum(tr["hold_out"], tr["rel_out"])).max() < ENV_TOL


@pytest.mark.parametrize("n", LENGTHS)
@pytest.mark.parametrize("kw", [dict(attack=10.0), dict(hold=200.0, hold_filter_order=2, release=20.0),
                                dict(attack=1000.0), dict(attack_filter_coefficient=-0.1)],
                         ids=["attack10", "hold200-order2", "attack1000", "coef01"])
def test_emulator_lengths_against_port(lib, kw, n):
    """Tracks shorter than one chunk, one sample either side of a chunk boundary, and several chunks; windows both
    shorter and longer than the track."""
    cfg = port.OracleConfig(limiter=port.OracleLimiterConfig(**kw))
    assert span_too_wide(cfg)
    x = port.synth_limiter_input(max(n, 64), seed=n + 3)[:n]
    out, engaged, ws_bytes = _limit(lib, x, cfg)
    assert ws_bytes > halo_workspace_bytes(cfg, n)
    tr = {}
    want = port.limit(x.astype(np.float64), cfg, tr)
    assert engaged == 1 and np.abs(out - want).max() < OUT_TOL
    env, _, _ = _limit(lib, x, cfg, gains=True)
    assert np.abs(env[:, 0] - tr["g_att"]).max() < ENV_TOL
    assert np.abs(env[:, 1] - np.maximum(tr["hold_out"], tr["rel_out"])).max() < ENV_TOL


def test_emulator_path_boundary(lib):
    """The halo kernel serves the default Config and an 8 ms attack at 44.1 kHz; the first attack past its span takes
    the wide-window path, which matches the oracle there too."""
    n = 12000
    x = port.synth_limiter_input(n, seed=5)
    for kw in (dict(), dict(attack=8.0)):
        cfg = port.OracleConfig(limiter=port.OracleLimiterConfig(**kw))
        assert not span_too_wide(cfg)
        out, _, ws_bytes = _limit(lib, x, cfg)
        assert ws_bytes == halo_workspace_bytes(cfg, n)
        assert np.abs(out - port.limit(x.astype(np.float64), cfg)).max() < OUT_TOL
    attack = 8.0
    while not span_too_wide(port.OracleConfig(limiter=port.OracleLimiterConfig(attack=attack))):
        attack = round(attack + 0.01, 2)
    for a, wide in ((round(attack - 0.01, 2), False), (attack, True)):
        cfg = port.OracleConfig(limiter=port.OracleLimiterConfig(attack=a))
        out, _, ws_bytes = _limit(lib, x, cfg)
        assert (ws_bytes > halo_workspace_bytes(cfg, n)) == wide, a
        assert np.abs(out - port.limit(x.astype(np.float64), cfg)).max() < OUT_TOL


def test_emulator_early_out_copies_input(lib):
    cfg = port.OracleConfig(limiter=port.OracleLimiterConfig(attack=10.0))
    x = (0.2 * port.synth_limiter_input(9300, 2)).astype(np.float32)
    out, engaged, ws_bytes = _limit(lib, x, cfg, fill=0xFF)
    assert ws_bytes > halo_workspace_bytes(cfg, len(x))
    assert engaged == 0 and np.array_equal(out, x)


@pytest.mark.parametrize("kw", [dict(attack=10.0), dict(attack=10.0, hold_filter_order=2, release_filter_order=2, release=20.0)],
                         ids=["order1", "order2"])
def test_emulator_poisoned_workspace_is_bit_identical(lib, kw):
    """Every plane and look-back word the path reads is written in the same call: workspaces that start as 0xFF or
    random bytes give the clean run's bits."""
    cfg = port.OracleConfig(limiter=port.OracleLimiterConfig(**kw))
    x = port.synth_limiter_input(14000, seed=17)
    rng = np.random.default_rng(3)
    for gains in (False, True):
        clean, _, ws_bytes = _limit(lib, x, cfg, gains=gains)
        for fill in (0xFF, rng.integers(0, 256, ws_bytes, dtype=np.uint8)):
            dirty, _, _ = _limit(lib, x, cfg, gains=gains, fill=fill)
            assert np.array_equal(dirty.view(np.uint32), clean.view(np.uint32))


def _wide_pipeline_config(**kw):
    return port.OracleConfig(max_piece_size=0.25, limiter=port.OracleLimiterConfig(attack=10.0, hold=200.0), **kw)


def test_emulator_stage_calls_against_port_main(lib):
    cfg = _wide_pipeline_config()
    assert span_too_wide(cfg)
    t, r = port.synth_target(40000, 61), port.synth_reference(33333, 62)
    outs, st, _, _, L = run_pipeline(cfg, t, r)
    want = port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True)
    for a, b in zip(outs, want):
        assert np.abs(a - b).max() < 1e-5
    assert st.limiter_engaged == 1
    # the planes sit behind the limiter's zeroed region: the layout grew by exactly the path's bytes
    halo = get_emul_plan(port.OracleConfig(max_piece_size=0.25)).layout(40000, 33333)
    assert L.workspace_bytes > halo.workspace_bytes


def test_emulator_batch_pipeline_reuses_slots(lib):
    """mgb_pipeline_* at depth 2, tracks of mixed lengths: every slot runs the wide-window path several times over
    memory the previous, longer or shorter, track left behind."""
    cfg = _wide_pipeline_config()
    ep = get_emul_plan(cfg)
    lengths = [40000, 9300, 31111, 40000, 12001, 27000]
    handle = C.c_void_p()
    lib.mgb_set_option(b"poison_alloc", 1)
    try:
        _native.check(lib, lib.mgb_pipeline_create(C.byref(ep.struct), 40000, 40000, 2, C.byref(handle)))
    finally:
        lib.mgb_set_option(b"poison_alloc", 0)
    try:
        for k, n in enumerate(lengths):
            t = aligned_copy(port.synth_target(n, 70 + k), np.float32)
            r = aligned_copy(port.synth_reference(30000 + 977 * k, 80 + k), np.float32)
            o = aligned((n, 2), np.float32)
            slot = C.c_int32()
            _native.check(lib, lib.mgb_pipeline_submit(handle, ptr(t), n, ptr(r), len(r), ptr(o), C.byref(slot)))
            assert slot.value == k % 2
            st = _native.TrackState()
            _native.check(lib, lib.mgb_pipeline_wait(handle, slot.value, C.byref(st)))
            want = port.main(t.astype(np.float64), r.astype(np.float64), cfg)[0]
            assert np.abs(o - want).max() < 1e-5, (k, n)
    finally:
        lib.mgb_pipeline_destroy(handle)


# ------------------------------------------------------------------------------------------------ device
@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    return torch


@pytest.fixture(scope="module")
def dlib(torch_cuda):
    return _native.load()


def _mg_config(sr=44100, **kw):
    import matchering_b200 as mg
    return mg.Config(internal_sample_rate=sr, limiter=mg.LimiterConfig(**kw))


def _launches(dlib, fn):
    """Kernel names launched by fn()."""
    dlib.mgb_profile_enable(1)
    try:
        fn()
    finally:
        cap = 4096
        names = C.create_string_buffer(1 << 17)
        ms = (C.c_float * cap)()
        got = dlib.mgb_profile_collect(names, len(names), ms, cap)
        dlib.mgb_profile_enable(0)
    return names.value.decode().split("\n")[:got]


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_NAMES)
def test_device_matches_reference_golden(dlib, golden, name):
    from matchering_b200.limiter import limit
    g = golden("limiter_windows.npz")
    sr, cfg, kw = golden_cases(g)[name]
    x, k = g["x"], int(g["every"])
    got = {}
    names = _launches(dlib, lambda: got.setdefault("y", limit(x.astype(np.float64), _mg_config(sr, **kw))))
    assert np.abs(got["y"][::k] - g[f"y_{name}"]).max() < OUT_TOL
    assert np.abs(got["y"] - fast_limit(x.astype(np.float64), cfg)).max() < OUT_TOL
    wide = span_too_wide(cfg)
    assert ("limiter_wide_apply_kernel" in names) == wide and ("limiter_kernel" in names) == (not wide)
    if wide:
        params = limiter_params(plan_mod.limiter_constants(cfg))
        import torch
        n = len(x)
        ws_bytes = int(dlib.mgb_limiter_workspace_bytes(C.byref(params), n))
        ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")
        xin = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()
        env = torch.empty_like(xin)
        engaged = torch.zeros(4, dtype=torch.int32, device="cuda")
        _native.check(dlib, dlib.mgb_test_limiter_gains(C.byref(params), xin.data_ptr(), env.data_ptr(), n, ws.data_ptr(), ws_bytes,
                                                        engaged.data_ptr(), None))
        env = env.cpu().numpy()
        assert np.abs(env[::k, 0] - g[f"att_{name}"]).max() < ENV_TOL
        assert np.abs(env[::k, 1] - g[f"rel_{name}"]).max() < ENV_TOL


@pytest.mark.gpu
@pytest.mark.parametrize("n", LENGTHS)
@pytest.mark.parametrize("kw", [dict(attack=10.0), dict(hold=200.0, hold_filter_order=2, release=20.0), dict(attack=1000.0)],
                         ids=["attack10", "hold200-order2", "attack1000"])
def test_device_lengths_against_port(dlib, kw, n):
    from matchering_b200.limiter import limit
    cfg = port.OracleConfig(limiter=port.OracleLimiterConfig(**kw))
    x = port.synth_limiter_input(max(n, 64), seed=n + 3)[:n]
    got = limit(x, _mg_config(**kw))
    assert np.abs(got - port.limit(x.astype(np.float64), cfg)).max() < OUT_TOL


@pytest.mark.gpu
def test_device_early_out_returns_input_object(dlib):
    from matchering_b200.limiter import limit
    x = (0.2 * port.synth_limiter_input(9300, 2)).astype(np.float64)
    assert limit(x, _mg_config(attack=10.0)) is x


@pytest.mark.gpu
@pytest.mark.parametrize("seconds,sr,kw", [(180, 44100, dict(attack=10.0, hold=200.0)), (600, 96000, dict(attack=5.0))],
                         ids=["3min-44k-attack10-hold200", "10min-96k-attack5"])
def test_device_long_inputs_against_fast_oracle(dlib, seconds, sr, kw):
    from matchering_b200.limiter import limit
    x = port.synth_limiter_input(sr * seconds, seed=seconds)
    cfg = port.OracleConfig(internal_sample_rate=sr, limiter=port.OracleLimiterConfig(**kw))
    assert span_too_wide(cfg)
    names = _launches(dlib, lambda: None)  # (drain)
    got = {}
    names = _launches(dlib, lambda: got.setdefault("y", limit(x, _mg_config(sr, **kw))))
    assert "limiter_wide_apply_kernel" in names and "limiter_kernel" not in names
    assert np.abs(got["y"] - fast_limit(x.astype(np.float64), cfg)).max() < OUT_TOL


@pytest.mark.gpu
def test_device_stages_main_against_port(dlib):
    import matchering_b200 as mg
    from matchering_b200 import stages
    t, r = port.synth_target(120000, 91), port.synth_reference(100000, 92)
    for sr, kw in ((44100, dict(attack=10.0, hold=200.0)), (384000, dict())):
        cfg = mg.Config(internal_sample_rate=sr, max_piece_size=0.2 if sr == 44100 else 0.05, limiter=mg.LimiterConfig(**kw))
        got = stages.main(t, r, cfg, True, True, True)
        want = port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True)
        for a, b in zip(got, want):
            assert a.shape == b.shape and np.abs(a - b).max() < 1e-5, (sr, kw)


@pytest.mark.gpu
def test_device_process_files_with_slow_attack(dlib, tmp_path):
    import matchering_b200 as mg
    from matchering_b200 import wavio
    n = 441000
    t = port.synth_target(n, 0, kind="white")
    r = port.synth_reference(n, 1, kind="quiet")
    wavio.write(str(tmp_path / "t.wav"), t, 44100, "FLOAT")
    wavio.write(str(tmp_path / "r.wav"), r, 44100, "FLOAT")
    cfg = mg.Config(limiter=mg.LimiterConfig(attack=10))
    mg.process(str(tmp_path / "t.wav"), str(tmp_path / "r.wav"), [mg.Result(str(tmp_path / "o.wav"), "FLOAT")], config=cfg)
    got, _ = wavio.read(str(tmp_path / "o.wav"))
    want = port.main(t.astype(np.float64), r.astype(np.float64), cfg)[0]
    assert np.abs(got - want).max() < 1e-5


@pytest.mark.gpu
def test_device_batch_master_many(dlib):
    import matchering_b200 as mg
    from matchering_b200 import stages
    from matchering_b200.batch import master_many
    cfg = mg.Config(max_piece_size=3.0, limiter=mg.LimiterConfig(attack=10.0, hold=200.0))
    pairs = [(port.synth_target(300000 - 40001 * k, 20 + k), port.synth_reference(280000, 40 + k)) for k in range(5)]
    got = master_many(pairs, cfg, depth=3)
    for (t, r), o in zip(pairs, got):
        want = stages.main(t, r, cfg)[0]
        assert o.shape == want.shape and np.abs(o - want).max() < 1e-6
        assert np.abs(o - port.main(t.astype(np.float64), r.astype(np.float64), cfg)[0]).max() < 1e-5
