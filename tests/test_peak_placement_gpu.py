"""Maxima at the kernels' seams on the H100 (tests/test_peak_placement.py on the device): the same events, positions,
lengths and tolerances at 8, 44.1, 96, 192 and 384 kHz, so that every loudness_kernel<OS>, every
true_peak_detect_kernel<L> and the true-peak halo-path limiter run on the device; then a 3-minute meter at 384 kHz
across several hundred look-back groups, 10 minutes of true-peak limiting at 96 kHz, and bit-identical repeats of
the meter at each oversampling factor."""
import ctypes as C

import numpy as np
import pytest

import port
import true_peak_oracle as tpo
from test_loudness_gpu import device_raw
import test_peak_placement as placement
from test_peak_placement import (CHUNK, CHUNK_TAILS, D_ULPS, GROUP, IMPULSE, LIMIT_TOL, MAIN, RATES, TILE, TILE_TAILS,
                                 TINY, TP_REL_TOL, assert_detector_matches, assert_meter_exact, background, detector_cases,
                                 limiter_case, limiter_positions, meter_case, positions, put_burst, put_over,
                                 tail_positions)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from matchering_b200 import _native
    return torch, _native.load()


def cuda(torch, x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()


def device_detect(dev, x, fs):
    """mgb_test_true_peak_detect on the device -> (d, d_max)."""
    from matchering_b200 import _native
    from matchering_b200.engine import _stream_ptr
    torch, lib = dev
    xd = cuda(torch, x)
    d = torch.full((len(x),), float("nan"), dtype=torch.float32, device="cuda")
    m = torch.zeros(4, dtype=torch.float32, device="cuda")
    _native.check(lib, lib.mgb_test_true_peak_detect(tpo.oversampling(fs), xd.data_ptr(), len(x), d.data_ptr(),
                                                     m.data_ptr(), _stream_ptr(xd.device)))
    return d.cpu().numpy(), float(m[0].item())


def device_limit(dev, x, cfg):
    """mgb_limit on the device, on a workspace filled with 0xFF."""
    from matchering_b200 import _native, plan
    from matchering_b200.engine import _stream_ptr
    torch, lib = dev
    params = _native.LimiterParams.from_constants(plan.limiter_constants(cfg))
    n = len(x)
    nbytes = int(lib.mgb_limiter_workspace_bytes(C.byref(params), n))
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")
    xd = cuda(torch, x)
    out = torch.empty_like(xd)
    engaged = torch.zeros(4, dtype=torch.int32, device="cuda")
    _native.check(lib, lib.mgb_limit(C.byref(params), xd.data_ptr(), out.data_ptr(), n, ws.data_ptr(), nbytes,
                                     engaged.data_ptr(), _stream_ptr(xd.device)))
    assert int(engaged[0].item()) == 1
    return out.cpu().numpy()


def launches(dev, fn):
    """Kernel names launched by fn()."""
    _, lib = dev
    lib.mgb_profile_enable(1)
    try:
        fn()
    finally:
        cap = 4096
        names = C.create_string_buffer(1 << 17)
        ms = (C.c_float * cap)()
        got = lib.mgb_profile_collect(names, len(names), ms, cap)
        lib.mgb_profile_enable(0)
    return names.value.decode().split("\n")[:got]


def meter(dev):
    torch, _ = dev
    return lambda x, fs: device_raw(cuda(torch, x), fs)


def check_meter_positions(dev, n, fs, where, both=True, burst=False):
    return placement.check_meter_positions(n, fs, where, both, meter(dev), burst)


# ---- the seams, as on the emulator -------------------------------------------------------------------------------------
@pytest.mark.parametrize("fs", RATES)
def test_meter_maxima_at_seams(dev, fs):
    worst = check_meter_positions(dev, MAIN, fs, positions(MAIN, fs, tiles=False))
    for n in CHUNK_TAILS:
        worst = max(worst, check_meter_positions(dev, n, fs, tail_positions(n), both=False))
    for n in TINY:
        worst = max(worst, check_meter_positions(dev, n, fs, range(n), both=False))
    print(f"meter at {fs} Hz: worst true-peak relative error {worst:.3g} (bound {TP_REL_TOL})")


def test_meter_maxima_at_group_edges(dev):
    worst = check_meter_positions(dev, placement.GROUP_TRACK, 44100, placement.group_positions(), both=False, burst=True)
    print(f"meter at the group edges: worst true-peak relative error {worst:.3g} (bound {TP_REL_TOL})")


@pytest.mark.parametrize("fs", RATES)
def test_momentary_max_of_a_burst_at_every_sub_block_and_chunk_edge(dev, fs):
    placement.check_bursts(placement.burst_track(fs), fs, meter(dev))


def test_short_term_max_of_a_burst_at_every_sub_block_edge(dev):
    placement.check_bursts(placement.burst_track(8000, short_term=True), 8000, meter(dev), short_term=True)


@pytest.mark.parametrize("fs", [8000, 44100, 96000])
def test_meter_true_peak_before_the_first_frame(dev, fs):
    for n in (13, MAIN):
        for c in (0, 1):
            x = placement.edge_case(n, fs, c)
            assert_meter_exact(device_raw(cuda(dev[0], x), fs), x, fs)


@pytest.mark.parametrize("fs", RATES)
def test_detector_at_every_frame(dev, fs):
    cases = [(MAIN, positions(MAIN, fs))]
    cases += [(n, tail_positions(n)) for n in CHUNK_TAILS + TILE_TAILS]
    cases += [(n, range(n)) for n in TINY]
    worst = 0.0
    for n, where in cases:
        x = background(n, fs)
        worst = max(worst, assert_detector_matches(*device_detect(dev, x, fs), x, fs, f"n={n} fs={fs} noise"))
        for label, x in detector_cases(n, fs, where):
            worst = max(worst, assert_detector_matches(*device_detect(dev, x, fs), x, fs, label))
    print(f"detector at {fs} Hz: worst {worst:.2f} ulps (bound {D_ULPS})")


@pytest.mark.parametrize("true_peak", [False, True], ids=["sample-peak", "true-peak"])
@pytest.mark.parametrize("fs", [44100, 96000, 192000])
def test_limiter_events_at_seams(dev, fs, true_peak):
    import matchering_b200 as mg
    cfg = mg.Config(internal_sample_rate=fs, true_peak=true_peak)
    for p in limiter_positions(MAIN):
        x = limiter_case(MAIN, fs, p, cfg.threshold)
        want = (tpo.limit if true_peak else port.limit)(x.astype(np.float64), cfg)
        err = float(np.abs(device_limit(dev, x, cfg) - want).max())
        assert err < LIMIT_TOL, (fs, true_peak, p, err)


@pytest.mark.parametrize("true_peak", [False, True], ids=["sample-peak", "true-peak"])
def test_limiter_events_at_seams_on_the_wide_window_path(dev, true_peak):
    import matchering_b200 as mg
    cfg = mg.Config(true_peak=true_peak, limiter=mg.LimiterConfig(attack=50))
    for p in [0, 1, CHUNK - 1, CHUNK, TILE - 1, TILE, 2 * TILE - 1, 2 * TILE, MAIN - 2, MAIN - 1]:
        x = limiter_case(MAIN, 44100, p, cfg.threshold)
        want = (tpo.limit if true_peak else port.limit)(x.astype(np.float64), cfg)
        err = float(np.abs(device_limit(dev, x, cfg) - want).max())
        assert err < LIMIT_TOL, (true_peak, p, err)


@pytest.mark.parametrize("fs", RATES)
def test_every_instance_runs_on_the_device(dev, fs):
    """The meter and the detector at this rate launch their kernels (mgb_profile_collect), and at 96 and 192 kHz the
    true-peak limiter takes the halo kernel."""
    import matchering_b200 as mg
    torch, _ = dev
    x = meter_case(MAIN, fs, CHUNK, 0)
    names = launches(dev, lambda: (device_raw(cuda(torch, x), fs), device_detect(dev, x, fs)))
    assert "loudness_kernel" in names and "true_peak_detect_kernel" in names, names
    if fs in (96000, 192000):
        cfg = mg.Config(internal_sample_rate=fs, true_peak=True)
        y = limiter_case(MAIN, fs, CHUNK, cfg.threshold)
        names = launches(dev, lambda: device_limit(dev, y, cfg))
        assert "true_peak_detect_kernel" in names and "limiter_kernel" in names, names


# ---- long tracks and repeats -------------------------------------------------------------------------------------------
def test_meter_three_minutes_at_384k_at_group_edges(dev):
    """69 M frames, 15000 chunks, 469 look-back groups: the events and the burst at the first, a middle and the last
    group edge, one call each, against the streaming oracle."""
    torch, _ = dev
    fs = 384000
    n = fs * 180
    rng = np.random.default_rng(384)
    bg = (rng.standard_normal((n, 2)) * 1e-3).astype(np.float32)
    span = GROUP * CHUNK
    last = (n - 1) // span
    for g in (1, last // 2, last):
        p = g * span
        x = bg.copy()
        put_burst(x, p, fs)
        put_over(x, p, g % 2)
        x[p, 1 - g % 2] = IMPULSE
        assert_meter_exact(device_raw(cuda(torch, x), fs), x, fs)


def test_true_peak_limit_ten_minutes_at_96k():
    """10 minutes at 96 kHz through mg.limit(true_peak=True): overs at 1.2 x the threshold at the first, a middle and
    the last chunk and tile edges, against the streaming oracle."""
    import matchering_b200 as mg
    from matchering_b200.limiter import limit
    fs = 96000
    n = fs * 600
    cfg = mg.Config(internal_sample_rate=fs, true_peak=True)
    rng = np.random.default_rng(96)
    x = (rng.standard_normal((n, 2)) * 1e-3).astype(np.float32)
    for k, p in enumerate([CHUNK - 1, TILE, (n // CHUNK // 2) * CHUNK, (n // TILE // 2) * TILE - 1,
                           (n - 1) // CHUNK * CHUNK, (n - 1) // TILE * TILE - 1, n - 1]):
        put_over(x, p, k % 2, 1.2 * cfg.threshold)
    got = limit(x, cfg).copy()  # (the result lives in a pooled buffer the next call reuses)
    assert float(np.abs(got - tpo.limit(x.astype(np.float64), cfg)).max()) < LIMIT_TOL


@pytest.mark.parametrize("fs", [44100, 96000, 384000], ids=["os4", "os2", "os1"])
def test_meter_repeats_bit_for_bit(dev, fs):
    """Two device runs of one meter call give the same bytes, at each oversampling factor, on 70 chunks (three
    look-back groups) with the events at the second group's edge."""
    torch, _ = dev
    n = 70 * CHUNK + 11
    x = meter_case(n, fs, GROUP * CHUNK, 1, burst=True)
    xd = cuda(torch, x)
    raw = device_raw(xd, fs)
    assert device_raw(xd, fs) == raw
    assert_meter_exact(raw, x, fs)
