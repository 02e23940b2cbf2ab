"""Maxima at the kernels' seams, on the CPU emulator: the meter's sample and true peaks, its momentary and short-term
maxima, the true-peak detector d at every frame, and the limiter's output, each with its one dominant event placed at
a track edge, a chunk edge, a detector tile edge, each of a thread's frames or a sub-block edge.

A maximum hides local errors: a kernel that gets a few frames wrong fails only when one of them holds the track's
maximum.  So every case here is a quiet background (float32 white noise at -60 dBFS) with one event that dominates:
  - an inter-sample over, x[p] = x[p + 1] = 0.7, whose interpolated peak lies between the two samples;
  - an impulse, x[p] = 0.9, whose true peak is its sample peak;
  - a burst one sub-block long at -10 dBFS from p, so that the momentary and short-term maxima hang on one
    sub-block's energy and therefore on the fold's slot arithmetic at that offset.  Bursts run on tracks of at
    least 4 sub-blocks at every rate, and of at least 30 at 8 and 44.1 kHz, and a guard requires the momentary
    (and there the short-term) count to be non-zero: on shorter tracks those maxima are -inf on both sides.
The meter's interpolated points before the first frame can hold the true peak at 4x oversampling (DESIGN.md, the
loudness meter); one case puts its maximum there.
The file takes about 4.5 minutes on the emulator (8 CPU threads), most of it in about 1,300 emulated meter calls.
The seams (csrc/loudness.cuh, csrc/true_peak.cuh): the meter's chunks of kLimiterCore = 4608 frames, 512 threads of
CORE_EPT = 9 frames each with a 6-frame halo, carries combined in groups of 32 chunks, 100 ms sub-blocks; the
detector's tiles of kTpTile = 2048 frames with a 6-frame halo.  A 2048-frame tile is no seam of the meter, so the
meter's short tails are chunk tails and the detector takes both.
"""
import ctypes as C
import math

import numpy as np
import pytest

from emul_harness import aligned, aligned_copy, emul_lib, ptr  # (puts oracle/ on sys.path)
import loudness as oracle
import port
import true_peak_oracle as tpo
import matchering_b200 as mg
from matchering_b200 import _native, plan
from test_loudness import assert_matches_oracle, emul_meter

CHUNK = 4608   # kLimiterCore: the meter's and the limiter's chunk
EPT = 9        # CORE_EPT: frames per meter thread
THREADS = 512  # meter threads per chunk
TILE = 2048    # kTpTile: the detector's tile
GROUP = 32     # chunks per lookback_fixed group
RATES = [8000, 44100, 96000, 192000, 384000]

# The meter's true peak against the float64 oracle, relative.  The kernel sums the same float64 products as upfirdn,
# so only the order of the additions and FMA contraction may move the last bits.  Measured worst case: 0.0 over every
# case of this file on the emulator; 1.3e-16 (one float64 ulp) over every case of tests/test_peak_placement_gpu.py on
# an NVIDIA H100 80GB HBM3 at a 700 W power limit.
TP_REL_TOL = 1e-12
# The detector d against the oracle, in float32 ulps of the oracle's value at that frame (np.spacing): the kernel
# interpolates with float32 taps and fmaf.  Measured worst case: 3.44 ulps at 44.1 kHz on both the emulator and the
# H100 above, and 0 at 192 and 384 kHz, where d is |x| itself.
D_ULPS = 4
LIMIT_TOL = 1e-5  # the limiter's parity bound (tests/test_true_peak_limiter.py)

OVER, IMPULSE = 0.7, 0.9
BURST = 10.0 ** (-10.0 / 20.0)
NOISE = 10.0 ** (-60.0 / 20.0)


def block(fs):
    return (fs + 5) // 10


def positions(n, fs, tiles=True):
    """Frames at which to place an event in a track of n frames: both track edges, the chunk edges k * 4608 - 8 ..
    + 7 for k = 1, 2, the detector's tile edges k * 2048 - 7 .. + 6 for the first two tiles and the last (`tiles`:
    a tile is no seam of the meter), every frame of two threads (37 and 511, the chunk's last), and the sub-block
    edges k * B - 1, k * B."""
    B = block(fs)
    p = set(range(8)) | set(range(n - 8, n))
    p |= {k * CHUNK + o for k in (1, 2) for o in range(-8, 8)}
    if tiles:
        p |= {k * TILE + o for k in {1, 2, (n - 1) // TILE} if k >= 1 for o in range(-7, 7)}
    p |= {k * EPT + o for k in (37, THREADS - 1) for o in range(EPT)}
    p |= {k * B + o for k in range(1, n // B + 1) for o in (-1, 0)}
    return sorted(q for q in p if 0 <= q < n)


MAIN = 2 * CHUNK + 3                              # three chunks, the last one 3 frames long
CHUNK_TAILS = [CHUNK + r for r in range(1, 8)]    # the last chunk shorter than the halo
TILE_TAILS = [2 * TILE + r for r in range(1, 8)]  # the last tile shorter than the halo
TINY = [7, 12, 13]                                # no longer than the interpolator: one chunk holds both edges


def tail_positions(n):
    return list(range(max(0, n - 8), n))


_BACKGROUND = {}


def background(n, fs):
    """Seeded float32 white noise at -60 dBFS, built once per (rate, length); callers copy it."""
    if (n, fs) not in _BACKGROUND:
        rng = np.random.default_rng(n * 7 + fs)
        _BACKGROUND[(n, fs)] = (rng.standard_normal((n, 2)) * NOISE).astype(np.float32)
    return _BACKGROUND[(n, fs)]


def put_over(x, p, c, a=OVER):
    q = min(p, len(x) - 2)  # (at the last frame: the pair ends there)
    x[q:q + 2, c] = a


def put_burst(x, p, fs):
    """A 997 Hz sine of -10 dBFS peak over one sub-block from frame p, both channels."""
    k = np.arange(min(block(fs), len(x) - p))
    x[p:p + len(k)] = (BURST * np.sin(2.0 * np.pi * 997.0 * k / fs))[:, None].astype(np.float32)


def meter_case(n, fs, p, over_channel, burst=False):
    """The background (with a burst from p if `burst`), the inter-sample over at p in `over_channel` and the impulse at
    p in the other (each channel's peaks are reported on their own, so one call checks both events)."""
    x = background(n, fs).copy()
    if burst:
        put_burst(x, p, fs)
    put_over(x, p, over_channel)
    x[p, 1 - over_channel] = IMPULSE
    return x


def assert_meter_exact(raw, x, fs):
    """Everything within test_loudness's bounds, the sample peaks equal and the true peaks within TP_REL_TOL."""
    assert_matches_oracle(raw, x, fs)
    got = _native.LoudnessResult.from_buffer_copy(raw)
    want = oracle.true_peak(np.asarray(x, np.float32).astype(np.float64), fs)
    rel = [abs(g - w) / w for g, w in zip(got.true_peak, want)]
    assert max(rel) <= TP_REL_TOL, (list(got.true_peak), list(want), rel)
    return max(rel)


def check_meter_positions(n, fs, where, both=True, meter=emul_meter, burst=False):
    """One meter call per position (and per channel of the over, `both`) -> the worst relative true-peak error."""
    worst = 0.0
    for p in where:
        for c in ((0, 1) if both else (p % 2,)):
            x = meter_case(n, fs, p, c, burst)
            try:
                worst = max(worst, assert_meter_exact(meter(x, fs), x, fs))
            except AssertionError as e:
                raise AssertionError(f"n={n} fs={fs} event at {p}, over in channel {c}: {e}") from None
    return worst


# ---- the meter ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fs", RATES)
def test_meter_maxima_at_seams_emulated(fs):
    check_meter_positions(MAIN, fs, positions(MAIN, fs, tiles=False))


@pytest.mark.parametrize("fs", RATES)
def test_meter_maxima_in_short_tails_emulated(fs):
    """(The over alternates between the channels: test_meter_maxima_at_seams_emulated runs it in both.)"""
    for n in CHUNK_TAILS:
        check_meter_positions(n, fs, tail_positions(n), both=False)
    for n in TINY:
        check_meter_positions(n, fs, range(n), both=False)


GROUP_TRACK = 33 * CHUNK + 1234  # 34 chunks, 35 sub-blocks at 44.1 kHz


def group_positions():
    return [k * CHUNK + o for k in (31, 32, 33) for o in range(-8, 8)]


def test_meter_maxima_at_group_edges_emulated():
    """A 34-chunk track: chunk edges 31, 32 and 33 around the first group edge of lookback_fixed (chunk 32), where the
    K-weighting carries change how they are combined.  The over alternates between the channels, and a burst from
    the same frame dominates every momentary and short-term value it touches."""
    check_meter_positions(GROUP_TRACK, 44100, group_positions(), both=False, burst=True)
    x = meter_case(GROUP_TRACK, 44100, group_positions()[0], 0, burst=True)
    got = _native.LoudnessResult.from_buffer_copy(emul_meter(x, 44100))
    assert got.momentary_count > 0 and got.short_term_count > 0  # (the checks above are not -inf against -inf)


# ---- momentary and short-term maxima: one sub-block of burst -----------------------------------------------------------
def burst_track(fs, short_term=False):
    """At least 4 sub-blocks and 2 chunks (30 sub-blocks for a short-term value), plus a 3-frame tail."""
    B = block(fs)
    return max((31 if short_term else 5) * B, 2 * CHUNK + 2 * B) + 3


def burst_positions(n, fs):
    """Burst starts: every sub-block edge k B - 1, k B, and the chunk edges k * 4608 - 1, k * 4608 (k = 1, 2); each
    burst ends inside the track."""
    B = block(fs)
    p = {0} | {k * B + o for k in range(1, n // B) for o in (-1, 0)} | {k * CHUNK + o for k in (1, 2) for o in (-1, 0)}
    return sorted(q for q in p if 0 <= q <= n - B)


def check_bursts(n, fs, meter=emul_meter, short_term=False):
    """The background with one burst at each start against the oracle; the meter must report momentary (and, with
    `short_term`, short-term) values, so that those comparisons are not -inf against -inf."""
    for p in burst_positions(n, fs):
        x = background(n, fs).copy()
        put_burst(x, p, fs)
        raw = meter(x, fs)
        try:
            assert_meter_exact(raw, x, fs)
        except AssertionError as e:
            raise AssertionError(f"n={n} fs={fs} burst from {p}: {e}") from None
        got = _native.LoudnessResult.from_buffer_copy(raw)
        assert got.momentary_count > 0 and math.isfinite(got.momentary_max), (n, fs)
        if short_term:
            assert got.short_term_count > 0 and math.isfinite(got.short_term_max), (n, fs)


@pytest.mark.parametrize("fs", RATES)
def test_momentary_max_of_a_burst_at_every_sub_block_and_chunk_edge_emulated(fs):
    check_bursts(burst_track(fs), fs)


def test_short_term_max_of_a_burst_at_every_sub_block_edge_emulated():
    """8 kHz: the shortest sub-blocks, so that a chunk touches the 7 sub-blocks kMeterSlots allows for."""
    check_bursts(burst_track(8000, short_term=True), 8000, short_term=True)


def test_burst_tracks_have_momentary_and_short_term_values():
    """The guard the burst checks rely on, restated on the track lengths: at least 4 complete sub-blocks everywhere,
    30 where short-term values are checked, and sub-block and chunk edges among the starts."""
    for fs in RATES:
        n = burst_track(fs)
        assert n // block(fs) >= 4 and n > 2 * CHUNK, fs
        assert {block(fs), CHUNK, 2 * CHUNK} <= set(burst_positions(n, fs)), fs
    assert burst_track(8000, short_term=True) // block(8000) >= 30
    assert GROUP_TRACK // block(44100) >= 30


# ---- the true peak before the first frame ------------------------------------------------------------------------------
EDGE = [1.0, -1.0, 1.0, -0.5]  # at 4x oversampling its true peak, 1.116, lies a quarter sample before frame 0


def edge_case(n, fs, c):
    """The background with EDGE from frame 0 in channel c, and EDGE mirrored onto the last frames of the other (whose
    interpolated points after the last frame stay below the in-signal maximum)."""
    x = background(n, fs).copy()
    x[:len(EDGE), c] = EDGE
    x[n - len(EDGE):, 1 - c] = EDGE[::-1]
    return x


def edge_peak_before_the_signal(x, fs):
    """Whether the largest |interpolated value| of channel 0 or 1 lies before frame 0 (upfirdn's full output)."""
    from scipy import signal
    L, h = oracle.true_peak_filter(fs)
    y = np.abs(signal.upfirdn(h, np.asarray(x, np.float64)[:, 0], up=L)[:(len(x) + 12) * L])
    return int(y.argmax()) < 6 * L


@pytest.mark.parametrize("fs", [8000, 44100, 96000])
def test_meter_true_peak_before_the_first_frame_emulated(fs):
    """The interpolated points before frame 0 hold this signal's true peak at 4x oversampling, so the meter must
    evaluate them; at 96 kHz (2x) the same signal peaks inside the track."""
    for n in (13, MAIN):
        for c in (0, 1):
            x = edge_case(n, fs, c)
            assert_meter_exact(emul_meter(x, fs), x, fs)
        assert edge_peak_before_the_signal(edge_case(n, fs, 0), fs) == (oracle.true_peak_filter(fs)[0] == 4)


def test_positions_cover_every_seam():
    """The generator places events on both sides of every seam (a guard against an edit that drops one)."""
    p = set(positions(MAIN, 8000))
    assert {0, 7, MAIN - 8, MAIN - 1} <= p
    assert {CHUNK - 8, CHUNK + 7, 2 * CHUNK - 8, 2 * CHUNK + 2} <= p
    assert {TILE - 7, TILE + 6, 4 * TILE - 7, 4 * TILE + 6} <= p
    assert {EPT * 511 + e for e in range(EPT)} <= p and {EPT * 37 + e for e in range(EPT)} <= p
    assert {800 * k + o for k in range(1, 12) for o in (-1, 0)} <= p
    # 8 kHz is the rate whose sub-blocks are shortest: a chunk touches the 7 kMeterSlots allow for
    assert (CHUNK - 1) // block(8000) + 2 == 7


# ---- the detector ------------------------------------------------------------------------------------------------------
def emul_detect(x, fs):
    """mgb_test_true_peak_detect on the emulator -> (d, d_max)."""
    lib = emul_lib()
    n = len(x)
    xa, d, m = aligned_copy(x, np.float32), aligned((n,), np.float32), aligned((4,), np.float32)
    d[...] = np.nan
    _native.check(lib, lib.mgb_test_true_peak_detect(tpo.oversampling(fs), ptr(xa), n, ptr(d), ptr(m), None))
    return np.array(d), float(m[0])


def ulps(got, want):
    """|got - want| in float32 ulps of want, frame by frame."""
    w32 = np.abs(want).astype(np.float32)
    return np.abs(got.astype(np.float64) - want) / np.spacing(np.maximum(w32, np.float32(np.finfo(np.float32).tiny)))


def assert_detector_matches(d, d_max, x, fs, where=""):
    want = tpo.true_peak_detector(np.asarray(x, np.float32).astype(np.float64), fs)
    err = ulps(d, want)
    assert err.max() <= D_ULPS, f"{where}: {err.max():.1f} ulps at frame {int(err.argmax())}"
    assert np.float32(d_max).tobytes() == d.max().tobytes(), where  # bit for bit
    return float(err.max())


def detector_cases(n, fs, where):
    for p in where:
        for c in (0, 1):
            for kind in ("over", "impulse"):
                x = background(n, fs).copy()
                if kind == "over":
                    put_over(x, p, c)
                else:
                    x[p, c] = IMPULSE
                yield f"n={n} fs={fs} {kind} at {p} in channel {c}", x


@pytest.mark.parametrize("fs", RATES)
def test_detector_at_every_frame_emulated(fs):
    cases = [(MAIN, positions(MAIN, fs))]
    cases += [(n, tail_positions(n)) for n in CHUNK_TAILS + TILE_TAILS]
    cases += [(n, range(n)) for n in TINY]
    for n, where in cases:
        x = background(n, fs)
        assert_detector_matches(*emul_detect(x, fs), x, fs, f"n={n} fs={fs} noise")
        for label, x in detector_cases(n, fs, where):
            assert_detector_matches(*emul_detect(x, fs), x, fs, label)


def test_detector_rejects_bad_arguments_emulated():
    lib = emul_lib()
    x, d, m = aligned((100, 2), np.float32), aligned((100,), np.float32), aligned((4,), np.float32)
    run = lambda os_, xp, n, dp, mp: lib.mgb_test_true_peak_detect(os_, xp, n, dp, mp, None)
    assert run(4, ptr(x), 100, ptr(d), ptr(m)) == _native.MGB_OK
    for bad in (0, 3, 8, -1):
        assert run(bad, ptr(x), 100, ptr(d), ptr(m)) == _native.MGB_ERR_INVALID, bad
    for frames in (0, -5):
        assert run(4, ptr(x), frames, ptr(d), ptr(m)) == _native.MGB_ERR_INVALID, frames
    odd = lambda a: C.c_void_p(a.ctypes.data + 4)
    assert run(4, None, 100, ptr(d), ptr(m)) == _native.MGB_ERR_INVALID
    assert run(4, ptr(x), 100, None, ptr(m)) == _native.MGB_ERR_INVALID
    assert run(4, ptr(x), 100, ptr(d), None) == _native.MGB_ERR_INVALID
    assert run(4, odd(x), 99, ptr(d), ptr(m)) == _native.MGB_ERR_INVALID
    assert run(4, ptr(x), 99, odd(d), ptr(m)) == _native.MGB_ERR_INVALID
    assert run(4, ptr(x), 99, ptr(d), odd(m)) == _native.MGB_ERR_INVALID


# ---- the limiter -------------------------------------------------------------------------------------------------------
def emul_limit(x, cfg):
    lib = emul_lib()
    params = _native.LimiterParams.from_constants(plan.limiter_constants(cfg))
    n = len(x)
    nbytes = int(lib.mgb_limiter_workspace_bytes(C.byref(params), n))
    ws = aligned((nbytes,), np.uint8)
    ws[...] = 0xFF
    xi, out, engaged = aligned_copy(x, np.float32), aligned((n, 2), np.float32), aligned((4,), np.int32)
    _native.check(lib, lib.mgb_limit(C.byref(params), ptr(xi), ptr(out), n, ptr(ws), nbytes, ptr(engaged), None))
    assert engaged[0] == 1
    return np.array(out)


def limiter_positions(n):
    """The limiter's seams: track edges, its chunk edges (k = 1, 2) and, in true-peak mode, the detector's tiles."""
    p = set(range(8)) | set(range(n - 8, n))
    p |= {k * CHUNK + o for k in (1, 2) for o in range(-8, 8)}
    p |= {k * TILE + o for k in {1, 2, (n - 1) // TILE} for o in range(-7, 7)}
    return sorted(q for q in p if 0 <= q < n)


def limiter_case(n, fs, p, thr):
    """The inter-sample over at 1.2 x the threshold at p, in the left channel at even p and the right at odd."""
    x = background(n, fs).copy()
    put_over(x, p, p % 2, 1.2 * thr)
    return x


def check_limiter_positions(cfg, n, where):
    fs = cfg.internal_sample_rate
    for p in where:
        x = limiter_case(n, fs, p, cfg.threshold)
        want = (tpo.limit if cfg.true_peak else port.limit)(x.astype(np.float64), cfg)
        err = float(np.abs(emul_limit(x, cfg) - want).max())
        assert err < LIMIT_TOL, (fs, cfg.true_peak, p, err)


@pytest.mark.parametrize("true_peak", [False, True], ids=["sample-peak", "true-peak"])
@pytest.mark.parametrize("fs", [44100, 96000, 192000])
def test_limiter_events_at_seams_emulated(fs, true_peak):
    cfg = mg.Config(internal_sample_rate=fs, true_peak=true_peak)
    check_limiter_positions(cfg, MAIN, limiter_positions(MAIN))


@pytest.mark.parametrize("true_peak", [False, True], ids=["sample-peak", "true-peak"])
def test_limiter_events_at_seams_on_the_wide_window_path_emulated(true_peak):
    from test_limiter_wide_windows import span_too_wide
    cfg = mg.Config(true_peak=true_peak, limiter=mg.LimiterConfig(attack=50))
    assert span_too_wide(cfg)
    where = [0, 1, CHUNK - 1, CHUNK, TILE - 1, TILE, 2 * TILE - 1, 2 * TILE, MAIN - 2, MAIN - 1]
    check_limiter_positions(cfg, MAIN, where)
