"""Dithered PCM encode on the CPU: the definition's properties (oracle), the shaping filter, mgb_pcm_encode_dithered on
the emulator against the oracle byte for byte, its argument checks, the batch pipeline's dithered PCM output, the
kernel under ThreadSanitizer and in other thread orders, and the Python surface."""
import ctypes as C
import os

import numpy as np
import pytest
from scipy import signal

from emul_harness import aligned, aligned_copy, emul_lib, get_emul_plan, ptr  # (puts oracle/ on sys.path)
import dither_oracle as do
import port
import matchering_b200 as mg
from matchering_b200 import _native
from matchering_b200 import dither as dither_mod

SEEDS = (0, 1, 2 ** 64 - 1)


def params_of(h=(), seed=0):
    p = _native.DitherParams()
    p.seed = seed
    p.taps = len(h)
    for k, v in enumerate(h):
        p.h[k] = float(v)
    return p


def emul_encode(x, bits, h=(), seed=0, p=None):
    """mgb_pcm_encode_dithered on the emulator -> int16 (N, 2) or uint8 (N, 6)."""
    lib = emul_lib()
    n = len(x)
    xs = aligned_copy(np.asarray(x, np.float32).reshape(n, 2))
    out = aligned((n, 2), np.int16) if bits == 16 else aligned((n, 6), np.uint8)
    out[...] = 0x5A  # bytes the encoder must overwrite
    _native.check(lib, lib.mgb_pcm_encode_dithered(C.byref(p if p is not None else params_of(h, seed)), ptr(xs), n, bits,
                                                   ptr(out), None))
    return np.array(out)


def sine(n, fs, f, dbfs, phase=0.3):
    t = np.arange(n) / fs
    a = 10 ** (dbfs / 20)
    return np.stack([a * np.sin(2 * np.pi * f * t + phase), a * np.sin(2 * np.pi * f * t + phase + 1.0)], 1).astype(np.float32)


def ntf_power(h, freqs):
    """|NTF(e^{j 2 pi f})|^2 at f in cycles per sample."""
    k = np.arange(1, len(h) + 1)
    return np.abs(1.0 - np.exp(-2j * np.pi * np.outer(freqs, k)) @ np.asarray(h)) ** 2


# ---- the definition (oracle) ----------------------------------------------------------------------------------------
def test_hash_matches_python_integers():
    rng = np.random.default_rng(1)
    n = np.concatenate([np.arange(5), rng.integers(0, 2 ** 40, 200), [2 ** 40 - 1]])
    for seed in SEEDS + (0x0123456789ABCDEF,):
        for c in (0, 1):
            got = do.tpdf(seed, n, c)
            for k, nn in enumerate(n):
                z = do.splitmix64_int(seed + (2 * int(nn) + c + 1) * do.GOLDEN)
                assert got[k] == ((z >> 40) - ((z >> 16) & 0xFFFFFF)) / 2 ** 24
    # the published first outputs of splitmix64 seeded with 0
    assert do.splitmix64_int(do.GOLDEN) == 0xE220A8397B1DCDAF


FS = 44100
BIG = 1 << 20


@pytest.fixture(scope="module")
def quiet_sine():
    return sine(BIG, FS, 1000.0, -70.0)


def test_flat_tpdf_error_statistics(quiet_sine):
    y, e = do.quantize(quiet_sine, 16, (), 7, return_error=True)
    err = y - quiet_sine.astype(np.float64) * 32767.0
    assert np.array_equal(err, e)  # no feedback: the output error is eps
    assert abs(err.mean()) < 0.01
    assert abs(err.var() / 0.25 - 1.0) < 0.03
    assert np.abs(e).max() < 1.5


def test_shaped_error_spectrum_follows_the_ntf(quiet_sine):
    h = dither_mod.shaping_filter(FS)
    y, e = do.quantize(quiet_sine, 16, h, 11, return_error=True)
    assert np.abs(e).max() < 1.5
    err = y - quiet_sine.astype(np.float64) * 32767.0
    assert abs(err.var() / (0.25 * (1.0 + np.sum(h ** 2))) - 1.0) < 0.03
    # Each 1024-frame segment restarts the loop, and the seams fill the NTF's notch (|NTF|^2 of -23 dB at 2.9 kHz) a
    # little: up to +1.5 dB there on this material (+0.8 dB with 8192-frame segments), against a spread of about
    # +-0.7 dB elsewhere.  So 1.5 dB holds everywhere but in the notch, and 2 dB there.
    for c in (0, 1):
        f, pxx = signal.welch(err[:, c], fs=1.0, nperseg=4096, return_onesided=False, detrend=False)
        want = 0.25 * ntf_power(h, f)
        dev = np.abs(10 * np.log10(pxx / want))
        notch = want < 0.25 * 10 ** (-20 / 10)
        assert dev[~notch].max() < 1.5, (c, float(dev[~notch].max()))
        assert dev[notch].max() < 2.0, (c, float(dev[notch].max()))


def test_dither_removes_truncation_harmonics():
    """A -90 dBFS 997 Hz sine at 16 bits: plain rounding leaves a 3rd harmonic far above the error's floor, flat TPDF
    leaves none."""
    x = sine(BIG, FS, 997.0, -90.0)
    u = x.astype(np.float64) * 32767.0
    k3 = int(round(3 * 997.0 / FS * 8192))

    def excess_db(err):
        _, pxx = signal.welch(err, fs=1.0, nperseg=8192)
        return 10 * np.log10(pxx[k3] / np.median(pxx))

    plain = do.plain(x, 32767.0) - u
    dithered = do.quantize(x, 16, (), 3) - u
    for c in (0, 1):
        assert excess_db(plain[:, c]) >= 25.0, c
        assert abs(excess_db(dithered[:, c])) <= 3.0, c


# ---- the shaping filter ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fs", [8000, 44100, 48000, 88200, 96000, 192000, 384000])
def test_shaping_filter_shape(fs):
    h = dither_mod.shaping_filter(fs)
    assert h.shape == (12,) and h.dtype == np.float64 and np.isfinite(h).all()
    h[0] = 0.0  # (a copy of the cached taps each time)
    assert dither_mod.shaping_filter(fs)[0] != 0.0
    # the design's NTF before truncation is monic: its first 12 taps after the leading 1 are these, at every length
    assert np.array_equal(dither_mod.shaping_filter(fs, 20)[:12], dither_mod.shaping_filter(fs))


def test_shaping_filter_at_44k1_and_its_weighted_noise():
    want = [1.6974, -1.2842, 0.0716, 0.4757, -0.2754, -0.2648, 0.1820, 0.0499, -0.1989, -0.0237, 0.1045, -0.0620]
    assert np.abs(dither_mod.shaping_filter(44100) - want).max() < 1e-4
    for fs, bound in ((44100, -9.0), (48000, -9.0), (88200, -12.0), (96000, -12.0)):
        assert dither_mod.weighted_noise_db(dither_mod.shaping_filter(fs), fs) <= bound, fs


# ---- the device encoder against the oracle (emulator) ---------------------------------------------------------------
FRAMES = [1, 7, 31, 32, 33, 1023, 1024, 1025, 3 * 1024 + 5]


def material(n, seed):
    """Full-scale material with a quiet passage, exact +-1, values beyond +-1, -0.0 and one NaN sample."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1.25, 1.25, (n, 2)).astype(np.float32)
    x[n // 3:2 * n // 3] *= np.float32(1e-4)
    special = [1.0, -1.0, -0.0, 0.0, 1.5, -3.0, np.nan, 1.0 - 2 ** -24, -1.0 + 2 ** -24, 0.5 / 32767]
    for k, v in enumerate(special):
        if 2 * k + 1 < 2 * n:
            x.reshape(-1)[(2 * k + 1) * 37 % (2 * n)] = v
    return x


def taps_of(K):
    if K == 12:
        return dither_mod.shaping_filter(44100)
    rng = np.random.default_rng(K)
    return rng.normal(0.0, 0.4, K)


@pytest.mark.parametrize("bits", [16, 24])
@pytest.mark.parametrize("K", [0, 1, 12, 32])
def test_encoder_matches_oracle_emulated(bits, K):
    h = taps_of(K)
    for i, n in enumerate(FRAMES):
        x = material(n, 100 * K + i)
        seed = SEEDS[i % len(SEEDS)]
        got = emul_encode(x, bits, h, seed)
        np.testing.assert_array_equal(got, do.encode(x, bits, h, seed), err_msg=f"{n} frames, seed {seed}")


@pytest.mark.parametrize("bits", [16, 24])
def test_zero_padded_taps_and_seeds_emulated(bits):
    n = 3 * 1024 + 5
    x = material(n, 5)
    h = dither_mod.shaping_filter(44100)
    for seed in SEEDS:
        want = do.encode(x, bits, h, seed)
        np.testing.assert_array_equal(emul_encode(x, bits, h, seed), want)
        np.testing.assert_array_equal(emul_encode(x, bits, np.concatenate([h, np.zeros(20)]), seed), want)
    # another seed is other noise; the seed's high bits count
    assert not np.array_equal(emul_encode(x, bits, h, 2 ** 63), emul_encode(x, bits, h, 0))


def test_frames_zero_writes_nothing_emulated():
    lib = emul_lib()
    xs, out = aligned((4, 2), np.float32), aligned((4, 2), np.int16)
    out[...] = 7
    assert lib.mgb_pcm_encode_dithered(C.byref(params_of()), ptr(xs), 0, 16, ptr(out), None) == _native.MGB_OK
    assert (out == 7).all()


def test_argument_errors_emulated():
    lib = emul_lib()
    n = 64
    xs, out = aligned((n, 2), np.float32), aligned((n, 6), np.uint8)

    def call(p=None, x=None, frames=n, bits=16, o=None):
        return lib.mgb_pcm_encode_dithered(C.byref(p if p is not None else params_of()), x if x is not None else ptr(xs),
                                           frames, bits, o if o is not None else ptr(out), None)
    assert call() == _native.MGB_OK and call(bits=24) == _native.MGB_OK
    for bits in (8, 15, 20, 32, 0, -16):
        assert call(bits=bits) == _native.MGB_ERR_UNSUPPORTED, bits
    for taps in (-1, 33, 1000):
        p = params_of()
        p.taps = taps
        assert call(p) == _native.MGB_ERR_INVALID, taps
    for bad in (float("nan"), float("inf"), -float("inf")):
        p = params_of([0.5, -0.25, 0.1])
        p.h[2] = bad
        assert call(p) == _native.MGB_ERR_INVALID, bad
        p.taps = 2  # a non-finite value beyond the taps is not read
        assert call(p) == _native.MGB_OK
    p = params_of()
    p.reserved = 1
    assert call(p) == _native.MGB_ERR_INVALID
    assert lib.mgb_pcm_encode_dithered(None, ptr(xs), n, 16, ptr(out), None) == _native.MGB_ERR_INVALID
    assert call(x=C.c_void_p(0)) == _native.MGB_ERR_INVALID
    assert call(o=C.c_void_p(0)) == _native.MGB_ERR_INVALID
    assert call(x=C.c_void_p(xs.ctypes.data + 8)) == _native.MGB_ERR_INVALID
    assert call(o=C.c_void_p(out.ctypes.data + 4)) == _native.MGB_ERR_INVALID
    assert call(frames=-1) == _native.MGB_ERR_INVALID


# ---- the batch pipeline ---------------------------------------------------------------------------------------------
def _pcm16(x):
    return np.clip(np.rint(np.asarray(x, np.float64) * 32767.0), -32768, 32767).astype(np.int16)


def test_pipeline_dithers_pcm_submits_emulated():
    """A depth-2 pipeline with dither: every PCM result, paired and profiled, 16- and 24-bit, is mgb_pcm_encode_dithered
    of the float32 result the same job gives through the float32 entry (which dither leaves alone).  Without dither the
    PCM results are mgb_pcm_encode's, as before.  Enabling dither twice or after a submit, or with bad parameters, is
    refused."""
    from test_reference_profile import emul_profile
    lib = emul_lib()
    cfg = port.OracleConfig(fft_size=1024, max_piece_size=0.3)
    ep = get_emul_plan(cfg)
    lengths = [20011, 19003]
    pcm_t = [_pcm16(port.synth_target(n, 190 + k) * 1.6) for k, n in enumerate(lengths)]
    targets = [(q.astype(np.float64) / 32768.0).astype(np.float32) for q in pcm_t]
    pcm_r = _pcm16(port.synth_reference(18000, 193))
    r = (pcm_r.astype(np.float64) / 32768.0).astype(np.float32)
    blob, _ = emul_profile(cfg, r)
    h = dither_mod.shaping_filter(cfg.internal_sample_rate)
    dp = params_of(h, 2 ** 64 - 5)

    def run(with_dither):
        hnd = C.c_void_p()
        _native.check(lib, lib.mgb_pipeline_create(C.byref(ep.struct), max(lengths), len(r), 2, C.byref(hnd)))
        results, keep = {}, []
        try:
            if with_dither:
                bad = params_of(h)
                bad.taps = 40
                assert lib.mgb_pipeline_enable_dither(hnd, C.byref(bad)) == _native.MGB_ERR_INVALID
                _native.check(lib, lib.mgb_pipeline_enable_dither(hnd, C.byref(dp)))
                assert lib.mgb_pipeline_enable_dither(hnd, C.byref(dp)) == _native.MGB_ERR_INVALID  # twice
            for k in range(len(targets)):
                for kind in ("float", 16, 24):
                    for profiled in (False, True):
                        slot = C.c_int32(-1)
                        if kind == "float":
                            tt, rr, o = aligned_copy(targets[k]), aligned_copy(r), aligned((len(targets[k]), 2), np.float32)
                            rc = (lib.mgb_pipeline_submit_profiled(hnd, ptr(tt), len(tt), ptr(blob), ptr(o), C.byref(slot))
                                  if profiled else lib.mgb_pipeline_submit(hnd, ptr(tt), len(tt), ptr(rr), len(rr), ptr(o),
                                                                           C.byref(slot)))
                        else:
                            o = aligned((len(targets[k]), 2), np.int16) if kind == 16 else aligned((len(targets[k]), 6),
                                                                                                   np.uint8)
                            tt, rr = aligned_copy(pcm_t[k]), aligned_copy(pcm_r)
                            rc = (lib.mgb_pipeline_submit_pcm_profiled(hnd, ptr(tt), 16, len(tt), ptr(blob), ptr(o), kind,
                                                                       C.byref(slot)) if profiled
                                  else lib.mgb_pipeline_submit_pcm(hnd, ptr(tt), 16, len(tt), ptr(rr), 16, len(rr), ptr(o),
                                                                   kind, C.byref(slot)))
                        _native.check(lib, rc)
                        _native.check(lib, lib.mgb_pipeline_wait(hnd, slot.value, None))
                        keep.append((tt, rr))
                        results[(k, kind, profiled)] = np.array(o)
            if with_dither:
                assert lib.mgb_pipeline_enable_dither(hnd, C.byref(dp)) == _native.MGB_ERR_INVALID  # after a submit
        finally:
            lib.mgb_pipeline_destroy(hnd)
        return results

    dithered, plain = run(True), run(False)
    for (k, kind, profiled), o in dithered.items():
        f32 = dithered[(k, "float", profiled)]
        np.testing.assert_array_equal(dithered[(k, "float", profiled)], plain[(k, "float", profiled)])
        if kind == "float":
            continue
        np.testing.assert_array_equal(o, emul_encode(f32, kind, p=dp), err_msg=str((k, kind, profiled)))
        np.testing.assert_array_equal(plain[(k, kind, profiled)], emul_plain_encode(f32, kind))
        assert not np.array_equal(o, plain[(k, kind, profiled)])


def emul_plain_encode(x, bits):
    lib = emul_lib()
    xs = aligned_copy(np.asarray(x, np.float32))
    out = aligned((len(x), 2), np.int16) if bits == 16 else aligned((len(x), 6), np.uint8)
    _native.check(lib, lib.mgb_pcm_encode(ptr(xs), bits, ptr(out), 2 * len(x), None))
    return np.array(out)


# ---- Python surface -------------------------------------------------------------------------------------------------
def test_result_validation():
    assert mg.pcm16("a.wav").dither is None and mg.pcm16("a.wav").dither_seed == 0
    r = mg.pcm16("a.wav", dither="shaped", dither_seed=5)
    assert (r.subtype, r.dither, r.dither_seed) == ("PCM_16", "shaped", 5)
    assert mg.pcm24("a.wav", dither="tpdf").dither == "tpdf"
    assert mg.Result("a.wav", "PCM_24", use_limiter=False, dither="tpdf", dither_seed=2 ** 64 - 1).dither_seed == 2 ** 64 - 1
    for subtype in ("PCM_32", "FLOAT", "DOUBLE"):
        with pytest.raises(ValueError):
            mg.Result("a.wav", subtype, dither="tpdf")
    for kind in ("TPDF", "rpdf", "", True):
        with pytest.raises(ValueError):
            mg.pcm16("a.wav", dither=kind)
    for seed in (-1, 2 ** 64, 1.5, "1", True):
        with pytest.raises(ValueError):
            mg.pcm16("a.wav", dither="tpdf", dither_seed=seed)
    assert mg.Result("a.wav", "FLOAT").dither is None  # no dither: every subtype as before


def test_non_wav_dither_is_refused(monkeypatch):
    from matchering_b200 import results
    monkeypatch.setattr(results, "_check_format", lambda ext, subtype=None: True)  # as if libsndfile knew FLAC
    with pytest.raises(ValueError):
        mg.Result("a.flac", "PCM_16", dither="shaped")
    assert mg.Result("a.flac", "PCM_16").dither is None


def test_params_of_each_kind():
    p = dither_mod.params("tpdf", 44100, 9)
    assert (p.seed, p.taps, p.reserved) == (9, 0, 0)
    p = dither_mod.params("shaped", 48000, 2 ** 64 - 1)
    assert p.seed == 2 ** 64 - 1 and p.taps == 12
    assert list(p.h[:12]) == list(dither_mod.shaping_filter(48000)) and not any(p.h[12:])
    with pytest.raises(ValueError):
        dither_mod.params("other", 44100)


# ---- the kernel under ThreadSanitizer and in other thread orders ----------------------------------------------------
HERE = "tests/test_dither.py::"
DUMP_ID = HERE + "test_dump_for_thread_orders_emulated"


def test_dump_for_thread_orders_emulated():
    """Every instance on a track with a partial last tile; with MGB_DITHER_DUMP set, the bytes go to that file (the
    thread-order runs below compare them with a forward run)."""
    raws = b""
    x = material(2 * 1024 + 37, 77)
    for bits in (16, 24):
        for K in (0, 12, 32):
            got = emul_encode(x, bits, taps_of(K), 3)
            np.testing.assert_array_equal(got, do.encode(x, bits, taps_of(K), 3))
            raws += got.tobytes()
    if os.environ.get("MGB_DITHER_DUMP"):
        with open(os.environ["MGB_DITHER_DUMP"], "wb") as f:
            f.write(raws)


@pytest.fixture(scope="module")
def other_runs(tmp_path_factory):
    from concurrent.futures import ThreadPoolExecutor

    import build_emul
    from test_emul_racecheck import run_group, tsan_env
    build_emul.build(racecheck=True)
    build_emul.build()
    base = tmp_path_factory.mktemp("dither_racecheck")
    jobs = {}
    env = tsan_env(str(base / "tsan"))
    env["MGB_EMUL_BUILD"] = "racecheck"
    jobs["tsan"] = ([DUMP_ID], env, str(base / "tsan"))
    for order in ("forward", "reverse", "seeded"):
        env = dict(os.environ, MGB_EMUL_ORDER=order, MGB_EMUL_SEED="4242", MGB_DITHER_DUMP=str(base / f"dump_{order}.bin"))
        jobs[order] = ([DUMP_ID], env, str(base / order))
    with ThreadPoolExecutor(max_workers=4) as ex:
        futures = {key: ex.submit(run_group, *job) for key, job in jobs.items()}
        done = {key: f.result() + (jobs[key][2],) for key, f in futures.items()}
    return done, base


def test_dither_kernel_has_no_data_races(other_runs):
    from test_emul_racecheck import reports
    rc, out, _, log_dir = other_runs[0]["tsan"]
    n, first = reports(log_dir)
    assert n == 0, f"{n} ThreadSanitizer report(s); the first:\n{first}"
    assert rc == 0, out


@pytest.mark.parametrize("order", ["reverse", "seeded"])
def test_dither_is_bit_identical_in_other_thread_orders(other_runs, order):
    done, base = other_runs
    for o in ("forward", order):
        rc, out, _, _ = done[o]
        assert rc == 0, out
    forward = (base / "dump_forward.bin").read_bytes()
    assert len(forward) > 0
    assert (base / f"dump_{order}.bin").read_bytes() == forward
