"""The loudness meter on the H100: the EBU cases through mg.loudness, full-size tracks against the float64 oracle,
repeatability, and the batch pipeline's metering."""
import math

import numpy as np
import pytest

import loudness as oracle
import port
from test_loudness import EBU, assert_matches_oracle, sine_steps

pytestmark = pytest.mark.gpu
C2_FRAMES = 44100 * 180


def raw_of(m):
    """The Loudness as comparable tuple (bit-identity)."""
    return (m.integrated, m.loudness_range, m.momentary_max, m.short_term_max, m.sample_peak, m.true_peak,
            m.true_peak_per_channel)


def device_raw(x, fs):
    """mgb_loudness's raw result for a CUDA float32 tensor."""
    import ctypes as C

    import torch

    from matchering_b200 import _native
    from matchering_b200.engine import _stream_ptr
    from matchering_b200.loudness import device_meter
    m = device_meter(fs, x.device)
    n = int(m.lib.mgb_loudness_workspace_bytes(C.byref(m.params), len(x)))
    ws = torch.full((n,), 0xFF, dtype=torch.uint8, device=x.device)
    out = torch.empty(C.sizeof(_native.LoudnessResult), dtype=torch.uint8, device=x.device)
    _native.check(m.lib, m.lib.mgb_loudness(C.byref(m.params), x.data_ptr(), len(x), ws.data_ptr(), n, out.data_ptr(),
                                            _stream_ptr(x.device)))
    return out.cpu().numpy().tobytes()


@pytest.mark.parametrize("fs", [48000, 44100])
@pytest.mark.parametrize("name,steps,want", EBU, ids=[e[0] for e in EBU])
def test_ebu_cases_numpy_and_cuda(fs, name, steps, want):
    import torch

    import matchering_b200 as mg
    x = sine_steps(fs, steps)
    a = mg.loudness(x, fs)
    b = mg.loudness(torch.from_numpy(x.astype(np.float32)).cuda(), fs)
    assert raw_of(a) == raw_of(b)
    for field, (value, tol) in want.items():
        assert abs(getattr(a, field) - value) <= tol, (field, getattr(a, field))


def test_c2_master_against_oracle_and_repeatable():
    import torch

    import matchering_b200 as mg
    from matchering_b200 import stages
    t, r = port.synth_target(C2_FRAMES, 0), port.synth_reference(C2_FRAMES, 1)
    (out,) = [o for o in stages.main(torch.from_numpy(t).cuda(), torch.from_numpy(r).cuda(), mg.Config(), True, False,
                                     False) if o is not None]
    raw = device_raw(out, 44100)
    assert device_raw(out, 44100) == raw  # bit-identical on a second run
    assert_matches_oracle(raw, out.cpu().numpy(), 44100)


def test_c5_hour_against_streaming_oracle():
    import torch
    n = 44100 * 3600
    x = port.synth_limiter_input(n, seed=0)
    raw = device_raw(torch.from_numpy(x).cuda(), 44100)
    assert_matches_oracle(raw, x, 44100)


def test_wrong_shapes_raise():
    import torch

    import matchering_b200 as mg
    for bad in (np.zeros((1000, 1), np.float32), np.zeros((1000, 6), np.float32), np.zeros(1000, np.float32)):
        with pytest.raises(ValueError):
            mg.loudness(bad, 44100)
    with pytest.raises(ValueError):
        mg.loudness(np.zeros((1000, 2), np.float32))  # no rate
    with pytest.raises(ValueError):
        mg.loudness(np.zeros((1000, 2), np.float32), 4000)
    with pytest.raises(ValueError):
        mg.loudness(torch.zeros((1000, 2), dtype=torch.float64, device="cuda"), 44100)


def _batch(n_tracks=8, seconds=30.0):
    rng = np.random.default_rng(11)
    lengths = [int(44100 * seconds) - int(rng.integers(0, 44100)) for _ in range(n_tracks)]
    pairs = [(port.synth_target(n, 100 + k), port.synth_reference(int(44100 * 20), 200 + k)) for k, n in enumerate(lengths)]
    return pairs


def test_master_many_meters_match_mg_loudness_and_poisoned_pipeline():
    import matchering_b200 as mg
    from matchering_b200 import _native
    from matchering_b200.batch import master_many
    cfg = mg.Config()
    pairs = _batch()
    profile = mg.analyze_reference(pairs[3][1], cfg)
    pairs[3] = (pairs[3][0], profile)
    plain = master_many(pairs, cfg, depth=3)
    outs, meters = master_many(pairs, cfg, depth=3, loudness=True)
    assert len(meters) == len(pairs) and all(isinstance(m, mg.Loudness) for m in meters)
    for o, m in zip(outs, meters):
        assert raw_of(m) == raw_of(mg.loudness(o, 44100))
        assert math.isfinite(m.integrated)
    for a, b in zip(plain, outs):  # metering leaves the outputs as they were (within the device's repeat bound)
        assert float(np.abs(a.astype(np.float64) - b).max()) <= 1e-6
    lib = _native.load()
    _native.check(lib, lib.mgb_set_option(b"poison_alloc", 1))
    try:
        outs_p, meters_p = master_many(pairs, cfg, depth=2, loudness=True)
    finally:
        lib.mgb_set_option(b"poison_alloc", 0)
    for o, m in zip(outs_p, meters_p):
        assert raw_of(m) == raw_of(mg.loudness(o, 44100))


def test_pipeline_pcm_submit_meters_float_output():
    import matchering_b200 as mg
    from matchering_b200.batch import MasteringPipeline
    cfg = mg.Config()
    (t, r), = _batch(1, 10.0)
    pcm = lambda x: np.clip(np.rint(x.astype(np.float64) * 32767.0), -32768, 32767).astype(np.int16)
    t16, r16 = pcm(t), pcm(r)
    with MasteringPipeline(cfg, len(t), len(r), depth=2, loudness=True) as pipe:
        out_f = np.empty((len(t), 2), np.float32)
        out16 = np.empty((len(t), 2), np.int16)
        _, m_pcm = pipe.wait_loudness(pipe.submit_pcm(t16, r16, out16))
        tf, rf = (t16.astype(np.float32) / 32768.0), (r16.astype(np.float32) / 32768.0)
        _, m_f = pipe.wait_loudness(pipe.submit(tf, rf, out_f))
    assert raw_of(m_f) == raw_of(mg.loudness(out_f, 44100))
    assert abs(m_pcm.integrated - m_f.integrated) <= 1e-4 and abs(m_pcm.true_peak - m_f.true_peak) <= 1e-3
    with MasteringPipeline(cfg, len(t), len(r), depth=2) as pipe:
        with pytest.raises(ValueError):
            pipe.wait_loudness(0)


def test_loudness_of_a_file_written_by_process(tmp_path):
    import matchering_b200 as mg
    from matchering_b200 import wavio
    t, r = port.synth_target(44100 * 12, 5), port.synth_reference(44100 * 12, 6)
    tp, rp, op = str(tmp_path / "t.wav"), str(tmp_path / "r.wav"), str(tmp_path / "out.wav")
    wavio.write(tp, t.astype(np.float64), 44100, "PCM_24")
    wavio.write(rp, r.astype(np.float64), 44100, "PCM_24")
    mg.process(tp, rp, [mg.pcm24(op)])
    m = mg.loudness(op)
    y, sr = mg.load(op, "target", str(tmp_path))
    assert sr == 44100
    assert raw_of(m) == raw_of(mg.loudness(y, 44100))
    want = oracle.measure(y.astype(np.float32).astype(np.float64), 44100)
    assert abs(m.integrated - want["integrated"]) <= 1e-6
    assert m.true_peak >= m.sample_peak
