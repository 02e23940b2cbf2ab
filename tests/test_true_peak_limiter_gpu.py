"""The limiter's true-peak mode on the H100: full-size inputs through mg.limit against the float64 oracle, a 24-bit file
at -1 dBTP through mg.process, master_many's meters with and without a profile, and run-to-run agreement."""
import math

import numpy as np
import pytest

import loudness
import port
import true_peak_oracle as tpo

pytestmark = pytest.mark.gpu
C2_FRAMES = 44100 * 180
TOL = 1e-5


def assert_repeats(a, b):
    """Two device runs of the limiter agree to within two float32 ulps near full scale.  The detector and its maximum
    are order-free, but the hold and release carries cross chunks by decoupled look-back, which stops at whichever
    predecessor has published by then: the same carry summed over other predecessors differs in the last bits, in
    either mode."""
    assert float(np.abs(np.asarray(a, np.float64) - b).max()) <= 2.5e-7


def tp_db(x, fs=44100):
    return 20.0 * math.log10(float(loudness.true_peak(np.asarray(x, np.float64), fs).max()))


def test_c2_job_through_limit_against_oracle_and_repeatable():
    import matchering_b200 as mg
    from matchering_b200.limiter import limit
    cfg = mg.Config(true_peak=True)
    x = port.synth_target(C2_FRAMES, 0) * np.float32(2.0)
    got = limit(x, cfg).copy()  # (the result lives in a pooled buffer the next call reuses)
    assert float(np.abs(got - tpo.limit(x.astype(np.float64), cfg)).max()) < TOL
    assert_repeats(limit(x, cfg), got)


def test_c5_hour_through_limit_against_oracle():
    import torch

    import matchering_b200 as mg
    from matchering_b200.limiter import limit
    cfg = mg.Config(true_peak=True)
    x = port.synth_limiter_input(44100 * 3600, 0)
    got = limit(torch.from_numpy(x).cuda(), cfg).cpu().numpy()
    assert float(np.abs(got - tpo.limit(x.astype(np.float64), cfg)).max()) < TOL


def test_limit_early_out_on_true_peaks():
    """Sample peaks below the threshold, true peak above: the limiter engages.  Both below: mg.limit returns its
    input object."""
    import matchering_b200 as mg
    from matchering_b200.limiter import limit
    from test_true_peak_limiter import _sine_between_samples
    cfg = mg.Config(true_peak=True)
    x = _sine_between_samples(44100, 1.0)
    assert limit(x, mg.Config()) is x
    got = limit(x, cfg)
    assert got is not x
    assert float(np.abs(got - tpo.limit(x.astype(np.float64), cfg)).max()) < TOL
    quiet = _sine_between_samples(44100, 0.9)
    assert limit(quiet, cfg) is quiet


def test_process_to_24_bit_file_at_minus_one_dbtp(tmp_path):
    import matchering_b200 as mg
    from matchering_b200 import wavio
    t, r = port.synth_target(44100 * 12, 5), port.synth_reference(44100 * 12, 6)
    tp, rp, op = str(tmp_path / "t.wav"), str(tmp_path / "r.wav"), str(tmp_path / "out.wav")
    wavio.write(tp, t.astype(np.float64), 44100, "PCM_24")
    wavio.write(rp, r.astype(np.float64), 44100, "PCM_24")
    cfg = mg.Config(threshold=10 ** (-1 / 20), true_peak=True)
    mg.process(tp, rp, [mg.pcm24(op)], config=cfg)
    m = mg.loudness(op)
    tt, _ = mg.load(tp, "target", str(tmp_path))
    rr, _ = mg.load(rp, "reference", str(tmp_path))
    want, _, _ = tpo.main(tt.astype(np.float32), rr.astype(np.float32), cfg)
    # the oracle's overshoot for this material, plus the 24-bit quantisation
    assert m.true_peak <= tp_db(want) + 1e-3
    assert m.true_peak <= -1.0 + 0.2


def _pairs(n_tracks=4, seconds=20.0):
    rng = np.random.default_rng(11)
    lengths = [int(44100 * seconds) - int(rng.integers(0, 44100)) for _ in range(n_tracks)]
    return [(port.synth_target(n, 100 + k), port.synth_reference(int(44100 * 15), 200 + k)) for k, n in enumerate(lengths)]


@pytest.mark.parametrize("with_profile", [False, True])
def test_master_many_meters_against_oracle(with_profile):
    import matchering_b200 as mg
    from matchering_b200 import stages
    from matchering_b200.batch import master_many
    cfg = mg.Config(true_peak=True)
    pairs = _pairs()
    refs = [r for _, r in pairs]
    if with_profile:  # a profile made without true_peak serves a true-peak Config
        pairs[1] = (pairs[1][0], mg.analyze_reference(pairs[1][1], mg.Config()))
    outs, meters = master_many(pairs, cfg, depth=2, loudness=True)
    outs2 = master_many(pairs, cfg, depth=2)
    for (t, _), r, o, o2, m in zip(pairs, refs, outs, outs2, meters):
        want, want_norm, _ = tpo.main(t, r, cfg)
        assert float(np.abs(o - want).max()) < TOL
        assert abs(m.true_peak - tp_db(want)) <= 1e-4
        assert float(np.abs(o.astype(np.float64) - o2).max()) <= 1e-6  # two device runs (the limiter's path is fixed)
    t, r = pairs[0][0], refs[0]
    _, _, norm = stages.main(t, r, cfg, False, False, True)
    assert abs(tp_db(norm) - 20.0 * math.log10(cfg.threshold)) <= 1e-4


def test_wide_window_path_against_oracle_and_repeatable():
    """The wide-window path (50 ms attack, order-2 hold and release) at 96 kHz: detector, then every limiter launch."""
    import matchering_b200 as mg
    from matchering_b200.limiter import limit
    cfg = mg.Config(internal_sample_rate=96000, true_peak=True,
                    limiter=mg.LimiterConfig(attack=50, hold_filter_order=2, release_filter_order=2))
    x = port.synth_limiter_input(96000 * 60, 3)
    got = limit(x, cfg).copy()  # (the result lives in a pooled buffer the next call reuses)
    assert float(np.abs(got - tpo.limit(x.astype(np.float64), cfg)).max()) < TOL
    assert_repeats(limit(x, cfg), got)
