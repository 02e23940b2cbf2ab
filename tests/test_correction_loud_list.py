"""RMS-correction steps 2..n from the convolution's loud lists (csrc/kernels.cuh: kLoudMid): a step reads
only the mid samples loud enough to clip and takes the others' part from the step-0 sums.  Checked on the
emulator and, marked gpu, on the device: against the oracle, and the coefficients against the full-plane
formulation (every counted mid sample, from the result, clipped at every step) on the same result.  Besides
ordinary material, three tracks leave the list path: a gain above 1 / kLoudMid from the first later step on,
one that crosses it between steps, and one with more loud samples than a list holds."""
import numpy as np
import pytest

import port

TOL = 1e-5        # sample-wise max-abs bound on the float32 outputs
LOUD_MID = 0.5    # kLoudMid
CAPACITY = 0.25   # loud entries per piece, as a fraction of the piece (loud_capacity)


def _clicks(n, seed):
    """Sparse clicks in silence: clipping at step 0 takes most of their energy, so the correction gain
    exceeds 2 from the first later step on."""
    rng = np.random.default_rng(seed)
    x = np.zeros((n, 2), np.float32)
    x[rng.choice(n, 20, replace=False)] = rng.uniform(-1, 1, (20, 2))
    return x


def _spiky(n, seed):
    """Quiet noise with rare large spikes: gain 1.9 at the first later step, above 2 at the next two."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, 2)) * 0.05
    x[rng.random(n) < 0.002] *= 200
    return x.astype(np.float32)


def _case(name):
    r = port.synth_reference(35000, 32)
    if name == "ordinary":
        return port.synth_target(40000, 31), r
    if name == "gain_above_limit":
        return _clicks(40000, 5), r
    if name == "gain_crosses_limit":
        return _spiky(40000, 5), r
    if name == "list_overflow":  # a nearly square-wave reference: 43 % of the result's mid samples are loud
        return port.synth_target(40000, 31), np.tanh(30 * r).astype(np.float32)
    raise KeyError(name)


CASES = ["ordinary", "gain_above_limit", "gain_crosses_limit", "list_overflow"]


def _full_plane_coefficients(result, steps, divisions, piece, reference_match_rms, eps, correction):
    """The coefficients of steps 1..steps-1 with every counted sample re-read: mid = (L + R) / 2 of the result,
    clip(mid * float32(gain)) in float32, squares summed in float64 (stages.py:151-168)."""
    m = ((result[:, 0] + result[:, 1]) * np.float32(0.5))[: divisions * piece].reshape(divisions, piece)
    out = []
    for k in range(1, steps):
        g = np.float32(np.prod(correction[:k]))
        c = np.clip(m * g, np.float32(-1), np.float32(1)).astype(np.float64)
        rms = np.sqrt((c * c).sum(axis=1) / piece)
        avg = np.sqrt(np.mean(rms * rms))
        loud = rms >= avg
        out.append(reference_match_rms / max(eps, np.sqrt(np.mean(rms[loud] ** 2))))
    return np.array(out)


def _check_case(name, outs, st, result, divisions, piece, cfg, t, r):
    steps = cfg.rms_correction_steps
    trace = {}
    want = port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True, trace=trace)
    # (float32 results: where the clicks' result peaks at 240 before the limiter, its error is relative to that)
    scale = max(1.0, np.abs(trace["pre_limiter"]).max())
    for got, ref in zip(outs, want):
        assert np.abs(np.asarray(got, dtype=np.float64) - ref).max() < TOL * scale
    assert st.steps_done == steps
    correction = np.array([st.correction[i] for i in range(steps)])
    np.testing.assert_allclose(correction, trace["correction"], rtol=1e-6, atol=0)
    gains = np.cumprod(correction)[:-1]  # accumulated gain of steps 1..steps-1
    m = (result[:, 0] + result[:, 1]) * np.float32(0.5)
    loud_share = (np.abs(m[: divisions * piece]).reshape(divisions, piece) >= LOUD_MID).mean(axis=1)
    # each case exercises what its name says
    if name == "ordinary":
        assert gains.max() * LOUD_MID < 1 and loud_share.max() < CAPACITY
    elif name == "gain_above_limit":
        assert gains.min() * LOUD_MID > 1
    elif name == "gain_crosses_limit":
        assert gains[0] * LOUD_MID < 1 < gains[-1] * LOUD_MID
    else:
        assert loud_share.max() > CAPACITY
    want = _full_plane_coefficients(result, steps, divisions, piece, st.reference_match_rms, cfg.min_value, correction)
    # the list path takes the quiet samples' part with the float64 gain, the full plane with its float32
    # rounding: the coefficients differ by up to the half of 2^-24 that the rounding moves the sums
    np.testing.assert_allclose(correction[1:], want, rtol=1e-7, atol=0)


def _compare(outs, want):
    for got, ref in zip(outs, want):
        assert np.abs(np.asarray(got, dtype=np.float64) - ref).max() < TOL


# ---- emulator ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("steps", [0, 1, 3, 4])
def test_step_counts_against_oracle_emulated(steps):
    from emul_harness import run_pipeline
    cfg = port.OracleConfig(fft_size=1024, max_piece_size=0.3, rms_correction_steps=steps)
    t, r = _case("ordinary")
    outs, st, _, _, _ = run_pipeline(cfg, t, r)
    _compare(outs, port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True))
    assert st.steps_done == steps


@pytest.mark.parametrize("name", CASES)
def test_loud_list_and_fallback_emulated(name):
    from emul_harness import run_pipeline
    cfg = port.OracleConfig(fft_size=1024, max_piece_size=0.3, rms_correction_steps=4)
    t, r = _case(name)
    outs, st, _, result, L = run_pipeline(cfg, t, r)
    _check_case(name, outs, st, np.array(result), L.target_divisions, L.target_piece, cfg, t, r)


# ---- device --------------------------------------------------------------------------------------------
def _run_device(steps, t, r):
    import torch
    import matchering_b200 as mg
    from matchering_b200.engine import TrackSession, get_plan, to_device_f32
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    cfg = mg.Config(fft_size=1024, max_piece_size=0.3, rms_correction_steps=steps)
    plan = get_plan(cfg)
    s = TrackSession(plan, len(t), len(r))
    td, rd = to_device_f32(t, plan.device), to_device_f32(r, plan.device)
    s.match_levels(td, rd)
    s.match_frequencies(td)
    s.correct_levels()
    outs = [o.cpu().numpy() for o in s.finalize(True, True, True)]
    return cfg, outs, s.read_state(), s.result.cpu().numpy(), s.layout


@pytest.mark.gpu
@pytest.mark.parametrize("steps", [0, 1, 3, 4])
def test_step_counts_against_oracle_device(steps):
    t, r = _case("ordinary")
    cfg, outs, st, _, _ = _run_device(steps, t, r)
    _compare(outs, port.main(t.astype(np.float64), r.astype(np.float64), cfg, True, True, True))
    assert st.steps_done == steps


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_loud_list_and_fallback_device(name):
    t, r = _case(name)
    cfg, outs, st, result, L = _run_device(4, t, r)
    _check_case(name, outs, st, result, L.target_divisions, L.target_piece, cfg, t, r)
