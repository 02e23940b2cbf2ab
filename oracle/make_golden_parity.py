"""ORACLE (test infrastructure only) -- generate tests/golden/reference_parity.npz and
tests/golden/reference_surface.json: what the UNMODIFIED reference (imported through
oracle/ref_shims.py) returns for the inputs of the parity tests in tests/test_oracle_port.py,
tests/test_checker_parity.py and tests/test_cabi_and_surface.py, so that those tests compare against
the reference without needing its source tree.

    python oracle/make_golden_parity.py

Outputs compared within a tolerance are too large to store whole: they are kept as every STRIDE-th row
plus sums (and, per channel, sums of squares) of the whole arrays.  Outputs compared for exact equality
(sliding maxima, mid/side, preview pieces) are kept as SHA-256 digests of their bytes.
"""
import hashlib
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import port  # noqa: E402
from ref_shims import import_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

MAIN_CASES = [(44100, 6.0), (96000, 2.5)]
MAIN_STRIDE = 1031
ATTACK_STRIDE = 5
PREVIEW_CASES = [30000, 9000, 12000 + 4000 * 3]
# the checker's error messages for the two rejected inputs of test_check_order_and_scaled_minimum_length
CHECKER_ERRORS = [("channels_22050", (3000, 3), "reference"), ("short_22050", (2000, 2), "target")]


def digest(a: np.ndarray) -> str:
    a = np.ascontiguousarray(a)
    return f"{a.dtype.str}{a.shape}:" + hashlib.sha256(a.tobytes()).hexdigest()


def identity_inputs():
    """The inputs of test_identities_against_reference_helpers (same seed, same draw order)."""
    rng = np.random.default_rng(5)
    g = np.abs(rng.standard_normal(5000)) * (rng.uniform(size=5000) > 0.7)
    pieces = rng.standard_normal((3, 20000))
    x = rng.standard_normal((1000, 2))
    return g, pieces, x


def main_inputs(sr, seconds):
    n = int(sr * seconds)
    return port.synth_target(n, 3).astype(np.float64), port.synth_reference(n - 777, 4).astype(np.float64)


def preview_inputs(n):
    target = 2.5 * port.synth_target(n, 41).astype(np.float64)
    result = port.synth_reference(n, 42).astype(np.float64) * (0.2 + np.abs(np.sin(np.linspace(0, 9, n))))[:, None]
    return target, result


def main():
    warnings.simplefilter("ignore")
    ref = import_reference()
    from matchering import Config, Result, dsp, preview_creator, stages
    from matchering.limiter import hyrax
    from matchering.log.codes import Code
    from matchering.log.exceptions import ModuleError
    from matchering.stage_helpers import match_frequencies as mf

    arrays, surface = {}, {}
    # ---- helper identities (exact ones as digests)
    g, pieces, x = identity_inputs()
    exact = {}
    for attack in (44, 45, 96):
        exact[f"attack_window_{attack}"] = digest(getattr(hyrax, "__sliding_window_fast")(g, attack, "attack"))
    for hold in (44, 45, 96, 3):
        exact[f"hold_window_{hold}"] = digest(getattr(hyrax, "__sliding_window_fast")(g, hold, "hold"))
    mid, side = dsp.lr_to_ms(x)
    exact["mid"], exact["side"] = digest(mid), digest(side)
    surface["identity_digests"] = exact
    att = getattr(hyrax, "__process_attack")(np.copy(g), Config())[0]
    arrays["process_attack_rows"] = att[::ATTACK_STRIDE]
    arrays["process_attack_sum"] = att.sum()
    arrays["attack_stride"] = np.int64(ATTACK_STRIDE)
    arrays["average_fft"] = getattr(mf, "__average_fft")(pieces, 44100, 4096)

    # ---- whole pipeline
    for sr, seconds in MAIN_CASES:
        t, r = main_inputs(sr, seconds)
        outs = stages.main(t, r, Config(internal_sample_rate=sr, max_piece_size=1.0), True, True, True)
        for name, a in zip(("limited", "no_limiter", "normalized"), outs):
            key = f"main_{sr}_{name}"
            arrays[key + "_rows"] = a[::MAIN_STRIDE]
            arrays[key + "_sum"] = a.sum(axis=0)
            arrays[key + "_sumsq"] = (a * a).sum(axis=0)
    arrays["main_stride"] = np.int64(MAIN_STRIDE)
    np.savez_compressed(os.path.join(OUT, "reference_parity.npz"), **arrays)

    # ---- preview pieces: the arrays the reference hands to its two `save` calls
    cfg = Config(internal_sample_rate=2000, preview_size=6, preview_analysis_step=2)
    original_save = preview_creator.save
    previews = {}
    for n in PREVIEW_CASES:
        saved = {}
        preview_creator.save = lambda file, arr, sr, subtype, name: saved.__setitem__(name, arr.copy())
        try:
            target, result = preview_inputs(n)
            preview_creator.create_preview(target, result, cfg, Result("t.wav", "PCM_16"), Result("r.wav", "PCM_16"))
        finally:
            preview_creator.save = original_save
        previews[str(n)] = {"target": digest(saved["target preview"]), "result": digest(saved["result preview"])}
    surface["preview_digests"] = previews

    # ---- public surface: Config attributes, log codes, checker warnings and errors
    theirs = Config(internal_sample_rate=48000, max_piece_size=7.5)
    surface["config_48000_7.5"] = {k: (vars(v) if k == "limiter" else v) for k, v in vars(theirs).items()}
    surface["log_codes"] = {c.name: int(c) for c in Code}
    sys.path[:0] = [os.path.dirname(HERE), os.path.join(os.path.dirname(HERE), "tests")]
    from test_checker_parity import CASES
    warnings_seen = {}
    for label, array, _ in CASES:
        seen = []
        ref.log(warning_handler=seen.append)
        try:
            ref.checker.check(array.copy(), 44100, Config(), "target")
        finally:
            ref.log()
        warnings_seen[label] = seen
    surface["checker_warnings"] = warnings_seen
    errors = {}
    for key, shape, name in CHECKER_ERRORS:
        try:
            ref.checker.check(np.zeros(shape), 22050, Config(), name)
            errors[key] = None
        except ModuleError as e:
            errors[key] = str(e)
    surface["checker_errors"] = errors
    with open(os.path.join(OUT, "reference_surface.json"), "w") as f:
        json.dump(surface, f, indent=1, sort_keys=True)
        f.write("\n")
    for name in ("reference_parity.npz", "reference_surface.json"):
        print(name, os.path.getsize(os.path.join(OUT, name)) // 1024, "KiB")


if __name__ == "__main__":
    main()
