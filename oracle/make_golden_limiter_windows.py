"""ORACLE (test infrastructure only) -- generate tests/golden/limiter_windows.npz by running the UNMODIFIED
reference limiter (imported through oracle/ref_shims.py) on limiter Configs whose windows are wider than the
limiter kernel's halo: slow attacks, long holds, an attack coefficient close to zero, the default limiter at
384 kHz, and windows longer than the track itself.

Run in the build container only:  python oracle/make_golden_limiter_windows.py
One input x (float32, FRAMES stereo frames) for every case.  Per case <name>, at every EVERY-th frame (11 is prime
to the kernels' 9 samples per thread and 4608 per chunk, so the kept frames fall on every position of both):
y_<name> = matchering.limiter.limit(x) (float64), att_<name> = the filtfilt'd attack gain and rel_<name> =
max(hold_out, release_out), both through hyrax's private helpers (float32); and cfg_<name> = the case's
(internal_sample_rate, LimiterConfig keyword arguments) as JSON.  Keeping every frame would make the file
about eight times larger; the tests check every frame against oracle/port.py, which this file pins.
"""
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

# (name, internal sample rate, LimiterConfig keyword arguments)
CASES = [
    ("attack10", 44100, dict(attack=10.0)),
    ("attack50", 44100, dict(attack=50.0)),
    ("hold200", 44100, dict(hold=200.0)),
    ("hold1000", 44100, dict(hold=1000.0)),             # hold window longer than the track
    ("attack1000", 44100, dict(attack=1000.0)),         # attack window (2 x 44100 samples) longer than the track
    ("coef01", 44100, dict(attack_filter_coefficient=-0.1)),
    ("default384k", 384000, dict()),
    # orders (2, 2): a 20 ms release, or the release section never rises above the hold section in half a second
    ("orders22", 44100, dict(attack=10.0, hold_filter_order=2, release_filter_order=2, release=20.0)),
]
FRAMES = 20011
EVERY = 11


def main():
    warnings.simplefilter("ignore")
    import_reference()
    from matchering import Config
    from matchering.defaults import LimiterConfig
    from matchering.limiter import hyrax, limit
    from matchering import dsp

    x32 = port.synth_limiter_input(FRAMES, seed=448)
    out = dict(x=x32, every=EVERY)
    x = x32.astype(np.float64)
    for name, sr, kw in CASES:
        cfg = Config(internal_sample_rate=sr, limiter=LimiterConfig(**kw))
        out[f"y_{name}"] = limit(x, cfg)[::EVERY]
        g = dsp.flip(1.0 / dsp.rectify(x, cfg.threshold))
        att, slided = getattr(hyrax, "__process_attack")(np.copy(g), cfg)
        rel = getattr(hyrax, "__process_release")(np.copy(slided), cfg)
        out[f"att_{name}"] = att[::EVERY].astype(np.float32)
        out[f"rel_{name}"] = rel[::EVERY].astype(np.float32)
        out[f"cfg_{name}"] = np.array(json.dumps([sr, kw]))
    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(os.path.join(OUT, "limiter_windows.npz"), **out)


if __name__ == "__main__":
    main()
