"""What linked versions cost on the device.  Prints one JSON line: the GPU and its power limit, then for a 3-minute mix
of the C2 recipe (instrumental + vocal-like part) and three versions (instrumental, a cappella, TV mix) against a
3-minute reference profile, the device time of
  - the main plus three versions as one linked job (stages.main_versions_device, the limited output), and
  - four independent jobs on the same data (stages.main_device per target),
in both peak modes, alternating, median and p10-p90 spread of repeats after a warm-up; CUDA events around each run.
Also the HBM floor of the linked detector and apply work: bytes those passes must move at 3.35 TB/s.
Read-only: writes nothing but stdout."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from album_loudness_cost import timed  # noqa: E402
from reference_profile_bench import gpu_info  # noqa: E402

SECONDS = 180
VERSIONS = 3
HBM_BYTES_PER_S = 3.35e12


def main():
    import numpy as np
    import torch

    import matchering_b200 as mg
    import port
    from matchering_b200 import analyze_reference, stages
    from matchering_b200.engine import get_plan, to_device_f32
    n = 44100 * SECONDS
    result = {}
    for tp in (False, True):
        cfg = mg.Config(true_peak=tp)
        dev = get_plan(cfg).device
        prof = analyze_reference(port.synth_reference(n, 1000), cfg)
        a = port.synth_target(n, 1).astype(np.float64) * 0.6
        b = port.synth_tonal(n, 2).astype(np.float64) * 0.35
        xs = [to_device_f32(np.ascontiguousarray(v.astype(np.float32)), dev) for v in (a + b, a, b, a + 0.5 * b)]
        result["true_peak" if tp else "sample_peak"] = timed({
            "linked": lambda: stages.main_versions_device(xs, prof, cfg, True, False, False),
            "independent": lambda: [stages.main_device(x, prof, cfg, True, False, False) for x in xs],
        })
    entries = 1 + VERSIONS
    # detector: read every entry's result (8 B/frame), write D (4 B/frame); apply: read D's halo-free share and every
    # entry's result, write every entry's output (8 + 8 B/frame per entry, plus D's 4 B/frame)
    detect = n * (8 * entries + 4)
    apply = n * (4 + 16 * entries)
    result["hbm_floor_ms"] = {"detect": round(detect / HBM_BYTES_PER_S * 1e3, 4),
                              "apply": round(apply / HBM_BYTES_PER_S * 1e3, 4)}
    gpu, power = gpu_info()
    torch.cuda.synchronize()
    print(json.dumps({"gpu": gpu, "power_limit": power, "seconds": SECONDS, "versions": VERSIONS, **result}))


if __name__ == "__main__":
    main()
