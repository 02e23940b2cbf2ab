"""What a native-rate master costs on the device.  Prints one JSON line: the GPU and its power limit, then for a 3-minute
target at 48 kHz and at 96 kHz against a 3-minute 44.1 kHz reference, the device time of the native job (stage 1 and
the FIR design on the analysis copy at 44.1 kHz, then mgb_match_frequencies_native, the RMS correction and the limited
output at the target's rate) and of the ordinary job on the same analysis copy (stages 1-4 at 44.1 kHz, the limited
output), and which convolution each ran (`mgb_track_state::conv_precise`).  The resampling that makes the analysis
copy is common to both and not timed.  CUDA events around each job, the two jobs alternating, median of repeats after
a warm-up.  Read-only: writes nothing but stdout."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from reference_profile_bench import gpu_info  # noqa: E402

REPEATS = 15
SECONDS = 180


def main():
    import torch

    import matchering_b200 as mg
    import port
    from matchering_b200.engine import TrackSession, get_native_plan, get_plan, to_device_f32
    from matchering_b200.resample import resample_on_device
    cfg = mg.Config()
    plan = get_plan(cfg)
    dev = plan.device
    r = to_device_f32(port.synth_reference(44100 * SECONDS, 1), dev)
    result = {}
    for rate in (48000, 96000):
        nplan = get_native_plan(cfg, rate, dev)
        xn = to_device_f32(port.synth_target(rate * SECONDS, 0), dev)
        xa = resample_on_device(xn, rate, 44100)
        analysis = TrackSession(plan, xa.shape[0], r.shape[0])
        native = TrackSession(nplan, xn.shape[0], None)
        ordinary = TrackSession(plan, xa.shape[0], r.shape[0])

        def native_job():
            analysis.match_levels(xa, r)
            analysis.design_frequencies()
            native.match_frequencies_native(analysis, xn)
            native.correct_levels()
            return native.finalize(True, False, False)

        def ordinary_job():
            ordinary.match_levels(xa, r)
            ordinary.match_frequencies(xa)
            ordinary.correct_levels()
            return ordinary.finalize(True, False, False)

        jobs = {"native": native_job, "ordinary": ordinary_job}
        for job in jobs.values():
            for _ in range(2):
                job()
        torch.cuda.synchronize()
        times = {k: [] for k in jobs}
        for _ in range(REPEATS):
            for k, job in jobs.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                job()
                b.record()
                b.synchronize()
                times[k].append(a.elapsed_time(b))
        ms = {k: float(np.median(v)) for k, v in times.items()}
        spread = {k: round(float(np.percentile(v, 90) - np.percentile(v, 10)), 4) for k, v in times.items()}
        result[f"native_{rate}_ms"] = round(ms["native"], 4)
        result[f"ordinary_on_44k1_copy_{rate}_ms"] = round(ms["ordinary"], 4)
        result[f"spread_p10_p90_{rate}_ms"] = spread
        result[f"native_fft_size_{rate}"] = nplan.tables.fft_size
        # which convolution ran (1: float64 transforms, chosen from the FIR's peak gain and the target's peak)
        result[f"conv_precise_{rate}"] = {"native": int(native.read_state().conv_precise),
                                          "ordinary": int(ordinary.read_state().conv_precise)}
        del xn, xa, analysis, native, ordinary, jobs
        torch.cuda.empty_cache()
    gpu, power = gpu_info()
    print(json.dumps({"gpu": gpu, "power_limit": power, "seconds": SECONDS, **result}))


if __name__ == "__main__":
    main()
