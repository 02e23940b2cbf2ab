"""What album loudness costs on the device.  Prints one JSON line: the GPU and its power limit, then
  - for an album of 12 3-minute tracks of the C2 recipe against a 3-minute reference profile, the device time of
    mgb_album_match + mgb_album_finalize_to_loudness at -14 and at -30 LUFS, and of mgb_album_match + 12 plain
    finalizes (the limited output), with the passes each search took;
  - mg.album_loudness of the 12 tracks against 12 mg.loudness calls (the samples already on the device).
Each group's variants alternate, median and p10-p90 spread of repeats after a warm-up; CUDA events around each run.
Read-only: writes nothing but stdout."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from reference_profile_bench import gpu_info  # noqa: E402

TRACKS = 12
REPEATS = 9
SECONDS = 180


def timed(jobs):
    import torch
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
    out = {f"{k}_ms": round(float(np.median(v)), 3) for k, v in times.items()}
    out.update({f"{k}_spread_p10_p90_ms": round(float(np.percentile(v, 90) - np.percentile(v, 10)), 3)
                for k, v in times.items()})
    return out


def main():
    import torch

    import matchering_b200 as mg
    import port
    from matchering_b200 import _native, analyze_reference
    from matchering_b200.engine import TrackSession, album_finalize_to_loudness, album_match, get_plan, to_device_f32
    from matchering_b200.loudness import device_meter
    cfg = mg.Config()
    plan = get_plan(cfg)
    dev = plan.device
    prof = analyze_reference(port.synth_reference(44100 * SECONDS, 1000), cfg)
    d_profile = prof.checked_blob(plan)
    xs = [to_device_f32(port.synth_target(44100 * SECONDS - 977 * k, k), dev) for k in range(TRACKS)]
    album = [TrackSession(plan, x.shape[0], None) for x in xs]
    passes = {}

    def plain():
        album_match(album, xs, d_profile)
        return [s.finalize(True, False, False) for s in album]

    def targeted(t):
        def job():
            album_match(album, xs, d_profile)
            passes[t] = album_finalize_to_loudness(album, t)[1]
        return job

    result = {"album": timed({"plain": plain, "target_m14": targeted(-14.0), "target_m30": targeted(-30.0)})}
    for t, rep in passes.items():
        r = _native.LoudnessTargetReport.from_buffer_copy(rep.cpu().numpy().tobytes())
        result["album"][f"passes_{int(-t)}"] = int(r.passes)
        result["album"][f"status_{int(-t)}"] = int(r.status)

    meter = device_meter(44100, dev)
    result["meter"] = timed({"album_loudness": lambda: meter.measure_album(xs),
                             "track_loudness_x12": lambda: [meter.measure(x) for x in xs]})
    gpu, power = gpu_info()
    print(json.dumps({"gpu": gpu, "power_limit": power, "tracks": TRACKS, "seconds": SECONDS, **result}))


if __name__ == "__main__":
    main()
