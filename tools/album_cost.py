"""What album mastering costs on the device.  Prints one JSON line: the GPU and its power limit, then for an album of 12
3-minute tracks of the C2 recipe against a 3-minute reference profile, the device time of the album (mgb_album_match,
then mgb_finalize per track, the limited output) and of 12 profiled single jobs on the same data (stages 1-4 each, the
limited output), the two alternating, median and p10-p90 spread of repeats after a warm-up; and the album's peak device
memory with every track resident.  CUDA events around each run.  Read-only: writes nothing but stdout."""
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


def main():
    import torch

    import matchering_b200 as mg
    import port
    from matchering_b200 import analyze_reference
    from matchering_b200.engine import TrackSession, album_match, get_plan, to_device_f32
    cfg = mg.Config()
    plan = get_plan(cfg)
    dev = plan.device
    prof = analyze_reference(port.synth_reference(44100 * SECONDS, 1000), cfg)
    d_profile = prof.checked_blob(plan)
    xs = [to_device_f32(port.synth_target(44100 * SECONDS - 977 * k, k), dev) for k in range(TRACKS)]
    album = [TrackSession(plan, x.shape[0], None) for x in xs]
    singles = [TrackSession(plan, x.shape[0], None) for x in xs]

    def album_job():
        album_match(album, xs, d_profile)
        return [s.finalize(True, False, False) for s in album]

    def single_jobs():
        outs = []
        for s, x in zip(singles, xs):
            s.match_levels_profiled(x, d_profile)
            s.match_frequencies(x)
            s.correct_levels()
            outs.append(s.finalize(True, False, False))
        return outs

    jobs = {"album": album_job, "singles": single_jobs}
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
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    album_job()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev)
    result = {f"{k}_ms": round(float(np.median(v)), 3) for k, v in times.items()}
    result.update({f"{k}_spread_p10_p90_ms": round(float(np.percentile(v, 90) - np.percentile(v, 10)), 3)
                   for k, v in times.items()})
    # the album's own memory: targets, sessions (workspace, state, stage-2 result) and the profile, resident for the whole
    # album, plus what one album run allocates on top (its workspace and the limited outputs)
    resident = sum(x.numel() * 4 for x in xs) + d_profile.numel()
    resident += sum(s.workspace.numel() + s.state.numel() + s.result.numel() * 4 for s in album)
    result["album_resident_mb"] = round(resident / 2 ** 20, 1)
    result["album_run_extra_mb"] = round((peak - base) / 2 ** 20, 1)
    result["album_peak_device_mb"] = round((resident + peak - base) / 2 ** 20, 1)
    result["conv_precise"] = [int(s.read_state().conv_precise) for s in album]
    gpu, power = gpu_info()
    print(json.dumps({"gpu": gpu, "power_limit": power, "tracks": TRACKS, "seconds": SECONDS, **result}))


if __name__ == "__main__":
    main()
