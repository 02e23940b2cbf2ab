"""Album workflow: 16 C2-recipe targets (3 minutes, 44.1 kHz) against one 3-minute reference, mastered with the
reference as samples in every job (pairs) and with one ReferenceProfile.  Prints one JSON line: the GPU and its
power limit, wall and device time per track for master_many and for stages.main on float64 numpy, whether every
profiled output is bit-identical to its paired one, and the largest difference between them next to the largest
difference between two runs of the same paired job (stage 3 sums per piece with float64 atomics, so the device does
not repeat a job bit for bit).  Read-only: writes nothing but stdout."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

TRACKS, FRAMES, ROUNDS = 16, 44100 * 180, 3


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:  # no nvidia-smi: the numbers still stand, without their card
        return f"unknown ({e})", "unknown"


def device_ms(lib):
    """Total device time (ms) of the launches recorded since profiling was switched on."""
    cap = 1 << 16
    ms = (C.c_float * cap)()
    n = lib.mgb_profile_collect(None, 0, ms, cap)
    return float(sum(ms[:n]))


def timed(lib, fn):
    import torch
    torch.cuda.synchronize()
    lib.mgb_profile_enable(1)
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    lib.mgb_profile_enable(0)
    return out, wall * 1e3 / TRACKS, device_ms(lib) / TRACKS


def main():
    import torch

    import matchering_b200 as mg
    import port
    from matchering_b200 import _native, stages
    from matchering_b200.batch import master_many
    lib = _native.load()
    cfg = mg.Config()
    reference = port.synth_reference(FRAMES, 1000)
    targets = [port.synth_target(FRAMES, k) for k in range(TRACKS)]
    ref64, targets64 = reference.astype(np.float64), [t.astype(np.float64) for t in targets]

    identical = True
    diff = {"profiled_vs_paired": 0.0, "paired_vs_paired": 0.0}
    last_paired = {}

    def maxdiff(xs, ys):
        return max(float(np.abs(np.asarray(x, np.float64) - y).max()) for x, y in zip(xs, ys))
    legs = {"master_many": {"paired": [], "profiled": []}, "stages_main_f64": {"paired": [], "profiled": []}}

    def run_master_many(kind):
        if kind == "paired":
            return master_many([(t, reference) for t in targets], cfg)
        prof = mg.analyze_reference(reference, cfg)  # once per album: part of the profiled leg's time
        return master_many([(t, prof) for t in targets], cfg)

    def run_stages(kind):
        if kind == "paired":
            return [stages.main(t, ref64, cfg)[0] for t in targets64]
        prof = mg.analyze_reference(ref64, cfg)
        return [stages.main(t, prof, cfg)[0] for t in targets64]

    runners = {"master_many": run_master_many, "stages_main_f64": run_stages}
    for name, fn in runners.items():  # warm-up: plans, pinned pools, sessions
        for kind in ("paired", "profiled"):
            fn(kind)
    for _ in range(ROUNDS):
        for name, fn in runners.items():
            outs = {}
            for kind in ("paired", "profiled"):
                outs[kind], wall, dev = timed(lib, lambda: fn(kind))
                legs[name][kind].append((wall, dev))
            identical &= all(np.array_equal(a, b) for a, b in zip(outs["paired"], outs["profiled"]))
            diff["profiled_vs_paired"] = max(diff["profiled_vs_paired"], maxdiff(outs["profiled"], outs["paired"]))
            if name in last_paired:
                diff["paired_vs_paired"] = max(diff["paired_vs_paired"], maxdiff(outs["paired"], last_paired[name]))
            last_paired[name] = outs["paired"]
            del outs
        torch.cuda.empty_cache()

    gpu, power = gpu_info()
    result = {"gpu": gpu, "power_limit": power, "tracks": TRACKS, "track_seconds": FRAMES / 44100, "rounds": ROUNDS,
              "bit_identical": bool(identical), "max_abs_diff_profiled_vs_paired": diff["profiled_vs_paired"],
              "max_abs_diff_paired_vs_paired": diff["paired_vs_paired"]}
    for name, kinds in legs.items():
        for kind, samples in kinds.items():
            walls, devs = zip(*samples)
            result[f"{name}_{kind}_wall_ms_per_track"] = round(float(np.median(walls)), 3)
            result[f"{name}_{kind}_device_ms_per_track"] = round(float(np.median(devs)), 4)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
