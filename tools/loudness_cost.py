"""What the loudness meter costs on the device.  Prints one JSON line: the GPU and its power limit; the device time
of mgb_loudness (CUDA events around the call, median of repeats) on the 3-minute C2 master and on the one-hour C5
buffer, each next to its HBM floor (8 B/frame at 3.35 TB/s); and the device time per track of master_many over 8
three-minute tracks with and without loudness=True (the library's per-launch events, summed).  Read-only: writes
nothing but stdout."""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from reference_profile_bench import device_ms, gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
REPEATS, TRACKS = 20, 8


def meter_ms(x, fs):
    """Median device time (ms) of mgb_loudness on a CUDA (N, 2) float32 tensor."""
    import torch

    from matchering_b200 import _native
    from matchering_b200.engine import _stream_ptr
    from matchering_b200.loudness import device_meter
    m = device_meter(fs, x.device)
    n = int(m.lib.mgb_loudness_workspace_bytes(C.byref(m.params), len(x)))
    ws = torch.empty(n, dtype=torch.uint8, device=x.device)
    out = torch.empty(C.sizeof(_native.LoudnessResult), dtype=torch.uint8, device=x.device)
    call = lambda: _native.check(m.lib, m.lib.mgb_loudness(C.byref(m.params), x.data_ptr(), len(x), ws.data_ptr(), n,
                                                           out.data_ptr(), _stream_ptr(x.device)))
    for _ in range(3):
        call()
    times = []
    for _ in range(REPEATS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def main():
    import torch

    import matchering_b200 as mg
    import port
    from matchering_b200 import _native, stages
    from matchering_b200.batch import master_many
    lib = _native.load()
    result = {}
    n2 = 44100 * 180
    t, r = port.synth_target(n2, 0), port.synth_reference(n2, 1)
    master = stages.main(torch.from_numpy(t).cuda(), torch.from_numpy(r).cuda(), mg.Config(), True, False, False)[0]
    for name, x in (("c2_master_3min", master), ("c5_hour", None)):
        if x is None:
            x = torch.from_numpy(port.synth_limiter_input(44100 * 3600, seed=0)).cuda()
        ms = meter_ms(x, 44100)
        floor = len(x) * 8 / HBM_BYTES_PER_S * 1e3
        result[f"{name}_frames"] = int(len(x))
        result[f"{name}_meter_ms"] = round(ms, 4)
        result[f"{name}_hbm_floor_ms"] = round(floor, 4)
        result[f"{name}_meter_over_floor"] = round(ms / floor, 2)
        del x
    torch.cuda.empty_cache()

    cfg = mg.Config()
    pairs = [(port.synth_target(n2, 10 + k), r) for k in range(TRACKS)]
    legs = {False: [], True: []}
    for flag in (False, True):  # warm-up
        master_many(pairs, cfg, loudness=flag)
    for _ in range(3):
        for flag in (False, True):
            torch.cuda.synchronize()
            lib.mgb_profile_enable(1)
            master_many(pairs, cfg, loudness=flag)
            torch.cuda.synchronize()
            lib.mgb_profile_enable(0)
            legs[flag].append(device_ms(lib) / TRACKS)
    result["master_many_device_ms_per_track"] = round(float(np.median(legs[False])), 4)
    result["master_many_loudness_device_ms_per_track"] = round(float(np.median(legs[True])), 4)
    gpu, power = gpu_info()
    print(json.dumps({"gpu": gpu, "power_limit": power, **result}))


if __name__ == "__main__":
    main()
