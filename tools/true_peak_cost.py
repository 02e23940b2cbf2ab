"""What the limiter's true-peak mode costs on the device.  Prints one JSON line: the GPU and its power limit, then for
3 minutes at 44.1 kHz and 10 minutes at 96 kHz (C5 material) the device time of mgb_limit with the default Config and
with Config(true_peak=True) (CUDA events around the call, median of repeats, the two alternating), and the detector
pass's HBM floor (12 B/frame: 8 read, 4 written, at 3.35 TB/s).  In true-peak mode the detector replaces the sample-peak
pass (8 B/frame read) and the limiter's first phase reads d (4 B/frame) instead of the samples (8 B/frame).
Read-only: writes nothing but stdout."""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from reference_profile_bench import gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
REPEATS = 20


def limiter_call(cfg, x):
    """A closure running mgb_limit of `cfg` on the CUDA (N, 2) float32 tensor x."""
    import torch

    from matchering_b200 import _native, plan
    from matchering_b200.engine import _stream_ptr
    lib = _native.load()
    params = _native.LimiterParams.from_constants(plan.limiter_constants(cfg))
    n = len(x)
    nbytes = int(lib.mgb_limiter_workspace_bytes(C.byref(params), n))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    out = torch.empty_like(x)
    engaged = torch.zeros(1, dtype=torch.int32, device=x.device)
    return lambda: _native.check(lib, lib.mgb_limit(C.byref(params), x.data_ptr(), out.data_ptr(), n, ws.data_ptr(), nbytes,
                                                    engaged.data_ptr(), _stream_ptr(x.device)))


def main():
    import torch

    import matchering_b200 as mg
    import port
    result = {}
    for name, fs, seconds in (("44k1_3min", 44100, 180), ("96k_10min", 96000, 600)):
        x = torch.from_numpy(port.synth_limiter_input(fs * seconds, 0)).cuda()
        calls = {"default": limiter_call(mg.Config(internal_sample_rate=fs), x),
                 "true_peak": limiter_call(mg.Config(internal_sample_rate=fs, true_peak=True), x)}
        for call in calls.values():
            for _ in range(3):
                call()
        times = {k: [] for k in calls}
        for _ in range(REPEATS):
            for k, call in calls.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                call()
                b.record()
                b.synchronize()
                times[k].append(a.elapsed_time(b))
        ms = {k: float(np.median(v)) for k, v in times.items()}
        result[f"{name}_frames"] = int(len(x))
        result[f"{name}_default_ms"] = round(ms["default"], 4)
        result[f"{name}_true_peak_ms"] = round(ms["true_peak"], 4)
        result[f"{name}_added_ms"] = round(ms["true_peak"] - ms["default"], 4)
        result[f"{name}_detector_hbm_floor_ms"] = round(len(x) * 12 / HBM_BYTES_PER_S * 1e3, 4)
        del x, calls
        torch.cuda.empty_cache()
    gpu, power = gpu_info()
    print(json.dumps({"gpu": gpu, "power_limit": power, **result}))


if __name__ == "__main__":
    main()
