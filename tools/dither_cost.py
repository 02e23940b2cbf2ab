"""What dither costs on the device.  Prints one JSON line: the GPU and its power limit, then for C2-sized (3 minutes at
44.1 kHz) and C3-sized (10 minutes at 96 kHz) stereo buffers, the device time of mgb_pcm_encode against
mgb_pcm_encode_dithered with flat TPDF (0 taps) and with the shaped filter (12 taps), at 16 and 24 bits: CUDA events
around each call, median of repeats, the three encoders alternating.  The HBM floor is the bytes each call moves (8 B
read plus 4 or 6 B written per frame) at 3.35 TB/s.  Read-only: writes nothing but stdout."""
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

REPEATS = 21
HBM_BYTES_PER_S = 3.35e12


def main():
    import torch

    import port
    from matchering_b200 import _native, dither
    from matchering_b200.engine import _stream_ptr
    lib = _native.load()
    result = {}
    for name, fs, seconds in (("c2_44k1_3min", 44100, 180), ("c3_96k_10min", 96000, 600)):
        n = fs * seconds
        x = torch.from_numpy(port.synth_target(n, 0)).cuda()
        st = _stream_ptr(x.device)
        for bits in (16, 24):
            out = torch.empty(n * 2 * bits // 8, dtype=torch.uint8, device=x.device)
            flat, shaped = dither.params("tpdf", fs, 1), dither.params("shaped", fs, 1)
            calls = {
                "plain": lambda: lib.mgb_pcm_encode(x.data_ptr(), bits, out.data_ptr(), 2 * n, st),
                "tpdf": lambda: lib.mgb_pcm_encode_dithered(C.byref(flat), x.data_ptr(), n, bits, out.data_ptr(), st),
                "shaped": lambda: lib.mgb_pcm_encode_dithered(C.byref(shaped), x.data_ptr(), n, bits, out.data_ptr(), st),
            }
            for call in calls.values():
                for _ in range(3):
                    _native.check(lib, call())
            times = {k: [] for k in calls}
            for _ in range(REPEATS):
                for k, call in calls.items():
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    _native.check(lib, call())
                    b.record()
                    b.synchronize()
                    times[k].append(a.elapsed_time(b))
            for k, v in times.items():
                result[f"{name}_pcm{bits}_{k}_us"] = round(1000 * float(np.median(v)), 1)
            result[f"{name}_pcm{bits}_hbm_floor_us"] = round(1e6 * n * (8 + 2 * bits // 8) / HBM_BYTES_PER_S, 1)
        result[f"{name}_frames"] = n
        del x, out
        torch.cuda.empty_cache()
    gpu, power = gpu_info()
    print(json.dumps({"gpu": gpu, "power_limit": power, **result}))


if __name__ == "__main__":
    main()
