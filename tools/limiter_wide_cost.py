"""Device time of the limiter's wide-window path (limiter_wide.cuh) against the halo kernel, on one GPU.

Buffers: a 3-minute 44.1 kHz limiter input and the one-hour BASELINE config-5 buffer (158.76 M frames), both from
oracle/port.py's synth_limiter_input.  Configs: attack 10 ms with hold 200 ms (3 minutes) or attack 10 ms (one hour)
on the wide-window path, and the default Config on the halo kernel, on the same buffers.  mgb_limit on device
buffers, timed with CUDA events (median of REPEATS), plus the per-kernel split from mgb_profile_collect, and the
path's HBM bytes per frame from its planes.  Prints one JSON line per run.  Usage:
    python tools/limiter_wide_cost.py [repeats]"""
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]

import port  # noqa: E402
import matchering_b200 as mg  # noqa: E402
from matchering_b200 import _native, plan as plan_mod  # noqa: E402


def model_bytes_per_frame(levels):
    """HBM bytes per frame the wide-window path moves, from its planes (each plane read once per use):
    gain kernel: input 8 in, g / prefix / suffix 12 out, block maxima 1/8 out; each sparse-table level 3 x 4/32;
    forward attack: suffix + prefix maxima of A's window 8 in, forward plane 8 out; backward: 8 in, g_att 4 out;
    apply: H's window 8, g 4, g_att 4, input 8 in, output 8 out.  Window reads of whole blocks hit L2."""
    return 8 + 12 + 0.125 + levels * 0.375 + 8 + 8 + 8 + 4 + 8 + 4 + 4 + 8 + 8


def run(lib, x_dev, n, cfg, repeats):
    lc = plan_mod.limiter_constants(cfg)
    params = _native.LimiterParams.from_constants(lc)
    ws_bytes = int(lib.mgb_limiter_workspace_bytes(C.byref(params), n))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    out = torch.empty_like(x_dev)
    engaged = torch.zeros(4, dtype=torch.int32, device="cuda")

    def call():
        _native.check(lib, lib.mgb_limit(C.byref(params), x_dev.data_ptr(), out.data_ptr(), n, ws.data_ptr(), ws_bytes,
                                         engaged.data_ptr(), None))
    call()
    times = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    lib.mgb_profile_enable(1)
    call()
    names = C.create_string_buffer(1 << 16)
    ms = (C.c_float * 256)()
    got = lib.mgb_profile_collect(names, len(names), ms, 256)
    lib.mgb_profile_enable(0)
    split = {}
    for k, t in zip(names.value.decode().split("\n"), list(ms)[:got]):
        split[k] = split.get(k, 0.0) + float(t)
    wide = "limiter_wide_apply_kernel" in split
    res = dict(frames=n, reach=lc.reach, hold=lc.hold, path="wide" if wide else "halo", median_ms=float(np.median(times)),
               min_ms=float(np.min(times)), workspace_bytes=ws_bytes, kernels_ms={k: round(v, 4) for k, v in split.items()})
    if wide:
        levels = names.value.decode().split("\n")[:got].count("limiter_wide_sparse_kernel")
        bpf = model_bytes_per_frame(levels)
        res.update(levels=levels, model_bytes_per_frame=bpf, model_GBps=bpf * n / (res["median_ms"] * 1e-3) / 1e9)
    return res


def main(repeats=10):
    torch.cuda.set_device(0)
    lib = _native.load()
    for label, n, wide_cfg in (("3min", 180 * 44100, mg.Config(limiter=mg.LimiterConfig(attack=10.0, hold=200.0))),
                               ("1hour", 3600 * 44100, mg.Config(limiter=mg.LimiterConfig(attack=10.0)))):
        x = port.synth_limiter_input(n, seed=0)
        x_dev = torch.from_numpy(x).cuda()
        del x
        for cname, cfg in (("wide", wide_cfg), ("default", mg.Config())):
            r = run(lib, x_dev, n, cfg, repeats if n < 1e8 else max(3, repeats // 3))
            print(json.dumps(dict(buffer=label, config=cname, **r)), flush=True)
        del x_dev
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 10)
