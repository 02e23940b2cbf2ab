"""What a loudness target costs on the device.  Prints one JSON line: the GPU and its power limit, then for the C2 job
(3 minutes at 44.1 kHz) and the C3 job (10 minutes at 96 kHz), after stages 1-3 ran once, the device time of stage 4's
limited output with mgb_finalize and with mgb_finalize_to_loudness at a quieter target (-30 LUFS: one pass) and a
louder one (-9 LUFS: several passes) -- each call captured once in a CUDA graph, so that the figure is device time and
not the host's ~100 launches; CUDA events around the graph's replay, median of repeats, the three alternating -- the
pass counts, and the kernel time of one fully skipped pass (the kernels launched after the first search step of the
one-pass run, from mgb_profile_collect, divided by the passes they cover; the pass's two memsets are not in it).
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

REPEATS = 15
QUIET, LOUD = -30.0, -9.0


def main():
    import torch

    import matchering_b200 as mg
    import port
    from matchering_b200 import _native
    from matchering_b200.engine import TrackSession, _stream_ptr, get_plan, to_device_f32
    from matchering_b200.loudness import device_meter, target_params
    lib = _native.load()
    result = {}
    for name, fs, seconds in (("c2_44k1_3min", 44100, 180), ("c3_96k_10min", 96000, 600)):
        cfg = mg.Config(internal_sample_rate=fs)
        plan = get_plan(cfg)
        dev = plan.device
        n = fs * seconds
        t = to_device_f32(port.synth_target(n, 0), dev)
        r = to_device_f32(port.synth_reference(n - 7 * fs, 1), dev)
        s = TrackSession(plan, n, r.shape[0])
        s.match_levels(t, r)
        s.match_frequencies(t)
        s.correct_levels()
        meter = device_meter(fs, dev)
        sb = int(lib.mgb_loudness_target_workspace_bytes(C.byref(meter.params), n))
        search = torch.empty(sb, dtype=torch.uint8, device=dev)
        out = torch.empty((n, 2), dtype=torch.float32, device=dev)
        rep = torch.empty(C.sizeof(_native.LoudnessTargetReport), dtype=torch.uint8, device=dev)
        P, L = C.byref(plan.struct), C.byref(s.layout)

        def finalize():
            _native.check(lib, lib.mgb_finalize(P, L, s.result.data_ptr(), out.data_ptr(), None, None, s.workspace.data_ptr(),
                                                s.state.data_ptr(), _stream_ptr(dev)))

        def to_loudness(target):
            tp = target_params(target)
            return lambda: _native.check(lib, lib.mgb_finalize_to_loudness(
                P, L, C.byref(meter.params), C.byref(tp), s.result.data_ptr(), out.data_ptr(), s.workspace.data_ptr(),
                search.data_ptr(), sb, s.state.data_ptr(), rep.data_ptr(), _stream_ptr(dev)))

        def report():
            return _native.LoudnessTargetReport.from_buffer_copy(rep.cpu().numpy().tobytes())

        calls = {"finalize": finalize, "quiet": to_loudness(QUIET), "loud": to_loudness(LOUD)}
        passes = {}
        for k, call in calls.items():
            for _ in range(2):
                call()
            if k != "finalize":
                rr = report()
                passes[k] = (int(rr.passes), int(rr.status), round(float(rr.integrated), 4))
        graphs = {}
        for k, call in calls.items():
            graphs[k] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graphs[k]):
                call()
        times = {k: [] for k in calls}
        for _ in range(REPEATS):
            for k, g in graphs.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                g.replay()
                b.record()
                b.synchronize()
                times[k].append(a.elapsed_time(b))
        ms = {k: float(np.median(v)) for k, v in times.items()}
        # one fully skipped pass: the kernels launched after the quiet run's first search step, per pass they cover
        torch.cuda.synchronize()
        lib.mgb_profile_enable(1)
        calls["quiet"]()
        lib.mgb_profile_enable(0)
        names = C.create_string_buffer(1 << 16)
        durations = (C.c_float * 4096)()
        count = lib.mgb_profile_collect(names, len(names), durations, 4096)
        kernel_names = names.value.decode().split("\n")[:count]
        first_step = kernel_names.index("loudness_target_step_kernel")
        skipped = sum(durations[first_step + 1:count])
        skipped_passes = _native.MGB_LOUDNESS_TARGET_MAX_PASSES - passes["quiet"][0]
        result[f"{name}_frames"] = n
        result[f"{name}_finalize_ms"] = round(ms["finalize"], 4)
        result[f"{name}_target_quiet_ms"] = round(ms["quiet"], 4)
        result[f"{name}_target_loud_ms"] = round(ms["loud"], 4)
        result[f"{name}_passes_quiet"] = passes["quiet"]
        result[f"{name}_passes_loud"] = passes["loud"]
        result[f"{name}_skipped_pass_kernel_ms"] = round(skipped / max(skipped_passes, 1), 4)
        del t, r, s, search, out, calls, graphs
        torch.cuda.empty_cache()
    gpu, power = gpu_info()
    result["passes_format"] = "(passes, status, measured LUFS)"
    result["targets_lufs"] = {"quiet": QUIET, "loud": LOUD}
    print(json.dumps({"gpu": gpu, "power_limit": power, **result}))


if __name__ == "__main__":
    main()
