"""Cost of the float64 convolution (convolve_precise_kernel) against the float32 one, on one H100.

Two 3-minute tracks at 44.1 kHz with the default Config: the benchmark's kind of target (white noise under an
envelope, pink reference: float32 path) and the same target low-passed at 8 kHz against a bright reference
(tanh of white noise: float64 path).  Prints, per track, which path ran and the median over REPEATS of the
mgb_match_frequencies call (spectrum mean, design, convolution), timed with CUDA events.  Usage:
    python tools/precise_cost.py [repeats]"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]

import port  # noqa: E402
import matchering_b200 as mg  # noqa: E402
from matchering_b200.engine import TrackSession, get_plan, to_device_f32  # noqa: E402

SR, N = 44100, 180 * 44100


def tracks():
    t = port.synth_target(N, 0)
    X = np.fft.rfft(t.astype(np.float64), axis=0)
    X[np.fft.rfftfreq(N, 1.0 / SR) > 8000] = 0
    lp = np.fft.irfft(X, n=N, axis=0).astype(np.float32)
    w = np.random.default_rng(1).uniform(-1, 1, (N, 2))
    bright = np.tanh(2.0 * w / np.abs(w).max()).astype(np.float32)
    return {"broadband/pink": (t, port.synth_reference(N, 1000)), "lp8k/bright": (lp, bright)}


def main(repeats=20):
    plan = get_plan(mg.Config())
    for name, (t, r) in tracks().items():
        s = TrackSession(plan, len(t), len(r))
        td, rd = to_device_f32(t, plan.device), to_device_f32(r, plan.device)
        times = []
        for i in range(repeats + 3):
            s.match_levels(td, rd)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            s.match_frequencies(td)
            b.record()
            torch.cuda.synchronize()
            if i >= 3:
                times.append(a.elapsed_time(b) * 1e3)
        st = s.read_state()
        print(f"{name:16s} conv_precise={st.conv_precise} match_frequencies median {np.median(times):8.1f} us "
              f"(min {min(times):.1f}, max {max(times):.1f}) on {torch.cuda.get_device_name()}")


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 20)
