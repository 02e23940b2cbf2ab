"""Synchronisation of the kernels, checked on the CPU without a GPU.

The emulator (tests/emul) runs a block's threads as fibers in a fixed order, so a missing barrier whose
reader runs after its writer still gives the right answer there.  Two checks close that gap:

- A ThreadSanitizer build of the emulator (build_emul.build(racecheck=True)): every emulated thread is a
  fiber, and happens-before edges exist only where CUDA gives them (cuda_emul.h lists them).  The
  controls prove that model on tiny kernels, at block sizes from 64 to 1024 threads (above 224, lanes of a
  warp share fibers in two alternating groupings; cuda_emul.h); the matrix then runs the emulator tests that
  reach every kernel and template instantiation at small shapes, and any report fails.
- The same matrix on the normal build with the threads of each round resumed in reverse and in a seeded
  random order (MGB_EMUL_ORDER).  The emulator tests hold every result to its oracle bound, and the
  limiter's output to bit-identity with a forward run.

Each matrix group runs in its own subprocess (libtsan has to be preloaded into the Python that loads the
instrumented library), and the groups run in parallel on up to 8 CPU cores.
"""
import ctypes as C
import glob
import os
import re
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import build_emul

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = "tests/test_emul_kernels.py::"

# Each group: emulator tests that together reach the kernels named in its comment, at the smallest shapes
# the suite has for them.  Shapes the matrix needs: three limiter chunks plus a partial one (9217 frames,
# 4608 * 5 + 77), a piece boundary inside a convolution frame (the stage-parity tracks), a silent channel
# (mono targets, one-sided digital silence), an overflowing loud list (the loud-list cases).
MATRIX = {
    # mgb_test_fft, float32 and float64, every size it accepts
    "fft": [K + "test_fft_matches_numpy"],
    # design_kernel on the direct and the operator path (operator_columns, transpose, smooth_operator),
    # with lowess_it 0 and > 0
    "design": [K + "test_fir_design_matches_oracle", K + "test_smoothing_operator_matches_direct_path_and_oracle",
               K + "test_fir_design_with_lowess_robustness_iterations"],
    # analyze_kernel, spectrum_mean, design_kernel and the convolution for every fft_size
    "fft_sizes": [K + "test_pipeline_other_configs", K + "test_pipeline_fft_size_16384"],
    # every convolution kernel launch_convolve_t can pick, with the twiddle_chain / tma / conv_persistent /
    # conv_fused switches, against float64 intermediates
    "convolution": ["tests/test_stage_parity.py::test_stage_parity_emulated",
                    K + "test_generic_convolution_kernel_matches_golden",
                    K + "test_persistent_convolution_and_chained_analysis_twiddles"],
    # convolve_precise_kernel on coloured material; the gain-crossing material through the float64 path
    "precise": ["tests/test_coloured_material.py::test_coloured_material_emulated",
                "tests/test_stage_parity.py::test_gain_crossing_stage_parity_emulated"],
    # loud_sumsq on its list path and its fallback with overflowing lists, correction_final and scale
    "correction": ["tests/test_correction_loud_list.py::test_loud_list_and_fallback_emulated",
                   K + "test_rms_correction_step_counts", K + "test_mono_and_near_mono_targets",
                   K + "test_tonal_material_with_digital_silence"],
    # the halo limiter with order capacity 1 and 2, by ticket and with lookback_inclusive=0, mgb_limit and
    # mgb_test_limiter_gains
    "limiter": [K + "test_limiter_matches_golden_several_chunks", K + "test_limiter_edge_lengths",
                K + "test_limiter_higher_filter_orders", K + "test_limiter_lookback_through_aggregates_only",
                K + "test_second_order_release_filter_over_many_chunks", K + "test_limiter_gain_envelopes_match_golden",
                K + "test_limiter_not_engaged_copies_input"],
    # every limiter_wide_* kernel
    "limiter_wide": ["tests/test_limiter_wide_windows.py::test_emulator_path_boundary",
                     "tests/test_limiter_wide_windows.py::test_emulator_poisoned_workspace_is_bit_identical",
                     "tests/test_limiter_wide_windows.py::test_emulator_early_out_copies_input"],
    # resample up and down, PCM encode / decode at 16 and 24 bit, window_energy and preview_piece,
    # check_peaks and check_equality
    "io_kernels": [K + "test_resampler_matches_oracle", K + "test_pcm_conversions_are_bit_exact",
                   K + "test_preview_kernels_match_golden", K + "test_checker_reductions"],
    # mgb_pipeline_* at depth 2, also through the PCM entry; mgb_host_upload / mgb_host_download and their
    # worker threads
    "pipeline_host": [K + "test_pipeline_entry_points_match_single_track_path", K + "test_pipeline_pcm_entry",
                      "tests/test_emul_hostio.py::test_upload_and_download_round_trip",
                      "tests/test_emul_hostio.py::test_stages_main_host_matches_staged_calls",
                      "tests/test_emul_hostio.py::test_limit_host_and_its_early_out"],
}



def split(ids):
    """One ThreadSanitizer run per parameter set of the convolution tests: they are the longest, and this way they
    spread over the cores (test ids as pytest prints them)."""
    import test_coloured_material
    import test_stage_parity
    cases = {"tests/test_stage_parity.py::test_stage_parity_emulated":
             [v.name for v in test_stage_parity.VARIANTS if v.emulated],
             "tests/test_stage_parity.py::test_gain_crossing_stage_parity_emulated": ["f1024_generic", "f4096_default"],
             "tests/test_coloured_material.py::test_coloured_material_emulated":
             # one coloured track per kernel the float64 path serves next to
             [f"{c}-{k}" for c, k in test_coloured_material.EMULATED if c in
              ("lp2k_bright", "butter16k_bright", "bass_bright", "upsampled22k_bright") or k == "f16384_global"]}
    return [[f"{i}[{p}]"] for i in ids if i in cases for p in cases[i]] + [[i] for i in ids if i not in cases]


# the race-checked runs, longest first: (name, test ids)
RACECHECK_RUNS = ([(f"{g}:{run[0].split('::')[1]}", run) for g in ("convolution", "precise") for run in split(MATRIX[g])] +
                  [(g, ids) for g, ids in MATRIX.items() if g not in ("convolution", "precise")])

CONTROLS_REPORTED = ["race_reader_above_writer", "race_reader_below_writer", "race_write_after_read",
                     "race_two_lanes_one_word", "race_kth_reset_on_entry"]
CONTROLS_CLEAN = ["ok_reader_above_writer", "ok_reader_below_writer", "ok_write_after_read", "ok_two_lanes_one_word",
                  "ok_shuffles", "ok_atomics", "ok_publish_poll", "ok_kth_twice"]
ORDERS = ["reverse", "seeded"]


def libtsan():
    path = subprocess.run(["g++", "-print-file-name=libtsan.so"], capture_output=True, text=True, check=True).stdout.strip()
    if not os.path.isabs(path):
        pytest.fail("g++ has no libtsan.so")
    return path


def tsan_env(log_dir, preload=True):
    env = dict(os.environ)
    env["TSAN_OPTIONS"] = f"halt_on_error=0:exitcode=66:log_path={os.path.join(log_dir, 'tsan')}"
    if preload:
        env["LD_PRELOAD"] = libtsan()
    return env


def reports(log_dir):
    """(number of reports, the first one: its two accesses' stacks down to the summary line)."""
    text = "".join(open(p, errors="replace").read() for p in sorted(glob.glob(os.path.join(log_dir, "tsan*"))))
    found = re.findall(r"WARNING: ThreadSanitizer.*?SUMMARY: ThreadSanitizer[^\n]*", text, flags=re.S)
    return len(found), (found[0] if found else text[-4000:])


def pytest_cmd(ids):
    flags = ["-s"] if sys.flags.no_user_site else []
    return [sys.executable, *flags, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", *ids]


def run_group(ids, env, log_dir):
    os.makedirs(log_dir, exist_ok=True)
    t0 = time.time()
    r = subprocess.run(pytest_cmd(ids), cwd=ROOT, env=env, capture_output=True, text=True)
    return r.returncode, r.stdout[-3000:] + r.stderr[-3000:], time.time() - t0


@pytest.fixture(scope="session")
def racecheck_build():
    return build_emul.build(racecheck=True), build_emul.build_racecheck_controls()


@pytest.fixture(scope="session")
def matrix_runs(racecheck_build, tmp_path_factory):
    """Every group under ThreadSanitizer, and on the normal build in each other order, 8 at a time."""
    build_emul.build()
    base = tmp_path_factory.mktemp("racecheck")
    jobs = {}
    for name, ids in RACECHECK_RUNS:
        log_dir = str(base / f"tsan_{re.sub(r'[^A-Za-z0-9_.-]', '_', name)}")
        env = tsan_env(log_dir)
        env["MGB_EMUL_BUILD"] = "racecheck"
        jobs[("tsan", name)] = (ids, env, log_dir)
    for group, ids in MATRIX.items():
        for order in ORDERS:
            env = dict(os.environ, MGB_EMUL_ORDER=order, MGB_EMUL_SEED="12345")
            jobs[(order, group)] = (ids, env, str(base / f"{order}_{group}"))
    t0 = time.time()
    with ThreadPoolExecutor(max_workers=8) as ex:
        futures = {key: ex.submit(run_group, *job) for key, job in jobs.items()}
        done = {key: f.result() + (jobs[key][2],) for key, f in futures.items()}
    print(f"race-check matrix: {len(jobs)} groups in {time.time() - t0:.0f} s")
    return done


@pytest.mark.parametrize("threads", [64, 256, 512, 1024])
@pytest.mark.parametrize("name", CONTROLS_REPORTED + CONTROLS_CLEAN)
def test_race_checker_controls(racecheck_build, tmp_path, name, threads):
    """A missing barrier, a write-after-read, two lanes writing one word and a radix select whose second call
    resets state the first call's result is still read from are reported, whatever the order of the threads
    involved and at every block size up to 1024; the same kernels with their barriers, shuffles, atomics, a
    publish/poll hand-off and design.cu's block_kth_smallest called twice are not."""
    _, exe = racecheck_build
    r = subprocess.run([exe, name, str(threads)], env=tsan_env(str(tmp_path), preload=False), capture_output=True,
                       text=True)
    n, first = reports(str(tmp_path))
    if name in CONTROLS_REPORTED:
        assert r.returncode == 66 and n >= 1, (r.returncode, r.stdout, r.stderr)
    else:
        assert r.returncode == 0 and n == 0, first


@pytest.mark.parametrize("group", [name for name, _ in RACECHECK_RUNS])
def test_kernels_have_no_data_races(matrix_runs, group):
    rc, out, seconds, log_dir = matrix_runs[("tsan", group)]
    n, first = reports(log_dir)
    assert n == 0, f"{n} ThreadSanitizer report(s) in {group}; the first:\n{first}"
    assert rc == 0, out
    print(f"{group}: {seconds:.0f} s under ThreadSanitizer")


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("group", list(MATRIX))
def test_kernels_pass_in_other_thread_orders(matrix_runs, group, order):
    rc, out, seconds, _ = matrix_runs[(order, group)]
    assert rc == 0, out


LIMITER_SNIPPET = r"""
import sys
import numpy as np
sys.path[:0] = ["tests", "oracle", "tests/emul"]
import port
import test_emul_kernels as t
from emul_harness import emul_lib
lib = emul_lib()
lib.mgb_set_option(b"limiter_ticket", int(sys.argv[1]))
x = port.synth_limiter_input(4608 * 5 + 77, seed=5)
cfgs = [port.OracleConfig(),  # the halo kernel, order capacity 1
        port.OracleConfig(limiter=port.OracleLimiterConfig(hold_filter_order=2, release_filter_order=2)),
        port.OracleConfig(limiter=port.OracleLimiterConfig(attack=10.0))]  # the wide-window kernels
np.save(sys.argv[2], np.stack([t._limit(lib, x, cfg)[0] for cfg in cfgs]))
# mgb_test_fft, float32 and float64, forward and inverse, at a size per transform kernel
import ctypes as C
from emul_harness import aligned, aligned_copy, ptr
from matchering_b200 import _native
ffts = []
for n, f64 in [(512, 0), (4096, 0), (16384, 0), (2048, 1), (8192, 1)]:
    rng = np.random.default_rng(n + f64)
    dt = np.complex128 if f64 else np.complex64
    xin = aligned_copy((rng.standard_normal((2, n)) + 1j * rng.standard_normal((2, n))).astype(dt))
    p = _native.Plan()
    p.fft_size = min(n, 8192) if n <= 8192 else n // 2
    p.n_lin, p.n_log, p.lowess_k, p.lowess_nfit = p.fft_size // 2 + 1, 10, 2, 2
    bufs = [aligned((1 << 20,), np.uint8) for _ in range(4)]
    p.d_tw_f32_F, p.d_tw_f32_2F, p.d_tw_f64_F, p.d_tw_f64_2F = [b.ctypes.data for b in bufs]
    _native.check(lib, lib.mgb_plan_fill_twiddles(C.byref(p), None))
    tw = bufs[1] if n > 8192 else (bufs[2] if f64 else bufs[0])
    for direction in (1, -1):
        out = aligned((2, n), dt)
        _native.check(lib, lib.mgb_test_fft(n, f64, direction, ptr(xin), ptr(out), 2, ptr(tw), None))
        ffts.append(out.view(np.uint8).ravel().copy())
np.save(sys.argv[2] + ".fft.npy", np.concatenate(ffts))
"""


def test_limiter_output_is_bit_identical_in_every_order(tmp_path):
    """The limiter and the FFTs are deterministic: their output may not depend on the order of the threads inside
    a block (the limiter with its chunks by block index and by ticket)."""
    build_emul.build()
    for ticket in ("0", "1"):
        outs = {}
        for order in ["forward", *ORDERS]:
            path = str(tmp_path / f"{order}_{ticket}.npy")
            env = dict(os.environ, MGB_EMUL_ORDER=order, MGB_EMUL_SEED="777")
            r = subprocess.run([sys.executable, *(["-s"] if sys.flags.no_user_site else []), "-c", LIMITER_SNIPPET,
                                ticket, path], cwd=ROOT, env=env, capture_output=True, text=True)
            assert r.returncode == 0, r.stderr[-3000:]
            outs[order] = (np.load(path), np.load(path + ".fft.npy"))
        for order in ORDERS:
            assert outs[order][0].tobytes() == outs["forward"][0].tobytes(), (order, ticket)
            assert outs[order][1].tobytes() == outs["forward"][1].tobytes(), (order, "fft")
