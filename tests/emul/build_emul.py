"""TEST INFRASTRUCTURE ONLY: compile matchering_b200/csrc/*.cu for the HOST through the
CUDA-on-CPU emulator (tests/emul/cuda_emul.h) into tests/emul/_build/libmatchering_b200_emul.so.
Same sources, same C ABI; device pointers are host pointers.

build(racecheck=True) makes the race-checking variant in tests/emul/_build_racecheck/: the kernel
sources built with ThreadSanitizer (-fsanitize=thread -O1 -g -DMGB_EMUL_RACECHECK), the scheduler
(cuda_emul.cpp) uninstrumented but telling ThreadSanitizer about its fibers and barriers.  The
process that loads it needs libtsan preloaded (LD_PRELOAD=$(g++ -print-file-name=libtsan.so))."""
from __future__ import annotations

import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SRC_DIR = os.path.join(ROOT, "matchering_b200", "csrc")
OUT_DIR = os.path.join(HERE, "_build")
LIB_PATH = os.path.join(OUT_DIR, "libmatchering_b200_emul.so")
RACECHECK_DIR = os.path.join(HERE, "_build_racecheck")
SOURCES = ["api.cu", "analyze.cu", "design.cu", "convolve.cu", "correct.cu", "limiter.cu", "pipeline.cu", "hostio.cu", "resample.cu"]
COMMON = ["-std=c++17", "-fPIC", "-DMGB_EMULATE", "-include", os.path.join(HERE, "cuda_emul.h"),
          "-Wno-unused-function", "-Wno-unknown-pragmas", "-fno-strict-aliasing"]
FLAGS = ["-O2", *COMMON]
RACECHECK_FLAGS = ["-O1", "-g", "-fsanitize=thread", "-DMGB_EMUL_RACECHECK", *COMMON]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("emulator build failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)


def build(force: bool = False, racecheck: bool = False) -> str:
    out_dir = RACECHECK_DIR if racecheck else OUT_DIR
    flags = RACECHECK_FLAGS if racecheck else FLAGS
    lib_path = os.path.join(out_dir, os.path.basename(LIB_PATH))
    os.makedirs(out_dir, exist_ok=True)
    deps_common = [os.path.join(SRC_DIR, f) for f in os.listdir(SRC_DIR) if f.endswith(".cuh")]
    deps_common += [os.path.join(HERE, "cuda_emul.h"), os.path.join(ROOT, "include", "matchering_b200.h")]
    jobs, objs = [], []
    for src in SOURCES:
        s = os.path.join(SRC_DIR, src)
        o = os.path.join(out_dir, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + deps_common):
            jobs.append(["g++", *flags, "-x", "c++", "-c", s, "-o", o])
    o = emul_object(out_dir, racecheck, force)
    objs.append(o)

    with ThreadPoolExecutor(max_workers=8) as ex:
        list(ex.map(_run, jobs))
    if jobs or _stale(lib_path, objs):
        _run(["g++", "-shared", *(["-fsanitize=thread"] if racecheck else []), "-o", lib_path, *objs])
    return lib_path


def emul_object(out_dir: str, racecheck: bool, force: bool = False) -> str:
    """The scheduler's object file in `out_dir` (never instrumented), rebuilt when stale."""
    s = os.path.join(HERE, "cuda_emul.cpp")
    o = os.path.join(out_dir, "cuda_emul.o")
    if force or _stale(o, [s, os.path.join(HERE, "cuda_emul.h")]):
        _run(["g++", "-O2", "-std=c++17", "-fPIC", "-DMGB_EMULATE", *(["-DMGB_EMUL_RACECHECK"] if racecheck else []),
              "-c", s, "-o", o])
    return o


def build_racecheck_controls(force: bool = False) -> str:
    """The race checker's controls (racecheck_controls.cu), an executable built like the race-checking library."""
    build(force, racecheck=True)
    # the controls include design.cu (for its radix select) and link the library's other objects
    objs = [os.path.join(RACECHECK_DIR, f.replace(".cu", ".o")) for f in SOURCES if f != "design.cu"]
    objs.append(os.path.join(RACECHECK_DIR, "cuda_emul.o"))
    s = os.path.join(HERE, "racecheck_controls.cu")
    exe = os.path.join(RACECHECK_DIR, "racecheck_controls")
    deps = [s, os.path.join(HERE, "cuda_emul.h"), os.path.join(SRC_DIR, "design.cu"), *objs]
    deps += [os.path.join(SRC_DIR, f) for f in os.listdir(SRC_DIR) if f.endswith(".cuh")]
    if force or _stale(exe, deps):
        _run(["g++", *RACECHECK_FLAGS, "-x", "c++", s, "-x", "none", *objs, "-o", exe])
    return exe


if __name__ == "__main__":
    import sys
    print(build(racecheck="--racecheck" in sys.argv[1:]))
