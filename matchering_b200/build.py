"""Build libmatchering_b200.so in-tree with nvcc for sm_90a, the H100 (no torch extension machinery: the
library has a plain C ABI and is loaded with ctypes).  `python -m matchering_b200.build`."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
SRC_DIR = os.path.join(PKG_DIR, "csrc")
OBJ_DIR = os.path.join(PKG_DIR, "_build")
LIB_PATH = os.path.join(PKG_DIR, "libmatchering_b200.so")
SOURCES = ["api.cu", "analyze.cu", "design.cu", "convolve.cu", "correct.cu", "limiter.cu", "pipeline.cu", "hostio.cu", "resample.cu"]
HEADERS = sorted(f for f in os.listdir(SRC_DIR) if f.endswith(".cuh")) + [os.path.join("..", "..", "include", "matchering_b200.h")]

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    *GENCODE,
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
]


def find_nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the CUDA library cannot be built")


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    nvcc = find_nvcc()
    os.makedirs(OBJ_DIR, exist_ok=True)
    headers = [os.path.normpath(os.path.join(SRC_DIR, h)) for h in HEADERS] + [os.path.abspath(__file__)]
    jobs = []
    objs = []
    for src in SOURCES:
        s = os.path.join(SRC_DIR, src)
        o = os.path.join(OBJ_DIR, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + headers):
            jobs.append((src, [nvcc, *NVCC_FLAGS, "-c", s, "-o", o]))

    def run(job):
        name, cmd = job
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = os.path.join(OBJ_DIR, name + ".log")
        with open(log, "w") as f:
            f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {name}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
        return name

    with ThreadPoolExecutor(max_workers=min(6, max(1, len(jobs)))) as ex:
        list(ex.map(run, jobs))
    if jobs or force or _stale(LIB_PATH, objs):
        # (--no-undefined: a symbol that only exists inside another file's anonymous namespace must fail here, not at dlopen)
        cmd = [nvcc, "-shared", *GENCODE, "-Xlinker", "--no-undefined", "-o", LIB_PATH, *objs]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
