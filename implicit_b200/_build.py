"""Builds libals_b200.so (sm_90a only) in-tree with plain nvcc -- no CMake, no torch extension.

    python -m implicit_b200._build [--force] [--verbose]

The built library lives next to the sources (implicit_b200/libals_b200.so) and is git-ignored.  nvcc
cross-compiles without a GPU.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "_obj")
LIB = os.path.join(HERE, "libals_b200.so")
SOURCES = ["api.cu", "csr.cu", "gen.cu", "gramian.cu", "cholesky.cu", "cholesky_tc.cu", "cholesky_short.cu", "dense.cu", "cholesky_wide.cu", "cholesky_xwide.cu", "cg.cu", "loss.cu", "topk.cu", "topk_tc.cu", "metrics.cu", "serve.cu", "refit.cu", "comm.cu"]
HEADERS = [os.path.join(CSRC, "common.h"), os.path.join(CSRC, "cholesky_device.cuh"), os.path.join(CSRC, "sm90.cuh"),
           os.path.join(HERE, "..", "include", "als_b200.h")]

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden", "-ccbin", "/usr/bin/g++",
    "--expt-relaxed-constexpr", "-I", "/usr/include",
]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    jobs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src.replace(".cu", ".o"))
        if force or _stale(o, [s] + HEADERS):
            cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
            jobs.append((src, cmd))

    def run(job):
        src, cmd = job
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, r

    failed = False
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        for src, r in ex.map(run, jobs):
            if verbose or r.returncode != 0:
                sys.stderr.write(f"--- {src}\n{r.stdout}{r.stderr}\n")
            failed |= r.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed building libals_b200.so")
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or _stale(LIB, objs):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-lcudart", "-ldl", "-lpthread", "-ccbin", "/usr/bin/g++"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed for libals_b200.so")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
