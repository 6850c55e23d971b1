"""Build the reference's OWN CUDA ALS solver (implicit/gpu/als.cu) into oracle/_ref/libref_gpu_als.so.

Test / bench infrastructure only (bench.py --impl reference-gpu; SURVEY.md section 8 rows R7).  The reference's CUDA
build needs rapids-cmake + RMM + RAFT (network), but the ALS solver itself depends only on cuBLAS and on the
Matrix / CSRMatrix *declarations*: oracle/ref_gpu/harness.cu includes implicit/gpu/als.cu from /root/reference where it
lies (nothing is copied), this script supplies a stand-in <rmm/device_uvector.hpp> in a /tmp scratch directory so that
implicit/gpu/matrix.h parses, and only the resulting shared object is written to oracle/_ref/ (git-ignored).
Compiled for sm_90a like the product: this is the "recompiled legacy kernel" baseline.

Usage:  python oracle/build_ref_gpu.py [--force]
"""
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref", "libref_gpu_als.so")
REFERENCE = os.environ.get("ALS_B200_REFERENCE", "/root/reference")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

RMM_STUB = """// stand-in for RMM (not installable offline): only what implicit/gpu/matrix.h needs to PARSE
#pragma once
#include <cstddef>
namespace rmm {
struct device_buffer {};
template <typename T> struct device_uvector {};
}  // namespace rmm
"""


def build(force=False, verbose=False):
    src = os.path.join(REFERENCE, "implicit", "gpu", "als.cu")
    if os.path.exists(OUT) and not force:
        return True
    if not os.path.exists(src):
        return False
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="als_b200_refgpu_")
    try:
        os.makedirs(os.path.join(tmp, "rmm"))
        with open(os.path.join(tmp, "rmm", "device_uvector.hpp"), "w") as fh:
            fh.write(RMM_STUB)
        cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
               "-ccbin", "/usr/bin/g++", "-I", tmp, "-I", REFERENCE, os.path.join(HERE, "ref_gpu", "harness.cu"), "-o", OUT,
               "-lcublas", "-lcudart", "-Xlinker", "--no-undefined"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
        return r.returncode == 0 and os.path.exists(OUT)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    ok = build(force="--force" in sys.argv, verbose=True)
    print("oracle/_ref/libref_gpu_als.so:", "built" if ok else "NOT built")
    sys.exit(0 if ok else 1)
