"""The Cholesky kernel above 128 factors (csrc/cholesky_xwide.cu) runs its tile products on the tensor cores and keeps
everything in registers and shared memory (no GPU needed: cuobjdump and ptxas)."""
import os
import shutil
import subprocess

import pytest

from implicit_b200 import _build


def _tool(name):
    exe = shutil.which(name) or os.path.join("/usr/local/cuda/bin", name)
    if not os.path.exists(exe):
        pytest.skip(f"{name} not available")
    return exe


def test_xwide_kernel_uses_hmma_without_spills(tmp_path):
    sass = subprocess.run([_tool("cuobjdump"), "-sass", _build.build()], capture_output=True, text=True).stdout
    per_kernel, fn = {}, None
    for line in sass.splitlines():
        if "Function :" in line:
            fn = line.split("Function :")[1].strip()
            per_kernel[fn] = []
        elif fn is not None:
            per_kernel[fn].append(line)
    body = [ln for name, lines in per_kernel.items() if "cholesky_xwide_kernel" in name for ln in lines]
    assert body, "cholesky_xwide_kernel is not in the library"
    assert any("HMMA" in ln for ln in body)
    assert not any(op in ln for ln in body for op in ("LDL", "STL"))

    cmd = [_build.NVCC] + _build.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(_build.CSRC, "cholesky_xwide.cu"),
                                          "-o", str(tmp_path / "x.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = r.stderr.splitlines()
    at = [i for i, ln in enumerate(lines) if "Compiling entry function" in ln and "cholesky_xwide_kernel" in ln]
    assert at
    props = " ".join(lines[at[0]:at[0] + 4])
    assert "0 bytes spill stores" in props and "0 bytes spill loads" in props and "0 bytes stack frame" in props
