"""The opt-in wgmma long-row kernel (csrc/cholesky_tc.cu, knob long_tc) against the oracle and against the default
mma.sync kernel.  Runs in a subprocess with a time limit: a synchronisation bug in a warp-specialised kernel shows up
as a hang, and that must fail this test only."""
import json
import os
import subprocess
import sys

import pytest

from helpers import CHOL_MAX

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _run(*args):
    r = subprocess.run([sys.executable, os.path.join(HERE, "_long_tc_case.py"), *args], capture_output=True, text=True, timeout=240)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_long_rows_tcgen05_matches_oracle_and_default_kernel():
    out = _run()
    print(out)
    for k in ("tc0", "tc1"):
        assert out[k]["max"] < CHOL_MAX and out[k]["empty_row_zero"]
    assert out["tc_vs_legacy_max"] < CHOL_MAX
    assert out["tc1"]["launches"] != out["tc0"]["launches"]  # the knob really switched kernels


def test_long_rows_tcgen05_not_used_with_weights_below_one():
    out = _run("below_one")
    print(out)
    assert out["tc1"]["launches"] == out["tc0"]["launches"]  # |c| - 1 < 0 somewhere: same (mma.sync) launches either way
    assert out["tc1"]["max"] < CHOL_MAX and out["tc_vs_legacy_max"] == 0.0
