"""The opt-in wgmma long-row kernel (csrc/cholesky_tc.cu, knob long_tc) against the oracle, against fp64 at its edges
and against the default mma.sync kernel.  Runs in a subprocess with a time limit: a synchronisation bug in a
warp-specialised kernel shows up as a hang, and that must fail this test only."""
import json
import os
import subprocess
import sys

import pytest

from helpers import CHOL_MAX

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _run(*args, timeout=240):
    r = subprocess.run([sys.executable, os.path.join(HERE, "_long_tc_case.py"), *args], capture_output=True, text=True,
                       timeout=timeout)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_long_rows_wgmma_matches_oracle_and_default_kernel():
    out = _run()
    print(out)
    for k in ("tc0", "tc1"):
        assert out[k]["max"] < CHOL_MAX and out[k]["empty_row_zero"]
    assert out["tc_vs_legacy_max"] < CHOL_MAX
    assert out["tc1"]["launches"] != out["tc0"]["launches"]  # the knob really switched kernels


def test_long_rows_wgmma_not_used_with_weights_below_one():
    out = _run("below_one")
    print(out)
    assert out["tc1"]["launches"] == out["tc0"]["launches"]  # |c| - 1 < 0 somewhere: same (mma.sync) launches either way
    assert out["tc1"]["max"] < CHOL_MAX and out["tc_vs_legacy_max"] == 0.0


@pytest.mark.parametrize("f", [64, 50, 63])
def test_long_rows_wgmma_edges_against_fp64(f):
    """Rows of 1 ... 8193 nonzeros around the stage, ring, producer and chunk edges; fewer rows than SMs, exactly four
    work items per SM and over 8 x 4 per SM; warm Y and Y with row norms over six decades; 64 factors and 50 and 63
    (64 padded).  Each case: one launch more than the default kernel (the wgmma kernel ran, the giant rows' chunks
    went to the mma.sync kernel), within 1.5x the fp32 reference's max and median row error against cholesky_truth
    (floors 2e-5 and 2e-6), and within CHOL_MAX of the default kernel."""
    out = _run("edges", str(f), timeout=600)
    bad = []
    for c in out["cases"]:
        print(f"f={f} rows={c['rows']} work={c['work']} (sm {out['sm']}) Y={c['Y']}: worst ratio max {c['max_ratio']:.2f} "
              f"median {c['median_ratio']:.2f} (default kernel {c['default_max_ratio']:.2f}); vs default "
              f"{c['tc_vs_default_max']:.2e}; launches {c['launches_tc']} / {c['launches_default']}")
        if not (c["finite"] and c["max_ratio"] <= 1.0 and c["median_ratio"] <= 1.0 and c["tc_vs_default_max"] < CHOL_MAX
                and c["launches_tc"] == c["launches_default"] + 1):
            bad.append(c)
    assert not bad
