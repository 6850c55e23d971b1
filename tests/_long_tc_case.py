"""Helper of tests/test_gpu_long_tc.py (run as a subprocess so that a hanging kernel cannot take the suite with it):
one Cholesky half over rows of 0 ... 3500 nonzeros with the wgmma long-row kernel (knob long_tc) and with the
mma.sync kernel, both against the oracle.  Prints one JSON line."""
import json
import os
import sys

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import oracle  # noqa: E402
from helpers import row_err  # noqa: E402
from implicit_b200 import _lib  # noqa: E402

below_one = len(sys.argv) > 1 and sys.argv[1] == "below_one"
rng = np.random.default_rng(17)
items, f = 6000, 64
lengths = [3500, 3072, 1000, 500, 65, 64, 63, 49, 48, 0, 17, 33] + rng.integers(49, 300, 1500).tolist()
rows, cols, vals = [], [], []
for u, n in enumerate(lengths):
    c = rng.choice(items, n, replace=False)
    rows += [u] * n
    cols += c.tolist()
    vals += (1 + 4 * rng.random(n)).tolist()
vals = np.array(vals, dtype=np.float32)
if below_one:
    vals[5] = 0.5  # one weight |c| - 1 < 0: the whole CSR must take the mma.sync kernel
Cui = sp.csr_matrix((vals, (rows, cols)), shape=(len(lengths), items))
Y = (rng.standard_normal((items, f)) * 0.1).astype(np.float32)
X0 = np.zeros((len(lengths), f), dtype=np.float32)
exp = X0.copy()
oracle.get("auto").least_squares(Cui, exp, Y, 0.05)
ctx = _lib.Context(0)
out = {}
res = {}
for tc in (0, 1):
    ctx.set_knob("long_tc", tc)
    C = _lib.DeviceCSR.upload(ctx, Cui)
    dX, dY = _lib.DeviceFactors.from_host(ctx, X0), _lib.DeviceFactors.from_host(ctx, Y)
    n0 = ctx.launch_count()
    _lib.least_squares(ctx, C, dX, dY, 0.05)
    res[tc] = dX.download()
    e = row_err(res[tc], exp)
    out[f"tc{tc}"] = {"max": float(e.max()), "median": float(np.median(e)), "empty_row_zero": bool(np.all(res[tc][9] == 0)),
                      "launches": int(ctx.launch_count() - n0)}
    for h in (C, dX, dY):
        h.close()
out["tc_vs_legacy_max"] = float(row_err(res[1], res[0]).max())
print(json.dumps(out))
