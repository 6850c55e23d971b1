"""Workload for profiler captures: a few C2 half-iterations (Cholesky by default, --cg for CG)."""
import os
import sys

os.environ.setdefault("OPENBLAS_NUM_THREADS", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from implicit_b200 import _lib, synthetic  # noqa: E402

cfgname = "C3" if "--c3" in sys.argv else "C2"
ctx = _lib.Context(0)
Cui, X0, Y0, cfg = synthetic.config(cfgname)
C = _lib.DeviceCSR.upload(ctx, Cui)
T = C.transpose()
X, Y = _lib.DeviceFactors.from_host(ctx, X0), _lib.DeviceFactors.from_host(ctx, Y0)
iters = 3
for it in range(iters):
    if "--cg" in sys.argv:
        _lib.least_squares_cg(ctx, C, X, Y, 0.01, 3)
        _lib.least_squares_cg(ctx, T, Y, X, 0.01, 3)
    else:
        _lib.least_squares(ctx, C, X, Y, 0.01)
        _lib.least_squares(ctx, T, Y, X, 0.01)
ctx.sync()
print("done", cfg)
