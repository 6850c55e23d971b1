"""Row error of the Cholesky half above 128 factors against fp64, next to the fp32 reference's own.

    python tools/xwide_precision.py [f ...]            (default: 512 896 1024)
    ALS_B200_LIB=variants/<name>.so python tools/xwide_precision.py 1024

Uses the data of tests/test_gpu_cholesky_wide.py (mixed_csr with giant rows and duplicates, 100 or 300 users, 2000
items) with cold and warm Y, and prints the max and median row error of the fp32 reference (oracle), of
als_least_squares (device Gramian) and of als_least_squares_with_gramian (the fp32 Gramian the reference uses).
A/B runs of kernel variants built with tools/build_variant.sh tell where the error of the path comes from.
"""
import os
import sys

os.environ.setdefault("OPENBLAS_NUM_THREADS", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import oracle  # noqa: E402
from helpers import mixed_csr, row_err  # noqa: E402
from implicit_b200 import _lib  # noqa: E402
from test_gpu_cholesky_wide import GIANTS, factors, truth_and_reference  # noqa: E402


def main():
    widths = [int(a) for a in sys.argv[1:]] or [512, 896, 1024]
    orc = oracle.get("auto")
    ctx = _lib.Context(0)
    print(f"library: {os.environ.get('ALS_B200_LIB', 'default')}")
    for f in widths:
        for state in ("cold", "warm"):
            users = 300 if f <= 384 else 100
            items, reg = 2000, 0.01
            Cui = mixed_csr(users, items, 1000 + f, giants=GIANTS, duplicates=True)
            Y = factors(state, items, f, seed=f)
            truth, exp = truth_and_reference(orc, Cui, Y, reg)
            Y64 = Y.astype(np.float64)
            YtY = (Y64.T @ Y64).astype(np.float32)
            C = _lib.DeviceCSR.upload(ctx, Cui)
            dY = _lib.DeviceFactors.from_host(ctx, Y)
            dX = _lib.DeviceFactors(ctx, users, f)
            _lib.least_squares(ctx, C, dX, dY, reg)
            e_ls = row_err(dX.download(), truth)
            _lib.least_squares_with_gramian(ctx, YtY, C, dX, dY, reg)
            e_wg = row_err(dX.download(), truth)
            for h in (C, dY, dX):
                h.close()
            e_ref = row_err(exp, truth)
            print(f"f={f:4d} {state}: reference max {e_ref.max():.2e} median {np.median(e_ref):.2e} | "
                  f"least_squares max {e_ls.max():.2e} median {np.median(e_ls):.2e} | "
                  f"with_gramian max {e_wg.max():.2e} median {np.median(e_wg):.2e}", flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
