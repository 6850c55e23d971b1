"""A Cholesky half whose normal equations are not positive definite on some row (helpers.bad_row_csr, lambda = 0 and
Y = I): every width family (f = 16 and 64 in cholesky.cu, 100 in cholesky_wide.cu, 200 in cholesky_xwide.cu) must name
the lowest such row, synchronously or through solver_status after the asynchronous half, and leave the context clean
for the next call.
"""
import numpy as np
import pytest

from helpers import bad_row_csr
from helpers import ctx, default_knobs, lib  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu
WIDTHS = [16, 64, 100, 200]


def upload(lib, ctx, f, csrs):
    """The CSRs on the device, then Y = I and X."""
    Yd = lib.DeviceFactors.from_host(ctx, np.eye(f, dtype=np.float32))
    return [lib.DeviceCSR.upload(ctx, C) for C in csrs] + [Yd, lib.DeviceFactors(ctx, csrs[0].shape[0], f)]


@pytest.mark.parametrize("f", WIDTHS)
def test_sync_half_names_lowest_bad_row(lib, ctx, f):
    d, clean, Yd, X = hs = upload(lib, ctx, f, [bad_row_csr(f, [30, 12]), bad_row_csr(f, [])])
    for solve in (lambda C: lib.least_squares(ctx, C, X, Yd, 0.0),
                  lambda C: lib.least_squares_with_gramian(ctx, np.eye(f, dtype=np.float32), C, X, Yd, 0.0),
                  lambda C: lib.half_pregram(ctx, C, X, Yd, 0.0, use_cg=False)):
        lib.gramian(ctx, Yd)
        with pytest.raises(ValueError, match=r"row 12\b"):
            solve(d)
        lib.gramian(ctx, Yd)
        solve(clean)  # the failure was reported once: the next call on the context succeeds
        np.testing.assert_allclose(X.download(), bad_row_csr(f, []).toarray() > 0, atol=1e-5)  # x = 1 on its items
    lib.solver_status(ctx)
    for h in hs:
        h.close()


@pytest.mark.parametrize("f", WIDTHS)
@pytest.mark.parametrize("second", [[], [30]], ids=["then_clean", "then_failing"])
def test_async_halves_report_the_lowest_bad_row(lib, ctx, f, second):
    """A failing asynchronous half, then a clean or a failing one: solver_status names the lower row, once."""
    lib.solver_status(ctx)
    first, then, Yd, X = hs = upload(lib, ctx, f, [bad_row_csr(f, [12]), bad_row_csr(f, second)])
    lib.gramian(ctx, Yd)
    lib.half_pregram_async(ctx, first, X, Yd, 0.0, use_cg=False)
    lib.half_pregram_async(ctx, then, X, Yd, 0.0, use_cg=False)
    with pytest.raises(ValueError, match=r"row 12\b"):
        lib.solver_status(ctx)
    lib.solver_status(ctx)  # a new collection period: clean
    for h in hs:
        h.close()
