"""The algebra behind csrc/cholesky_short.cu, restated in numpy float32 and checked on the CPU against the oracle
(the reference's own `least_squares` when oracle/_ref is built): for a row with n nonzeros

    x = (G + V^T D V)^-1 V^T c+  =  P W_u^T E (I + E K E)^-1 E^-1 c+,    G = R^T R,  P = R^-1,  W = Y P,  K = W_u W_u^T

This is test infrastructure for the DESIGN.md section 4.1b claim that the n x n route is as accurate in fp32 as
the F x F normal equations; the CUDA kernels themselves are covered by tests/test_gpu_parity.py."""
import numpy as np
import pytest
import scipy.linalg as sl

import oracle
from helpers import cholesky_truth, row_err
from implicit_b200 import synthetic


def pushthrough_rows_fp32(Cui, Y, reg):
    f = Y.shape[1]
    G = (Y.T @ Y).astype(np.float32).astype(np.float64) + reg * np.eye(f)  # fp32 Gramian, like the device
    R = np.linalg.cholesky(G).T
    P = np.linalg.inv(R).astype(np.float32)  # fp64 factorisation, fp32 result (whiten_factor_kernel)
    W = (Y @ P).astype(np.float32)           # whiten_rows_kernel
    X = np.zeros((Cui.shape[0], f), dtype=np.float32)
    for u in range(Cui.shape[0]):
        s, e = Cui.indptr[u], Cui.indptr[u + 1]
        if s == e:
            continue
        idx, c = Cui.indices[s:e], Cui.data[s:e].astype(np.float32)
        w = np.abs(c) - 1
        assert (w >= 0).all()  # rows with negative weights never take this path
        E = np.sqrt(np.maximum(w, 1e-10)).astype(np.float32)
        Wu = W[idx]
        M = (np.eye(len(idx), dtype=np.float32) + E[:, None] * (Wu @ Wu.T).astype(np.float32) * E[None, :]).astype(np.float32)
        rhs = (np.where(c > 0, c, 0) / E).astype(np.float32)
        L = np.linalg.cholesky(M)
        sv = sl.solve_triangular(L.T, sl.solve_triangular(L, rhs, lower=True).astype(np.float32), lower=False).astype(np.float32)
        X[u] = (P @ (Wu.T @ (E * sv)).astype(np.float32)).astype(np.float32)
    return X


@pytest.mark.parametrize("warm", [False, True])
@pytest.mark.parametrize("neg", [0.0, 0.1])
def test_pushthrough_matches_reference_solve(warm, neg):
    orc = oracle.get("auto")
    Cui = synthetic.power_law_csr(600, 400, 9000, 77, neg)  # ~15 nonzeros per row: all "short" at f=64
    X, Y = synthetic.initial_factors(600, 400, 64)
    if warm:
        oracle.fit(Cui, X, Y, iterations=2, use_cg=False, kind=orc.name)
    exp = X.copy()
    orc.least_squares(Cui, exp, Y, 0.01)
    got = pushthrough_rows_fp32(Cui, Y, 0.01)
    # fp64 truth, to show the two fp32 routes are equally far from it
    truth = cholesky_truth(Cui, Y, 0.01)
    e_ref, e_new = row_err(exp, truth), row_err(got, truth)
    print(f"warm={warm} neg={neg}: reference vs fp64 max {e_ref.max():.2e}; push-through vs fp64 max {e_new.max():.2e}; "
          f"push-through vs reference max {row_err(got, exp).max():.2e}")
    assert row_err(got, exp).max() < 1e-4          # the parity bar of north_star
    assert e_new.max() < max(2 * e_ref.max(), 2e-5)  # and no less accurate than the F x F route
