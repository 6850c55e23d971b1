"""Models wider than 128 factors (the reference's CUDA solver takes up to 1024, implicit/gpu/als.cu:177-178; its CPU
path any width): CG half, loss, top-k and the fit loop at 192 / 260 / 512 factors against the oracle (the Gramian:
test_gpu_gramian_widths.py)."""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from helpers import row_err
from implicit_b200 import AlternatingLeastSquares, synthetic

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from implicit_b200 import _lib

    return _lib


@pytest.fixture(scope="module")
def ctx(lib):
    c = lib.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def orc():
    return oracle.get("auto")


def _case(users, items, nnz, f, seed):
    Cui = synthetic.power_law_csr(users, items, nnz, seed, 0.05)
    rng = np.random.default_rng(seed)
    X = (rng.standard_normal((users, f)) * 0.1).astype(np.float32)
    Y = (rng.standard_normal((items, f)) * 0.1).astype(np.float32)
    return Cui, X, Y


@pytest.mark.parametrize("f", [192, 260, 512])
def test_wide_cg_half_matches_oracle(lib, ctx, orc, f):
    Cui, X, Y = _case(400, 300, 9000, f, seed=900 + f)
    exp = X.copy()
    orc.least_squares_cg(Cui, exp, Y, 0.01, cg_steps=3)
    C = lib.DeviceCSR.upload(ctx, Cui)
    dX, dY = lib.DeviceFactors.from_host(ctx, X), lib.DeviceFactors.from_host(ctx, Y)
    lib.least_squares_cg(ctx, C, dX, dY, 0.01, 3)
    e = row_err(dX.download(), exp)
    print(f"wide cg f={f}: max {e.max():.2e} median {np.median(e):.2e}")
    assert e.max() < 1e-4 and np.median(e) < 1e-5
    for h in (C, dX, dY):
        h.close()


def test_wide_cg_giant_and_empty_rows(lib, ctx, orc):
    rng = np.random.default_rng(41)
    users, items, f = 24, 7000, 256
    rows, cols, vals = [], [], []
    for u, n in enumerate([6500, 3100, 0, 17] + [60] * 20):
        c = rng.choice(items, n, replace=False)
        rows += [u] * n
        cols += c.tolist()
        vals += (1 + 4 * rng.random(n)).tolist()
    Cui = sp.csr_matrix((np.array(vals, dtype=np.float32), (rows, cols)), shape=(users, items))
    Y = (rng.standard_normal((items, f)) * 0.1).astype(np.float32)
    X = (rng.standard_normal((users, f)) * 0.1).astype(np.float32)
    exp = X.copy()
    orc.least_squares_cg(Cui, exp, Y, 0.05, cg_steps=3)
    C = lib.DeviceCSR.upload(ctx, Cui)
    dX, dY = lib.DeviceFactors.from_host(ctx, X), lib.DeviceFactors.from_host(ctx, Y)
    lib.least_squares_cg(ctx, C, dX, dY, 0.05, 3)
    got = dX.download()
    assert np.all(got[2] == 0)
    assert row_err(got, exp).max() < 1e-4
    for h in (C, dX, dY):
        h.close()


@pytest.mark.parametrize("f", [192, 384])
def test_wide_loss_matches_oracle(lib, ctx, orc, f):
    Cui, X, Y = _case(300, 250, 5000, f, seed=700 + f)
    C = lib.DeviceCSR.upload(ctx, Cui)
    dX, dY = lib.DeviceFactors.from_host(ctx, X), lib.DeviceFactors.from_host(ctx, Y)
    got = lib.calculate_loss(ctx, C, dX, dY, 0.01)
    assert got == pytest.approx(orc.calculate_loss(Cui, X, Y, 0.01), rel=1e-5)
    for h in (C, dX, dY):
        h.close()


def test_wide_topk_matches_oracle(lib, ctx, orc):
    f, k = 192, 10
    rng = np.random.default_rng(77)
    items = (rng.standard_normal((2000, f)) * 0.3).astype(np.float32)
    query = (rng.standard_normal((60, f)) * 0.3).astype(np.float32)
    liked = synthetic.power_law_csr(60, 2000, 900, 8)
    di, dq = lib.DeviceFactors.from_host(ctx, items), lib.DeviceFactors.from_host(ctx, query)
    dl = lib.DeviceCSR.upload(ctx, liked)
    ids, sc = lib.topk(ctx, di, dq, k, liked=dl)
    eids, esc = orc.topk(items, query, k, filter_query_items=liked)
    np.testing.assert_allclose(sc, esc, rtol=1e-5, atol=1e-6)
    diff = ids != eids
    assert diff.mean() < 0.01
    for h in (di, dq, dl):
        h.close()


def test_wide_fit_and_recommend(orc):
    """factors=200 through the public class: the loss falls like the oracle's fit and recommend returns the true top items."""
    Cui = synthetic.power_law_csr(600, 400, 15000, 12)
    losses = []
    model = AlternatingLeastSquares(factors=200, use_cg=True, iterations=3, calculate_training_loss=True, random_state=3)
    X0, Y0 = synthetic.initial_factors(600, 400, 200)
    model.user_factors, model.item_factors = X0.copy(), Y0.copy()
    model.fit(Cui, show_progress=False, callback=lambda i, t, l: losses.append(l))
    Xo, Yo = X0.copy(), Y0.copy()
    oracle.fit(Cui, Xo, Yo, iterations=3, use_cg=True, kind=orc.name)
    exp_loss = orc.calculate_loss(Cui, Xo, Yo, 0.01)
    assert losses[0] > losses[-1]
    assert losses[-1] == pytest.approx(exp_loss, rel=2e-3)
    ids, scores = model.recommend(np.arange(20), Cui[:20], N=5)
    full = np.array(model.user_factors)[:20] @ np.array(model.item_factors).T
    full[Cui[:20].nonzero()] = -np.inf
    assert (ids[:, 0] == full.argmax(axis=1)).mean() > 0.9
    with pytest.raises(ValueError):
        AlternatingLeastSquares(factors=200, use_cg=False)
    with pytest.raises(ValueError):
        AlternatingLeastSquares(factors=2000)
