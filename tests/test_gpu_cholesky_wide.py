"""The Cholesky half above 128 factors (cholesky_xwide.cu: padded widths ld = 256 ... 1024, blocked by 64-column panels
with A in a global workspace per CTA) against fp64, and the public methods that use it on wide models.

Every ld class runs at its full width and below it, including widths where fe = roundup(f, 64) < ld, so that the
zero padding columns [f, fe), which are factored, ride along.  Bars are 1.5x the fp32 reference's own
max and median row error against the same fp64 truth, with floors 2e-5 and 2e-6 (those of the fp32 kernels in
test_gpu_cholesky_widths.py).
"""
import numpy as np
import pytest
import scipy.sparse as sp

from helpers import cholesky_truth, mixed_csr, row_err, topk_mismatches, topk_noise
from helpers import ctx, default_knobs, lib, orc, sm  # noqa: F401  (fixtures)
from implicit_b200 import AlternatingLeastSquares, synthetic

pytestmark = pytest.mark.gpu

#: every padded class 256 ... 1024 at its full width and below it (f = 129 factors 192 columns of 256)
WIDTHS = [129, 192, 200, 255, 256, 257, 384, 500, 512, 640, 768, 896, 1000, 1024]
#: giant rows: 2 and 4 chunks of 2048 plus a finish item each (kSplitNnz, kChunkNnz in csrc/common.h)
GIANTS = (3073, 6145)


def bars(e_ref, f=0):
    """1.5x the fp32 reference's max and median row error against the truth, with floors 2e-5 and 2e-6 (those of the
    fp32 kernels in test_gpu_cholesky_widths.py).  At fe = 1024 (f > 960) the median floor is 2.5e-6.  Measured on one
    H100 80GB HBM3 with tools/xwide_precision.py on this module's warm data: the median row error is 1.6e-6 to 1.9e-6
    at f = 896 and 2.0e-6 to 2.3e-6 at f = 1024.  The fp32 reference reaches 1.0e-6 and 1.2e-6 there.  Fp32
    accumulation in the tile routine, the lo * lo term, triangular solves in place of inverses and correctly rounded
    pivots each leave the f = 1024 median within 2% of 2.0e-6 or worse (DESIGN.md section 4.1d)."""
    return max(2e-5, 1.5 * e_ref.max()), max(2.5e-6 if f > 960 else 2e-6, 1.5 * np.median(e_ref))


def within(got, truth, bar_max, bar_med):
    e = row_err(got, truth)
    return e.max(), np.median(e), bool(np.isfinite(got).all()) and e.max() <= bar_max and np.median(e) <= bar_med


def row_slice(Cui, r0, r1):
    """Rows [r0, r1) of a CSR with its stored entries as they are (duplicates and explicit zeros kept)."""
    s, e = Cui.indptr[r0], Cui.indptr[r1]
    return sp.csr_matrix((Cui.data[s:e], Cui.indices[s:e], Cui.indptr[r0:r1 + 1] - s), shape=(r1 - r0, Cui.shape[1]))


def truth_and_reference(orc, Cui, Y, reg, block=32):
    """(fp64 truth, fp32 reference) of one Cholesky half, on row slices with one fp64 Y^T Y: the fp64 batch of a
    slice stays near 0.3 GB at 1024 factors."""
    Y64 = Y.astype(np.float64)
    G64 = Y64.T @ Y64
    G32 = G64.astype(np.float32)
    truth = np.zeros((Cui.shape[0], Y.shape[1]))
    exp = np.zeros((Cui.shape[0], Y.shape[1]), dtype=np.float32)
    for r0 in range(0, Cui.shape[0], block):
        r1 = min(r0 + block, Cui.shape[0])
        part = row_slice(Cui, r0, r1)
        truth[r0:r1] = cholesky_truth(part, Y, reg, YtY=G64)
        out = np.zeros((r1 - r0, Y.shape[1]), dtype=np.float32)
        orc._least_squares(G32, part.indptr, part.indices, part.data.astype(np.float32), out, Y, reg, 0)
        exp[r0:r1] = out
    return truth, exp


def factors(state, rows, f, seed):
    """cold: the all-positive initialisation U(0, 0.01); warm: mixed signs at the scale of a fitted model."""
    rng = np.random.default_rng(seed)
    if state == "cold":
        return rng.random((rows, f), dtype=np.float32) * np.float32(0.01)
    return (rng.standard_normal((rows, f), dtype=np.float32) * np.float32(0.1)).astype(np.float32)


@pytest.mark.parametrize("state", ["cold", "warm"])
@pytest.mark.parametrize("f", WIDTHS)
def test_wide_cholesky_half_against_fp64(lib, ctx, orc, f, state):
    """One seeded CSR (rows at every short-class boundary, empty rows, negative confidences, weights below zero,
    stored zeros, duplicates, giant rows of 3073 and 6145 nonzeros) through als_least_squares and
    als_least_squares_with_gramian against fp64.  Empty rows must be exactly zero.  Then the item half from the
    device-resident X, checked on a slice of items: non-zero columns [f, fe) in X would enter its Gramian and normal
    equations.  (Columns [fe, ld) are zero from allocation and upload and no solver reads them, so no result shows a
    kernel that leaves them alone instead of writing zeros.)  The item
    half takes confidences |c| + 1 and a regularization of 1% of ||X||_F^2: with 100 users X^T X has rank 100 < f, and
    after a cold half X's norms are large, so that reg = 0.01 would leave the item systems singular in fp32."""
    users = 300 if f <= 384 else 100
    items, reg = 2000, 0.01
    Cui = mixed_csr(users, items, 1000 + f, giants=GIANTS, duplicates=True)
    empty = np.diff(Cui.indptr) == 0
    Y = factors(state, items, f, seed=f)
    truth, exp = truth_and_reference(orc, Cui, Y, reg)
    bar_max, bar_med = bars(row_err(exp, truth), f)
    Y64 = Y.astype(np.float64)
    YtY = (Y64.T @ Y64).astype(np.float32)
    C = lib.DeviceCSR.upload(ctx, Cui)
    dY = lib.DeviceFactors.from_host(ctx, Y)
    results, dX_keep = {}, None
    for name in ("least_squares", "with_gramian"):
        dX = lib.DeviceFactors.from_host(ctx, np.full((users, f), np.nan, np.float32))
        if name == "with_gramian":
            lib.least_squares_with_gramian(ctx, YtY, C, dX, dY, reg)
        else:
            lib.least_squares(ctx, C, dX, dY, reg)
        got = dX.download()
        results[name] = within(got, truth, bar_max, bar_med) + (bool(np.all(got[empty] == 0)),)
        if name == "least_squares":
            dX_keep, X_got = dX, got
        else:
            dX.close()
    C.close()
    dY.close()

    # the item half from the X left on the device, checked on its first 96 items (and all of its empty ones)
    Ciu = Cui.T.tocsr()
    Ciu.data = np.abs(Ciu.data) + 1
    reg_i = 0.01 * float(np.square(X_got.astype(np.float64)).sum())
    dYn = lib.DeviceFactors.from_host(ctx, np.full((items, f), np.nan, np.float32))
    Ci = lib.DeviceCSR.upload(ctx, Ciu)
    lib.least_squares(ctx, Ci, dYn, dX_keep, reg_i)
    got_i = dYn.download()
    for h in (Ci, dYn, dX_keep):
        h.close()
    n_chk = 96
    truth_i, exp_i = truth_and_reference(orc, row_slice(Ciu, 0, n_chk), X_got, reg_i)
    bar_max_i, bar_med_i = bars(row_err(exp_i, truth_i), f)
    results["item half"] = within(got_i[:n_chk], truth_i, bar_max_i, bar_med_i) + (
        bool(np.all(got_i[np.diff(Ciu.indptr) == 0] == 0)),)

    print(f"f={f} {state}: bars {bar_max:.2e} / {bar_med:.2e}; item half {bar_max_i:.2e} / {bar_med_i:.2e}")
    for name, (mx, md, ok, zero) in results.items():
        bm, bd = (bar_max_i, bar_med_i) if name == "item half" else (bar_max, bar_med)
        print(f"   {name:13s} worst ratio max {mx / bm:.2f} median {md / bd:.2f}, empty rows zero {zero}")
    bad = {n: r for n, r in results.items() if not (r[2] and r[3])}
    assert not bad


def _solve_and_check(lib, ctx, orc, Cui, Y, reg=0.01):
    truth, exp = truth_and_reference(orc, Cui, Y, reg)
    bar_max, bar_med = bars(row_err(exp, truth), Y.shape[1])
    C = lib.DeviceCSR.upload(ctx, Cui)
    dY = lib.DeviceFactors.from_host(ctx, Y)
    dX = lib.DeviceFactors.from_host(ctx, np.full((Cui.shape[0], Y.shape[1]), np.nan, np.float32))
    lib.least_squares(ctx, C, dX, dY, reg)
    got = dX.download()
    for h in (C, dY, dX):
        h.close()
    mx, md, ok = within(got, truth, bar_max, bar_med)
    zero = bool(np.all(got[np.diff(Cui.indptr) == 0] == 0))
    print(f"   worst ratio max {mx / bar_max:.2f} median {md / bar_med:.2f}, empty rows zero {zero}")
    return ok and zero


def _csr_of_lengths(lens, items, seed):
    rng = np.random.default_rng(seed)
    lens = np.asarray(lens)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    cols = np.concatenate([rng.choice(items, n, replace=n > items) for n in lens] + [np.zeros(0, int)]).astype(np.int32)
    vals = (1 + 4 * rng.random(int(indptr[-1]))).astype(np.float32)
    vals[rng.random(len(vals)) < 0.1] *= -1
    return sp.csr_matrix((vals, cols, indptr), shape=(len(lens), items))


def test_wide_cholesky_grid_and_workspace_edges(lib, ctx, orc, sm):
    """Fewer work items than SMs; several times more rows than resident CTAs, so that every CTA reuses its
    workspace; a CSR whose only row is a giant one (pass 0: its four chunks and nothing else; pass 1: one finish
    item), at the narrowest and the widest class."""
    items = 3000
    cases = {
        "few items, f=512": (_csr_of_lengths([0, 1, 5, 64, 200, 33, 1], items, 1), 512),
        "rows >> CTAs, f=256": (_csr_of_lengths(np.random.default_rng(2).integers(0, 40, 8 * 2 * sm), items, 2), 256),
        "one giant row, f=256": (_csr_of_lengths([6145], items, 3), 256),
        "one giant row, f=1024": (_csr_of_lengths([6145], items, 4), 1024),
    }
    ok = {}
    for name, (Cui, f) in cases.items():
        print(name)
        ok[name] = _solve_and_check(lib, ctx, orc, Cui, factors("warm", items, f, seed=f))
    assert all(ok.values()), ok


@pytest.mark.parametrize("f", [256, 1024])
def test_wide_cholesky_failure_names_first_bad_row(lib, ctx, orc, f):
    """regularization=0 and a Y whose last column is non-zero on item 7 only: a row that stores a zero for item 7
    subtracts y_7 y_7^T and leaves that column of A zero, so its normal equations are singular.  Rows 5 and 9 do;
    the call raises ValueError naming row 5.  The next call on the same context succeeds."""
    items = 2500
    rng = np.random.default_rng(f)
    Y = (rng.standard_normal((items, f)) * 0.1).astype(np.float32)
    Y[:, -1] = 0
    Y[7, -1] = 1
    lens = [0, 0, 30, 12, 3100, 40, 0, 7, 6145, 25, 16]
    Cui = _csr_of_lengths(lens, items, 5)
    Cui.data = np.abs(Cui.data)
    Cui.indices[Cui.indices == 7] = 8  # item 7 only where placed below
    for u in (5, 9):
        Cui.indices[Cui.indptr[u]] = 7
        Cui.data[Cui.indptr[u]] = 0.0
    C = lib.DeviceCSR.upload(ctx, Cui)
    dY = lib.DeviceFactors.from_host(ctx, Y)
    dX = lib.DeviceFactors.from_host(ctx, np.zeros((len(lens), f), np.float32))
    with pytest.raises(ValueError, match="row 5"):
        lib.least_squares(ctx, C, dX, dY, 0.0)
    for h in (C, dY, dX):
        h.close()
    assert _solve_and_check(lib, ctx, orc, _csr_of_lengths(lens, items, 6), factors("warm", items, f, seed=3))


@pytest.fixture(scope="module", params=[200, 512])
def wide_model(request):
    f = request.param
    Cui = synthetic.power_law_csr(600, 400, 15000, 12)
    model = AlternatingLeastSquares(factors=f, use_cg=True, iterations=3, random_state=3)
    X0, Y0 = synthetic.initial_factors(600, 400, f)
    model.user_factors, model.item_factors = X0.copy(), Y0.copy()
    model.fit(Cui, show_progress=False)
    return model, Cui


def test_wide_model_recalculate(orc, wide_model):
    """recalculate_user / recalculate_item against fp64 with the model's own Gramians, and a batch equals its
    scalars."""
    model, Cui = wide_model
    X, Y = np.array(model.user_factors), np.array(model.item_factors)
    ok = {}
    for side, M, other, gram in (("user", Cui, Y, model.YtY), ("item", Cui.T.tocsr(), X, model.XtX)):
        ids = np.arange(0, M.shape[0], 3)
        rows = M[ids]
        fn = model.recalculate_user if side == "user" else model.recalculate_item
        got = fn(ids, rows)
        truth = cholesky_truth(rows, other, model.regularization, YtY=gram)
        exp = np.zeros_like(got)
        orc._least_squares(np.asarray(gram, np.float32), rows.indptr, rows.indices, rows.data.astype(np.float32), exp,
                           other, model.regularization, 0)
        bar_max, bar_med = bars(row_err(exp, truth), model.factors)
        mx, md, good = within(got, truth, bar_max, bar_med)
        print(f"f={model.factors} {side}: worst ratio max {mx / bar_max:.2f} median {md / bar_med:.2f}")
        for n in (0, 5, len(ids) - 1):
            np.testing.assert_allclose(fn(ids[n], M[ids[n]]), got[n], rtol=1e-4, atol=1e-7)
        ok[side] = good
    assert all(ok.values()), ok


def test_wide_model_recommend_and_similar_items(wide_model):
    """recommend(recalculate_user=True) ranks the items by the recalculated factors; similar_items(recalculate_item=True)
    by cosine against the recalculated item."""
    model, Cui = wide_model
    Y = np.array(model.item_factors, dtype=np.float64)
    users = np.arange(0, 60, 2)
    N = 10
    ids, scores = model.recommend(users, Cui[users], N=N, recalculate_user=True)
    q = model.recalculate_user(users, Cui[users]).astype(np.float64)
    full = q @ Y.T
    full[Cui[users].nonzero()] = -np.inf
    ref_ids = np.argsort(-full, axis=1, kind="stable")[:, :N]
    ref_scores = np.take_along_axis(full, ref_ids, axis=1)
    _, bad = topk_mismatches(ids, scores, ref_ids, ref_scores, topk_noise(q, Y))
    assert not bad.any()

    item = 17
    ids, scores = model.similar_items(item, N=N, recalculate_item=True, item_users=Cui.T.tocsr()[item])
    v = model.recalculate_item(item, Cui.T.tocsr()[item]).astype(np.float64)
    cos = (Y @ v) / np.maximum(np.linalg.norm(Y, axis=1) * np.linalg.norm(v), 1e-30)
    assert len(ids) == N and np.isfinite(scores).all()
    # every returned item is within fp32 noise of the N-th best cosine
    assert np.all(cos[ids] >= np.sort(cos)[-N] - 1e-5)


def test_wide_model_partial_fit():
    """partial_fit_users / partial_fit_items grow the factor matrices and store the recalculated rows."""
    f = 200
    Cui = synthetic.power_law_csr(300, 250, 6000, 21)
    model = AlternatingLeastSquares(factors=f, use_cg=True, iterations=2, random_state=1)
    model.fit(Cui, show_progress=False)
    new_users = np.array([3, 310, 305])
    rows = Cui[[10, 20, 30]]
    want = model.recalculate_user(new_users, rows)
    model.partial_fit_users(new_users, rows)
    assert model.user_factors.shape == (311, f)
    np.testing.assert_allclose(model.user_factors[new_users], want, rtol=1e-4, atol=1e-7)
    Ciu = Cui.T.tocsr()
    new_items = np.array([1, 260])
    irows = Ciu[[5, 6]]
    irows = sp.csr_matrix((irows.data, irows.indices, irows.indptr), shape=(2, model.user_factors.shape[0]))
    want_i = model.recalculate_item(new_items, irows)
    model.partial_fit_items(new_items, irows)
    assert model.item_factors.shape == (261, f)
    np.testing.assert_allclose(model.item_factors[new_items], want_i, rtol=1e-4, atol=1e-7)
    assert np.isfinite(model.user_factors).all() and np.isfinite(model.item_factors).all()
