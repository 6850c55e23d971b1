"""GPU parity tests proper: every call goes Python -> ctypes -> C-ABI (include/als_b200.h) -> sm_90a kernels,
and is compared with the CPU oracle (the reference's own compiled Cython when oracle/_ref is present,
else its C restatement) on the same seeded inputs, and with the committed golden vectors."""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from helpers import CHOL_MAX, cholesky_truth, golden_cases, load_golden, row_err
from implicit_b200 import synthetic

pytestmark = pytest.mark.gpu

ORACLE = None


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


def _case(users, items, nnz, f, seed, neg=0.0, warm=True, orc=None):
    """Seeded CSR + factors; `warm` runs two reference iterations so the state is well conditioned."""
    Cui = synthetic.power_law_csr(users, items, nnz, seed, neg)
    X, Y = synthetic.initial_factors(users, items, f)
    if warm:
        oracle.fit(Cui, X, Y, iterations=2, use_cg=False, kind=orc.name if orc else "auto")
    return Cui, X, Y


def _gpu_half(lib, ctx, Cui, X, Y, reg, use_cg, cg_steps=3):
    C = lib.DeviceCSR.upload(ctx, Cui)
    dX = lib.DeviceFactors.from_host(ctx, X)
    dY = lib.DeviceFactors.from_host(ctx, Y)
    if use_cg:
        lib.least_squares_cg(ctx, C, dX, dY, reg, cg_steps)
    else:
        lib.least_squares(ctx, C, dX, dY, reg)
    out = dX.download()
    for h in (C, dX, dY):
        h.close()
    return out


# ---------------------------------------------------------------------------------------- R4 Gramian
@pytest.mark.parametrize("f", [16, 40, 64, 100, 128])
def test_gramian(lib, ctx, f):
    rng = np.random.default_rng(f)
    Y = (rng.standard_normal((5000, f)) * 0.3).astype(np.float32)
    d = lib.DeviceFactors.from_host(ctx, Y)
    G = lib.gramian(ctx, d)
    d.close()
    G64 = Y.astype(np.float64).T @ Y.astype(np.float64)
    assert np.abs(G - G64).max() / np.abs(G64).max() < 1e-6


# ---------------------------------------------------------------------------------------- R1 Cholesky half
@pytest.mark.parametrize("f", [16, 32, 40, 64])
@pytest.mark.parametrize("neg", [0.0, 0.1])
def test_cholesky_half_matches_oracle(lib, ctx, orc, f, neg):
    Cui, X, Y = _case(700, 450, 9000, f, seed=100 + f, neg=neg, orc=orc)
    exp = X.copy()
    orc.least_squares(Cui, exp, Y, 0.01)
    got = _gpu_half(lib, ctx, Cui, X, Y, 0.01, use_cg=False)
    e = row_err(got, exp)
    print(f"cholesky f={f} neg={neg}: max {e.max():.2e} median {np.median(e):.2e}")
    assert e.max() < CHOL_MAX  # rtol 1e-4 per factor row (north_star); expected ~1e-6


@pytest.mark.parametrize("name", [n for n in golden_cases() if n.startswith("chol")])
def test_cholesky_half_matches_golden(lib, ctx, name):
    rc, Cui, _, _, z = load_golden(name)
    got = _gpu_half(lib, ctx, Cui, z["X"], z["Y"], 0.01, use_cg=False)
    assert row_err(got, z["Xh"]).max() < CHOL_MAX


def test_cholesky_cold_start_and_empty_rows(lib, ctx, orc):
    """First half-iteration from the rng.random()*0.01 start, with empty rows (-> exact zeros)."""
    Cui, X, Y = _case(600, 400, 5000, 64, seed=7, warm=False)
    Cui = Cui.tolil()
    Cui[5, :] = 0
    Cui[77, :] = 0
    Cui = Cui.tocsr()
    Cui.eliminate_zeros()
    exp = X.copy()
    orc.least_squares(Cui, exp, Y, 0.01)
    got = _gpu_half(lib, ctx, Cui, X, Y, 0.01, use_cg=False)
    assert np.all(got[5] == 0) and np.all(got[77] == 0)
    assert row_err(got, exp).max() < CHOL_MAX


def test_cholesky_giant_rows(lib, ctx, orc):
    """Rows above the split threshold take the chunk + finish path; explicit zeros and duplicates too."""
    rng = np.random.default_rng(3)
    users, items, f = 64, 9000, 64
    rows, cols, vals = [], [], []
    for u, n in enumerate([8000, 3073, 3072, 4100] + [40] * 60):
        c = rng.choice(items, n, replace=False)
        rows += [u] * n
        cols += c.tolist()
        vals += (1 + 4 * rng.random(n)).tolist()
    Cui = sp.csr_matrix((np.array(vals, dtype=np.float32), (rows, cols)), shape=(users, items))
    Y = (rng.standard_normal((items, f)) * 0.1).astype(np.float32)
    X = np.zeros((users, f), dtype=np.float32)
    exp = X.copy()
    orc.least_squares(Cui, exp, Y, 0.05)
    got = _gpu_half(lib, ctx, Cui, X, Y, 0.05, use_cg=False)
    e = row_err(got, exp)
    print("giant rows:", e[:4], "rest max", e[4:].max())
    assert e.max() < CHOL_MAX


def test_cholesky_explicit_zeros_and_duplicates(lib, ctx, orc):
    """SURVEY.md 8(a) notes (i),(ii): duplicates are NOT merged, a stored 0.0 subtracts y y^T."""
    rng = np.random.default_rng(9)
    f = 32
    indptr = np.array([0, 5, 9], dtype=np.int32)
    indices = np.array([1, 1, 3, 7, 2, 0, 4, 4, 6], dtype=np.int32)  # duplicates, unsorted
    data = np.array([2.0, 3.0, 0.0, -1.5, 1.0, 4.0, 0.0, 2.5, -0.5], dtype=np.float32)
    Cui = sp.csr_matrix((data, indices, indptr), shape=(2, 8))
    Y = (rng.standard_normal((8, f)) * 0.2).astype(np.float32)
    X = np.zeros((2, f), dtype=np.float32)
    exp = X.copy()
    orc.least_squares(Cui, exp, Y, 0.5)
    got = _gpu_half(lib, ctx, Cui, X, Y, 0.5, use_cg=False)
    assert row_err(got, exp).max() < CHOL_MAX


def test_cholesky_not_positive_definite_raises(lib, ctx):
    """_als.pyx:131-138 -> ValueError naming the row."""
    Cui = sp.csr_matrix(np.array([[0.0, 0.0], [1.0, 0.0]], dtype=np.float32))
    Cui = sp.csr_matrix((np.array([1.0], dtype=np.float32), np.array([0], dtype=np.int32), np.array([0, 0, 1], dtype=np.int32)), shape=(2, 2))
    Y = np.zeros((2, 16), dtype=np.float32)
    X = np.zeros((2, 16), dtype=np.float32)
    with pytest.raises(ValueError, match="row 1"):
        _gpu_half(lib, ctx, Cui, X, Y, 0.0, use_cg=False)


# ---------------------------------------------------------------------------------------- R2 CG half
@pytest.mark.parametrize("f", [16, 32, 40, 64, 100, 128])
def test_cg_half_matches_oracle(lib, ctx, orc, f):
    Cui, X, Y = _case(700, 450, 12000, f, seed=200 + f, neg=0.05, orc=orc)
    exp = X.copy()
    orc.least_squares_cg(Cui, exp, Y, 0.01, cg_steps=3)
    got = _gpu_half(lib, ctx, Cui, X, Y, 0.01, use_cg=True)
    e = row_err(got, exp)
    print(f"cg f={f}: max {e.max():.2e} median {np.median(e):.2e}")
    assert e.max() < 1e-4 and np.median(e) < 1e-5


@pytest.mark.parametrize("name", [n for n in golden_cases() if n.startswith("cg")])
def test_cg_half_matches_golden(lib, ctx, name):
    rc, Cui, _, _, z = load_golden(name)
    got = _gpu_half(lib, ctx, Cui, z["X"], z["Y"], 0.01, use_cg=True)
    assert row_err(got, z["Xh"]).max() < 1e-4


def test_cg_giant_and_empty_rows(lib, ctx, orc):
    rng = np.random.default_rng(4)
    users, items, f = 40, 9000, 128
    rows, cols, vals = [], [], []
    for u, n in enumerate([9000, 3100, 0, 17] + [60] * 36):
        c = rng.choice(items, n, replace=False)
        rows += [u] * n
        cols += c.tolist()
        vals += (1 + 4 * rng.random(n)).tolist()
    Cui = sp.csr_matrix((np.array(vals, dtype=np.float32), (rows, cols)), shape=(users, items))
    Y = (rng.standard_normal((items, f)) * 0.1).astype(np.float32)
    X = (rng.standard_normal((users, f)) * 0.1).astype(np.float32)
    exp = X.copy()
    orc.least_squares_cg(Cui, exp, Y, 0.05, cg_steps=3)
    got = _gpu_half(lib, ctx, Cui, X, Y, 0.05, use_cg=True)
    assert np.all(got[2] == 0)
    e = row_err(got, exp)
    print("cg giant:", e[:4], "rest", e[4:].max())
    assert e.max() < 1e-4


def test_cg_steps_zero_and_many(lib, ctx, orc):
    Cui, X, Y = _case(300, 200, 4000, 32, seed=31, orc=orc)
    for steps in (0, 1, 8):
        exp = X.copy()
        orc.least_squares_cg(Cui, exp, Y, 0.01, cg_steps=steps)
        got = _gpu_half(lib, ctx, Cui, X, Y, 0.01, use_cg=True, cg_steps=steps)
        assert row_err(got, exp).max() < 2e-4, steps


# ---------------------------------------------------------------------------------------- R6 loss
@pytest.mark.parametrize("f", [16, 64, 128])
def test_loss_matches_oracle(lib, ctx, orc, f):
    Cui, X, Y = _case(500, 350, 8000, f, seed=300 + f, neg=0.1, orc=orc)
    C = lib.DeviceCSR.upload(ctx, Cui)
    dX, dY = lib.DeviceFactors.from_host(ctx, X), lib.DeviceFactors.from_host(ctx, Y)
    got = lib.calculate_loss(ctx, C, dX, dY, 0.01)
    assert got == pytest.approx(orc.calculate_loss(Cui, X, Y, 0.01), rel=1e-5)


def test_loss_known_answers(lib, ctx):
    """tests/als_test.py:304-324"""
    ratings = sp.coo_matrix(([1.0], ([0], [0])), shape=(1, 2)).tocsr()
    C = lib.DeviceCSR.upload(ctx, ratings)
    dY = lib.DeviceFactors.from_host(ctx, np.array([[0.0], [1.0]], dtype="float32"))
    dX = lib.DeviceFactors.from_host(ctx, np.array([[1.0]], dtype="float32"))
    assert lib.calculate_loss(ctx, C, dX, dY, 0) == pytest.approx(1.0)
    assert lib.calculate_loss(ctx, C, dX, dY, 1.0) == pytest.approx(2.0)


# ---------------------------------------------------------------------------------------- N3 transpose
def test_device_transpose_is_exactly_scipy(lib, ctx):
    Cui = synthetic.power_law_csr(3000, 1700, 60000, 55, 0.05)
    C = lib.DeviceCSR.upload(ctx, Cui)
    T = C.transpose().download()
    exp = Cui.T.tocsr()
    np.testing.assert_array_equal(T.indptr, exp.indptr)
    np.testing.assert_array_equal(T.indices, exp.indices)
    np.testing.assert_array_equal(T.data, exp.data)


# ---------------------------------------------------------------------------------------- R5 fit
@pytest.mark.parametrize("name", golden_cases())
def test_fit_matches_golden(name):
    from implicit_b200 import AlternatingLeastSquares

    rc, Cui, X0, Y0, z = load_golden(name)
    m = AlternatingLeastSquares(factors=rc["factors"], regularization=0.01, use_cg=rc["use_cg"],
                                iterations=rc["iterations"], calculate_training_loss=True)
    m.user_factors, m.item_factors = X0, Y0
    losses = []
    m.fit(Cui, show_progress=False, callback=lambda it, t, loss: losses.append(loss))
    e = np.concatenate([row_err(m.user_factors, z["X"]), row_err(m.item_factors, z["Y"])])
    print(name, f"max {e.max():.2e} median {np.median(e):.2e} loss {losses[-1]} vs {float(z['loss'])}")
    assert len(losses) == rc["iterations"]
    if rc["use_cg"]:
        assert losses[-1] == pytest.approx(float(z["loss"]), rel=2e-3)
        assert np.median(e) < 1e-2
    else:
        assert e.max() < CHOL_MAX
        assert losses[-1] == pytest.approx(float(z["loss"]), rel=1e-5)


def test_fit_c1_matches_oracle_cholesky_and_cg(orc):
    """BASELINE.json configs[0]: 10k x 5k, 50k nnz, factors=16, 3 iterations."""
    from implicit_b200 import AlternatingLeastSquares

    Cui, X0, Y0, cfg = synthetic.config("C1")
    for use_cg in (False, True):
        Xe, Ye = X0.copy(), Y0.copy()
        oracle.fit(Cui, Xe, Ye, iterations=3, use_cg=use_cg, kind=orc.name)
        m = AlternatingLeastSquares(factors=16, use_cg=use_cg, iterations=3)
        m.user_factors, m.item_factors = X0.copy(), Y0.copy()
        m.fit(Cui, show_progress=False)
        e = np.concatenate([row_err(m.user_factors, Xe), row_err(m.item_factors, Ye)])
        print("C1", "cg" if use_cg else "chol", f"max {e.max():.2e} median {np.median(e):.2e} p99 {np.percentile(e, 99):.2e}")
        if use_cg:
            assert np.median(e) < 1e-4 and np.percentile(e, 99) < 2e-3
        else:
            assert e.max() < CHOL_MAX


def test_fit_alpha_and_dtype(orc):
    """alpha scaling happens on device (cpu/als.py:133-134); float64 input is cast (:129-130)."""
    from implicit_b200 import AlternatingLeastSquares

    Cui, X0, Y0 = _case(300, 200, 3000, 32, seed=41, warm=False)
    Xe, Ye = X0.copy(), Y0.copy()
    oracle.fit(Cui, Xe, Ye, iterations=2, use_cg=False, alpha=2.5, kind=orc.name)
    m = AlternatingLeastSquares(factors=32, use_cg=False, iterations=2, alpha=2.5)
    m.user_factors, m.item_factors = X0.copy(), Y0.copy()
    m.fit(Cui.astype(np.float64), show_progress=False)
    assert max(row_err(m.user_factors, Xe).max(), row_err(m.item_factors, Ye).max()) < CHOL_MAX


# ---------------------------------------------------------------------------------------- R3 top-k
def _topk_gpu(lib, ctx, items, query, k, **kw):
    di, dq = lib.DeviceFactors.from_host(ctx, items), lib.DeviceFactors.from_host(ctx, query)
    liked = kw.pop("liked", None)
    dl = lib.DeviceCSR.upload(ctx, liked) if liked is not None else None
    out = lib.topk(ctx, di, dq, k, liked=dl, **kw)
    for h in (di, dq, dl):
        if h is not None:
            h.close()
    return out


@pytest.mark.parametrize("f", [16, 64, 100, 128])
@pytest.mark.parametrize("k", [1, 10, 64, 100])
def test_topk_matches_oracle(lib, ctx, orc, f, k):
    rng = np.random.default_rng(f * 1000 + k)
    items = (rng.standard_normal((3000, f)) * 0.3).astype(np.float32)
    query = (rng.standard_normal((150, f)) * 0.3).astype(np.float32)
    liked = synthetic.power_law_csr(150, 3000, 2500, 8)
    filt = np.array([0, 5, 17, 2999])
    ids, sc = _topk_gpu(lib, ctx, items, query, k, liked=liked, filter_items=filt)
    eids, esc = orc.topk(items, query, k, filter_query_items=liked, filter_items=filt)
    np.testing.assert_allclose(sc, esc, rtol=1e-5, atol=1e-6)  # tests/gpu_test.py:49-51 uses rtol=1e-6 on its data
    diff = ids != eids
    # indices must be identical except where two candidates tie to within fp32 summation-order noise
    assert diff.mean() < 0.01
    if diff.any():
        assert np.abs(sc[diff] - esc[diff]).max() < 1e-5
    assert not np.isin(ids, filt).any()


def test_topk_exact_ties_follow_select_h(lib, ctx, orc):
    """Integer-valued factors give exact ties: ids must be bit-identical to select.h's heap semantics."""
    rng = np.random.default_rng(5)
    items = rng.integers(0, 4, size=(700, 16)).astype(np.float32)
    items[:, 3:] = 0
    q = rng.integers(0, 3, size=(40, 16)).astype(np.float32)
    q[:, 3:] = 0
    for k in (1, 5, 32, 64, 100, 700, 1000):
        a = orc.topk(items, q, k)
        b = _topk_gpu(lib, ctx, items, q, k)
        np.testing.assert_array_equal(a[0], b[0], err_msg=f"k={k}")
        np.testing.assert_array_equal(a[1], b[1], err_msg=f"k={k}")


def test_topk_norms_and_zero_tail(lib, ctx, orc):
    rng = np.random.default_rng(6)
    items = (rng.standard_normal((50, 32))).astype(np.float32)
    q = (rng.standard_normal((7, 32))).astype(np.float32)
    norms = np.linalg.norm(items, axis=1).astype(np.float32)
    a = orc.topk(items, q, 60, item_norms=norms)
    b = _topk_gpu(lib, ctx, items, q, 60, item_norms=norms)
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_allclose(a[1], b[1], rtol=1e-5, atol=1e-6)
    assert np.all(b[0][:, 50:] == 0) and np.all(b[1][:, 50:] == 0)  # topk.pyx:20-21


def test_topk_query_rows(lib, ctx, orc):
    rng = np.random.default_rng(7)
    items = rng.standard_normal((500, 64)).astype(np.float32)
    users = rng.standard_normal((300, 64)).astype(np.float32)
    rows = np.array([5, 299, 0, 17, 5])
    di, dq = lib.DeviceFactors.from_host(ctx, items), lib.DeviceFactors.from_host(ctx, users)
    ids, sc = lib.topk(ctx, di, dq, 10, query_rows=rows)
    eids, esc = orc.topk(items, users[rows], 10)
    np.testing.assert_array_equal(ids, eids)
    np.testing.assert_allclose(sc, esc, rtol=1e-5)


# ---------------------------------------------------------------------------------------- full size, sampled
def test_c2_full_size_sampled_rows_match_oracle(lib, ctx, orc):
    """BASELINE.json configs[1] at FULL size (360k x 300k, 17M nnz, f=64, Cholesky): one user half on the GPU;
    a fixed sample of rows -- including the longest ones, which take the split path -- is re-solved by the
    oracle on the sub-CSR of just those rows (each row's solve depends only on its own nonzeros and Y)."""
    Cui, X0, Y0, cfg = synthetic.config("C2")
    lens = np.diff(Cui.indptr)
    rng = np.random.default_rng(0)
    sample = np.unique(np.concatenate([np.argsort(-lens)[:8], rng.choice(cfg["users"], 400, replace=False),
                                       np.where(lens == 0)[0][:2]]))
    got = _gpu_half(lib, ctx, Cui, X0, Y0, 0.01, use_cg=False)
    sub = Cui[sample]
    # (1) solver parity on IDENTICAL inputs: the reference's _least_squares (implicit/cpu/_als.pyx:76) is given
    #     the Gramian the GPU computed, so only the per-row accumulate + Cholesky differ.
    dY = lib.DeviceFactors.from_host(ctx, Y0)
    G_gpu = lib.gramian(ctx, dY)
    dY.close()
    exp_same = np.zeros((len(sample), 64), dtype=np.float32)
    orc._least_squares(G_gpu, sub.indptr, sub.indices, sub.data.astype("float32"), exp_same, Y0, 0.01)
    e_same = row_err(got[sample], exp_same)
    # (2) the reference end to end: its own np.dot(Y.T, Y) is an fp32 sgemm over 300k all-positive rows whose
    #     rounding noise (reported below against fp64) is amplified by the cold-start conditioning.
    exp = np.zeros((len(sample), 64), dtype=np.float32)
    orc.least_squares(sub, exp, Y0, 0.01)
    e = row_err(got[sample], exp)
    G64 = Y0.astype(np.float64).T @ Y0.astype(np.float64)
    g_gpu = np.abs(G_gpu - G64).max() / np.abs(G64).max()
    g_ref = np.abs(np.dot(Y0.T, Y0) - G64).max() / np.abs(G64).max()
    print(f"C2 sampled rows, same Gramian: max {e_same.max():.2e} median {np.median(e_same):.2e}; "
          f"reference end to end: max {e.max():.2e} median {np.median(e):.2e}; "
          f"Gramian rel err vs fp64: gpu {g_gpu:.1e} reference sgemm {g_ref:.1e}; longest row {lens.max()}")
    # (3) ground truth in fp64 for the sampled rows: at this cold start the normal equations have condition
    #     number ~2e2 (Y^T Y of all-positive factors is rank-1 dominated), so fp32 LAPACK itself is ~1e-4 off
    #     on the worst rows; the GPU result must be no further from the truth than the reference is.
    truth = cholesky_truth(sub, Y0, 0.01, YtY=G64)
    e_gpu_truth, e_ref_truth = row_err(got[sample], truth), row_err(exp, truth)
    print(f"vs fp64 truth: gpu max {e_gpu_truth.max():.2e} median {np.median(e_gpu_truth):.2e}; "
          f"reference max {e_ref_truth.max():.2e} median {np.median(e_ref_truth):.2e}")
    assert np.median(e_same) < 1e-5 and e_same.max() < 5e-4
    assert e.max() < 1e-3 and np.median(e) < 1e-4
    assert e_gpu_truth.max() < max(CHOL_MAX, 1.5 * e_ref_truth.max())
    assert np.median(e_gpu_truth) < max(1e-5, 1.5 * np.median(e_ref_truth))
    assert g_gpu < 1e-6
    assert not np.isnan(got).any()


# ---------------------------------------------------------------------------------------- multi-GPU entry points on one GPU
def test_shard_gramian_pregram_and_slices_match_plain_path(lib, ctx, orc):
    """als_gramian_shard + als_least_squares*_pregram (the multi-GPU half) on a single rank, over two row
    slices of the CSR, must reproduce the plain half; a slice view downloads as the rows it covers."""
    Cui, X, Y = _case(900, 500, 15000, 64, seed=77, orc=orc)
    for use_cg in (False, True):
        exp = _gpu_half(lib, ctx, Cui, X, Y, 0.01, use_cg=use_cg)
        C = lib.DeviceCSR.upload(ctx, Cui)
        dX, dY = lib.DeviceFactors.from_host(ctx, X), lib.DeviceFactors.from_host(ctx, Y)
        lib.gramian_shard(ctx, dY, 0, 500)
        for r0, r1 in ((0, 400), (400, 900)):
            S = C.slice_rows(r0, r1)
            lib.half_pregram(ctx, S, dX, dY, 0.01, use_cg, 3)
            if r0 == 400:
                got = S.download()
                ref = Cui[400:900]
                np.testing.assert_array_equal(got.indptr, ref.indptr)
                np.testing.assert_array_equal(got.indices, ref.indices)
                np.testing.assert_array_equal(got.data, ref.data)
            S.close()
        np.testing.assert_array_equal(dX.download(), exp)


# ---------------------------------------------------------------------------------------- short-row (n x n) path
@pytest.mark.parametrize("f", [32, 40, 64])
def test_cholesky_short_row_classes_and_deferrals(lib, ctx, orc, f):
    """cholesky_short.cu: rows at every class boundary (1, 15, 16, 17, 31, 32, 33, 47, 48, 49 nonzeros ...), an
    empty row, rows the path must hand back (|c| < 1, an explicit zero, a negative confidence below 1 in size)
    and rows it keeps (negative confidences of size >= 1, c == 1 exactly), against the oracle."""
    rng = np.random.default_rng(1000 + f)
    items = 4000
    lengths = [0, 1, 2, 7, 8, 9, 15, 16, 17, 24, 31, 32, 33, 40, 47, 48, 49, 63, 64, 65, 100] * 40
    rows, cols, vals = [], [], []
    for u, n in enumerate(lengths):
        c = rng.choice(items, n, replace=False)
        v = 1 + 4 * rng.random(n)
        kind = u % 7
        if n and kind == 1:
            v[0] = 0.5          # weight |c| - 1 < 0: deferred to the full-size kernel
        elif n and kind == 2:
            v[0] = 0.0          # explicit zero: subtracts y y^T, deferred
        elif n and kind == 3:
            v[: n // 2 + 1] *= -1  # disliked with confidence >= 1: stays on the short path
        elif n and kind == 4:
            v[0] = 1.0          # weight exactly 0
        elif n and kind == 5:
            v[0] = -0.25        # deferred
        rows += [u] * n
        cols += c.tolist()
        vals += v.tolist()
    users = len(lengths)
    Cui = sp.csr_matrix((np.array(vals, dtype=np.float32), (rows, cols)), shape=(users, items))
    assert (Cui.data == 0).sum() > 0  # the explicit zeros are stored
    Y = (rng.standard_normal((items, f)) * 0.2).astype(np.float32)
    X = np.zeros((users, f), dtype=np.float32)
    exp = X.copy()
    orc.least_squares(Cui, exp, Y, 0.05)
    got = _gpu_half(lib, ctx, Cui, X, Y, 0.05, use_cg=False)
    e = row_err(got, exp)
    lens = np.diff(Cui.indptr)
    print(f"f={f}: max {e.max():.2e}; by class <=16 {e[lens <= 16].max():.2e}, <=32 {e[(lens > 16) & (lens <= 32)].max():.2e}, "
          f"<=48 {e[(lens > 32) & (lens <= 48)].max():.2e}, longer {e[lens > 48].max():.2e}")
    assert np.all(got[lens == 0] == 0)
    assert e.max() < CHOL_MAX
