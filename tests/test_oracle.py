"""CPU-only: pins the oracle (oracle/als_oracle.c) against
  (1) the golden vectors generated from the reference's own compiled Cython (tests/golden/),
  (2) what that compiled reference returned for direct comparisons (tests/golden/ref_checks.npz,
      tests/golden/make_golden_ref.py),
  (3) the known-answer / property tests the reference holds for this path."""
import os
import sys

import numpy as np
import pytest
from scipy.sparse import csr_matrix

import oracle
from helpers import CHOL_MAX, GOLDEN, cholesky_truth, golden_cases, load_golden, row_err

sys.path.insert(0, GOLDEN)
import make_golden_ref  # noqa: E402

PORT = oracle.get("port")
REF = np.load(os.path.join(GOLDEN, "ref_checks.npz"))


@pytest.mark.parametrize("name", golden_cases())
def test_port_matches_golden_warm_half(name):
    """One half-iteration from the stored (well conditioned) state: the tight per-half parity bar."""
    rc, Cui, _, _, z = load_golden(name)
    Xh = z["X"].copy()
    if rc["use_cg"]:
        PORT.least_squares_cg(Cui, Xh, z["Y"], 0.01, cg_steps=3)
    else:
        PORT.least_squares(Cui, Xh, z["Y"], 0.01)
    assert row_err(Xh, z["Xh"]).max() < 1e-5


@pytest.mark.parametrize("name", golden_cases())
def test_port_matches_golden_fit(name):
    rc, Cui, X, Y, z = load_golden(name)
    oracle.fit(Cui, X, Y, regularization=0.01, iterations=rc["iterations"], use_cg=rc["use_cg"], kind="port")
    e = np.concatenate([row_err(X, z["X"]), row_err(Y, z["Y"])])
    loss = PORT.calculate_loss(Cui, X, Y, 0.01)
    if rc["use_cg"]:
        # truncated CG from the near rank-1 random start is chaotic in factor space (SURVEY.md 8(c)):
        # two correct fp32 executions agree in loss, not row by row
        assert abs(loss - float(z["loss"])) / float(z["loss"]) < 2e-3
        assert np.median(e) < 1e-2
    else:
        assert e.max() < CHOL_MAX
        assert abs(loss - float(z["loss"])) / float(z["loss"]) < 1e-5


@pytest.mark.parametrize("name", golden_cases())
def test_port_loss_and_topk_match_golden(name):
    rc, Cui, _, _, z = load_golden(name)
    loss = PORT.calculate_loss(Cui, z["X"], z["Y"], 0.01)
    assert loss == pytest.approx(float(z["loss"]), rel=1e-6)
    ids, scores = PORT.topk(z["Y"], z["X"][:64], 10, filter_query_items=Cui[:64], filter_items=np.array([0, 3, 7]))
    np.testing.assert_allclose(scores, z["topk_scores"], rtol=1e-5, atol=1e-7)
    # ids may differ only where the reference's own scores tie to within rounding
    diff = ids != z["topk_ids"]
    if diff.any():
        assert np.abs(scores[diff] - z["topk_scores"][diff]).max() < 1e-6


@pytest.mark.parametrize("name", [n for n in golden_cases() if n.startswith("chol")])
def test_cholesky_truth_matches_golden_half(name):
    """tests/helpers.cholesky_truth, the fp64 yardstick of the GPU kernel tests, against the reference's own fp32 half
    (golden Xh) from the stored warm state, with its own fp64 Gramian and with a caller-supplied one (_least_squares)."""
    rc, Cui, _, _, z = load_golden(name)
    Y = z["Y"]
    truth = cholesky_truth(Cui, Y, 0.01)
    e = row_err(z["Xh"], truth)
    YtY = (Y.astype(np.float64).T @ Y.astype(np.float64) * 0.5).astype(np.float32)  # any SPD Gramian will do
    got = np.zeros_like(z["X"])
    PORT._least_squares(YtY, Cui.indptr, Cui.indices, Cui.data.astype(np.float32), got, Y, 0.01)
    e_g = row_err(got, cholesky_truth(Cui, Y, 0.01, YtY=YtY))
    print(f"{name}: fp32 reference vs cholesky_truth max {e.max():.2e}; with a supplied Gramian max {e_g.max():.2e}")
    assert e.max() < 1e-5 and e_g.max() < 1e-5


def test_cholesky_truth_counts_zeros_duplicates_and_negatives():
    """Stored zeros subtract y y^T, duplicates are not merged, negative confidences weigh |c| - 1 with no right-hand
    side, empty rows are zero: the same as the oracle's fp32 solve of _als.pyx:96-130."""
    rng = np.random.default_rng(12)
    indptr = np.array([0, 5, 9, 9, 12], dtype=np.int32)
    indices = np.array([1, 1, 3, 7, 2, 0, 4, 4, 6, 5, 2, 5], dtype=np.int32)
    data = np.array([2.0, 3.0, 0.0, -1.5, 1.0, 4.0, 0.0, 2.5, -0.5, 3.0, 0.5, 3.0], dtype=np.float32)
    Cui = csr_matrix((data, indices, indptr), shape=(4, 8))
    Y = (rng.standard_normal((8, 16)) * 0.4).astype(np.float32)
    exp = np.zeros((4, 16), dtype=np.float32)
    PORT.least_squares(Cui, exp, Y, 0.5)
    truth = cholesky_truth(Cui, Y, 0.5)
    assert np.all(truth[2] == 0)
    assert row_err(exp, truth).max() < 1e-5
    merged = Cui.copy()
    merged.sum_duplicates()
    assert row_err(cholesky_truth(merged, Y, 0.5), truth).max() > 1e-3  # merging duplicates is a different problem


@pytest.mark.parametrize("use_cg", [False, True])
def test_port_matches_compiled_reference(use_cg):
    """One half from a warm state against the reference's compiled least_squares / least_squares_cg."""
    tag = "cg" if use_cg else "chol"
    Cui, Xw, Yw = make_golden_ref.half_inputs(use_cg)
    Xb = Xw.copy()
    if use_cg:
        PORT.least_squares_cg(Cui, Xb, Yw, 0.01, cg_steps=3)
    else:
        PORT.least_squares(Cui, Xb, Yw, 0.01)
    assert row_err(Xb, REF[f"half_{tag}_Xa"]).max() < 1e-5
    assert PORT.calculate_loss(Cui, Xw, Yw, 0.01) == pytest.approx(float(REF[f"half_{tag}_loss"]), rel=1e-6)


def test_port_matches_compiled_reference_on_a_wide_model():
    """192 factors (the widths of tests/test_gpu_wide.py): the checker itself must not care about the width."""
    Cui, X, Y = make_golden_ref.wide_inputs()
    Xb = X.copy()
    PORT.least_squares_cg(Cui, Xb, Y, 0.01, cg_steps=3)
    assert row_err(Xb, REF["wide_Xa"]).max() < 1e-5
    assert PORT.calculate_loss(Cui, X, Y, 0.01) == pytest.approx(float(REF["wide_loss"]), rel=1e-6)
    ib, sb = PORT.topk(Y, REF["wide_Xa"][:20], 7, filter_query_items=Cui[:20])
    np.testing.assert_allclose(sb, REF["wide_topk_scores"], rtol=1e-5, atol=1e-7)
    assert (REF["wide_topk_ids"] == ib).mean() > 0.98


# ---- the reference's own known-answer tests for this path ------------------------------------------
@pytest.mark.parametrize("use_cg", [False, True])
def test_factorize(use_cg):
    """tests/als_test.py:142-186: X Y^T must reconstruct a 7x6 binary matrix to 1e-3."""
    counts = csr_matrix(
        [[1, 1, 0, 1, 0, 0], [0, 1, 1, 1, 0, 0], [1, 0, 1, 0, 0, 0], [1, 1, 0, 0, 0, 0], [0, 0, 1, 1, 0, 1],
         [0, 1, 0, 0, 0, 1], [0, 0, 0, 0, 1, 1]], dtype=np.float64)
    rng = np.random.default_rng(23)
    X = (rng.random((7, 6), dtype=np.float32) * 0.01).astype(np.float32)
    Y = (rng.random((6, 6), dtype=np.float32) * 0.01).astype(np.float32)
    oracle.fit(counts, X, Y, regularization=0, iterations=15, use_cg=use_cg, alpha=2.0, kind="port")
    rec = X.dot(Y.T)
    dense = counts.toarray()
    for r in range(7):
        for c in range(6):
            assert dense[r, c] == pytest.approx(rec[r, c], abs=1e-3)


def test_calculate_loss_simple():
    """tests/als_test.py:304-324: the only user liked item 0; factors are perfectly wrong -> loss 1.0 (lambda=0),
    2.0 (lambda=1)."""
    from scipy.sparse import coo_matrix

    ratings = coo_matrix(([1.0], ([0], [0])), shape=(1, 2)).tocsr()
    item_factors = np.array([[0.0], [1.0]], dtype="float32")
    user_factors = np.array([[1.0]], dtype="float32")
    assert PORT.calculate_loss(ratings, user_factors, item_factors, 0) == pytest.approx(1.0)
    assert PORT.calculate_loss(ratings, user_factors, item_factors, 1.0) == pytest.approx(2.0)


def test_empty_rows_are_zeroed():
    """_als.pyx:98-100 / :182-184"""
    Cui = csr_matrix(np.array([[0, 0, 0], [1, 0, 2], [0, 0, 0]], dtype=np.float32))
    Y = np.random.default_rng(0).random((3, 8), dtype=np.float32)
    for cg in (False, True):
        X = np.ones((3, 8), dtype=np.float32)
        (PORT.least_squares_cg if cg else PORT.least_squares)(Cui, X, Y, 0.1)
        assert np.all(X[0] == 0) and np.all(X[2] == 0) and np.any(X[1] != 0)


def test_cholesky_failure_raises():
    """_als.pyx:131-138: singular normal equations with no regularization raise ValueError."""
    Cui = csr_matrix(np.array([[1.0, 0.0]], dtype=np.float32))
    Y = np.zeros((2, 4), dtype=np.float32)
    X = np.zeros((1, 4), dtype=np.float32)
    with pytest.raises(ValueError):
        PORT.least_squares(Cui, X, Y, 0.0)


def test_select_tie_semantics():
    """implicit/cpu/select.h:12-39: strict `>` admission, evict the lexicographic (score, col) minimum,
    output descending by (score, col); rows shorter than k keep their zero tail (topk.pyx:20-21)."""
    items = np.array([[5.0], [5.0], [7.0]], dtype=np.float32)
    ids, sc = PORT.topk(items, np.array([[1.0]], dtype=np.float32), 2)
    assert ids.tolist() == [[2, 1]] and sc.tolist() == [[7.0, 5.0]]
    items = np.array([[7.0], [5.0], [5.0]], dtype=np.float32)
    ids, sc = PORT.topk(items, np.array([[1.0]], dtype=np.float32), 2)
    assert ids.tolist() == [[0, 1]]
    items = np.array([[1.0], [1.0], [1.0], [1.0]], dtype=np.float32)
    ids, _ = PORT.topk(items, np.array([[1.0]], dtype=np.float32), 3)
    assert ids.tolist() == [[2, 1, 0]]
    ids, sc = PORT.topk(items[:2], np.array([[1.0]], dtype=np.float32), 4)
    assert ids.tolist() == [[1, 0, 0, 0]] and sc.tolist() == [[1.0, 1.0, 0.0, 0.0]]


def test_select_matches_compiled_reference_on_ties():
    rng = np.random.default_rng(5)
    items = rng.integers(0, 4, size=(200, 3)).astype(np.float32)  # many exact ties
    q = rng.integers(0, 3, size=(17, 3)).astype(np.float32)
    for k in (1, 5, 32, 250):
        b = PORT.topk(items, q, k)
        np.testing.assert_array_equal(REF[f"ties_k{k}_ids"], b[0])
        np.testing.assert_array_equal(REF[f"ties_k{k}_scores"], b[1])
