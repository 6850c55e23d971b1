"""Shared helpers for the test-suite: parity metric and golden-case reconstruction."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from implicit_b200 import synthetic  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

#: Parity bars (north_star: rtol=1e-4 fp32 per factor row).  Row error = ||a - b||_2 / max(||b||_2, 1% of the
#: median row norm): elementwise rtol is unsatisfiable even by the reference against itself (SURVEY.md 8(c)).
CHOL_MAX = 1e-4
#: Truncated CG(3) amplifies rounding: the reference's own fp32 vs fp64 runs differ by up to 7e-4 on
#: iteration 1 (SURVEY.md 8(c)), so a half-iteration is gated on median / p99 and max only on a
#: converged fit.
CG_MEDIAN = 5e-5
CG_P99 = 1e-3
CG_CONVERGED_MAX = 1e-4


def row_err(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    num = np.linalg.norm(a - b, axis=1)
    den = np.linalg.norm(b, axis=1)
    floor = 0.01 * np.median(den) if len(den) else 0.0
    return num / np.maximum(np.maximum(den, floor), 1e-30)


def cholesky_truth(Cui, Y, reg, YtY=None):
    """The Cholesky half in fp64: for every row u, x_u = (G + reg I + Y_u^T diag(|c| - 1) Y_u)^-1 Y_u^T c+ with
    G = YtY (the caller's, cast to fp64) or the fp64 Y^T Y.  Every stored entry counts like _als.pyx:96-130: an
    explicit zero subtracts y y^T, duplicates are not merged.  Empty rows are zero (_als.pyx:98-100)."""
    Y64 = np.asarray(Y, dtype=np.float64)
    f = Y64.shape[1]
    G = Y64.T @ Y64 if YtY is None else np.asarray(YtY, dtype=np.float64)
    G = G + reg * np.eye(f)
    lens = np.diff(Cui.indptr)
    rows = np.nonzero(lens)[0]
    A = np.empty((len(rows), f, f))
    b = np.empty((len(rows), f))
    for n, u in enumerate(rows):
        s, e = Cui.indptr[u], Cui.indptr[u + 1]
        Yu, c = Y64[Cui.indices[s:e]], np.asarray(Cui.data[s:e], dtype=np.float64)
        A[n] = G + (Yu.T * (np.abs(c) - 1.0)) @ Yu
        b[n] = Yu.T @ np.maximum(c, 0.0)
    X = np.zeros((Cui.shape[0], f))
    if len(rows):
        X[rows] = np.linalg.solve(A, b[:, :, None])[:, :, 0]
    return X


def topk_noise(queries, items):
    """Per-row fp32 summation noise of a score q . i: 4 eps |q| max_i |i|, as an (n, 1) column.  The query side is
    per row (a kernel must hold its accuracy however small a query is next to the others); the item side is the
    largest item, because every item of a row competes for the same k slots."""
    q = np.linalg.norm(np.asarray(queries, dtype=np.float64), axis=1)[:, None]
    return 4 * np.finfo(np.float32).eps * q * np.linalg.norm(np.asarray(items, dtype=np.float64), axis=1).max()


def topk_mismatches(ids, scores, ref_ids, ref_scores, noise):
    """Near-tie classification of two top-k results (SURVEY.md section 8(d)): where the ids at a rank differ, the
    two scores at that rank must agree within `noise` (a scalar or an (n, 1) column from topk_noise).
    Returns (same, bad): the boolean arrays of equal ids and of true mismatches."""
    same = ids == ref_ids
    bad = (~same) & (np.abs(np.asarray(scores, np.float64) - np.asarray(ref_scores, np.float64)) > noise)
    return same, bad


def golden_cases():
    """The fit fixtures (chol_*, cg_*); eval_metrics.npz belongs to tests/test_evaluation.py."""
    return sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz") and f.startswith(("chol_", "cg_")))


def load_golden(name):
    """Returns (recipe dict, Cui, X0, Y0, expected npz dict)."""
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    rc = {k[len("recipe_"):]: z[k].item() for k in z.files if k.startswith("recipe_")}
    Cui = synthetic.power_law_csr(rc["users"], rc["items"], rc["nnz"], rc["seed"], rc["neg"])
    X0, Y0 = synthetic.initial_factors(rc["users"], rc["items"], rc["factors"], seed=42)
    return rc, Cui, X0, Y0, z


# ----------------------------------------------------------------------------- evaluation fixtures
class TableModel:
    """Stands in for a fitted model: `recommend` returns precomputed ranked ids (no GPU involved)."""

    def __init__(self, table):
        self.table = table

    def recommend(self, userid, user_items, N=10, **kwargs):
        ids = self.table[np.asarray(userid)][:, :N]
        return ids, np.zeros(ids.shape, dtype=np.float32)


def eval_case(users, items, K, seed):
    """Seeded (model, train, test): a random ranking per user, a test CSR with duplicates and empty rows."""
    import scipy.sparse as sp

    rng = np.random.default_rng(seed)
    table = np.argsort(rng.random((users, items)), axis=1)[:, :max(K, 1)].astype(np.int32)
    n = rng.integers(0, min(items, 2 * K) + 1, size=users)
    n[rng.random(users) < 0.2] = 0  # users without withheld items are skipped (evaluation.pyx:421-422)
    indptr = np.concatenate([[0], np.cumsum(n)]).astype(np.int32)
    indices = rng.integers(0, items, size=int(indptr[-1])).astype(np.int32)  # duplicates on purpose
    test = sp.csr_matrix((np.ones(len(indices), dtype=np.float32), indices, indptr), shape=(users, items))
    train = sp.random(users, items, density=0.05, format="csr", dtype=np.float32, random_state=seed)
    return TableModel(table), train, test
