"""Shared helpers for the test-suite: parity metric and golden-case reconstruction."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

ROOT =os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
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
    X = np.zeros((Cui.shape[0], f))
    nonempty = np.nonzero(lens)[0]
    for r0 in range(0, len(nonempty), 1024):  # blocks of rows: A stays small at 128 factors and many rows
        rows = nonempty[r0:r0 + 1024]
        A = np.empty((len(rows), f, f))
        b = np.empty((len(rows), f))
        for n, u in enumerate(rows):
            s, e = Cui.indptr[u], Cui.indptr[u + 1]
            Yu, c = Y64[Cui.indices[s:e]], np.asarray(Cui.data[s:e], dtype=np.float64)
            A[n] = G + (Yu.T * (np.abs(c) - 1.0)) @ Yu
            b[n] = Yu.T @ np.maximum(c, 0.0)
        X[rows] = np.linalg.solve(A, b[:, :, None])[:, :, 0]
    return X


#: every knob of als_ctx_set_knob and its default (include/als_b200.h, csrc/common.h)
KNOB_DEFAULTS = dict(short_max=48, short_serial=0, whiten_fma=0, gramian_fma=0, topk_legacy=0,
                     long_tc=0, cg_nv=2)


# ----------------------------------------------------------------------------- fixtures of the kernel-path modules
# A GPU module that compares kernel paths imports these by name: one context per module, every knob at its default
# before and after each test, and a failure at once when a knob is set in the environment.
@pytest.fixture(scope="module")
def lib():
    set_in_env = sorted(f"ALS_B200_{k.upper()}" for k in KNOB_DEFAULTS if f"ALS_B200_{k.upper()}" in os.environ)
    if set_in_env:  # a "default path" test would silently run another path
        pytest.fail(f"knob environment variables are set: {', '.join(set_in_env)}; unset them to run these tests")
    from implicit_b200 import _lib

    return _lib


@pytest.fixture(scope="module")
def ctx(lib):
    c = lib.Context(0)
    yield c
    c.close()


@pytest.fixture(autouse=True)
def default_knobs(ctx):
    """Every test starts and ends with every knob at its default."""
    for k, v in KNOB_DEFAULTS.items():
        ctx.set_knob(k, v)
    yield
    for k, v in KNOB_DEFAULTS.items():
        ctx.set_knob(k, v)


@pytest.fixture(scope="module")
def orc():
    import oracle

    return oracle.get("auto")


@pytest.fixture(scope="module")
def sm(ctx):
    return ctx.info()["sm_count"]


def factors_of(kind, rows, f, seed):
    rng = np.random.default_rng(seed)
    if kind == "mixed":
        return rng.standard_normal((rows, f), dtype=np.float32)
    if kind == "cold":  # the all-positive initialisation (implicit/cpu/als.py:144-147)
        return rng.random((rows, f), dtype=np.float32) * np.float32(0.01)
    if kind == "decades":  # row norms spread over six decades
        Y = rng.standard_normal((rows, f), dtype=np.float32)
        return (Y * (10.0 ** rng.uniform(-6, 0, size=(rows, 1)))).astype(np.float32)
    if kind == "zero_rows":
        Y = rng.standard_normal((rows, f), dtype=np.float32)
        Y[rng.random(rows) < 0.3] = 0
        Y[-1] = 0
        return Y
    raise ValueError(kind)


def worst_ratio(err, bar):
    """max(err / bar); entries with bar == 0 must have err == 0."""
    err, bar = np.asarray(err, np.float64), np.asarray(bar, np.float64)
    if np.any((bar == 0) & (err != 0)):
        return np.inf
    return float(np.max(np.where(bar > 0, err / np.where(bar > 0, bar, 1), 0.0), initial=0.0))


def mixed_csr(users, items, seed, giants=(3073, 3500, 4100), duplicates=False):
    """Rows at every short-row class boundary, giant rows past the split threshold (> 3072; rows 3, 50, 97, ...
    get the lengths `giants`, sampled with repeats where a length exceeds `items`), negative confidences, weights
    |c| - 1 below zero and stored zeros.  duplicates=True repeats the first column of every ninth row at its end."""
    rng = np.random.default_rng(seed)
    lengths = [0, 1, 8, 9, 15, 16, 17, 24, 25, 31, 32, 33, 40, 41, 47, 48, 49, 64, 65, 200]
    lens = [lengths[u % len(lengths)] for u in range(users)]
    for i, n in enumerate(giants):
        lens[3 + 47 * i] = n
    rows, cols, vals = [], [], []
    for u, n in enumerate(lens):
        c = rng.choice(items, n, replace=n > items)
        v = 1 + 4 * rng.random(n)
        kind = u % 9
        if n and kind == 1:
            v[0] = 0.5      # weight below zero
        elif n and kind == 2:
            v[0] = 0.0      # stored zero
        elif n and kind == 3:
            v[: n // 2 + 1] *= -1
        elif n and kind == 4:
            v[0] = -0.25
        rows += [u] * n
        cols += c.tolist()
        vals += v.tolist()
    if not duplicates:
        Cui = sp.csr_matrix((np.array(vals, dtype=np.float32), (rows, cols)), shape=(users, items))
    else:  # built from indptr so that nothing merges the repeats
        indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        for u in range(5, users, 9):
            if lens[u] >= 2:
                cols[indptr[u + 1] - 1] = cols[indptr[u]]
        Cui = sp.csr_matrix((np.array(vals, dtype=np.float32), np.array(cols, dtype=np.int32), indptr),
                            shape=(users, items))
    assert (Cui.data == 0).sum() > 0
    return Cui


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
