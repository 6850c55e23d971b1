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


def _nnz_dots(Y64, V, indices, owner, out=None):
    """d_k = y_k . v_owner(k) for every stored entry, in blocks of ~4M products (bounded memory at 1024 factors)."""
    d = np.empty(len(indices)) if out is None else out
    block = max(1, (1 << 22) // max(1, Y64.shape[1]))
    for k0 in range(0, len(indices), block):
        k1 = min(len(indices), k0 + block)
        d[k0:k1] = np.einsum("kf,kf->k", Y64[indices[k0:k1]], V[owner[k0:k1]])
    return d


def _csr_parts64(Cui, r0=0, r1=None):
    """(indptr rebased to 0, indices, data as fp64, owner row of every entry) of rows [r0, r1), duplicates kept."""
    r1 = Cui.shape[0] if r1 is None else r1
    indptr = np.asarray(Cui.indptr[r0:r1 + 1], dtype=np.int64)
    s, e = int(indptr[0]), int(indptr[-1])
    indptr = indptr - s
    owner = np.repeat(np.arange(r1 - r0), np.diff(indptr))
    return indptr, np.asarray(Cui.indices[s:e]), np.asarray(Cui.data[s:e], dtype=np.float64), owner


def _rows_times_Y(coef, indices, indptr, Y64):
    """sum_k coef_k y_k per row: the sparse matrix (coef, indices, indptr) times Y (duplicates add, as in the loop)."""
    M = sp.csr_matrix((coef, indices, indptr), shape=(len(indptr) - 1, Y64.shape[0]))
    return np.asarray(M @ Y64)


def cg_truth(Cui, X0, Y, reg, cg_steps, YtY=None):
    """The CG half in fp64: _least_squares_cg (_als.pyx:154-248, oracle_least_squares_cg) with the same recurrences
    and the same 1e-20 thresholds on rsold (skip the row, x unchanged) and rsnew (stop after that step), vectorised
    over rows.  A = G + reg I with G = YtY (the caller's, cast to fp64) or the fp64 Y^T Y.  Every stored entry counts:
    a stored zero weighs |c| - 1 = -1, duplicates are not merged.  Empty rows are zero (:182-184).
    Returns (X, rs0, stop, rs_last): rs0 the initial r.r of every row (0 for empty rows), stop the number of CG steps
    applied to the row (0 for empty rows and rows skipped on rsold), rs_last its r.r after the last of those steps
    (rs0 where none ran), so that rows which broke on rsnew are those with rs_last < 1e-20."""
    Y64 = np.asarray(Y, dtype=np.float64)
    n, f = Cui.shape[0], Y64.shape[1]
    A = (Y64.T @ Y64 if YtY is None else np.asarray(YtY, dtype=np.float64)) + reg * np.eye(f)
    indptr, indices, c, owner = _csr_parts64(Cui)
    w, pos = np.abs(c) - 1.0, np.maximum(c, 0.0)
    nonempty = np.diff(indptr) > 0
    X = np.array(X0, dtype=np.float64)
    X[~nonempty] = 0.0
    # r = b - A x = sum_k (c_k^+ - (|c_k| - 1) y_k.x) y_k - (G + reg I) x          (:187-201)
    r = _rows_times_Y(pos - w * _nnz_dots(Y64, X, indices, owner), indices, indptr, Y64) - X @ A
    r[~nonempty] = 0.0
    p = r.copy()
    rsold = np.einsum("uf,uf->u", r, r)
    rs0, rs_last = rsold.copy(), rsold.copy()
    stop = np.zeros(n, dtype=np.int64)
    active = nonempty & (rsold >= 1e-20)  # :206-207
    for s in range(cg_steps):
        rows = np.nonzero(active)[0]
        if not len(rows):
            break
        # Ap = (G + reg I) p + sum_k (|c_k| - 1) (y_k.p) y_k                           (:212-222)
        Ap = p @ A + _rows_times_Y(w * _nnz_dots(Y64, p, indices, owner), indices, indptr, Y64)
        alpha = rsold[rows] / np.einsum("uf,uf->u", p[rows], Ap[rows])   # :225
        X[rows] += alpha[:, None] * p[rows]                               # :228
        r[rows] -= alpha[:, None] * Ap[rows]                              # :231-232
        rsnew = np.einsum("uf,uf->u", r[rows], r[rows])                   # :234
        stop[rows], rs_last[rows] = s + 1, rsnew
        go = rsnew >= 1e-20                                               # :235-236
        active[rows[~go]] = False
        rows, rsnew = rows[go], rsnew[go]
        p[rows] = r[rows] + (rsnew / rsold[rows])[:, None] * p[rows]     # :239-242
        p[~active] = 0.0  # stopped rows take no further part
        rsold[rows] = rsnew
    return X, rs0, stop, rs_last


def loss_truth(Cui, X, Y, reg, rows=None):
    """The training loss in fp64 the way _calculate_loss computes it (_als.pyx:259-308, oracle_calculate_loss), row
    by row: r = Y^T Y x_u + sum_k ((c_k > 0 ? -2 c_k : 0) + (|c_k| - 1) y_k.x_u) y_k, loss += r.x_u + sum_k |c_k| --
    not through the expansion <Y^T Y, X^T X>_F + sum_k (...) that the device uses.
    rows = (r0, r1) restricts the sums over users to those rows of Cui and X (a shard).
    Returns (loss, terms, scale): terms are those of als_calculate_loss for the rows, [0] = sum_u (r.x_u + sum_k |c_k|)
    + reg sum_u |x_u|^2, [1] = sum_k |c_k|, [2] = reg |Y|^2; loss = (terms[0] + terms[2]) / (terms[1] + U I - nnz)
    with U and nnz of the rows (the loss of Cui for the whole range).  scale holds the same sums with every product
    replaced by the product of absolute values: the size of the rounding an fp32 evaluation of each term can carry."""
    r0, r1 = (0, Cui.shape[0]) if rows is None else rows
    Y64 = np.asarray(Y, dtype=np.float64)
    Xr = np.asarray(X, dtype=np.float64)[r0:r1]
    indptr, indices, c, owner = _csr_parts64(Cui, r0, r1)
    conf = np.abs(c)
    terms, scale = np.zeros(3), np.zeros(3)
    for k, (Yk, Xk) in enumerate(((Y64, Xr), (np.abs(Y64), np.abs(Xr)))):
        d = _nnz_dots(Yk, Xk, indices, owner)
        temp = (np.where(c > 0, -2.0 * c, 0.0) + (conf - 1.0) * d if k == 0
                else np.where(c > 0, 2.0 * c, 0.0) + np.abs(conf - 1.0) * d)
        r = Xk @ (Yk.T @ Yk) + _rows_times_Y(temp, indices, indptr, Yk)    # :282-298
        out = terms if k == 0 else scale
        out[0] = np.einsum("uf,uf->", r, Xk) + conf.sum() + reg * np.einsum("uf,uf->", Xk, Xk)  # :300-301, :307
        out[1] = conf.sum()
        out[2] = reg * np.einsum("if,if->", Yk, Yk)                         # :303-304
    den = terms[1] + float(r1 - r0) * float(Cui.shape[1]) - float(len(c))
    return (terms[0] + terms[2]) / den, terms, scale


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


def bad_row_csr(f, bad_rows, users=40):
    """With lambda = 0 and Y = I (f items), row u's normal equations are I + the e_i e_i^T of its four items (confidence
    2); a row in bad_rows also holds three stored zeros on item 0, which subtract 3 e_0 e_0^T: not positive definite."""
    rng = np.random.default_rng(1)
    cols = [list(rng.choice(f, 4, replace=False)) + [0] * 3 * (u in bad_rows) for u in range(users)]
    vals = np.concatenate([[2.0] * 4 + [0.0] * 3 * (u in bad_rows) for u in range(users)]).astype(np.float32)
    indptr = np.cumsum([0] + [len(c) for c in cols]).astype(np.int32)
    return sp.csr_matrix((vals, np.concatenate(cols).astype(np.int32), indptr), shape=(users, f))


def check_bad_row_in_second_segment(lib, ctx, host):
    """A bad row beyond the first segment of a segmented device- or host-resident CSR: the synchronous half and, after
    the asynchronous one, solver_status name it.  Leaves the segment_nnz knob set."""
    f, bad = 16, 30
    C = bad_row_csr(f, [bad])
    ctx.set_knob("segment_nnz", C.nnz // 3 + 1)
    d = lib.DeviceCSR.upload(ctx, C, host=host)
    assert d.host_resident == host and d.segment_count > 1
    assert C.indptr[bad] > C.nnz // 3 + 1  # the bad row lies beyond the first segment
    Yd, X = lib.DeviceFactors.from_host(ctx, np.eye(f, dtype=np.float32)), lib.DeviceFactors(ctx, C.shape[0], f)
    with pytest.raises(ValueError, match=f"row {bad}\\b"):
        lib.least_squares(ctx, d, X, Yd, 0.0)
    lib.gramian(ctx, Yd)
    lib.half_pregram_async(ctx, d, X, Yd, 0.0, use_cg=False)
    with pytest.raises(ValueError, match=f"row {bad}\\b"):
        lib.solver_status(ctx)
    for h in (d, Yd, X):
        h.close()


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


def select_h(scores, k):
    """The top-k that select.h's heap (implicit/cpu/select.h:12-39) leaves, restated without the heap, for rows of
    scores of any float type.  With kk = min(k, I), T the kk-th largest score of a row and g the number of items
    above T: every item above T is kept, and the m = kk - g items with the largest columns <= c* among those scoring
    exactly T, where c* is the column of the kk-th item scoring >= T in column order.  Output descending by score,
    equal scores larger column first; ids and scores are zero past kk (topk.pyx:20-21)."""
    S = np.atleast_2d(np.asarray(scores))
    n, I = S.shape
    kk = min(k, I)
    ids = np.zeros((n, k), dtype=np.int32)
    out = np.zeros((n, k), dtype=S.dtype)
    if kk == 0:
        return ids, out
    for r in range(n):
        s = S[r]
        T = np.partition(s, I - kk)[I - kk]
        above = np.flatnonzero(s > T)
        c_star = np.flatnonzero(s >= T)[kk - 1]
        tied = np.flatnonzero(s[:c_star + 1] == T)
        sel = np.concatenate([above, tied[len(tied) - (kk - len(above)):]])
        sel = sel[np.lexsort((-sel, -s[sel]))]
        ids[r, :kk], out[r, :kk] = sel, s[sel]
    return ids, out


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
