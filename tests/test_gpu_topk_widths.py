"""The top-k (csrc/topk.cu, csrc/topk_tc.cu) against select.h and fp64 at every factor width, k class and grid edge.

Every case states which path topk_device dispatches it to (restated in `expected_path`) and checks that this path ran:
the mma.sync kernel topk_kernel<F, TQ> (up to 128 padded factors and k <= 1048), the wgmma kernel (64 padded factors,
k <= 16, >= 1024 queries), or scores + segmented sort (wider models and larger k), seen from the number of `topk`
launches in the profile (one per pass of the sort) and the launch count.

  * Exact ties: integer factors in -2..2 (30 % zero item rows, a few zero query rows) give scores that are exact in
    fp32 and in every kernel's split (TF32 hi / lo, fp16 hi / lo with power-of-two scales, FMA), so ids and scores
    must equal the reference's bit for bit, with and without liked lists, filter lists, item norms and query_rows.
  * fp64: the score of every returned id against its fp64 product, within a per-path error bound, and the ids against
    select.h applied to the fp64 scores away from near-ties.
  * Grid and tile edges of topk_kernel<F, TQ>, the sort in several passes, and the public model class.
"""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from helpers import factors_of, select_h, topk_mismatches, topk_noise, worst_ratio
from helpers import ctx, default_knobs, lib, orc, sm  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

U = np.finfo(np.float32).eps / 2
NEG = -np.finfo(np.float32).max  # a filtered item's score (topk.pyx:51-56)
KINDS = ["mixed", "cold", "decades", "zero_rows"]


@pytest.fixture(scope="module", autouse=True)
def profiling(ctx):
    ctx.profile(True)
    yield
    ctx.profile(False)


# ---------------------------------------------------------------------------------------- the dispatch, restated
def padded(f):
    return (f + 15) // 16 * 16 if f <= 128 else (f + 127) // 128 * 128


def tk_cfg(F, TQ):
    """TkCfg<F, TQ> of csrc/topk.cu: query rows per CTA, items per tile, CTAs per SM."""
    QB, IT = 16 * TQ, 128 if F <= 64 else 64
    alias = IT * (F + 4) >= QB * (IT + 4)
    return QB, IT, 2 if alias and F <= 64 else 1


def expected_path(f, n_query, n_items, k, norms=False, n_filter=0, liked_max=0):
    """(path, passes) of topk_device: the wgmma kernel, the mma.sync kernel at TQ = 4 or 1, or the sort."""
    ld, keff = padded(f), min(k, n_items)
    if (ld == 64 and 1 <= keff <= 16 and not norms and n_query >= 1024 and n_items >= 256
            and n_items - n_filter - liked_max >= keff):
        return "wgmma", 1
    if (keff > 64 and keff * 16 * 2 * 4 + 96 * 1024 > 227 * 1024) or ld > 128:
        rows_per_pass = max(1, min(n_query, (3 << 29) // (n_items * 24), (2 ** 31 - 1) // n_items))
        return "sort", -(-n_query // rows_per_pass)
    return ("mma.sync TQ=4" if keff <= 64 else "mma.sync TQ=1"), 1


def unsorted_rows(m):
    d = np.diff(m.indices.astype(np.int64))
    starts = np.zeros(len(m.indices), bool)
    starts[m.indptr[:-1][np.diff(m.indptr) > 0]] = True
    return bool((d < 0)[~starts[1:]].any())


def run_topk(lib, ctx, items, queries, k, liked=None, filter_items=None, item_norms=None, query_rows=None):
    """lib.topk on fresh device handles: (ids, scores, path, passes), the path as the launches show it."""
    di, dq = lib.DeviceFactors.from_host(ctx, items), lib.DeviceFactors.from_host(ctx, queries)
    dl = lib.DeviceCSR.upload(ctx, liked) if liked is not None else None
    try:
        ctx.profile_read()
        n0 = ctx.launch_count()
        ids, sc = lib.topk(ctx, di, dq, k, query_rows=query_rows, liked=dl, filter_items=filter_items,
                           item_norms=item_norms)
        n = ctx.launch_count() - n0
        passes = ctx.profile_read()["topk"][1]
    finally:
        for h in (dl, dq, di):
            if h is not None:
                h.close()
    n -= filter_items is not None and len(filter_items) > 0           # the filter mask
    if liked is not None and liked.nnz:
        n -= 1 + 2 * unsorted_rows(liked)                             # the order check and the sorted copy
    path = {1: "mma.sync", 4: "wgmma"}.get(n) if passes == 1 else None
    if n == 3 * passes:
        path = "sort"
    return ids, sc, path, passes


def check_path(got_path, got_passes, want, what):
    path, passes = want
    assert (got_path, got_passes) == (path.split(" ")[0], passes), f"{what}: expected {want}, ran {got_path} x{got_passes}"


# ---------------------------------------------------------------------------------------- data
def tie_factors(rng, rows, f, zero_frac=0.3):
    Y = rng.integers(-2, 3, size=(rows, f)).astype(np.float32)
    Y[rng.random(rows) < zero_frac] = 0
    return Y


def liked_csr(rng, Q, I, max_len=40, shuffle=True, dup=True):
    """A liked CSR with rows of 0..max_len columns, in random order with repeats when shuffle / dup."""
    lists = []
    for _ in range(Q):
        cols = rng.choice(I, min(int(rng.integers(0, max_len + 1)), I), replace=False)
        if not shuffle:
            cols = np.sort(cols)
        if dup and len(cols) > 2:
            cols = np.concatenate([cols, cols[:2]])
        lists.append(cols)
    indptr = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int32)
    ind = np.concatenate(lists).astype(np.int32) if indptr[-1] else np.zeros(0, np.int32)
    return sp.csr_matrix((np.ones(len(ind), np.float32), ind, indptr), shape=(Q, I))


def model_norms(Y):
    """item norms as the model computes them (implicit/cpu/matrix_factorization_base.py item_norms)"""
    n = np.linalg.norm(Y, axis=-1)
    n[n == 0] = 1e-10
    return n.astype(np.float32)


VARIANTS = ["plain", "liked", "filter", "norms", "query_rows", "all"]


def variant(v, rng, Q, I, items):
    """keyword arguments of one case: liked (unsorted, repeats), filter_items (repeats), item norms, query_rows."""
    kw = {}
    n_query = Q
    if v in ("query_rows", "all"):
        kw["query_rows"] = rng.integers(0, Q, size=Q + 13).astype(np.int32)
        n_query = Q + 13
    if v in ("liked", "all"):
        kw["liked"] = liked_csr(rng, n_query, I)
    if v in ("filter", "all"):
        kw["filter_items"] = rng.integers(0, I, size=max(1, I // 60)).astype(np.int32)
    if v in ("norms", "all"):
        kw["item_norms"] = model_norms(items)
    return kw


def dispatch_args(kw):
    return dict(norms="item_norms" in kw, n_filter=len(kw.get("filter_items", ())),
                liked_max=int(np.diff(kw["liked"].indptr).max()) if "liked" in kw else 0)


def reference(orc, items, users, k, kw):
    q = users if kw.get("query_rows") is None else users[kw["query_rows"]]
    return orc.topk(items, q, k, item_norms=kw.get("item_norms"), filter_query_items=kw.get("liked"),
                    filter_items=kw.get("filter_items"))


def k_classes(I):
    """1; the TQ = 4 / 1 switch at 64; 1048, the last k the mma.sync kernel takes, and 1049; I - 1, I and past I."""
    return sorted({1, 16, 17, 64, 65, 1048, 1049, I - 1, I, I + 7})


# (f, queries): every padded class of the mma.sync kernel, full and padded; the wgmma kernel (>= 1024 queries);
# the sort, every model wider than 128 factors
MMA_WIDTHS = [3, 16, 17, 32, 40, 48, 64, 65, 80, 96, 100, 112, 128]
SORT_WIDTHS = [129, 200, 256, 384, 512, 1000, 1024]
WIDTH_CASES = [(f, 40) for f in MMA_WIDTHS] + [(50, 1100), (64, 1100)] + [(f, 40) for f in SORT_WIDTHS]
WIDTH_IDS = [f"f{f}-q{q}" for f, q in WIDTH_CASES]


# ---------------------------------------------------------------------------------------- exact ties
@pytest.mark.parametrize("f,Q", WIDTH_CASES, ids=WIDTH_IDS)
def test_topk_exact_ties_bit_equal_to_select_h(lib, ctx, orc, f, Q):
    rng = np.random.default_rng(f * 31 + Q)
    users = tie_factors(rng, Q, f, zero_frac=0)
    users[[1, Q // 2, Q - 1]] = 0  # every item ties at 0
    seen = set()
    for I in (1500, 97):
        items = tie_factors(rng, I, f)
        for v in VARIANTS:
            kw = variant(v, rng, Q, I, items)
            for k in k_classes(I):
                want = expected_path(f, len(kw.get("query_rows", users)), I, k, **dispatch_args(kw))
                ids, sc, path, passes = run_topk(lib, ctx, items, users, k, **kw)
                what = f"f={f} I={I} {v} k={k}"
                check_path(path, passes, want, what)
                seen.add(want[0])
                eids, esc = reference(orc, items, users, k, kw)
                np.testing.assert_array_equal(ids, eids, err_msg=what)
                np.testing.assert_array_equal(sc, esc, err_msg=what)
    print(f"exact ties f={f} Q={Q}: paths {sorted(seen)}")


# ---------------------------------------------------------------------------------------- fp64
def gamma(n):
    """|fl(q . i) - q . i| <= gamma_n |q| . |i| for an fp32 dot product of length n, FMA or not (Higham 3.1)"""
    return n * U / (1 - n * U)


def check_against_fp64(users, items, ids, sc, k, path, ld, liked=None, flt=None, items64=None, abs_items64=None):
    """Returns the worst ratio of |score - fp64| to the path's bar; asserts ids, filtering and the filtered tail.
    Bars: the tensor-core kernels topk_noise (4 eps |q| max|i| per query row); the sort's FMA scores gamma_ld |q|.|i|
    per returned id, and its largest value over the row's items where two rankings are compared."""
    items64 = items.astype(np.float64) if items64 is None else items64
    S = users.astype(np.float64) @ items64.T
    mask = np.zeros(S.shape, bool)
    if liked is not None:
        mask[np.repeat(np.arange(S.shape[0]), np.diff(liked.indptr)), liked.indices] = True
    if flt is not None:
        mask[:, flt] = True
    S[mask] = NEG
    keff = min(k, S.shape[1])
    ids, sc = ids[:, :keff], sc[:, :keff]
    got = np.take_along_axis(S, ids, axis=1)
    absdot = np.abs(users.astype(np.float64)) @ (np.abs(items64) if abs_items64 is None else abs_items64).T
    if path == "sort":
        g = gamma(ld)
        bar = g * np.take_along_axis(absdot, ids, axis=1)
        noise = g * absdot.max(axis=1, keepdims=True)
    else:
        # topk_noise, or where nothing cancels (all-positive factors) the accumulation bound: 3 ld / 8 MMA results
        # added into a truncating fp32 accumulator (each off by < eps of the sum of |terms|) and the split's dropped
        # lo parts (< 6 eps |q_j i_j|).  On all-positive factors at 128 factors the error reaches ~2x topk_noise.
        g = (3 * ld / 8 + 6) * 2 * U
        tn = topk_noise(users, items)
        bar = np.maximum(tn, g * np.take_along_axis(absdot, ids, axis=1))
        noise = np.maximum(tn, g * absdot.max(axis=1, keepdims=True))
    live = got > NEG
    ratio = worst_ratio(np.abs(sc - got)[live], bar[live])
    assert ratio <= 1.0, f"score error {ratio:.3f} x the bar"
    eids, esc = select_h(S, k)
    eids, esc = eids[:, :keff], esc[:, :keff]
    # the r-th largest of scores each within `noise` of the truth is within `noise` of the r-th largest truth
    _, bad = topk_mismatches(ids, sc, eids, esc, noise)
    assert bad.sum() == 0, f"{bad.sum()} ids differ from fp64 select.h away from near-ties"
    n_live = (~mask).sum(axis=1)
    for r in range(len(S)):  # no filtered id while unfiltered items remain; the filtered tail follows select.h
        assert live[r, :min(keff, n_live[r])].all(), f"row {r}: a filtered id ranked before an unfiltered one"
        np.testing.assert_array_equal(ids[r, n_live[r]:], eids[r, n_live[r]:], err_msg=f"row {r}: filtered tail")
        assert (sc[r, n_live[r]:] == NEG).all()
    return ratio


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("f,Q", WIDTH_CASES, ids=WIDTH_IDS)
def test_topk_against_fp64(lib, ctx, f, Q, kind):
    """Bars: the tensor-core kernels 4 eps |q| max|i| per query row (topk_noise: split operands, fp32 accumulation);
    the sort's FMA scores gamma_ld |q| . |i| per returned id.  Near-ties (two ranks within the bar) may order either
    way."""
    I = 1500
    rng = np.random.default_rng(f * 7 + Q + len(kind))
    items, users = factors_of(kind, I, f, seed=f + 1), factors_of(kind, Q, f, seed=f + 2)
    liked = liked_csr(rng, Q, I, max_len=60)
    flt = rng.integers(0, I, size=30).astype(np.int32)
    worst = {}
    for k in k_classes(I):
        want = expected_path(f, Q, I, k, n_filter=len(flt), liked_max=int(np.diff(liked.indptr).max()))
        ids, sc, path, passes = run_topk(lib, ctx, items, users, k, liked=liked, filter_items=flt)
        check_path(path, passes, want, f"f={f} {kind} k={k}")
        r = check_against_fp64(users, items, ids, sc, k, path, padded(f), liked, flt)
        worst[want[0]] = max(worst.get(want[0], 0.0), r)
    print(f"fp64 f={f} Q={Q} {kind}: worst |score - fp64| / bar " + ", ".join(f"{p} {w:.3f}" for p, w in worst.items()))


# ---------------------------------------------------------------------------------------- grid and tile edges
@pytest.mark.parametrize("k", [33, 100], ids=["TQ4", "TQ1"])
@pytest.mark.parametrize("f", [32, 64, 128])
def test_topk_kernel_grid_and_tile_edges(lib, ctx, sm, f, k):
    """topk_kernel<F, TQ> with one and two query blocks past a full grid and a ragged last block, and two full grids
    plus one (CTAs take a second and a third block); items 1, 31, 32, 33 and around one and three tiles.  The liked
    lists differ from row to row, so a cursor kept from a CTA's previous block would filter the wrong columns.  The
    exact integer scores make select.h on the fp64 product the reference, bit for bit.  (Item counts of 64 or fewer
    leave k_eff <= 64, which runs TQ = 4.)"""
    rng = np.random.default_rng(f + k)
    ran = set()
    F = padded(f)
    IT = tk_cfg(F, 4)[1]
    for I in sorted({1, 31, 32, 33, IT - 1, IT, IT + 1, 3 * IT + 37}):
        keff = min(k, I)
        TQ = 4 if keff <= 64 else 1
        QB, IT, ctas = tk_cfg(F, TQ)
        grid = sm * ctas
        items = tie_factors(rng, I, f)
        for n_query in (QB * (grid + 1) + QB // 2 + 1, QB * (grid + 2) + 3, QB * (2 * grid + 1) + QB - 1):
            users = tie_factors(rng, n_query, f, zero_frac=0.01)
            liked = liked_csr(rng, n_query, I, max_len=min(I, 9), shuffle=False, dup=False)
            want = expected_path(f, n_query, I, k, liked_max=int(np.diff(liked.indptr).max()))
            assert want[0] == f"mma.sync TQ={TQ}"
            ids, sc, path, passes = run_topk(lib, ctx, items, users, k, liked=liked)
            check_path(path, passes, want, f"f={f} I={I} Q={n_query} k={k}")
            S = (users.astype(np.float64) @ items.astype(np.float64).T).astype(np.float32)  # exact
            S[np.repeat(np.arange(n_query), np.diff(liked.indptr)), liked.indices] = NEG
            eids, esc = oracle.port.select(S, k)
            np.testing.assert_array_equal(ids, eids, err_msg=f"I={I} Q={n_query}")
            np.testing.assert_array_equal(sc, esc, err_msg=f"I={I} Q={n_query}")
            ran.add((TQ, IT, n_query // QB))
    print(f"grid edges f={f} k={k}: (TQ, items per tile, full query blocks) {sorted(ran)}")


# ---------------------------------------------------------------------------------------- the sort in several passes
@pytest.mark.parametrize("data", ["ties", "fp64"])
@pytest.mark.parametrize("f,k", [(64, 1100), (200, 10)])
def test_topk_by_sort_in_several_passes(lib, ctx, f, k, data):
    """2^20 + 3 items leave room for 63 rows per pass: 130 queries run as passes of 63, 63 and 4."""
    Q, I = 130, (1 << 20) + 3
    rng = np.random.default_rng(f + k)
    if data == "ties":
        items, users = tie_factors(rng, I, f), tie_factors(rng, Q, f, zero_frac=0.05)
    else:
        items, users = factors_of("mixed", I, f, seed=1), factors_of("decades", Q, f, seed=2)
    liked = liked_csr(rng, Q, I, max_len=300)
    flt = rng.integers(0, I, size=500).astype(np.int32)
    want = expected_path(f, Q, I, k, n_filter=len(flt), liked_max=int(np.diff(liked.indptr).max()))
    assert want == ("sort", 3)
    ids, sc, path, passes = run_topk(lib, ctx, items, users, k, liked=liked, filter_items=flt)
    check_path(path, passes, want, f"f={f} k={k} {data}")
    worst = 0.0
    items64 = items.astype(np.float64)
    abs_items64 = np.abs(items64) if data == "fp64" else None
    for r0 in range(0, Q, 10):  # row blocks: a full score matrix would take a gigabyte
        r1 = min(Q, r0 + 10)
        sub = liked[r0:r1]
        if data == "ties":
            S = (users[r0:r1].astype(np.float64) @ items64.T).astype(np.float32)  # exact
            S[np.repeat(np.arange(r1 - r0), np.diff(sub.indptr)), sub.indices] = NEG
            S[:, flt] = NEG
            eids, esc = oracle.port.select(S, k)
            np.testing.assert_array_equal(ids[r0:r1], eids, err_msg=f"rows {r0}..{r1}")
            np.testing.assert_array_equal(sc[r0:r1], esc, err_msg=f"rows {r0}..{r1}")
        else:
            worst = max(worst, check_against_fp64(users[r0:r1], items, ids[r0:r1], sc[r0:r1], k, "sort", padded(f),
                                                  sub, flt, items64, abs_items64))
    print(f"sort in 3 passes f={f} k={k} {data}: worst |score - fp64| / bar {worst:.3f}")


# ---------------------------------------------------------------------------------------- the public class
def _tie_model(f, users, n_items, seed):
    from implicit_b200.als import AlternatingLeastSquares

    rng = np.random.default_rng(seed)
    m = AlternatingLeastSquares(factors=f, random_state=0)
    m.user_factors = tie_factors(rng, users, f, zero_frac=0.05)
    m.item_factors = tie_factors(rng, n_items, f)
    return m


class TopkModel:
    """A stand-in model whose recommend is the reference's (matrix_factorization_base.py recommend, no items=)."""

    def __init__(self, orc, X, Y):
        self.orc, self.X, self.Y = orc, X, Y

    def recommend(self, userid, user_items, N=10, **kwargs):
        return self.orc.topk(self.Y, self.X[np.asarray(userid)], N, filter_query_items=user_items)


@pytest.mark.parametrize("f,N", [(200, 10), (200, 1200), (64, 1100)])
def test_public_class_with_tied_scores(orc, f, N):
    """recommend (also with filter_items and items=), similar_items and ranking_metrics_at_k on a model with integer
    factors, against the reference's logic on orc.topk: at 200 factors every call takes the sort, at 64 factors
    N > 1048 does."""
    from implicit_b200 import evaluation
    from oracle import evaluation_oracle

    users, n_items = 300, 2000
    m = _tie_model(f, users, n_items, seed=f + N)
    X, Y = m.user_factors, m.item_factors
    rng = np.random.default_rng(N)
    train = sp.random(users, n_items, density=0.02, format="csr", dtype=np.float32, random_state=f)
    uids = np.arange(0, users, 3)
    liked = train[uids]

    ids, sc = m.recommend(uids, liked, N=N)
    eids, esc = orc.topk(Y, X[uids], N, filter_query_items=liked)
    np.testing.assert_array_equal(ids, eids)
    np.testing.assert_array_equal(sc, esc)

    flt = rng.integers(0, n_items, size=50)
    ids, sc = m.recommend(uids, liked, N=N, filter_items=flt)
    eids, esc = orc.topk(Y, X[uids], N, filter_query_items=liked, filter_items=flt)
    np.testing.assert_array_equal(ids, eids)
    np.testing.assert_array_equal(sc, esc)

    subset = rng.choice(n_items, 1500, replace=False)
    ids, sc = m.recommend(uids, liked, N=N, items=subset)
    items = np.sort(subset)
    coo = liked.tocoo()  # matrix_factorization_base.py _filter_items_from_sparse_matrix: liked ids -> positions
    pos = np.clip(np.searchsorted(items, coo.col), 0, len(items) - 1)
    keep = items[pos] == coo.col
    fq = sp.csr_matrix((np.ones(keep.sum(), np.float32), (coo.row[keep], pos[keep])), shape=(len(uids), len(items)))
    eids, esc = orc.topk(Y[items], X[uids], min(N, len(items)), filter_query_items=fq)
    np.testing.assert_array_equal(ids, items[eids])
    np.testing.assert_array_equal(sc, esc)

    norms = np.linalg.norm(Y, axis=-1)
    norms[norms == 0] = 1e-10
    iids = np.arange(0, n_items, 37)
    ids, sc = m.similar_items(iids, N=N)
    eids, esc = orc.topk(Y, Y[iids], N, item_norms=norms)
    np.testing.assert_array_equal(ids, eids)
    np.testing.assert_array_equal(sc, esc / norms[iids][:, None])

    test = sp.random(users, n_items, density=0.01, format="csr", dtype=np.float32, random_state=f + 1)
    K = N
    got = evaluation.ranking_metrics_at_k(m, train, test, K=K, show_progress=False)
    exp = evaluation_oracle.ranking_metrics_at_k(TopkModel(orc, X, Y), train, test, K=K)
    for key in ("precision", "map", "ndcg", "auc"):
        assert got[key] == pytest.approx(exp[key], rel=1e-12, abs=0), key
    print(f"public class f={f} N={N}: " + ", ".join(f"{key} {got[key]:.6f}" for key in ("precision", "map", "ndcg", "auc")))
