"""The serving cases tests/golden/serving.npz pins: recommend, rank_items and similar_* called with host ids (lists, numpy
arrays and scalars) on seeded models, and what each returned or raised.  tests/golden/make_golden_serving.py records
them; tests/test_gpu_serving_golden.py replays them.  Every input is rebuilt here from its seed."""
import numpy as np
import scipy.sparse as sp

USERS, ITEMS = 1100, 1200
WIDTHS = (16, 40, 64, 100, 128, 192, 512, 1024)
ZERO_ROWS = (3, 77)  # zero in both factor matrices: norm 1e-10


def model(ctx, f):
    from implicit_b200 import AlternatingLeastSquares

    rng = np.random.default_rng(1000 + f)
    m = AlternatingLeastSquares(factors=f, iterations=1, regularization=0.1, random_state=1)
    m._ctx = ctx
    X = rng.standard_normal((USERS, f), dtype=np.float32)
    Y = rng.standard_normal((ITEMS, f), dtype=np.float32)
    X[list(ZERO_ROWS)] = 0
    Y[list(ZERO_ROWS)] = 0
    m.user_factors, m.item_factors = X, Y
    return m


def liked(rows, per_row=9, seed=1, positive=False):
    """A scipy CSR of `rows` rows over the items: unsorted rows, duplicate columns, empty rows and, unless `positive`
    (a recalculation's confidences), stored zeros and negative values."""
    rng = np.random.default_rng(seed)
    counts = rng.integers(0, 2 * per_row, rows)
    counts[::7] = 0
    indptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    indices = rng.integers(0, ITEMS, indptr[-1]).astype(np.int32)
    dup = rng.random(len(indices)) < 0.1
    indices[1:][dup[1:]] = indices[:-1][dup[1:]]
    data = rng.uniform(-2, 3, len(indices)).astype(np.float32)
    data[rng.random(len(data)) < 0.1] = 0
    if positive:
        data = np.abs(data) + np.float32(1)
    return sp.csr_matrix((data, indices, indptr), shape=(rows, ITEMS))


def item_users(rows, seed):
    """A scipy CSR of `rows` rows over the users, positive confidences, for recalculate_item."""
    M = liked(rows, seed=seed, positive=True)
    return sp.csr_matrix((M.data, M.indices % USERS, M.indptr), shape=(rows, USERS))


def device_csr(M):
    import torch

    ip, ix, v = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in
                 (M.indptr.astype(np.int64), M.indices.astype(np.int64), M.data))
    return torch.sparse_csr_tensor(ip, ix, v, size=M.shape)


def cases():
    """[(name, factors, method, kwargs, cuda, liked_max)]: `cuda` when the same call with the ids as a CUDA array must
    return the same values (2-D); `liked_max` the als._LIKED_NNZ_MAX to call with (None: unchanged)."""
    out = []

    def add(name, f, method, cuda=True, liked_max=None, **kw):
        out.append((name, f, method, kw, cuda, liked_max))

    rng = np.random.default_rng(7)
    u60 = rng.integers(0, USERS, 60)
    i40 = np.concatenate([list(ZERO_ROWS), rng.integers(0, ITEMS, 38)])
    u25 = np.concatenate([[3], rng.integers(0, USERS, 24)])
    sub = rng.integers(0, ITEMS, 80)  # unsorted, with duplicates
    fl = rng.integers(0, ITEMS, 40)
    for f in WIDTHS:
        add(f"rec_f{f}", f, "recommend", userid=u60, user_items=liked(60, seed=f), N=10)
        add(f"rec_scalar_f{f}", f, "recommend", userid=7, user_items=liked(8, per_row=20, seed=f)[[3]], N=10)
        add(f"sim_items_f{f}", f, "similar_items", itemid=i40, N=10)
        add(f"sim_users_f{f}", f, "similar_users", userid=u25, N=10)
        add(f"sim_items_subset_f{f}", f, "similar_items", itemid=i40, N=12, items=sub)
        add(f"sim_items_filter_f{f}", f, "similar_items", itemid=i40, N=10, filter_items=fl)
        add(f"sim_scalar_f{f}", f, "similar_items", itemid=77, N=10)
        add(f"rec_recalc_f{f}", f, "recommend", userid=u60[:20], user_items=liked(20, seed=f, positive=True), N=10,
            recalculate_user=True)
        add(f"sim_recalc_f{f}", f, "similar_items", itemid=i40[:20], N=10, recalculate_item=True,
            item_users=item_users(20, seed=f))

    # each top-k kernel: mma.sync (few queries), wgmma (64 factors, >= 1024 queries, k <= 16), by-sort (k > 1048)
    L = liked(USERS, seed=4)
    users = np.arange(USERS)
    add("rec_mma", 64, "recommend", userid=users[:40], user_items=L[:40], N=10)
    add("rec_wgmma", 64, "recommend", userid=users, user_items=L, N=16)
    add("rec_wgmma_noliked", 64, "recommend", userid=users, user_items=None, N=10, filter_already_liked_items=False)
    add("rec_bysort", 64, "recommend", userid=users[:30], user_items=L[:30], N=1100)
    add("rec_zero_tail", 64, "recommend", userid=users[:20], user_items=L[:20], N=ITEMS + 9)
    add("rec_zero_tail_f192", 192, "recommend", userid=users[:20], user_items=L[:20], N=ITEMS + 9)
    add("sim_zero_tail", 40, "similar_users", userid=u25[:10], N=USERS + 5)

    # filter_items and ids of every accepted kind
    L20 = liked(20, seed=5)
    u20 = u60[:20]
    add("rec_filter_list", 64, "recommend", userid=u20, user_items=L20, N=12, filter_items=fl.tolist())
    add("rec_filter_i32", 64, "recommend", userid=u20, user_items=L20, N=12, filter_items=fl.astype(np.int32))
    add("rec_filter_i16", 64, "recommend", cuda=False, userid=u20, user_items=L20, N=12, filter_items=fl.astype(np.int16))
    add("rec_filter_f64", 64, "recommend", cuda=False, userid=u20, user_items=L20, N=12, filter_items=fl.astype(float))
    add("rec_filter_scalar", 64, "recommend", cuda=False, userid=u20, user_items=L20, N=12, filter_items=5)
    add("rec_filter_empty", 64, "recommend", userid=u20, user_items=L20, N=12, filter_items=[])
    add("rec_ids_list", 64, "recommend", userid=u20.tolist(), user_items=L20, N=12)
    add("rec_ids_i32", 64, "recommend", userid=u20.astype(np.int32), user_items=L20, N=12)
    add("rec_ids_i16", 64, "recommend", cuda=False, userid=u20.astype(np.int16), user_items=L20, N=12)
    add("rec_ids_u32", 64, "recommend", cuda=False, userid=u20.astype(np.uint32), user_items=L20, N=12)
    add("rec_ids_f64", 64, "recommend", cuda=False, userid=u20.astype(float), user_items=L20, N=12)
    add("rec_ids_empty", 64, "recommend", userid=np.array([], dtype=np.int64), user_items=None, N=12,
        filter_already_liked_items=False)
    add("rec_no_liked", 40, "recommend", userid=u20, user_items=None, N=12, filter_already_liked_items=False)

    # items=: a subset, unsorted with duplicates, some of it liked
    L30 = liked(20, per_row=30, seed=6)
    s = sub.copy()
    s[:10] = L30.indices[:10]
    for kind, items in (("i64", s), ("list", s.tolist()), ("i32", s.astype(np.int32)), ("i16", s.astype(np.int16)),
                        ("u32", s.astype(np.uint32))):
        add(f"rec_items_{kind}", 64, "recommend", cuda=kind in ("i64", "list", "i32"), userid=u20, user_items=L30,
            N=15, items=items)
    add("rec_items_big_n", 16, "recommend", userid=u20, user_items=L30, N=500, items=s)
    add("rec_items_filter_empty", 64, "recommend", userid=u20, user_items=L30, N=15, items=s, filter_items=[])
    add("rec_items_scalar", 128, "recommend", userid=9, user_items=L30[[4]], N=15, items=s)
    # a filter numpy finds false next to items: it filters positions of the sorted subset
    for kind, zero in (("array", np.array([0])), ("int", 0), ("i64", np.int64(0))):
        add(f"rec_items_filter_zero_{kind}", 64, "recommend", cuda=False, userid=u20, user_items=L30, N=15, items=s,
            filter_items=zero)
    add("rec_n0", 64, "recommend", userid=u20, user_items=L30, N=0)
    Lp = liked(20, seed=8, positive=True)
    add("rec_recalc_items", 64, "recommend", userid=u20, user_items=Lp, N=10, recalculate_user=True, items=s)
    add("rec_recalc_scalar", 64, "recommend", userid=4, user_items=Lp[[2]], N=10, recalculate_user=True)
    add("rank_items", 40, "rank_items", userid=u20, user_items=None, selected_items=[9, 3, 400, 3, 17, 1100])
    add("rank_items_i32", 40, "rank_items", userid=u20, user_items=None,
        selected_items=np.array([9, 3, 400, 3, 17, 1100], dtype=np.int32))
    add("rank_items_scalar", 40, "rank_items", userid=11, user_items=None, selected_items=[5, 2, 8])

    # a liked filter split into batches of at most 700 nonzeros
    L400 = liked(400, seed=5)
    u400 = np.arange(400)
    add("rec_liked_batches", 64, "recommend", liked_max=700, userid=u400, user_items=L400, N=11)
    add("rec_liked_batches_items", 64, "recommend", liked_max=700, userid=u400, user_items=L400, N=11,
        items=np.arange(0, ITEMS, 2))
    add("rec_liked_batches_recalc", 64, "recommend", liked_max=700, userid=u400,
        user_items=liked(400, seed=5, positive=True), N=11, recalculate_user=True)

    # similar_*: subsets and filters of every kind, recalculation of one item
    add("sim_subset_list", 64, "similar_items", itemid=i40, N=10, items=sub.tolist())
    add("sim_subset_i32", 64, "similar_items", itemid=i40, N=10, items=sub.astype(np.int32))
    add("sim_subset_i16", 64, "similar_items", cuda=False, itemid=i40, N=10, items=sub.astype(np.int16))
    add("sim_subset_big_n", 64, "similar_items", itemid=i40, N=100, items=sub)
    add("sim_users_subset", 100, "similar_users", userid=u25, N=30, users=sub[sub < USERS])
    add("sim_users_filter", 64, "similar_users", userid=u25, N=10, filter_users=fl[fl < USERS].tolist())
    add("sim_filter_outside", 64, "similar_items", cuda=False, itemid=i40, N=10,
        filter_items=np.array([-5, 4, ITEMS, ITEMS + 3, 7]))
    add("sim_filter_i16", 64, "similar_items", cuda=False, itemid=i40, N=10, filter_items=fl.astype(np.int16))
    add("sim_filter_empty", 64, "similar_items", itemid=i40, N=10, filter_items=[])
    add("sim_scalar_user", 40, "similar_users", userid=3, N=10)
    add("sim_subset_filter_zero", 64, "similar_items", cuda=False, itemid=i40, N=10, items=sub, filter_items=np.array([0]))
    add("sim_users_subset_filter_zero", 64, "similar_users", cuda=False, userid=u25, N=10, users=sub[sub < USERS],
        filter_users=0)
    add("sim_negative_n0", 64, "similar_items", cuda=False, itemid=np.array([-1, 2]), N=0)
    add("sim_negative_n0_scalar", 64, "similar_users", cuda=False, userid=-3, N=0)
    add("sim_scalar_subset", 40, "similar_items", itemid=12, N=10, items=sub)
    add("sim_recalc_scalar", 64, "similar_items", cuda=False, itemid=5, N=10, recalculate_item=True,
        item_users=item_users(1, seed=9))
    add("sim_recalc_scalar_f512", 512, "similar_items", cuda=False, itemid=5, N=10, recalculate_item=True,
        item_users=item_users(1, seed=10))
    add("sim_recalc_subset", 64, "similar_items", itemid=i40[:20], N=10, recalculate_item=True,
        item_users=item_users(20, seed=11), items=sub)

    # refusals: the exception and message of the host path, checked in its order
    Le = liked(20, seed=12)
    bad_u = u20.copy()
    bad_u[5] = USERS
    neg_u = u20.copy()
    neg_u[3] = -1
    for name, kw in (
        ("userid_high", dict(userid=bad_u)),
        ("userid_negative", dict(userid=neg_u)),
        ("userid_and_items", dict(userid=bad_u, items=[0, ITEMS])),
        ("userid_and_filter", dict(userid=neg_u, filter_items=[ITEMS])),
        ("userid_and_items_and_filter", dict(userid=bad_u, items=[0, 5], filter_items=[3])),
        ("filter_high", dict(filter_items=[0, ITEMS])),
        ("filter_negative", dict(filter_items=np.array([4, -2]))),
        ("items_high", dict(items=[0, ITEMS])),
        ("items_negative", dict(items=np.array([-1, 4]))),
        ("items_empty", dict(items=[])),
        ("items_float", dict(items=np.array([1.0, 2.0]))),
        ("items_and_filter_list", dict(items=[0, 5], filter_items=[3])),
        ("items_and_filter_array", dict(items=[0, 5], filter_items=np.array([3, 4]))),
        ("items_and_filter_high", dict(items=[0, 5], filter_items=[ITEMS])),
        ("rows", dict(user_items=Le[:5])),
        ("rows_recalc", dict(user_items=Le[:5], recalculate_user=True)),
        ("not_csr", dict(user_items=Le.toarray())),
        ("device_csr_items", dict(user_items="device", items=[0, 5, 9])),
        ("items_high_device_csr", dict(user_items="device", items=[0, ITEMS])),
    ):
        kw = dict(kw)
        kw.setdefault("userid", u20)
        kw.setdefault("user_items", Le)
        add(f"rec_err_{name}", 64, "recommend", cuda=False, N=5, **kw)
    wide = sp.hstack([Le, sp.csr_matrix((20, 4), dtype=np.float32)]).tocsr()
    add("rec_err_liked_width", 64, "recommend", cuda=False, userid=u20, user_items=wide, N=5)
    add("rec_err_negative_n", 64, "recommend", cuda=False, userid=u20, user_items=Le, N=-1)
    add("rec_err_negative_n_items", 64, "recommend", cuda=False, userid=u20, user_items=Le, N=-1, items=[3, 1, 2])
    add("sim_err_negative_n", 64, "similar_items", cuda=False, itemid=i40, N=-2)
    add("sim_err_negative_n_and_id", 64, "similar_items", cuda=False, itemid=np.array([-1, 2]), N=-2)
    for name, method, kw in (
        ("id_high", "similar_items", dict(itemid=np.array([0, ITEMS]))),
        ("id_high_list", "similar_items", dict(itemid=[4, ITEMS + 2])),
        ("id_high_scalar", "similar_items", dict(itemid=ITEMS)),
        ("id_negative", "similar_items", dict(itemid=np.array([2, -1, -4]))),
        ("id_negative_scalar", "similar_users", dict(userid=-3)),
        ("id_negative_and_subset", "similar_items", dict(itemid=[-2, 1], items=[5, 6, 7])),
        ("id_float", "similar_items", dict(itemid=np.array([1.0, 2.0]))),
        ("id_high_and_subset", "similar_items", dict(itemid=[ITEMS], items=[1, ITEMS])),
        ("subset_high", "similar_items", dict(itemid=[1, 2], items=[1, ITEMS])),
        ("subset_negative", "similar_users", dict(userid=[1, 2], users=np.array([-1, 2]))),
        ("subset_empty", "similar_items", dict(itemid=[1, 2], items=[])),
        ("subset_float", "similar_items", dict(itemid=[1, 2], items=np.array([1.0, 3.0]))),
        ("subset_and_filter", "similar_items", dict(itemid=[1, 2], items=[1, 2], filter_items=[3])),
        ("subset_and_filter_array", "similar_items", dict(itemid=[1, 2], items=[1, 2], filter_items=np.array([3, 4]))),
        ("subset_and_filter_users", "similar_users", dict(userid=[1, 2], users=[1, 2], filter_users=[3])),
    ):
        add(f"sim_err_{name}", 64, method, cuda=False, N=5, **kw)
    return out


def call(m, method, kw):
    """m.<method>(**kw), with user_items="device" standing for the kwargs' liked filter as a CUDA CSR.  Every scipy CSR
    is passed as a copy: the liked remap of items= writes zeros into the data of the CSR it is given."""
    kw = {k: v.copy() if sp.issparse(v) else v for k, v in kw.items()}
    if isinstance(kw.get("user_items"), str):
        kw["user_items"] = device_csr(liked(len(np.atleast_1d(kw["userid"])), seed=12))
    return getattr(m, method)(**kw)
