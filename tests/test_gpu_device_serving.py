"""recommend, rank_items and similar_* with their ids in CUDA memory: the call hands back CUDA arrays, bitwise the ids
and scores of the same call with numpy ids (which goes through the host adapter; a scipy liked filter of the same
float32 entries).  tests/test_gpu_serving_golden.py ties the numpy-id calls to recorded results.  PyTorch plays the
producer; the package itself never imports it.
"""
import gc
import os

import numpy as np
import pytest
import scipy.sparse as sp

from helpers import KNOB_DEFAULTS

torch = pytest.importorskip("torch")

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs PyTorch with CUDA as the producer")]


class Cai:
    """A tensor behind an interface dict of our choosing (version 2, or version 3 naming a stream)."""

    def __init__(self, t, **override):
        self.t = t
        self.__cuda_array_interface__ = dict(t.__cuda_array_interface__, **override)


class CaiCSR:
    def __init__(self, indptr, indices, data, shape):
        self.indptr, self.indices, self.data, self.shape = indptr, indices, data, shape


@pytest.fixture(scope="module")
def ctx():
    names = [f"ALS_B200_{k.upper()}" for k in list(KNOB_DEFAULTS) + ["segment_nnz", "host_csr"]]
    set_in_env = sorted(n for n in names if n in os.environ)
    if set_in_env:
        pytest.fail(f"knob environment variables are set: {', '.join(set_in_env)}; unset them to run these tests")
    from implicit_b200 import _lib

    c = _lib.Context(0)
    yield c
    c.close()


USERS, ITEMS = 1300, 1200


def model(ctx, f, users=USERS, items=ITEMS, seed=0, zero_rows=()):
    from implicit_b200 import AlternatingLeastSquares

    rng = np.random.default_rng(seed + f)
    m = AlternatingLeastSquares(factors=f, iterations=1, regularization=0.1, random_state=1)
    m._ctx = ctx
    X = rng.standard_normal((users, f), dtype=np.float32)
    Y = rng.standard_normal((items, f), dtype=np.float32)
    Y[list(zero_rows)] = 0
    X[list(zero_rows)] = 0
    m.user_factors, m.item_factors = X, Y
    return m


@pytest.fixture(scope="module")
def models(ctx):
    return {f: model(ctx, f, zero_rows=(3, 77)) for f in (16, 40, 64, 100, 128, 192, 512, 1024)}


def liked_csr(rows, cols, per_row=9, seed=1):
    """Unsorted rows, duplicate columns, stored zeros, negative values and empty rows."""
    rng = np.random.default_rng(seed)
    counts = rng.integers(0, 2 * per_row, rows)
    counts[::7] = 0
    indptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    indices = rng.integers(0, cols, indptr[-1]).astype(np.int32)
    dup = rng.random(len(indices)) < 0.1
    indices[1:][dup[1:]] = indices[:-1][dup[1:]]
    data = rng.uniform(-2, 3, len(indices)).astype(np.float32)
    data[rng.random(len(data)) < 0.1] = 0
    M = sp.csr_matrix((data, indices, indptr), shape=(rows, cols))
    assert not M.has_sorted_indices and (M.data == 0).any() and (M.data < 0).any()
    return M


def device_csr(M, index_dtype=np.int64):
    ip, ix, v = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in
                 (M.indptr.astype(index_dtype), M.indices.astype(index_dtype), M.data))
    return torch.sparse_csr_tensor(ip, ix, v, size=M.shape)


def cu(a, dtype=np.int64):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=dtype))).cuda()


def host(x):
    cai = x.__cuda_array_interface__
    assert cai["version"] == 3 and cai["stream"] is None
    return torch.as_tensor(x, device="cuda").cpu().numpy()


def same(got, want):
    gi, gs = host(got[0]), host(got[1])
    wi, ws = np.atleast_2d(want[0]), np.atleast_2d(want[1])
    assert gi.dtype == wi.dtype and gs.dtype == ws.dtype == np.float32, (gi.dtype, wi.dtype, gs.dtype)
    assert gi.shape == wi.shape and np.array_equal(gi, wi)
    assert np.array_equal(gs.view(np.uint32), ws.view(np.uint32))


# ---- recommend --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f", [16, 40, 64, 100, 128, 192, 1024])
def test_recommend_matches_host(models, f):
    m = models[f]
    rng = np.random.default_rng(f)
    users = rng.integers(0, USERS, 150)
    L = liked_csr(len(users), ITEMS, seed=f)
    fl = rng.integers(0, ITEMS, 40)
    for dtype in (np.int32, np.int64):
        for N in (7, ITEMS + 9):
            same(m.recommend(cu(users, dtype), L, N=N), m.recommend(users.astype(dtype), L, N=N))
            same(m.recommend(cu(users, dtype), device_csr(L), N=N), m.recommend(users, L, N=N))
        same(m.recommend(cu(users, dtype), L, N=12, filter_items=cu(fl, dtype)),
             m.recommend(users, L, N=12, filter_items=fl))
        same(m.recommend(cu(users, dtype), L, N=12, filter_items=fl), m.recommend(users, L, N=12, filter_items=fl))
        same(m.recommend(cu(users, dtype), None, N=12, filter_already_liked_items=False),
             m.recommend(users, None, N=12, filter_already_liked_items=False))


@pytest.mark.parametrize("f", [16, 64, 128])
def test_recommend_with_items_matches_host(models, f):
    m = models[f]
    rng = np.random.default_rng(f + 1)
    users = rng.integers(0, USERS, 120)
    L = liked_csr(len(users), ITEMS, per_row=30, seed=f)
    subset = rng.integers(0, ITEMS, 300)  # unsorted, with duplicates
    subset[:20] = L.indices[:20]
    for dtype in (np.int32, np.int64):
        want = m.recommend(users, L, N=15, items=subset.astype(dtype))
        same(m.recommend(cu(users), L, N=15, items=subset.astype(dtype)), want)
        same(m.recommend(cu(users), L, N=15, items=cu(subset, dtype)), want)
        same(m.recommend(cu(users), device_csr(L), N=15, items=cu(subset, dtype)), want)
        same(m.recommend(cu(users), device_csr(L), N=500, items=subset.astype(dtype)),
             m.recommend(users, L, N=500, items=subset.astype(dtype)))


@pytest.mark.parametrize("f", [40, 64])
def test_recommend_recalculate_user_matches_host(models, f):
    m = models[f]
    users = np.arange(30, 230)
    L = abs(liked_csr(len(users), ITEMS, seed=3))
    L.data += np.float32(1)
    want = m.recommend(users, L, N=10, recalculate_user=True)
    same(m.recommend(cu(users, np.int32), L, N=10, recalculate_user=True), want)
    same(m.recommend(cu(users), device_csr(L), N=10, recalculate_user=True), want)
    subset = np.arange(5, ITEMS, 3)
    same(m.recommend(cu(users), device_csr(L), N=10, recalculate_user=True, items=cu(subset)),
         m.recommend(users, L, N=10, recalculate_user=True, items=subset))


def test_interface_wrappers_and_producer_stream(models):
    m = models[64]
    users = np.arange(0, 500, 3)
    L = liked_csr(len(users), ITEMS, seed=9)
    want = m.recommend(users, L, N=10, filter_items=np.arange(100))
    truth, fl_truth = cu(users, np.int32), cu(np.arange(100))
    same(m.recommend(Cai(truth, version=2), L, N=10, filter_items=Cai(fl_truth, version=2)), want)
    u, fl = torch.zeros_like(truth), torch.zeros_like(fl_truth)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)  # the ids land some 0.1 s after the call is made
        u.copy_(truth)
        fl.copy_(fl_truth)
    s = side.cuda_stream
    got = m.recommend(Cai(u, version=3, stream=s), L, N=10, filter_items=Cai(fl, version=3, stream=s))
    same(got, want)


def test_each_topk_path(ctx):
    """mma.sync (few queries), wgmma (64 factors, k <= 16, >= 1024 queries), by-sort (k past the register lists)."""
    m = model(ctx, 64, users=2100, items=1500)
    L = liked_csr(2100, 1500, seed=4)
    users = np.arange(2100)
    for q, N in ((40, 10), (2100, 10), (40, 1200), (2100, 16)):
        same(m.recommend(cu(users[:q]), L[:q], N=N), m.recommend(users[:q], L[:q], N=N))
        same(m.recommend(cu(users[:q]), device_csr(L[:q]), N=N), m.recommend(users[:q], L[:q], N=N))
    same(m.recommend(cu(users), L, N=10, items=np.arange(0, 1500, 2)),
         m.recommend(users, L, N=10, items=np.arange(0, 1500, 2)))


def test_liked_batches(models, monkeypatch):
    from implicit_b200 import als

    m = models[64]
    users = np.arange(400)
    L = liked_csr(400, ITEMS, seed=5)
    monkeypatch.setattr(als, "_LIKED_NNZ_MAX", 700)
    assert len(als.liked_batches(L.sorted_indices().indptr, 700)) > 3
    same(m.recommend(cu(users), L, N=11), m.recommend(users, L, N=11))
    subset = np.arange(0, ITEMS, 2)
    same(m.recommend(cu(users), L, N=11, items=cu(subset)), m.recommend(users, L, N=11, items=subset))
    Lr = abs(L)
    Lr.data += np.float32(1)
    same(m.recommend(cu(users), Lr, N=11, recalculate_user=True), m.recommend(users, Lr, N=11, recalculate_user=True))


def test_rank_items(models):
    m = models[40]
    users, sel = np.arange(50), np.array([9, 3, 400, 3, 17, 1100])
    same(m.rank_items(cu(users), None, sel), m.rank_items(users, None, sel))
    same(m.rank_items(cu(users), None, cu(sel, np.int32)), m.rank_items(users, None, sel.astype(np.int32)))


# ---- similar_* --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f", [16, 40, 64, 100, 128, 192, 512, 1024])
def test_similar_matches_host(models, f):
    m = models[f]
    from implicit_b200 import _lib

    n = m._device_norms("item")
    assert np.array_equal(host(n).view(np.uint32), m.item_norms.view(np.uint32))
    assert np.array_equal(host(m._device_norms("user")).view(np.uint32), m.user_norms.view(np.uint32))
    rng = np.random.default_rng(f)
    items = np.concatenate([[3, 77], rng.integers(0, ITEMS, 60)])  # rows 3 and 77 are zero: norm 1e-10
    users = np.concatenate([[3], rng.integers(0, USERS, 30)])
    subset = rng.integers(0, ITEMS, 50)
    for dtype in (np.int32, np.int64):
        same(m.similar_items(cu(items, dtype), N=10), m.similar_items(items, N=10))
        same(m.similar_users(cu(users, dtype), N=10), m.similar_users(users, N=10))
        same(m.similar_items(cu(items, dtype), N=10, filter_items=cu(subset)), m.similar_items(items, N=10, filter_items=subset))
        same(m.similar_items(cu(items, dtype), N=10, items=cu(subset, dtype)),
             m.similar_items(items, N=10, items=subset.astype(dtype)))
        same(m.similar_users(cu(users, dtype), N=60, users=subset), m.similar_users(users, N=60, users=subset))
    assert isinstance(m._dev_norms["item"], _lib.DeviceSnapshot)


def test_similar_items_recalculated(models):
    m = models[64]
    items = np.arange(20, 60)
    M = abs(liked_csr(len(items), USERS, seed=8))
    M.data += np.float32(1)
    want = m.similar_items(items, N=9, recalculate_item=True, item_users=M)
    same(m.similar_items(cu(items), N=9, recalculate_item=True, item_users=device_csr(M)), want)
    same(m.similar_items(cu(items), N=9, recalculate_item=True, item_users=M), want)


# ---- refusals ---------------------------------------------------------------------------------------------------
def message(fn, exc):
    with pytest.raises(exc) as e:
        fn()
    return type(e.value), str(e.value)


def test_refusals_match_host(models):
    m = models[64]
    users = np.arange(20)
    L = liked_csr(20, ITEMS)
    cases = [
        (dict(userid=[1, USERS]), IndexError),
        (dict(userid=[-1, 2]), IndexError),
        (dict(filter_items=[ITEMS]), IndexError),
        (dict(items=[0, ITEMS]), IndexError),
        (dict(items=[0, 5], filter_items=[3]), ValueError),
        (dict(user_items=L[:5]), ValueError),
    ]
    for kw, exc in cases:
        uid = np.asarray(kw.pop("userid", users))
        li = kw.pop("user_items", L[:len(uid)])
        want = message(lambda: m.recommend(uid, li, N=5, **kw), exc)
        dev = {k: cu(v) for k, v in kw.items()}
        assert message(lambda: m.recommend(cu(uid), li, N=5, **dev), exc) == want
        assert message(lambda: m.recommend(cu(uid), li, N=5, **kw), exc) == want
    want = message(lambda: m.similar_items(np.arange(5), items=[1, ITEMS]), IndexError)
    assert message(lambda: m.similar_items(cu(np.arange(5)), items=cu([1, ITEMS])), IndexError) == want
    want = message(lambda: m.similar_items(np.arange(5), items=[1, 2], filter_items=[3]), ValueError)
    assert message(lambda: m.similar_items(cu(np.arange(5)), items=[1, 2], filter_items=[3]), ValueError) == want
    assert message(lambda: m.similar_items(cu([0, ITEMS])), IndexError)[1] == "itemid out of range"


def test_bad_id_arrays_refused(models):
    m = models[64]
    L = liked_csr(4, ITEMS)
    with pytest.raises(ValueError, match="typestr"):
        m.recommend(torch.zeros(4, device="cuda"), L)
    with pytest.raises(ValueError, match="1-D"):
        m.recommend(torch.zeros((2, 2), dtype=torch.int64, device="cuda"), L)
    with pytest.raises(ValueError, match="typestr"):
        m.similar_items(torch.zeros(4, dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError, match="1-D"):
        m.similar_users(torch.zeros((2, 2), dtype=torch.int32, device="cuda"))


# ---- outputs ----------------------------------------------------------------------------------------------------
def test_outputs(ctx):
    m = model(ctx, 32)
    users = np.arange(10)
    ids, scores = m.recommend(cu(users), None, N=6, filter_already_liked_items=False)
    want = m.recommend(users, None, N=6, filter_already_liked_items=False)
    for x, dt in ((ids, "<i4"), (scores, "<f4")):
        cai = x.__cuda_array_interface__
        assert cai["shape"] == (10, 6) and cai["typestr"] == dt and cai["stream"] is None and cai["version"] == 3
    t_ids, t_scores = torch.as_tensor(ids, device="cuda"), torch.as_tensor(scores, device="cuda")
    del ids, scores, m
    gc.collect()
    assert np.array_equal(t_ids.cpu().numpy(), want[0]) and np.array_equal(t_scores.cpu().numpy(), want[1])
    m = model(ctx, 32)
    ids, scores = m.recommend(cu([], np.int32), None, N=6, filter_already_liked_items=False)
    assert host(ids).shape == (0, 6) and host(scores).shape == (0, 6)
    ids, _ = m.similar_items(cu(np.arange(4)), N=3, items=np.arange(9, dtype=np.int64))
    assert host(ids).dtype == np.int64


def test_device_factors_are_never_downloaded(ctx, monkeypatch):
    from implicit_b200 import _lib

    rng = np.random.default_rng(11)
    X = rng.standard_normal((USERS, 64), dtype=np.float32)
    Y = rng.standard_normal((ITEMS, 64), dtype=np.float32)
    ref = model(ctx, 64)
    ref.user_factors, ref.item_factors = X, Y
    m = model(ctx, 64)
    m.user_factors, m.item_factors = torch.from_numpy(X).cuda(), torch.from_numpy(Y).cuda()
    calls = []
    real = _lib.DeviceFactors.download
    monkeypatch.setattr(_lib.DeviceFactors, "download", lambda self, *a, **k: calls.append(1) or real(self, *a, **k))
    users, subset = np.arange(100), np.arange(3, ITEMS, 4)
    L = liked_csr(100, ITEMS)
    got = [m.recommend(cu(users), device_csr(L), N=10, items=cu(subset)),
           m.similar_items(cu(np.arange(40)), N=10, items=cu(subset)),
           m.similar_users(cu(np.arange(40)), N=10, users=subset),
           m.similar_items(cu(np.arange(40)), N=10)]
    assert not calls and not m._host_fresh["user"] and not m._host_fresh["item"]
    monkeypatch.undo()
    want = [ref.recommend(users, L, N=10, items=subset), ref.similar_items(np.arange(40), N=10, items=subset),
            ref.similar_users(np.arange(40), N=10, users=subset), ref.similar_items(np.arange(40), N=10)]
    for g, w in zip(got, want):
        same(g, w)
