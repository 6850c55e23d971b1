"""Every device allocation of a call can fail without leaking: with the alloc_fail_at knob set to n, the n-th allocation
through the pool (or a DeviceBlock) of the call fails.  Swept over n = 1, 2, ... until the call succeeds, each failure
must raise and leave the pool's used bytes where a successful run of the same call leaves them; the successful run at
the end must give bitwise the outputs of the first.  Sizes are tiny: the sweep covers every allocation of each call.
PyTorch plays the producer of the CUDA inputs; the package itself never imports it."""
import contextlib
import gc

import numpy as np
import pytest
import scipy.sparse as sp

torch = pytest.importorskip("torch")

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs PyTorch with CUDA as the producer")]

F = 64


@pytest.fixture(scope="module")
def ctx():
    from implicit_b200 import _lib

    c = _lib.Context(0)
    yield c
    c.close()


@contextlib.contextmanager
def knob(ctx, name, value):
    old = ctx.get_knob(name)
    ctx.set_knob(name, value)
    try:
        yield
    finally:
        ctx.set_knob(name, old)


def used(ctx):
    gc.collect()
    torch.cuda.synchronize()
    ctx.sync()
    return ctx.mem_peak()[0]


def host(a):
    if isinstance(a, torch.Tensor):
        return a.cpu().numpy()
    if hasattr(a, "__cuda_array_interface__"):
        return torch.as_tensor(a, device="cuda").cpu().numpy()
    if isinstance(a, (tuple, list)):
        return [host(x) for x in a]
    return np.array(a, copy=True)


def sweep(ctx, run, on=None):
    """run() -> the call's outputs (numpy arrays, or lists of them), with every handle it made closed or dropped.  on:
    the context the call allocates through (default ctx); the pool's counters are the device's."""
    from implicit_b200 import _lib

    on = on or ctx
    want = host(run())
    base = used(ctx)
    n = 1
    while True:
        on.set_knob("alloc_fail_at", n)
        try:
            got = host(run())
        except (_lib.AlsError, ValueError, RuntimeError, MemoryError) as e:
            err = str(e)  # checked below, once the traceback no longer holds the call's frames
        else:
            break
        # the failure is the injected one (its message may be replaced by the caller's refusal)
        assert on.get_knob("alloc_fail_at") == 0, f"allocation {n}: {err}"
        assert used(ctx) == base, f"allocation {n} failed ({err}) and left {used(ctx) - base} bytes of the pool in use"
        n += 1
    on.set_knob("alloc_fail_at", 0)
    assert n > 1, "the call made no allocation through the pool"
    assert used(ctx) == base

    def same(a, b):
        if isinstance(a, list):
            assert len(a) == len(b)
            for x, y in zip(a, b):
                same(x, y)
        else:
            np.testing.assert_array_equal(a, b)

    same(got, want)
    return n - 1


def matrix(rows, cols, nnz, seed, max_row=None):
    rng = np.random.default_rng(seed)
    m = sp.random(rows, cols, density=nnz / (rows * cols), format="csr", random_state=rng, dtype=np.float32)
    m.data = (1.0 + 4.0 * m.data).astype(np.float32)
    if max_row is not None:  # short rows: at most max_row entries each
        m = sp.csr_matrix(m.multiply(sp.csr_matrix((rng.random((rows, cols)) < max_row / cols).astype(np.float32))))
        m.data[m.data == 0] = 1.0
    m.sort_indices()
    return m


def factors(n, seed):
    return (np.random.default_rng(seed).standard_normal((n, F)) * 0.1).astype(np.float32)


def torch_csr(m):
    return torch.sparse_csr_tensor(torch.from_numpy(m.indptr.astype(np.int64)), torch.from_numpy(m.indices.astype(np.int64)),
                                   torch.from_numpy(m.data), size=m.shape).cuda()


def download(c):
    try:
        m = c.download()
        return [m.indptr, m.indices, m.data]
    finally:
        c.close()


def test_upload_segments(ctx):
    from implicit_b200 import _lib

    C = matrix(300, 200, 6000, 1)
    with knob(ctx, "segment_nnz", 1000):
        sweep(ctx, lambda: download(_lib.DeviceCSR.upload(ctx, C)))


def test_host_upload_and_transpose_in_windows(ctx):
    from implicit_b200 import _lib

    C = matrix(400, 300, 20000, 2)

    def run():
        c = _lib.DeviceCSR.upload(ctx, C, host=True)
        try:
            return download(c.transpose())
        finally:
            c.close()

    with knob(ctx, "segment_nnz", 500):
        sweep(ctx, run)


def test_from_device(ctx):
    from implicit_b200 import _lib

    T = torch_csr(matrix(300, 200, 5000, 3))
    sweep(ctx, lambda: download(_lib.DeviceCSR.from_device(ctx, T)))


@pytest.mark.parametrize("resident", ["device", "host"])
@pytest.mark.parametrize("cg", [False, True])
def test_least_squares(ctx, resident, cg):
    from implicit_b200 import _lib

    C = matrix(2000, 300, 12000, 4, max_row=12)
    X0, Y0 = factors(2000, 5), factors(300, 6)
    Y = _lib.DeviceFactors.from_host(ctx, Y0)

    def run():
        c = _lib.DeviceCSR.upload(ctx, C, host=resident == "host")
        X = _lib.DeviceFactors.from_host(ctx, X0)
        try:
            if cg:
                _lib.least_squares_cg(ctx, c, X, Y, 0.1)
            else:
                _lib.least_squares(ctx, c, X, Y, 0.1)
            return X.download()
        finally:
            X.close()
            c.close()

    with knob(ctx, "segment_nnz", 3000 if resident == "host" else 0):
        sweep(ctx, run)
    Y.close()


def model(ctx, users, items, seed):
    from implicit_b200 import AlternatingLeastSquares

    m = AlternatingLeastSquares(factors=F, iterations=1, regularization=0.1, random_state=1)
    m._ctx = ctx
    m.user_factors, m.item_factors = factors(users, seed), factors(items, seed + 1)
    return m


def test_fit(ctx):
    C = matrix(500, 400, 8000, 7)

    def run():
        m = model(ctx, 500, 400, 8)
        m.fit(C, show_progress=False)
        return [np.array(m.user_factors), np.array(m.item_factors)]

    sweep(ctx, run)


def test_recommend_subset_with_device_liked(ctx):
    m = model(ctx, 300, 500, 9)
    users = torch.arange(0, 300, 3, device="cuda")
    liked = torch_csr(matrix(100, 500, 2000, 10))
    subset = torch.arange(3, 500, 7, device="cuda")
    sweep(ctx, lambda: list(m.recommend(users, liked, N=10, items=subset)))


def test_similar_items_subset(ctx):
    m = model(ctx, 300, 500, 11)
    subset = np.arange(1, 500, 5)
    sweep(ctx, lambda: list(m.similar_items(np.arange(0, 500, 7), N=10, items=subset)))


def test_partial_fit_users_growing(ctx):
    R = matrix(40, 500, 600, 12)

    def run():
        m = model(ctx, 300, 500, 13)
        m.partial_fit_users(torch.arange(280, 320, device="cuda"), R)
        return [np.array(m.user_factors), np.array(m.item_factors)]

    sweep(ctx, run)


def test_topk_by_sort(ctx):
    from implicit_b200 import _lib

    items = _lib.DeviceFactors.from_host(ctx, factors(3000, 14))
    queries = _lib.DeviceFactors.from_host(ctx, factors(20, 15))
    sweep(ctx, lambda: list(_lib.topk(ctx, items, queries, 1200)))
    items.close()
    queries.close()


def test_ranking_metrics(ctx):
    from implicit_b200 import evaluation

    m = model(ctx, 400, 300, 16)
    train, test = matrix(400, 300, 6000, 17), matrix(400, 300, 2000, 18)
    sweep(ctx, lambda: [np.array(sorted(evaluation.ranking_metrics_at_k(m, train, test, K=10, show_progress=False).items()),
                                 dtype=object)[:, 1].astype(np.float64)])


def test_bm25_weight(ctx):
    from implicit_b200 import nearest_neighbours
    from implicit_b200.nearest_neighbours import bm25_weight

    C = matrix(300, 200, 5000, 19).tocoo()
    order = np.random.default_rng(20).permutation(C.nnz)
    coo = sp.coo_matrix((C.data[order], (C.row[order], C.col[order])), shape=C.shape)
    T = torch_csr(matrix(300, 200, 5000, 21))

    def run():
        w = bm25_weight(T)
        d = torch.as_tensor(w.data).cpu().numpy().copy()
        del w
        return [bm25_weight(coo).data, d]

    sweep(ctx, run, on=nearest_neighbours._context())


def test_generate(ctx):
    from implicit_b200 import _lib

    sweep(ctx, lambda: download(_lib.DeviceCSR.generate(ctx, 500, 400, 8000, 22)))
