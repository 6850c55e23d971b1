"""Inputs and outputs in CUDA memory: a CSR whose arrays live on the device (a torch.sparse_csr_tensor, or a CuPy-like
object exposing __cuda_array_interface__), factors assigned from CUDA tensors and device snapshots of the factors.

A device CSR is copied on the device into the same layout as the scipy CSR it equals, so every fit, solve and top-k
from it must give bitwise the results of the scipy call.  PyTorch plays the producer; the package itself never imports
it.
"""
import gc
import os
import types

import numpy as np
import pytest
import scipy.sparse as sp

from helpers import KNOB_DEFAULTS, mixed_csr

torch = pytest.importorskip("torch")

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs PyTorch with CUDA as the producer")]
REG = 0.1


class Cai:
    """A tensor behind an interface dict of our choosing (a CuPy array would export version 3 with its stream)."""

    def __init__(self, t, **override):
        self.t = t
        self.__cuda_array_interface__ = dict(t.__cuda_array_interface__, **override)


class CaiCSR:
    """What fit() sees of a cupyx.scipy.sparse.csr_matrix: shape and three arrays exposing the interface."""

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
    c.set_knob("segment_nnz", 0)
    c.close()


@pytest.fixture(scope="module")
def C():
    """Unsorted rows, duplicates, stored zeros, negative confidences, empty rows and rows past the giant-row split."""
    C = mixed_csr(600, 500, 7, duplicates=True)
    assert not C.has_sorted_indices and (C.data == 0).any() and (C.data < 0).any() and (np.diff(C.indptr) == 0).any()
    return C


def scipy_csr(C, index_dtype, value_dtype, seed=3):
    """C with values of value_dtype (fp64 values get bits below fp32's resolution, so that the device cast has something
    to round) and indices of index_dtype where scipy keeps them (it narrows indices that fit int32)."""
    data = C.data.astype(value_dtype)
    if value_dtype == np.float64:
        data = data + np.random.default_rng(seed).uniform(-1e-7, 1e-7, len(data)) * data
    return sp.csr_matrix((data, C.indices.astype(index_dtype), C.indptr.astype(index_dtype)), shape=C.shape)


def as_float32(M):
    """The float32 scipy CSR of M's values rounded, entry for entry.  (scipy's astype would also merge M's duplicates
    and sort its rows, which a device CSR of fp64 values does not.)"""
    return sp.csr_matrix((M.data.astype(np.float32), M.indices, M.indptr), shape=M.shape)


def device_csr(M, kind, index_dtype=None):
    """M (scipy) in CUDA memory, its indptr and indices of index_dtype (default: M's): a torch.sparse_csr_tensor, or a
    CaiCSR of torch tensors."""
    index_dtype = index_dtype or M.indices.dtype
    ip, ix, v = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in
                 (M.indptr.astype(index_dtype), M.indices.astype(index_dtype), M.data))
    if kind == "torch":
        return torch.sparse_csr_tensor(ip, ix, v, size=M.shape)
    return CaiCSR(ip, ix, v, M.shape)


def model(ctx, f, use_cg, alpha=1.0, iterations=2):
    from implicit_b200 import AlternatingLeastSquares

    m = AlternatingLeastSquares(factors=f, iterations=iterations, use_cg=use_cg, regularization=REG, alpha=alpha,
                                random_state=1)
    m._ctx = ctx
    return m


def fit(ctx, M, f, use_cg, X0, Y0, alpha=1.0):
    m = model(ctx, f, use_cg, alpha)
    m.user_factors, m.item_factors = X0, Y0
    m.fit(M, show_progress=False)
    return m.user_factors.copy(), m.item_factors.copy()


def initial(M, f, seed=5):
    rng = np.random.default_rng(seed)
    return (rng.random((M.shape[0], f), dtype=np.float32) * np.float32(0.01),
            rng.random((M.shape[1], f), dtype=np.float32) * np.float32(0.01))


SOLVERS = [(False, 16), (False, 64), (False, 128), (True, 16), (True, 64), (True, 128), (True, 192)]
# (container, index dtype, value dtype, alpha)
INPUTS = [("torch", np.int32, np.float32, 1.0), ("torch", np.int64, np.float64, 2.5), ("cai", np.int32, np.float64, 1.0),
          ("cai", np.int64, np.float32, 0.75)]


@pytest.mark.parametrize("use_cg,f", SOLVERS)
@pytest.mark.parametrize("kind,index_dtype,value_dtype,alpha", INPUTS)
def test_fit_from_device_csr_bitwise(ctx, C, use_cg, f, kind, index_dtype, value_dtype, alpha):
    M = scipy_csr(C, index_dtype, value_dtype)
    X0, Y0 = initial(M, f)
    want = fit(ctx, as_float32(M), f, use_cg, X0, Y0, alpha)
    D = device_csr(M, kind, index_dtype)
    ix = D.indices if kind == "cai" else D.col_indices()
    assert ix.element_size() == np.dtype(index_dtype).itemsize
    got = fit(ctx, D, f, use_cg, X0, Y0, alpha)
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("use_cg", [False, True])
def test_fit_from_segmented_device_csr_bitwise(ctx, C, use_cg):
    """The same knob as ALS_B200_SEGMENT_NNZ, set on the live context: the device CSR is cut into row-block segments."""
    from implicit_b200 import _lib

    M = scipy_csr(C, np.int64, np.float64)
    D = device_csr(M, "torch", np.int64)
    M = as_float32(M)
    X0, Y0 = initial(M, 64)
    want = fit(ctx, M, 64, use_cg, X0, Y0)
    ctx.set_knob("segment_nnz", M.nnz // 3)
    try:
        d = _lib.DeviceCSR.from_device(ctx, D)
        got = d.download()
        assert d.segment_count >= 3 and np.array_equal(got.indices, M.indices) and np.array_equal(got.data, M.data)
        d.close()
        seg = fit(ctx, M, 64, use_cg, X0, Y0)
        got = fit(ctx, D, 64, use_cg, X0, Y0)
    finally:
        ctx.set_knob("segment_nnz", 0)
    for a, b, c in zip(got, seg, want):
        assert np.array_equal(a, b) and np.array_equal(a, c)


def test_device_csr_is_copied_not_aliased(ctx, C):
    from implicit_b200 import _lib

    M = scipy_csr(C, np.int32, np.float32)
    D = device_csr(M, "cai")
    d = _lib.DeviceCSR.from_device(ctx, D)
    D.data.zero_()
    D.indices.fill_(-1)
    torch.cuda.synchronize()
    assert not d.host_resident
    got = d.download()
    assert np.array_equal(got.indptr, M.indptr) and np.array_equal(got.indices, M.indices)
    assert np.array_equal(got.data, M.data)


# ---- refusals: what als_csr_upload64 refuses, named the same way ------------------------------------------------
def host_arrays(M):
    return np.ascontiguousarray(M.indptr, dtype=np.int64), np.ascontiguousarray(M.indices), \
        np.ascontiguousarray(M.data, dtype=np.float32)


def upload64_message(ctx, M, indptr, indices, nnz):
    import ctypes

    from implicit_b200 import _lib

    h = ctypes.c_void_p()
    data = np.ascontiguousarray(M.data, dtype=np.float32)
    rc = ctx.lib.als_csr_upload64(ctx.h, M.shape[0], M.shape[1], nnz, _lib.ptr(indptr), _lib.ptr(indices),
                                  indices.dtype.itemsize, _lib.ptr(data), 0, ctypes.byref(h))
    assert rc == _lib.ALS_E_INVALID
    return ctx.lib.als_last_error().decode()


def refused(ctx, D, use_cg=False):
    m = model(ctx, 16, use_cg)
    with pytest.raises(ValueError) as e:
        m.fit(D, show_progress=False)
    return str(e.value)


def same_words(device_msg, host_msg):
    assert device_msg.startswith("als_csr_upload_device: ") and host_msg.startswith("als_csr_upload64: ")
    assert device_msg.split(": ", 1)[1] == host_msg.split(": ", 1)[1], (device_msg, host_msg)


@pytest.mark.parametrize("index_dtype", [np.int32, np.int64])
def test_refuses_an_index_out_of_range(ctx, C, index_dtype):
    from implicit_b200 import _lib

    M = scipy_csr(C, index_dtype, np.float32)
    ip, ix, _ = host_arrays(M)
    ix = ix.astype(index_dtype)
    for pos, v in ((int(ip[123]) + 1, M.shape[1]), (M.nnz - 1, -3)):
        bad = ix.copy()
        bad[pos] = v
        Mb = types.SimpleNamespace(shape=M.shape, indptr=ip, indices=bad, data=M.data)
        with pytest.raises(ValueError) as host:
            _lib.DeviceCSR.upload_rows(ctx, Mb, 0, M.shape[0])
        dev = refused(ctx, CaiCSR(torch.from_numpy(ip).cuda(), torch.from_numpy(bad.astype(index_dtype)).cuda(),
                                  torch.from_numpy(M.data).cuda(), M.shape))
        same_words(dev, str(host.value))
        assert f"indices[{pos}] = {v} is outside [0, {M.shape[1]})" in dev


def test_refuses_a_non_monotone_indptr(ctx, C):
    from implicit_b200 import _lib

    M = scipy_csr(C, np.int32, np.float32)
    ip, ix, v = host_arrays(M)
    nm = ip.copy()
    nm[100] = nm[101] + 1
    Mb = types.SimpleNamespace(shape=M.shape, indptr=nm, indices=ix, data=v)
    with pytest.raises(ValueError) as host:
        _lib.DeviceCSR.upload_rows(ctx, Mb, 0, M.shape[0])
    dev = refused(ctx, device_csr(types.SimpleNamespace(shape=M.shape, indptr=nm, indices=ix, data=v), "torch"))
    same_words(dev, str(host.value))
    assert "indptr is not monotone at row 100" in dev


def test_refuses_an_nnz_mismatch(ctx, C):
    M = scipy_csr(C, np.int64, np.float32)
    ip, ix, v = host_arrays(M)
    short = ip.copy()
    short[-1] -= 1  # the arrays hold one entry more than the indptr counts
    host = upload64_message(ctx, M, short, ix, M.nnz)
    dev = refused(ctx, CaiCSR(torch.from_numpy(short).cuda(), torch.from_numpy(ix).cuda(), torch.from_numpy(v).cuda(),
                              M.shape))
    same_words(dev, host)
    assert f"= {M.nnz - 1} != nnz = {M.nnz}" in dev


def test_refuses_host_memory_strided_indices_and_a_mask(ctx, C):
    M = scipy_csr(C, np.int64, np.float32)
    ip, ix, v = (torch.from_numpy(a).cuda() for a in host_arrays(M))
    host_ix = np.ascontiguousarray(M.indices, dtype=np.int64)
    fake = types.SimpleNamespace(__cuda_array_interface__=dict(shape=host_ix.shape, typestr="<i8", strides=None,
                                                               data=(host_ix.ctypes.data, False), version=3))
    msg = refused(ctx, CaiCSR(ip, fake, v, M.shape))
    assert "indices is not device memory" in msg
    wide = torch.stack([ix, ix], 1).reshape(-1)
    msg = refused(ctx, CaiCSR(ip, wide[::2], v, M.shape))
    assert "indices" in msg and "not contiguous" in msg
    msg = refused(ctx, CaiCSR(ip, ix, Cai(v, mask=Cai(v).__cuda_array_interface__), M.shape))
    assert "data" in msg and "mask" in msg
    # the host path is untouched by the device one: the same matrix from scipy fits
    model(ctx, 16, False).fit(M, show_progress=False)


def test_producer_stream_is_honoured(ctx, C):
    """The values are written on a side stream behind a long sleep, and fit() is called at once: it must wait."""
    M = scipy_csr(C, np.int32, np.float32)
    X0, Y0 = initial(M, 64)
    want = fit(ctx, M, 64, False, X0, Y0)
    ip, ix, truth = (torch.from_numpy(a).cuda() for a in host_arrays(M))
    v = torch.zeros_like(truth)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)  # some 0.1 s of spinning before the values land
        v.copy_(truth)
    s = side.cuda_stream
    D = CaiCSR(Cai(ip, version=3, stream=s), Cai(ix, version=3, stream=s), Cai(v, version=3, stream=s), M.shape)
    got = fit(ctx, D, 64, False, X0, Y0)
    torch.cuda.synchronize()
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


# ---- factors from and to CUDA memory ----------------------------------------------------------------------------
@pytest.mark.parametrize("use_cg,f", [(False, 64), (True, 40), (True, 192)])
def test_factor_assignment_from_cuda_tensors(ctx, C, use_cg, f):
    M = scipy_csr(C, np.int32, np.float32)
    X0, Y0 = initial(M, f)
    want = fit(ctx, M, f, use_cg, X0, Y0)
    got = fit(ctx, M, f, use_cg, torch.from_numpy(X0).cuda(), torch.from_numpy(Y0).cuda())
    wide_x = torch.full((X0.shape[0], f + 7), float("nan"), device="cuda")
    wide_y = torch.full((Y0.shape[0], f + 33), float("nan"), device="cuda")
    wide_x[:, :f] = torch.from_numpy(X0)
    wide_y[:, :f] = torch.from_numpy(Y0)
    strided = fit(ctx, M, f, use_cg, wide_x[:, :f], wide_y[:, :f])
    for a, b, c in zip(got, strided, want):
        assert np.array_equal(a, c) and np.array_equal(b, c)
    m = model(ctx, f, use_cg)
    m.user_factors = wide_x[:, :f]
    assert np.array_equal(m.user_factors, X0)  # the lazy download of an assigned device array
    m.item_factors = torch.zeros((3, f + 1), device="cuda")
    with pytest.raises(ValueError, match="do not match"):
        m.fit(M, show_progress=False)
    with pytest.raises(ValueError, match="typestr"):
        m.user_factors = torch.zeros((3, f), dtype=torch.float64, device="cuda")


def test_factor_snapshots(ctx, C):
    M = scipy_csr(C, np.int32, np.float32)
    X0, Y0 = initial(M, 40)
    m = model(ctx, 40, True)
    m.user_factors, m.item_factors = X0, Y0
    m.fit(M, show_progress=False)
    s = m.user_factors_device
    cai = s.__cuda_array_interface__
    assert cai["shape"] == (M.shape[0], 40) and cai["strides"] == (4 * 48, 4) and cai["typestr"] == "<f4"
    assert cai["version"] == 3 and cai["stream"] is None
    u = torch.as_tensor(s, device="cuda")
    i = torch.as_tensor(m.item_factors_device, device="cuda")
    del s
    gc.collect()
    assert np.array_equal(u.cpu().numpy(), m.user_factors) and np.array_equal(i.cpu().numpy(), m.item_factors)
    before = u.cpu().numpy().copy()
    m.fit(M * np.float32(2), show_progress=False)
    assert not np.array_equal(m.user_factors, before)
    assert np.array_equal(u.cpu().numpy(), before)
    del m
    gc.collect()
    assert np.array_equal(u.cpu().numpy(), before)  # the snapshot outlives the model


# ---- the other entry points -------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fitted(ctx, C):
    M = abs(scipy_csr(C, np.int32, np.float32))
    M.data += np.float32(1)
    m = model(ctx, 64, False, alpha=2.0, iterations=3)
    m.fit(M, show_progress=False)
    return m, M


@pytest.mark.parametrize("recalculate_user", [False, True])
@pytest.mark.parametrize("kind", ["torch", "cai"])
def test_recommend_with_device_user_items(fitted, kind, recalculate_user):
    m, M = fitted
    users = np.arange(17, 317)
    rows = M[users]
    want = m.recommend(users, rows, N=12, recalculate_user=recalculate_user)
    got = m.recommend(users, device_csr(rows, kind), N=12, recalculate_user=recalculate_user)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    one = m.recommend(5, device_csr(M[5], kind), N=7, recalculate_user=recalculate_user)
    ref = m.recommend(5, M[5], N=7, recalculate_user=recalculate_user)
    assert np.array_equal(one[0], ref[0]) and np.array_equal(one[1], ref[1])


@pytest.mark.parametrize("kind", ["torch", "cai"])
def test_recalculate_and_partial_fit_with_device_csrs(ctx, fitted, kind):
    m, M = fitted
    users = np.arange(0, 300)
    assert np.array_equal(m.recalculate_user(users, device_csr(M[users], kind)), m.recalculate_user(users, M[users]))
    Mt = M.T.tocsr()
    assert np.array_equal(m.recalculate_item(9, device_csr(Mt[9], kind)), m.recalculate_item(9, Mt[9]))
    Mt = Mt[:50]
    Mt = sp.csr_matrix((Mt.data, Mt.indices, Mt.indptr), shape=(50, 640))  # the 40 new users' columns, empty
    out = []
    for wrap in (lambda x: x, lambda x: device_csr(x, kind, np.int64)):
        p = model(ctx, 64, False, alpha=2.0)
        p.user_factors, p.item_factors = m.user_factors, m.item_factors
        p.partial_fit_users(np.arange(590, 640), wrap(M[:50]))  # 40 new users
        p.partial_fit_items(np.arange(480, 530), wrap(Mt))  # 30 new items
        out.append((p.user_factors.copy(), p.item_factors.copy()))
    for a, b in zip(*out):
        assert np.array_equal(a, b)


def test_unsupported_places_refuse_a_device_csr(ctx, fitted):
    from implicit_b200 import evaluation
    from implicit_b200.distributed import RowBlock

    m, M = fitted
    D = device_csr(M, "torch")
    with pytest.raises(ValueError, match="CUDA memory"):
        evaluation.ranking_metrics_at_k(m, D, M, K=5, show_progress=False)
    with pytest.raises(ValueError, match="CUDA memory"):
        evaluation.train_test_split(D)
    with pytest.raises(ValueError, match="CUDA memory"):
        model(ctx, 64, False).fit(RowBlock(D, 0, M.shape[0]), show_progress=False)
    with pytest.raises(ValueError, match="items="):
        m.recommend(np.arange(3), device_csr(M[:3], "torch"), items=np.arange(10))
