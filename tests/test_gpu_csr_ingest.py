"""Every way a CSR enters the library: the three upload entries, with and without a segment cap, of a whole matrix and
of a row shard whose indptr starts mid-matrix.  Uploads, downloads, transposes and row slices are exact integer
permutations, so each case must reproduce scipy bit for bit and take the expected layout.
"""
import ctypes
import os

import numpy as np
import pytest

from helpers import KNOB_DEFAULTS, mixed_csr
from implicit_b200.utils import CudaArray

pytestmark = pytest.mark.gpu
KNOBS = dict(KNOB_DEFAULTS, segment_nnz=0, host_csr=0)
ENTRIES = ["upload", "upload64_i32", "upload64_i64", "upload_host64"]
SHARD = (150, 480)  # rows of the row-shard cases


@pytest.fixture(scope="module")
def lib():
    set_in_env = sorted(n for n in (f"ALS_B200_{k.upper()}" for k in KNOBS) if n in os.environ)
    if set_in_env:  # the default-cap cases would silently be segmented or host-resident
        pytest.fail(f"knob environment variables are set: {', '.join(set_in_env)}; unset them to run these tests")
    from implicit_b200 import _lib

    return _lib


@pytest.fixture(scope="module")
def ctx(lib):
    c = lib.Context(0)
    yield c
    c.close()


@pytest.fixture(autouse=True)
def knobs(ctx):
    for k, v in KNOBS.items():
        ctx.set_knob(k, v)
    yield
    for k, v in KNOBS.items():
        ctx.set_knob(k, v)


@pytest.fixture(scope="module")
def C():
    return mixed_csr(600, 500, 7, duplicates=True)


def call_upload(lib, ctx, entry, rows, cols, nnz, indptr, indices, data, row_offset):
    """(rc, handle, message) of one entry point, given the arrays as they are (a shard's indptr not rebased)."""
    h = ctypes.c_void_p()
    if entry == "upload":
        rc = ctx.lib.als_csr_upload(ctx.h, rows, cols, nnz, lib.ptr(indptr.astype(np.int32)),
                                    lib.ptr(indices.astype(np.int32)), lib.ptr(data), row_offset, ctypes.byref(h))
    else:
        ix = indices.astype(np.int64 if entry == "upload64_i64" else np.int32)
        fn = ctx.lib.als_csr_upload_host64 if entry == "upload_host64" else ctx.lib.als_csr_upload64
        rc = fn(ctx.h, rows, cols, nnz, lib.ptr(indptr.astype(np.int64)), lib.ptr(ix), ix.dtype.itemsize, lib.ptr(data),
                row_offset, ctypes.byref(h))
    return rc, h, ctx.lib.als_last_error().decode()


def expected_segments(indptr, cap):
    """The segment count of the greedy cut into whole rows of at most `cap` nonzeros (at least one row each)."""
    ip = np.asarray(indptr, dtype=np.int64) - indptr[0]
    rows, a, n = len(ip) - 1, 0, 0
    while a < rows:
        b = max(int(np.searchsorted(ip, ip[a] + cap, side="right")) - 1, a + 1)
        a, n = b, n + 1
    return max(n, 1)


def assert_rows(lib, ctx, d, want):
    """als_csr_download and als_csr_download64 both return `want` exactly."""
    rows, nnz = want.shape[0], want.nnz
    for wide in (False, True):
        ip = np.zeros(rows + 1, dtype=np.int64 if wide else np.int32)
        ix, dv = np.zeros(nnz, dtype=np.int32), np.zeros(nnz, dtype=np.float32)
        fn = ctx.lib.als_csr_download64 if wide else ctx.lib.als_csr_download
        lib.check(fn(ctx.h, d.h, lib.ptr(ip), lib.ptr(ix), lib.ptr(dv)))
        assert np.array_equal(ip, want.indptr) and np.array_equal(ix, want.indices), wide
        assert np.array_equal(dv, want.data), wide


@pytest.mark.parametrize("shard", [False, True], ids=["whole", "shard"])
@pytest.mark.parametrize("capped", [False, True], ids=["cap0", "cap_thirds"])
@pytest.mark.parametrize("entry", ENTRIES)
def test_ingest(lib, ctx, C, entry, capped, shard):
    r0, r1 = SHARD if shard else (0, C.shape[0])
    want = C[r0:r1]
    cap = want.nnz // 3 if capped else 0
    ctx.set_knob("segment_nnz", cap)
    host = entry == "upload_host64"
    rc, h, msg = call_upload(lib, ctx, entry, r1 - r0, C.shape[1], want.nnz, C.indptr[r0:r1 + 1], C.indices, C.data, r0)
    assert rc == 0, msg
    d = lib.DeviceCSR(ctx, h)
    assert d.host_resident == host
    assert d.segment_count == (expected_segments(want.indptr, cap) if capped else 1)
    if capped:
        assert d.segment_count > 1
    assert d.shape3 == (r1 - r0, C.shape[1], want.nnz)
    assert_rows(lib, ctx, d, want)

    if shard:
        with pytest.raises(lib.AlsError, match="row shards cannot be transposed"):
            d.transpose()
    else:
        t = d.transpose()
        assert t.host_resident == host
        T = C.T.tocsr()
        assert t.segment_count == (expected_segments(T.indptr, cap) if capped else 1)
        assert_rows(lib, ctx, t, T)
        t.close()

    if not shard and not host:
        # slices that cross the end of the first segment (or the middle of an unsegmented CSR)
        first_end = int(np.searchsorted(C.indptr, cap, side="right")) - 1 if capped else 300
        assert 10 < first_end < C.shape[0] - 40
        for a, b in ((0, first_end + 5), (first_end - 7, first_end + 40), (first_end - 3, C.shape[0])):
            s = d.slice_rows(a, b)
            assert s.shape3 == (b - a, C.shape[1], int(C.indptr[b] - C.indptr[a]))
            assert_rows(lib, ctx, s, C[a:b])
            s.close()
    d.close()


@pytest.mark.parametrize("entry", ENTRIES)
def test_refusals(lib, ctx, C, entry):
    who = {"upload": "als_csr_upload", "upload_host64": "als_csr_upload_host64"}.get(entry, "als_csr_upload64")
    nm = C.indptr.copy()
    nm[100] = nm[101] + 1
    cases = [((nm, C.nnz), f"{who}: indptr is not monotone at row 100"),
             ((C.indptr, C.nnz - 1), f"{who}: indptr[rows] - indptr[0] = {C.nnz} != nnz = {C.nnz - 1}")]
    for (ip, nnz), want in cases:
        rc, _, msg = call_upload(lib, ctx, entry, C.shape[0], C.shape[1], nnz, ip, C.indices, C.data, 0)
        assert rc == lib.ALS_E_INVALID and msg == want


EDGES = ["nnz0", "rows0", "cols1", "cols65536", "cols65537", "column3072", "column3073", "unsorted"]


def edge_csr(name):
    """A CSR at an edge of the transpose of a one-segment device CSR: no entries, no rows, one column, the column counts
    around 2^16 where the radix sort takes one more bit, a column of 3072 entries (the longest transposed row the
    schedule keeps whole) or 3073 (chunked), else 4000 random entries.  Each row keeps its entries in the order drawn:
    unsorted, with repeated columns."""
    import scipy.sparse as sp

    rng = np.random.default_rng(5)
    rows, cols, n = (3200 if name.startswith("column") else 500), 300, 4000
    if name in ("nnz0", "rows0"):
        rows, n = (0 if name == "rows0" else rows), 0
    elif name.startswith("cols"):
        cols = int(name[4:])
    r, c = (rng.integers(0, rows, n), rng.integers(0, cols, n)) if n else (np.zeros(0, np.int64), np.zeros(0, np.int64))
    if name.startswith("cols"):
        c[0] = cols - 1
    elif name.startswith("column"):  # column 7 holds exactly that many entries, in distinct rows
        m = int(name[6:])
        c[c == 7] = 8
        r, c = np.concatenate([r, rng.permutation(rows)[:m]]), np.concatenate([c, np.full(m, 7)])
    order = np.argsort(r, kind="stable")
    indptr = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=rows))]).astype(np.int32)
    data = (1 + 4 * rng.random(len(r))).astype(np.float32)
    C = sp.csr_matrix((data, c[order].astype(np.int32), indptr), shape=(rows, cols))
    if name == "unsorted":
        merged = C.copy()
        merged.sum_duplicates()
        assert not C.has_sorted_indices and merged.nnz < C.nnz
    return C


@pytest.mark.parametrize("name", EDGES)
def test_device_transpose_edges(lib, ctx, name):
    """The transpose of a one-segment device CSR is scipy's, and complete when the call returns: solves over it, made
    after the input is destroyed and after a second transpose, and its use at once as a liked filter (top-k and
    restrict_columns) give bitwise what the upload of scipy's transpose gives."""
    C = edge_csr(name)
    T = C.T.tocsr()
    f, reg, k = 32, 0.1, 10  # 32 factors: no top-k batch takes the wgmma kernel, which needs 64
    rng = np.random.default_rng(6)
    X0 = rng.standard_normal((T.shape[0], f), dtype=np.float32)
    Y = lib.DeviceFactors.from_host(ctx, rng.standard_normal((T.shape[1], f), dtype=np.float32))
    subset = np.sort(rng.choice(T.shape[1], T.shape[1] // 2, replace=False)).astype(np.int32)
    sub = lib.DeviceSnapshot.from_host(ctx, subset) if len(subset) else None
    sub_ids = sub.cuda() if sub is not None else CudaArray(0, (0,), 4, 1, 0)
    Q = lib.DeviceFactors.from_host(ctx, X0)
    u = lib.DeviceCSR.upload(ctx, T)
    d = lib.DeviceCSR.upload(ctx, C)
    assert d.segment_count == 1 and not d.host_resident

    liked = d.transpose()
    got, want = lib.topk(ctx, Y, Q, k, liked=liked), lib.topk(ctx, Y, Q, k, liked=u)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    r_got, r_want = liked.restrict_columns(sub_ids), u.restrict_columns(sub_ids)
    assert_rows(lib, ctx, r_got, r_want.download())

    t, t2 = d.transpose(), d.transpose()
    d.close()
    for use_cg in (False, True):
        out = []
        for m in (t, u):
            X = lib.DeviceFactors.from_host(ctx, X0)
            if use_cg:
                lib.least_squares_cg(ctx, m, X, Y, reg)
            else:
                lib.least_squares(ctx, m, X, Y, reg)
            out.append(X.download())
            X.close()
        assert np.array_equal(out[0], out[1]), "cg" if use_cg else "cholesky"
    for h in (liked, t, t2):
        assert h.segment_count == 1 and not h.host_resident
        assert_rows(lib, ctx, h, T)
    for h in (liked, t, t2, u, r_got, r_want, Q, Y) + ((sub,) if sub is not None else ()):
        h.close()
