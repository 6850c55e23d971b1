"""CPU: how a CSR reaches the device by its size, and how recommend splits a query batch whose already-liked
matrix would reach 2^31 nonzeros."""
import numpy as np
import pytest

from implicit_b200 import _lib, als


def test_upload_route():
    assert _lib.csr_upload_route(0) == "int32"
    assert _lib.csr_upload_route(2**31 - 2) == "int32"  # the largest nnz the int32 upload takes
    assert _lib.csr_upload_route(2**31 - 1) == "int64"
    assert _lib.csr_upload_route(5 * 2**31) == "int64"


def test_liked_batches_cover_all_rows_under_the_limit():
    rng = np.random.default_rng(0)
    lens = rng.integers(0, 50, size=1000)
    indptr = np.concatenate([[0], np.cumsum(lens)])
    for limit in (49, 50, 100, 777, int(indptr[-1]), int(indptr[-1]) + 5):
        b = als.liked_batches(indptr, limit)
        assert b[0][0] == 0 and b[-1][1] == 1000
        assert all(e0 == s1 for (_, e0), (s1, _) in zip(b[:-1], b[1:]))
        sizes = [int(indptr[e] - indptr[s]) for s, e in b]
        assert max(sizes) <= limit
        # greedy: adding the next row to a batch would pass the limit
        assert all(int(indptr[e + 1] - indptr[s]) > limit for s, e in b[:-1])
    assert als.liked_batches(indptr, int(indptr[-1])) == [(0, 1000)]


def test_liked_batches_single_row_at_the_limit():
    indptr = np.array([0, 3, 3 + 2**31 - 2, 2**31 + 5], dtype=np.int64)
    assert als.liked_batches(indptr, 2**31 - 2) == [(0, 1), (1, 2), (2, 3)]
    assert als.liked_batches(np.array([0, 0, 10, 10]), 10) == [(0, 3)]
    with pytest.raises(ValueError, match="row 1"):
        als.liked_batches(np.array([0, 1, 12]), 10)


def test_liked_batches_empty():
    assert als.liked_batches(np.array([0]), 10) == []
