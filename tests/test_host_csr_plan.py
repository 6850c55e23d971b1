"""CPU-only: where fit() keeps Cui / Ciu (implicit_b200._lib.csr_residency), at the edges of its memory count."""
import pytest

from implicit_b200 import _lib

GIB = 1 << 30


def need(users, items, nnz, factors):
    """The smallest free byte count that keeps the pair on the device: the function's own threshold, found by bisection."""
    lo, hi = 0, 1 << 50
    while lo < hi:
        mid = (lo + hi) // 2
        if _lib.csr_residency(users, items, nnz, factors, mid) == "device":
            hi = mid
        else:
            lo = mid + 1
    return lo


def test_threshold_is_sharp():
    n = need(1000, 500, 10_000, 64)
    assert _lib.csr_residency(1000, 500, 10_000, 64, n) == "device"
    assert _lib.csr_residency(1000, 500, 10_000, 64, n - 1) == "host"


def test_small_matrix_counts_the_fixed_margin():
    # one nonzero, one row, one column: the 1 GiB for scratch and fragmentation dominates
    n = need(1, 1, 1, 1)
    assert GIB < n < GIB + 4096
    assert _lib.csr_residency(1, 1, 1, 1, GIB) == "host"


def test_empty_matrix():
    assert _lib.csr_residency(0, 0, 0, 16, 2 * GIB) == "device"
    assert _lib.csr_residency(0, 0, 0, 16, 0) == "host"


def test_both_orientations_and_the_transpose_temporaries():
    # below 2^31 - 1 nonzeros the transpose sorts the whole matrix: 16 + 20 bytes per nonzero
    nnz = 1_000_000_000
    n = need(1000, 1000, nnz, 16)
    assert 36 * nnz < n < 36 * nnz + 2 * GIB
    # above it the sorts go by pieces of 2^28 nonzeros: 16 bytes per nonzero plus one piece
    nnz = 4_000_000_000
    n = need(1000, 1000, nnz, 16)
    assert 16 * nnz + 20 * 2**28 < n < 16 * nnz + 20 * 2**28 + 2 * GIB


def test_one_h100_limit():
    # 80 GB of HBM holds a 2.159 B-nonzero fit (C2-like shape, f = 64) but not a 5.4 B one
    free = 79 * 10**9
    assert _lib.csr_residency(40000 * 127, 20000 * 127, 2_159_000_000, 64, free) == "device"
    assert _lib.csr_residency(40000 * 320, 20000 * 320, 5_440_000_000, 64, free) == "host"


@pytest.mark.parametrize("factors,ld", [(1, 16), (16, 16), (17, 32), (100, 112), (128, 128), (129, 256), (1024, 1024)])
def test_factor_matrices_use_the_padded_width(factors, ld):
    users, items = 1_000_000, 500_000
    base = need(users, items, 0, 16)
    # X, Y and two whitened copies of the larger side, at the device row stride
    extra = 4 * (ld - 16) * (users + items) + 2 * 4 * (ld - 16) * max(users, items)
    assert need(users, items, 0, factors) == base + extra


def test_more_free_memory_never_moves_to_host():
    for nnz in (0, 10**6, 3 * 10**9):
        n = need(10**6, 10**5, nnz, 64)
        for free in (n, n + 1, 2 * n, 1 << 50):
            assert _lib.csr_residency(10**6, 10**5, nnz, 64, free) == "device"
