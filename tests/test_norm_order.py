"""CPU: the summation order the device row norms (als_factors_row_norms) follow is numpy's.  The norms of similar_items
are np.linalg.norm(F, axis=-1), i.e. sqrt(add.reduce(F * F, axis=-1)) with numpy's float32 pairwise summation; the
device kernel emulates that order, and this test pins it against the numpy that is installed, bit for bit, at every
factor width a model can have."""
import numpy as np
import pytest


def pairwise(x):
    """numpy's pairwise float32 sum of x (its add.reduce over a contiguous axis), step by step."""
    n = len(x)
    if n < 8:
        r = np.float32(0)
        for v in x:
            r = np.float32(r + v)
        return r
    if n <= 128:
        r = x[:8].copy()
        i = 8
        while i < n - n % 8:
            r = (r + x[i:i + 8]).astype(np.float32)
            i += 8
        res = np.float32(np.float32(np.float32(r[0] + r[1]) + np.float32(r[2] + r[3])) +
                         np.float32(np.float32(r[4] + r[5]) + np.float32(r[6] + r[7])))
        for v in x[i:]:
            res = np.float32(res + v)
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return np.float32(pairwise(x[:n2]) + pairwise(x[n2:]))


def emulated_norms(F):
    return np.array([np.sqrt(pairwise((r * r).astype(np.float32))) for r in F], dtype=np.float32)


@pytest.mark.parametrize("block", range(8))
def test_pairwise_order_is_numpys(block):
    rng = np.random.default_rng(block)
    for f in range(1 + 128 * block, 129 + 128 * block):
        F = (rng.standard_normal((4, f)) * rng.uniform(1e-3, 1e3, (4, 1))).astype(np.float32)
        F[0] = 0  # a zero row: norm 0 (written as 1e-10 by the callers)
        F[1, ::3] = 0
        want = np.linalg.norm(F, axis=-1)
        assert want.dtype == np.float32
        got = emulated_norms(F)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f
