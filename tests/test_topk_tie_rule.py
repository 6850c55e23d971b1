"""The tie rule of select.h (implicit/cpu/select.h:12-39), restated without the heap in tests/helpers.py:select_h, and
the way csrc/topk.cu's by-sort path applies it to a sorted row, both checked on the CPU against the oracle's heap on
small integer rows full of exact ties.  The GPU kernels themselves are covered by tests/test_gpu_topk_widths.py."""
import numpy as np
import pytest

import oracle
from helpers import select_h

NEG = np.float32(-np.finfo(np.float32).max)  # a filtered item (topk.pyx:51-56)


def by_sort_row(s, k):
    """sorted_rows_to_topk_kernel on one row of float32 scores: sort by (score, column) descending, then g (the
    first position scoring T), e (one past the last) and r (the T-items with a column <= c*) by binary search."""
    I = len(s)
    kk = min(k, I)
    order = np.lexsort((-np.arange(I), -s))  # the descending sort of the 64-bit keys (score, column)
    ss, cols = s[order], order
    T = ss[kk - 1]
    g = int(np.searchsorted(-ss[:kk], -T, side="left"))
    e = kk + int(np.searchsorted(-ss[kk:], -T, side="right"))
    m, r = kk - g, kk - g
    if e > kk:
        lo, hi = m, min(kk, e - g)
        while lo < hi:
            c = (lo + hi + 1) // 2
            if c + int((cols[:g] < cols[e - c]).sum()) <= kk:
                lo = c
            else:
                hi = c - 1
        r = lo
    pos = np.concatenate([np.arange(g), np.arange(e - r, e - r + m)])
    ids, out = np.zeros(k, np.int32), np.zeros(k, np.float32)
    ids[:kk], out[:kk] = cols[pos], ss[pos]
    return ids, out


def tie_rows(rng, rows, I):
    """Integer scores in a narrow range (many ties), some entries at -FLT_MAX, and a few all-equal rows."""
    S = rng.integers(-3, 4, size=(rows, I)).astype(np.float32)
    S[rng.random((rows, I)) < rng.random((rows, 1)) * 0.6] = NEG
    S[0] = 0
    S[1] = NEG
    S[2, :] = 1
    S[2, rng.integers(0, I)] = 2
    return S


@pytest.mark.parametrize("I", [1, 2, 3, 7, 16, 33, 100])
def test_select_h_restatement_matches_the_heap(I):
    rng = np.random.default_rng(I)
    S = tie_rows(rng, 300, I)
    for k in sorted({1, 2, 3, I // 2 + 1, I - 1, I, I + 1, I + 7} - {0}):
        eids, esc = oracle.port.select(S, k)
        ids, sc = select_h(S, k)
        np.testing.assert_array_equal(ids, eids, err_msg=f"I={I} k={k}")
        np.testing.assert_array_equal(sc, esc, err_msg=f"I={I} k={k}")


def test_smallest_case_keeps_the_largest_tied_column_below_c_star():
    """Scores [1, 1, 1, 2], k = 2: the heap holds (1, c0), (1, c1) after two columns; c2 does not enter (not strictly
    better) and c3 evicts the smallest column.  The first k of a (score, smaller column first) order would give c0."""
    s = np.array([[1, 1, 1, 2]], dtype=np.float32)
    assert oracle.port.select(s, 2)[0].tolist() == [[3, 1]]
    assert select_h(s, 2)[0].tolist() == [[3, 1]]
    assert by_sort_row(s[0], 2)[0].tolist() == [3, 1]


@pytest.mark.parametrize("I", [1, 5, 33, 257, 1000])
def test_by_sort_decode_matches_the_heap(I):
    rng = np.random.default_rng(100 + I)
    S = tie_rows(rng, 120, I)
    for k in sorted({1, 2, 17, I // 3 + 1, I - 1, I, I + 7} - {0}):
        eids, esc = oracle.port.select(S, k)
        for r in range(len(S)):
            ids, sc = by_sort_row(S[r], k)
            np.testing.assert_array_equal(ids, eids[r], err_msg=f"I={I} k={k} row {r}")
            np.testing.assert_array_equal(sc, esc[r], err_msg=f"I={I} k={k} row {r}")


def test_cold_items_tie_at_zero():
    """An ALS item without interactions solves to exactly zero, so every cold item scores exactly 0 for every user:
    integer factors in -2..2 with 30 % zero item rows, as a 200-factor model would have them."""
    rng = np.random.default_rng(9)
    Y = rng.integers(-2, 3, size=(3000, 200)).astype(np.float32)
    Y[rng.random(3000) < 0.3] = 0
    X = rng.integers(-2, 3, size=(50, 200)).astype(np.float32)
    S = (X.astype(np.float64) @ Y.T.astype(np.float64)).astype(np.float32)  # exact: integers below 2^24
    for k in (10, 1200, 3000):
        eids, esc = oracle.port.select(S, k)
        np.testing.assert_array_equal(select_h(S, k)[0], eids)
        for r in range(0, 50, 7):
            np.testing.assert_array_equal(by_sort_row(S[r], k)[0], eids[r], err_msg=f"k={k} row {r}")
