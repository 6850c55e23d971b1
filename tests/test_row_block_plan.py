"""CPU-only: the planning of a multi-GPU fit from row blocks.  The user split the ranks agree on from the block table and
their own indptrs (block_cuts, summed) must be exactly nnz_balanced_splits of the whole indptr, the split of a fit from
the whole matrix; a malformed table must raise the same ValueError on every rank; row_block must tile the rows."""
import numpy as np
import pytest

from implicit_b200.distributed import row_block
from implicit_b200.utils import (BLOCK_FIELDS, block_cuts, check_block_table, nnz_balanced_splits,
                                 simulate_block_splits)


def table_of(indptr, bounds, items=7):
    """The block table of ranks holding rows [bounds[p], bounds[p + 1]) of a matrix with this indptr, and their local
    indptrs (offset like a slice of scipy's, which need not start at 0)."""
    users = len(indptr) - 1
    rows = [(bounds[p], bounds[p + 1] - bounds[p], users, items, int(indptr[bounds[p + 1]] - indptr[bounds[p]]), 0)
            for p in range(len(bounds) - 1)]
    return np.array(rows, dtype=np.int64), [indptr[bounds[p]:bounds[p + 1] + 1] for p in range(len(bounds) - 1)]


def random_bounds(rng, users, W, empty=()):
    """Uneven block boundaries; the ranks in `empty` hold no rows."""
    inner = np.sort(rng.integers(0, users + 1, size=W - 1))
    bounds = np.concatenate([[0], inner, [users]]).astype(np.int64)
    for p in empty:
        if p == W - 1:
            bounds[p] = users
        else:
            bounds[p + 1] = bounds[p]
    return np.maximum.accumulate(bounds)


def indptr_of(rng, users, kind):
    if kind == "empty":
        lengths = np.zeros(users, dtype=np.int64)
    elif kind == "giant":  # a few rows hold most nonzeros: several targets fall in one row
        lengths = rng.integers(0, 4, size=users)
        giants = rng.choice(users, min(users, 3), replace=False)
        lengths[giants] = rng.integers(500, 5000, size=len(giants))
    else:
        lengths = rng.zipf(1.6, size=users).clip(max=300) * rng.integers(0, 2, size=users)
    return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)


@pytest.mark.parametrize("row_cost", [0, 20, 60])
@pytest.mark.parametrize("W", [1, 2, 3, 8])
@pytest.mark.parametrize("kind", ["random", "giant", "empty"])
def test_block_split_is_the_whole_matrix_split(W, row_cost, kind):
    rng = np.random.default_rng(W * 100 + row_cost + len(kind))
    for users in (0, 1, 5, 37, 400):
        indptr = indptr_of(rng, users, kind)
        want = nnz_balanced_splits(indptr, W, row_cost)
        cases = [random_bounds(rng, users, W) for _ in range(12)]
        cases.append(np.array([0] + [users] * W))         # the first rank holds everything
        cases.append(np.array([0] * W + [users]))         # the last rank holds everything
        cases.append(np.linspace(0, users, W + 1).astype(np.int64))
        if W > 2:
            cases += [random_bounds(rng, users, W, empty=(0,)), random_bounds(rng, users, W, empty=(W - 1,)),
                      random_bounds(rng, users, W, empty=(W // 2,))]
        for bounds in cases:
            table, ips = table_of(indptr, bounds)
            got = simulate_block_splits(table, ips, row_cost)
            assert np.array_equal(got, want), (users, bounds, got, want)


@pytest.mark.parametrize("row_cost", [0, 20, 60])
@pytest.mark.parametrize("W", [2, 3, 8])
def test_targets_on_block_boundaries(W, row_cost):
    """Blocks cut exactly where nnz_balanced_splits cuts (and one row either side): every target lies on, or next to,
    a block boundary."""
    rng = np.random.default_rng(W + row_cost)
    indptr = indptr_of(rng, 300, "random")
    want = nnz_balanced_splits(indptr, W, row_cost)
    for shift in (-1, 0, 1):
        bounds = np.clip(want + shift, 0, 300)
        bounds[0], bounds[-1] = 0, 300
        bounds = np.maximum.accumulate(bounds)
        table, ips = table_of(indptr, bounds)
        assert np.array_equal(simulate_block_splits(table, ips, row_cost), want), (shift, bounds)


def test_each_target_has_one_owner():
    """Every inner cut comes from exactly one rank (or none, when it is 0): the sum over ranks adds no two cuts."""
    rng = np.random.default_rng(5)
    indptr = indptr_of(rng, 200, "random")
    for W in (2, 3, 8):
        table, ips = table_of(indptr, random_bounds(rng, 200, W))
        parts = np.array([block_cuts(table, ip, p, 20) for p, ip in enumerate(ips)])
        assert ((parts != 0).sum(axis=0) <= 1).all()


def bad_tables():
    """(name, table, rank the error names): every malformed table a set of ranks can send."""
    good = np.array([(0, 3, 10, 4, 5, 0), (3, 0, 10, 4, 0, 0), (3, 7, 10, 4, 9, 0)], dtype=np.int64)

    def edit(p, field, value):
        t = good.copy()
        t[p, BLOCK_FIELDS.index(field)] = value
        return t

    return [
        ("gap", edit(2, "first_row", 4), 2),
        ("overlap", edit(2, "first_row", 2), 2),
        ("out_of_order", np.array([good[0], (3, 7, 10, 4, 9, 0), (10, 0, 10, 4, 0, 0)])[[0, 2, 1]], 1),
        ("short", edit(2, "rows", 6), 2),
        ("users", edit(1, "users", 11), 1),
        ("items", edit(2, "items", 5), 2),
        ("past_the_end", edit(2, "rows", 8), 2),
        ("negative_first_row", np.array([(-1, 4, 10, 4, 5, 0), (3, 7, 10, 4, 9, 0)]), 0),
    ]


@pytest.mark.parametrize("name,table,rank", bad_tables(), ids=[b[0] for b in bad_tables()])
def test_bad_table_raises_the_same_error_on_every_rank(name, table, rank):
    messages = set()
    for _ in range(len(table)):  # every rank checks the same all-gathered table
        with pytest.raises(ValueError, match=f"rank {rank}'s row block") as e:
            check_block_table(table.copy())
        messages.add(str(e.value))
    assert len(messages) == 1


def test_good_table_totals():
    table = np.array([(0, 3, 10, 4, 5, 0), (3, 0, 10, 4, 0, 0), (3, 7, 10, 4, 9, 0)], dtype=np.int64)
    assert check_block_table(table) == (10, 4, 14)
    assert check_block_table(np.array([(0, 0, 0, 4, 0, 0)])) == (0, 4, 0)


@pytest.mark.parametrize("W", [1, 2, 3, 8, 13])
@pytest.mark.parametrize("users", [0, 1, 5, 12, 1001])
def test_row_block_tiles_the_rows(users, W):
    blocks = [row_block(users, r, W) for r in range(W)]
    assert blocks[0][0] == 0 and blocks[-1][1] == users
    for (a0, a1), (b0, _) in zip(blocks, blocks[1:]):
        assert a0 <= a1 == b0
    sizes = [b - a for a, b in blocks]
    assert max(sizes) - min(sizes) <= 1


def test_row_block_refuses_bad_ranks():
    with pytest.raises(ValueError):
        row_block(10, 3, 3)
    with pytest.raises(ValueError):
        row_block(10, 0, 0)
