"""ranking_metrics_at_k from distributed.RowBlocks, the checks that come before any device work: a partial block without
a process group, and blocks that do not tile the rows or whose train and test rows differ on a process group of several
ranks (the all-gather of the block table is stood in for by a group that hands out the other ranks' extents)."""
import numpy as np
import pytest
import scipy.sparse as sp

from implicit_b200.utils import BLOCK_FIELDS


def matrices(users=40, items=30, seed=0):
    train = sp.random(users, items, density=0.2, format="csr", dtype=np.float32, random_state=seed)
    test = sp.random(users, items, density=0.1, format="csr", dtype=np.float32, random_state=seed + 1)
    return train, test


class NoDevice:
    """A context that fails any call but the all-gather; the all-gather returns the other ranks' block extents."""

    def __init__(self, rank, others):
        self.rank, self.others = rank, others

    def allgather_bytes(self, payload):
        rows = list(self.others)
        rows.insert(self.rank, np.frombuffer(payload, dtype=np.int64).reshape(2, len(BLOCK_FIELDS)))
        return np.stack(rows).tobytes()

    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the blocks were checked")


class Group:
    def __init__(self, rank, world, ctx):
        self.rank, self.world, self.ctx = rank, world, ctx


def extents(first, rows, users, items, nnz=0):
    return [first, rows, users, items, nnz, 0]


def test_partial_block_without_a_group_is_refused():
    from implicit_b200 import evaluation
    from implicit_b200.als import AlternatingLeastSquares
    from implicit_b200.distributed import RowBlock

    train, test = matrices()
    model = AlternatingLeastSquares(factors=8)
    with pytest.raises(ValueError, match="every row"):
        evaluation.ranking_metrics_at_k(model, RowBlock(train[5:], 5, 40), RowBlock(test[5:], 5, 40), show_progress=False)
    with pytest.raises(ValueError, match="every row"):
        evaluation.ranking_metrics_at_k(model, RowBlock(train, 0, 40), RowBlock(test[:-1], 0, 40), show_progress=False)
    assert model._ctx is None  # no context was created


@pytest.mark.parametrize("rank", [0, 1, 2])
def test_mismatched_blocks_raise_the_same_error_on_every_rank(rank):
    """W = 3 over 40 rows: rank 1's train block is rows [10, 25), its test block rows [10, 30); every rank checks the
    same table and raises the same ValueError naming rank 1.  A gap in the tiling is refused the same way."""
    from implicit_b200 import evaluation
    from implicit_b200.als import AlternatingLeastSquares
    from implicit_b200.distributed import RowBlock

    train, test = matrices()
    tr = [(0, 10), (10, 15), (25, 15)]
    te = [(0, 10), (10, 20), (30, 10)]
    blocks = [np.array([extents(*tr[p], 40, 30), extents(*te[p], 40, 30)], dtype=np.int64) for p in range(3)]
    others = [b for p, b in enumerate(blocks) if p != rank]
    model = AlternatingLeastSquares(factors=8, process_group=Group(rank, 3, NoDevice(rank, others)))
    (f0, n0), (f1, n1) = tr[rank], te[rank]
    with pytest.raises(ValueError, match="rank 1's train block holds rows"):
        evaluation.ranking_metrics_at_k(model, RowBlock(train[f0:f0 + n0], f0, 40), RowBlock(test[f1:f1 + n1], f1, 40),
                                        show_progress=False)

    gap = [(0, 10), (12, 18), (30, 10)]
    blocks = [np.array([extents(*gap[p], 40, 30), extents(*gap[p], 40, 30)], dtype=np.int64) for p in range(3)]
    others = [b for p, b in enumerate(blocks) if p != rank]
    model = AlternatingLeastSquares(factors=8, process_group=Group(rank, 3, NoDevice(rank, others)))
    f, n = gap[rank]
    with pytest.raises(ValueError, match="train_user_items: rank 1's row block starts at row 12"):
        evaluation.ranking_metrics_at_k(model, RowBlock(train[f:f + n], f, 40), RowBlock(test[f:f + n], f, 40),
                                        show_progress=False)
