"""CPU: the item split of a row-sharded fit, planned from the column counts of the matrix (what the ranks all-reduce),
equals the split planned from the indptr of its transpose."""
import numpy as np
import pytest
import scipy.sparse as sp

from implicit_b200 import synthetic
from implicit_b200.utils import column_splits, nnz_balanced_splits


def cases():
    yield "power_law", synthetic.power_law_csr(3000, 1500, 60000, 3)
    yield "power_law_neg", synthetic.power_law_csr(500, 4000, 9000, 11, negative_fraction=0.2)
    rng = np.random.default_rng(5)
    dense = (rng.random((40, 30)) < 0.1) * rng.random((40, 30))
    dense[::4] = 0     # empty rows
    dense[:, 3::5] = 0  # empty columns
    yield "empty_rows_and_columns", sp.csr_matrix(dense.astype(np.float32))
    yield "empty", sp.csr_matrix((7, 5), dtype=np.float32)


@pytest.mark.parametrize("name,C", list(cases()), ids=lambda v: v if isinstance(v, str) else "")
def test_column_splits_equal_transpose_splits(name, C):
    counts = np.bincount(C.indices, minlength=C.shape[1])
    T = C.T.tocsr()
    for W in (1, 2, 3, 8, C.shape[1] + 3):
        for row_cost in (0, 20, 60):
            got = column_splits(counts, W, row_cost)
            assert np.array_equal(got, nnz_balanced_splits(T.indptr, W, row_cost)), (W, row_cost)
            assert len(got) == W + 1 and got[0] == 0 and got[-1] == C.shape[1] and np.all(np.diff(got) >= 0)
