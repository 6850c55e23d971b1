"""Input-handling helpers with the reference's semantics (implicit/utils.py:65-83, :155-169;
implicit/recommender_base.py:9)."""
import time
import warnings

import numpy as np
import scipy.sparse


class ParameterWarning(Warning):
    """implicit/utils.py:155"""


class ModelFitError(Exception):
    """implicit/recommender_base.py:9"""


def check_csr(user_items):
    """implicit/utils.py:159-169: non-CSR input is converted with a ParameterWarning."""
    if not isinstance(user_items, scipy.sparse.csr_matrix):
        class_name = user_items.__class__.__name__
        start = time.time()
        user_items = user_items.tocsr()
        warnings.warn(
            f"Method expects CSR input, and was passed {class_name} instead. "
            f"Converting to CSR took {time.time() - start} seconds",
            ParameterWarning,
        )
    return user_items


def check_random_state(random_state):
    """implicit/utils.py:65-83: int / None / RandomState / Generator -> np.random.Generator."""
    if isinstance(random_state, np.random.RandomState):
        return np.random.default_rng(random_state.randint(2**31))
    return np.random.default_rng(random_state)


def nnz_balanced_splits(indptr, parts, row_cost=0):
    """Row boundaries [0 = s_0 <= ... <= s_parts = rows] giving every part the same share of
    nnz + row_cost * rows (SURVEY.md section 8(e): nnz-balanced, not row-balanced, shards; row_cost adds the
    per-row fixed work -- the factorisation -- in units of nonzeros)."""
    indptr = np.asarray(indptr, dtype=np.int64)
    rows = len(indptr) - 1
    if row_cost:
        indptr = indptr + row_cost * np.arange(rows + 1, dtype=np.int64)
    nnz = int(indptr[-1] - indptr[0])
    targets = indptr[0] + (nnz * np.arange(1, parts, dtype=np.int64)) // max(parts, 1)
    cuts = np.searchsorted(indptr, targets, side="left")
    splits = np.concatenate([[0], np.clip(cuts, 0, rows), [rows]]).astype(np.int64)
    return np.maximum.accumulate(splits)


def column_splits(col_counts, parts, row_cost=0):
    """nnz_balanced_splits of the transpose, planned from the entries per column of the matrix: the transpose's indptr
    is their running sum."""
    counts = np.asarray(col_counts, dtype=np.int64)
    return nnz_balanced_splits(np.concatenate([[0], np.cumsum(counts)]), parts, row_cost)
