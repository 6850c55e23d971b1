"""Ranking evaluation: the main batch consumer of ``recommend`` (SURVEY.md section 8(f) N4).

Mirrors ``implicit.evaluation`` (implicit/evaluation.pyx): ``ranking_metrics_at_k`` :366-475 and its four
single-metric wrappers :236-363, plus ``train_test_split`` :14-48.  The reference walks the users in
batches of 1000 through ``model.recommend`` and scores each returned id against an ``unordered_set`` of
the user's withheld items in a scalar loop.  Here the batches are sized for the fused top-k kernel (one
launch covers ``BATCH`` users) and the per-user bookkeeping is whole-batch array arithmetic on the
returned ``(users, K)`` id matrix; the four sums are the same quantities, accumulated in float64.

For this package's ``AlternatingLeastSquares`` the ids never leave the device: each batch is one
``als_ranking_metrics`` call (top-k, then one metrics pass over the ids and the batch's withheld items,
csrc/metrics.cu) that returns the batch's six fp64 sums, and the host only adds them up in batch order.  The
numbers are the array path's up to fp64 summation order.  Such a model fitted on a process group of several
ranks is evaluated from ``distributed.RowBlock``s: each rank scores the users of its own train / test blocks and
one all-reduce sums the six values (plus a failure flag), so every rank returns the same dict and no rank holds
the whole matrices.  Any other model with a ``recommend`` method goes through the array path.

``leave_k_out_split`` (:141-233) is dataset preparation rather than a caller of the hot path; it is provided with the
reference's contract (every eligible user leaves exactly K entries in the test matrix, train + test == input, a
reserved share of users stays train-only, the same ValueErrors).  The reference draws its shuffle from numpy's
global generator there (:128), so the split itself is seeded here and is not bit-comparable.

Every function here takes scipy CSRs (or RowBlocks of them); a CSR in CUDA memory is refused with ValueError.
"""
import numpy as np
from scipy.sparse import csr_matrix

from .als import AlternatingLeastSquares, _Ingest
from .distributed import RowBlock
from .utils import BLOCK_FIELDS, check_block_table, check_random_state, is_device_csr

def _host_only(*matrices):
    """ValueError for a CSR in CUDA memory, which evaluation does not read."""
    if any(is_device_csr(m) for m in matrices):
        raise ValueError("evaluation takes scipy CSRs: a CSR in CUDA memory is not supported here")


#: users per ``recommend`` call (the reference uses 1000, evaluation.pyx:417; any value gives the same sums)
BATCH = 16384


def train_test_split(ratings, train_percentage=0.8, random_state=None):
    """Random split of the stored entries into (train, test) CSR matrices (evaluation.pyx:14-48).

    One uniform draw per stored entry, in COO order: ``< train_percentage`` goes to train.  Negative
    test entries are dropped (:44-45)."""
    _host_only(ratings)
    ratings = ratings.tocoo()
    rng = check_random_state(random_state)
    draw = rng.random(len(ratings.data))
    in_train = draw < train_percentage
    parts = []
    for keep in (in_train, ~in_train):
        parts.append(csr_matrix((ratings.data[keep], (ratings.row[keep], ratings.col[keep])),
                                shape=ratings.shape, dtype=ratings.dtype))
    train, test = parts
    test.data[test.data < 0] = 0
    test.eliminate_zeros()
    return train, test


def leave_k_out_split(ratings, K=1, train_only_size=0.0, random_state=None):
    """'Leave K out': every eligible user (more than K + 1 stored entries, evaluation.pyx:191) gives K randomly
    chosen entries to the test matrix; `train_only_size` is the fraction of users kept out of the test set
    (:194-198).  Returns (train, test) CSR matrices of the input's shape with train + test == ratings."""
    _host_only(ratings)
    if K < 1:
        raise ValueError("The 'K' must be >= 1.")
    if not 0.0 <= train_only_size < 1.0:
        raise ValueError("The 'train_only_size' must be in the range (0.0 <= x < 1.0).")
    ratings = ratings.tocoo()
    rng = check_random_state(random_state)
    users, items, data = ratings.row, ratings.col, ratings.data
    unique_users, counts = np.unique(users, return_counts=True)
    candidate = counts > K + 1
    if train_only_size > 0.0:
        size = max(1, int(len(unique_users) * train_only_size))  # _choose, :73-75
        reserved = rng.choice(len(unique_users), size=size, replace=False)
        # positions (not ids) drawn from range(len(unique_users)) are matched against the ids, as in :195-197
        candidate &= ~np.isin(unique_users, reserved)
    in_candidates = np.isin(users, unique_users[candidate])
    # K random entries per candidate user: shuffle the entries, stable-sort by user, take the first K of each run
    pos = np.flatnonzero(in_candidates)
    pos = pos[rng.permutation(len(pos))]
    pos = pos[np.argsort(users[pos], kind="stable")]
    run_start = np.flatnonzero(np.r_[True, users[pos][1:] != users[pos][:-1]]) if len(pos) else np.zeros(0, dtype=int)
    rank_in_run = np.arange(len(pos)) - np.repeat(run_start, np.diff(np.r_[run_start, len(pos)]))
    test_pos = pos[rank_in_run < K]
    is_test = np.zeros(len(users), dtype=bool)
    is_test[test_pos] = True
    test = csr_matrix((data[is_test], (users[is_test], items[is_test])), shape=ratings.shape, dtype=ratings.dtype)
    train = csr_matrix((data[~is_test], (users[~is_test], items[~is_test])), shape=ratings.shape, dtype=ratings.dtype)
    return train, test


def _withheld_keys(test_user_items):
    """Sorted unique ``user * items + item`` keys of the test matrix and the per-user count of DISTINCT
    withheld items (the reference's ``likes`` is a set, evaluation.pyx:436-438: duplicates count once)."""
    users, items = test_user_items.shape
    indptr = np.asarray(test_user_items.indptr, dtype=np.int64)
    rows = np.repeat(np.arange(users, dtype=np.int64), np.diff(indptr))
    keys = np.unique(rows * items + np.asarray(test_user_items.indices, dtype=np.int64))
    distinct = np.bincount(keys // items, minlength=users) if len(keys) else np.zeros(users, dtype=np.int64)
    return keys, distinct


def ranking_metrics_at_k(model, train_user_items, test_user_items, K=10, show_progress=True, num_threads=1):
    """precision / map / ndcg / auc at K over the users that have withheld items (evaluation.pyx:366-475).

    ``model.recommend(batch, train_user_items[batch], N=K)`` supplies the ranked ids (liked training
    items filtered, the recommend default).  Per user, with ``L`` distinct withheld items and
    ``hit_i`` = "rank i is withheld":
      precision  sum hit_i / sum min(K, L)                                     (:440, :451-452, :470)
      map        mean over users of  sum_i hit_i * (hits so far) / (i+1) / min(K, L)          (:453, :460)
      ndcg       mean of  sum_i hit_i / log2(i+2) / sum_{j<min(K,L)} 1/log2(j+2)              (:454, :446)
      auc        mean of [sum_{miss i} hits before i + (hits + L)/2 * (items - L - misses)] / (L (items - L))
                                                                                (:455-461)

    For an ``AlternatingLeastSquares`` the metrics are computed on the device; ``test_user_items`` must then have
    one column per item of the model.  On a process group of several ranks, ``train_user_items`` and
    ``test_user_items`` may be ``distributed.RowBlock``s of the same rows on each rank; without one, or on one
    rank, a RowBlock must hold every row.
    """
    _host_only(train_user_items, test_user_items)
    if isinstance(model, AlternatingLeastSquares):
        return _device_ranking_metrics(model, train_user_items, test_user_items, int(K), show_progress)
    if isinstance(train_user_items, RowBlock):
        train_user_items = train_user_items.whole()
    if isinstance(test_user_items, RowBlock):
        test_user_items = test_user_items.whole()
    if not isinstance(train_user_items, csr_matrix):
        train_user_items = train_user_items.tocsr()
    if not isinstance(test_user_items, csr_matrix):
        test_user_items = test_user_items.tocsr()
    K = int(K)
    users, items = test_user_items.shape
    keys, distinct = _withheld_keys(test_user_items)
    to_generate = np.arange(users, dtype=np.int32)[np.ediff1d(test_user_items.indptr) > 0]  # :421-422

    gain, gain_sum = _gains(K)
    rank = np.arange(1, K + 1, dtype=np.float64)

    relevant = pr_div = mean_ap = ndcg = mean_auc = 0.0
    total = 0
    progress = None
    if show_progress:
        from tqdm.auto import tqdm

        progress = tqdm(total=len(to_generate))
    for start in range(0, len(to_generate), BATCH):
        batch = to_generate[start:start + BATCH]
        ids, _ = model.recommend(batch, train_user_items[batch], N=K)
        ids = np.asarray(ids).reshape(len(batch), -1).astype(np.int64)
        width = ids.shape[1]  # == K unless the model returned fewer columns
        q = batch.astype(np.int64)[:, None] * items + ids
        pos = np.searchsorted(keys, q)
        hit = np.zeros(q.shape, dtype=bool)
        inside = pos < len(keys)
        hit[inside] = keys[pos[inside]] == q[inside]
        hitf = hit.astype(np.float64)
        L = distinct[batch].astype(np.float64)
        cap = np.minimum(float(K), L)

        cum_hits = np.cumsum(hitf, axis=1)
        hits = cum_hits[:, -1] if width else np.zeros(len(batch))
        misses = float(K) - hits  # ranks the model did not fill count as misses, as in the scalar loop
        relevant += hits.sum()
        pr_div += cap.sum()
        mean_ap += ((hitf * cum_hits / rank[:width]).sum(axis=1) / cap).sum()
        ndcg += ((hitf * gain[:width]).sum(axis=1) / gain_sum[cap.astype(np.int64) - 1]).sum()
        neg = items - L
        # a miss at rank i adds the hits seen so far; unfilled ranks (width < K) all come after every hit
        auc = ((1.0 - hitf) * cum_hits).sum(axis=1) + (K - width) * hits
        auc += (hits + L) / 2.0 * (neg - misses)
        mean_auc += (auc / (L * neg)).sum()
        total += len(batch)
        if progress is not None:
            progress.update(len(batch))
    if progress is not None:
        progress.close()
    return {
        "precision": relevant / pr_div,
        "map": mean_ap / total,
        "ndcg": ndcg / total,
        "auc": mean_auc / total,
    }


def _gains(K):
    """The nDCG gain of each rank, 1 / log2(rank + 1), and its running sum (the ideal DCG of min(K, L) hits)."""
    gain = 1.0 / np.log2(np.arange(2, K + 2))
    return gain, np.cumsum(gain)


def _ratios(sums):
    """The metrics from the six sums (hits, sum min(K, L), AP, nDCG, AUC, users), divided like the array path."""
    relevant, pr_div, mean_ap, ndcg, mean_auc, total = (float(v) for v in sums)
    return {"precision": np.float64(relevant / pr_div), "map": np.float64(mean_ap / total),
            "ndcg": np.float64(ndcg / total), "auc": np.float64(mean_auc / total)}


def _device_ranking_metrics(model, train, test, K, show_progress):
    pg = model.process_group
    if pg is not None and pg.world > 1 and (isinstance(train, RowBlock) or isinstance(test, RowBlock)):
        return _row_block_metrics(model, train, test, K, show_progress)
    train = train.whole() if isinstance(train, RowBlock) else train
    test = test.whole() if isinstance(test, RowBlock) else test
    if not isinstance(train, csr_matrix):
        train = train.tocsr()
    if not isinstance(test, csr_matrix):
        test = test.tocsr()
    return _ratios(_device_sums(model, train, test, 0, K, show_progress))


def _device_sums(model, train, test, first_row, K, show_progress):
    """The six sums over the users with withheld items among rows [first_row, first_row + test.shape[0]) of the
    whole matrices, whose rows train / test hold: one device call per BATCH of them, added in batch order."""
    to_generate = np.arange(test.shape[0], dtype=np.int32)[np.ediff1d(test.indptr) > 0]  # :421-422
    if K == 0 and len(to_generate):
        raise IndexError("K = 0: there is no ideal DCG of 0 ranks")  # what the array path raises
    gain, gain_sum = _gains(K)
    sums = np.zeros(6)
    progress = None
    if show_progress:
        from tqdm.auto import tqdm

        progress = tqdm(total=len(to_generate))
    for start in range(0, len(to_generate), BATCH):
        batch = to_generate[start:start + BATCH]
        sums += model._ranking_sums(first_row + batch.astype(np.int64), train[batch], test[batch], K, gain, gain_sum)
        if progress is not None:
            progress.update(len(batch))
    if progress is not None:
        progress.close()
    return sums


def _row_block_metrics(model, train, test, K, show_progress):
    """ranking_metrics_at_k on a process group of several ranks, each holding the RowBlocks of the same rows of train
    and test.  The ranks all-gather both blocks' extents and check them like fit does, so a bad tiling, or train and
    test blocks of different rows, raises the same ValueError on every rank.  Each rank then sums its own users, and one
    all-reduce adds the six sums and a failure flag: a rank that failed raises its error, the others an AlsError."""
    pg, ctx = model.process_group, model.ctx
    W = pg.world
    ing = _Ingest(ctx, "evaluation")
    blocks = [b if isinstance(b, RowBlock) else RowBlock(b, 0, b.shape[0]) for b in (train, test)]

    def read():
        ms = [b.csr() for b in blocks]
        return ms, [(b.first_row, m.shape[0], b.users, m.shape[1], int(m.indptr[-1]) - int(m.indptr[0]), 0)
                    for b, m in zip(blocks, ms)]

    out, err = ing.run(read)
    mine = out[1] if err is None else [(0, 0, 0, 0, 0, 1)] * 2
    # both blocks' extents and whether this rank could read them (96 bytes)
    table = np.frombuffer(ctx.allgather_bytes(np.array(mine, dtype=np.int64).tobytes()), dtype=np.int64)
    table = table.reshape(W, 2, len(BLOCK_FIELDS))
    ing.fail(err, table[:, :, -1].any())
    for side, name in enumerate(("train_user_items", "test_user_items")):
        try:
            check_block_table(table[:, side])  # the same table on every rank: the same error on every rank
        except ValueError as e:
            raise ValueError(f"{name}: {e}") from None
    if table[0, 0, 2] != table[0, 1, 2]:
        raise ValueError(f"train_user_items has {table[0, 0, 2]} rows, test_user_items {table[0, 1, 2]}")
    for p in range(W):
        (f0, r0), (f1, r1) = table[p, 0, :2], table[p, 1, :2]
        if f0 != f1 or r0 != r1:
            raise ValueError(f"rank {p}'s train block holds rows [{f0}, {f0 + r0}) and its test block rows [{f1}, {f1 + r1}):"
                             " each rank's blocks must hold the same rows")
    (m_train, m_test) = out[0]
    sums, err = ing.run(lambda: _device_sums(model, m_train, m_test, blocks[1].first_row, K, show_progress))
    total = ctx.allreduce(np.append(sums if err is None else np.zeros(6), 0.0 if err is None else 1.0))
    ing.fail(err, total[-1] > 0)
    return _ratios(total[:6])


def precision_at_k(model, train_user_items, test_user_items, K=10, show_progress=True, num_threads=1):
    """evaluation.pyx:236-267"""
    return ranking_metrics_at_k(model, train_user_items, test_user_items, K, show_progress, num_threads)["precision"]


def mean_average_precision_at_k(model, train_user_items, test_user_items, K=10, show_progress=True, num_threads=1):
    """evaluation.pyx:270-299"""
    return ranking_metrics_at_k(model, train_user_items, test_user_items, K, show_progress, num_threads)["map"]


def ndcg_at_k(model, train_user_items, test_user_items, K=10, show_progress=True, num_threads=1):
    """evaluation.pyx:302-331"""
    return ranking_metrics_at_k(model, train_user_items, test_user_items, K, show_progress, num_threads)["ndcg"]


def AUC_at_k(model, train_user_items, test_user_items, K=10, show_progress=True, num_threads=1):
    """evaluation.pyx:334-363"""
    return ranking_metrics_at_k(model, train_user_items, test_user_items, K, show_progress, num_threads)["auc"]
