"""ranking_metrics_at_k on the device (als_ranking_metrics, csrc/metrics.cu) for this package's model, against the array
path fed by the same model's recommend (forced through a proxy that exposes only `recommend`) and against the scalar
restatement of the reference (oracle/evaluation_oracle.py), to rel 1e-12: only the fp64 summation order differs.

Every top-k path (mma.sync at f = 32, wgmma at f = 64 with more than 1024 queries, the segmented sort at f = 200 and
above the k-list limit), K at the edges of the k-lists and above the items, users without withheld items, duplicate,
unsorted and stored-zero test entries, unsorted and empty train rows, a user whose filter leaves fewer than K items
(the filtered tail is ranked), item 0 withheld (ranks past the items are id 0) and exact score ties (integer factors).
Also: repeatability, errors, row blocks (one-rank communicator, emulated W = 3, mismatched blocks, two GPUs).

Run as a script (one process per GPU, RANK / WORLD_SIZE / MASTER_* set), this file is the worker of the two-GPU test.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if __name__ == "__main__":
    sys.path.insert(0, ROOT)
from oracle import evaluation_oracle  # noqa: E402

pytestmark = pytest.mark.gpu
KEYS = ("precision", "map", "ndcg", "auc")


class Proxy:
    """Only `recommend`: ranking_metrics_at_k takes its array path."""

    def __init__(self, model):
        self.model = model

    def recommend(self, *args, **kwargs):
        return self.model.recommend(*args, **kwargs)


def shuffled_rows(m, rng):
    """The same CSR with the entries of every row in random order."""
    m = m.tocsr()
    rows = np.repeat(np.arange(m.shape[0]), np.diff(m.indptr))
    order = np.lexsort((rng.random(m.nnz), rows))
    out = sp.csr_matrix((m.data[order], m.indices[order], m.indptr.copy()), shape=m.shape)
    out.has_sorted_indices = False
    return out


def case(users, items, f, seed, ties=False, crowded=True, **model_args):
    """(model, train, test).  crowded: user 1 likes all but 3 items, so its filter leaves fewer than K."""
    from implicit_b200.als import AlternatingLeastSquares

    rng = np.random.default_rng(seed)
    if ties:  # small integers: exact scores, many equal, so rank order decides AP and nDCG
        X = rng.integers(-2, 3, (users, f)).astype(np.float32)
        Y = rng.integers(-2, 3, (items, f)).astype(np.float32)
    else:
        X = (rng.standard_normal((users, f)) * 0.3).astype(np.float32)
        Y = (rng.standard_normal((items, f)) * 0.3).astype(np.float32)
    model = AlternatingLeastSquares(factors=f, random_state=0, **model_args)
    model.user_factors, model.item_factors = X, Y
    train = sp.random(users, items, density=0.05, format="lil", dtype=np.float32, random_state=seed)
    train[::7] = 0  # empty train rows
    if crowded:
        train[1, :] = 1.0
        train[1, [0, items // 2, items - 1]] = 0
    train = sp.csr_matrix(train)
    train.eliminate_zeros()
    train = shuffled_rows(train, rng)
    n = rng.integers(0, 12, size=users)
    n[rng.random(users) < 0.2] = 0  # users without withheld items
    indptr = np.concatenate([[0], np.cumsum(n)])
    indices = rng.integers(0, items, size=int(indptr[-1]))  # duplicates and unsorted rows
    zero_hit = rng.random(users) < 0.1
    first = indptr[:-1][(n > 0) & zero_hit]
    indices[first] = 0  # item 0 withheld
    data = np.ones(len(indices), dtype=np.float32)
    data[rng.random(len(data)) < 0.05] = 0.0  # stored zeros count: only indices are read
    test = sp.csr_matrix((data, indices.astype(np.int32), indptr.astype(np.int32)), shape=(users, items))
    return model, train, test


def assert_close(got, exp):
    for k in KEYS:
        assert got[k] == pytest.approx(exp[k], rel=1e-12, abs=0), (k, got[k], exp[k])


PATHS = [(32, 1, 300), (32, 10, 300), (32, 16, 300), (32, 17, 300), (32, 64, 300), (32, 65, 300), (32, 400, 300),
         (64, 1, 300), (64, 10, 300), (64, 16, 300), (64, 17, 300),  # K <= 16: the wgmma kernel
         (200, 10, 300), (200, 65, 300), (200, 400, 300),           # by-sort
         (32, 1200, 1500)]                                          # by-sort above the k-list limit


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("f,K,items", PATHS)
def test_device_metrics_match_array_path_and_oracle(f, K, items, ties):
    from implicit_b200 import evaluation

    # the wgmma kernel takes a batch only when every row keeps K unfiltered items, so no crowded user at f = 64
    model, train, test = case(1600, items, f, seed=f * 1000 + K, ties=ties, crowded=f != 64)
    got = evaluation.ranking_metrics_at_k(model, train, test, K=K, show_progress=False)
    host = evaluation.ranking_metrics_at_k(Proxy(model), train, test, K=K, show_progress=False)
    exp = evaluation_oracle.ranking_metrics_at_k(model, train, test, K=K)
    assert_close(got, host)
    assert_close(got, exp)


@pytest.mark.parametrize("batch", [7, None])
@pytest.mark.parametrize("f", [32, 200])
def test_batch_sizes(f, batch, monkeypatch):
    from implicit_b200 import evaluation

    if batch is not None:
        monkeypatch.setattr(evaluation, "BATCH", batch)
    model, train, test = case(300, 120, f, seed=5, ties=True)
    for K in (10, 130):
        got = evaluation.ranking_metrics_at_k(model, train, test, K=K, show_progress=False)
        assert_close(got, evaluation.ranking_metrics_at_k(Proxy(model), train, test, K=K, show_progress=False))
        assert_close(got, evaluation_oracle.ranking_metrics_at_k(model, train, test, K=K))
        for name, fn in (("precision", evaluation.precision_at_k), ("map", evaluation.mean_average_precision_at_k),
                         ("ndcg", evaluation.ndcg_at_k), ("auc", evaluation.AUC_at_k)):
            assert fn(model, train, test, K=K, show_progress=False) == got[name]


def test_repeatable_bits():
    from implicit_b200 import evaluation

    model, train, test = case(1600, 300, 64, seed=11, crowded=False)
    a = evaluation.ranking_metrics_at_k(model, train, test, K=10, show_progress=False)
    b = evaluation.ranking_metrics_at_k(model, train, test, K=10, show_progress=False)
    assert all(np.float64(a[k]).tobytes() == np.float64(b[k]).tobytes() for k in KEYS)


def test_errors_match_array_path():
    from implicit_b200 import _lib, evaluation

    model, train, test = case(200, 100, 32, seed=3)
    big = sp.vstack([train, train[:5]]).tocsr()
    big_test = sp.vstack([test, sp.csr_matrix(np.ones((5, 100), dtype=np.float32))]).tocsr()
    wide = sp.hstack([train, sp.csr_matrix((200, 4), dtype=np.float32)]).tocsr()
    cases = [(big, big_test, IndexError),        # users outside the model
             (wide, test, _lib.AlsError),       # train columns are not the model's items
             (train[:150], test, IndexError)]   # test rows past train's
    for tr, te, want in cases:
        for m in (model, Proxy(model)):
            with pytest.raises(want):
                evaluation.ranking_metrics_at_k(m, tr, te, K=10, show_progress=False)


def uneven_blocks(users):
    return [0, users // 5, users // 5, users]  # W = 3, rank 1's block empty


def test_emulated_row_blocks_sum_to_the_whole():
    """Rank p's sums (its own block of train and test rows, query rows first_row + local row) added over W = 3 uneven
    blocks, one empty, are the whole matrices' sums."""
    from implicit_b200 import evaluation

    model, train, test = case(1600, 300, 32, seed=21, ties=True)
    whole = evaluation._device_sums(model, train, test, 0, 10, False)
    b = uneven_blocks(train.shape[0])
    parts = [evaluation._device_sums(model, train[b[p]:b[p + 1]], test[b[p]:b[p + 1]], b[p], 10, False) for p in range(3)]
    assert sum(parts) == pytest.approx(whole, rel=1e-12)
    assert_close(evaluation._ratios(sum(parts)), evaluation.ranking_metrics_at_k(Proxy(model), train, test, K=10,
                                                                                show_progress=False))


def spawn(envs, *args, timeout=900):
    """Runs this file once per environment in `envs` and returns (returncode, output) of each; a process still running
    at the timeout is killed, so a rank stuck in a collective cannot outlive the test."""
    procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), *args], env=dict(os.environ, **env),
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for env in envs]
    try:
        outs = [p.communicate(timeout=timeout)[0] for p in procs]
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    return [(p.returncode, o) for p, o in zip(procs, outs)]


def test_row_blocks_on_one_rank():
    """In a process of its own (the library loads NCCL with RTLD_GLOBAL): one_rank_worker."""
    ((rc, out),) = spawn([{}], "one-rank", timeout=600)
    assert rc == 0 and "ONE_RANK_EVAL OK" in out, out[-3000:]


def one_rank_worker():
    from implicit_b200 import _lib, evaluation
    from implicit_b200.distributed import ProcessGroup, RowBlock

    model, train, test = case(1600, 300, 32, seed=31)
    want = evaluation.ranking_metrics_at_k(model, train, test, K=10, show_progress=False)
    ctx = _lib.Context(0)
    ctx.comm_init(0, 1, _lib.comm_unique_id())
    model, _, _ = case(1600, 300, 32, seed=31, process_group=ProcessGroup(0, 1, ctx))
    users = train.shape[0]
    got = evaluation.ranking_metrics_at_k(model, RowBlock(train, 0, users), RowBlock(test, 0, users), K=10,
                                          show_progress=False)
    ok = all(np.float64(got[k]).tobytes() == np.float64(want[k]).tobytes() for k in KEYS)
    print(f"one-rank communicator, whole RowBlocks: {got} (plain matrices: {want})", flush=True)
    try:
        evaluation.ranking_metrics_at_k(model, RowBlock(train[10:], 10, users), RowBlock(test[10:], 10, users), K=10,
                                        show_progress=False)
        ok = False
    except ValueError as e:
        print(f"partial block refused: {e}", flush=True)
    ctx.close()
    print("ONE_RANK_EVAL", "OK" if ok else "FAILED", flush=True)
    sys.exit(0 if ok else 1)


def test_two_gpu_row_blocks():
    from implicit_b200 import _lib

    if _lib.device_count() < 2:
        pytest.skip("needs two GPUs")
    port = 29700 + os.getpid() % 90
    envs = [dict(RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
            for r in range(2)]
    for rc, out in spawn(envs):
        assert rc == 0, out[-3000:]
        assert "EVAL_BLOCK_CHECK OK" in out, out[-3000:]


def worker():
    """One rank of the two-GPU test: rank 0 holds about 10 % of the rows.  Both ranks must return the single-GPU dict
    (rel 1e-12) and identical dicts; an out-of-range index in rank 1's test block makes both ranks raise."""
    from implicit_b200 import _lib, evaluation
    from implicit_b200.distributed import RowBlock, init_process_group

    pg = init_process_group()
    rank = pg.rank
    model, train, test = case(3000, 400, 32, seed=41, device=rank)
    single = evaluation.ranking_metrics_at_k(model, train, test, K=10, show_progress=False)
    model, _, _ = case(3000, 400, 32, seed=41, process_group=pg)
    users = train.shape[0]
    b = [0, users // 10, users]
    r0, r1 = b[rank], b[rank + 1]
    got = evaluation.ranking_metrics_at_k(model, RowBlock(train[r0:r1], r0, users), RowBlock(test[r0:r1], r0, users),
                                          K=10, show_progress=False)
    ok = all(got[k] == pytest.approx(single[k], rel=1e-12, abs=0) for k in KEYS)
    mine = np.array([got[k] for k in KEYS])
    both = np.frombuffer(pg.ctx.allgather_bytes(mine.tobytes()), dtype=np.float64).reshape(2, 4)
    ok &= bool(np.array_equal(both[0].view(np.int64), both[1].view(np.int64)))
    print(f"rank {rank}: rows [{r0}, {r1}): {got} (single GPU {single}); ranks identical: {ok}", flush=True)

    bad = test[r0:r1].copy()
    if rank == 1:
        row = int(np.flatnonzero(np.diff(bad.indptr))[0])
        bad.indices[bad.indptr[row]] = test.shape[1] + 3
    raised = None
    try:
        evaluation.ranking_metrics_at_k(model, RowBlock(train[r0:r1], r0, users), RowBlock(bad, r0, users), K=10,
                                        show_progress=False)
    except (ValueError, _lib.AlsError) as e:
        raised = e
    want = ValueError if rank == 1 else _lib.AlsError
    print(f"rank {rank}: bad index in rank 1's test block: {type(raised).__name__}: {raised}", flush=True)
    ok &= type(raised) is want
    pg.barrier()
    print(f"rank {rank} EVAL_BLOCK_CHECK", "OK" if ok else "FAILED", flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    one_rank_worker() if sys.argv[1:] == ["one-rank"] else worker()
