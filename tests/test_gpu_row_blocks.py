"""A multi-GPU fit from row blocks (distributed.RowBlock): every rank holds only its own, possibly uneven, block of
user rows.  Emulated for W ranks in one process and one context, like test_gpu_shard_ingest.py: rank p cuts its block
into one piece per rank (block_pieces), rank q stacks the pieces meant for it (DeviceCSR.concat_rows).  The stacked
user shards must be exactly the shards of today's ingest from the whole matrix, so every later step, and the fit, is
bitwise today's.  Also: concat_rows on its own, a bad index named by its global row, rank 0's device memory, the fit
on a one-rank communicator, and (on two GPUs) the fit itself.

Run as a script (one process per GPU, RANK / WORLD_SIZE / MASTER_* set), this file is the worker of the two-GPU test.
"""
import importlib.util
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if __name__ == "__main__":
    sys.path.insert(0, ROOT)
from helpers import KNOB_DEFAULTS, mixed_csr
from test_gpu_csr_ingest import expected_segments
from test_gpu_shard_ingest import assert_csr_equal, emulate, matrix, solve
from implicit_b200 import synthetic
from implicit_b200.utils import column_splits, nnz_balanced_splits, simulate_block_splits

pytestmark = pytest.mark.gpu
KNOBS = dict(KNOB_DEFAULTS, segment_nnz=0)


@pytest.fixture(scope="module")
def lib():
    set_in_env = sorted(n for n in (f"ALS_B200_{k.upper()}" for k in KNOBS) if n in os.environ)
    if set_in_env:
        pytest.fail(f"knob environment variables are set: {', '.join(set_in_env)}; unset them to run these tests")
    from implicit_b200 import _lib

    return _lib


@pytest.fixture(scope="module")
def ctx(lib):
    c = lib.Context(0)
    yield c
    c.close()


@pytest.fixture(autouse=True)
def knobs(ctx):
    for k, v in KNOBS.items():
        ctx.set_knob(k, v)
    yield
    for k, v in KNOBS.items():
        ctx.set_knob(k, v)


def uneven_bounds(users, W, seed):
    """Random block boundaries, one rank with no rows at all when W > 2."""
    rng = np.random.default_rng(seed)
    b = np.concatenate([[0], np.sort(rng.integers(0, users + 1, size=W - 1)), [users]]).astype(np.int64)
    if W > 2:
        b[W // 2 + 1] = b[W // 2]
    return np.maximum.accumulate(b)


def block_table(C, bounds):
    return np.array([(bounds[p], bounds[p + 1] - bounds[p], C.shape[0], C.shape[1],
                      C.indptr[bounds[p + 1]] - C.indptr[bounds[p]], 0) for p in range(len(bounds) - 1)], dtype=np.int64)


def emulate_blocks(lib, ctx, C, bounds, row_cost, alpha=1.0):
    """(shards, merged, usplit, isplit): every rank's Cui_s and Ciu_s as a fit from the row blocks `bounds` builds them."""
    from implicit_b200.als import block_pieces

    W, (users, items) = len(bounds) - 1, C.shape
    usplit = simulate_block_splits(block_table(C, bounds), [C.indptr[bounds[p]:bounds[p + 1] + 1] for p in range(W)],
                                   row_cost)
    cut = [block_pieces(ctx, C[bounds[p]:bounds[p + 1]], bounds[p], usplit) for p in range(W)]
    shards, counts = [], np.zeros(items, dtype=np.int64)
    for q in range(W):
        s = lib.DeviceCSR.concat_rows(ctx, [cut[p][q] for p in range(W)], items, usplit[q])
        if alpha != 1.0:
            s.scale(alpha)
        counts += s.column_counts()
        shards.append(s)
    for ps in cut:
        for x in ps:
            x.close()
    isplit = column_splits(counts, W, row_cost)
    pieces = [s.transpose_pieces(isplit) for s in shards]
    merged = [lib.DeviceCSR.merge_rows(ctx, [pieces[p][q] for p in range(W)], users, isplit[q]) for q in range(W)]
    for ps in pieces:
        for x in ps:
            x.close()
    return shards, merged, usplit, isplit


@pytest.mark.parametrize("capped", [False, True], ids=["cap0", "cap_small"])
@pytest.mark.parametrize("alpha", [1.0, 2.5])
@pytest.mark.parametrize("W", [2, 3, 8])
@pytest.mark.parametrize("kind", ["mixed", "tiny"])
def test_stacked_shards_are_the_whole_matrix_shards(lib, ctx, kind, W, alpha, capped):
    C = matrix(kind)
    scaled = C.copy()
    scaled.data = scaled.data * np.float32(alpha)
    cap = max(C.nnz // (2 * W * W), 2) if capped else 0
    ctx.set_knob("segment_nnz", cap)
    for row_cost in (20, 60):
        for seed in (0, 1):
            bounds = uneven_bounds(C.shape[0], W, seed + 10 * W)
            shards, merged, usplit, isplit = emulate_blocks(lib, ctx, C, bounds, row_cost, alpha)
            old_shards, old_merged, old_usplit, old_isplit = emulate(lib, ctx, C, W, row_cost, alpha)
            assert np.array_equal(usplit, old_usplit) and np.array_equal(isplit, old_isplit)
            for q in range(W):
                ref = lib.DeviceCSR.upload_rows(ctx, scaled, usplit[q], usplit[q + 1])
                want = ref.download()
                assert_csr_equal(shards[q], want)
                assert shards[q].shape3 == ref.shape3
                assert shards[q].segment_count == ref.segment_count == expected_segments(want.indptr, cap or 2**31 - 1)
                assert_csr_equal(merged[q], old_merged[q].download())
                assert merged[q].segment_count == old_merged[q].segment_count
                ref.close()
            for h in shards + merged + old_shards + old_merged:
                h.close()


@pytest.mark.parametrize("name", ["chol64", "chol200", "cg64"])
def test_solves_over_stacked_shards_are_bitwise(lib, ctx, name):
    f, use_cg = {"chol64": (64, False), "chol200": (200, False), "cg64": (64, True)}[name]
    C, W = matrix("mixed"), 3
    users, items = C.shape
    X, Y = synthetic.initial_factors(users, items, f, seed=f)
    shards, merged, usplit, _ = emulate_blocks(lib, ctx, C, uneven_bounds(users, W, 4), 20 if use_cg else 60)
    for q in range(W):
        ref = lib.DeviceCSR.upload_rows(ctx, C, usplit[q], usplit[q + 1])
        a, b = solve(lib, ctx, shards[q], X, Y, use_cg), solve(lib, ctx, ref, X, Y, use_cg)
        assert isinstance(a, np.ndarray) and np.array_equal(a.view(np.int32), b.view(np.int32)), q
        ref.close()
    for h in shards + merged:
        h.close()


def test_concat_rows(lib, ctx):
    C = matrix("mixed")
    users, items = C.shape
    cuts = [0, 0, 90, 91, 91, 400, users]  # empty pieces at the start, in the middle and a one-row piece
    up = [lib.DeviceCSR.upload_rows(ctx, C, cuts[k], cuts[k + 1]) for k in range(len(cuts) - 1)]

    one = lib.DeviceCSR.concat_rows(ctx, [up[2]], items, 5)  # n = 1: a copy
    assert_csr_equal(one, C[90:91])
    stacked = lib.DeviceCSR.concat_rows(ctx, up, items, 0)
    assert_csr_equal(stacked, C)
    assert stacked.segment_count == 1
    empty = lib.DeviceCSR.concat_rows(ctx, [up[0], up[3]], items, 0)
    assert empty.shape3 == (0, items, 0)

    whole = lib.DeviceCSR.upload(ctx, C)  # row-slice views: their indptrs do not start at 0
    views = [whole.slice_rows(cuts[k], cuts[k + 1]) for k in range(len(cuts) - 1)]
    assert_csr_equal(lib.DeviceCSR.concat_rows(ctx, views[::-1], items, 0),
                     sp.vstack([C[cuts[k]:cuts[k + 1]] for k in reversed(range(len(cuts) - 1))]).tocsr())

    cap = C.nnz // 7  # segmented pieces, and a result above the cap
    ctx.set_knob("segment_nnz", cap)
    seg = [lib.DeviceCSR.upload_rows(ctx, C, 0, 400), lib.DeviceCSR.upload_rows(ctx, C, 400, users)]
    assert seg[0].segment_count > 1
    for pieces in (seg, up, seg[::-1]):
        out = lib.DeviceCSR.concat_rows(ctx, pieces, items, 3)
        want = sp.vstack([p.download() for p in pieces]).tocsr()
        assert_csr_equal(out, want)
        assert out.segment_count == expected_segments(want.indptr, cap) > 1
        X, Y = synthetic.initial_factors(want.shape[0] + 3, items, 32, seed=2)
        ref = lib.DeviceCSR.upload(ctx, want, row_offset=3)
        a, b = solve(lib, ctx, out, X, Y, False), solve(lib, ctx, ref, X, Y, False)
        assert np.array_equal(a.view(np.int32), b.view(np.int32))  # the stacked CSR's schedule and row_offset
        for h in (out, ref):
            h.close()

    host = lib.DeviceCSR.upload(ctx, C[:50], host=True)
    with pytest.raises(lib.AlsError, match="host-resident") as e:
        lib.DeviceCSR.concat_rows(ctx, [up[2], host], items, 0)
    assert e.value.code == lib.ALS_E_UNSUPPORTED
    for h in up + views + seg + [one, stacked, empty, whole, host]:
        h.close()


def test_bad_index_in_a_block_names_its_global_row(lib, ctx):
    from implicit_b200.als import block_pieces

    C = matrix("mixed")
    usplit = nnz_balanced_splits(C.indptr, 3, 60)
    first = 250
    block = C[first:].copy()
    row = 120
    while block.indptr[row + 1] == block.indptr[row]:
        row += 1
    block.indices[block.indptr[row]] = C.shape[1] + 3
    with pytest.raises(ValueError, match=f"row {first + row} holds column index {C.shape[1] + 3}, which is outside"):
        block_pieces(ctx, block, first, usplit)
    nm = C[first:].copy()
    nm.indptr[40] = nm.indptr[41] + 1
    with pytest.raises(ValueError, match=f"not monotone at row {first + 40}\\b"):
        block_pieces(ctx, nm, first, usplit)


def load_tool():
    spec = importlib.util.spec_from_file_location("row_block_ingest_bench",
                                                  os.path.join(ROOT, "tools", "row_block_ingest_bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_rank_memory_of_the_block_ingest(lib, ctx):
    """Rank 0 of 8 in the 204M-nonzero case, with twice its even share of the rows as its block: its pool peak stays
    within today's sharded ingest plus 8 bytes per nonzero of its block (the block's pieces, alive until the exchange),
    and it builds today's shards."""
    tool = load_tool()
    W, row_cost = 8, 60
    C = tool.tiling(12)
    assert C.nnz >= 200_000_000
    bounds = tool.uneven_bounds(C.shape[0], W)
    _, old, s_old, m_old = tool.rank0_sharded(ctx, C, W, row_cost)
    _, new, s_new, m_new, block_nnz = tool.rank0_blocks(ctx, C, W, row_cost, bounds)
    print(f"rank 0 of {W}: sharded ingest peak {old / 1e9:.2f} GB, from its block of {block_nnz} nonzeros "
          f"{new / 1e9:.2f} GB")
    assert block_nnz > C.nnz // W
    assert new <= old + 8 * block_nnz
    for a, b in ((s_new, s_old), (m_new, m_old)):
        assert a.shape3 == b.shape3 and a.segment_count == b.segment_count
        a.close()
        b.close()


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


def test_fit_from_a_block_on_one_rank():
    """In a process of its own (the library loads NCCL with RTLD_GLOBAL): one_rank_worker."""
    ((rc, out),) = spawn([{}], "one-rank", timeout=600)
    assert rc == 0 and "ONE_RANK_BLOCK OK" in out, out[-3000:]


def fit_factors(C, pg=None, **kw):
    from implicit_b200 import AlternatingLeastSquares

    users, items = C.shape if not hasattr(C, "users") else (C.users, C.user_items.shape[1])
    X0, Y0 = synthetic.initial_factors(users, items, 64)
    m = AlternatingLeastSquares(factors=64, iterations=3, calculate_training_loss=True, process_group=pg, **kw)
    m.user_factors, m.item_factors = X0.copy(), Y0.copy()
    losses = []
    m.fit(C, show_progress=False, callback=lambda it, t, loss: losses.append(loss))
    return np.array(m.user_factors), np.array(m.item_factors), losses[-1]


def bitwise(a, b):
    return all(np.array_equal(x.view(np.int32), y.view(np.int32)) for x, y in zip(a[:2], b[:2]))


def one_rank_worker():
    """fit(RowBlock(C, 0, users)) on a one-rank communicator and without a process group is bitwise fit(C); a block
    of only some rows is refused without a process group and on one rank."""
    from implicit_b200 import _lib
    from implicit_b200.distributed import ProcessGroup, RowBlock

    C = synthetic.power_law_csr(3000, 2000, 90000, 7)
    users = C.shape[0]
    ctx = _lib.Context(0)
    ctx.comm_init(0, 1, _lib.comm_unique_id())
    pg = ProcessGroup(0, 1, ctx)
    ok = True
    for use_cg in (False, True):
        want = fit_factors(C, use_cg=use_cg, alpha=2.5)
        for label, group in (("no process group", None), ("one-rank communicator", pg)):
            got = fit_factors(RowBlock(C, 0, users), group, use_cg=use_cg, alpha=2.5)
            same = bitwise(got, want) and got[2] == want[2]
            print(f"{'cg' if use_cg else 'cholesky'}, {label}: RowBlock fit bitwise the plain fit: {same}", flush=True)
            ok &= same
    coo = RowBlock(C.tocoo(), 0, users)  # converted with the usual warning
    from implicit_b200.utils import ParameterWarning

    with pytest.warns(ParameterWarning):
        got = fit_factors(coo, use_cg=True)
    ok &= bitwise(got, fit_factors(C, use_cg=True))
    # fit() takes the block ingest only on several ranks; its collectives, exchange and stack run here on one
    from implicit_b200 import AlternatingLeastSquares

    for cap, alpha in ((0, 1.0), (C.nnz // 5, 2.5)):
        ctx.set_knob("segment_nnz", cap)
        m = AlternatingLeastSquares(factors=64, alpha=alpha, process_group=pg)
        new = m._ingest_row_blocks(RowBlock(C, 0, users), 60)
        old = m._ingest_shards(C.astype(np.float32), 60)
        same = new[4] == (users, C.shape[1], C.nnz) and all(np.array_equal(a, b) for a, b in zip(new[2:4], old[2:4]))
        for a, b in zip(new[:2], old[:2]):
            x, y = a.download(), b.download()
            same &= a.segment_count == b.segment_count and np.array_equal(x.indptr, y.indptr) and \
                np.array_equal(x.indices, y.indices) and np.array_equal(x.data.view(np.int32), y.data.view(np.int32))
            a.close()
            b.close()
        print(f"segment cap {cap}: one-rank ingest from a block equals the ingest from the matrix: {same}", flush=True)
        ok &= same
    ctx.set_knob("segment_nnz", 0)
    bad, row = C.copy(), 1234
    while bad.indptr[row + 1] == bad.indptr[row]:
        row += 1
    bad.indices[bad.indptr[row]] = C.shape[1]
    try:
        AlternatingLeastSquares(factors=64, process_group=pg)._ingest_row_blocks(RowBlock(bad, 0, users), 60)
        ok = False
    except ValueError as e:
        print(f"bad index refused: {e}", flush=True)
        ok &= f"row {row} " in str(e)
    for group in (None, pg):
        for block in (RowBlock(C[10:], 10, users), RowBlock(C[:-1], 0, users)):
            try:
                fit_factors(block, group)
                ok = False
                print("a partial block was fitted on one rank", flush=True)
            except ValueError as e:
                print(f"partial block refused: {e}", flush=True)
    ctx.close()
    print("ONE_RANK_BLOCK", "OK" if ok else "FAILED", flush=True)
    sys.exit(0 if ok else 1)


def test_two_gpu_fit_from_row_blocks():
    from implicit_b200 import _lib

    if _lib.device_count() < 2:
        pytest.skip("needs two GPUs")
    port = 29800 + os.getpid() % 90
    envs = [dict(RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
            for r in range(2)]
    for rc, out in spawn(envs):
        assert rc == 0, out[-3000:]
        assert "ROW_BLOCK_CHECK OK" in out, out[-3000:]


def worker():
    """One rank of the two-GPU test: rank 0 holds about 10 % of the rows, rank 1 the rest.  Fits from the blocks
    against the same ranks' fits from the whole matrix; a bad index in rank 1's block; mismatched `users`."""
    from implicit_b200 import _lib
    from implicit_b200.distributed import RowBlock, init_process_group

    pg = init_process_group()
    rank = pg.rank
    C = synthetic.power_law_csr(30000, 20000, 900000, 5)
    users = C.shape[0]
    bounds = [0, users // 10, users]
    r0, r1 = bounds[rank], bounds[rank + 1]
    ok = True
    for use_cg in (False, True):
        whole = fit_factors(C, pg, use_cg=use_cg, alpha=2.5)
        got = fit_factors(RowBlock(C[r0:r1], r0, users), pg, use_cg=use_cg, alpha=2.5)
        same = bitwise(got, whole) and abs(got[2] - whole[2]) <= 1e-12 * abs(whole[2])
        print(f"rank {rank}: {'cg' if use_cg else 'cholesky'} fit from rows [{r0}, {r1}) bitwise the whole-matrix fit: "
              f"{same} (loss {got[2]!r} vs {whole[2]!r})", flush=True)
        ok &= same

    block = C[r0:r1].copy()
    if rank == 1:
        row = 50
        while block.indptr[row + 1] == block.indptr[row]:
            row += 1
        block.indices[block.indptr[row]] = C.shape[1] + 7
    cases = [("bad index in rank 1's block", RowBlock(block, r0, users), ValueError if rank == 1 else _lib.AlsError),
             ("mismatched users", RowBlock(C[r0:r1], r0, users + rank), ValueError)]
    for label, blk, want in cases:
        raised = None
        try:
            fit_factors(blk, pg, use_cg=False)
        except (ValueError, _lib.AlsError) as e:
            raised = e
        print(f"rank {rank}: {label}: {type(raised).__name__}: {raised}", flush=True)
        ok &= type(raised) is want
        if label.startswith("bad index") and rank == 1:
            ok &= f"row {r0 + row} " in str(raised)
    pg.barrier()
    print(f"rank {rank} ROW_BLOCK_CHECK", "OK" if ok else "FAILED", flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    one_rank_worker() if sys.argv[1:] == ["one-rank"] else worker()
