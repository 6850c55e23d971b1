"""The row-sharded ingest of a multi-GPU fit (DeviceCSR.upload_rows, column_counts, transpose_pieces, merge_rows),
emulated for W ranks in one process and one context: every rank's shard of user_items and its pieces of the
transpose are built on the one device, and the pieces every rank made for rank q are merged as rank q would merge
what it receives.  The merged shards must be scipy's transpose bit for bit, the planned item split today's, every
solve over them bitwise what the same solve gives over slice_rows of the whole device transpose, and the loss terms
equal up to the arrival order of their fp64 atomics.

Run as a script (one process per GPU, RANK / WORLD_SIZE / MASTER_* set), this file is the worker of the two-GPU test.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp

if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from helpers import KNOB_DEFAULTS, bad_row_csr, mixed_csr
from test_gpu_csr_ingest import expected_segments
from implicit_b200 import synthetic
from implicit_b200.utils import column_splits, nnz_balanced_splits

pytestmark = pytest.mark.gpu
KNOBS = dict(KNOB_DEFAULTS, segment_nnz=0)
REG = 0.01


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


def with_empty_columns(C):
    """C with an empty column after every 50th one and five empty columns at the end."""
    C = C.copy()
    C.indices = (C.indices + C.indices // 50).astype(C.indices.dtype)
    return sp.csr_matrix((C.data, C.indices, C.indptr), shape=(C.shape[0], C.shape[1] + C.shape[1] // 50 + 5))


def matrix(kind):
    if kind == "mixed":  # giant rows, duplicates, stored zeros, negative values, empty rows and empty columns
        return with_empty_columns(mixed_csr(600, 500, 7, duplicates=True))
    # fewer rows and columns than some W: ranks with no users and item windows with no columns
    return sp.csr_matrix(np.array([[0, 2, 0], [1, 0, 0], [0, 0, 0], [3, -1, 0], [0, 5, 0]], dtype=np.float32))


def emulate(lib, ctx, C, W, row_cost, alpha=1.0):
    """(shards, merged, usplit, isplit): every rank's Cui_s and Ciu_s as a W-rank fit builds them."""
    usplit = nnz_balanced_splits(C.indptr, W, row_cost)
    shards, counts = [], np.zeros(C.shape[1], dtype=np.int64)
    for p in range(W):
        s = lib.DeviceCSR.upload_rows(ctx, C, usplit[p], usplit[p + 1])
        if alpha != 1.0:
            s.scale(alpha)
        counts += s.column_counts()
        shards.append(s)
    isplit = column_splits(counts, W, row_cost)
    pieces = [s.transpose_pieces(isplit) for s in shards]
    merged = [lib.DeviceCSR.merge_rows(ctx, [pieces[p][q] for p in range(W)], C.shape[0], isplit[q]) for q in range(W)]
    for ps in pieces:
        for x in ps:
            x.close()
    return shards, merged, usplit, isplit


def old_ingest(lib, ctx, C, alpha=1.0):
    """The whole-matrix ingest a multi-GPU fit used before: upload, scale, device transpose."""
    Cui = lib.DeviceCSR.upload(ctx, C)
    if alpha != 1.0:
        Cui.scale(alpha)
    return Cui, Cui.transpose()


def assert_csr_equal(d, want):
    got = d.download()
    assert got.shape == want.shape
    assert np.array_equal(got.indptr, want.indptr) and np.array_equal(got.indices, want.indices)
    assert np.array_equal(got.data.view(np.int32), want.data.view(np.int32))  # bits: -0.0 and stored zeros too


@pytest.mark.parametrize("capped", [False, True], ids=["cap0", "cap_small"])
@pytest.mark.parametrize("alpha", [1.0, 2.5])
@pytest.mark.parametrize("W", [2, 3, 8])
@pytest.mark.parametrize("kind", ["mixed", "tiny"])
def test_merged_shards_are_scipy_transpose(lib, ctx, kind, W, alpha, capped):
    C = matrix(kind)
    scaled = C.copy()
    scaled.data = scaled.data * np.float32(alpha)
    T = scaled.T.tocsr()
    cap = max(C.nnz // (2 * W * W), 2) if capped else 0  # below the size of a piece: shards, pieces and merges segmented
    ctx.set_knob("segment_nnz", cap)
    for row_cost in (20, 60):  # the CG and the Cholesky split
        shards, merged, usplit, isplit = emulate(lib, ctx, C, W, row_cost, alpha)
        Cui, Ciu = old_ingest(lib, ctx, C, alpha)
        assert np.array_equal(isplit, nnz_balanced_splits(Ciu.indptr_host(), W, row_cost))
        assert usplit[-1] == C.shape[0] and isplit[-1] == C.shape[1]
        for p in range(W):
            u0, u1, i0, i1 = usplit[p], usplit[p + 1], isplit[p], isplit[p + 1]
            assert_csr_equal(shards[p], scaled[u0:u1])
            assert_csr_equal(merged[p], T[i0:i1])
            if capped:
                assert shards[p].segment_count == expected_segments(scaled[u0:u1].indptr, cap)
                assert merged[p].segment_count == expected_segments(T[i0:i1].indptr, cap)
        if capped and kind == "mixed":
            assert any(s.segment_count > 1 for s in shards)
            pieces = shards[0].transpose_pieces(isplit)
            assert any(x.segment_count > 1 for x in pieces)
            T0 = scaled[:usplit[1]].T.tocsr()
            for q, x in enumerate(pieces):  # rows of piece q: its item window; columns: global user ids
                assert_csr_equal(x, T0[isplit[q]:isplit[q + 1]])
                assert x.segment_count == expected_segments(T0[isplit[q]:isplit[q + 1]].indptr, cap)
                x.close()
        if kind == "tiny" and W == 8:
            assert any(usplit[p] == usplit[p + 1] for p in range(W))
            assert any(isplit[p] == isplit[p + 1] for p in range(W))
        for h in shards + merged + [Cui, Ciu]:
            h.close()


SOLVES = {  # name: (factors, use_cg, knobs)
    "chol16": (16, False, {}), "chol64": (64, False, {}), "chol100": (100, False, {}), "chol200": (200, False, {}),
    "chol64_long_tc": (64, False, {"long_tc": 1}), "chol64_short_max0": (64, False, {"short_max": 0}),
    "cg64": (64, True, {}), "cg200": (200, True, {}),
}


def solve(lib, ctx, C, X0, Y, use_cg):
    """X after one half over C from X0 (downloaded), or the ValueError's message."""
    dX, dY = lib.DeviceFactors.from_host(ctx, X0), lib.DeviceFactors.from_host(ctx, Y)
    try:
        if use_cg:
            lib.least_squares_cg(ctx, C, dX, dY, REG, 3)
        else:
            lib.least_squares(ctx, C, dX, dY, REG)
        out = dX.download()
    except ValueError as e:
        out = str(e)
    dX.close()
    dY.close()
    return out


@pytest.mark.parametrize("state", ["cold", "warm"])
@pytest.mark.parametrize("name", list(SOLVES))
def test_solves_over_shards_are_bitwise(lib, ctx, name, state):
    f, use_cg, knobs = SOLVES[name]
    C, W = matrix("mixed"), 3
    users, items = C.shape
    X, Y = synthetic.initial_factors(users, items, f, seed=f)
    Cui, Ciu = old_ingest(lib, ctx, C)
    if state == "warm":  # one whole-matrix iteration first
        dX, dY = lib.DeviceFactors.from_host(ctx, X), lib.DeviceFactors.from_host(ctx, Y)
        lib.least_squares_cg(ctx, Cui, dX, dY, REG, 3)
        lib.least_squares_cg(ctx, Ciu, dY, dX, REG, 3)
        X, Y = dX.download(), dY.download()
        dX.close()
        dY.close()
    for k, v in knobs.items():
        ctx.set_knob(k, v)
    shards, merged, usplit, isplit = emulate(lib, ctx, C, W, 20 if use_cg else 60)
    for side, new, whole, split, X0, Yo in (("user", shards, Cui, usplit, X, Y), ("item", merged, Ciu, isplit, Y, X)):
        for p in range(W):
            old = whole.slice_rows(split[p], split[p + 1])
            a, b = solve(lib, ctx, new[p], X0, Yo, use_cg), solve(lib, ctx, old, X0, Yo, use_cg)
            if isinstance(b, str):
                assert a == b, (side, p)
            else:
                assert isinstance(a, np.ndarray) and np.array_equal(a.view(np.int32), b.view(np.int32)), (side, p)
                # the rows outside the shard are untouched: the merged shard carries its row_offset
                assert np.array_equal(np.delete(a, np.arange(split[p], split[p + 1]), axis=0),
                                      np.delete(X0, np.arange(split[p], split[p + 1]), axis=0))
            dX, dY = lib.DeviceFactors.from_host(ctx, X0), lib.DeviceFactors.from_host(ctx, Yo)
            # fp64 sums accumulated with atomics in arrival order: the same call twice may differ in the last bits
            ta, tb = lib.loss_terms(ctx, new[p], dX, dY, REG), lib.loss_terms(ctx, old, dX, dY, REG)
            assert np.allclose(ta, tb, rtol=1e-12, atol=0), (side, p, ta - tb)
            for h in (dX, dY, old):
                h.close()
    for h in shards + merged + [Cui, Ciu]:
        h.close()


def test_bad_row_in_merged_shard_is_named_globally(lib, ctx):
    f, bad, W = 16, 30, 3
    B = bad_row_csr(f, [bad])      # its row `bad` is not positive definite against Y = I, at lambda = 0
    C = B.T.tocsr()                # users x items whose transpose is B
    shards, merged, _, isplit = emulate(lib, ctx, C, W, 60)
    q = int(np.searchsorted(isplit, bad, side="right")) - 1
    assert 0 < isplit[q] <= bad < isplit[q + 1]
    assert_csr_equal(merged[q], C.T.tocsr()[isplit[q]:isplit[q + 1]])
    eye = lib.DeviceFactors.from_host(ctx, np.eye(f, dtype=np.float32))
    out = lib.DeviceFactors(ctx, B.shape[0], f)
    with pytest.raises(ValueError, match=f"row {bad}\\b"):
        lib.least_squares(ctx, merged[q], out, eye, 0.0)
    for h in shards + merged + [eye, out]:
        h.close()


def test_shard_upload_refuses_bad_rows(lib, ctx):
    C = matrix("mixed")
    bad = C.copy()
    bad.indices = bad.indices.copy()
    bad.indices[bad.indptr[400]] = C.shape[1] + 3
    lib.DeviceCSR.upload_rows(ctx, bad, 0, 300).close()  # the bad index lies outside these rows
    with pytest.raises(ValueError, match="is outside"):
        lib.DeviceCSR.upload_rows(ctx, bad, 300, 600)
    nm = C.copy()
    nm.indptr = nm.indptr.copy()
    nm.indptr[450] = nm.indptr[451] + 1
    with pytest.raises(ValueError, match="not monotone at row"):
        lib.DeviceCSR.upload_rows(ctx, nm, 300, 600)


def spawn(envs, *args, timeout=900):
    """Runs this file once per environment in `envs` (extra arguments `args`) and returns (returncode, output) of each.
    A process still running at the timeout is killed: a hung rank must not outlive the test on the GPU."""
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


def test_exchange_over_a_one_rank_communicator():
    """als_comm_exchange_csr and als_comm_allreduce_i64 through NCCL on one GPU (one_rank_worker).  In a process of its
    own: the library loads NCCL with RTLD_GLOBAL, and a later `import torch` in the same process would bind to it."""
    ((rc, out),) = spawn([{}], "one-rank", timeout=600)
    assert rc == 0 and "ONE_RANK_EXCHANGE OK" in out, out[-3000:]


def one_rank_worker():
    """A one-rank communicator sends each piece to itself.  The received piece (laid out without a schedule) must be
    the piece bit for bit, and a solve over it, which builds its schedule at first use, bitwise the solve over the same
    matrix uploaded; with and without a segment cap."""
    from implicit_b200 import _lib as lib

    ctx = lib.Context(0)
    ctx.comm_init(0, 1, lib.comm_unique_id())
    v = np.array([3, -(2**40) - 1, 2**53 + 1, 0], dtype=np.int64)
    assert np.array_equal(ctx.allreduce_i64(v), v)
    C = matrix("mixed")
    users, items = C.shape
    for cap in (0, C.nnz // 20):
        ctx.set_knob("segment_nnz", cap)
        for r0, r1 in ((100, 400), (0, users), (7, 7)):  # a shard mid-matrix, the whole matrix, no rows (nnz 0)
            rows = sp.vstack([sp.csr_matrix((r0, items), dtype=np.float32), C[r0:r1]]).tocsr()
            want = rows.T.tocsr()  # items x r1: the global user ids of rows [r0, r1)
            s = lib.DeviceCSR.upload_rows(ctx, C, r0, r1)
            (piece,) = s.transpose_pieces([0, items])
            (got,) = ctx.exchange_csr([piece])
            assert_csr_equal(piece, want)
            assert_csr_equal(got, want)
            if cap and want.nnz:
                assert got.segment_count == expected_segments(want.indptr, cap) > 1
            ref = lib.DeviceCSR.upload(ctx, want)
            X0, Y = synthetic.initial_factors(items, r1, 64, seed=3)
            for use_cg in (False, True):
                a, b = solve(lib, ctx, got, X0, Y, use_cg), solve(lib, ctx, ref, X0, Y, use_cg)
                assert np.array_equal(a.view(np.int32), b.view(np.int32)), (cap, r0, r1, use_cg)
            for h in (s, piece, got, ref):
                h.close()
            print(f"segment cap {cap}, rows [{r0}, {r1}): {want.nnz} nonzeros exchanged exactly", flush=True)
    ctx.close()
    print("ONE_RANK_EXCHANGE OK", flush=True)


def test_rank_memory_is_a_fraction_of_the_whole_ingest(lib, ctx):
    """Rank 0 of an 8-rank fit on 204M nonzeros: the pool's peak while it builds Cui_s and Ciu_s, counting the pieces
    it receives from the 7 other ranks from the start, against the peak of the whole-matrix upload and transpose."""
    W, row_cost = 8, 60
    C = synthetic.block_diagonal_tiling(synthetic.power_law_csr(40000, 20000, 17_000_000, 31), 12)
    assert C.nnz >= 200_000_000
    base, _ = ctx.mem_peak()
    Cui, Ciu = old_ingest(lib, ctx, C)
    _, peak = ctx.mem_peak()
    old = peak - base
    Cui.close()
    Ciu.close()

    usplit = nnz_balanced_splits(C.indptr, W, row_cost)
    isplit = column_splits(np.bincount(C.indices, minlength=C.shape[1]), W, row_cost)
    received = []
    for p in range(1, W):  # what the other ranks send to rank 0
        s = lib.DeviceCSR.upload_rows(ctx, C, usplit[p], usplit[p + 1])
        pieces = s.transpose_pieces(isplit)
        received.append(pieces[0])
        for x in pieces[1:] + [s]:
            x.close()
    ctx.mem_peak()  # restart the mark
    s0 = lib.DeviceCSR.upload_rows(ctx, C, usplit[0], usplit[1])
    pieces = s0.transpose_pieces(isplit)
    for x in pieces[1:]:  # sent, then freed
        x.close()
    m0 = lib.DeviceCSR.merge_rows(ctx, [pieces[0]] + received, C.shape[0], isplit[0])
    _, peak = ctx.mem_peak()
    new = peak - base
    print(f"whole ingest peak {old / 1e9:.2f} GB, rank 0 of {W} {new / 1e9:.2f} GB ({C.nnz} nonzeros)")
    assert new < old / 3
    assert m0.shape3 == (isplit[1], C.shape[0], int(np.bincount(C.indices, minlength=C.shape[1])[:isplit[1]].sum()))
    for x in [s0, m0, pieces[0]] + received:
        x.close()


def test_two_gpu_fit_with_sharded_ingest():
    from implicit_b200 import _lib

    if _lib.device_count() < 2:
        pytest.skip("needs two GPUs")
    port = 29900 + os.getpid() % 90
    envs = [dict(RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
            for r in range(2)]
    for rc, out in spawn(envs):
        assert rc == 0, out[-3000:]
        assert "SHARD_INGEST_CHECK OK" in out, out[-3000:]


def worker():
    """One rank of the two-GPU test: fits with the sharded ingest against the same fits with the whole-matrix ingest,
    per-rank memory, and a bad column index in rank 1's rows."""
    from implicit_b200 import AlternatingLeastSquares, _lib
    from implicit_b200.distributed import init_process_group

    pg = init_process_group()
    ctx, rank, world = pg.ctx, pg.rank, pg.world
    U, I, f = 30000, 20000, 64
    Cui = synthetic.power_law_csr(U, I, 900000, 5)
    X0, Y0 = synthetic.initial_factors(U, I, f)
    ok = True

    class OldIngest(AlternatingLeastSquares):
        def _ingest_shards(self, Cui_host, row_cost):
            Cui, Ciu = old_ingest(_lib, self.ctx, Cui_host, self.alpha)
            usplit = nnz_balanced_splits(Cui_host.indptr, world, row_cost)
            isplit = nnz_balanced_splits(Ciu.indptr_host(), world, row_cost)
            return (Cui.slice_rows(usplit[rank], usplit[rank + 1]), Ciu.slice_rows(isplit[rank], isplit[rank + 1]),
                    usplit, isplit)

    def fit(cls, use_cg, alpha):
        m = cls(factors=f, use_cg=use_cg, iterations=3, alpha=alpha, calculate_training_loss=True, process_group=pg)
        m.user_factors, m.item_factors = X0.copy(), Y0.copy()
        m.fit(Cui, show_progress=False)
        return np.array(m.user_factors), np.array(m.item_factors)

    for use_cg, alpha in ((False, 1.0), (True, 2.5)):
        new, old = fit(AlternatingLeastSquares, use_cg, alpha), fit(OldIngest, use_cg, alpha)
        same = all(np.array_equal(a.view(np.int32), b.view(np.int32)) for a, b in zip(new, old))
        print(f"rank {rank}: {'cg' if use_cg else 'cholesky'} fit, sharded ingest bitwise equal: {same}", flush=True)
        ok &= same

    peaks = []
    for cls in (AlternatingLeastSquares, OldIngest):
        m = cls(factors=f, process_group=pg)
        base, _ = ctx.mem_peak()
        shards = m._ingest_shards(Cui, 20)[:2]
        _, peak = ctx.mem_peak()
        peaks.append(peak - base)
        for s in shards:
            s.close()
    print(f"rank {rank}: ingest peak {peaks[0] / 1e6:.1f} MB sharded, {peaks[1] / 1e6:.1f} MB whole", flush=True)
    ok &= peaks[0] < 0.65 * peaks[1]

    usplit = nnz_balanced_splits(Cui.indptr, world, 60)
    bad = Cui.copy()
    bad.indices = bad.indices.copy()
    row = usplit[1]
    while bad.indptr[row + 1] == bad.indptr[row]:
        row += 1
    bad.indices[bad.indptr[row]] = I + 7  # in rank 1's rows only
    raised = None
    try:
        m = AlternatingLeastSquares(factors=f, use_cg=False, iterations=1, process_group=pg)
        m.fit(bad, show_progress=False)
    except (ValueError, _lib.AlsError) as e:
        raised = e
    print(f"rank {rank}: bad index in row {row}: {type(raised).__name__}: {raised}", flush=True)
    want = ValueError if rank == 1 else _lib.AlsError
    ok &= type(raised) is want
    pg.barrier()
    print(f"rank {rank} SHARD_INGEST_CHECK", "OK" if ok else "FAILED", flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    one_rank_worker() if sys.argv[1:] == ["one-rank"] else worker()
