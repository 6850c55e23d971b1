"""CSRs held as row-block segments (more nonzeros than the segment cap): the layout must never change a result.

Small cases force the cap with the segment_nnz knob on mixed_csr data (duplicates, empty rows, giant rows, negative
confidences, stored zeros) and compare every CSR call bit for bit with the one-segment run.  One case runs a real
matrix above 2^31 nonzeros: a block-diagonal tiling of a base CSR, where every block of the factors must equal block 0.
"""
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import scipy.sparse as sp

from helpers import CHOL_MAX, KNOB_DEFAULTS, cholesky_truth, factors_of, mixed_csr, row_err

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REG = 0.05


@pytest.fixture(scope="module")
def lib():
    names = [f"ALS_B200_{k.upper()}" for k in list(KNOB_DEFAULTS) + ["segment_nnz"]]
    set_in_env = sorted(n for n in names if n in os.environ)
    if set_in_env:  # a one-segment reference run would silently be segmented too
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
    """Every test starts and ends with every knob at its default and one-segment CSRs (segment_nnz = 0)."""
    for k, v in dict(KNOB_DEFAULTS, segment_nnz=0).items():
        ctx.set_knob(k, v)
    yield
    for k, v in dict(KNOB_DEFAULTS, segment_nnz=0).items():
        ctx.set_knob(k, v)


@pytest.fixture(scope="module")
def C():
    return mixed_csr(600, 500, 7, duplicates=True)


def caps_of(C):
    """Forced caps: below the longest row, exactly a giant row's length, right after the giant row 50, about 3 parts."""
    lens = np.diff(C.indptr)
    return {"below_longest": int(lens.max()) - 100, "giant_length": int(lens[50]), "after_giant": int(C.indptr[51]),
            "thirds": C.nnz // 3 + 1}


CAPS = ["below_longest", "giant_length", "after_giant", "thirds"]


def upload(lib, ctx, C, cap):
    ctx.set_knob("segment_nnz", cap)
    d = lib.DeviceCSR.upload(ctx, C)
    if cap:
        assert d.segment_count > 1
    else:
        assert d.segment_count == 1
    return d


def cholesky_half(lib, ctx, C, Y, cap, YtY=None):
    d = upload(lib, ctx, C, cap)
    Yd = lib.DeviceFactors.from_host(ctx, Y)
    X = lib.DeviceFactors(ctx, C.shape[0], Y.shape[1])
    if YtY is None:
        lib.least_squares(ctx, d, X, Yd, REG)
    else:
        lib.least_squares_with_gramian(ctx, YtY, d, X, Yd, REG)
    # the item half from the device-resident X, over the device transpose (segmented like its input)
    t = d.transpose()
    if cap:
        assert t.segment_count > 1
    Y2 = lib.DeviceFactors(ctx, C.shape[1], Y.shape[1])
    lib.least_squares(ctx, t, Y2, X, REG)
    out = X.download(), Y2.download()
    for h in (t, d, Yd, X, Y2):
        h.close()
    return out


@pytest.mark.parametrize("cap", CAPS)
def test_transpose_equals_scipy(lib, ctx, C, cap):
    want = C.T.tocsr()
    c = caps_of(C)[cap]
    d = upload(lib, ctx, C, c)
    for src in ("segmented", "single"):
        if src == "single":  # one-segment input, transposed into segmented output
            d.close()
            d = upload(lib, ctx, C, 0)
            ctx.set_knob("segment_nnz", c)
        t = d.transpose()
        assert t.segment_count > 1
        got = t.download()
        assert np.array_equal(got.indptr, want.indptr)
        assert np.array_equal(got.indices, want.indices)
        assert np.array_equal(got.data, want.data)
        back = d.download()
        assert np.array_equal(back.indptr, C.indptr) and np.array_equal(back.indices, C.indices)
        assert np.array_equal(back.data, C.data)
        t.close()
    d.close()


@pytest.mark.parametrize("f", [16, 48, 64, 100, 200])
@pytest.mark.parametrize("kind", ["cold", "mixed"])
def test_cholesky_half_bitwise(lib, ctx, C, f, kind):
    Y = factors_of(kind, C.shape[1], f, 11)
    ref = cholesky_half(lib, ctx, C, Y, 0)
    for cap in CAPS:
        got = cholesky_half(lib, ctx, C, Y, caps_of(C)[cap])
        assert np.array_equal(got[0], ref[0]), (cap, "user half")
        assert np.array_equal(got[1], ref[1]), (cap, "item half")
    YtY = (Y.astype(np.float64).T @ Y).astype(np.float32)
    ref = cholesky_half(lib, ctx, C, Y, 0, YtY)
    got = cholesky_half(lib, ctx, C, Y, caps_of(C)["thirds"], YtY)
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])


@pytest.mark.parametrize("f", [64, 200])
def test_cg_half_bitwise(lib, ctx, C, f):
    Y = factors_of("mixed", C.shape[1], f, 3)
    X0 = factors_of("mixed", C.shape[0], f, 4)

    def run(cap):
        d = upload(lib, ctx, C, cap)
        Yd, X = lib.DeviceFactors.from_host(ctx, Y), lib.DeviceFactors.from_host(ctx, X0)
        lib.least_squares_cg(ctx, d, X, Yd, REG, 3)
        out = X.download()
        for h in (d, Yd, X):
            h.close()
        return out

    ref = run(0)
    for cap in CAPS:
        assert np.array_equal(run(caps_of(C)[cap]), ref), cap


def test_loss(lib, ctx, C):
    Y = factors_of("mixed", C.shape[1], 64, 5)
    X = factors_of("mixed", C.shape[0], 64, 6)
    Yd, Xd = lib.DeviceFactors.from_host(ctx, Y), lib.DeviceFactors.from_host(ctx, X)
    d = upload(lib, ctx, C, 0)
    ref = lib.calculate_loss(ctx, d, Xd, Yd, REG)
    d.close()
    for cap in CAPS:
        d = upload(lib, ctx, C, caps_of(C)[cap])
        got = lib.calculate_loss(ctx, d, Xd, Yd, REG)
        assert abs(got - ref) <= 1e-6 * abs(ref), (cap, got, ref)
        d.close()


def test_alpha_scaling(lib, ctx, C):
    Y = factors_of("mixed", C.shape[1], 64, 8)
    out = []
    for cap in (0, caps_of(C)["thirds"]):
        d = upload(lib, ctx, C, cap)
        d.scale(3.5)
        back = d.download()
        assert np.array_equal(back.data, C.data * np.float32(3.5))
        Yd, X = lib.DeviceFactors.from_host(ctx, Y), lib.DeviceFactors(ctx, C.shape[0], 64)
        lib.least_squares(ctx, d, X, Yd, REG)
        out.append(X.download())
        for h in (d, Yd, X):
            h.close()
    assert np.array_equal(out[0], out[1])


def test_bad_row_in_second_segment(lib, ctx):
    """lambda = 0 and Y = I: a row whose three stored zeros subtract 3 e_0 e_0^T is not positive definite."""
    f, users = 16, 40
    rng = np.random.default_rng(1)
    rows, cols, vals = [], [], []
    for u in range(users):
        for i in rng.choice(f, 4, replace=False):
            rows.append(u)
            cols.append(int(i))
            vals.append(2.0)
    bad = 30
    rows += [bad] * 3
    cols += [0] * 3
    vals += [0.0] * 3
    order = np.lexsort((np.arange(len(rows)), rows))
    rows, cols, vals = np.array(rows)[order], np.array(cols)[order], np.array(vals, dtype=np.float32)[order]
    indptr = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=users))]).astype(np.int32)
    C = sp.csr_matrix((vals, cols.astype(np.int32), indptr), shape=(users, f))
    Y = np.eye(f, dtype=np.float32)
    d = upload(lib, ctx, C, C.nnz // 3 + 1)
    assert C.indptr[bad] > C.nnz // 3 + 1  # the bad row lies beyond the first segment
    Yd, X = lib.DeviceFactors.from_host(ctx, Y), lib.DeviceFactors(ctx, users, f)
    with pytest.raises(ValueError, match=f"row {bad}\\b"):
        lib.least_squares(ctx, d, X, Yd, 0.0)
    lib.gramian(ctx, Yd)
    lib.half_pregram_async(ctx, d, X, Yd, 0.0, use_cg=False)
    with pytest.raises(ValueError, match=f"row {bad}\\b"):
        lib.solver_status(ctx)
    for h in (d, Yd, X):
        h.close()


@pytest.mark.parametrize("f", [16, 64])
def test_slice_rows_across_segments(lib, ctx, C, f):
    Y = factors_of("mixed", C.shape[1], f, 9)
    cap = caps_of(C)["thirds"]
    d = upload(lib, ctx, C, cap)
    Yd = lib.DeviceFactors.from_host(ctx, Y)
    Xfull, Xsh = lib.DeviceFactors(ctx, C.shape[0], f), lib.DeviceFactors(ctx, C.shape[0], f)
    lib.least_squares(ctx, d, Xfull, Yd, REG)
    first_seg_end = int(np.searchsorted(C.indptr, cap, side="right")) - 1
    cuts = [0, first_seg_end - 7, first_seg_end + 5, C.shape[0]]  # shards that cross segment boundaries
    lib.gramian(ctx, Yd)
    for r0, r1 in zip(cuts[:-1], cuts[1:]):
        s = d.slice_rows(r0, r1)
        assert s.shape3 == (r1 - r0, C.shape[1], int(C.indptr[r1] - C.indptr[r0]))
        got = s.download()
        assert np.array_equal(got.indices, C[r0:r1].indices) and np.array_equal(got.data, C[r0:r1].data)
        lib.half_pregram(ctx, s, Xsh, Yd, REG, use_cg=False)
        s.close()
    # each shard decides its fp16 operand scale and short-row path from its own rows, like a multi-GPU shard
    assert row_err(Xsh.download(), Xfull.download()).max() < CHOL_MAX
    for h in (d, Yd, Xfull, Xsh):
        h.close()


@pytest.mark.parametrize("index_dtype", [np.int32, np.int64])
def test_upload64(lib, ctx, C, index_dtype):
    import ctypes

    def up(indptr, indices, nnz=None, cap=0):
        ctx.set_knob("segment_nnz", cap)
        h = ctypes.c_void_p()
        rc = ctx.lib.als_csr_upload64(ctx.h, C.shape[0], C.shape[1], C.nnz if nnz is None else nnz, lib.ptr(indptr),
                                      lib.ptr(indices), indices.dtype.itemsize, lib.ptr(C.data), 0, ctypes.byref(h))
        return rc, h

    indptr = C.indptr.astype(np.int64)
    indices = C.indices.astype(index_dtype)
    for cap in (0, caps_of(C)["thirds"]):
        rc, h = up(indptr, indices, cap=cap)
        assert rc == 0
        d = lib.DeviceCSR(ctx, h)
        assert (d.segment_count > 1) == (cap > 0)
        ip = np.zeros(C.shape[0] + 1, dtype=np.int64)
        ix = np.zeros(C.nnz, dtype=np.int32)
        dv = np.zeros(C.nnz, dtype=np.float32)
        lib.check(ctx.lib.als_csr_download64(ctx.h, d.h, lib.ptr(ip), lib.ptr(ix), lib.ptr(dv)))
        assert np.array_equal(ip, C.indptr) and np.array_equal(ix, C.indices) and np.array_equal(dv, C.data)
        d.close()
    for pos, v in ((17, -1), (C.nnz - 1, C.shape[1])):
        bad = indices.copy()
        bad[pos] = v
        rc, _ = up(indptr, bad)
        assert rc == lib.ALS_E_INVALID
        assert f"indices[{pos}] = {v} is outside" in ctx.lib.als_last_error().decode()
    nm = indptr.copy()
    nm[100] = nm[101] + 1
    rc, _ = up(nm, indices)
    assert rc == lib.ALS_E_INVALID and "not monotone" in ctx.lib.als_last_error().decode()
    rc, _ = up(indptr, indices, nnz=C.nnz - 1)
    assert rc == lib.ALS_E_INVALID and "!= nnz" in ctx.lib.als_last_error().decode()


def _model(lib, ctx, use_cg, f=32):
    from implicit_b200 import AlternatingLeastSquares

    m = AlternatingLeastSquares(factors=f, iterations=3, use_cg=use_cg, regularization=REG, random_state=1)
    m._ctx = ctx
    return m


@pytest.mark.parametrize("use_cg", [False, True])
def test_public_fit_bitwise(lib, ctx, C, use_cg):
    Cp = abs(C)  # the public class takes what a user passes: positive confidences
    Cp.data += np.float32(1)
    out = []
    for cap in (0, caps_of(C)["thirds"]):
        ctx.set_knob("segment_nnz", cap)
        m = _model(lib, ctx, use_cg)
        m.fit(Cp, show_progress=False)
        rec = m.recalculate_user(np.arange(0, 300), Cp[:300])
        m.partial_fit_items(np.arange(400, 650), Cp.T.tocsr()[:250])  # 150 new items
        out.append((m.user_factors.copy(), m.item_factors.copy(), rec))
    for a, b in zip(out[0], out[1]):
        assert np.array_equal(a, b)


def test_recommend_batch_split(lib, ctx, C, monkeypatch):
    from implicit_b200 import als

    Cp = abs(C)
    m = _model(lib, ctx, True)
    m.fit(Cp, show_progress=False)
    users = np.arange(0, 400)
    want = m.recommend(users, Cp[users], N=10)
    want_rec = m.recommend(users, Cp[users], N=10, recalculate_user=True)
    monkeypatch.setattr(als, "_LIKED_NNZ_MAX", 5000)  # rows 3 and 50 alone hold > 3000
    assert len(als.liked_batches(Cp[users].indptr, 5000)) > 3
    for w, got in ((want, m.recommend(users, Cp[users], N=10)),
                   (want_rec, m.recommend(users, Cp[users], N=10, recalculate_user=True))):
        assert np.array_equal(got[0], w[0]) and np.array_equal(got[1], w[1])


def test_topk_refuses_segmented_liked(lib, ctx, C):
    Y = lib.DeviceFactors.from_host(ctx, factors_of("mixed", C.shape[1], 32, 1))
    Q = lib.DeviceFactors.from_host(ctx, factors_of("mixed", C.shape[0], 32, 2))
    d = upload(lib, ctx, C, caps_of(C)["thirds"])
    with pytest.raises(lib.AlsError, match="segments"):
        lib.topk(ctx, Y, Q, 10, liked=d)
    for h in (d, Y, Q):
        h.close()


def test_two_gpu_fit_with_segments():
    from implicit_b200 import _lib

    if _lib.device_count() < 2:
        pytest.skip("needs two GPUs")
    port = 29900 + os.getpid() % 90
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port), ALS_B200_SEGMENT_NNZ="200000")
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tools", "multi_gpu_check.py")], env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=600)[0] for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o[-2000:]
        assert "MULTI_GPU_CHECK OK" in o


# ---------------------------------------------------------------------------------------- above 2^31 nonzeros
R_BLOCKS = 127


def test_fit_above_2_31_nonzeros(lib, ctx):
    import oracle

    orc = oracle.get("auto")
    import torch

    from implicit_b200 import AlternatingLeastSquares, synthetic

    base = synthetic.power_law_csr(40000, 20000, 17_000_000, 31)
    Ub, Ib = base.shape
    nnz = R_BLOCKS * base.nnz
    assert nnz >= 2**31
    free, total = torch.cuda.mem_get_info()
    need_dev = 48e9
    try:
        avail_host = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    except (ValueError, OSError):
        avail_host = 0
    need_host = 34e9
    if free < need_dev or avail_host < need_host:
        pytest.skip(f"needs {need_dev / 1e9:.0f} GB free on the device and {need_host / 1e9:.0f} GB of host memory; "
                    f"{free / 1e9:.1f} GB and {avail_host / 1e9:.1f} GB are available")
    t0 = time.perf_counter()
    Cui = synthetic.block_diagonal_tiling(base, R_BLOCKS)
    assert Cui.nnz == nnz and Cui.indices.dtype == np.int64
    f = 32

    # the device transpose: segmented both ways, indptr as predicted from the base
    d = lib.DeviceCSR.upload(ctx, Cui)
    t = d.transpose()
    assert d.segment_count >= 3 and t.segment_count >= 3
    counts = np.tile(np.bincount(base.indices, minlength=Ib), R_BLOCKS)
    assert np.array_equal(t.indptr_host(), np.concatenate([[0], np.cumsum(counts)]))
    used = free - torch.cuda.mem_get_info()[0]
    t.close()
    d.close()
    print(f"\nupload + transpose of {nnz} nonzeros: {used / 1e9:.1f} GB of device memory")

    X0, Y0 = synthetic.initial_factors(Ub, Ib, f, seed=3)
    for use_cg in (False, True):
        m = AlternatingLeastSquares(factors=f, iterations=1, use_cg=use_cg, regularization=REG)
        m._ctx = ctx
        m.user_factors = np.tile(X0, (R_BLOCKS, 1))
        m.item_factors = np.tile(Y0, (R_BLOCKS, 1))
        m.fit(Cui, show_progress=False)
        X = m.user_factors.reshape(R_BLOCKS, Ub, f)
        Y = m.item_factors.reshape(R_BLOCKS, Ib, f)
        # the per-row arithmetic does not depend on position: every block equals block 0
        assert (X == X[0]).all(), "user blocks differ"
        assert (Y == Y[0]).all(), "item blocks differ"
        if not use_cg:
            # block 0 against fp64, with the bars of the Cholesky width tests: 1.5x the fp32 reference's max and
            # median row error, floors 8e-5 and 8e-6 (fp16-split long-row kernels up to 64 padded factors).  Both the
            # truth and the reference see the whole matrix's Gramian, R Y_b^T Y_b.
            halves = ((base, np.tile(Y0, (R_BLOCKS, 1)), Y0, X[0]), (base.T.tocsr(), m.user_factors, X[0], Y[0]))
            for Cb, Yfull, Yb, got in halves:
                Y64 = Yb.astype(np.float64)
                truth = cholesky_truth(Cb, Yb, REG, YtY=R_BLOCKS * (Y64.T @ Y64))
                wide = sp.csr_matrix((Cb.data, Cb.indices, Cb.indptr), shape=(Cb.shape[0], Yfull.shape[0]))
                exp = np.zeros((Cb.shape[0], f), dtype=np.float32)
                orc.least_squares(wide, exp, np.array(Yfull, dtype=np.float32), REG)  # a writable copy
                e_ref, e = row_err(exp, truth), row_err(got, truth)
                bar_max, bar_med = max(8e-5, 1.5 * e_ref.max()), max(8e-6, 1.5 * np.median(e_ref))
                print(f"block 0 row error max {e.max():.2e} median {np.median(e):.2e}; fp32 reference "
                      f"{e_ref.max():.2e} {np.median(e_ref):.2e}")
                assert e.max() <= bar_max and np.median(e) <= bar_med
        m._ctx = None
    print(f"fit_above_2_31: {time.perf_counter() - t0:.0f} s")
