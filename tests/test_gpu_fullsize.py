"""Full-size parity (BASELINE.json configs C2, C3, C5) on the GPU against the CPU oracle: what bench.py times is
what these tests check.  Every call goes Python -> ctypes -> C-ABI -> sm_90a kernels.

  C2  (360k x 300k, 17M nnz, f=64, Cholesky): a WARM user half (after one GPU iteration) on a row sample against
      the reference's _least_squares with the same Gramian, asserted at 1e-4; and the 3-iteration fit bench.py
      times against the oracle's 3-iteration fit of the whole matrix.
  C3  (138k x 27k, 20M nnz, f=128, CG(3)): a warm CG half on a row sample (median / max per tests/helpers.py) and
      the converged 15-iteration fit (CG_CONVERGED_MAX).
  C5  (1M x 1M, f=64, k=10, liked filter): 2000 sampled query rows against the oracle's topk with the near-tie
      classification of SURVEY.md section 8(d).
  N1  als_least_squares_with_gramian against the reference's _least_squares(YtY, ...) directly.
"""
import numpy as np
import pytest

import oracle
from helpers import CG_CONVERGED_MAX, CG_MEDIAN, CG_P99, CHOL_MAX, row_err, topk_mismatches, topk_noise
from implicit_b200 import synthetic

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from implicit_b200 import _lib

    return _lib


@pytest.fixture(scope="module")
def ctx(lib):
    c = lib.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def orc():
    return oracle.get("auto")


@pytest.fixture(scope="module")
def c2():
    return synthetic.config("C2")


def _sample_rows(lens, n, seed):
    rng = np.random.default_rng(seed)
    return np.unique(np.concatenate([np.argsort(-lens)[:8], rng.choice(len(lens), n, replace=False),
                                     np.where(lens == 0)[0][:2]]))


# ---------------------------------------------------------------------------------------- C2
def test_c2_warm_half_matches_reference_at_1e4(lib, ctx, orc, c2):
    """One full GPU iteration from the cold start, then the user half of iteration 2: a 410-row sample (the longest
    rows, which take the split path, included) is re-solved by the reference's _least_squares (_als.pyx:76-142)
    from the same Y and the same Gramian."""
    Cui, X0, Y0, cfg = c2
    C = lib.DeviceCSR.upload(ctx, Cui)
    T = C.transpose()
    X, Y = lib.DeviceFactors.from_host(ctx, X0), lib.DeviceFactors.from_host(ctx, Y0)
    lib.least_squares(ctx, C, X, Y, 0.01)
    lib.least_squares(ctx, T, Y, X, 0.01)
    Y1 = Y.download()
    G = lib.gramian(ctx, Y)
    lib.least_squares(ctx, C, X, Y, 0.01)
    got = X.download()
    for h in (T, C, X, Y):
        h.close()
    lens = np.diff(Cui.indptr)
    sample = _sample_rows(lens, 400, 0)
    sub = Cui[sample]
    exp_same = np.zeros((len(sample), 64), dtype=np.float32)
    orc._least_squares(G, sub.indptr, sub.indices, sub.data.astype("float32"), exp_same, Y1, 0.01)
    exp = np.zeros((len(sample), 64), dtype=np.float32)
    orc.least_squares(sub, exp, Y1, 0.01)  # the reference's own np.dot(Y.T, Y)
    e_same, e = row_err(got[sample], exp_same), row_err(got[sample], exp)
    print(f"C2 warm user half, {len(sample)} rows (longest {lens.max()}): same Gramian max {e_same.max():.2e} median "
          f"{np.median(e_same):.2e}; reference end to end max {e.max():.2e} median {np.median(e):.2e}")
    assert e_same.max() < CHOL_MAX and np.median(e_same) < 1e-5
    assert e.max() < CHOL_MAX and np.median(e) < 1e-5


def test_c2_three_iteration_fit_matches_oracle(lib, ctx, orc, c2):
    """The fit bench.py times end to end (C2, 3 iterations, injected initial factors) against the oracle's
    3-iteration fit of the WHOLE matrix; every row of both factor matrices is compared."""
    from implicit_b200 import AlternatingLeastSquares

    Cui, X0, Y0, cfg = c2
    # The reference twice: in fp32 -- what the GPU has to match -- and in fp64 (the `floating` fused type of
    # _als.pyx:76-77), which is the ground truth both are measured against.  Three
    # iterations from this cold start (condition number ~2e2 in the first half, the reference's own sgemm Gramian off
    # by 1e-6) amplify every rounding difference ~50x, so "as close to the fp64 fit as the reference itself" is the bar
    # that means something; the row-by-row distance to the reference and the training loss are reported and bounded too.
    Xe, Ye = X0.copy(), Y0.copy()
    Xt, Yt = X0.astype(np.float64), Y0.astype(np.float64)
    for a, b in ((Xe, Ye), (Xt, Yt)):  # (one after the other: OpenBLAS aborts when two OpenMP teams call it at once)
        oracle.fit(Cui, a, b, regularization=0.01, iterations=3, use_cg=False, kind=orc.name)
    m = AlternatingLeastSquares(factors=64, regularization=0.01, use_cg=False, iterations=3)
    m.user_factors, m.item_factors = X0.copy(), Y0.copy()
    m.fit(Cui, show_progress=False)
    gx, gy = np.array(m.user_factors), np.array(m.item_factors)
    e = np.concatenate([row_err(gx, Xe), row_err(gy, Ye)])
    e_gpu = np.concatenate([row_err(gx, Xt), row_err(gy, Yt)])
    e_ref = np.concatenate([row_err(Xe, Xt), row_err(Ye, Yt)])

    def q(v):
        return f"max {v.max():.2e} p99.9 {np.quantile(v, 0.999):.2e} median {np.median(v):.2e}"

    print(f"C2 3-iteration fit, all {len(e)} rows: GPU vs fp32 reference {q(e)} (rows above 1e-4: {(e > CHOL_MAX).sum()}); "
          f"vs the fp64 reference fit: GPU {q(e_gpu)}, fp32 reference {q(e_ref)}")
    assert np.median(e_gpu) < max(1e-5, 1.5 * np.median(e_ref))
    assert np.quantile(e_gpu, 0.999) < max(CHOL_MAX, 1.5 * np.quantile(e_ref, 0.999))
    assert e_gpu.max() < max(CHOL_MAX, 1.5 * e_ref.max())
    assert np.median(e) < 1e-4 and e.max() < 1e-3
    loss_g = orc.calculate_loss(Cui, gx, gy, 0.01)
    loss_e = orc.calculate_loss(Cui, Xe, Ye, 0.01)
    print(f"   training loss: GPU factors {loss_g:.7f}, reference factors {loss_e:.7f}")
    assert abs(loss_g - loss_e) < 1e-4 * abs(loss_e)


# ---------------------------------------------------------------------------------------- C3
def test_c3_warm_cg_half_and_converged_fit(lib, ctx, orc):
    """C3 at full size.  (1) a CG(3) user half from a warm state (after one GPU iteration) on a row sample against
    the reference's least_squares_cg (_als.pyx:154-248): median / p99 / max per tests/helpers.py;
    (2) the converged 15-iteration fit against the oracle's: max <= CG_CONVERGED_MAX (SURVEY.md section 8(c))."""
    Cui, X0, Y0, cfg = synthetic.config("C3")
    f = cfg["factors"]
    C = lib.DeviceCSR.upload(ctx, Cui)
    T = C.transpose()
    X, Y = lib.DeviceFactors.from_host(ctx, X0), lib.DeviceFactors.from_host(ctx, Y0)
    for _ in range(2):  # a conditioned state: two GPU iterations
        lib.least_squares_cg(ctx, C, X, Y, 0.01, 3)
        lib.least_squares_cg(ctx, T, Y, X, 0.01, 3)
    X1, Y1 = X.download(), Y.download()
    lib.least_squares_cg(ctx, C, X, Y, 0.01, 3)
    got = X.download()
    lens = np.diff(Cui.indptr)
    sample = _sample_rows(lens, 2000, 3)
    sub = Cui[sample]
    exp = X1[sample].copy()
    orc.least_squares_cg(sub, exp, Y1, 0.01, cg_steps=3)
    e = row_err(got[sample], exp)
    print(f"C3 warm CG half, {len(sample)} rows: max {e.max():.2e} p99 {np.quantile(e, 0.99):.2e} median {np.median(e):.2e}")
    assert np.median(e) < CG_MEDIAN and np.quantile(e, 0.99) < CG_P99 and e.max() < 1e-3
    for h in (T, C, X, Y):
        h.close()
    # (2) converged: 15 iterations on both sides from the same initial factors.  Truncated CG(3) is chaotic in factor
    # space, so the yardstick is the reference against ITSELF from initial factors perturbed in the last bit (1e-7
    # relative); that needs two 15-iteration CPU fits, which is why this part runs the C3 recipe at quarter scale
    # (34.5k x 6.75k, 5M nonzeros, f = 128).
    Cui, X0, Y0, cfg = synthetic.config("C3", scale=0.25)
    C = lib.DeviceCSR.upload(ctx, Cui)
    T = C.transpose()
    X, Y = lib.DeviceFactors.from_host(ctx, X0), lib.DeviceFactors.from_host(ctx, Y0)
    for _ in range(15):
        lib.least_squares_cg(ctx, C, X, Y, 0.01, 3)
        lib.least_squares_cg(ctx, T, Y, X, 0.01, 3)
    gx, gy = X.download(), Y.download()
    for h in (T, C, X, Y):
        h.close()
    rng = np.random.default_rng(99)
    Xe, Ye = X0.copy(), Y0.copy()
    Xp = (X0 * (1 + 1e-7 * rng.standard_normal(X0.shape))).astype(np.float32)
    Yp = (Y0 * (1 + 1e-7 * rng.standard_normal(Y0.shape))).astype(np.float32)
    for a_, b_ in ((Xe, Ye), (Xp, Yp)):
        oracle.fit(Cui, a_, b_, regularization=0.01, iterations=15, use_cg=True, cg_steps=3, kind=orc.name)
    e15 = np.concatenate([row_err(gx, Xe), row_err(gy, Ye)])
    eself = np.concatenate([row_err(Xp, Xe), row_err(Yp, Ye)])
    print(f"C3 converged (15 iterations), all {len(e15)} rows: GPU vs reference max {e15.max():.2e} p99 {np.quantile(e15, 0.99):.2e} "
          f"median {np.median(e15):.2e}; reference vs itself from 1e-7-perturbed factors: max {eself.max():.2e} "
          f"p99 {np.quantile(eself, 0.99):.2e} median {np.median(eself):.2e}")
    assert np.median(e15) < max(CG_MEDIAN, 3 * np.median(eself))
    assert np.quantile(e15, 0.99) < max(CG_CONVERGED_MAX, 3 * np.quantile(eself, 0.99))
    assert e15.max() < max(10 * CG_CONVERGED_MAX, 3 * eself.max())
    # the converged objective agrees regardless of where in factor space the two runs sit
    loss_g = orc.calculate_loss(Cui, gx, gy, 0.01)
    loss_e = orc.calculate_loss(Cui, Xe, Ye, 0.01)
    print(f"   training loss: GPU factors {loss_g:.6f}, reference factors {loss_e:.6f}")
    assert abs(loss_g - loss_e) < 2e-3 * abs(loss_e)


# ---------------------------------------------------------------------------------------- C5
def test_c5_sampled_queries_match_oracle_topk(lib, ctx, orc):
    """recommend at the C5 shape (1M users x 1M items, f=64, k=10, liked items filtered): 2000 sampled query rows
    through the fused GEMM + top-k against the reference's topk (topk.pyx:15-67, select.h).  Ids must be equal
    wherever the k-th / (k+1)-th score gap exceeds fp32 summation noise; at near-ties the score at each rank must
    still match to rtol 1e-6-ish (tests/gpu_test.py:49-51 uses the same rule on tie-free inputs)."""
    Q = I = 1_000_000
    f, k, nq = 64, 10, 2000
    rng = np.random.default_rng(5)
    users = rng.standard_normal((Q, f), dtype=np.float32) * np.float32(0.1)
    items = rng.standard_normal((I, f), dtype=np.float32) * np.float32(0.1)
    rows = np.sort(np.random.default_rng(55).choice(Q, nq, replace=False)).astype(np.int32)
    liked = synthetic.power_law_csr(nq, I, 20 * nq, 5)  # the liked lists of the sampled users
    di = lib.DeviceFactors.from_host(ctx, items)
    dq = lib.DeviceFactors.from_host(ctx, users[rows])
    dl = lib.DeviceCSR.upload(ctx, liked)
    ids, sc = lib.topk(ctx, di, dq, k, liked=dl)
    for h in (dl, dq, di):
        h.close()
    eids, esc = orc.topk(items, users[rows], k, filter_query_items=liked)
    # near-tie classification: where the ids differ, the scores at that rank must agree within summation noise
    same, bad = topk_mismatches(ids, sc, eids, esc, topk_noise(users[rows], items))
    print(f"C5 sample: {nq} queries x {I} items, ids equal {same.mean():.6f}, near-tie swaps {(~same).sum() - bad.sum()}, "
          f"true mismatches {bad.sum()}; score rel err max {np.abs(sc - esc).max() / np.abs(esc).max():.2e}")
    assert bad.sum() == 0
    assert same.mean() > 0.999
    np.testing.assert_allclose(sc, esc, rtol=2e-5, atol=1e-7)


# ---------------------------------------------------------------------------------------- N1
@pytest.mark.parametrize("f", [32, 64, 128])
def test_least_squares_with_gramian_matches_reference(lib, ctx, orc, f):
    """als_least_squares_with_gramian (recalculate_user / partial_fit, implicit/cpu/als.py:221-240) against the
    reference's _least_squares(YtY, indptr, indices, data, X, Y, regularization) with the same YtY."""
    Cui = synthetic.power_law_csr(3000, 2000, 90000, 11)
    X, Y = synthetic.initial_factors(3000, 2000, f)
    oracle.fit(Cui, X, Y, iterations=2, use_cg=False, kind=orc.name)
    YtY = np.dot(Y.T, Y).astype(np.float32)
    exp = np.zeros_like(X)
    orc._least_squares(YtY, Cui.indptr, Cui.indices, Cui.data.astype("float32"), exp, Y, 0.01)
    C = lib.DeviceCSR.upload(ctx, Cui)
    dX, dY = lib.DeviceFactors.from_host(ctx, np.zeros_like(X)), lib.DeviceFactors.from_host(ctx, Y)
    lib.least_squares_with_gramian(ctx, YtY, C, dX, dY, 0.01)
    got = dX.download()
    for h in (C, dX, dY):
        h.close()
    e = row_err(got, exp)
    print(f"with_gramian f={f}: max {e.max():.2e} median {np.median(e):.2e}")
    assert e.max() < CHOL_MAX


# ---------------------------------------------------------------------------------------- tensor-core top-k at mid size
@pytest.mark.parametrize("k", [1, 10, 16])
def test_topk_tcgen05_path_matches_oracle_and_legacy_kernel(lib, ctx, orc, k):
    """The wgmma kernel (csrc/topk_tc.cu: batches of >= 1024 queries, 64 factors, k <= 16) against the reference's
    topk and against the mma.sync kernel (knob topk_legacy), with a liked CSR, a global filter list, a ragged last
    query tile and a ragged last item tile."""
    Q, I, f = 3000 + 37, 5000 + 113, 64
    rng = np.random.default_rng(100 + k)
    users = rng.standard_normal((Q, f), dtype=np.float32) * np.float32(0.3)
    items = rng.standard_normal((I, f), dtype=np.float32) * np.float32(0.3)
    liked = synthetic.power_law_csr(Q, I, 25 * Q, 9)
    flt = np.sort(rng.choice(I, 200, replace=False)).astype(np.int32)
    di, dq = lib.DeviceFactors.from_host(ctx, items), lib.DeviceFactors.from_host(ctx, users)
    dl = lib.DeviceCSR.upload(ctx, liked)
    ids, sc = lib.topk(ctx, di, dq, k, liked=dl, filter_items=flt)
    ctx.set_knob("topk_legacy", 1)
    ids_old, sc_old = lib.topk(ctx, di, dq, k, liked=dl, filter_items=flt)
    ctx.set_knob("topk_legacy", 0)
    # a row subset through query_rows (the recommend() path)
    rows = np.sort(rng.choice(Q, 1500, replace=False)).astype(np.int32)
    dl2 = lib.DeviceCSR.upload(ctx, liked[rows])
    ids_r, sc_r = lib.topk(ctx, di, dq, k, query_rows=rows, liked=dl2)
    for h in (dl2, dl, dq, di):
        h.close()
    eids, esc = orc.topk(items, users, k, filter_query_items=liked, filter_items=flt)
    same, bad = topk_mismatches(ids, sc, eids, esc, topk_noise(users, items))
    print(f"wgmma top-k k={k}: ids equal to the reference {same.mean():.6f} (true mismatches {bad.sum()}), to the mma.sync kernel "
          f"{(ids == ids_old).mean():.6f}; score rel err {np.abs(sc - esc).max() / np.abs(esc).max():.2e}")
    assert bad.sum() == 0 and same.mean() > 0.999
    np.testing.assert_allclose(sc, esc, rtol=2e-5, atol=1e-6)
    assert (ids == ids_old).mean() > 0.999
    e2, s2 = orc.topk(items, users[rows], k, filter_query_items=liked[rows])
    assert (ids_r == e2).mean() > 0.999
    np.testing.assert_allclose(sc_r, s2, rtol=2e-5, atol=1e-6)


def test_topk_tcgen05_exact_ties_follow_select_h(lib, ctx, orc):
    """Integer-valued factors make every score exact, so ties are real: ids must equal the reference's bit for bit
    (select.h: at the k-th-score boundary the smaller column wins; equal scores come out larger column first)."""
    Q, I, f, k = 2048, 4096, 64, 10
    rng = np.random.default_rng(7)
    users = rng.integers(-2, 3, size=(Q, f)).astype(np.float32)
    items = rng.integers(-2, 3, size=(I, f)).astype(np.float32)
    di, dq = lib.DeviceFactors.from_host(ctx, items), lib.DeviceFactors.from_host(ctx, users)
    ids, sc = lib.topk(ctx, di, dq, k)
    dq.close()
    di.close()
    eids, esc = orc.topk(items, users, k)
    np.testing.assert_array_equal(sc, esc)
    np.testing.assert_array_equal(ids, eids)


def test_topk_very_large_k_falls_back_to_a_full_sort(lib, ctx, orc):
    """k beyond what the shared-memory k-lists hold (~1100): scores to HBM + one stable segmented sort.  The reference's
    select.h accepts any k (rank_items, N = all items); ids and scores must match it, including the liked / filtered
    items that come back at -FLT_MAX once the unfiltered ones run out."""
    Q, I, f, k = 37, 4000, 64, 3900
    rng = np.random.default_rng(3)
    users = rng.standard_normal((Q, f), dtype=np.float32)
    items = rng.standard_normal((I, f), dtype=np.float32)
    liked = synthetic.power_law_csr(Q, I, 60 * Q, 4)
    flt = np.sort(rng.choice(I, 150, replace=False)).astype(np.int32)
    di, dq = lib.DeviceFactors.from_host(ctx, items), lib.DeviceFactors.from_host(ctx, users)
    dl = lib.DeviceCSR.upload(ctx, liked)
    ids, sc = lib.topk(ctx, di, dq, k, liked=dl, filter_items=flt)
    for h in (dl, dq, di):
        h.close()
    eids, esc = orc.topk(items, users, k, filter_query_items=liked, filter_items=flt)
    live = esc > -1e38
    np.testing.assert_allclose(sc, esc, rtol=2e-5, atol=1e-5)
    assert (ids[live] == eids[live]).mean() > 0.999
    # the filtered tail ties at -FLT_MAX: which of those items survive and in what order is pure heap semantics
    # (select.h: the first k columns fill the heap, later better items evict the smallest column first)
    np.testing.assert_array_equal(ids[~live], eids[~live])
