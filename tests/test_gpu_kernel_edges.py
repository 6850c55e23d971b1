"""The tensor-core kernels at their tile, ring and range edges, against fp64.

Every kernel path (and every measurement knob, which must not change results beyond fp32 rounding) is compared with
a plain fp64 computation of the same operation.  Shapes come from the device's SM count, so that CTAs get zero, one,
two and three-plus tiles, ragged last tiles and ring wrap-arounds.  Each bar is an error model stated next to it, and
the measured worst ratio (error / bar) is printed beside it.
"""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from helpers import (CG_MEDIAN, KNOB_DEFAULTS, cholesky_truth, factors_of, mixed_csr, row_err, topk_mismatches,
                     topk_noise, worst_ratio)
from helpers import ctx, default_knobs, lib, orc, sm  # noqa: F401  (fixtures)
from implicit_b200 import synthetic

pytestmark = pytest.mark.gpu


def row_counts(sm):
    """1 row; one tile +- 1; one tile per CTA; three tiles on some CTAs with a ragged last tile; about a million."""
    return [1, 127, 128, 129, 128 * sm, 128 * (2 * sm + 1) + 37, (1 << 20) + 5]


KINDS = ["mixed", "cold", "decades", "zero_rows"]


# ---------------------------------------------------------------------------------------- Gramian
def gramian_paths(f):
    if (f + 15) // 16 * 16 == 64:  # the path follows the padded width: 49..63 factors run the wgmma kernel too
        return {"wgmma": {}, "gramian_fma": {"gramian_fma": 1}}
    return {"fma": {}}


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("f", [16, 40, 49, 63, 64, 100, 128])
def test_gramian_elementwise_against_fp64(lib, ctx, sm, f, kind):
    """Error model: an fp32-faithful Gramian is the fp64 one up to a few ulps of the sum of |terms| per entry, so
    |G - G64| <= 1e-6 (|Y|^T |Y|) elementwise -- the normwise 1e-6 of C2 applied entry by entry, which a wrong
    off-diagonal entry that is small next to the diagonal cannot hide under.
    The FMA kernels (every width but 64, and gramian_fma) sum about 4000 rows per thread in fp32 at a million rows,
    whose round-to-nearest walk reaches ~sqrt(4000) ulps: there the bar is 3e-6 (measured on one H100: 2.2e-6 with row
    norms over six decades, under 1e-6 for the other data).  The wgmma kernel adds chains of 64 rows into its fp32
    accumulators and stays under 1e-6 at every size.  (An mma.sync variant measured 8-11e-6 at a million rows and was
    removed.)"""
    worst = {}
    for rows in row_counts(sm):
        Y = factors_of(kind, rows, f, seed=rows + f)
        Y64 = Y.astype(np.float64)
        G64 = Y64.T @ Y64
        A = np.abs(Y64)
        bar = 1e-6 * (A.T @ A)
        d = lib.DeviceFactors.from_host(ctx, Y)
        for name, knobs in gramian_paths(f).items():
            for k, v in knobs.items():
                ctx.set_knob(k, v)
            G = lib.gramian(ctx, d)
            for k in knobs:
                ctx.set_knob(k, KNOB_DEFAULTS[k])
            scale = 3.0 if name != "wgmma" and rows > 1e6 else 1.0
            r = worst_ratio(np.abs(G - G64), scale * bar)
            worst[(name, rows)] = r
        d.close()
    for (name, rows), r in sorted(worst.items()):
        print(f"Gramian f={f} {kind} {name} rows={rows}: worst |G - G64| / bar = {r:.3f}")
    bad = {key: r for key, r in worst.items() if not r <= 1.0}
    assert not bad, f"Gramian outside 1e-6 |Y|^T|Y|: {bad}"


def test_gramian_shard_window_feeds_the_half(lib, ctx, orc, sm):
    """als_gramian_shard on a window [37, 37 + 128 sm + 5) of Y (the TMA map starts at an offset pointer), then a
    Cholesky half with that device-resident Gramian, against cholesky_truth with the window's fp64 Gramian.
    Error model: the fp32 reference's own distance to the truth (it gets the same window Gramian), x 1.5."""
    f, r0 = 64, 37
    n = 128 * sm + 5
    items = r0 + n + 300
    rng = np.random.default_rng(21)
    Y = (rng.standard_normal((items, f)) * 0.1).astype(np.float32)
    Cui = synthetic.power_law_csr(1500, items, 30000, 22)
    Gw = Y[r0:r0 + n].astype(np.float64).T @ Y[r0:r0 + n].astype(np.float64)
    truth = cholesky_truth(Cui, Y, 0.05, YtY=Gw)
    exp = np.zeros((Cui.shape[0], f), dtype=np.float32)
    orc._least_squares(Gw.astype(np.float32), Cui.indptr, Cui.indices, Cui.data.astype(np.float32), exp, Y, 0.05)
    C = lib.DeviceCSR.upload(ctx, Cui)
    dX, dY = lib.DeviceFactors.from_host(ctx, np.zeros((Cui.shape[0], f), np.float32)), lib.DeviceFactors.from_host(ctx, Y)
    lib.gramian_shard(ctx, dY, r0, n)
    lib.half_pregram(ctx, C, dX, dY, 0.05, use_cg=False)
    got = dX.download()
    for h in (C, dX, dY):
        h.close()
    e, e_ref = row_err(got, truth), row_err(exp, truth)
    print(f"shard window [{r0}, {r0 + n}): GPU vs fp64 max {e.max():.2e} median {np.median(e):.2e}; "
          f"fp32 reference max {e_ref.max():.2e} median {np.median(e_ref):.2e}")
    assert e.max() <= max(2e-5, 1.5 * e_ref.max())
    assert np.median(e) <= max(2e-6, 1.5 * np.median(e_ref))


# ---------------------------------------------------------------------------------------- W and Z
def whitening_truth(G_dev, f, reg):
    """fp64 P = R^-1 (G + reg I = R^T R) and G^-1 from the regularised Gramian the device factorises, G + reg I
    rounded to fp32: building them from the fp64 Gramian, or adding reg in fp64, would amplify the rounding of the
    device's Gramian by cond(G + reg I) (up to ~1e3 here)."""
    Greg = (G_dev + np.float32(reg) * np.eye(f, dtype=np.float32)).astype(np.float64)
    R = np.linalg.cholesky(Greg).T
    P = np.linalg.inv(R)
    P = np.triu(P)
    return P, P @ P.T


def chunked_ratios(Y, W, Z, P, Ginv, chunk=1 << 17):
    f = Y.shape[1]
    rel = max(1e-6, (f + 2) * 2.0 ** -24)
    rw = rz = 0.0
    absP, absGi = np.abs(P), np.abs(Ginv)
    for s in range(0, len(Y), chunk):
        Y64 = Y[s:s + chunk].astype(np.float64)
        A = np.abs(Y64)
        rz = max(rz, worst_ratio(np.abs(Z[s:s + chunk] - Y64 @ Ginv), rel * (A @ absGi)))
        rw = max(rw, worst_ratio(np.abs(W[s:s + chunk] - Y64 @ P), rel * (A @ absP) + 2.0 ** -38))
    return rw, rz


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("f", [33, 48, 49, 63, 64])
def test_whitened_factors_against_fp64(lib, ctx, sm, f, kind):
    """W = Y P and Z = Y G^-1 of the short-row path (als_whitened_factors): the wgmma apply (64 padded factors,
    49..64 real ones, at least 128 rows) and the fp32 FMA tiles (whiten_fma, and every other width).
    Error model: |Z - Zt| <= e |Y||G^-1| and |W - Wt| <= e |Y||P| + 2^-38 elementwise, e = max(1e-6, (f + 2) 2^-24):
    the textbook bound of a length-f fp32 dot product plus the fp32 rounding of P or G^-1 and of the result (measured
    on one H100: Z reaches 1.2e-6 relative at a million rows, where 64M entries sample the tail).  2^-38 is the
    absolute floor of the fp16 hi / lo storage of 2^14 W (22 bits down to 2^-17 of |W| <= 1)."""
    reg = 0.01
    worst = {}
    counts = row_counts(sm) if f == 64 else row_counts(sm)[:-1]
    for rows in counts:
        Y = factors_of(kind, rows, f, seed=7 * rows + f)
        d = lib.DeviceFactors.from_host(ctx, Y)
        for fma in (0, 1):
            ctx.set_knob("whiten_fma", fma)
            W, Z = lib.whitened_factors(ctx, d, reg)
            G_dev = lib.gramian(ctx, d)
            P, Ginv = whitening_truth(G_dev, f, reg)
            worst[(fma, rows)] = chunked_ratios(Y, W, Z, P, Ginv)
        ctx.set_knob("whiten_fma", 0)
        d.close()
    for (fma, rows), (rw, rz) in sorted(worst.items()):
        print(f"W/Z f={f} {kind} whiten_fma={fma} rows={rows}: worst W ratio {rw:.3f}, Z ratio {rz:.3f}")
    bad = {key: r for key, r in worst.items() if not max(r) <= 1.0}
    assert not bad, f"W or Z outside its bar: {bad}"


# ---------------------------------------------------------------------------------------- Cholesky half, every knob
KNOB_SETTINGS = {
    "default": {},
    "short_max=0": {"short_max": 0},
    "short_max=16": {"short_max": 16},
    "short_max=32": {"short_max": 32},
    "short_serial": {"short_serial": 1},
    "whiten_fma": {"whiten_fma": 1},
    "gramian_fma": {"gramian_fma": 1},
}


@pytest.mark.parametrize("state", ["cold", "warm"])
def test_cholesky_half_under_every_knob(lib, ctx, orc, state):
    """One seeded CSR through the Cholesky half under every knob setting, against cholesky_truth.
    Error model: within 1.5x the fp32 reference's own max and median row error against the same truth, with floors
    2e-5 (max) and 2e-6 (median)."""
    users, items, f, reg = 2400, 4500, 64, 0.01
    Cui = mixed_csr(users, items, 5)
    X, Y = synthetic.initial_factors(users, items, f, seed=9)
    if state == "warm":
        pos = Cui.copy()
        pos.data = np.abs(pos.data) + 1
        oracle.fit(pos, X, Y, iterations=1, use_cg=False, kind=orc.name)
    truth = cholesky_truth(Cui, Y, reg)
    exp = np.zeros((users, f), dtype=np.float32)
    orc.least_squares(Cui, exp, Y, reg)
    e_ref = row_err(exp, truth)
    bar_max, bar_med = max(2e-5, 1.5 * e_ref.max()), max(2e-6, 1.5 * np.median(e_ref))
    C = lib.DeviceCSR.upload(ctx, Cui)
    dY = lib.DeviceFactors.from_host(ctx, Y)
    results = {}
    for name, knobs in KNOB_SETTINGS.items():
        for k, v in knobs.items():
            ctx.set_knob(k, v)
        dX = lib.DeviceFactors.from_host(ctx, np.zeros((users, f), np.float32))
        lib.least_squares(ctx, C, dX, dY, reg)
        got = dX.download()
        dX.close()
        for k in knobs:
            ctx.set_knob(k, KNOB_DEFAULTS[k])
        e = row_err(got, truth)
        results[name] = (e.max(), np.median(e), bool(np.isfinite(got).all()))
    C.close()
    dY.close()
    print(f"{state}: fp32 reference vs fp64 max {e_ref.max():.2e} median {np.median(e_ref):.2e} -> bars {bar_max:.2e} / {bar_med:.2e}")
    for name, (mx, md, fin) in results.items():
        print(f"   {name:14s} max {mx:.2e} ({mx / bar_max:.2f} of bar) median {md:.2e} ({md / bar_med:.2f} of bar)")
    bad = {n: r for n, r in results.items() if not (r[2] and r[0] <= bar_max and r[1] <= bar_med)}
    assert not bad


# ---------------------------------------------------------------------------------------- caller-supplied Gramian
@pytest.mark.parametrize("which", ["zero", "five_percent"])
def test_least_squares_with_gramian_that_does_not_bound_Y(lib, ctx, orc, which):
    """als_least_squares_with_gramian feeds the caller's YtY to the short-row path, whose fp16 storage of 2^14 W
    assumes YtY >= Y^T Y - reg I.  With YtY = 0 (W = 10 Y at reg 0.01) or the Gramian of 5% of Y's rows that premise
    fails; the result must still be the reference's (_least_squares with the same YtY).
    Error model: the fp32 reference's own distance to cholesky_truth, x 1.5 on the median (floor 2e-6) and x 3 on the
    max (floor 2e-5).  With YtY = 0 a row's normal equations are reg I plus a rank-n update (n < 64), condition
    number ~1e6, so every fp32 solve carries rounding noise of order 1e-2 on its worst rows; the worst of ~3000
    such rows is itself noisy, hence the wider factor on the max."""
    users, items, f, reg = 3000, 2000, 64, 0.01
    rng = np.random.default_rng(31)
    Cui = synthetic.power_law_csr(users, items, 30000, 32)
    lens = np.diff(Cui.indptr)
    assert (lens <= 48).sum() * 16 >= items  # enough short rows to take the short-row path
    Y = rng.standard_normal((items, f), dtype=np.float32)
    if which == "zero":
        YtY = np.zeros((f, f), dtype=np.float32)
    else:
        sub = Y[rng.random(items) < 0.05].astype(np.float64)
        YtY = (sub.T @ sub).astype(np.float32)
    truth = cholesky_truth(Cui, Y, reg, YtY=YtY)
    exp = np.zeros((users, f), dtype=np.float32)
    orc._least_squares(YtY, Cui.indptr, Cui.indices, Cui.data.astype(np.float32), exp, Y, reg)
    e_ref = row_err(exp, truth)
    C = lib.DeviceCSR.upload(ctx, Cui)
    dX, dY = lib.DeviceFactors.from_host(ctx, np.zeros((users, f), np.float32)), lib.DeviceFactors.from_host(ctx, Y)
    lib.least_squares_with_gramian(ctx, YtY, C, dX, dY, reg)
    got = dX.download()
    for h in (C, dX, dY):
        h.close()
    e = row_err(got, truth)
    print(f"YtY {which}: GPU vs fp64 max {e.max():.2e} median {np.median(e):.2e} (non-finite rows "
          f"{(~np.isfinite(got).all(axis=1)).sum()}); fp32 reference max {e_ref.max():.2e} median {np.median(e_ref):.2e}; "
          f"GPU vs reference max {row_err(got, exp).max():.2e}")
    assert np.isfinite(got).all()
    assert e.max() <= max(2e-5, 3 * e_ref.max())
    assert np.median(e) <= max(2e-6, 1.5 * np.median(e_ref))


# ---------------------------------------------------------------------------------------- CG, every cg_nv
@pytest.mark.parametrize("f", [64, 128])
@pytest.mark.parametrize("nv", [1, 2, 4])
def test_cg_half_under_cg_nv(lib, ctx, orc, f, nv):
    """The CG kernel with 1, 2 or 4 float4 words per lane against the oracle, with the bars of the CG parity tests."""
    Cui = synthetic.power_law_csr(700, 450, 12000, 200 + f, 0.05)
    X, Y = synthetic.initial_factors(700, 450, f)
    oracle.fit(Cui, X, Y, iterations=2, use_cg=False, kind=orc.name)
    exp = X.copy()
    orc.least_squares_cg(Cui, exp, Y, 0.01, cg_steps=3)
    ctx.set_knob("cg_nv", nv)
    C = lib.DeviceCSR.upload(ctx, Cui)
    dX, dY = lib.DeviceFactors.from_host(ctx, X), lib.DeviceFactors.from_host(ctx, Y)
    lib.least_squares_cg(ctx, C, dX, dY, 0.01, 3)
    got = dX.download()
    for h in (C, dX, dY):
        h.close()
    e = row_err(got, exp)
    print(f"cg_nv={nv} f={f}: max {e.max():.2e} median {np.median(e):.2e}")
    assert e.max() < 1e-4 and np.median(e) < CG_MEDIAN


# ---------------------------------------------------------------------------------------- top-k on wgmma
def _launches(ctx, fn):
    n0 = ctx.launch_count()
    out = fn()
    return out, ctx.launch_count() - n0


def _check_ids(ids, sc, eids, esc, noise, what):
    same, bad = topk_mismatches(ids, sc, eids, esc, noise)
    assert bad.sum() == 0, f"{what}: {bad.sum()} ids differ away from near-ties"
    return same


TILE_EDGE_SHAPES = [(q, i, 64) for q in (1024, 1025, 256 * 5 + 1, 256 * 5 + 128, 256 * 6 + 129)
                    for i in (256, 257, 64 * 40 + 1)] + [(1025, 257, 50), (256 * 6 + 129, 64 * 40 + 1, 50)]


@pytest.mark.parametrize("n_query,n_items,f", TILE_EDGE_SHAPES,
                         ids=[f"{q}-{i}" + ("" if f == 64 else f"-f{f}") for q, i, f in TILE_EDGE_SHAPES])
def test_topk_wgmma_tile_edges(lib, ctx, orc, n_query, n_items, f):
    """Query counts that leave a CTA's second warpgroup without queries or with one; 256 items (four tiles, no ring
    wrap), 257 and 64 m + 1 (a one-item last tile); k = 1 and 16 on the wgmma kernel and k = 17 on the mma.sync
    kernel; a liked CSR and a global filter list; 64 factors, and 50 (64 padded, 14 zero columns) at two shapes.
    Ids must equal the reference's away from near-ties (noise per row: 4 eps |q| max|i|) and the mma.sync kernel's,
    scores to rtol 2e-5."""
    rng = np.random.default_rng(n_query * 7 + n_items)
    users = (rng.standard_normal((n_query, f)) * 0.3).astype(np.float32)
    items = (rng.standard_normal((n_items, f)) * 0.3).astype(np.float32)
    liked = synthetic.power_law_csr(n_query, n_items, 8 * n_query, n_query + 1)
    flt = np.sort(rng.choice(n_items, 20, replace=False)).astype(np.int32)
    noise = topk_noise(users, items)
    di, dq, dl = lib.DeviceFactors.from_host(ctx, items), lib.DeviceFactors.from_host(ctx, users), lib.DeviceCSR.upload(ctx, liked)
    try:
        for k in (1, 16, 17):
            ctx.set_knob("topk_legacy", 1)
            (lids, lsc), n_legacy = _launches(ctx, lambda: lib.topk(ctx, di, dq, k, liked=dl, filter_items=flt))
            ctx.set_knob("topk_legacy", 0)
            (ids, sc), n_default = _launches(ctx, lambda: lib.topk(ctx, di, dq, k, liked=dl, filter_items=flt))
            assert (n_default == n_legacy) == (k > 16), f"k={k}: the wgmma kernel must run exactly when k <= 16"
            eids, esc = orc.topk(items, users, k, filter_query_items=liked, filter_items=flt)
            same = _check_ids(ids, sc, eids, esc, noise, f"k={k} vs reference")
            _check_ids(ids, sc, lids, lsc, noise, f"k={k} vs mma.sync")
            np.testing.assert_allclose(sc, esc, rtol=2e-5, atol=1e-6)
            assert not np.isin(ids, flt).any()
            print(f"top-k Q={n_query} I={n_items} k={k}: ids equal {same.mean():.5f}, launches {n_default} (mma.sync {n_legacy})")
    finally:
        for h in (dl, dq, di):
            h.close()


def test_topk_wgmma_row_with_exactly_k_unfiltered_items(lib, ctx, orc):
    """The wgmma kernel skips filtered items instead of ranking them at -FLT_MAX, which is exact while every row keeps
    k unfiltered items; the dispatch bound is I - n_filter - longest liked row >= k.  At equality one row has exactly
    k candidates: its ids must be exactly the reference's set, its scores the reference's."""
    f, k, Q, I = 64, 16, 1100, 256
    rng = np.random.default_rng(77)
    users = (rng.standard_normal((Q, f)) * 0.3).astype(np.float32)
    items = (rng.standard_normal((I, f)) * 0.3).astype(np.float32)
    flt = np.sort(rng.choice(I, 40, replace=False)).astype(np.int32)
    rest = np.setdiff1d(np.arange(I), flt)
    lists = [np.sort(rng.choice(rest, rng.integers(0, 30), replace=False)) for _ in range(Q)]
    lists[5] = np.sort(rng.choice(rest, I - 40 - k, replace=False))  # exactly k unfiltered items left
    indptr = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int32)
    liked = sp.csr_matrix((np.ones(indptr[-1], np.float32), np.concatenate(lists).astype(np.int32), indptr), shape=(Q, I))
    di, dq, dl = lib.DeviceFactors.from_host(ctx, items), lib.DeviceFactors.from_host(ctx, users), lib.DeviceCSR.upload(ctx, liked)
    ctx.set_knob("topk_legacy", 1)
    _, n_legacy = _launches(ctx, lambda: lib.topk(ctx, di, dq, k, liked=dl, filter_items=flt))
    ctx.set_knob("topk_legacy", 0)
    (ids, sc), n_default = _launches(ctx, lambda: lib.topk(ctx, di, dq, k, liked=dl, filter_items=flt))
    for h in (dl, dq, di):
        h.close()
    assert n_default != n_legacy  # the bound holds with equality: the wgmma kernel runs
    eids, esc = orc.topk(items, users, k, filter_query_items=liked, filter_items=flt)
    assert sorted(ids[5]) == sorted(eids[5]) == sorted(np.setdiff1d(rest, lists[5]))
    np.testing.assert_allclose(sc[5], esc[5], rtol=2e-5, atol=1e-6)
    _check_ids(ids, sc, eids, esc, topk_noise(users, items), "exact-k case")


def test_topk_wgmma_query_rows_with_repeats(lib, ctx, orc):
    f, k = 64, 10
    rng = np.random.default_rng(78)
    users = (rng.standard_normal((700, f)) * 0.3).astype(np.float32)
    items = (rng.standard_normal((3000, f)) * 0.3).astype(np.float32)
    rows = rng.integers(0, 700, size=1300).astype(np.int32)  # many repeats, 1300 >= 1024 queries
    di, dq = lib.DeviceFactors.from_host(ctx, items), lib.DeviceFactors.from_host(ctx, users)
    ids, sc = lib.topk(ctx, di, dq, k, query_rows=rows)
    di.close()
    dq.close()
    eids, esc = orc.topk(items, users[rows], k)
    _check_ids(ids, sc, eids, esc, topk_noise(users[rows], items), "query_rows")
    np.testing.assert_allclose(sc, esc, rtol=2e-5, atol=1e-6)
    first = {}
    for n, r in enumerate(rows):  # a repeated row gives the same answer every time
        if r in first:
            np.testing.assert_array_equal(ids[n], ids[first[r]])
        first.setdefault(r, n)


@pytest.mark.parametrize("k,f", [(1, 64), (16, 64), (1, 50), (16, 50)], ids=["1", "16", "1-f50", "16-f50"])
def test_topk_wgmma_small_query_norms_against_fp64(lib, ctx, k, f):
    """Query rows at 10^U(-6, 0) of the largest one, at 64 factors and at 50 (64 padded).  Error model: the score of
    every returned id is the fp64 product to within 4 eps |q| max|i| (per query row: the kernel must keep its
    relative accuracy however small a query is next to the others; the item side is absolute, DESIGN.md section 4.3);
    ids equal the fp64 top-k and the mma.sync kernel's away from near-ties."""
    Q, I = 1500, 2000
    rng = np.random.default_rng(79 + k + f)
    users = rng.standard_normal((Q, f)).astype(np.float32)
    users = (users * 10.0 ** rng.uniform(-6, 0, size=(Q, 1))).astype(np.float32)
    items = rng.standard_normal((I, f)).astype(np.float32)
    S = users.astype(np.float64) @ items.astype(np.float64).T
    eids = np.argsort(-S, axis=1, kind="stable")[:, :k]
    esc = np.take_along_axis(S, eids, axis=1)
    noise = topk_noise(users, items)
    di, dq = lib.DeviceFactors.from_host(ctx, items), lib.DeviceFactors.from_host(ctx, users)
    ids, sc = lib.topk(ctx, di, dq, k)
    ctx.set_knob("topk_legacy", 1)
    lids, lsc = lib.topk(ctx, di, dq, k)
    ctx.set_knob("topk_legacy", 0)
    di.close()
    dq.close()
    err = np.abs(sc - np.take_along_axis(S, ids, axis=1)) / noise
    lerr = np.abs(lsc - np.take_along_axis(S, lids, axis=1)) / noise
    print(f"small query norms k={k}: worst |score - fp64| / (4 eps |q| max|i|): wgmma {err.max():.3f}, mma.sync {lerr.max():.3f}")
    assert err.max() <= 1.0 and lerr.max() <= 1.0
    _check_ids(ids, sc, eids, esc, noise, "vs fp64")
    _check_ids(ids, sc, lids, lsc, noise, "vs mma.sync")


# ---------------------------------------------------------------------------------------- unsorted liked lists
@pytest.mark.parametrize("path", ["mma_sync", "wgmma", "by_sort"])
def test_topk_unsorted_liked_with_duplicates(lib, ctx, orc, path):
    """The ABI takes any liked CSR; the reference filters batch_distances[i, liked.indices] (topk.pyx:51-54), which
    does not care about order or repeats.  Each row's columns reversed, with duplicates, through the mma.sync kernel
    (a small batch), the wgmma kernel (a large one at 64 factors) and the full sort (k > 1100)."""
    f = 64
    Q, I, k = {"mma_sync": (200, 3000, 10), "wgmma": (1100, 3000, 10), "by_sort": (37, 3000, 1200)}[path]
    rng = np.random.default_rng(81)
    users = (rng.standard_normal((Q, f)) * 0.3).astype(np.float32)
    items = (rng.standard_normal((I, f)) * 0.3).astype(np.float32)
    base = synthetic.power_law_csr(Q, I, 40 * Q, 82)
    lists = []
    for q in range(Q):
        cols = base.indices[base.indptr[q]:base.indptr[q + 1]][::-1]
        if len(cols) > 2:
            cols = np.concatenate([cols[:2], cols])  # duplicates, still descending at the front
        lists.append(cols)
    indptr = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int32)
    liked = sp.csr_matrix((np.ones(indptr[-1], np.float32), np.concatenate(lists).astype(np.int32), indptr), shape=(Q, I))
    assert not liked.has_sorted_indices
    di, dq, dl = lib.DeviceFactors.from_host(ctx, items), lib.DeviceFactors.from_host(ctx, users), lib.DeviceCSR.upload(ctx, liked)
    ids, sc = lib.topk(ctx, di, dq, k, liked=dl)
    ids2, sc2 = lib.topk(ctx, di, dq, k, liked=dl)  # the second call reuses what the first one learnt
    for h in (dl, dq, di):
        h.close()
    eids, esc = orc.topk(items, users, k, filter_query_items=base)
    leaked = sum(np.isin(ids[q][sc[q] > -1e38], lists[q]).sum() for q in range(Q))
    print(f"unsorted liked, {path}: liked items returned {leaked}")
    assert leaked == 0
    np.testing.assert_array_equal(ids, ids2)
    np.testing.assert_allclose(sc, esc, rtol=2e-5, atol=1e-6)
    _check_ids(ids, sc, eids, esc, topk_noise(users, items), path)
