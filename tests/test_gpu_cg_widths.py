"""The CG half at every factor width, under every cg_nv setting, at its early exits and schedule edges, against fp64.

csrc/cg.cu follows the padded width ld = 16 ceil(f / 16): up to 128 it compiles run_cg<ld, NV> with NV = 1, 2 or 4
float4 words per lane (knob cg_nv), in lane groups of L = ld / (4 NV) lanes rounded up to a power of two, so that the
words of some lanes are masked (Lane::ok) at ld = 48, 80, 96 and 112; above 128 it runs run_cg<ld, ld / 128> for
ld = 256 ... 1024.  Rows past 3072 nonzeros are walked in 2048-nonzero chunks whose partial sums a per-row combine
kernel adds up, with a per-row done flag once the row's CG stopped.  Every class runs at its full width and below it.

The yardstick is tests/helpers.cg_truth, the reference's recurrences in fp64.  Bars are 1.5x the fp32 reference's
own median row error and MAX_FACTOR (WIDE_MAX_FACTOR above 128) times its max row error against that truth, with the
floors of the Cholesky modules (2e-5, 2e-6): truncated CG amplifies rounding (up to 7e-4 of a row at iteration 1),
so the reference term sets the bar wherever it is larger than the floors.  The measured worst ratios are printed per case.  Every case asserts that no row's fp64 initial
residual r.r lies within a factor 100 of the 1e-20 skip threshold, so that a branch decided differently in fp32 and
in fp64 cannot pass for a kernel error.
"""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from helpers import KNOB_DEFAULTS, cg_truth, cholesky_truth, mixed_csr, row_err
from helpers import ctx, default_knobs, lib, orc, sm  # noqa: F401  (fixtures)
from implicit_b200 import synthetic

pytestmark = pytest.mark.gpu

#: every ld / 16 class 1 .. 8 at its full width and below it (the Cholesky width module's), plus 81 and 95
WIDTHS = [1, 15, 16, 17, 31, 32, 40, 48, 49, 56, 63, 64, 65, 79, 80, 81, 95, 96, 100, 112, 127, 128]
#: every ld / 128 class 2 .. 8 at its full width and below it
WIDE = [129, 256, 257, 384, 385, 512, 513, 640, 641, 768, 769, 896, 897, 1024]
#: the largest whole row, then giant rows of 2, 4 and 10 chunks of 2048 (kSplitNnz, kChunkNnz in csrc/common.h), and
#: six more giant rows: nine in all, so that the combine grid (8 rows per CTA) has a second, ragged CTA
GIANTS = (3072, 3073, 6145, 20000, 3073, 4097, 3500, 8193, 3100, 5000)
REG = 0.01


#: factor on the fp32 reference's own worst row error.  1.5x holds for the median everywhere (worst measured ratio
#: 0.95 of the bar); the worst row is a noisier statistic.  Measured on one H100 80GB HBM3 at 400 W: up to 3.35x the
#: reference's worst row at 128 factors or fewer (f = 17 cold, cg_nv = 4; 2.4e-4 there) and 10.4x above (f = 896
#: warm, where the reference's own worst row is already 2.3e-2).  Those rows' normal equations are made nearly
#: singular by weights |c| - 1 < 0 (stored zeros, |c| < 1) on a near rank-one Y; three CG steps from there amplify
#: rounding by orders of magnitude, so two correct fp32 summation orders land far apart on them (not isolated
#: further).  The factors below keep a margin of 1.2x over those measurements.
MAX_FACTOR, WIDE_MAX_FACTOR = 4.0, 12.5
#: floor of the item half's max bar, 4x the fp32 floor.  A cold user half leaves X with some rows far off (see above);
#: the device forms X^T X with fp32 FMA chains (1e-6 |X|^T |X| elementwise, test_gpu_gramian_widths.py), the reference
#: with a blocked BLAS product.  Measured on one H100 80GB HBM3 at 400 W: up to 4.2e-5 (f = 64 cold) where the
#: reference's worst item row is 6.5e-6; medians stay at 0.13 ... 0.16 of their bar.
ITEM_MAX_FLOOR = 8e-5


def bars(e_ref, max_factor=MAX_FACTOR):
    return max(2e-5, max_factor * e_ref.max()), max(2e-6, 1.5 * np.median(e_ref))


def assert_branch_margin(rs0):
    """Every row's fp64 r.r before the first step is 0 or at least 100x away from 1e-20 on either side."""
    near = (rs0 != 0) & (rs0 > 1e-22) & (rs0 < 1e-18)
    assert not near.any(), f"rows with r.r within 100x of 1e-20: {np.nonzero(near)[0][:10]} {rs0[near][:10]}"


def check(got, truth, bar_max, bar_med, empty):
    """(max, median, ok): finite, within the bars, empty rows exactly zero."""
    e = row_err(got, truth)
    ok = bool(np.isfinite(got).all()) and e.max() <= bar_max and np.median(e) <= bar_med and bool(np.all(got[empty] == 0))
    return e.max() / bar_max, np.median(e) / bar_med, ok


def cg_gpu(lib, ctx, C, X0, dY, steps, nv=None, keep=False, reg=REG):
    """One CG half on the device from X0 (every row is written or kept: X0 is the warm start)."""
    if nv is not None:
        ctx.set_knob("cg_nv", nv)
    dX = lib.DeviceFactors.from_host(ctx, X0)
    lib.least_squares_cg(ctx, C, dX, dY, reg, steps)
    ctx.set_knob("cg_nv", KNOB_DEFAULTS["cg_nv"])
    got = dX.download()
    if keep:
        return got, dX
    dX.close()
    return got


def start_state(orc, Cui, f, state, users, items, seed):
    X, Y = synthetic.initial_factors(users, items, f, seed=seed)
    if state == "warm":  # one reference CG iteration on |c| + 1
        pos = Cui.copy()
        pos.data = np.abs(pos.data) + 1
        oracle.fit(pos, X, Y, iterations=1, use_cg=True, kind=orc.name)
    return X, Y


def reference(orc, Cui, X0, Y, steps=3, max_factor=MAX_FACTOR):
    """(truth, bars, the fp32 reference's row errors) of one CG half from X0."""
    truth, rs0, stop, _ = cg_truth(Cui, X0, Y, REG, steps)
    assert_branch_margin(rs0)
    exp = X0.copy()
    orc.least_squares_cg(Cui, exp, Y, REG, cg_steps=steps)
    e_ref = row_err(exp, truth)
    return truth, bars(e_ref, max_factor), e_ref


def halves(lib, ctx, orc, Cui, X0, Y, nvs, pregram):
    """The user half under each cg_nv, the pregram entry on a window of Y, and the item half from the device-resident
    X of the default run.  Returns {name: (max ratio, median ratio, ok)} and the printed bars."""
    users, items = Cui.shape
    f = Y.shape[1]
    mf = MAX_FACTOR if f <= 128 else WIDE_MAX_FACTOR
    empty = np.diff(Cui.indptr) == 0
    truth, (bar_max, bar_med), e_ref = reference(orc, Cui, X0, Y, max_factor=mf)
    C = lib.DeviceCSR.upload(ctx, Cui)
    dY = lib.DeviceFactors.from_host(ctx, Y)
    results, dX_default, X_default = {}, None, None
    for nv in nvs:
        if nv == KNOB_DEFAULTS["cg_nv"] or nv is None:
            got, dX_default = cg_gpu(lib, ctx, C, X0, dY, 3, nv, keep=True)
            X_default = got
        else:
            got = cg_gpu(lib, ctx, C, X0, dY, 3, nv)
        results[f"cg_nv={nv}" if nv else "default"] = check(got, truth, bar_max, bar_med, empty)
    notes = [f"fp32 reference vs fp64 max {e_ref.max():.2e} median {np.median(e_ref):.2e} -> bars {bar_max:.2e} / "
             f"{bar_med:.2e}"]
    if pregram:  # als_gramian_shard on a window of Y, then the CG half with that device-resident Gramian
        r0, n = 37, items // 2
        Gw = Y[r0:r0 + n].astype(np.float64).T @ Y[r0:r0 + n].astype(np.float64)
        truth_w, rs0_w, _, _ = cg_truth(Cui, X0, Y, REG, 3, YtY=Gw)
        assert_branch_margin(rs0_w)
        exp_w = X0.copy()
        oracle.get("port").least_squares_cg_with_gramian(Gw.astype(np.float32), Cui, exp_w, Y, REG, cg_steps=3)
        bw = bars(row_err(exp_w, truth_w), mf)
        dX = lib.DeviceFactors.from_host(ctx, X0)
        lib.gramian_shard(ctx, dY, r0, n)
        lib.half_pregram(ctx, C, dX, dY, REG, use_cg=True, cg_steps=3)
        results["pregram"] = check(dX.download(), truth_w, *bw, empty)
        dX.close()
        notes.append(f"pregram window [{r0}, {r0 + n}) bars {bw[0]:.2e} / {bw[1]:.2e}")
    C.close()
    dY.close()
    # the item half, from the X the default run left on the device: non-zero padding columns there would enter this
    # half's Gramian and dot products, which a download cannot show
    Ciu = Cui.T.tocsr()
    truth_i, bi, _ = reference(orc, Ciu, Y, X_default, max_factor=mf)
    bi = (max(ITEM_MAX_FLOOR, bi[0]), bi[1])
    Ci = lib.DeviceCSR.upload(ctx, Ciu)
    dYn = lib.DeviceFactors.from_host(ctx, Y)
    lib.least_squares_cg(ctx, Ci, dYn, dX_default, REG, 3)
    results["item half"] = check(dYn.download(), truth_i, *bi, np.diff(Ciu.indptr) == 0)
    for h in (Ci, dYn, dX_default):
        h.close()
    notes.append(f"item half bars {bi[0]:.2e} / {bi[1]:.2e}")
    assert f == X_default.shape[1]
    return results, notes


def report(tag, results, notes):
    print(f"{tag}: " + "; ".join(notes))
    for name, (rmax, rmed, ok) in results.items():
        print(f"   {name:10s} worst ratio max {rmax:.2f} median {rmed:.2f} {'' if ok else 'FAIL'}")
    bad = {n: r for n, r in results.items() if not r[2]}
    assert not bad, f"{tag}: {bad}"


@pytest.mark.parametrize("state", ["cold", "warm"])
@pytest.mark.parametrize("f", WIDTHS)
def test_cg_half_at_every_width(lib, ctx, orc, f, state):
    """One seeded CSR (rows at every short-class boundary, empty rows, negative confidences, weights below zero,
    stored zeros, duplicates, the largest whole row and nine giant rows of 2 ... 10 chunks) through the user half
    under cg_nv = 1, 2 and 4, then the pregram entry on a window of Y and the item half from the device-resident X,
    each against cg_truth at cg_steps = 3 from the same start.  Every row must be finite, empty rows exactly zero."""
    users, items = 2400, 6000
    Cui = mixed_csr(users, items, 70 + f, giants=GIANTS, duplicates=True)
    assert (np.diff(Cui.indptr) > 3072).sum() >= 9
    X0, Y = start_state(orc, Cui, f, state, users, items, seed=f)
    results, notes = halves(lib, ctx, orc, Cui, X0, Y, (1, 2, 4), pregram=True)
    report(f"f={f} {state}", results, notes)


@pytest.mark.parametrize("state", ["cold", "warm"])
@pytest.mark.parametrize("f", WIDE)
def test_wide_cg_half_against_fp64(lib, ctx, orc, f, state):
    """The wide kernels (a whole warp per nonzero, ld / 128 float4 words per lane; cg_nv does not apply) on a
    smaller CSR of the same kinds, with empty rows and giant rows of 2 and 3 chunks: both halves against cg_truth,
    and the pregram entry at f = 513."""
    users, items = 600, 1500
    Cui = mixed_csr(users, items, 170 + f, giants=(3072, 3073, 6145), duplicates=True)
    X0, Y = start_state(orc, Cui, f, state, users, items, seed=f)
    results, notes = halves(lib, ctx, orc, Cui, X0, Y, (None,), pregram=f == 513)
    report(f"f={f} {state}", results, notes)


# ---------------------------------------------------------------------------------------- cg_steps
@pytest.mark.parametrize("f", [16, 80, 128, 200])
def test_cg_steps_against_fp64(lib, ctx, orc, f):
    """cg_steps = 0 (X unchanged bit for bit except that empty rows become zero), 1 and 3 against cg_truth; then
    3f steps (converged: most rows leave the loop on rsnew < 1e-20, whole rows and giant rows alike) against
    cholesky_truth, with 1.5x the fp32 reference's own distance to that solution as the bar (floors 2e-5, 2e-6)."""
    users, items = 500, 1500
    Cui = mixed_csr(users, items, 300 + f, giants=(3073, 6145), duplicates=True)
    empty = np.diff(Cui.indptr) == 0
    rng = np.random.default_rng(f)
    Y = (rng.standard_normal((items, f)) * 0.1).astype(np.float32)  # well conditioned: CG converges within 3f steps
    X0 = (rng.standard_normal((users, f)) * 0.1).astype(np.float32)
    C = lib.DeviceCSR.upload(ctx, Cui)
    dY = lib.DeviceFactors.from_host(ctx, Y)
    results = {}
    got0 = cg_gpu(lib, ctx, C, X0, dY, 0)
    results["steps=0"] = (0.0, 0.0, bool(np.array_equal(got0[~empty], X0[~empty]) and np.all(got0[empty] == 0)))
    for steps in (1, 3):
        truth, (bm, bd), _ = reference(orc, Cui, X0, Y, steps)
        results[f"steps={steps}"] = check(cg_gpu(lib, ctx, C, X0, dY, steps), truth, bm, bd, empty)
    steps = 3 * f
    chol = cholesky_truth(Cui, Y, REG)
    _, rs0, stop, _ = cg_truth(Cui, X0, Y, REG, steps)
    assert_branch_margin(rs0)
    broke = (stop < steps) & ~empty
    assert broke.sum() > 0.9 * (~empty).sum() and broke[np.diff(Cui.indptr) > 3072].all()
    exp = X0.copy()
    orc.least_squares_cg(Cui, exp, Y, REG, cg_steps=steps)
    bm, bd = bars(row_err(exp, chol))
    results[f"steps={steps}"] = check(cg_gpu(lib, ctx, C, X0, dY, steps), chol, bm, bd, empty)
    C.close()
    dY.close()
    report(f"f={f} (converged bars {bm:.2e} / {bd:.2e}; rows that broke on rsnew: {broke.sum()})", results, [])


# ---------------------------------------------------------------------------------------- early exits
def early_exit_case(f, seed):
    """Y spans e0 and e1 only (e0-items at 5e-10 ... 1e-9, e1-items three times larger) and reg = 0: rows observing only
    e0-items converge in one step, rows observing both (half and half) in two, since A = Y^T Y + W is diagonal and r0
    lies in span(e0, e1).  Before the last step r.r is above 1e-15; after it, of order (2^-24)^2 r0.r0, below 1e-22 in
    fp32 as in fp64.  Rows observing only zero items, with x0 = 5 e2 (reg = 0 and the Gramian's row 2 is zero, so
    r = 0 exactly), take the rsold skip.  Every kind as whole rows (40 nonzeros) and as giant rows (3500: two
    chunks).  Returns (Cui, X0, Y, kind per row)."""
    rng = np.random.default_rng(seed)
    n_pool = 1000
    Y = np.zeros((3 * n_pool, f), dtype=np.float32)
    Y[n_pool:2 * n_pool, 0] = 5e-10 * (1 + rng.random(n_pool))
    Y[2 * n_pool:, 1] = 1.5e-9 * (1 + rng.random(n_pool))
    kinds = ["skip", "one", "two"] * 12
    lens = [3500 if u % 4 == 3 else 40 for u in range(len(kinds))]
    cols, indptr = [], [0]
    pools = [np.arange(n_pool), np.arange(n_pool, 2 * n_pool), np.arange(2 * n_pool, 3 * n_pool)]
    for kind, n in zip(kinds, lens):
        if kind == "two":
            c = np.concatenate([rng.choice(pools[1], n // 2, replace=True), rng.choice(pools[2], n - n // 2, replace=True)])
        else:
            c = rng.choice(pools[0 if kind == "skip" else 1], n, replace=True)
        cols.append(c)
        indptr.append(indptr[-1] + n)
    vals = (1 + 4 * rng.random(indptr[-1])).astype(np.float32)
    Cui = sp.csr_matrix((vals, np.concatenate(cols).astype(np.int32), np.array(indptr, dtype=np.int32)),
                        shape=(len(kinds), 3 * n_pool))
    X0 = np.zeros((len(kinds), f), dtype=np.float32)
    X0[np.array(kinds) == "skip", 2] = 5.0
    return Cui, X0, Y, np.array(kinds)


@pytest.mark.parametrize("f,nv", [(48, 1), (48, 2), (48, 4), (80, 1), (80, 4), (300, None)])
def test_cg_early_exits(lib, ctx, orc, f, nv):
    """The rsold < 1e-20 skip (X bit for bit unchanged) and the rsnew < 1e-20 break after step 1 or 2, on whole rows
    and on giant rows (chunk + combine kernels and the done flag: a giant row that ignored its flag would take a third
    step from stale state), under cg_nv = 1, 2, 4 and on the wide kernel, against cg_truth at cg_steps = 3."""
    Cui, X0, Y, kinds = early_exit_case(f, 7 + f)
    truth, rs0, stop, rs_last = cg_truth(Cui, X0, Y, 0.0, 3)
    assert np.all(rs0[kinds == "skip"] == 0) and np.all(stop[kinds == "skip"] == 0)
    assert np.all(rs0[kinds != "skip"] > 1e-18)
    assert np.all(stop[kinds == "one"] == 1) and np.all(stop[kinds == "two"] == 2)
    assert np.all(rs_last[kinds != "skip"] < 1e-22)
    exp = X0.copy()
    orc.least_squares_cg(Cui, exp, Y, 0.0, cg_steps=3)
    bm, bd = bars(row_err(exp, truth))
    C = lib.DeviceCSR.upload(ctx, Cui)
    dY = lib.DeviceFactors.from_host(ctx, Y)
    got = cg_gpu(lib, ctx, C, X0, dY, 3, nv, reg=0.0)
    C.close()
    dY.close()
    giant = np.diff(Cui.indptr) > 3072
    results = {"skip rows unchanged": (0.0, 0.0, bool(np.array_equal(got[kinds == "skip"], X0[kinds == "skip"])))}
    for kind in ("one", "two"):
        for where, sel in (("whole", ~giant), ("giant", giant)):
            rows = (kinds == kind) & sel
            results[f"{kind} {where}"] = check(got[rows], truth[rows], bm, bd, np.zeros(rows.sum(), bool))
    report(f"f={f} cg_nv={nv} bars {bm:.2e} / {bd:.2e}", results, [])


# ---------------------------------------------------------------------------------------- schedule edges
@pytest.mark.parametrize("f", [16, 96, 256])
def test_cg_schedule_edges(lib, ctx, orc, sm, f):
    """More whole-row work items than cg_rows_kernel's capped grid has warps (6 SMs x 8) and more chunk slots than
    cg_chunk_kernel's grid has warps (the same cap): both grid-stride loops wrap.  Giant rows of 3073 nonzeros (two
    slots each), short rows of 1 ... 40; against cg_truth at cg_steps = 2."""
    warps = 6 * sm * 8
    n_giant, n_short = warps // 2 + 3, warps + 101
    rng = np.random.default_rng(f)
    lens = np.concatenate([np.full(n_giant, 3073), rng.integers(1, 41, n_short), np.zeros(50, np.int64)])
    rng.shuffle(lens)
    items = 4000
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    nnz = int(indptr[-1])
    vals = (1 + 4 * rng.random(nnz)).astype(np.float32)
    vals[rng.random(nnz) < 0.1] *= -1
    Cui = sp.csr_matrix((vals, rng.integers(0, items, nnz).astype(np.int32), indptr), shape=(len(lens), items))
    X0, Y = synthetic.initial_factors(len(lens), items, f, seed=f)
    assert 2 * n_giant > warps and (lens <= 3072).sum() > warps
    truth, _, e_ref = reference(orc, Cui, X0, Y, steps=2)
    C = lib.DeviceCSR.upload(ctx, Cui)
    dY = lib.DeviceFactors.from_host(ctx, Y)
    got = cg_gpu(lib, ctx, C, X0, dY, 2)
    C.close()
    dY.close()
    giant = lens > 3072
    results, notes = {}, []
    for where, sel in (("whole rows", ~giant), ("giant rows", giant)):  # giant rows carry more rounding: own bars
        bm, bd = bars(e_ref[sel])
        results[where] = check(got[sel], truth[sel], bm, bd, lens[sel] == 0)
        notes.append(f"{where} bars {bm:.2e} / {bd:.2e}")
    report(f"f={f} sm={sm}: {n_short} short rows, {2 * n_giant} chunk slots, {warps} warps", results, notes)
