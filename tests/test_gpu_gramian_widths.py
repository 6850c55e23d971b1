"""The Gramian G = Y^T Y at every factor width, on every kernel path, at its partition edges and at the row counts of
real models, against fp64.

csrc/gramian.cu follows the padded width F: gramian_partial_kernel<F / 16> up to 128 (2 SMs CTAs stride over steps of
32 rows), gramian_tc_kernel on wgmma at 64 (dense.cu, from 128 rows on, unless gramian_fma is set) and
gramian_wide_kernel above 128 (one 64 x 64 tile of G per CTA and part of nparts = min(ceil(rows / 64),
4 SMs / (F / 64)^2 + 1, 64) parts of rows, staged 16 rows at a time).  Every kernel folds its fp32 register tile into a
second accumulator after at most 256 rows, and the partials are added in fp64 in a fixed order.

Error model: an fp32-faithful Gramian is the fp64 one up to a few units of 2^-24 of the sum of |terms| per entry, so
|G - G64| <= 1e-6 (|Y|^T |Y|) elementwise, on every path and at every row count: the normwise 1e-6 of C2 applied entry
by entry, which a wrong off-diagonal entry that is small next to the diagonal cannot hide under.  The worst ratio
(error / bar) of every case is printed.

From 2^20 rows on, row r of Y is row r mod PERIOD of a seeded block (PERIOD odd, so no kernel stride lines up with
it): the fp64 truth is then q G_block + G_prefix, exact to fp64 rounding, at the host cost of two passes over the block
with numpy's BLAS on one thread.  Above 128 factors those counts compare sampled columns G[:, S] = Y^T Y[:, S] against
the bar |Y|^T |Y[:, S]|, S holding the first and last column of every 64-column tile and column f - 1: every row of G
is present, so every CTA tile (bi, bj) of the wide kernel is checked, its diagonal entries included.
"""
import numpy as np
import pytest

import oracle
from helpers import KNOB_DEFAULTS, cg_truth, cholesky_truth, factors_of, mixed_csr, row_err, worst_ratio
from helpers import ctx, default_knobs, lib, orc, sm  # noqa: F401  (fixtures)
from test_gpu_cg_widths import WIDE_MAX_FACTOR, assert_branch_margin
from test_gpu_cg_widths import bars as cg_bars
from test_gpu_cholesky_wide import bars as cholesky_bars
from test_gpu_loss_widths import WIDTHS

pytestmark = pytest.mark.gpu

KINDS = ["mixed", "cold", "decades", "zero_rows"]
REL = 1e-6
MILLION = (1 << 20) + 5
TEN_MILLION = 10_000_000 + 3
#: widths that also run 10M + 3 rows (C4's user count; 1024 factors would need 40 GB of host memory)
TEN_MILLION_WIDTHS = (64, 128, 256)
#: rows of the repeating block of Y from 2^20 rows on
PERIOD = (1 << 16) + 1
CHUNK = 1 << 14


def ceil_div(a, b):
    return -(-a // b)


def padded(f):
    return 16 * ceil_div(f, 16) if f <= 128 else 128 * ceil_div(f, 128)


def paths(f):
    """{name: knobs}: the path follows the padded width, so 49..63 factors run the wgmma kernel too."""
    if padded(f) == 64:
        return {"wgmma": {}, "gramian_fma": {"gramian_fma": 1}}
    return {"fma": {}}


def wide_partition(rows, F, sm):
    """(nparts, rows_per_part) of gramian_wide_kernel, as launch_gramian computes them."""
    T = F // 64
    n = max(1, min(ceil_div(max(rows, 1), 64), 4 * sm // (T * T) + 1, 64))
    return n, ceil_div(ceil_div(max(rows, 1), n), 16) * 16


def row_counts(f, sm):
    """1 row; the wide kernel's 16-row staging +- 1; the FMA kernel's 32-row step +- 1; the wgmma box and TMA switch
    at 128 rows +- 1; then the grid edges of the path, 2^20 + 5 and, at TEN_MILLION_WIDTHS, 10M + 3."""
    F = padded(f)
    counts = [1, 15, 16, 17, 31, 32, 33, 127, 128, 129]
    if F <= 128:
        g = 2 * sm  # CTAs of gramian_partial_kernel
        counts += [32 * g, 32 * g + 1, 32 * g * 9 + 5]  # a step per CTA; CTA 0 takes two; a fold, then a ragged step
        if F == 64:
            counts += [128 * sm, 128 * (2 * sm + 1) + 37]  # wgmma: a tile per CTA; three on some, the last ragged
    else:
        cap = min(4 * sm // (F // 64) ** 2 + 1, 64)
        parts = {r: wide_partition(r, F, sm) for r in range(64 * cap + 1, 64 * cap + 4096)}
        short = next(r for r, (n, p) in parts.items() if 0 < r - (n - 1) * p < p)
        empty = [r for r, (n, p) in parts.items() if (n - 1) * p >= r]
        assert wide_partition(64 * (cap - 1) - 7, F, sm)[0] == cap - 1  # ceil(rows / 64) sets nparts
        counts += [64 * (cap - 1) - 7, short]  # ... and the last part short
        # trailing parts left empty by the rounding of rows_per_part (none exist from 768 padded factors on)
        counts += empty[:1]
        counts += [cap * 600 + 5]  # parts of 608 rows: two folds, then a run of 96 rows
    counts.append(MILLION)
    if f in TEN_MILLION_WIDTHS:
        counts.append(TEN_MILLION)
    return sorted(set(c for c in counts if c >= 1))


def sampled_columns(f):
    return sorted({c for t in range(0, f, 64) for c in (t, min(t + 63, f - 1))} | {f - 1})


def gram64(Y, cols):
    """(Y^T Y[:, cols], |Y|^T |Y[:, cols]|) in fp64, over chunks of rows."""
    f = Y.shape[1]
    G, A = np.zeros((f, len(cols))), np.zeros((f, len(cols)))
    for s in range(0, len(Y), CHUNK):
        Y64 = Y[s:s + CHUNK].astype(np.float64)
        G += Y64.T @ Y64[:, cols]
        Y64 = np.abs(Y64, out=Y64)
        A += Y64.T @ Y64[:, cols]
    return G, A


def truth(block, rows, cols):
    """(G64[:, cols], bar[:, cols]) of the Y whose row r is block[r % len(block)]."""
    q, rem = divmod(rows, len(block)) if len(block) else (0, 0)
    G, A = gram64(block[:rem], cols)
    if q:
        Gb, Ab = gram64(block, cols)
        G, A = G + q * Gb, A + q * Ab
    return G, REL * A


def upload_periodic(lib, ctx, block, rows):
    d = lib.DeviceFactors(ctx, rows, block.shape[1])
    for r0 in range(0, rows, len(block)):
        d.upload(block[:min(len(block), rows - r0)], row0=r0)
    return d


def with_knobs(ctx, knobs, fn):
    for k, v in knobs.items():
        ctx.set_knob(k, v)
    try:
        return fn()
    finally:
        for k in knobs:
            ctx.set_knob(k, KNOB_DEFAULTS[k])


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("f", WIDTHS)
def test_gramian_against_fp64(lib, ctx, sm, f, kind):
    """Every path of the width at every count of row_counts, elementwise within 1e-6 |Y|^T|Y| (every entry below 2^20
    rows and up to 128 factors, sampled columns above), and two calls on the same Y return the same bits."""
    seed = 1000 * f + KINDS.index(kind)
    big = factors_of(kind, PERIOD, f, seed)
    worst, unstable = {}, []
    for rows in row_counts(f, sm):
        block = big if rows >= MILLION else factors_of(kind, rows, f, seed + rows)
        cols = sampled_columns(f) if rows >= MILLION and f > 128 else list(range(f))
        G64, bar = truth(block, rows, cols)
        d = upload_periodic(lib, ctx, block, rows)
        for name, knobs in paths(f).items():
            G1 = with_knobs(ctx, knobs, lambda: lib.gramian(ctx, d))
            G2 = with_knobs(ctx, knobs, lambda: lib.gramian(ctx, d))
            if not np.array_equal(G1.view(np.uint32), G2.view(np.uint32)):
                unstable.append((name, rows))
            worst[(name, rows)] = worst_ratio(np.abs(G1[:, cols] - G64), bar)
        d.close()
    for (name, rows), r in sorted(worst.items()):
        print(f"Gramian f={f} {kind} {name} rows={rows}: worst |G - G64| / bar = {r:.3f}")
    bad = {key: r for key, r in worst.items() if not r <= 1.0}
    assert not bad, f"Gramian outside 1e-6 |Y|^T|Y|: {bad}"
    assert not unstable, f"two calls returned different bits: {unstable}"


def test_gramian_bits_do_not_depend_on_the_context_history(lib, sm):
    """A context that already ran other widths and row counts returns the bits of a fresh context.  The calls regrow
    gram_partials (the per-CTA partials) from nothing with a wide call, again with a wider one, then with a narrow call
    after the wide ones, and reuse a larger buffer holding another call's partials from there on.  A wide call never
    regrows it after a narrow one: nparts F^2 <= (4 SMs / T^2 + 1) 4096 T^2 stays under the 2 SMs 128^2 floats that any
    narrow or wgmma call allocates, for T = F / 64 <= 16 (asserted below)."""
    sequence = [(384, 4001, {}), (1024, 50001, {}), (128, 100003, {}), (256, 20011, {}), (64, 10007, {}),
                (64, 10007, {"gramian_fma": 1}), (16, 777, {}), (1000, 3001, {})]
    for F in range(256, 1025, 128):
        nparts, _ = wide_partition(1 << 30, F, sm)
        assert nparts * F * F < 2 * sm * 128 * 128
    used = lib.Context(0)
    try:
        differ = []
        for f, rows, knobs in sequence:
            Y = factors_of("mixed", rows, f, seed=f + rows)
            got = []
            for c in (used, None):
                c = c or lib.Context(0)
                d = lib.DeviceFactors.from_host(c, Y)
                got.append(with_knobs(c, knobs, lambda: lib.gramian(c, d)))
                d.close()
                if c is not used:
                    c.close()
            if not np.array_equal(got[0].view(np.uint32), got[1].view(np.uint32)):
                differ.append((f, rows, knobs))
        assert not differ, f"bits differ from a fresh context's: {differ}"
    finally:
        used.close()


@pytest.mark.parametrize("f", [16, 40, 63, 64, 100, 128, 256, 1024])
def test_gramian_shard_windows(lib, ctx, sm, f):
    """als_gramian_shard on windows of Y, read back with als_gramian_read, against the window's fp64 Gramian within
    1e-6 |W|^T|W| elementwise (an empty window exactly 0): starts off every 16- and 128-row boundary (the wgmma path's
    TMA map starts at an offset pointer), windows of 0 and 1 rows, fewer than 128 rows (64 factors fall back to the FMA
    kernel there), a window ending on Y's last row, and the whole of Y."""
    rows = 128 * sm + 300
    Y = factors_of("mixed", rows, f, seed=77 + f)
    windows = [(37, 128 * sm + 5), (5, 0), (rows - 1, 1), (200, 1), (19, 100), (rows - 517, 517), (1, rows - 1),
               (0, rows)]
    dY = lib.DeviceFactors.from_host(ctx, Y)
    worst = {}
    for name, knobs in paths(f).items():
        for r0, n in windows:
            G = with_knobs(ctx, knobs, lambda: (lib.gramian_shard(ctx, dY, r0, n), lib.gramian_read(ctx, dY))[1])
            G64, bar = truth(Y[r0:r0 + n], n, list(range(f)))
            worst[(name, r0, n)] = worst_ratio(np.abs(G - G64), bar)
    dY.close()
    for (name, r0, n), r in worst.items():
        print(f"Gramian shard f={f} {name} rows [{r0}, {r0 + n}): worst |G - G64| / bar = {r:.3f}")
    bad = {key: r for key, r in worst.items() if not r <= 1.0}
    assert not bad, f"shard Gramian outside 1e-6 |W|^T|W|: {bad}"


@pytest.mark.parametrize("solver", ["cholesky", "cg"])
def test_wide_half_from_a_million_rows(lib, ctx, orc, solver):
    """One xwide Cholesky half and one wide CG half at f = 256 with Y of 2^20 + 5 rows (mixed signs at the scale of a
    fitted model, test_gpu_cholesky_wide.py's warm state) and 300 users, against cholesky_truth / cg_truth given the
    chunked fp64 Gramian, under the bars of test_gpu_cholesky_wide.py / test_gpu_cg_widths.py: 1.5x the fp32
    reference's own max and median row error (CG: its max times WIDE_MAX_FACTOR), with floors 2e-5 and 2e-6.  The
    reference gets that Gramian rounded to fp32 through _least_squares, so it never forms a 2^20-row Gramian itself.
    CG starts from X0 at the scale of the solution (about 1e-4 here): from X0 at 0.1 three fp32 steps cancel a residual
    1e4 times larger than b, and the fp32 reference lands 1.4e-4 from the truth at the median.  On the host, a relative
    error of 1e-4 on G's diagonal moves the rows of either half by 1e-4, 50 times their median bar."""
    f, users, items, reg = 256, 300, MILLION, 0.01
    block = factors_of("mixed", PERIOD, f, seed=5) * np.float32(0.1)
    G64, _ = truth(block, items, list(range(f)))
    G32 = G64.astype(np.float32)
    Y = np.tile(block, (ceil_div(items, PERIOD), 1))[:items]
    Cui = mixed_csr(users, items, 31, giants=(3073, 6145), duplicates=True)
    X0 = factors_of("mixed", users, f, seed=6) * np.float32(1e-4)
    if solver == "cholesky":
        t = cholesky_truth(Cui, Y, reg, YtY=G64)
        exp = np.zeros((users, f), dtype=np.float32)
        orc._least_squares(G32, Cui.indptr, Cui.indices, Cui.data.astype(np.float32), exp, Y, reg, 0)
        bar_max, bar_med = cholesky_bars(row_err(exp, t), f)
    else:
        t, rs0, _, _ = cg_truth(Cui, X0, Y, reg, 3, YtY=G64)
        assert_branch_margin(rs0)
        exp = X0.copy()
        oracle.get("port").least_squares_cg_with_gramian(G32, Cui, exp, Y, reg, cg_steps=3)
        bar_max, bar_med = cg_bars(row_err(exp, t), WIDE_MAX_FACTOR)
    C = lib.DeviceCSR.upload(ctx, Cui)
    dY = upload_periodic(lib, ctx, block, items)
    dX = lib.DeviceFactors.from_host(ctx, X0)
    if solver == "cholesky":
        lib.least_squares(ctx, C, dX, dY, reg)
    else:
        lib.least_squares_cg(ctx, C, dX, dY, reg, 3)
    got = dX.download()
    for h in (C, dY, dX):
        h.close()
    e = row_err(got, t)
    print(f"{solver} half f={f} from {items} rows: GPU vs fp64 max {e.max():.2e} median {np.median(e):.2e}; bars "
          f"{bar_max:.2e} / {bar_med:.2e}; ratios {e.max() / bar_max:.2f} / {np.median(e) / bar_med:.2f}")
    assert np.isfinite(got).all() and e.max() <= bar_max and np.median(e) <= bar_med
