"""The Cholesky half at every factor width, and across the range of the long-row kernels' fp16 operand scale, against
fp64.

The kernel follows the padded width ld = 16 ceil(f / 16): ld / 16 = 1 .. 4 run the mma.sync long-row kernel of
cholesky.cu (with the short-row path of cholesky_short.cu from ld = 32, on the wgmma pre-pass at ld = 64), 5 .. 8 the
wide kernel of cholesky_wide.cu.  Every class runs at its full width and below it, so that zero padding columns ride
along.  Bars are those of the edge module's Cholesky tests, 1.5x the fp32 reference's own max and median row error
against the same fp64 truth, with floors scaled to the precision of each kernel's operands (bars()).
"""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from helpers import KNOB_DEFAULTS, cholesky_truth, mixed_csr, row_err
from helpers import ctx, default_knobs, lib, orc  # noqa: F401  (fixtures)
from implicit_b200 import synthetic

pytestmark = pytest.mark.gpu

#: every ld / 16 class 1 .. 8 at its full width and below it
WIDTHS = [1, 15, 16, 17, 31, 32, 40, 48, 49, 56, 63, 64, 65, 79, 80, 96, 100, 112, 127, 128]
#: giant rows: the largest whole row, then 2, 4 and 10 chunks of 2048 (kSplitNnz, kChunkNnz in csrc/common.h)
GIANTS = (3072, 3073, 6145, 20000)


def bars(e_ref, fp16=False):
    """1.5x the fp32 reference's max and median row error against the truth, with floors 2e-5 and 2e-6; 4x those
    floors (8e-5, 8e-6, still inside the parity bar CHOL_MAX) for the long-row kernels of 16 ... 64 padded factors
    (fp16=True), which gather v = sigma sqrt|w| y as fp16 hi + lo pairs.  Measured on one H100 80GB HBM3 at 400 W: the
    mma.sync kernel, which adds all three hi / lo products of a tile into one fp32 accumulator, reaches 3.5e-5 (1.8x
    the fp32 floor) on the 20000-nonzero row at f = 1 and medians of 4.2e-6 (2.1x) with confidences 1 + 4U, where
    the fp32 reference reaches 3.9e-6 and 6e-7; the wgmma kernel (long_tc) reaches medians of 2e-6 (1.0x) there."""
    k = 4.0 if fp16 else 1.0
    return max(k * 2e-5, 1.5 * e_ref.max()), max(k * 2e-6, 1.5 * np.median(e_ref))


def reference_half(orc, Cui, Y, reg):
    """(fp64 truth, the fp32 reference's result) of one Cholesky half."""
    truth = cholesky_truth(Cui, Y, reg)
    exp = np.zeros((Cui.shape[0], Y.shape[1]), dtype=np.float32)
    orc.least_squares(Cui, exp, Y, reg)
    return truth, exp


def within(got, truth, bar_max, bar_med):
    e = row_err(got, truth)
    return e.max(), np.median(e), bool(np.isfinite(got).all()) and e.max() <= bar_max and np.median(e) <= bar_med


@pytest.mark.parametrize("state", ["cold", "warm"])
@pytest.mark.parametrize("f", WIDTHS)
def test_cholesky_half_at_every_width(lib, ctx, orc, f, state):
    """One seeded CSR (rows at every short-class boundary, empty rows, negative confidences, weights below zero,
    stored zeros, duplicates, giant rows of 3072 ... 20000 nonzeros) through the user half under the default knobs,
    short_max=0 and als_least_squares_with_gramian (the fp32 Gramian of Y: recalculate_user), each against
    cholesky_truth.  Empty rows must be exactly zero.  Then the item half from the device-resident X of the default
    run, against cholesky_truth(Ciu, X): padding columns left non-zero in X would enter that half's Gramian and
    normal equations, which a download cannot show."""
    users, items, reg = 2400, 6000, 0.01
    Cui = mixed_csr(users, items, 50 + f, giants=GIANTS, duplicates=True)
    empty = np.diff(Cui.indptr) == 0
    X, Y = synthetic.initial_factors(users, items, f, seed=f)
    if state == "warm":
        pos = Cui.copy()
        pos.data = np.abs(pos.data) + 1
        oracle.fit(pos, X, Y, iterations=1, use_cg=False, kind=orc.name)
    truth, exp = reference_half(orc, Cui, Y, reg)
    e_ref = row_err(exp, truth)
    fp16 = f <= 64
    bar_max, bar_med = bars(e_ref, fp16)
    Y64 = Y.astype(np.float64)
    YtY = (Y64.T @ Y64).astype(np.float32)
    C = lib.DeviceCSR.upload(ctx, Cui)
    dY = lib.DeviceFactors.from_host(ctx, Y)
    results, dX_default = {}, None
    for name, knobs in {"default": {}, "short_max=0": {"short_max": 0}, "with_gramian": {}}.items():
        for k, v in knobs.items():
            ctx.set_knob(k, v)
        dX = lib.DeviceFactors.from_host(ctx, np.full((users, f), np.nan, np.float32))
        if name == "with_gramian":
            lib.least_squares_with_gramian(ctx, YtY, C, dX, dY, reg)
        else:
            lib.least_squares(ctx, C, dX, dY, reg)
        for k in knobs:
            ctx.set_knob(k, KNOB_DEFAULTS[k])
        got = dX.download()
        results[name] = within(got, truth, bar_max, bar_med) + (bool(np.all(got[empty] == 0)),)
        if name == "default":
            dX_default, X_default = dX, got
        else:
            dX.close()
    C.close()
    dY.close()

    # the item half, from the X the default run left on the device
    Ciu = Cui.T.tocsr()
    truth_i, exp_i = reference_half(orc, Ciu, X_default, reg)
    e_ref_i = row_err(exp_i, truth_i)
    bar_max_i, bar_med_i = bars(e_ref_i, fp16)
    Ci = lib.DeviceCSR.upload(ctx, Ciu)
    dYn = lib.DeviceFactors.from_host(ctx, np.full((items, f), np.nan, np.float32))
    lib.least_squares(ctx, Ci, dYn, dX_default, reg)
    got_i = dYn.download()
    for h in (Ci, dYn, dX_default):
        h.close()
    results["item half"] = within(got_i, truth_i, bar_max_i, bar_med_i) + (
        bool(np.all(got_i[np.diff(Ciu.indptr) == 0] == 0)),)

    print(f"f={f} {state}: fp32 reference vs fp64 max {e_ref.max():.2e} median {np.median(e_ref):.2e} -> bars "
          f"{bar_max:.2e} / {bar_med:.2e}; item half {bar_max_i:.2e} / {bar_med_i:.2e}")
    for name, (mx, md, ok, zero) in results.items():
        bm, bd = (bar_max_i, bar_med_i) if name == "item half" else (bar_max, bar_med)
        print(f"   {name:13s} worst ratio max {mx / bm:.2f} median {md / bd:.2f}, empty rows zero {zero}")
    bad = {n: r for n, r in results.items() if not (r[2] and r[3])}
    assert not bad


# ---------------------------------------------------------------------------------------- operand-scale range
#: kernel -> (factors, knobs); short_max=0 puts every row on the long-row kernel
SCALE_KERNELS = {"NB=1": (16, {"short_max": 0}), "NB=3": (48, {"short_max": 0}), "NB=4": (64, {"short_max": 0}),
                 "long_tc": (64, {"short_max": 0, "long_tc": 1}), "wide": (100, {})}


def scale_csr(kind, seed):
    """300 rows of 49 ... 400 nonzeros, one empty row and one giant row of 3073 (two chunks and a finish item); every
    |c| >= 1 and no stored zeros (the long_tc kernel stays eligible), a quarter of the confidences negative.
    kind sets |c|: all exactly 1 (max| |c| - 1 | = 0), {1, 1 + 2^-23}, 1 + 4U, or 1 + 4U alpha-scaled to 1e4."""
    users, items = 300, 4000
    rng = np.random.default_rng(seed)
    lens = rng.integers(49, 401, users)
    lens[7], lens[11] = 3073, 0
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    cols = np.concatenate([rng.choice(items, n, replace=False) for n in lens]).astype(np.int32)
    n = int(indptr[-1])
    mag = {"ones": np.ones(n),
           "one_ulp": np.where(rng.random(n) < 0.5, 1.0, 1.0 + 2.0 ** -23),
           "1+4U": 1 + 4 * rng.random(n),
           "alpha": 2000.0 * (1 + 4 * rng.random(n))}[kind]
    vals = np.where(rng.random(n) < 0.25, -mag, mag).astype(np.float32)
    return sp.csr_matrix((vals, cols, indptr), shape=(users, items))


@pytest.mark.parametrize("kernel", list(SCALE_KERNELS))
def test_cholesky_operand_scale_range(lib, ctx, orc, kernel):
    """Y scaled by 2^s, s in {-60, ..., 40}, with four kinds of confidences.  Both long-row kernels gather
    v = sigma sqrt|w| y in fp16 with sigma = 2^k bringing sqrt(max|w|) max|y| just below 2^14, and solve
    (sigma^2 A) x = sigma^2 b: at factors of order 1e-16, sigma^2 must not overflow fp32.  The wide kernel (fp32
    throughout) is the control.  Bars of test_cholesky_half_at_every_width (see bars()); a case is skipped only where
    the fp32 reference's own result is not finite.  Before sigma's exponent was clamped, every factor width of the
    long-row kernels failed with "cholesky failed on row 0" at s = -60 (and at s = -52 with confidences {1, 1 + 2^-23}):
    sigma = 2^64 or more made sigma^2 = inf, and the factorisation of sigma^2 (Y^T Y + reg I + ...) non-finite."""
    f, knobs = SCALE_KERNELS[kernel]
    reg = 0.01
    base = np.random.default_rng(3).standard_normal((4000, f)).astype(np.float32)
    results, skipped = {}, []
    for kind in ("ones", "one_ulp", "1+4U", "alpha"):
        Cui = scale_csr(kind, 11)
        for s in (-60, -52, -40, -20, 0, 20, 40):
            Y = (base * np.float32(2.0 ** s)).astype(np.float32)
            truth = cholesky_truth(Cui, Y, reg)
            exp = np.zeros((Cui.shape[0], f), dtype=np.float32)
            try:
                orc.least_squares(Cui, exp, Y, reg)
            except ValueError:
                exp[:] = np.nan
            if not np.isfinite(exp).all():
                skipped.append((kind, s))
                continue
            bar_max, bar_med = bars(row_err(exp, truth), fp16=kernel != "wide")
            dY = lib.DeviceFactors.from_host(ctx, Y)
            dX = lib.DeviceFactors.from_host(ctx, np.zeros((Cui.shape[0], f), np.float32))
            launches = {}
            for tc in ((0, 1) if kernel == "long_tc" else (None,)):
                C = lib.DeviceCSR.upload(ctx, Cui)  # a fresh handle: the weight range it caches costs a launch
                dX.upload(np.full((Cui.shape[0], f), np.nan, np.float32))  # every row must be written
                for k, v in knobs.items():
                    ctx.set_knob(k, v)
                if tc is not None:
                    ctx.set_knob("long_tc", tc)
                n0 = ctx.launch_count()
                try:
                    lib.least_squares(ctx, C, dX, dY, reg)
                    got = dX.download()
                    err = None
                except ValueError as exc:
                    got, err = None, str(exc)
                launches[tc] = ctx.launch_count() - n0
                for k in list(knobs) + ["long_tc"]:
                    ctx.set_knob(k, KNOB_DEFAULTS[k])
                C.close()
            dY.close()
            dX.close()
            if kernel == "long_tc":  # the wgmma kernel ran: one launch more (its chunks go to the mma.sync kernel)
                assert launches[1] == launches[0] + 1, f"{kind} s={s}: launches {launches}"
            if err is not None:
                results[(kind, s)] = (np.inf, np.inf, False, err)
            else:
                mx, md, ok = within(got, truth, bar_max, bar_med)
                results[(kind, s)] = (mx / bar_max, md / bar_med, ok, "")
    for (kind, s), (rmax, rmed, ok, err) in results.items():
        print(f"{kernel} {kind:8s} s={s:4d}: worst ratio max {rmax:.2f} median {rmed:.2f} {err}")
    print(f"{kernel}: skipped (fp32 reference not finite): {skipped}")
    bad = {key: r for key, r in results.items() if not r[2]}
    assert not bad, f"outside the bar: {bad}"
