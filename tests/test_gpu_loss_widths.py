"""The training loss at every factor width and on row shards, against fp64.

csrc/loss.cu evaluates sum_u x_u^T (Y^T Y) x_u as <Y^T Y, X^T X>_F from two fp32 Gramians, and the per-nonzero terms
((c > 0 ? -2c : 0) + (|c| - 1) d) d + |c| with d = y . x in fp32, summed in fp64: loss_nnz_kernel<ld> for ld <= 128 (a
group of ld / 4 lanes rounded up to a power of two per nonzero, so lanes idle at ld = 48, 80, 96 and 112) and
loss_nnz_wide_kernel<ld / 128> above.  The yardstick is tests/helpers.loss_truth, the reference's row-by-row
evaluation in fp64, which does not use that expansion.

Error model: max(1.5 |reference - truth|, K S / denominator), S being the loss's numerator with every product replaced
by the product of absolute values (loss_truth's scale): fp32 Gramians and dot products carry rounding of a few
2^-24 of the absolute sums they add, whatever the cancellation between the terms.
"""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from helpers import loss_truth, mixed_csr
from helpers import ctx, default_knobs, lib, orc  # noqa: F401  (fixtures)
from implicit_b200 import synthetic

pytestmark = pytest.mark.gpu

#: every ld / 16 class at <= 128 and every ld / 128 class above, each at its full width and below it
WIDTHS = [15, 16, 31, 32, 47, 48, 63, 64, 79, 80, 95, 96, 111, 112, 127, 128,
          129, 256, 257, 384, 385, 512, 513, 640, 641, 768, 769, 896, 897, 1024]
GIANTS = (3072, 3073, 6145, 20000, 3073, 4097, 3500, 8193, 3100, 5000)
REG = 0.01
#: K of the error model, one unit of 2^-24 (6e-8) of the absolute sums; the fp32 reference stays within 1e-8 and an
#: fp32 evaluation of the device's expansion on the host within 3e-10 of S / denominator on this data
K = 2.0 ** -24


def case(f):
    """The CSR of the CG width modules (smaller above 128 factors, where the reference iterations cost f^2 a row)."""
    if f <= 128:
        users, items = 2400, 6000
        return users, items, mixed_csr(users, items, 70 + f, giants=GIANTS, duplicates=True)
    users, items = 600, 1500
    return users, items, mixed_csr(users, items, 170 + f, giants=(3072, 3073, 6145), duplicates=True)


@pytest.mark.parametrize("f", WIDTHS)
def test_loss_at_every_width(lib, ctx, orc, f):
    """calculate_loss from a cold state, a warm one (one reference CG iteration) and a near-converged one (four), on
    data with giant rows, empty rows, negative confidences, stored zeros and duplicates, against loss_truth."""
    users, items, Cui = case(f)
    pos = Cui.copy()
    pos.data = np.abs(pos.data) + 1
    X, Y = synthetic.initial_factors(users, items, f, seed=f)
    C = lib.DeviceCSR.upload(ctx, Cui)
    results = {}
    for state, its in (("cold", 0), ("warm", 1), ("near-converged", 3)):
        if its:
            oracle.fit(pos, X, Y, iterations=its, use_cg=True, kind=orc.name)
        truth, terms, scale = loss_truth(Cui, X, Y, REG)
        den = terms[1] + float(users) * float(items) - float(Cui.nnz)
        ref = orc.calculate_loss(Cui, X, Y, REG)
        dX, dY = lib.DeviceFactors.from_host(ctx, X), lib.DeviceFactors.from_host(ctx, Y)
        got = lib.calculate_loss(ctx, C, dX, dY, REG)
        dX.close()
        dY.close()
        bar = max(1.5 * abs(ref - truth), K * (scale[0] + scale[2]) / den)
        results[state] = (truth, abs(got - truth) / bar, abs(ref - truth) / ((scale[0] + scale[2]) / den),
                          abs(got - truth) / ((scale[0] + scale[2]) / den))
    C.close()
    for state, (truth, r, kref, kgot) in results.items():
        print(f"f={f} {state:14s} loss {truth:.6e}: |GPU - truth| / bar {r:.2f}; in units of S / den: reference "
              f"{kref:.2e}, GPU {kgot:.2e}")
    bad = {s: r[1] for s, r in results.items() if not r[1] <= 1.0}
    assert not bad, f"f={f}: outside the bar: {bad}"


def host_rows(Cui, r0, r1):
    """Rows [r0, r1) of Cui with every stored entry kept (no canonicalisation)."""
    s, e = Cui.indptr[r0], Cui.indptr[r1]
    return sp.csr_matrix((Cui.data[s:e], Cui.indices[s:e], Cui.indptr[r0:r1 + 1] - s), shape=(r1 - r0, Cui.shape[1]))


@pytest.mark.parametrize("f", [64, 100, 256])
def test_loss_terms_on_shards(lib, ctx, orc, f):
    """als_calculate_loss on row shards made with DeviceCSR.slice_rows and with upload(row_offset=...), starting at
    0, in the middle and on a giant row: each of the three terms against loss_truth over that row range (terms[0] within K
    times its absolute sum, terms[1], a sum of fp32 |c| in fp64, within 1e-12), and the shards'
    terms summed into the loss of the whole.  terms[2] = reg tr(Y^T Y) comes from the device's fp32 Gramian, whose
    bar is 1e-6 |Y|^T |Y| elementwise (test_gpu_gramian_widths.py); measured on one H100 80GB HBM3 at 400 W: 3.2e-7 of
    its absolute sum at 6000 items."""
    users, items, Cui = case(f)
    giant = 3 + 47 * 1  # mixed_csr's second giant length (3073) sits on row 50
    assert Cui.indptr[giant + 1] - Cui.indptr[giant] == 3073
    bounds = [0, giant, users // 2, users]
    X, Y = synthetic.initial_factors(users, items, f, seed=f)
    pos = Cui.copy()
    pos.data = np.abs(pos.data) + 1
    oracle.fit(pos, X, Y, iterations=1, use_cg=True, kind=orc.name)
    C = lib.DeviceCSR.upload(ctx, Cui)
    dX, dY = lib.DeviceFactors.from_host(ctx, X), lib.DeviceFactors.from_host(ctx, Y)
    whole = lib.calculate_loss(ctx, C, dX, dY, REG)
    truth, terms_all, scale_all = loss_truth(Cui, X, Y, REG)
    worst, sums = {}, {"slice": np.zeros(3), "row_offset": np.zeros(3)}
    for r0, r1 in zip(bounds[:-1], bounds[1:]):
        _, terms, scale = loss_truth(Cui, X, Y, REG, rows=(r0, r1))
        bar = np.array([K * scale[0], 1e-12 * scale[1], 1e-6 * scale[2]])
        for how in ("slice", "row_offset"):
            S = C.slice_rows(r0, r1) if how == "slice" else lib.DeviceCSR.upload(ctx, host_rows(Cui, r0, r1), row_offset=r0)
            t = lib.loss_terms(ctx, S, dX, dY, REG)
            S.close()
            worst[(how, r0)] = np.abs(t - terms) / bar
            sums[how] += [t[0], t[1], 0.0]
            sums[how][2] = t[2]
    for h in (C, dX, dY):
        h.close()
    den = float(users) * float(items) - float(Cui.nnz)
    bar = K * (scale_all[0] + scale_all[2]) / (terms_all[1] + den)
    for (how, r0), r in worst.items():
        print(f"f={f} {how:10s} shard from row {r0:5d}: |terms - truth| / bar {np.array2string(r, precision=2)}")
    summed = {how: (s[0] + s[2]) / (s[1] + den) for how, s in sums.items()}
    print(f"f={f}: whole {whole:.8e} truth {truth:.8e}; summed shards " +
          ", ".join(f"{how} {v:.8e}" for how, v in summed.items()) + f"; bar {bar:.2e}")
    assert all(np.all(r <= 1.0) for r in worst.values()), worst
    assert abs(whole - truth) <= bar and all(abs(v - truth) <= bar for v in summed.values())
