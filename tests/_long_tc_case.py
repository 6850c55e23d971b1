"""Helper of tests/test_gpu_long_tc.py (run as a subprocess so that a hanging kernel cannot take the suite with it).

    _long_tc_case.py [below_one]   one Cholesky half over rows of 0 ... 3500 nonzeros with the wgmma long-row kernel
                                   (knob long_tc) and with the mma.sync kernel, both against the oracle
    _long_tc_case.py edges F       the wgmma kernel at its edges with F factors, against fp64 (see edges())

Prints one JSON line."""
import json
import os
import sys

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import oracle  # noqa: E402
from helpers import cholesky_truth, factors_of, row_err  # noqa: E402
from implicit_b200 import _lib, synthetic  # noqa: E402

#: rows at the kernel's edges: 32-nonzero stages, the 8-stage ring (256 nonzeros a lap), rows under 128 nonzeros that
#: leave some of the 4 producers idle, the largest whole row and giant rows of 2 and 5 chunks (kSplitNnz = 3072,
#: kChunkNnz = 2048); rows of 1 ... 33 nonzeros reach this kernel only with short_max=0
EDGE_LENGTHS = [49, 63, 64, 65, 95, 96, 97, 127, 128, 129, 255, 256, 257, 511, 512, 513, 3072, 3073, 8193,
                1, 15, 16, 17, 31, 32, 33]


def edge_lengths(rows):
    return np.array([EDGE_LENGTHS[u % len(EDGE_LENGTHS)] for u in range(rows)])


def work_items(lens):
    """Length of the work list: whole rows plus the chunks of rows over 3072 nonzeros (api.cu build_schedule)."""
    return int(np.where(lens > 3072, -(-lens // 2048), 1).sum())


def edge_csr(rows, items, seed):
    """Every |c| >= 1 (a quarter of them <= -1, a tenth exactly +-1) and no stored zeros: the CSR stays eligible."""
    rng = np.random.default_rng(seed)
    lens = edge_lengths(rows)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    cols = np.concatenate([rng.choice(items, n, replace=False) for n in lens]).astype(np.int32)
    n = int(indptr[-1])
    mag = np.where(rng.random(n) < 0.1, 1.0, 1 + 4 * rng.random(n))
    vals = np.where(rng.random(n) < 0.25, -mag, mag).astype(np.float32)
    return sp.csr_matrix((vals, cols, indptr), shape=(rows, items))


def solve(ctx, Cui, Y, reg, knobs):
    for k, v in knobs.items():
        ctx.set_knob(k, v)
    C = _lib.DeviceCSR.upload(ctx, Cui)
    dX = _lib.DeviceFactors.from_host(ctx, np.full((Cui.shape[0], Y.shape[1]), np.nan, np.float32))
    dY = _lib.DeviceFactors.from_host(ctx, Y)
    n0 = ctx.launch_count()
    _lib.least_squares(ctx, C, dX, dY, reg)
    n = ctx.launch_count() - n0
    X = dX.download()
    for h in (C, dX, dY):
        h.close()
    return X, n


def edges(f):
    """Three row counts: fewer rows than SMs (grid = rows); work lists of exactly 4 items per SM (one batch of four
    rows per CTA); and over 8 x 4 items per SM, so that the 4 b slots and the 2 solver panels of each CTA wrap many
    times.  Y after one ALS iteration ("warm") and with row norms over six decades.  Every row goes to the long-row
    kernels (short_max=0); each case runs with long_tc=1 and with the default mma.sync kernel."""
    ctx = _lib.Context(0)
    sm = ctx.info()["sm_count"]
    orc = oracle.get("auto")
    items, reg = 9000, 0.01
    X0, Y0 = synthetic.initial_factors(2000, items, f, seed=f)
    oracle.fit(synthetic.power_law_csr(2000, items, 60000, 5), X0, Y0, iterations=1, use_cg=False, kind=orc.name)
    Ys = {"warm": Y0, "decades": factors_of("decades", items, f, seed=f + 1) * np.float32(0.1)}
    counts = [2 * len(EDGE_LENGTHS)]
    for target in (4 * sm, 8 * 4 * sm + 1):
        rows = target
        while work_items(edge_lengths(rows)) > target:
            rows -= 1
        counts.append(rows)
    assert counts[0] < sm and work_items(edge_lengths(counts[1])) == 4 * sm
    out = []
    for rows in counts:
        Cui = edge_csr(rows, items, rows + f)
        for yname, Y in Ys.items():
            truth = cholesky_truth(Cui, Y, reg)
            exp = np.zeros((rows, f), dtype=np.float32)
            orc.least_squares(Cui, exp, Y, reg)
            e_ref = row_err(exp, truth)
            bar_max, bar_med = max(2e-5, 1.5 * e_ref.max()), max(2e-6, 1.5 * np.median(e_ref))
            res = {}
            for tc in (0, 1):
                res[tc] = solve(ctx, Cui, Y, reg, {"short_max": 0, "long_tc": tc})
            ctx.set_knob("short_max", 48)
            ctx.set_knob("long_tc", 0)
            e = row_err(res[1][0], truth)
            out.append({"rows": rows, "work": work_items(np.diff(Cui.indptr)), "Y": yname,
                        "finite": bool(np.isfinite(res[1][0]).all()),
                        "max_ratio": float(e.max() / bar_max), "median_ratio": float(np.median(e) / bar_med),
                        "default_max_ratio": float(row_err(res[0][0], truth).max() / bar_max),
                        "tc_vs_default_max": float(row_err(res[1][0], res[0][0]).max()),
                        "launches_tc": res[1][1], "launches_default": res[0][1]})
    ctx.close()
    return {"sm": sm, "cases": out}


def oracle_case(below_one):
    rng = np.random.default_rng(17)
    items, f = 6000, 64
    lengths = [3500, 3072, 1000, 500, 65, 64, 63, 49, 48, 0, 17, 33] + rng.integers(49, 300, 1500).tolist()
    rows, cols, vals = [], [], []
    for u, n in enumerate(lengths):
        c = rng.choice(items, n, replace=False)
        rows += [u] * n
        cols += c.tolist()
        vals += (1 + 4 * rng.random(n)).tolist()
    vals = np.array(vals, dtype=np.float32)
    if below_one:
        vals[5] = 0.5  # one weight |c| - 1 < 0: the whole CSR must take the mma.sync kernel
    Cui = sp.csr_matrix((vals, (rows, cols)), shape=(len(lengths), items))
    Y = (rng.standard_normal((items, f)) * 0.1).astype(np.float32)
    X0 = np.zeros((len(lengths), f), dtype=np.float32)
    exp = X0.copy()
    oracle.get("auto").least_squares(Cui, exp, Y, 0.05)
    ctx = _lib.Context(0)
    out = {}
    res = {}
    for tc in (0, 1):
        ctx.set_knob("long_tc", tc)
        C = _lib.DeviceCSR.upload(ctx, Cui)
        dX, dY = _lib.DeviceFactors.from_host(ctx, X0), _lib.DeviceFactors.from_host(ctx, Y)
        n0 = ctx.launch_count()
        _lib.least_squares(ctx, C, dX, dY, 0.05)
        res[tc] = dX.download()
        e = row_err(res[tc], exp)
        out[f"tc{tc}"] = {"max": float(e.max()), "median": float(np.median(e)), "empty_row_zero": bool(np.all(res[tc][9] == 0)),
                          "launches": int(ctx.launch_count() - n0)}
        for h in (C, dX, dY):
            h.close()
    out["tc_vs_legacy_max"] = float(row_err(res[1], res[0]).max())
    return out


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "edges":
        print(json.dumps(edges(int(sys.argv[2]))))
    else:
        print(json.dumps(oracle_case(len(sys.argv) > 1 and sys.argv[1] == "below_one")))
