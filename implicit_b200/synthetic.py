"""Deterministic synthetic inputs for the ALS hot path (SURVEY.md section 8(d)).

Power-law CSR generator and the named configurations of BASELINE.json (C1..C4).  Pure numpy/scipy,
host side; used by bench.py, the tests and the golden-vector script so that every party builds
bit-identical inputs from a seed.
"""
import numpy as np
import scipy.sparse as sp

#: name -> shape, nnz, factors, solver, seed
CONFIGS = {
    "C1": dict(users=10_000, items=5_000, nnz=50_000, factors=16, use_cg=False, seed=1),
    "C2": dict(users=360_000, items=300_000, nnz=17_000_000, factors=64, use_cg=False, seed=2),
    "C3": dict(users=138_000, items=27_000, nnz=20_000_000, factors=128, use_cg=True, seed=3),
    "C4": dict(users=10_000_000, items=1_000_000, nnz=500_000_000, factors=64, use_cg=False, seed=4),
}


def plaw(rng, n, N, a):
    """Truncated power law p(j) ~ (j+1)^-a on [0, N) by inverse CDF."""
    x = ((N ** (1.0 - a) - 1.0) * rng.random(n) + 1.0) ** (1.0 / (1.0 - a))
    return np.clip(np.floor(x) - 1, 0, N - 1).astype(np.int64)


def power_law_csr(users, items, nnz_target, seed, negative_fraction=0.0):
    """CSR (users x items) float32 with sorted, de-duplicated indices; values 1 + 4*U[0,1).

    negative_fraction > 0 negates a fixed share of the values (correctness-only variant that
    exercises the negative-confidence branch, implicit/cpu/_als.pyx:115-118).
    """
    rng = np.random.default_rng(seed)
    m = int(1.25 * nnz_target)
    u = plaw(rng, m, users, 0.5)
    i = plaw(rng, m, items, 0.8)
    pu = rng.permutation(users)
    pi = rng.permutation(items)
    key = np.unique(pu[u] * np.int64(items) + pi[i])
    if len(key) > nnz_target:
        key = np.sort(rng.choice(key, nnz_target, replace=False))
    row = key // items
    col = (key % items).astype(np.int32)
    data = (1.0 + 4.0 * rng.random(len(key), dtype=np.float32)).astype(np.float32)
    if negative_fraction > 0:
        neg = np.random.default_rng(seed + 1000).random(len(key)) < negative_fraction
        data[neg] *= -1
    indptr = np.zeros(users + 1, dtype=np.int64)
    indptr[1:] = np.cumsum(np.bincount(row, minlength=users))
    indptr = indptr.astype(np.int32 if len(key) < 2**31 else np.int64)
    return sp.csr_matrix((data, col, indptr), shape=(users, items))


def block_diagonal_tiling(base, R):
    """R copies of `base` on the diagonal: block r holds users r U_b ... and items r I_b ....  Index arrays are int64
    once the result passes 2^31 nonzeros, as scipy builds them; filled block by block without temporaries of the
    whole size (the large-CSR test and tools/large_csr_bench.py: beyond 2^31 nonzeros at a few minutes of host time)."""
    Ub, Ib = base.shape
    nb = base.nnz
    idx = np.int64 if R * nb >= 2**31 else np.int32
    indices = np.empty(R * nb, dtype=idx)
    indptr = np.empty(R * Ub + 1, dtype=idx)
    ip = base.indptr.astype(np.int64)
    for r in range(R):
        indices[r * nb:(r + 1) * nb] = base.indices
        indices[r * nb:(r + 1) * nb] += r * Ib
        indptr[r * Ub:(r + 1) * Ub] = ip[:-1] + r * nb
    indptr[-1] = R * nb
    return sp.csr_matrix((np.tile(base.data, R), indices, indptr), shape=(R * Ub, R * Ib))


def initial_factors(users, items, factors, seed=42):
    """Same distribution as implicit/cpu/als.py:144-147: rng.random((n, f), float32) * 0.01."""
    rng = np.random.default_rng(seed)
    X = rng.random((users, factors), dtype=np.float32) * np.float32(0.01)
    Y = rng.random((items, factors), dtype=np.float32) * np.float32(0.01)
    return X, Y


def config(name, scale=1.0, negative_fraction=0.0):
    """Returns (Cui, X0, Y0, cfg) for a named configuration; scale < 1 shrinks rows/cols/nnz together."""
    cfg = dict(CONFIGS[name])
    users = max(8, int(cfg["users"] * scale))
    items = max(8, int(cfg["items"] * scale))
    nnz = max(8, int(cfg["nnz"] * scale))
    Cui = power_law_csr(users, items, nnz, cfg["seed"], negative_fraction)
    X0, Y0 = initial_factors(users, items, cfg["factors"])
    cfg.update(users=users, items=items, nnz=int(Cui.nnz))
    return Cui, X0, Y0, cfg
