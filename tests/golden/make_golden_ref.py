"""Generates tests/golden/ref_checks.npz: what the reference's OWN compiled code (oracle/_ref, built by
oracle/build_ref.py from a checkout of the reference) returns for the direct comparisons of tests/test_oracle.py.
Run where the reference checkout exists:

    OPENBLAS_NUM_THREADS=1 python tests/golden/make_golden_ref.py

Inputs are NOT stored: the CSRs and factors are rebuilt from implicit_b200.synthetic and seeded generators, and the
warm state a half starts from is the C port's own 2-iteration fit (oracle/als_oracle.c, deterministic).  Every row
the reference computed is stored.
"""
import os
import sys

os.environ.setdefault("OPENBLAS_NUM_THREADS", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import oracle  # noqa: E402
from implicit_b200 import synthetic  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def half_inputs(use_cg):
    """(Cui, warm X, warm Y) of test_port_matches_compiled_reference: the port's 2-iteration fit."""
    Cui = synthetic.power_law_csr(500, 300, 6000, 77, negative_fraction=0.05)
    Xw, Yw = synthetic.initial_factors(500, 300, 48)
    oracle.fit(Cui, Xw, Yw, iterations=2, use_cg=use_cg, kind="port")
    return Cui, Xw, Yw


def wide_inputs():
    Cui = synthetic.power_law_csr(200, 150, 3000, 78, negative_fraction=0.05)
    rng = np.random.default_rng(5)
    X = (rng.standard_normal((200, 192)) * 0.1).astype(np.float32)
    Y = (rng.standard_normal((150, 192)) * 0.1).astype(np.float32)
    return Cui, X, Y


def ref_half_case():
    """tests/test_oracle.py::test_port_matches_compiled_reference: one half of the reference from a warm state."""
    ref = oracle.get("ref")
    out = {}
    for tag, use_cg in (("chol", False), ("cg", True)):
        Cui, Xw, Yw = half_inputs(use_cg)
        Xa = Xw.copy()
        if use_cg:
            ref.least_squares_cg(Cui, Xa, Yw, 0.01, cg_steps=3)
        else:
            ref.least_squares(Cui, Xa, Yw, 0.01)
        out.update({f"half_{tag}_Xa": Xa,
                    f"half_{tag}_loss": np.float64(ref.calculate_loss(Cui, Xw, Yw, 0.01))})
    return out


def wide_case():
    """tests/test_oracle.py::test_port_matches_compiled_reference_on_a_wide_model (192 factors)."""
    ref = oracle.get("ref")
    Cui, X, Y = wide_inputs()
    Xa = X.copy()
    ref.least_squares_cg(Cui, Xa, Y, 0.01, cg_steps=3)
    ia, sa = ref.topk(Y, Xa[:20], 7, filter_query_items=Cui[:20])
    return {"wide_Xa": Xa,
            "wide_loss": np.float64(ref.calculate_loss(Cui, X, Y, 0.01)), "wide_topk_ids": ia, "wide_topk_scores": sa}


def ties_case():
    """tests/test_oracle.py::test_select_matches_compiled_reference_on_ties: integer scores, many exact ties."""
    ref = oracle.get("ref")
    rng = np.random.default_rng(5)
    items = rng.integers(0, 4, size=(200, 3)).astype(np.float32)
    q = rng.integers(0, 3, size=(17, 3)).astype(np.float32)
    out = {}
    for k in (1, 5, 32, 250):
        ids, scores = ref.topk(items, q, k)
        out[f"ties_k{k}_ids"], out[f"ties_k{k}_scores"] = ids, scores
    return out


def main():
    out = {}
    for case in (ref_half_case, wide_case, ties_case):
        out.update(case())
    path = os.path.join(HERE, "ref_checks.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
