"""Generates tests/golden/serving.npz: what recommend, rank_items and similar_* returned or raised for host ids, for
every case of tests/_serving_cases.py.  Needs an H100 and PyTorch with CUDA (for the liked filter in CUDA memory):

    python tests/golden/make_golden_serving.py [OUT.npz]

Per case: NAME__ids and NAME__scores (as returned: dtype and shape included), or NAME__exc and NAME__msg (the type
name and message of the exception raised).  The inputs are rebuilt from their seeds.
"""
import os
import sys

os.environ.setdefault("OPENBLAS_NUM_THREADS", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import _serving_cases as sc  # noqa: E402
from implicit_b200 import _lib, als  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "serving.npz")
    ctx = _lib.Context(0)
    models = {f: sc.model(ctx, f) for f in sc.WIDTHS}
    default = als._LIKED_NNZ_MAX
    out = {}
    for name, f, method, kw, _, liked_max in sc.cases():
        als._LIKED_NNZ_MAX = default if liked_max is None else liked_max
        try:
            ids, scores = sc.call(models[f], method, kw)
            out[f"{name}__ids"], out[f"{name}__scores"] = ids, scores
            print(name, ids.dtype, ids.shape)
        except Exception as e:  # noqa: BLE001 -- a refusal is recorded, whatever it is
            out[f"{name}__exc"], out[f"{name}__msg"] = np.str_(type(e).__name__), np.str_(str(e))
            print(name, type(e).__name__, e)
    als._LIKED_NNZ_MAX = default
    np.savez_compressed(path, **out)


if __name__ == "__main__":
    main()
