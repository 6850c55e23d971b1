#!/usr/bin/env python
"""ranking_metrics_at_k end to end, device metrics pass against the array path, on a C5-shaped workload.

    python tools/eval_bench.py [--users 1000000] [--items 1000000] [--factors 64] [--K 10] [--reps 3] [--out DIR]

Train: synthetic.power_law_csr with 20 entries per user; test: 5 uniformly drawn items per user; the model's factors are
synthetic.initial_factors.  `device` is ranking_metrics_at_k(model, ...) (one als_ranking_metrics call per batch);
`host` is the same call through a proxy that exposes only `recommend`, so the ids and scores come back to the host and
the metrics are computed there in numpy.  Both run in one process, after one warm-up each, alternated `reps` times;
the best and median wall-clock seconds of each are reported with the card name and power limit, as one JSON line (and
DIR/eval_bench.json).  The two dicts must agree to rel 1e-12.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


class Proxy:
    def __init__(self, model):
        self.model = model

    def recommend(self, *args, **kwargs):
        return self.model.recommend(*args, **kwargs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=1_000_000)
    ap.add_argument("--factors", type=int, default=64)
    ap.add_argument("--K", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import scipy.sparse as sp

    from implicit_b200 import AlternatingLeastSquares, evaluation, synthetic

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    U, I = args.users, args.items
    train = synthetic.power_law_csr(U, I, 20 * U, 7)
    rng = np.random.default_rng(8)
    test = sp.csr_matrix((np.ones(5 * U, dtype=np.float32), rng.integers(0, I, 5 * U).astype(np.int32),
                          np.arange(0, 5 * U + 1, 5, dtype=np.int64)), shape=(U, I))
    X, Y = synthetic.initial_factors(U, I, args.factors)
    model = AlternatingLeastSquares(factors=args.factors)
    model.user_factors, model.item_factors = X, Y

    def run(m):
        t = time.perf_counter()
        r = evaluation.ranking_metrics_at_k(m, train, test, K=args.K, show_progress=False)
        return time.perf_counter() - t, r

    run(model)
    run(Proxy(model))
    times = {"device": [], "host": []}
    for _ in range(args.reps):
        t, dev = run(model)
        times["device"].append(t)
        t, host = run(Proxy(model))
        times["host"].append(t)
    rel = max(abs(dev[k] - host[k]) / abs(host[k]) for k in host)
    res = dict(gpu=gpu, users=U, items=I, factors=args.factors, K=args.K, train_nnz=int(train.nnz), test_nnz=int(test.nnz),
               reps=args.reps, agree_rel=rel, agree=bool(rel <= 1e-12), metrics={k: float(v) for k, v in dev.items()})
    for k, v in times.items():
        res[f"{k}_best_s"], res[f"{k}_median_s"] = min(v), float(np.median(v))
    res["speedup_median"] = res["host_median_s"] / res["device_median_s"]
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "eval_bench.json"), "w") as f:
            f.write(line + "\n")
    sys.exit(0 if res["agree"] else 1)


if __name__ == "__main__":
    main()
