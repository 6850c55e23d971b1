#!/usr/bin/env python
"""Latency of recommend and similar_items called with host ids, one call at a time, on one GPU.

    python tools/host_serving_latency.py [--calls 50] [--label NAME] [--out DIR]

A model of bench.py's C5 shape: 1M users x 1M items at 64 factors (default_rng(5).standard_normal * 0.1), factors
assigned from host arrays, a liked-items CSR of 20 nonzeros per user (synthetic.power_law_csr).  Each call goes from
numpy ids in to numpy (ids, scores) out, ending in a device synchronise (host clock):
  recommend        1, 64 and 4096 users, k = 10, with their liked rows as a scipy CSR and without a liked filter
  recommend_items  64 users ranked over 10,000 items (items=...), their liked rows as a scipy CSR
  similar_items    1 and 64 items, k = 10
Every call is warmed up once; the calls are then made round-robin --calls times.  Prints one JSON line (and writes
DIR/host_serving_latency_<label>.json): per call the median and the 10th / 90th percentiles in ms, a digest of its last
outputs (to compare two versions of the code), and the card's name and power limit read in the same run.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--label", default="run")
    ap.add_argument("--scale", type=float, default=1.0, help="shrink users and items together (rehearsal only)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from implicit_b200 import AlternatingLeastSquares, synthetic

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    Q = I = max(100_000, int(1_000_000 * args.scale))
    f, k = 64, 10
    rng = np.random.default_rng(5)
    m = AlternatingLeastSquares(factors=f, random_state=0)
    m.user_factors = rng.standard_normal((Q, f), dtype=np.float32) * np.float32(0.1)
    m.item_factors = rng.standard_normal((I, f), dtype=np.float32) * np.float32(0.1)
    liked = synthetic.power_law_csr(Q, I, 20 * Q, 5)
    pick = np.random.default_rng(6)
    users = {n: pick.choice(Q, n, replace=False) for n in (1, 64, 4096)}
    rows = {n: liked[u] for n, u in users.items()}
    subset = pick.choice(I, 10_000, replace=False)
    sim = {n: pick.choice(I, n, replace=False) for n in (1, 64)}

    calls = {}
    for n in (1, 64, 4096):
        calls[f"recommend_{n}_liked"] = lambda n=n: m.recommend(users[n], rows[n], N=k)
        calls[f"recommend_{n}"] = lambda n=n: m.recommend(users[n], None, N=k, filter_already_liked_items=False)
    calls["recommend_items_64_liked"] = lambda: m.recommend(users[64], rows[64], N=k, items=subset)
    for n in (1, 64):
        calls[f"similar_items_{n}"] = lambda n=n: m.similar_items(sim[n], N=k)

    def timed(fn):
        m.ctx.sync()
        t = time.perf_counter()
        out = fn()
        m.ctx.sync()
        return time.perf_counter() - t, out

    last = {name: timed(fn)[1] for name, fn in calls.items()}  # warm-up
    times = {name: [] for name in calls}
    for _ in range(args.calls):
        for name, fn in calls.items():
            dt, last[name] = timed(fn)
            times[name].append(dt)

    def digest(out):
        h = hashlib.sha256()
        for a in out:
            h.update(str(a.dtype).encode() + str(a.shape).encode() + np.ascontiguousarray(a).tobytes())
        return h.hexdigest()[:16]

    result = {
        "tool": "host_serving_latency", "label": args.label, "gpu": gpu, "users": Q, "items": I, "factors": f, "k": k,
        "calls": args.calls,
        "ms": {name: {"median": 1e3 * float(np.median(t)), "p10": 1e3 * float(np.percentile(t, 10)),
                      "p90": 1e3 * float(np.percentile(t, 90))} for name, t in times.items()},
        "digest": {name: digest(out) for name, out in last.items()},
    }
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"host_serving_latency_{args.label}.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
