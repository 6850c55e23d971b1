#!/usr/bin/env python
"""recommend and similar_items with ids in CUDA memory against the same calls with numpy ids, on one GPU.

    python tools/device_serving_bench.py [--reps 5] [--out DIR]

Data of bench.py's C5 shape: 1M users x 1M items at 64 factors (default_rng(5).standard_normal * 0.1), a liked-items CSR
of 20 nonzeros per user (synthetic.power_law_csr).  The factors are assigned from CUDA tensors, as a GPU pipeline hands
them over.  Timed, each call from its inputs where a user would hold them to its outputs where the next stage reads
them, ending in a device synchronise (host clock):
  recommend  67,584 users, k = 10, their liked rows as a scipy CSR.  numpy: numpy ids in, numpy (ids, scores) out.
             torch: torch ids in, the CUDA outputs wrapped by torch.as_tensor.
  similar    similar_items of 10,000 items, N = 10.  "first": the first call after the factors were assigned (both
             compute the norms on the device), re-assigned before every rep; "steady": the call again, norms cached.
Every path is warmed up once; the paths alternate --reps times and the medians are reported in ms, with the card name
and power limit read in the same run, as one JSON line (and DIR/device_serving_bench.json).  Each pair of paths must
give bitwise the same ids and scores.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="shrink users and items together (rehearsal only)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    from implicit_b200 import AlternatingLeastSquares, _lib, synthetic

    if not torch.cuda.is_available():
        raise SystemExit("device_serving_bench needs a GPU and PyTorch with CUDA")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    Q = I = max(100_000, int(1_000_000 * args.scale))
    f, k, batch, n_similar = 64, 10, min(67_584, Q), 10_000
    rng = np.random.default_rng(5)
    X = rng.standard_normal((Q, f), dtype=np.float32) * np.float32(0.1)
    Y = rng.standard_normal((I, f), dtype=np.float32) * np.float32(0.1)
    liked = synthetic.power_law_csr(Q, I, 20 * Q, 5)
    Xd, Yd = torch.from_numpy(X).cuda(), torch.from_numpy(Y).cuda()
    ctx = _lib.Context(0)

    def model():
        m = AlternatingLeastSquares(factors=f, random_state=0)
        m._ctx = ctx
        m.user_factors, m.item_factors = Xd, Yd
        return m

    mn, mt = model(), model()  # the numpy and the torch path each keep their own caches
    users = np.arange(batch, dtype=np.int64)
    rows = liked[:batch]
    users_d = torch.from_numpy(users).cuda()
    sim = np.arange(0, I, I // n_similar, dtype=np.int64)[:n_similar]
    sim_d = torch.from_numpy(sim).cuda()
    torch.cuda.synchronize()

    def timed(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t, out

    def torch_out(r):
        return torch.as_tensor(r[0], device="cuda"), torch.as_tensor(r[1], device="cuda")

    def reassign(m):  # the state right after a pipeline hands the factors over
        def go():
            m.user_factors, m.item_factors = Xd, Yd
            torch.cuda.synchronize()
        return go

    paths = {
        "recommend_numpy": (None, lambda: mn.recommend(users, rows, N=k)),
        "recommend_torch": (None, lambda: torch_out(mt.recommend(users_d, rows, N=k))),
        "similar_first_numpy": (reassign(mn), lambda: mn.similar_items(sim, N=k)),
        "similar_first_torch": (reassign(mt), lambda: torch_out(mt.similar_items(sim_d, N=k))),
        "similar_steady_numpy": (None, lambda: mn.similar_items(sim, N=k)),
        "similar_steady_torch": (None, lambda: torch_out(mt.similar_items(sim_d, N=k))),
    }
    last, times = {}, {name: [] for name in paths}
    for name, (prep, fn) in paths.items():  # warm-up
        if prep:
            prep()
        last[name] = timed(fn)[1]
    for _ in range(args.reps):
        for name, (prep, fn) in paths.items():
            if prep:
                prep()
            dt, last[name] = timed(fn)
            times[name].append(dt)

    def bitwise(a, b):
        return all(np.array_equal(x, y.cpu().numpy()) for x, y in zip(last[a], last[b]))

    med = {name: 1e3 * float(np.median(t)) for name, t in times.items()}
    out = {
        "tool": "device_serving_bench", "gpu": gpu, "users": Q, "items": I, "factors": f, "k": k,
        "recommend_batch": batch, "similar_items": n_similar, "reps": args.reps, "median_ms": med,
        "all_ms": {name: [1e3 * x for x in t] for name, t in times.items()},
        "bitwise": {"recommend": bitwise("recommend_numpy", "recommend_torch"),
                    "similar_first": bitwise("similar_first_numpy", "similar_first_torch"),
                    "similar_steady": bitwise("similar_steady_numpy", "similar_steady_torch")},
    }
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "device_serving_bench.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
