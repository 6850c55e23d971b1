#!/usr/bin/env python
"""partial_fit_users with ids in CUDA memory against the same call with numpy ids, on one GPU.

    python tools/device_partial_fit_bench.py [--reps 5] [--out DIR]

A model of bench.py's C5 shape: 1M users x 1M items at 64 factors (default_rng(5).standard_normal * 0.1), assigned from
CUDA tensors, as a GPU pipeline hands them over; the user factors are re-assigned before every timed call, so every call
starts from the state right after a fit or an assignment.  Timed, host clock ending in a device synchronise:
  partial_fit  partial_fit_users of 1,000 and of 10,000 users, a tenth of them new ids past the last user (the matrix
               grows), their rows a scipy CSR of 20 nonzeros per user.  numpy: numpy int64 ids; torch: torch int64 ids.
  next_call    what the next device call then pays before it can read the user factors: the upload of the whole
               matrix the numpy call left on the host (nothing for the torch call, whose replica is current).
Every path is warmed up once; the paths alternate --reps times and the medians are reported in ms, with the card name
and power limit read in the same run, as one JSON line (and DIR/device_partial_fit_bench.json).  Both paths must leave
bitwise the same user factors.
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
        raise SystemExit("device_partial_fit_bench needs a GPU and PyTorch with CUDA")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    Q = I = max(100_000, int(1_000_000 * args.scale))
    f = 64
    rng = np.random.default_rng(5)
    X = rng.standard_normal((Q, f), dtype=np.float32) * np.float32(0.1)
    Y = rng.standard_normal((I, f), dtype=np.float32) * np.float32(0.1)
    Xd, Yd = torch.from_numpy(X).cuda(), torch.from_numpy(Y).cuda()
    ctx = _lib.Context(0)

    def model():
        m = AlternatingLeastSquares(factors=f, random_state=0)
        m._ctx = ctx
        m.user_factors, m.item_factors = Xd, Yd
        return m

    mn, mt = model(), model()
    cases = {}
    for n in (1_000, 10_000):
        new = n // 10
        ids = np.concatenate([rng.choice(Q, n - new, replace=False), Q + np.arange(new)]).astype(np.int64)
        rng.shuffle(ids)
        cases[n] = (ids, torch.from_numpy(ids).cuda(), synthetic.power_law_csr(n, I, 20 * n, n))
    torch.cuda.synchronize()

    def timed(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t

    def run(m, ids, rows):
        m.user_factors = Xd  # the state right after a fit or an assignment
        torch.cuda.synchronize()
        return timed(lambda: m.partial_fit_users(ids, rows)), timed(lambda: m._device_factors("user"))

    paths = {}
    for n, (ids, ids_d, rows) in cases.items():
        paths[f"numpy_{n}"] = (mn, ids, rows)
        paths[f"torch_{n}"] = (mt, ids_d, rows)
    times = {name: ([], []) for name in paths}
    bitwise = {}
    for name, p in paths.items():  # warm-up
        run(*p)
    for _ in range(args.reps):
        for name, p in paths.items():
            fit_s, next_s = run(*p)
            times[name][0].append(fit_s)
            times[name][1].append(next_s)
            if name.startswith("torch_"):  # both models now hold this case's refit
                bitwise[int(name[6:])] = bool(np.array_equal(mn.user_factors.view(np.uint32),
                                                             mt.user_factors.view(np.uint32)))

    out = {
        "tool": "device_partial_fit_bench", "gpu": gpu, "users": Q, "items": I, "factors": f, "reps": args.reps,
        "median_ms": {name: {"partial_fit": 1e3 * float(np.median(t[0])), "next_call": 1e3 * float(np.median(t[1]))}
                      for name, t in times.items()},
        "all_ms": {name: {"partial_fit": [1e3 * x for x in t[0]], "next_call": [1e3 * x for x in t[1]]}
                   for name, t in times.items()},
        "bitwise": bitwise,
    }
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "device_partial_fit_bench.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
