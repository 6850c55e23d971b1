#!/usr/bin/env python
"""A C2 fit end to end from host arrays against the same fit from CUDA arrays, on one GPU.

    python tools/cuda_input_bench.py [--iterations 3] [--reps 3] [--out DIR]

C2 is synthetic.power_law_csr (360k x 300k, 17M nonzeros, seed 2) at 64 factors, Cholesky.  One timed call covers:
  host    factors assigned from numpy, fit() from the scipy CSR, both factor matrices read back to numpy
  device  factors assigned from CUDA tensors, fit() from a torch.sparse_csr_tensor on the device, both factor matrices
          handed out as *_factors_device snapshots wrapped by torch.as_tensor
Each call starts from the inputs where a user would hold them and ends in a device synchronise; the time is the host
clock around it.  Every path is warmed up once, then the two alternate --reps times; the medians are reported in
row-updates/s (iterations x (users + items) / seconds) with the card name and power limit, as one JSON line (and
DIR/cuda_input_bench.json).  The two paths must give bitwise the same factors.
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
    ap.add_argument("--iterations", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    from implicit_b200 import AlternatingLeastSquares, _lib, synthetic

    if not torch.cuda.is_available():
        raise SystemExit("cuda_input_bench needs a GPU and PyTorch with CUDA")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    Cui, X0, Y0, cfg = synthetic.config("C2")
    users, items = Cui.shape
    D = torch.sparse_csr_tensor(*(torch.from_numpy(a).cuda() for a in (Cui.indptr, Cui.indices, Cui.data)),
                                size=Cui.shape)
    Xd, Yd = torch.from_numpy(X0).cuda(), torch.from_numpy(Y0).cuda()
    torch.cuda.synchronize()
    ctx = _lib.Context(0)

    def model():
        m = AlternatingLeastSquares(factors=cfg["factors"], use_cg=False, iterations=args.iterations, random_state=0)
        m._ctx = ctx
        return m

    def host():
        m = model()
        t = time.perf_counter()
        m.user_factors, m.item_factors = X0, Y0
        m.fit(Cui, show_progress=False)
        out = m.user_factors, m.item_factors
        return time.perf_counter() - t, out

    def device():
        m = model()
        torch.cuda.synchronize()
        t = time.perf_counter()
        m.user_factors, m.item_factors = Xd, Yd
        m.fit(D, show_progress=False)
        out = torch.as_tensor(m.user_factors_device, device="cuda"), torch.as_tensor(m.item_factors_device, device="cuda")
        torch.cuda.synchronize()
        return time.perf_counter() - t, out

    paths = {"host": host, "device": device}
    last = {name: fn()[1] for name, fn in paths.items()}  # warm-up
    times = {name: [] for name in paths}
    for _ in range(args.reps):
        for name, fn in paths.items():
            dt, last[name] = fn()
            times[name].append(dt)
    bitwise = all(np.array_equal(h, d.cpu().numpy()) for h, d in zip(last["host"], last["device"]))
    rows = args.iterations * (users + items)
    med = {name: float(np.median(t)) for name, t in times.items()}
    out = {
        "tool": "cuda_input_bench", "gpu": gpu, "config": "C2", "users": users, "items": items, "nnz": int(Cui.nnz),
        "factors": cfg["factors"], "solver": "cholesky", "iterations": args.iterations, "reps": args.reps,
        "seconds": {name: [round(t, 4) for t in ts] for name, ts in times.items()},
        "median_seconds": {name: round(t, 4) for name, t in med.items()},
        "row_updates_per_s": {name: float(f"{rows / t:.4g}") for name, t in med.items()},
        "ms_per_iteration": {name: round(1e3 * t / args.iterations, 2) for name, t in med.items()},
        "bitwise_equal_factors": bool(bitwise),
    }
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "cuda_input_bench.json"), "w") as f:
            f.write(line + "\n")
    if not bitwise:
        raise SystemExit("the device path's factors differ from the host path's")


if __name__ == "__main__":
    main()
