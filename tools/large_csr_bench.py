#!/usr/bin/env python
"""Above 2^31 nonzeros: upload, device transpose and one iteration of each solver on a CSR held as row-block segments.

    python tools/large_csr_bench.py [--blocks 127] [--out DIR]

The matrix is a block-diagonal tiling of a 40k x 20k power-law base (about 17M nonzeros per block, 2.16B at 127
blocks, 5.1M users x 2.5M items).  Reports, as one JSON line (and DIR/large_csr_bench.json):
  upload_s      DeviceCSR.upload of the scipy matrix (int64 indptr and indices, narrowed while staged)
  transpose_s   the device transpose into a segmented CSR
  chol_f64      one Cholesky iteration (user + item half) at 64 factors: ms and nonzeros per second (2 nnz / time)
  cg_f128       one CG iteration (3 steps) at 128 factors: the same
  device_gb     device memory taken by the two CSRs and everything the transpose needed (cudaMemGetInfo before and
                after: the stream-ordered pool keeps what it freed, so this covers the transpose's peak)
Compare the rates with bench.py --config C2 (Cholesky, 64 factors) and C3 (CG, 128 factors) on the same box.
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
    ap.add_argument("--blocks", type=int, default=127)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    from implicit_b200 import _lib, synthetic

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    base = synthetic.power_law_csr(40000, 20000, 17_000_000, 31)
    t0 = time.perf_counter()
    Cui_host = synthetic.block_diagonal_tiling(base, args.blocks)
    build_s = time.perf_counter() - t0
    nnz = int(Cui_host.nnz)
    users, items = Cui_host.shape
    ctx = _lib.Context(0)
    free0 = torch.cuda.mem_get_info()[0]

    t0 = time.perf_counter()
    Cui = _lib.DeviceCSR.upload(ctx, Cui_host)
    ctx.sync()
    upload_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    Ciu = Cui.transpose()
    ctx.sync()
    transpose_s = time.perf_counter() - t0
    device_gb = (free0 - torch.cuda.mem_get_info()[0]) / 1e9
    del Cui_host

    res = dict(gpu=gpu, nnz=nnz, users=users, items=items, segments=[Cui.segment_count, Ciu.segment_count],
               host_build_s=round(build_s, 1), upload_s=round(upload_s, 2), transpose_s=round(transpose_s, 2),
               device_gb=round(device_gb, 1))
    for name, f, use_cg in (("chol_f64", 64, False), ("cg_f128", 128, True)):
        X = _lib.DeviceFactors(ctx, users, f)
        Y = _lib.DeviceFactors(ctx, items, f)
        X.fill_uniform(1, 0.01)
        Y.fill_uniform(2, 0.01)

        def iteration():
            if use_cg:
                _lib.least_squares_cg(ctx, Cui, X, Y, 0.01, 3)
                _lib.least_squares_cg(ctx, Ciu, Y, X, 0.01, 3)
            else:
                _lib.least_squares(ctx, Cui, X, Y, 0.01)
                _lib.least_squares(ctx, Ciu, Y, X, 0.01)

        iteration()  # warm-up: schedules, scratch, module loading
        ctx.sync()
        times = []
        for _ in range(3):
            ctx.timer_start()
            iteration()
            times.append(ctx.timer_stop())
        ms = float(np.median(times))
        res[name] = dict(ms=round(ms, 1), nnz_per_s=float(f"{2 * nnz / (ms / 1e3):.4g}"), runs_ms=[round(t, 1) for t in times])
        X.close()
        Y.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "large_csr_bench.json"), "w") as fh:
            fh.write(line + "\n")
    Ciu.close()
    Cui.close()
    ctx.close()


if __name__ == "__main__":
    main()
