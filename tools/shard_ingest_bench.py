#!/usr/bin/env python
"""Ingest of one rank of a W-rank fit against the whole-matrix ingest, on one GPU.

    python tools/shard_ingest_bench.py [--blocks 127] [--world 8] [--out DIR]

The matrix is the block-diagonal tiling of tools/large_csr_bench.py (2.16B nonzeros at 127 blocks).  Reports, as one
JSON line (and DIR/shard_ingest_bench.json):
  whole         DeviceCSR.upload + transpose of the whole matrix, what every rank of a multi-GPU fit did before the
                sharded ingest: seconds, and the device memory pool's peak over the ingest (als_mem_peak) in GB
  rank0         rank 0's part of the sharded ingest, emulated in one process: upload_rows of its user rows, column
                counts, transpose_pieces, then merge_rows of its piece with the pieces the other W - 1 ranks built for it
                (built beforehand on the same device and counted in the peak from the start, as if already received).
                The NCCL exchange is not part of it: it needs W GPUs (an all-to-all of about 8 nnz / W bytes per rank).
Times are host clocks around work that ends in a device synchronise.
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
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from implicit_b200 import _lib, synthetic
    from implicit_b200.utils import column_splits, nnz_balanced_splits

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    C = synthetic.block_diagonal_tiling(synthetic.power_law_csr(40000, 20000, 17_000_000, 31), args.blocks)
    W, row_cost = args.world, 60
    ctx = _lib.Context(0)
    res = dict(gpu=gpu, nnz=int(C.nnz), users=C.shape[0], items=C.shape[1], world=W)

    base, _ = ctx.mem_peak()
    t0 = time.perf_counter()
    Cui = _lib.DeviceCSR.upload(ctx, C)
    Ciu = Cui.transpose()
    ctx.sync()
    whole_s = time.perf_counter() - t0
    _, peak = ctx.mem_peak()
    res["whole"] = dict(s=round(whole_s, 3), peak_gb=round((peak - base) / 1e9, 2))
    Cui.close()
    Ciu.close()

    usplit = nnz_balanced_splits(C.indptr, W, row_cost)
    isplit = column_splits(np.bincount(C.indices, minlength=C.shape[1]), W, row_cost)
    received = []
    for p in range(1, W):
        s = _lib.DeviceCSR.upload_rows(ctx, C, usplit[p], usplit[p + 1])
        pieces = s.transpose_pieces(isplit)
        received.append(pieces[0])
        for x in pieces[1:] + [s]:
            x.close()
    ctx.mem_peak()
    times = {}
    t0 = time.perf_counter()
    s0 = _lib.DeviceCSR.upload_rows(ctx, C, usplit[0], usplit[1])
    ctx.sync()
    times["upload_rows"] = time.perf_counter() - t0
    t1 = time.perf_counter()
    s0.column_counts()
    times["column_counts"] = time.perf_counter() - t1
    t1 = time.perf_counter()
    pieces = s0.transpose_pieces(isplit)
    ctx.sync()
    times["transpose_pieces"] = time.perf_counter() - t1
    for x in pieces[1:]:
        x.close()
    t1 = time.perf_counter()
    m0 = _lib.DeviceCSR.merge_rows(ctx, [pieces[0]] + received, C.shape[0], isplit[0])
    ctx.sync()
    times["merge_rows"] = time.perf_counter() - t1
    total = time.perf_counter() - t0
    _, peak = ctx.mem_peak()
    res["rank0"] = dict(s=round(total, 3), peak_gb=round((peak - base) / 1e9, 2), shard_nnz=int(C.indptr[usplit[1]]),
                        merged_nnz=m0.shape3[2], steps_s={k: round(v, 3) for k, v in times.items()})
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "shard_ingest_bench.json"), "w") as fh:
            fh.write(line + "\n")
    for x in [s0, m0, pieces[0]] + received:
        x.close()
    ctx.close()


if __name__ == "__main__":
    main()
