#!/usr/bin/env python
"""Rank 0's ingest of a W-rank fit from row blocks against today's sharded ingest from the whole matrix, on one GPU.

    python tools/row_block_ingest_bench.py [--blocks 12] [--world 8] [--out DIR]

The matrix is the block-diagonal tiling of tools/large_csr_bench.py (204M nonzeros at 12 blocks, the case of
test_rank_memory_is_a_fraction_of_the_whole_ingest).  Rank 0's row block is uneven: twice its even share of the rows.
Reports, as one JSON line (and DIR/row_block_ingest_bench.json):
  sharded   rank 0's part of the ingest from the whole scipy matrix: upload_rows of its user shard, column counts,
            transpose_pieces, merge_rows with the pieces the other ranks built for it
  blocks    rank 0's part of the ingest from its row block: its rows uploaded in one piece per rank (block_pieces), a
            copy of its own piece (the receive buffer of the exchange), concat_rows with the pieces the other ranks cut
            for it, then the same column counts, transpose_pieces and merge_rows
Each: host seconds around work that ends in a device synchronise, and the device pool's peak (als_mem_peak) in GB.
What the other ranks send to rank 0 is built beforehand on the same device and counted in the peak from the start, as
if already received; the NCCL exchanges are not part of it (they need W GPUs).
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


def tiling(blocks):
    from implicit_b200 import synthetic

    return synthetic.block_diagonal_tiling(synthetic.power_law_csr(40000, 20000, 17_000_000, 31), blocks)


def uneven_bounds(users, W):
    """Rank 0 holds twice its even share of the rows; the other ranks split the rest evenly."""
    first = min(2 * users // W, users)
    return np.concatenate([[0], first + (users - first) * np.arange(W, dtype=np.int64) // max(W - 1, 1)])[:W + 1]


def _peak(ctx, base):
    _, peak = ctx.mem_peak()
    return peak - base


def _sent_transposes(ctx, C, usplit, isplit):
    """The transpose pieces ranks 1 .. W - 1 send to rank 0."""
    from implicit_b200 import _lib

    out = []
    for p in range(1, len(usplit) - 1):
        s = _lib.DeviceCSR.upload_rows(ctx, C, usplit[p], usplit[p + 1])
        pieces = s.transpose_pieces(isplit)
        out.append(pieces[0])
        for x in pieces[1:] + [s]:
            x.close()
    return out


def rank0_sharded(ctx, C, W, row_cost):
    """(seconds, peak bytes, Cui_s, Ciu_s) of rank 0's ingest from the whole matrix."""
    from implicit_b200 import _lib
    from implicit_b200.utils import column_splits, nnz_balanced_splits

    usplit = nnz_balanced_splits(C.indptr, W, row_cost)
    isplit = column_splits(np.bincount(C.indices, minlength=C.shape[1]), W, row_cost)
    received = _sent_transposes(ctx, C, usplit, isplit)
    base, _ = ctx.mem_peak()
    t0 = time.perf_counter()
    s0 = _lib.DeviceCSR.upload_rows(ctx, C, usplit[0], usplit[1])
    s0.column_counts()
    pieces = s0.transpose_pieces(isplit)
    for x in pieces[1:]:  # sent, then freed
        x.close()
    m0 = _lib.DeviceCSR.merge_rows(ctx, [pieces[0]] + received, C.shape[0], isplit[0])
    ctx.sync()
    seconds = time.perf_counter() - t0
    for x in [pieces[0]] + received:
        x.close()
    return seconds, _peak(ctx, base), s0, m0


def rank0_blocks(ctx, C, W, row_cost, bounds):
    """(seconds, peak bytes, Cui_s, Ciu_s, block nnz) of rank 0's ingest from its row block [bounds[0], bounds[1])."""
    from implicit_b200 import _lib
    from implicit_b200.als import block_pieces
    from implicit_b200.utils import column_splits, nnz_balanced_splits

    users, items = C.shape
    usplit = nnz_balanced_splits(C.indptr, W, row_cost)  # what the ranks plan from the block table (block_cuts)
    isplit = column_splits(np.bincount(C.indices, minlength=items), W, row_cost)
    others = []  # the pieces ranks 1 .. W - 1 cut out of their blocks for rank 0
    for p in range(1, W):
        ps = block_pieces(ctx, C[bounds[p]:bounds[p + 1]], bounds[p], usplit)
        others.append(ps[0])
        for x in ps[1:]:
            x.close()
    received = _sent_transposes(ctx, C, usplit, isplit)
    block = C[bounds[0]:bounds[1]]
    base, _ = ctx.mem_peak()
    t0 = time.perf_counter()
    pieces = block_pieces(ctx, block, bounds[0], usplit)
    own = _lib.DeviceCSR.concat_rows(ctx, [pieces[0]], items, 0)  # what the exchange allocates for rank 0's own piece
    for x in pieces:
        x.close()
    s0 = _lib.DeviceCSR.concat_rows(ctx, [own] + others, items, usplit[0])
    for x in [own] + others:
        x.close()
    s0.column_counts()
    tp = s0.transpose_pieces(isplit)
    for x in tp[1:]:
        x.close()
    m0 = _lib.DeviceCSR.merge_rows(ctx, [tp[0]] + received, users, isplit[0])
    ctx.sync()
    seconds = time.perf_counter() - t0
    for x in [tp[0]] + received:
        x.close()
    return seconds, _peak(ctx, base), s0, m0, int(block.nnz)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=12)
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from implicit_b200 import _lib

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    C = tiling(args.blocks)
    W, row_cost = args.world, 60
    bounds = uneven_bounds(C.shape[0], W)
    ctx = _lib.Context(0)
    res = dict(gpu=gpu, nnz=int(C.nnz), users=C.shape[0], items=C.shape[1], world=W,
               rank0_rows=int(bounds[1] - bounds[0]))
    s, peak, a, b = rank0_sharded(ctx, C, W, row_cost)
    res["sharded"] = dict(s=round(s, 3), peak_gb=round(peak / 1e9, 2))
    a.close()
    b.close()
    s, peak, a, b, block_nnz = rank0_blocks(ctx, C, W, row_cost, bounds)
    res["blocks"] = dict(s=round(s, 3), peak_gb=round(peak / 1e9, 2), block_nnz=block_nnz)
    a.close()
    b.close()
    ctx.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "row_block_ingest_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
