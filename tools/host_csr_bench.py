#!/usr/bin/env python
"""Host-resident CSRs at scale: the streamed solves against the device-resident ones on the same matrix.

    python tools/host_csr_bench.py [--blocks 127] [--huge-blocks 320] [--out DIR]

The matrix is the block-diagonal tiling of tools/large_csr_bench.py (about 17M nonzeros per block, 2.16B at 127
blocks).  Reports, as one JSON line (and DIR/host_csr_bench.json):
  gpu             name and power limit of the card, read in this call
  h2d_gbps        measured page-locked host-to-device bandwidth (1 GiB copies, CUDA events)
  device / host   for each residency: upload_s, transpose_s, device_gb (device memory the two CSRs and the transpose
                  took), chol_f64_ms (one Cholesky iteration at 64 factors) and cg_f128_ms (one CG iteration, 3 steps,
                  at 128 factors), each the median of 3 timed iterations after one warm-up
  streamed_gb     bytes one iteration copies to the device when host-resident (indices + values of Cui and Ciu)
  model_ms        max(resident time, streamed_gb / h2d_gbps): what the streamed iteration would take if copies hid
                  perfectly behind compute; ratio = host time / model_ms
  rows_equal      sampled factor rows of the host-resident and the device-resident runs are bitwise equal
  huge            with enough host memory (MemAvailable), fit() of --huge-blocks blocks (both orientations larger
                  than device memory) for one Cholesky iteration at 32 factors with automatic residency; else why not
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


def mem_available_gb():
    with open("/proc/meminfo") as fh:
        for line in fh:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) / 1e6
    return 0.0


def h2d_gbps(torch):
    n = 1 << 30
    src = torch.empty(n, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(n, dtype=torch.uint8, device="cuda")
    dst.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rates = []
    for _ in range(5):
        t0.record()
        dst.copy_(src, non_blocking=True)
        t1.record()
        t1.synchronize()
        rates.append(n / (t0.elapsed_time(t1) / 1e3) / 1e9)
    del src, dst
    torch.cuda.empty_cache()
    return float(np.median(rates))


def run(lib, ctx, Cui_host, host, torch, sample):
    users, items = Cui_host.shape
    free0 = torch.cuda.mem_get_info()[0]
    t0 = time.perf_counter()
    Cui = lib.DeviceCSR.upload(ctx, Cui_host, host=host)
    ctx.sync()
    upload_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    Ciu = Cui.transpose()
    ctx.sync()
    transpose_s = time.perf_counter() - t0
    res = dict(upload_s=round(upload_s, 2), transpose_s=round(transpose_s, 2),
               device_gb=round((free0 - torch.cuda.mem_get_info()[0]) / 1e9, 1),
               segments=[Cui.segment_count, Ciu.segment_count])
    rows = {}
    for name, f, use_cg in (("chol_f64_ms", 64, False), ("cg_f128_ms", 128, True)):
        X = lib.DeviceFactors(ctx, users, f)
        Y = lib.DeviceFactors(ctx, items, f)
        X.fill_uniform(1, 0.01)
        Y.fill_uniform(2, 0.01)

        def iteration():
            if use_cg:
                lib.least_squares_cg(ctx, Cui, X, Y, 0.01, 3)
                lib.least_squares_cg(ctx, Ciu, Y, X, 0.01, 3)
            else:
                lib.least_squares(ctx, Cui, X, Y, 0.01)
                lib.least_squares(ctx, Ciu, Y, X, 0.01)

        iteration()
        ctx.sync()
        times = []
        for _ in range(3):
            ctx.timer_start()
            iteration()
            ctx.sync()  # the timer's stop event is on the compute stream, which waits for every staged copy
            times.append(ctx.timer_stop())
        res[name] = round(float(np.median(times)), 1)
        rows[name] = (np.concatenate([X.download(int(r), 1) for r in sample[0]]),
                      np.concatenate([Y.download(int(r), 1) for r in sample[1]]))
        X.close()
        Y.close()
    Ciu.close()
    Cui.close()
    return res, rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=127)
    ap.add_argument("--huge-blocks", type=int, default=320)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    from implicit_b200 import AlternatingLeastSquares, _lib, synthetic

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    out = dict(gpu=gpu, mem_available_gb=round(mem_available_gb(), 1))
    out["h2d_gbps"] = round(h2d_gbps(torch), 2)
    base = synthetic.power_law_csr(40000, 20000, 17_000_000, 31)
    Cui_host = synthetic.block_diagonal_tiling(base, args.blocks)
    nnz = int(Cui_host.nnz)
    out.update(nnz=nnz, users=Cui_host.shape[0], items=Cui_host.shape[1])
    rng = np.random.default_rng(0)
    sample = (rng.integers(0, Cui_host.shape[0], 64), rng.integers(0, Cui_host.shape[1], 64))
    ctx = _lib.Context(0)
    res_dev, rows_dev = run(_lib, ctx, Cui_host, False, torch, sample)
    res_host, rows_host = run(_lib, ctx, Cui_host, True, torch, sample)
    out["device"], out["host"] = res_dev, res_host
    out["rows_equal"] = all(np.array_equal(a, b) for k in rows_dev for a, b in zip(rows_dev[k], rows_host[k]))
    streamed = 2 * 8 * nnz
    out["streamed_gb"] = round(streamed / 1e9, 2)
    for k in ("chol_f64_ms", "cg_f128_ms"):
        model = max(res_dev[k], streamed / (out["h2d_gbps"] * 1e9) * 1e3)
        out[k.replace("_ms", "_model_ms")] = round(model, 1)
        out[k.replace("_ms", "_ratio")] = round(res_host[k] / model, 3)
    del Cui_host

    # both orientations beyond device memory: host input 12 bytes per nonzero (int64 indices), pinned 16 per nonzero
    huge_nnz = args.huge_blocks * base.nnz
    need_gb = (12 + 16) * huge_nnz / 1e9 + 8
    if args.huge_blocks <= 0:
        out["huge"] = "not run: --huge-blocks 0"
    elif mem_available_gb() < need_gb:
        out["huge"] = f"not run: {huge_nnz} nonzeros need about {need_gb:.0f} GB of host memory, " \
                      f"{mem_available_gb():.0f} GB available"
    else:
        C = synthetic.block_diagonal_tiling(base, args.huge_blocks)
        m = AlternatingLeastSquares(factors=32, iterations=1, use_cg=False, regularization=0.01, random_state=1)
        m._ctx = ctx
        uploads = []
        real = _lib.DeviceCSR.upload.__func__
        _lib.DeviceCSR.upload = classmethod(lambda cls, *a, **k: uploads.append(k.get("host", False)) or real(cls, *a, **k))
        t0 = time.perf_counter()
        m.fit(C, show_progress=False)
        fit_s = time.perf_counter() - t0
        _lib.DeviceCSR.upload = classmethod(real)
        X = m.user_factors.reshape(args.huge_blocks, base.shape[0], 32)
        out["huge"] = dict(nnz=huge_nnz, host_resident=bool(uploads and uploads[0]), fit_1_iter_s=round(fit_s, 1),
                           blocks_equal=bool((X == X[0]).all()))
        m._ctx = None
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "host_csr_bench.json"), "w") as fh:
            fh.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
