#!/usr/bin/env python
"""fit()'s default initial factors on one GPU: numpy's draw on the host plus its upload, against the same draw computed
on the device (als_factors_fill_pcg64), and what the difference does to a whole fit.

    python tools/init_bench.py [--configs C2,1Mx1M] [--reps 5] [--out DIR]

Shapes, f = 64: C2 (synthetic.CONFIGS["C2"], 360k x 300k, from the host generator) and 1M x 1M (20M nonzeros from the
device generator, csrc/gen.cu, downloaded once).  In one process, alternated, --reps times each, medians in ms:
  host     both sides drawn as the parent code drew them, default_rng(1).random((n, 64), float32) * float32(0.01),
           then DeviceFactors.from_host (a pageable upload that synchronises), host clock;
  device   the host bookkeeping (pcg64.get_state / after_float32_draws / set_state, host clock) and both sides'
           als_factors_create + fill, host clock ending in a synchronise; the two fill kernels alone are timed with CUDA
           events on the context's stream and set against the bytes they write (4 rows f per side) and the data sheet's
           3.35 TB/s of HBM3;
  fit      fit(torch CSR, iterations=3, Cholesky) with random_state=1 and no factors set, against the same fit with
           device factors set beforehand (so it draws nothing), host clock.
The host and device draws must be bitwise equal.  One JSON line, with the card name and power limit read in the same
run (and DIR/init_bench.json).
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

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
F = 64
SCALE = np.float32(0.01)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C2,1Mx1M")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    from implicit_b200 import AlternatingLeastSquares, _lib, pcg64, synthetic

    if not torch.cuda.is_available():
        raise SystemExit("init_bench needs a GPU and PyTorch with CUDA")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    ctx = _lib.Context(0)
    result = {"tool": "init_bench", "gpu": gpu, "reps": args.reps, "factors": F, "configs": {}}
    for name in args.configs.split(","):
        if name == "C2":
            cfg = synthetic.CONFIGS["C2"]
            M = synthetic.power_law_csr(cfg["users"], cfg["items"], cfg["nnz"], cfg["seed"])
        elif name == "1Mx1M":
            g = _lib.DeviceCSR.generate(ctx, 1_000_000, 1_000_000, 20_000_000, 7)
            M = g.download()
            g.close()
        else:
            raise SystemExit(f"unknown config {name}")
        users, items = M.shape
        D = torch.sparse_csr_tensor(*(torch.from_numpy(np.ascontiguousarray(a)).cuda()
                                      for a in (M.indptr.astype(np.int32), M.indices.astype(np.int32), M.data)),
                                    size=M.shape)

        def host_draw():
            rng = np.random.default_rng(1)
            return [_lib.DeviceFactors.from_host(ctx, rng.random((n, F), dtype=np.float32) * SCALE)
                    for n in (users, items)]

        def device_draw():
            t = time.perf_counter()
            rng = np.random.default_rng(1)
            st = pcg64.get_state(rng)
            starts = []
            for n in (users, items):
                starts.append(st)
                st = pcg64.after_float32_draws(st, n * F)
            pcg64.set_state(rng, st)
            book = time.perf_counter() - t
            out = [_lib.DeviceFactors(ctx, n, F) for n in (users, items)]
            ctx.sync()
            ctx.timer_start()
            for d, s in zip(out, starts):
                d.fill_pcg64(s, SCALE)
            kernel_ms = ctx.timer_stop()
            ctx.sync()
            return out, book * 1e3, kernel_ms

        def fit(preset):
            m = AlternatingLeastSquares(factors=F, iterations=3, use_cg=False, random_state=1)
            m._ctx = ctx
            if preset is not None:
                m.user_factors, m.item_factors = preset
            torch.cuda.synchronize()
            t = time.perf_counter()
            m.fit(D, show_progress=False)
            ms = 1e3 * (time.perf_counter() - t)
            return ms, m

        # warm-up and the bitwise check
        a = host_draw()
        b, _, _ = device_draw()
        for x, y in zip(a, b):
            assert np.array_equal(x.download().view(np.uint32), y.download().view(np.uint32)), "host and device draws differ"
        preset = [torch.as_tensor(d.snapshot(), device="cuda") for d in b]
        del a, b
        fit(None)
        fit(preset)
        times = {"host": [], "device": [], "device_bookkeeping": [], "fill_kernels": [], "fit_drawing": [],
                 "fit_preset": []}
        for _ in range(args.reps):
            ctx.sync()
            t = time.perf_counter()
            a = host_draw()
            ctx.sync()
            times["host"].append(1e3 * (time.perf_counter() - t))
            del a
            t = time.perf_counter()
            b, book, kern = device_draw()
            times["device"].append(1e3 * (time.perf_counter() - t))
            times["device_bookkeeping"].append(book)
            times["fill_kernels"].append(kern)
            del b
            times["fit_drawing"].append(fit(None)[0])
            times["fit_preset"].append(fit(preset)[0])
        med = {k: float(np.median(v)) for k, v in times.items()}
        nbytes = 4 * (users + items) * F
        result["configs"][name] = {
            "users": users, "items": items, "nnz": int(M.nnz), "median_ms": med, "all_ms": times,
            "fill_bytes": nbytes, "fill_gb_per_s": nbytes / med["fill_kernels"] / 1e6,
            "fill_share_of_hbm_datasheet": nbytes / HBM_BYTES_PER_S / (med["fill_kernels"] / 1e3),
        }
        del D, M, preset
        torch.cuda.empty_cache()
    ctx.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "init_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
