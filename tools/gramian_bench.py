"""Device time of the Gramian G = Y^T Y, alternating library builds in one run (A/B of csrc/gramian.cu).

    python tools/gramian_bench.py                         # this tree's library
    python tools/gramian_bench.py variants/old.so implicit_b200/libals_b200.so --rounds 3

Each round runs every library once, in order, in a fresh process (ALS_B200_LIB) and prints one JSON line per case and
library, then the median over rounds.  Y is filled on the device (U(0, 0.01), the cold start), so that no host memory
bounds the size.  A case times `reps` calls of als_gramian_shard over all of Y's rows (the launch of als_gramian
without its copy of G to the host) with CUDA events, after `warmup` untimed calls.  The card's name and power limit
are read in the same run.  A variant of gramian.cu builds with VARIANT_SRC=gramian VARIANT_FILE=<its source>
tools/build_variant.sh <name>.
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
#: (factors, rows): 64 runs the wgmma kernel, 128 the FMA partial kernel, 256 and 1024 the wide kernel
CASES = [(64, 1 << 20), (64, 10_000_000), (128, 1 << 20), (128, 10_000_000), (256, 1 << 20), (256, 10_000_000),
         (1024, 1 << 20)]


def worker(warmup=5, reps=50):
    sys.path.insert(0, ROOT)
    from implicit_b200 import _lib

    ctx = _lib.Context(0)
    for f, rows in CASES:
        d = _lib.DeviceFactors(ctx, rows, f)
        d.fill_uniform(7, 0.01)
        for _ in range(warmup):
            _lib.gramian_shard(ctx, d, 0, rows)
        ctx.timer_start()
        for _ in range(reps):
            _lib.gramian_shard(ctx, d, 0, rows)
        ms = ctx.timer_stop() / reps
        d.close()
        print(json.dumps(dict(lib=os.environ.get("ALS_B200_LIB", "tree"), f=f, rows=rows, ms=round(ms, 4),
                              GBps=round(4.0 * rows * f / ms / 1e6, 1))), flush=True)
    ctx.close()


def main(libs, rounds):
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(card=card)), flush=True)
    times = {}
    for _ in range(rounds):
        for lib in libs:
            env = dict(os.environ)
            if lib != "tree":
                env["ALS_B200_LIB"] = os.path.abspath(lib)
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker"], env=env, capture_output=True,
                                 text=True, check=True).stdout
            for line in out.splitlines():
                print(line, flush=True)
                r = json.loads(line)
                times.setdefault((r["f"], r["rows"]), {}).setdefault(lib, []).append(r["ms"])
    print(f"median of {rounds} rounds, ms per call ({card}):")
    for (f, rows), per_lib in sorted(times.items()):
        cells = "  ".join(f"{os.path.basename(lib)} {sorted(v)[len(v) // 2]:.3f}" for lib, v in per_lib.items())
        print(f"  f={f:5d} rows={rows:9d}: {cells}")


if __name__ == "__main__":
    if "--worker" in sys.argv:
        worker()
    else:
        args = [a for a in sys.argv[1:] if not a.startswith("--")]
        n = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 3
        if "--rounds" in sys.argv:
            args.remove(str(n))
        main(args or ["tree"], n)
