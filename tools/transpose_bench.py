"""Time and pool peak of the device transpose (als_csr_transpose), alternating library builds in one run.

    python tools/transpose_bench.py                                      # this tree's library
    python tools/transpose_bench.py variants/parent.so implicit_b200/libals_b200.so --rounds 2 --configs C2,C3

Each round runs every library once, in order, in a fresh process (ALS_B200_LIB) and prints one JSON line per
configuration and library.  C2 and C3 are the host-generated matrices of bench.py (generated once, kept in a temporary
directory for the run), uploaded; C4 is generated on the device (DeviceCSR.generate), as bench.py's C4.  After one
untimed transpose and halves, four figures are taken, the times as the median of `reps`:
  transpose_ms       the transpose alone, host clock from its call to ctx.sync();
  with_half_ms       the transpose and a Cholesky half over it (the item half of a fit, Y = the user factors);
  fit_order_ms       the first iteration of a fit in its order: the transpose, the user half over the input, then the
                     item half over the transpose, from the same initial factors every time;
  peak_bytes         the pool's peak during one transpose over what was in use before it (ctx.mem_peak()).
The card's name and power limit are read in the same run.
"""
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIGS = ["C2", "C3", "C4"]


def worker(cache, configs, reps=5):
    sys.path.insert(0, ROOT)
    import scipy.sparse as sp

    from implicit_b200 import _lib, synthetic

    ctx = _lib.Context(0)
    for name in configs:
        cfg = synthetic.CONFIGS[name]
        if name == "C4":
            Cui = _lib.DeviceCSR.generate(ctx, cfg["users"], cfg["items"], cfg["nnz"], cfg["seed"])
        else:
            host = sp.load_npz(os.path.join(cache, name + ".npz"))
            Cui = _lib.DeviceCSR.upload(ctx, host)
            del host
        users, items, nnz = Cui.shape3
        Y, X = _lib.DeviceFactors(ctx, users, cfg["factors"]), _lib.DeviceFactors(ctx, items, cfg["factors"])

        def transpose(halves):
            Y.fill_uniform(42, 0.01)
            X.fill_uniform(43, 0.01)
            ctx.sync()
            t0 = time.perf_counter()
            T = Cui.transpose()
            if halves == 2:
                _lib.least_squares(ctx, Cui, Y, X, 0.01)
            if halves:
                _lib.least_squares(ctx, T, X, Y, 0.01)
            ctx.sync()
            dt = time.perf_counter() - t0
            T.close()
            return dt * 1e3

        transpose(2)
        alone = sorted(transpose(0) for _ in range(reps))
        with_half = sorted(transpose(1) for _ in range(reps))
        fit_order = sorted(transpose(2) for _ in range(reps))
        ctx.sync()
        used0, _ = ctx.mem_peak()
        T = Cui.transpose()
        ctx.sync()
        _, peak = ctx.mem_peak()
        T.close()
        print(json.dumps(dict(lib=os.environ.get("ALS_B200_LIB", "tree"), config=name, nnz=nnz,
                              transpose_ms=round(alone[reps // 2], 3), with_half_ms=round(with_half[reps // 2], 3),
                              fit_order_ms=round(fit_order[reps // 2], 3), peak_bytes=peak - used0,
                              transpose_runs=[round(x, 3) for x in alone],
                              with_half_runs=[round(x, 3) for x in with_half],
                              fit_order_runs=[round(x, 3) for x in fit_order])), flush=True)
        for h in (Cui, X, Y):
            h.close()
    ctx.close()


def main(libs, rounds, configs):
    sys.path.insert(0, ROOT)
    import scipy.sparse as sp

    from implicit_b200 import synthetic

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(card=card)), flush=True)
    with tempfile.TemporaryDirectory() as cache:
        for name in configs:
            if name != "C4":
                sp.save_npz(os.path.join(cache, name + ".npz"), synthetic.config(name)[0], compressed=False)
        for _ in range(rounds):
            for lib in libs:
                env = dict(os.environ)
                if lib != "tree":
                    env["ALS_B200_LIB"] = os.path.abspath(lib)
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", cache, ",".join(configs)],
                                   env=env, capture_output=True, text=True)
                print(r.stdout, end="", flush=True)
                if r.returncode:
                    sys.exit(f"{lib}: the worker failed\n{r.stderr}")


if __name__ == "__main__":
    if "--worker" in sys.argv:
        i = sys.argv.index("--worker")
        worker(sys.argv[i + 1], sys.argv[i + 2].split(","))
    else:
        args = [a for a in sys.argv[1:] if not a.startswith("--")]
        n = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 1
        if "--rounds" in sys.argv:
            args.remove(str(n))
        configs = sys.argv[sys.argv.index("--configs") + 1] if "--configs" in sys.argv else ",".join(CONFIGS)
        if "--configs" in sys.argv:
            args.remove(configs)
        main(args or ["tree"], n, configs.split(","))
