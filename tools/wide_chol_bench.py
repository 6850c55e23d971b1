"""Times the Cholesky half above 128 factors (csrc/cholesky_xwide.cu).

    python tools/wide_chol_bench.py [--no-host]

1. recalculate_user (als_least_squares_with_gramian) for 1,000 and 10,000 users at f = 192, 256, 512 and 1024:
   device time of the Cholesky kernels (CUDA events of the library's profiler), averaged over 3 calls after a warm-up;
2. the same 1,000 users through the reference's compiled Cython (_als._least_squares) on the host cores (oracle/_ref);
3. one Cholesky half at f = 256 on the C3-shaped CSR (138k x 27k, 20M nonzeros).
The rate is 2 (nnz fe^2 (nt + 1) / (2 nt) + R fe^3 / 3) / time with fe = roundup(f, 64) = 64 nt and R the non-empty
rows: the multiply-adds of the nt (nt + 1) / 2 tiles of the normal equations plus those of the factorisation, two flops
each (the unit of the tensor cores' quoted peak).  Device times are the Cholesky kernels only; the host time is the
reference's end-to-end wall time.  The card name and power
limit are read in the same run.
"""
import os
import subprocess
import sys
import time

os.environ.setdefault("OPENBLAS_NUM_THREADS", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from implicit_b200 import _lib, synthetic  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def work(C, f):
    nt = -(-f // 64)
    fe = 64 * nt
    R = int((np.diff(C.indptr) > 0).sum())
    return 2 * (C.nnz * fe * fe * (nt + 1) / (2 * nt) + R * fe ** 3 / 3)


def device_ms(ctx, fn, reps=3):
    fn()  # warm-up: scratch sizing, schedule
    ctx.profile(True)
    ctx.profile_read()
    for _ in range(reps):
        fn()
    prof = ctx.profile_read()
    ctx.profile(False)
    return (prof["cholesky"][0] + prof["cholesky_finish"][0]) / reps


def main():
    host = "--no-host" not in sys.argv
    ctx = _lib.Context(0)
    print(f"card: {card()}; host cores: {os.cpu_count()}")
    items = 20000
    for f in (192, 256, 512, 1024):
        rng = np.random.default_rng(f)
        Y = (rng.standard_normal((items, f)) * 0.1).astype(np.float32)
        YtY = (Y.astype(np.float64).T @ Y).astype(np.float32)
        dY = _lib.DeviceFactors.from_host(ctx, Y)
        for n in (1000, 10000):
            Cui = synthetic.power_law_csr(n, items, 50 * n, 7 + f)
            C = _lib.DeviceCSR.upload(ctx, Cui)
            dX = _lib.DeviceFactors(ctx, n, f)
            ms = device_ms(ctx, lambda: _lib.least_squares_with_gramian(ctx, YtY, C, dX, dY, 0.01))
            line = (f"recalculate_user f={f:4d} users={n:5d} nnz={Cui.nnz:7d}: device {ms:8.2f} ms, "
                    f"{work(Cui, f) / ms / 1e9:6.1f} TFLOP/s")
            if host and n == 1000:
                import oracle

                orc = oracle.get("ref")
                X = np.zeros((n, f), np.float32)
                t = time.perf_counter()
                orc._least_squares(YtY, Cui.indptr, Cui.indices, Cui.data.astype(np.float32), X, Y, 0.01, 0)
                line += f"; reference Cython end to end on the host {1e3 * (time.perf_counter() - t):9.1f} ms"
            print(line, flush=True)
            C.close()
            dX.close()
        dY.close()

    Cui, _, _, cfg = synthetic.config("C3")
    f = 256
    rng = np.random.default_rng(5)
    Y = (rng.random((cfg["items"], f), dtype=np.float32) * np.float32(0.01))
    C = _lib.DeviceCSR.upload(ctx, Cui)
    dY = _lib.DeviceFactors.from_host(ctx, Y)
    dX = _lib.DeviceFactors(ctx, cfg["users"], f)
    ms = device_ms(ctx, lambda: _lib.least_squares(ctx, C, dX, dY, 0.01))
    print(f"Cholesky half f=256 on C3 ({cfg['users']}x{cfg['items']}, {Cui.nnz} nnz): device {ms:.1f} ms, "
          f"{work(Cui, f) / ms / 1e9:.1f} TFLOP/s", flush=True)
    for h in (C, dY, dX):
        h.close()
    ctx.close()


if __name__ == "__main__":
    main()
