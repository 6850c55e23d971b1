"""wgmma apply (csrc/dense.cu) against an fp64 product: W = Y P and Z = Y G^-1 on C2-sized factor matrices,
with the fp32 FMA tiles (ALS_B200_WHITEN_FMA=1 in a second process) as the comparison point, and its timing."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from implicit_b200 import _lib

ctx = _lib.Context(0)
rng = np.random.default_rng(7)
for rows, kind in ((1000, "normal"), (300000, "cold"), (360037, "normal")):
    Y0 = (rng.random((rows, 64), dtype=np.float32) * 0.01) if kind == "cold" else (rng.standard_normal((rows, 64)).astype(np.float32) * 0.1)
    Y = _lib.DeviceFactors.from_host(ctx, Y0)
    W, Z = _lib.whitened_factors(ctx, Y, 0.01)
    Y64 = Y0.astype(np.float64)
    G = Y64.T @ Y64 + 0.01 * np.eye(64)
    R = np.linalg.cholesky(G).T
    P = np.linalg.inv(R)
    Wt, Zt = Y64 @ P, Y64 @ np.linalg.inv(G)
    def err(a, b):
        return np.abs(a - b).max() / np.abs(b).max(), np.median(np.linalg.norm(a - b, axis=1) / np.linalg.norm(b, axis=1))
    ew, ez = err(W, Wt), err(Z, Zt)
    print(f"rows {rows} ({kind}): W max-rel {ew[0]:.2e} row-median {ew[1]:.2e} | Z max-rel {ez[0]:.2e} row-median {ez[1]:.2e} | cond(G) {np.linalg.cond(G):.1e}", flush=True)
    Gt = Y64.T @ Y64
    for knob, name in ((0, "wgmma"), (1, "fma")):
        ctx.set_knob("gramian_fma", knob)
        Gg = _lib.gramian(ctx, Y)
        ctx.profile(True); ctx.profile_read()
        for _ in range(5):
            _lib.gramian(ctx, Y)
        p = ctx.profile_read(); ctx.profile(False)
        print(f"   gramian {name}: max-rel {np.abs(Gg - Gt).max() / np.abs(Gt).max():.2e}, asymmetry {np.abs(Gg - Gg.T).max() / np.abs(Gt).max():.1e}, "
              f"{p['gramian'][0] / 5 * 1e3:.1f} us per call = {rows * 256 / (p['gramian'][0] / 5 * 1e-3) / 1e9:.0f} GB/s", flush=True)
    ctx.set_knob("gramian_fma", 0)
    del Y
print("DENSE_CHECK done")
