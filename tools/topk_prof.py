"""Workload for profiler captures of the fused top-k: Q queries (default 2 waves of 128-row CTAs) x 1M items, f=64, k=10."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from implicit_b200 import _lib, synthetic
ctx = _lib.Context(0)
Q = int(sys.argv[1]) if len(sys.argv) > 1 else 37888
I, f, k = 1_000_000, 64, 10
rng = np.random.default_rng(5)
users = rng.standard_normal((Q, f), dtype=np.float32) * np.float32(0.1)
items = rng.standard_normal((I, f), dtype=np.float32) * np.float32(0.1)
liked = synthetic.power_law_csr(Q, I, 20 * Q, 5)
di, dq = _lib.DeviceFactors.from_host(ctx, items), _lib.DeviceFactors.from_host(ctx, users)
dl = _lib.DeviceCSR.upload(ctx, liked)
ctx.profile(True)
for rep in range(2):
    ids, sc = _lib.topk(ctx, di, dq, k, liked=dl)
    p = ctx.profile_read()
    print(f"topk Q={Q}: kernel {p['topk'][0]:.2f} ms -> {Q * I / p['topk'][0] / 1e6:.1f} G candidates/s", flush=True)
