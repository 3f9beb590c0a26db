"""Cost of the wgmma skinny GEMV at the large-v2 decoder shapes (stand-alone launches, weights from HBM every time)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from willow_inference_server_b200 import _lib  # noqa: E402

h = _lib.Handle.frontend(0)
rng = np.random.default_rng(0)
for name, N, K in (("qkv", 3840, 1280), ("o/cq/co", 1280, 1280), ("fc1", 5120, 1280), ("fc2", 1280, 5120), ("vocab", 51968, 1280)):
    x = rng.standard_normal((5, K)).astype(np.float32)
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float16)
    out, us = h.debug_gemv_tc(x, w, None, iters=200)
    want = x.astype(np.float16).astype(np.float32) @ w.astype(np.float32).T
    print(f"{name:8s} N={N:6d} K={K:5d}: {us:7.2f} us per launch, {N * K * 2 / us / 1e3:7.1f} GB/s, max err {np.abs(out - want).max():.2e}", flush=True)
