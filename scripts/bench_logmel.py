#!/usr/bin/env python
"""The log-mel stage alone on the H100: B = 1, 8 and 32 windows of 30 s, 80 and 128 bins, PCM already on the device.

    python scripts/bench_logmel.py [--reps 50] [--warmup 5] [--lib path/to/libwisb200.so]

Each call is one wisb_logmel (offsets / lengths upload, the power kernel and the clamp pass) timed by the library's
CUDA events (``timing()["logmel_ms"]``); the features stay on the device.  Configurations are taken round-robin, one
call each per rep, so every one sees the same share of the card's and the host's noise.  Per configuration: median,
min, max, 10th / 90th percentiles and windows per second.  ``--lib`` loads another build of the library (to compare
two kernels on one card).  The card's name, power limit and max SM clock are read in the same call.  Writes one JSON
line to stdout."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_SAMPLES = 480000
BATCHES = (1, 8, 32)
MELS = (80, 128)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--lib", default=None)
    args = ap.parse_args()
    import torch

    from willow_inference_server_b200 import _lib
    from oracle import logmel as om

    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    if not torch.cuda.is_available():
        raise SystemExit("bench_logmel measures on the GPU: no CUDA device")
    dev = torch.device("cuda", 0)
    pcm = torch.from_numpy(np.concatenate([om.synth_utterance(N_SAMPLES, 1234 + i) for i in range(max(BATCHES))])).to(dev)
    handles = {m: _lib.Handle.frontend(0, m) for m in MELS}
    configs = [(m, b) for m in MELS for b in BATCHES]
    times = {c: [] for c in configs}

    def call(m, b):
        h = handles[m]
        off = (np.arange(b, dtype=np.int64) * N_SAMPLES)
        h.logmel(pcm.data_ptr(), off, np.full(b, N_SAMPLES, np.int32), to_host=False, keep=True, pcm_on_device=True,
                 pcm_dtype=_lib.PCM_F32, B=b)
        return h.timing()["logmel_ms"]

    for _ in range(args.warmup):
        for c in configs:
            call(*c)
    for _ in range(args.reps):
        for c in configs:
            times[c].append(call(*c))
    out = {"card": card(), "lib": os.path.relpath(_lib.LIB_PATH, ROOT), "reps": args.reps, "configs": []}
    for (m, b), t in times.items():
        t = np.asarray(t)
        med = float(np.median(t))
        out["configs"].append({"n_mels": m, "B": b, "ms_median": round(med, 4), "ms_min": round(float(t.min()), 4),
                               "ms_p10": round(float(np.percentile(t, 10)), 4),
                               "ms_p90": round(float(np.percentile(t, 90)), 4), "ms_max": round(float(t.max()), 4),
                               "windows_per_s": round(b / (med / 1e3), 1)})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
