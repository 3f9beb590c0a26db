#!/usr/bin/env python
"""Whisper.align measurement at large-v2 (synthetic weights, default alignment heads: 320): 1 and 16 windows of 30 s,
100-token texts, median filter width 7.  Splits the call into encoder (+ cross K/V), teacher-forced passes, capture
kernels (a separate run with per-kernel events), filter and DTW, and times beam-5 generate of 104 tokens (<|endoftext|>
suppressed) on the same windows beside it.
Prints one JSON object, with the GPU's name and power limit.

    python scripts/bench_align.py [size] [reps]
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from willow_inference_server_b200 import _lib, weights as W  # noqa: E402

START = [50258, 50259, 50359]
PROMPT = START + [50363]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def synth(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.float64) / 16000.0
    return (0.3 * np.sin(2 * np.pi * (200.0 + 300.0 * t) * t) + 0.05 * rng.standard_normal(n)).astype(np.float32)


def main():
    size = sys.argv[1] if len(sys.argv) > 1 else "large-v2"
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    dims = W.WhisperDims.for_size(size)
    tensors = W.synth_engine_tensors(dims, seed=0)
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    del tensors
    h = _lib.Handle.from_host(buf, 0)
    del buf
    out = {"size": size, "gpu": gpu_info(), "text_tokens": 100, "width": 7, "runs": {}}
    rng = np.random.default_rng(7)
    for B in (1, 16):
        pcm = [synth(480000, 100 + i) for i in range(B)]
        off = np.cumsum([0] + [480000] * (B - 1)).astype(np.int64)
        mel = h.logmel(np.concatenate(pcm), off, np.full(B, 480000, np.int32))
        texts = [[int(t) for t in rng.integers(300, dims.eot, 100)] for _ in range(B)]
        res = {}
        h.align(mel, START, texts, 3000, 7)  # warm-up (workspaces, module load)
        wall, stages = [], []
        for _ in range(reps):
            t0 = time.perf_counter()
            h.align(mel, START, texts, 3000, 7)
            wall.append((time.perf_counter() - t0) * 1e3)
            stages.append(h.align_timing())
        res["align_ms"] = round(float(np.median(wall)), 2)
        for k in ("encoder_ms", "passes_ms", "filter_ms", "dtw_ms"):
            res[k] = round(float(np.median([s[k] for s in stages])), 3)
        res["passes"] = stages[-1]["passes"]
        h.set_option("profile", 1)
        h.align(mel, START, texts, 3000, 7)
        res["capture_ms_profiled"] = round(h.align_timing()["capture_ms"], 3)
        h.set_option("profile", 0)
        prompts = np.asarray([PROMPT] * B, np.int32)
        # <|endoftext|> suppressed and max_length 208: exactly 104 generated tokens, about the length of the aligned text
        h.generate(mel, prompts, 5, 1.0, 1.0, 208, [dims.eot])
        gen = []
        for _ in range(reps):
            t0 = time.perf_counter()
            h.generate(mel, prompts, 5, 1.0, 1.0, 208, [dims.eot])
            gen.append((time.perf_counter() - t0) * 1e3)
        res["generate_beam5_ms"] = round(float(np.median(gen)), 2)
        out["runs"][str(B)] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
