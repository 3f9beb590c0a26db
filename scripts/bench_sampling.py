#!/usr/bin/env python
"""Cost of sampling on the H100: large-v2 with bench.py's seeded synthetic weights (peaked), <|endoftext|> suppressed and
a fixed max_length so that every arm generates the same number of tokens; arms alternated rep by rep in one process.

    python scripts/bench_sampling.py [--reps 10] [--reps2 2] [--profile-reps 2]

Arms:
  one 3.84 s window: greedy (beam 1), beam 5, best-of-5 sampling at T = 0.2, top-k 0 (5 rows: persistent decoder pass)
  64 windows: best-of-5 sampling at T = 0.2, top-k 0 (320 rows: batched decoder pass)
Per arm: median decode time per generated step (the library's CUDA events: decode_ms / decode_steps), then from a
separate torch.profiler run the device time per step of the search kernels (partial and tail).  The card's name and
power limit are read in the same call.  Writes one JSON line to stdout."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload constants shared with the headline benchmark)
from scripts.bench_processors import card  # noqa: E402

T, TOPK, N = 0.2, 0, 5
KERNELS = ("topk_partial_kernel", "sample_tail_kernel", "search_tail_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--reps2", type=int, default=2)
    ap.add_argument("--profile-reps", type=int, default=2)
    args = ap.parse_args()
    import torch

    from willow_inference_server_b200 import _lib, audio, weights as W

    if not torch.cuda.is_available():
        raise SystemExit("bench_sampling measures on the GPU: no CUDA device")
    dims = W.WhisperDims.for_size(bench.MODEL)
    host, _ = bench.make_blob_host(dims)
    h = _lib.Handle.from_host(host.numpy(), 0)
    del host
    prompt = np.array([bench.PROMPT], np.int32)
    mel1 = audio.log_mel_batch([bench.synth_utterance(bench.AUDIO_SAMPLES, seed=1234)], h)
    mel64 = audio.log_mel_batch([bench.synth_utterance(bench.AUDIO_SAMPLES, seed=1234 + i) for i in range(64)], h)
    ml = bench.MAX_LENGTH
    seeds1, seeds64 = np.arange(1, dtype=np.uint64), np.arange(64, dtype=np.uint64)

    def beam(b):
        def run():
            ids, _ = h.generate(mel1, prompt, b, 1.0, 1.0, ml, [dims.eot])
            assert len(ids[0]) == bench.N_OUT
            return h.timing()
        return run

    def sample(mel, seeds):
        def run():
            ids, _ = h.generate_sample(mel, np.repeat(prompt, len(seeds), 0), N, TOPK, T, seeds, 1.0, ml, [dims.eot])
            assert all(len(s) == bench.N_OUT for hyps in ids for s in hyps)
            return h.timing()
        return run

    arms = {"greedy_1x3.84s": beam(1), "beam5_1x3.84s": beam(5), "bestof5_T0.2_1x3.84s": sample(mel1, seeds1),
            "bestof5_T0.2_64x3.84s": sample(mel64, seeds64)}
    for fn in arms.values():  # warm-up: allocations, graph capture
        fn()
        fn()
    res = {k: [] for k in arms}
    for i in range(args.reps):
        for k, fn in arms.items():
            if k.endswith("64x3.84s") and i >= args.reps2:
                continue
            t = fn()
            res[k].append(t["decode_ms"] / t["decode_steps"])
    from torch.profiler import ProfilerActivity, profile

    out = {"card": card(), "model": bench.MODEL, "reps": args.reps, "steps": bench.N_OUT, "arms": {}}
    for k, fn in arms.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.profile_reps):
                fn()
            torch.cuda.synchronize()
        tot = dict.fromkeys(KERNELS, 0.0)
        for e in prof.key_averages():
            for kk in KERNELS:
                if kk in e.key:
                    tot[kk] += e.device_time_total
        steps = args.profile_reps * bench.N_OUT
        out["arms"][k] = {"step_ms_median": round(float(np.median(res[k])), 4), "step_ms_min": round(min(res[k]), 4),
                          "search_kernels_us_per_step": {kk: round(v / steps, 2) for kk, v in tot.items() if v}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
