#!/usr/bin/env python
"""Cost of the history processors (repetition_penalty, no_repeat_ngram_size) on the H100: large-v2 with bench.py's seeded
synthetic weights, the settings (p, n) = (1, 0) and (1.1, 3) alternated rep by rep in one process.

    python scripts/bench_processors.py [--reps 20] [--reps2 2] [--profile-reps 3]

Workloads (bench.py's shapes, <|endoftext|> suppressed so that every setting generates the same number of tokens):
  configs1 : beam 5, one 3.84 s utterance, 15 generated tokens (persistent decoder pass)
  configs2 : beam 5, 64 mixed 3.84 / 10 / 30 s windows in one engine call (batched decoder pass, per-window lengths)
Per setting and workload: median decode time per generated step (the library's CUDA events: decode_ms / decode_steps)
and median call time; then, in a separate profiled run (torch.profiler, CUDA activities), the mean device time per
step of the two search kernels (topk_partial_kernel and search_tail_kernel).  The card's name and power limit are read
in the same call.  Writes one JSON line to stdout and nothing else."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload constants shared with the headline benchmark)

SETTINGS = [(1.0, 0), (1.1, 3)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--reps2", type=int, default=2)
    ap.add_argument("--profile-reps", type=int, default=3)
    args = ap.parse_args()
    import torch

    from willow_inference_server_b200 import _lib, audio, weights as W

    if not torch.cuda.is_available():
        raise SystemExit("bench_processors measures on the GPU: no CUDA device")
    dims = W.WhisperDims.for_size(bench.MODEL)
    host, _ = bench.make_blob_host(dims)
    h = _lib.Handle.from_host(host.numpy(), 0)
    del host
    prompt = np.array([bench.PROMPT], np.int32)
    mel1 = audio.log_mel_batch([bench.synth_utterance(bench.AUDIO_SAMPLES, seed=1234)], h)
    durs = [61440] * 22 + [160000] * 21 + [480000] * 21
    np.random.default_rng(1234).shuffle(durs)
    mel2 = audio.log_mel_batch([bench.synth_utterance(n, 1234 + i) for i, n in enumerate(durs)], h)
    max2 = np.asarray([2 * bench.n_out_for(n) for n in durs], np.int32)
    n_out2 = [bench.n_out_for(n) for n in durs]

    def run1(p, n):
        ids, _ = h.generate(mel1, prompt, bench.BEAM, 1.0, 1.0, bench.MAX_LENGTH, [dims.eot], repetition_penalty=p,
                            no_repeat_ngram_size=n)
        assert len(ids[0]) == bench.N_OUT, (len(ids[0]), bench.N_OUT)
        return h.timing()

    def run2(p, n):
        ids, _ = h.generate(mel2, np.repeat(prompt, len(durs), 0), bench.BEAM, 1.0, 1.0, max2, [dims.eot],
                            repetition_penalty=p, no_repeat_ngram_size=n)
        assert [len(x) for x in ids] == n_out2, "decode lengths are not the pinned ones"
        return h.timing()

    for s in SETTINGS:  # warm-up: allocations, graph capture, both workloads, both settings
        for _ in range(2):
            run1(*s)
        run2(*s)
    res = {s: {"c1": [], "c2": []} for s in SETTINGS}
    for _ in range(args.reps):  # alternated: both settings see the same share of the host's and the card's noise
        for s in SETTINGS:
            t = run1(*s)
            res[s]["c1"].append((t["decode_ms"] / t["decode_steps"], t["generate_ms"]))
    for _ in range(args.reps2):
        for s in SETTINGS:
            t = run2(*s)
            res[s]["c2"].append((t["decode_ms"] / t["decode_steps"], t["generate_ms"]))

    # separate profiled run: device time of the two search kernels per step
    from torch.profiler import ProfilerActivity, profile

    kern = {}
    for s in SETTINGS:
        for wl, fn, steps in (("c1", run1, bench.N_OUT), ("c2", run2, max(n_out2))):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.profile_reps):
                    fn(*s)
                torch.cuda.synchronize()
            tot = {"topk_partial_kernel": 0.0, "search_tail_kernel": 0.0}
            for e in prof.key_averages():
                for k in tot:
                    if k in e.key:
                        tot[k] += e.device_time_total  # microseconds over every call
            kern[(s, wl)] = {k: round(v / (args.profile_reps * steps), 2) for k, v in tot.items()}

    out = {"card": card(), "model": bench.MODEL, "reps": args.reps, "reps2": args.reps2, "settings": {}}
    for s in SETTINGS:
        c1, c2 = np.asarray(res[s]["c1"]), np.asarray(res[s]["c2"])
        out["settings"][f"p={s[0]},n={s[1]}"] = {
            "configs1": {"step_ms_median": round(float(np.median(c1[:, 0])), 4),
                         "step_ms_min": round(float(c1[:, 0].min()), 4), "step_ms_max": round(float(c1[:, 0].max()), 4),
                         "call_ms_median": round(float(np.median(c1[:, 1])), 3),
                         "search_kernels_us_per_step": kern[(s, "c1")]},
            "configs2": {"step_ms_median": round(float(np.median(c2[:, 0])), 4),
                         "call_ms_median": round(float(np.median(c2[:, 1])), 2),
                         "search_kernels_us_per_step": kern[(s, "c2")]},
        }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
