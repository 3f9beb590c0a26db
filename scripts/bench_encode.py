#!/usr/bin/env python
"""What an explicit encoder output saves on the H100: large-v2 with bench.py's seeded synthetic weights, faster-whisper's
per-window call sequence detect_language -> generate (beam 5) -> align, on 1 and on 16 windows.

    python scripts/bench_encode.py [--reps 10] [--reps16 4]

Three arms, alternated rep by rep in one process so that each sees the same share of the host's and the card's noise:
  features       : the three calls on the features, option encoder_cache off (each call encodes)
  features_cache : the same with encoder_cache on (it serves <= 2 windows encoded in one group)
  encoder_output : Whisper.encode(features) once (device form), then the three calls on its output
The time of an arm is the host clock around its calls (each returns after a stream synchronise); the encoder_output
arm also reports its encode call alone.  generate suppresses <|endoftext|> so that every arm decodes bench.py's 15
tokens.  The card's name and power limit are read in the same call.  Writes one JSON line to stdout and nothing else."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload constants shared with the headline benchmark)

ARMS = ("features", "features_cache", "encoder_output")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--reps16", type=int, default=4)
    args = ap.parse_args()
    import torch

    from willow_inference_server_b200 import _lib, audio, models, weights as W

    if not torch.cuda.is_available():
        raise SystemExit("bench_encode measures on the GPU: no CUDA device")
    dims = W.WhisperDims.for_size(bench.MODEL)
    host, _ = bench.make_blob_host(dims)
    h = _lib.Handle.from_host(host.numpy(), 0)
    del host
    m = models.Whisper(None, device="cuda", _handles=[h])
    text = [int(t) for t in np.random.default_rng(7).integers(300, dims.eot, 20)]

    def sequence(arm, feats, n):
        h.set_option("encoder_cache", 1 if arm == "features_cache" else 0)
        t0 = time.perf_counter()
        src, t_enc = feats, 0.0
        if arm == "encoder_output":
            src = m.encode(feats)
            t_enc = time.perf_counter() - t0
        m.detect_language(src)
        out = m.generate(src, [bench.PROMPT] * n, beam_size=bench.BEAM, max_length=bench.MAX_LENGTH,
                         suppress_tokens=[-1, dims.eot])
        m.align(src, bench.PROMPT[:3], [text] * n, 3000)
        t = time.perf_counter() - t0
        assert all(len(r.sequences_ids[0]) == bench.N_OUT for r in out)
        return 1e3 * t, 1e3 * t_enc, [r.sequences_ids[0] for r in out]

    result = {"card": card(), "model": bench.MODEL, "windows": {}}
    for n, reps in ((1, args.reps), (16, args.reps16)):
        durs = [bench.AUDIO_SAMPLES] * n
        mel = audio.log_mel_batch([bench.synth_utterance(k, 1234 + i) for i, k in enumerate(durs)], h)
        feats = models.StorageView.from_array(mel)
        for arm in ARMS:  # warm-up: allocations, graphs, plans
            sequence(arm, feats, n)
        times = {a: [] for a in ARMS}
        enc_ms, tokens = [], {}
        for _ in range(reps):
            for arm in ARMS:
                t, te, ids = sequence(arm, feats, n)
                times[arm].append(t)
                tokens.setdefault(arm, ids)
                if arm == "encoder_output":
                    enc_ms.append(te)
        assert tokens["encoder_output"] == tokens["features"] == tokens["features_cache"], "the arms decode differently"
        med = {a: round(float(np.median(v)), 2) for a, v in times.items()}
        result["windows"][str(n)] = {
            "reps": reps, "median_ms": med, "min_ms": {a: round(float(np.min(v)), 2) for a, v in times.items()},
            "encode_ms_median": round(float(np.median(enc_ms)), 2),
            "saved_ms_per_window_vs_features": round((med["features"] - med["encoder_output"]) / n, 2),
        }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
