#!/usr/bin/env python
"""Windows with different beam sizes and prompts: one engine call per class of options, against one mixed call
(wisb_generate with per-window options, every window its own beam / prompt / length limit in one shared decoder pass
per token), against
the batcher fed by concurrent submits of the same windows.  Synthetic large-v2 weights (peaked, as bench.py), features
computed once; <|endoftext|> is suppressed and every window has its own max_length, so each window generates a fixed
number of tokens (3.5 per second of audio) in every arm and the arms do the same search work.

Mixes:
  wis_default : 32 x 3.84 s at beam 1 + 16 x 30 s at beam 3 (WIS: beam_size 1 below 12 s, long_beam_size 3 above) +
                8 x 10 s at beam 1 with another language token
  adverse     : 1 x 30 s at beam 8 among 63 x 3.84 s greedy windows (every window keeps 8 rows: 8x the rows)

Arms run alternated rep by rep in one process.  Prints one JSON object: per mix and arm the call time (wall, host clock
around calls that end in a device synchronise), engine calls, decode steps and decode time per step summed over the
arm's engine calls (the batcher's through a wrapper around the model it calls), and the number of windows whose
tokens differ from the per-class arm (with, for each, the first differing position and both scores), plus the card's name
and power limit read in the same run."""
import argparse
import json
import math
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from willow_inference_server_b200 import _lib, models, weights as W  # noqa: E402
from willow_inference_server_b200.batcher import TranscribeBatcher  # noqa: E402

EN = [50258, 50259, 50359, 50363]
DE = [50258, 50261, 50359, 50363]
S3, S10, S30 = 61440, 160000, 480000
MIXES = {
    "wis_default": [(32, S3, 1, EN), (16, S30, 3, EN), (8, S10, 1, DE)],
    "adverse": [(63, S3, 1, EN), (1, S30, 8, EN)],
}


def synth(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.float64) / 16000.0
    return (0.3 * np.sin(2 * np.pi * (200.0 + 300.0 * t) * t) + 0.05 * rng.standard_normal(n)).astype(np.float32)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = (s.strip() for s in q.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001 -- reported, not fatal
        return {"error": repr(e)}


class Mix:
    def __init__(self, h, classes, seed):
        self.classes = classes
        durs, beams, prompts, cls = [], [], [], []
        for c, (n, dur, beam, prompt) in enumerate(classes):
            durs += [dur] * n
            beams += [beam] * n
            prompts += [prompt] * n
            cls += [c] * n
        pcm = [synth(d, seed + i) for i, d in enumerate(durs)]
        off = np.cumsum([0] + [len(p) for p in pcm[:-1]]).astype(np.int64)
        self.mel = h.logmel(np.concatenate(pcm), off, np.asarray(durs, np.int32))
        self.n_out = np.asarray([int(math.ceil(3.5 * d / 16000.0)) + 1 for d in durs], np.int32)
        self.max_len = 2 * self.n_out   # min(max_length / 2, max_length - 4) = n_out new tokens
        self.beams = np.asarray(beams, np.int32)
        self.prompts = np.asarray(prompts, np.int32)
        self.cls = np.asarray(cls)
        self.audio_s = sum(durs) / 16000.0


class Timed:
    """models.Whisper as the batcher sees it, summing each engine call's decode steps and decode time"""

    def __init__(self, model, handle):
        self.model, self.h = model, handle
        self.per_window_options, self.dims, self.n_mels = True, model.dims, model.n_mels
        self.calls = self.steps = self.decode_ms = 0

    def generate(self, *a, **kw):
        out = self.model.generate(*a, **kw)
        t = self.h.timing()
        self.calls += 1
        self.steps += t["decode_steps"]
        self.decode_ms += t["decode_ms"]
        return out


def run_arm(arm, h, batcher, timed, mix, eot):
    """-> (wall s, decode steps, decode ms, tokens, scores)"""
    n = len(mix.beams)
    ids, scores = [None] * n, [0.0] * n
    steps = dec_ms = 0.0
    t0 = time.perf_counter()
    if arm == "per_class":
        for c in range(len(mix.classes)):
            idx = np.flatnonzero(mix.cls == c)
            got = h.generate(np.ascontiguousarray(mix.mel[idx]), mix.prompts[idx], int(mix.beams[idx[0]]), 1.0, 1.0,
                             mix.max_len[idx], [eot])
            t = h.timing()
            steps += t["decode_steps"]
            dec_ms += t["decode_ms"]
            for j, i in enumerate(idx):
                ids[i], scores[i] = got[0][j], got[1][j]
    elif arm == "mixed":
        ids, scores = h.generate(mix.mel, mix.prompts, mix.beams, 1.0, 1.0, mix.max_len, [eot])
        t = h.timing()
        steps, dec_ms = t["decode_steps"], t["decode_ms"]
    else:
        timed.calls = timed.steps = timed.decode_ms = 0
        futs = [None] * n

        def submit(i):
            futs[i] = batcher.submit(mix.mel[i : i + 1], list(mix.prompts[i]), beam_size=int(mix.beams[i]),
                                           max_length=int(mix.max_len[i]), suppress_tokens=[-1, eot], return_scores=True)
        threads = [threading.Thread(target=submit, args=(i,)) for i in range(n)]
        [t.start() for t in threads]
        [t.join() for t in threads]
        for i, f in enumerate(futs):
            r = f.result(timeout=600)[0]
            ids[i], scores[i] = r.sequences_ids[0], r.scores[0]
        steps, dec_ms, calls = timed.steps, timed.decode_ms, timed.calls
    if arm == "per_class":
        calls = len(mix.classes)
    elif arm == "mixed":
        calls = 1
    wall = time.perf_counter() - t0
    return wall, steps, dec_ms, calls, ids, scores


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="large-v2")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--mixes", default="wis_default,adverse")
    args = ap.parse_args()
    dims = W.WhisperDims.for_size(args.size)
    tensors = W.synth_engine_tensors(dims, seed=0, script=(4, 3.3, 1.67))
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    del tensors
    h = _lib.Handle.from_host(buf, 0)
    del buf
    model = models.Whisper(None, device="cuda", _handles=[h])
    out = {"size": args.size, "card": card(), "mixes": {}}
    arms = ("per_class", "mixed", "batcher")
    timed = Timed(model, h)
    with TranscribeBatcher(timed, max_batch=64, max_wait_ms=50) as b:
        for name in args.mixes.split(","):
            mix = Mix(h, MIXES[name], 1234)
            for arm in arms:  # warm-up: graphs, workspaces
                run_arm(arm, h, b, timed, mix, dims.eot)
            runs = {a: [] for a in arms}
            results = {}
            for rep in range(args.reps):
                for k in range(len(arms)):
                    arm = arms[(k + rep) % len(arms)]     # rotate the order rep by rep
                    wall, steps, dec_ms, calls, ids, sc = run_arm(arm, h, b, timed, mix, dims.eot)
                    runs[arm].append({"wall_ms": round(wall * 1e3, 1), "engine_calls": calls, "decode_steps": steps,
                                      "decode_ms": round(dec_ms, 1), "ms_per_step": round(dec_ms / steps, 3)})
                    results[arm] = (ids, sc)
            ref_ids, ref_sc = results["per_class"]
            diffs = {}
            for arm in ("mixed", "batcher"):
                ids, sc = results[arm]
                d = []
                for i in range(len(ids)):
                    if list(ids[i]) != list(ref_ids[i]):
                        pos = next((t for t, (a, c) in enumerate(zip(ids[i], ref_ids[i])) if a != c), min(len(ids[i]), len(ref_ids[i])))
                        d.append({"window": i, "beam": int(mix.beams[i]), "first_diff": pos, "score": round(float(sc[i]), 5),
                                  "per_class_score": round(float(ref_sc[i]), 5)})
                diffs[arm] = {"windows_differing": len(d), "detail": d[:16]}
            assert all(len(x) == k for x, k in zip(ref_ids, mix.n_out)), "a window did not generate its fixed length"
            med = {a: float(np.median([r["wall_ms"] for r in runs[a]])) for a in arms}
            out["mixes"][name] = {"classes": [{"windows": n, "seconds": d / 16000.0, "beam": bm, "prompt": p}
                                              for n, d, bm, p in MIXES[name]],
                                  "windows": int(len(mix.beams)), "audio_s": round(mix.audio_s, 1),
                                  "rows_mixed": int(len(mix.beams) * mix.beams.max()), "rows_real": int(mix.beams.sum()),
                                  "median_wall_ms": med, "mixed_over_per_class": round(med["mixed"] / med["per_class"], 3),
                                  "runs": runs, "token_diffs_vs_per_class": diffs}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
