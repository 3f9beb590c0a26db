"""Previous-text prompts on synthetic large-v2: the wide prefill (option wide_prefill=1) against the prefill of at most 8
positions per pass (0), alternated rep by rep in one process.

Prompts are shaped like faster-whisper's: [<|startofprev|>] + earlier text and timestamps + <|startoftranscript|>
<|en|> <|transcribe|> (+ <|notimestamps|> with timestamps off), 4 to 227 tokens (--lens).  <|endoftext|> is suppressed
and max_length set so that every arm generates GEN tokens.  Workloads: 1 window at beam 5 (the persistent pass) and 16
windows at beam 5 (the batched pass).  Per arm: the median call time (device events, encoder included), decode steps,
and the prefill's share of the call: prefill = decode time of a 1-token call minus one step, a step being the decode
time difference between the GEN-token and the 1-token call over GEN - 1.

    python scripts/bench_prompt.py [--reps 5] [--lens 4,9,32,128,227] [--out bench_prompt.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from willow_inference_server_b200 import _lib, weights as W  # noqa: E402

GEN = 20
SOT, SOT_PREV, NO_TS, EOT = 50258, 50361, 50363, 50257


def prompt_of(n, ts, rng):
    tail = [SOT, 50259, 50359] + ([] if ts else [NO_TS])
    if n == len(tail):
        return tail
    prev = []
    t = NO_TS + 1
    while len(prev) < n - 1 - len(tail):
        prev += [t, *(int(x) for x in rng.integers(0, EOT, 4)), t + 40]
        t = NO_TS + 1 + (t - NO_TS + 49) % 1400                     # timestamps of one 30-s window: <= <|30.00|>
    return [SOT_PREV] + prev[: n - 1 - len(tail)] + tail


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    ap.add_argument("--lens", default="4,9,32,128,227", help="prompt lengths, comma-separated")
    args = ap.parse_args()
    import subprocess
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    dims = W.WhisperDims.for_size("large-v2")
    tensors = W.synth_engine_tensors(dims, seed=0)
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    del tensors
    h = _lib.Handle.from_host(buf, 0)
    rng = np.random.default_rng(0)
    mel = (rng.standard_normal((16, 80, 3000)) * 0.5).astype(np.float32)
    rows = []
    for n_win in (1, 16):
        for ts in (False, True):
            for plen in (int(x) for x in args.lens.split(",")):
                P = np.repeat(np.array([prompt_of(plen, ts, rng)], np.int32), n_win, 0)
                ml20, ml1 = max(2 * GEN, plen + GEN), plen + 1
                res = {0: {"t": [], "d20": [], "d1": []}, 1: {"t": [], "d20": [], "d1": []}}
                out = {}
                for rep in range(args.reps + 1):                   # rep 0 warms every shape up
                    for arm in (0, 1):
                        h.set_option("wide_prefill", arm)
                        ids, _ = h.generate(mel[:n_win], P, 5, max_length=ml20, extra_suppress=[EOT], timestamps=ts)
                        t20 = h.timing()
                        h.generate(mel[:n_win], P, 5, max_length=ml1, extra_suppress=[EOT], timestamps=ts)
                        t1 = h.timing()
                        out[arm] = (ids, t20["decode_steps"])
                        if rep:
                            res[arm]["t"].append(t20["generate_ms"])
                            res[arm]["d20"].append(t20["decode_ms"])
                            res[arm]["d1"].append(t1["decode_ms"])
                h.set_option("wide_prefill", 1)
                row = {"windows": n_win, "timestamps": ts, "prompt_len": plen, "same_tokens": out[0][0] == out[1][0],
                       "all_gen_tokens": all(len(s) == GEN for s in out[0][0] + out[1][0])}
                for arm in (0, 1):
                    t, d20, d1 = (float(np.median(res[arm][k])) for k in ("t", "d20", "d1"))
                    step = (d20 - d1) / (GEN - 1)
                    pre = max(0.0, d1 - step)
                    row[f"arm{arm}"] = {"call_ms": round(t, 3), "spread_ms": round(float(np.ptp(res[arm]["t"])), 3),
                                        "decode_steps": out[arm][1], "prefill_ms": round(pre, 3),
                                        "prefill_share": round(pre / t, 3)}
                rows.append(row)
                print(json.dumps(row), flush=True)
    result = {"gpu": gpu, "gen_tokens": GEN, "beam": 5, "reps": args.reps, "time": time.strftime("%Y-%m-%d %H:%M"),
              "rows": rows}
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps({"gpu": gpu}))


if __name__ == "__main__":
    main()
