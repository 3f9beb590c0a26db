"""The cost of the no-speech probability on synthetic large-v2: the same generate call without and with the request
(no_speech_out), alternated rep by rep in one process.

Workloads, one per way the probability is obtained:
  * headline: 1 window, beam 5, 4-token prompt (fused prefill: one reduction over the prefill pass's logits);
  * prefix_2x5: 2 windows, beam 1, 5-token prompt [<|startofprev|>, text, sot, lang, task] (the persistent one-pass
    prefix, run with logits);
  * fw_227_1 / fw_227_16: 1 and 16 windows, beam 5, faster-whisper's 227-token previous-text prompt (the wide prefill,
    the gather of the SOT rows and one vocabulary GEMM over them);
  * batch_64: 64 windows, beam 5, 4-token prompt (the batched pass, fused prefill).
Per workload: the median call time of each arm (device events, encoder included), their difference, decode steps.  Ids
and scores must be byte-identical between the arms (asserted).  The card's name and power limit are read in the same run.

    python scripts/bench_no_speech.py [--reps 7] [--out bench_no_speech.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from willow_inference_server_b200 import _lib, weights as W  # noqa: E402

SOT, SOT_PREV, NO_TS, EOT = 50258, 50361, 50363, 50257
HEAD = [SOT, 50259, 50359, NO_TS]


def fw_prompt(n, rng):
    """[<|startofprev|>] + earlier text + <|startoftranscript|> <|en|> <|transcribe|>: sot at n - 3"""
    return [SOT_PREV] + [int(x) for x in rng.integers(0, EOT, n - 4)] + [SOT, 50259, 50359]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    dims = W.WhisperDims.for_size("large-v2")
    tensors = W.synth_engine_tensors(dims, seed=0)
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    del tensors
    h = _lib.Handle.from_host(buf, 0)
    rng = np.random.default_rng(0)
    mel = (rng.standard_normal((64, 80, 3000)) * 0.5).astype(np.float32)
    fw = fw_prompt(227, rng)
    workloads = [("headline", 1, HEAD, 5), ("prefix_2x5", 2, [SOT_PREV, 1234, SOT, 50259, 50359], 1),
                 ("fw_227_1", 1, fw, 5), ("fw_227_16", 16, fw, 5), ("batch_64", 64, HEAD, 5)]
    rows = []
    for name, n, prompt, beam in workloads:
        P = np.repeat(np.array([prompt], np.int32), n, 0)
        ml = max(40, len(prompt) + 20)                              # at most 20 new tokens
        times = {0: [], 1: []}
        out, ns = {}, np.zeros(n, np.float32)
        for rep in range(args.reps + 1):                            # rep 0 warms every shape up
            for arm in (0, 1):
                ids, scores = h.generate(mel[:n], P, beam, max_length=ml, no_speech_out=ns if arm else None)
                t = h.timing()
                out[arm] = (ids, np.asarray(scores, np.float32).tobytes(), t["decode_steps"])
                if rep:
                    times[arm].append(t["generate_ms"])
            assert out[0] == out[1], f"{name}: the request changed ids, scores or decode steps"
        med = {arm: float(np.median(times[arm])) for arm in (0, 1)}
        row = {"workload": name, "windows": n, "beam": beam, "prompt_len": len(prompt), "decode_steps": out[0][2],
               "off_ms": round(med[0], 3), "on_ms": round(med[1], 3), "delta_ms": round(med[1] - med[0], 3),
               "off_spread_ms": round(float(np.ptp(times[0])), 3), "on_spread_ms": round(float(np.ptp(times[1])), 3),
               "no_speech_prob": [float(x) for x in ns[:4]]}
        rows.append(row)
        print(json.dumps(row), flush=True)
    result = {"gpu": gpu, "reps": args.reps, "time": time.strftime("%Y-%m-%d %H:%M"), "rows": rows}
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps({"gpu": gpu}))


if __name__ == "__main__":
    main()
