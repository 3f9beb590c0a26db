"""Write tests/golden/history_processors_hf.npz: what transformers' ``RepetitionPenaltyLogitsProcessor`` and
``NoRepeatNGramLogitsProcessor`` make of crafted rows, with ``input_ids`` = the row's generated tokens, for the three
vocabulary sizes (51864, 51865, 51866).

The rows cover negative, zero and positive logits on history ids, duplicate ids, repetition_penalty 0.5, 1.1 and 2,
no_repeat_ngram_size 1..4 (including gen + 1 < n and self-overlapping histories such as ``a a a a``), histories holding
timestamp ids, and both processors together (penalty first, as the engine applies them).

A row's logits are not stored: they are ``standard_normal(V, float32) * 3`` from ``numpy.random.default_rng(seed)``,
then the history ids listed in ``set_idx`` get the float32 values ``set_val`` (to place negative, zero and positive
logits on them).  Stored per row: vocabulary size, p, n, gen, history (padded with -1), seed, the set ids / values
(padded with -1 / 0) and every id whose output differs from the input with its output value (padded with -1 / 0).
``tests/test_history_processors.py`` replays the rows through ``tests.proc_oracle.history_processors``.

    python scripts/gen_golden_history_processors_hf.py      (needs transformers; run from the repository root)
"""
from __future__ import annotations

import os

import numpy as np
import torch
from transformers.generation.logits_process import NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor

VOCABS = (51864, 51865, 51866)
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "history_processors_hf.npz")
HMAX, SMAX, CMAX = 24, 8, 32


def row_logits(V, seed, set_idx, set_val):
    x = np.random.default_rng(seed).standard_normal(V, dtype=np.float32) * np.float32(3.0)
    x[list(set_idx)] = np.asarray(set_val, np.float32)
    return x


def hf_process(hist, x, p, n):
    scores = torch.from_numpy(x.copy())[None]
    ids = torch.tensor([list(hist)], dtype=torch.long)
    if p != 1:
        scores = RepetitionPenaltyLogitsProcessor(p)(ids, scores)
    if n > 0:
        scores = NoRepeatNGramLogitsProcessor(n)(ids, scores)
    return scores[0].numpy()


def cases(V):
    """(p, n, hist, {id: logit}) rows."""
    ts = V - 1500 + 7                                 # a timestamp id of this vocabulary (near the top)
    a, b, c, d = 1000, 2345, 17, 40000
    out = []
    for p in (0.5, 1.1, 2.0):
        out.append((p, 0, [a, b, c], {a: -2.5, b: 0.0, c: 3.25}))               # negative / zero / positive
        out.append((p, 0, [a, b, a, a, c, b], {a: -1.75, b: 4.5, c: -0.125}))   # duplicates: penalised once
        out.append((p, 0, [ts, a, ts + 3, ts], {ts: 2.0, ts + 3: -3.0}))        # timestamp ids in the history
        out.append((p, 0, [], {}))                                               # gen 0: nothing to penalise
    for n in (1, 2, 3, 4):
        out.append((1.0, n, [a, b, a, b, a], {}))                # alternating history
        out.append((1.0, n, [a, a, a, a], {}))                   # self-overlapping
        out.append((1.0, n, [a, b, c, d, a, b, c], {}))          # the suffix repeats an earlier n-gram
        out.append((1.0, n, [c, ts, a, c, ts], {}))              # timestamps inside n-grams
        out.append((1.0, n, [a] * max(n - 2, 0), {}))            # gen + 1 < n (n >= 2): nothing banned
        out.append((1.0, n, [a] * (n - 1), {}))                  # gen + 1 == n: the first n-gram can only be banned
        out.append((1.0, n, [], {}))
    out.append((1.1, 2, [a, b, a, b, c, a], {a: -4.0, b: 1.5, c: 0.0}))   # both processors
    out.append((2.0, 3, [a, a, a, b, a, a], {a: 6.0, b: -6.0}))
    out.append((0.5, 1, [b, c, b], {b: -0.5, c: 0.75}))
    return out


def main():
    rows = {k: [] for k in ("V", "p", "n", "gen", "hist", "seed", "set_idx", "set_val", "out_idx", "out_val")}
    seed = 5000
    for V in VOCABS:
        for p, n, hist, setv in cases(V):
            seed += 1
            x = row_logits(V, seed, list(setv), list(setv.values()))
            y = hf_process(hist, x, p, n)
            diff = np.flatnonzero(y != x)
            assert len(hist) <= HMAX and len(setv) <= SMAX and diff.size <= CMAX
            rows["V"].append(V)
            rows["p"].append(p)
            rows["n"].append(n)
            rows["gen"].append(len(hist))
            rows["hist"].append(list(hist) + [-1] * (HMAX - len(hist)))
            rows["seed"].append(seed)
            rows["set_idx"].append(list(setv) + [-1] * (SMAX - len(setv)))
            rows["set_val"].append(list(setv.values()) + [0.0] * (SMAX - len(setv)))
            rows["out_idx"].append(list(diff) + [-1] * (CMAX - diff.size))
            rows["out_val"].append(list(y[diff]) + [0.0] * (CMAX - diff.size))
    np.savez_compressed(
        OUT, V=np.asarray(rows["V"], np.int32), p=np.asarray(rows["p"], np.float32), n=np.asarray(rows["n"], np.int32),
        gen=np.asarray(rows["gen"], np.int32), hist=np.asarray(rows["hist"], np.int32),
        seed=np.asarray(rows["seed"], np.int64), set_idx=np.asarray(rows["set_idx"], np.int32),
        set_val=np.asarray(rows["set_val"], np.float32), out_idx=np.asarray(rows["out_idx"], np.int32),
        out_val=np.asarray(rows["out_val"], np.float32))
    print(f"{len(rows['V'])} rows -> {os.path.normpath(OUT)} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
