"""Write tests/golden/timestamp_rules_hf.npz: what transformers' ``WhisperTimeStampLogitsProcessor`` disables on crafted
rows that reach every branch of Whisper's timestamp rules, for the three vocabulary geometries (multilingual 51865,
English-only 51864, large-v3-sized 51866) and several ``max_initial_timestamp_index`` values.

A row's logits are not stored: they are ``standard_normal(V, float32) * 3`` from ``numpy.random.default_rng(seed)``,
then ``shift`` is added to every timestamp logit (float32).  The shift places rule 5 (timestamp log-sum-exp against
the best text logit) at a chosen margin, measured on the row as processed by rules 1-4.  Stored per row: geometry
index, max_initial_timestamp_index, gen, history (padded with -1), seed, shift and the packed bitmask of the ids the
processor set to -inf.  ``tests/test_timestamp_rules.py`` replays the rows through the oracle's rules.

    python scripts/gen_golden_timestamp_rules_hf.py      (needs transformers; run from the repository root)
"""
from __future__ import annotations

import os
from types import SimpleNamespace

import numpy as np
import torch
from transformers.generation.logits_process import WhisperTimeStampLogitsProcessor

# (n_vocab, eot, no_timestamps)
GEOMETRIES = [(51865, 50257, 50363), (51864, 50256, 50362), (51866, 50257, 50364)]
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "timestamp_rules_hf.npz")
HMAX = 8


def row_logits(V, seed, shift, ts_begin):
    x = np.random.default_rng(seed).standard_normal(V, dtype=np.float32) * np.float32(3.0)
    x[ts_begin:] += np.float32(shift)
    return x


def hf_process(V, eot, no_ts, max_init, hist, logits, detect=True):
    cfg = SimpleNamespace(no_timestamps_token_id=no_ts, eos_token_id=eot, bos_token_id=eot,
                          max_initial_timestamp_index=max_init, _detect_timestamp_from_logprob=detect)
    prompt = [eot + 1, eot + 2, eot + 102]  # three stand-in prompt ids: only the length matters (begin_index)
    proc = WhisperTimeStampLogitsProcessor(cfg, begin_index=len(prompt))
    ids = torch.tensor([prompt + list(hist)], dtype=torch.long)
    return proc(ids, torch.from_numpy(logits.copy())[None])[0].numpy()


def cases(V, eot, no_ts):
    """(max_init, hist, rule-5 margin or None) covering every branch."""
    T = lambda i: no_ts + 1 + i  # noqa: E731
    last = V - 1 - (no_ts + 1)
    out = []
    for mi in (0, 1, 50, 1500):                       # rule 2 and the clamp, including one past the vocabulary
        out.append((mi, [], None))
    out += [
        (50, [T(3)], None),                           # gen 1 after a timestamp: 3a
        (50, [T(3), 500], None),                      # rule 4 at <= t
        (0, [T(3), 500], None),                       # max_initial has no effect after the first step
        (50, [T(0), 500, T(20)], None),               # 3b, rule 4 at < t
        (50, [T(0), 500, T(20), T(20)], None),        # 3a after a pair
        (50, [T(0), 500, T(20), T(25), 700], None),   # rule 4 after a pair
        (50, [500, 600, 700], None),                  # no timestamp yet: rules 1 and 5 only
        (50, [500, T(40)], None),                     # 3b without an earlier timestamp
        (50, [T(0), 9, T(last)], None),               # 3b at the last timestamp id: only it and eot..ts_begin-1 stay
        (50, [T(0), 9, T(0)], None),                  # 3b at the first timestamp id (text / timestamp boundary)
        (50, [T(0), 9, 10, 11, 12, 13, 14], None),
    ]
    for m in (1e-3, -1e-3, 0.5, -0.5, 4.0, -4.0):   # rule 5 either side of the decision
        out.append((50, [T(3), 500], m))
        out.append((50, [500, 600], m))
    out.append((50, [T(0), 500, T(20)], 1e-3))      # rule 5 when 3b has already turned the text off
    return out


def main():
    rows = {k: [] for k in ("geom", "max_init", "gen", "hist", "seed", "shift", "disabled")}
    seed = 1000
    for g, (V, eot, no_ts) in enumerate(GEOMETRIES):
        ts_begin = no_ts + 1
        for mi, hist, margin in cases(V, eot, no_ts):
            seed += 1
            shift = 0.0
            if margin is not None:
                x = row_logits(V, seed, 0.0, ts_begin)
                y = hf_process(V, eot, no_ts, mi, hist, x, detect=False).astype(np.float64)
                ts_lse = np.logaddexp.reduce(y[ts_begin:])
                shift = float(margin - (ts_lse - y[:ts_begin].max()))
            x = row_logits(V, seed, shift, ts_begin)
            y = hf_process(V, eot, no_ts, mi, hist, x)
            dis = np.zeros(max(v for v, _, _ in GEOMETRIES), bool)
            dis[:V] = np.isneginf(y)
            assert np.array_equal(y[~dis[:V]], x[~dis[:V]])  # the processor only ever disables
            rows["geom"].append(g)
            rows["max_init"].append(mi)
            rows["gen"].append(len(hist))
            rows["hist"].append(list(hist) + [-1] * (HMAX - len(hist)))
            rows["seed"].append(seed)
            rows["shift"].append(shift)
            rows["disabled"].append(np.packbits(dis))
    np.savez_compressed(
        OUT, geometries=np.asarray(GEOMETRIES, np.int32), geom=np.asarray(rows["geom"], np.int32),
        max_init=np.asarray(rows["max_init"], np.int32), gen=np.asarray(rows["gen"], np.int32),
        hist=np.asarray(rows["hist"], np.int32), seed=np.asarray(rows["seed"], np.int64),
        shift=np.asarray(rows["shift"], np.float32), disabled=np.stack(rows["disabled"]))
    print(f"{len(rows['geom'])} rows -> {os.path.normpath(OUT)} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
