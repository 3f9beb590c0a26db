"""Write tests/golden/sampling_warpers_hf.npz: the sampling distribution transformers builds from crafted rows with
``TemperatureLogitsWarper`` followed by ``TopKLogitsWarper`` (skipped for top-k 0, the whole vocabulary) and a
softmax, for temperatures 0.2, 0.5, 1 and 1.5 and top-k 0, 2, 5 and 16.

Rows: three vocabulary sizes (40, 300, 2000), float32 logits standard_normal * 3 from numpy.random.default_rng(seed)
with a quarter of the ids set to -inf (what the engine's masks and rules leave), and no two finite logits equal, so
that no tie sits at the top-k boundary (HF keeps every token tied with the k-th value; the engine breaks ties by the
lowest id, which tests/test_sampling.py checks on its own).  Stored: the logits [rows, 2000] (-inf padding past V),
V per row, and probs [rows, len(T), len(K), 2000].

    python scripts/gen_golden_sampling_hf.py      (needs transformers; run from the repository root)
"""
from __future__ import annotations

import os

import numpy as np
import torch
from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper

VOCABS = (40, 300, 2000)
TEMPS = (0.2, 0.5, 1.0, 1.5)
TOPKS = (0, 2, 5, 16)
VMAX = 2000
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "sampling_warpers_hf.npz")


def row_logits(V, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(V, dtype=np.float32) * np.float32(3.0)
    x[rng.choice(V, V // 4, replace=False)] = -np.inf
    fin = x[np.isfinite(x)]
    assert np.unique(fin).size == fin.size
    return x


def main():
    rows, vs = [], []
    for V in VOCABS:
        for seed in range(3):
            rows.append(row_logits(V, 1000 * V + seed))
            vs.append(V)
    logits = np.full((len(rows), VMAX), -np.inf, np.float32)
    probs = np.zeros((len(rows), len(TEMPS), len(TOPKS), VMAX), np.float64)
    for i, x in enumerate(rows):
        logits[i, : x.size] = x
        for a, t in enumerate(TEMPS):
            for b, k in enumerate(TOPKS):
                s = torch.from_numpy(x.copy())[None]
                ids = torch.zeros((1, 1), dtype=torch.long)
                s = TemperatureLogitsWarper(t)(ids, s)
                if k:
                    s = TopKLogitsWarper(k)(ids, s)
                probs[i, a, b, : x.size] = torch.softmax(s.double(), -1)[0].numpy()
    np.savez_compressed(OUT, logits=logits, V=np.asarray(vs, np.int32), temps=np.asarray(TEMPS),
                        topks=np.asarray(TOPKS, np.int32), probs=probs)
    print("wrote", OUT, logits.shape)


if __name__ == "__main__":
    main()
