#!/usr/bin/env python
"""Generate tests/golden/logmel_*.npz and host_logic.json by RUNNING THE REFERENCE.

Needs a checkout of the reference server (its directory as the first argument):
    python scripts/gen_golden_logmel.py <path to willow-inference-server>

Imports the reference's own ``wis.audio`` (wis/audio.py:28-159) and records its
outputs on seeded inputs.  The inputs are not stored: tests regenerate them from
``oracle.logmel.synth_utterance`` / the recipes in CASES below.
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, sys.argv[1])

from wis import audio as ref_audio  # noqa: E402  (the reference itself)

from oracle import logmel as om  # noqa: E402


def case_inputs():
    """name -> float32 pcm (unpadded)."""
    rng = np.random.default_rng(20260923)
    t30 = np.arange(480000, dtype=np.float64) / 16000.0
    return {
        "synth_3p84s": om.synth_utterance(61440, seed=1234),
        "synth_10p688s": om.synth_utterance(171008, seed=1235),
        "synth_29p248s": om.synth_utterance(467968, seed=1236),
        "zeros_30s": np.zeros(480000, np.float32),
        "sine_fullscale_30s": np.sin(2 * np.pi * 440.0 * t30).astype(np.float32),
        "noise_30s": (0.5 * rng.standard_normal(480000)).astype(np.float32),
        "long_35s_trimmed": om.synth_utterance(560000, seed=1237),
        "tiny_1sample": np.array([0.25], np.float32),
    }


def main():
    out_dir = os.path.join(ROOT, "tests", "golden")
    os.makedirs(out_dir, exist_ok=True)
    inputs = case_inputs()
    for name, pcm in inputs.items():
        padded = ref_audio.pad_or_trim(pcm)
        mel = ref_audio.log_mel_spectrogram(padded).numpy()
        assert mel.shape == (80, 3000) and mel.dtype == np.float32
        rec = {
            "n_samples": np.int64(pcm.shape[0]),
            "sub": mel[:, ::16].copy(),  # every 16th frame, all mel bins
            "sum64": np.float64(mel.astype(np.float64).sum()),
            "abs64": np.float64(np.abs(mel.astype(np.float64)).sum()),
            "max": np.float32(mel.max()),
            "min": np.float32(mel.min()),
        }
        if name == "synth_3p84s":
            rec["full"] = mel  # mostly the constant padded floor -> compresses well
        np.savez_compressed(os.path.join(out_dir, f"logmel_{name}.npz"), **rec)
        print(name, mel.shape, float(mel.min()), float(mel.max()))

    # ---- host logic goldens: chunk_iter window tables and LCS merges (wis/audio.py:106-159)
    host = {"chunk_iter": {}, "lcs": []}
    for secs in (31, 44, 60, 75, 180, 30.0001):
        n = int(round(secs * 16000))
        x = np.zeros(n, np.float32)
        host["chunk_iter"][str(n)] = [
            [int(c.shape[0]), int(s[0]), int(s[1]), int(s[2])] for c, s in ref_audio.chunk_iter(x)
        ]

    class Tok:
        all_special_ids = [50257, 50258, 50259, 50359, 50363]

    lcs_cases = [
        [[1, 2, 3, 4, 5, 6, 50257], [4, 5, 6, 7, 8, 9], [8, 9, 10, 11]],
        [[10, 11, 12, 13], [12, 13, 14, 15]],
        [[1, 2, 3], [7, 8, 9]],
        [[5, 6, 7, 8, 9, 10], [9, 10]],
        [[50258, 1, 2, 3, 4], [3, 4, 5, 50257], [4, 5, 6]],
        [[1, 2, 3, 4, 5, 6, 7, 8], [2, 3, 4, 9]],
    ]
    for seqs in lcs_cases:
        tokens = [(s, (0, 0, 0)) for s in seqs]
        merged = ref_audio.find_longest_common_sequence(tokens, Tok())
        host["lcs"].append({"in": seqs, "special": Tok.all_special_ids, "out": [int(v) for v in merged]})
    with open(os.path.join(out_dir, "host_logic.json"), "w") as f:
        json.dump(host, f, indent=1)
    print("chunk tables:", {k: len(v) for k, v in host["chunk_iter"].items()})


if __name__ == "__main__":
    main()
