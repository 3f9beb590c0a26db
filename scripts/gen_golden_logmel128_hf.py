#!/usr/bin/env python
"""Generate tests/golden/logmel128_hf.npz: the 128-bin log-mel of the large-v3 family as HF transformers computes it
(``WhisperFeatureExtractor(feature_size=128)``, an independent implementation of openai-whisper's front end), and
transformers' 128-bin Slaney filterbank itself.

    python scripts/gen_golden_logmel128_hf.py

The inputs are not stored: tests regenerate them from ``oracle.logmel.synth_utterance`` and the seeds in CASES."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from transformers import WhisperFeatureExtractor  # noqa: E402
from transformers.audio_utils import mel_filter_bank  # noqa: E402

from oracle import logmel as om  # noqa: E402

CASES = {"synth_3p84s": (61440, 1234), "synth_10p688s": (171008, 1235), "synth_30s": (480000, 1236),
         "synth_1s": (16000, 1237)}  # name -> (samples, seed)


def main():
    fe = WhisperFeatureExtractor(feature_size=128)
    # (float32 rounds the float64 filterbank by < 2e-9, well inside the 1e-8 the tests ask)
    rec = {"filters": mel_filter_bank(201, 128, 0.0, 8000.0, 16000, norm="slaney", mel_scale="slaney").T.astype(np.float32)}
    for name, (n, seed) in CASES.items():
        pcm = om.synth_utterance(n, seed)
        mel = fe(pcm, sampling_rate=16000, return_tensors="np").input_features[0]
        assert mel.shape == (128, 3000)
        rec[name + "_n"] = np.array([n, seed], np.int64)
        rec[name + "_sub"] = mel[:, ::16].astype(np.float32)  # every 16th frame, all bins
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "logmel128_hf.npz"), **rec)


if __name__ == "__main__":
    main()
