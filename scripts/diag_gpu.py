#!/usr/bin/env python
"""GPU diagnostics: numerical error of the CUDA path vs the oracle on the small synthetic models (used to set the
test tolerances) -- needs a GPU."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.gpu_common import PROMPT, mel_inputs, model_pair  # noqa: E402

for cfg in [(128, 2, 2, 11, (10, 8.0)), (256, 4, 3, 5, (12, 8.0)), (384, 6, 4, 2, (14, 8.0))]:
    dims, oracle, h = model_pair(*cfg)
    mel = mel_inputs(4)
    enc = oracle.encode(mel)
    got = h.debug_encode(mel)
    print("cfg", cfg[:3], "enc max err %.3e (ref std %.2f)" % (np.abs(got - enc.numpy()).max(), enc.std()))
    toks = PROMPT + [100, 2000, 30000, 41000, 12, 50000, 7, 999, 4242]
    want = oracle.forced_logits(enc[0], toks).numpy()
    lg = h.debug_forced_logits(mel[:1], toks)
    print("   logits max err %.3e mean err %.3e (std %.2f)" % (np.abs(lg - want).max(), np.abs(lg - want).mean(), want.std()))
    for beam in (1, 5):
        tr = []
        res = oracle.generate(mel, [PROMPT] * 4, beam_size=beam, enc=enc, trace=tr)
        ids, sc = h.generate(mel, [PROMPT] * 4, beam_size=beam)
        for i in range(4):
            w = res[i].sequences_ids[0]
            print("   beam", beam, "utt", i, "match" if ids[i] == w else "DIFF", "len", len(w), len(ids[i]),
                  "min margin %.4f" % min(tr[i]), "score %.4f vs %.4f" % (sc[i], res[i].scores[0] / (1 if beam > 1 else 1)))
