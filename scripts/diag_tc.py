"""Diagnostics for the wgmma cross-attention of the batched pass: teacher-forced logits with 1..8 positions per pass,
tensor-core kernel vs SIMT kernel vs the fp32 oracle, error per position."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests.gpu_common import PROMPT, mel_inputs, model_pair  # noqa: E402

dims, oracle, h = model_pair()
mel = mel_inputs(4)[:1]
toks = PROMPT + [100, 2000, 30000, 41000, 12, 50000, 7, 999]
want = oracle.forced_logits(oracle.encode(mel)[0], toks).numpy()
h.set_option("decoder_batch", 2)
for tc in (0, 1):
    h.set_option("cross_tc", tc)
    for chunk in (1, 2, 3, 5, 8):
        h.set_option("debug_chunk", chunk)
        got = h.debug_forced_logits(mel, toks)
        err = np.abs(got - want).max(axis=1)
        print("cross_tc", tc, "chunk", chunk, "err per position:", " ".join("%.3f" % e for e in err), flush=True)
h.set_option("debug_chunk", 1)
h.set_option("cross_tc", 1)
h.set_option("decoder_batch", 1)
# multi-utterance, one row per utterance everywhere (2-token prompt: the prefix pass has one row per utterance too)
mel16 = mel_inputs(16)
p2 = np.asarray([[50258, 50363]] * 16, np.int32)
a, _ = h.generate(mel16, p2, beam_size=1, max_length=24)
h.set_option("cross_tc", 0)
b, _ = h.generate(mel16, p2, beam_size=1, max_length=24)
h.set_option("cross_tc", 1)
print("greedy 16 utterances, prompt of 2: tc == simt for", sum(x == y for x, y in zip(a, b)), "of 16")
a, _ = h.generate(mel16, np.asarray([PROMPT] * 16, np.int32), beam_size=1, max_length=24)
h.set_option("cross_tc", 0)
b, _ = h.generate(mel16, np.asarray([PROMPT] * 16, np.int32), beam_size=1, max_length=24)
h.set_option("cross_tc", 1)
print("greedy 16 utterances, prompt of 4: tc == simt for", sum(x == y for x, y in zip(a, b)), "of 16")
