"""Warp-MMA persistent pass (option mega_mma = 1, the default) vs SIMT persistent pass: teacher-forced logit error against the oracle (tiny model), then
the large-v2 headline step timed with both."""
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests.gpu_common import PROMPT, mel_inputs, model_pair, robust_cases  # noqa: E402

for cfg in ((128, 2, 2, 11), (256, 4, 3, 7)):
    dims, oracle, h = model_pair(*cfg)
    mel = mel_inputs(6)
    toks = PROMPT + [100, 2000, 30000, 41000, 12, 50000, 7, 999]
    want = oracle.forced_logits(oracle.encode(mel[:1])[0], toks).numpy()
    for mma in (0, 1):
        h.set_option("mega_mma", mma)
        got = h.debug_forced_logits(mel[:1], toks)
        print("d", cfg[0], "mega_mma", mma, "logit err per position:", " ".join("%.3f" % e for e in np.abs(got - want).max(axis=1)), flush=True)
    for beam in (1, 5):
        res, robust = robust_cases(oracle, mel, [PROMPT] * 6, beam, n_probe=2)
        for mma in (0, 1):
            h.set_option("mega_mma", mma)
            got = [h.generate(mel[i : i + 1], [PROMPT], beam_size=beam)[0][0] for i in range(6)]
            bad = [i for i in robust if got[i] != res[i].sequences_ids[0]]
            print("d", cfg[0], "beam", beam, "mega_mma", mma, "robust", robust, "mismatches", bad, flush=True)
    h.set_option("mega_mma", 1)

import bench  # noqa: E402
from willow_inference_server_b200 import _lib, weights as W  # noqa: E402

dims = W.WhisperDims.for_size("large-v2")
host, _ = bench.make_blob_host(dims, pinned=False)
h = _lib.Handle.from_host(host.numpy(), 0)
del host
pcm = bench.synth_utterance(bench.AUDIO_SAMPLES, 1234)
mel = h.logmel(pcm, [0], [len(pcm)])
P = np.asarray([bench.PROMPT], np.int32)
ids = {}
for mma in (0, 1, 0, 1):
    h.set_option("mega_mma", mma)
    for _ in range(3):
        out, _ = h.generate(mel, P, bench.BEAM, 1.0, 1.0, bench.MAX_LENGTH, [dims.eot])
    t = h.timing()
    ids[mma] = out[0]
    print("large-v2 mega_mma", mma, "decode_ms %.3f" % t["decode_ms"], "generate_ms %.3f" % t["generate_ms"], "tokens", out[0][:6], flush=True)
print("large-v2 tokens equal between the two passes:", ids[0] == ids[1])
