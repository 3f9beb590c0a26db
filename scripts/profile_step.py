#!/usr/bin/env python
"""Run N steps of the bench workload (large-v2, beam 5, one 3.84 s utterance) with nothing else around them, for a
profiler, e.g. Nsight Compute:

  ncu --metrics gpu__time_duration.sum --csv --log-file launches.csv python scripts/profile_step.py --steps 1
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from willow_inference_server_b200 import _lib, weights as W  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=1)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--model", default="large-v2")
ap.add_argument("--no-graphs", action="store_true")
args = ap.parse_args()

import torch  # noqa: E402

dims = W.WhisperDims.for_size(args.model)
host, _ = bench.make_blob_host(dims)
h = _lib.Handle.from_host(host.numpy(), 0)
if args.no_graphs:
    h.set_option("use_graphs", 0)

pcm = torch.from_numpy(bench.synth_utterance(bench.AUDIO_SAMPLES, 1234)).cuda()
off, ns = np.zeros(1, np.int64), np.array([bench.AUDIO_SAMPLES], np.int32)
prompts = np.array([bench.PROMPT], np.int32)
for i in range(args.warmup + args.steps):
    h.logmel(pcm.data_ptr(), off, ns, to_host=False, keep=True, pcm_on_device=True, pcm_dtype=_lib.PCM_F32, B=1)
    ids, _ = h.generate(None, prompts, bench.BEAM, 1.0, 1.0, bench.MAX_LENGTH, [dims.eot], B=1)
    t = h.timing()
    print("step", i, {k: round(v, 3) for k, v in t.items()}, flush=True)
