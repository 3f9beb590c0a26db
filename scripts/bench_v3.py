#!/usr/bin/env python
"""The large-v3 family against large-v2 on the H100, in one process, models alternated rep by rep.

    python scripts/bench_v3.py [--reps 10] [--reps2 2]

Models (seeded synthetic weights, peaked like bench.py's): large-v3 (128 mels, 32 / 32 layers), large-v3-turbo
(128 mels, 32 / 4 layers) and large-v2 (80 mels, 32 / 32).  Workloads:
  configs1 : beam 5, one 3.84 s utterance, 15 generated tokens pinned (<|endoftext|> suppressed), PCM on the device
  configs2 : beam 5, 64 mixed 3.84 / 10 / 30 s windows in one engine call (per-window pinned lengths)
Per model and workload: median device time (the library's CUDA events: log-mel + generate), audio-seconds per second
and the wisb_get_timing stage split (log-mel, encoder, cross K/V, decode, decode steps), plus the bytes one persistent
decoder pass streams (bench.py's formula).  The card's name and power limit are read in the same call.  Writes one JSON
line to stdout and nothing else."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload constants and formulas shared with the headline benchmark)

MODELS = ["large-v3", "large-v3-turbo", "large-v2"]


def prompt_for(dims):
    return [dims.sot, dims.lang_first, dims.transcribe, dims.no_timestamps]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--reps2", type=int, default=2)
    args = ap.parse_args()
    import torch

    from willow_inference_server_b200 import _lib, weights as W

    if not torch.cuda.is_available():
        raise SystemExit("bench_v3 measures on the GPU: no CUDA device")
    dev = torch.device("cuda", 0)
    st = {}
    for name in MODELS:
        dims = W.WhisperDims.for_size(name)
        host, _ = bench.make_blob_host(dims)
        h = _lib.Handle.from_host(host.numpy(), 0)
        del host
        pcm = bench.synth_utterance(bench.AUDIO_SAMPLES, seed=1234)
        durs = [61440] * 22 + [160000] * 21 + [480000] * 21
        np.random.default_rng(1234).shuffle(durs)
        pcm2 = [bench.synth_utterance(n, 1234 + i) for i, n in enumerate(durs)]
        st[name] = dict(
            dims=dims, h=h, prompt=np.array([prompt_for(dims)], np.int32),
            pcm=torch.from_numpy(pcm).to(dev), pcm2=torch.from_numpy(np.concatenate(pcm2)).to(dev),
            off2=np.cumsum([0] + durs[:-1]).astype(np.int64), ns2=np.asarray(durs, np.int32),
            max2=np.asarray([2 * bench.n_out_for(n) for n in durs], np.int32), n_out2=[bench.n_out_for(n) for n in durs],
            audio2=sum(durs) / 16000.0, t1=[], t2=[], stages1=[], stages2=[])

    def run1(s):
        h = s["h"]
        h.logmel(s["pcm"].data_ptr(), np.zeros(1, np.int64), np.array([bench.AUDIO_SAMPLES], np.int32), to_host=False,
                 keep=True, pcm_on_device=True, pcm_dtype=_lib.PCM_F32, B=1)
        tl = h.timing()["logmel_ms"]
        ids, _ = h.generate(None, s["prompt"], bench.BEAM, 1.0, 1.0, bench.MAX_LENGTH, [s["dims"].eot], B=1)
        assert len(ids[0]) == bench.N_OUT, (len(ids[0]), bench.N_OUT)
        return tl, h.timing()

    def run2(s):
        h, B = s["h"], len(s["ns2"])
        h.logmel(s["pcm2"].data_ptr(), s["off2"], s["ns2"], to_host=False, keep=True, pcm_on_device=True,
                 pcm_dtype=_lib.PCM_F32, B=B)
        tl = h.timing()["logmel_ms"]
        ids, _ = h.generate(None, np.repeat(s["prompt"], B, 0), bench.BEAM, 1.0, 1.0, s["max2"], [s["dims"].eot], B=B)
        assert [len(x) for x in ids] == s["n_out2"], "decode lengths are not the pinned ones"
        return tl, h.timing()

    for s in st.values():  # warm-up: allocations, graph capture, both workloads
        for _ in range(2):
            run1(s)
        run2(s)
    for _ in range(args.reps):  # alternated: every model sees the same share of the host's and the card's noise
        for s in st.values():
            tl, t = run1(s)
            s["t1"].append(tl + t["generate_ms"])
            s["stages1"].append([tl, t["encoder_ms"], t["cross_kv_ms"], t["decode_ms"], t["decode_steps"]])
    for _ in range(args.reps2):
        for s in st.values():
            tl, t = run2(s)
            s["t2"].append(tl + t["generate_ms"])
            s["stages2"].append([tl, t["encoder_ms"], t["cross_kv_ms"], t["decode_ms"], t["decode_steps"]])
    keys = ["logmel_ms", "encoder_ms", "cross_kv_ms", "decode_ms", "decode_steps"]
    out = {"card": card(), "reps": args.reps, "reps2": args.reps2, "models": {}}
    for name, s in st.items():
        dims = s["dims"]
        m1, m2 = float(np.median(s["t1"])), float(np.median(s["t2"]))
        st1 = dict(zip(keys, (float(v) for v in np.median(np.asarray(s["stages1"]), 0))))
        st2 = dict(zip(keys, (float(v) for v in np.median(np.asarray(s["stages2"]), 0))))
        out["models"][name] = {
            "layers": [dims.n_enc_layers, dims.n_dec_layers], "n_mels": dims.n_mels, "n_vocab": dims.n_vocab,
            "decoder_pass_gb": round(bench.decoder_pass_bytes(dims) / 1e9, 3),
            "vocab_projection_gb": round(2 * dims.n_vocab * dims.d_model / 1e9, 3),
            "configs1": {"ms_median": round(m1, 3), "ms_min": round(float(min(s["t1"])), 3),
                         "ms_max": round(float(max(s["t1"])), 3),
                         "audio_s_per_s": round(bench.AUDIO_SECONDS / (m1 / 1e3), 1),
                         "per_token_ms": round(st1["decode_ms"] / max(st1["decode_steps"], 1), 4), "stages": st1},
            "configs2": {"ms_median": round(m2, 2), "audio_s_per_s": round(s["audio2"] / (m2 / 1e3), 1), "stages": st2},
        }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
