#!/usr/bin/env python
"""Batched-decode measurement at large-v2 (BASELINE.json configs[2]: batch 64, mixed 3.84 / 10 / 30 s utterances, beam 5).
Prints one JSON object with stage times; used to iterate on the batched decoder pass (bench.py reports the same thing as
the `configs2` key)."""
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from willow_inference_server_b200 import _lib, weights as W  # noqa: E402

PROMPT = [50258, 50259, 50359, 50363]


def synth(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.float64) / 16000.0
    return (0.3 * np.sin(2 * np.pi * (200.0 + 300.0 * t) * t) + 0.05 * rng.standard_normal(n)).astype(np.float32)


def main():
    size = sys.argv[1] if len(sys.argv) > 1 else "large-v2"
    B = int(sys.argv[2]) if len(sys.argv) > 2 else 64
    reps = int(sys.argv[3]) if len(sys.argv) > 3 else 2
    dims = W.WhisperDims.for_size(size)
    t0 = time.time()
    tensors = W.synth_engine_tensors(dims, seed=0)
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    del tensors
    h = _lib.Handle.from_host(buf, 0)
    del buf
    for kv in filter(None, os.environ.get("WISB_OPTS", "").split(",")):  # e.g. WISB_OPTS=cross_tc=0,batch_pdl=0
        k, v = kv.split("=")
        h.set_option(k, int(v))
    load_s = time.time() - t0
    durs = ([61440] * 22 + [160000] * 21 + [480000] * 21)
    rng = np.random.default_rng(1234)
    rng.shuffle(durs)
    durs = durs[:B] if B <= 64 else (durs * (B // 64 + 1))[:B]
    pcm = [synth(n, 1234 + i) for i, n in enumerate(durs)]
    flat = np.concatenate(pcm)
    off = np.cumsum([0] + [len(p) for p in pcm[:-1]]).astype(np.int64)
    ns = np.asarray([len(p) for p in pcm], np.int32)
    n_out = [int(math.ceil(3.5 * n / 16000.0)) + 1 for n in durs]
    max_len = np.asarray([2 * k for k in n_out], np.int32)
    audio_s = float(sum(durs)) / 16000.0
    out = {"size": size, "B": B, "audio_s": round(audio_s, 1), "load_s": round(load_s, 1), "runs": []}
    for order in ("shuffled", "sorted"):
        idx = np.arange(B) if order == "shuffled" else np.argsort(-ns, kind="stable")
        for rep in range(reps):
            t1 = time.perf_counter()
            mel = h.logmel(flat, off[idx], ns[idx], to_host=False, keep=True)
            tl = h.timing()["logmel_ms"]
            ids, _ = h.generate(None, np.asarray([PROMPT] * B, np.int32), 5, 1.0, 1.0, max_len[idx], [dims.eot], B=B)
            wall = time.perf_counter() - t1
            t = h.timing()
            assert [len(x) for x in ids] == [n_out[i] for i in idx]
            out["runs"].append({"order": order, "rep": rep, "wall_s": round(wall, 4), "x_realtime_wall": round(audio_s / wall, 1),
                                "logmel_ms": round(tl, 2), "encoder_ms": round(t["encoder_ms"], 1), "cross_kv_ms": round(t["cross_kv_ms"], 1),
                                "decode_ms": round(t["decode_ms"], 1), "passes": int(t["decode_steps"]), "launches": int(t["launches"]),
                                "x_realtime_dev": round(audio_s / ((tl + t["generate_ms"]) * 1e-3), 1)})
    if os.environ.get("WISB_PROFILE"):
        # per-kernel-family CUDA-event sums (eager launches): a run with 2 generated tokens and a full run; the difference
        # is the decode loop alone.  gemm / cross-attention / LayerNorm+embed / self-attention (+ conv1 on the encoder side)
        h.set_option("profile", 1)
        prof = {}
        for name, ml in (("short", np.full(B, 6, np.int32)), ("full", max_len)):
            h.logmel(flat, off, ns, to_host=False, keep=True)
            h.generate(None, np.asarray([PROMPT] * B, np.int32), 5, 1.0, 1.0, ml, [dims.eot], B=B)
            t = h.timing()
            prof[name] = {k: round(t[k], 2) for k in ("gemm_ms", "attn_ms", "ln_ms", "conv1_ms", "decode_ms", "encoder_ms", "decode_steps")}
        prof["decode_only"] = {k: round(prof["full"][k] - prof["short"][k], 2) for k in prof["full"]}
        prof["legend"] = "decode_only: gemm_ms = wgmma GEMMs, attn_ms = cross-attention, ln_ms = LayerNorm/residual/embed, conv1_ms = self-attention"
        out["profile"] = prof
        h.set_option("profile", 0)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
