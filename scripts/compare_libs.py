"""Run one fixed set of Whisper.generate calls on two builds of libwisb200.so and check that their token ids and scores
are byte-identical.  Used to show that a change to the decoding loop leaves every result unchanged.

Model: the peaked synthetic model of the tests (d_model 128, timestamp-scripted).  Calls: greedy, beam 5, per-window
beams (with dead rows), timestamps, the history processors and best-of-5 sampling at top-k 0 and 4, each on 1 and 2
windows (the warp-MMA and the SIMT persistent passes) and on 16 windows (the batched pass).  Each library runs in a
process of its own.

    python scripts/compare_libs.py LIB_A LIB_B [--out compare_libs.json]
"""
import argparse
import json
import os
import pickle
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PROMPT = [50258, 50259, 50359, 50363]
TS_PROMPTS = [[50258, 50259, 50359], [50258, 50260, 50359], [50258, 50259, 50358], [50258, 50262, 50358]]
PROC = dict(repetition_penalty=1.3, no_repeat_ngram_size=3)
MODES = {"greedy": ((1,), False, {}), "beam5": ((5,), False, {}), "mixed": ((1, 3, 2, 1), False, {}),
         "timestamps": ((2, 1, 3), True, {}), "history": ((3, 1, 2), False, PROC)}


def run_all(lib_path):
    from willow_inference_server_b200 import _lib, weights as W
    from tests.gpu_common import RAMP, SCRIPT, mel_inputs

    _lib.LIB_PATH = lib_path
    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=2)
    tensors = W.synth_engine_tensors(dims, seed=11, eot_ramp=RAMP, script=SCRIPT, ts_script=(2, 5, 8))
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    h = _lib.Handle.from_host(buf, 0)
    mel16 = np.ascontiguousarray(mel_inputs(16))
    out = {}
    for impl in (1, 0):
        h.set_option("mega_mma", impl)
        for n in (1, 2, 16):
            if n == 16 and impl == 0:
                continue  # (the batched pass does not depend on mega_mma)
            mel = np.ascontiguousarray(mel16[:n])
            for mode, (beams, ts, proc) in MODES.items():
                b = np.asarray([beams[i % len(beams)] for i in range(n)], np.int32)
                src = TS_PROMPTS if ts else [PROMPT]
                prompts = np.asarray([src[i % len(src)] for i in range(n)], np.int32)
                ids, sc = h.generate(mel, prompts, beam_size=b, timestamps=ts, **proc)
                out[f"{mode} n={n} mma={impl}"] = (ids, np.asarray(sc, np.float32).tobytes())
            for topk in (0, 4):
                seeds = np.arange(100, 100 + n, dtype=np.uint64)
                ids, sc = h.generate_sample(mel, np.asarray([PROMPT] * n, np.int32), 5, topk, 0.8, seeds, max_length=60)
                out[f"sample topk={topk} n={n} mma={impl}"] = (ids, np.asarray(sc, np.float32).tobytes())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="*")
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--result", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        with open(args.result, "wb") as f:
            pickle.dump(run_all(args.child), f)
        return
    assert len(args.libs) == 2, "two library paths"
    import tempfile

    res = []
    with tempfile.TemporaryDirectory() as tmp:
        for i, lib in enumerate(args.libs):
            path = os.path.join(tmp, f"{i}.pkl")
            subprocess.run([sys.executable, os.path.abspath(__file__), "--child", os.path.abspath(lib), "--result", path],
                           check=True, cwd=ROOT)
            with open(path, "rb") as f:
                res.append(pickle.load(f))
    a, b = res
    differ = sorted(k for k in a if a[k] != b.get(k))
    summary = {"calls": len(a), "identical": len(a) - len(differ), "differ": differ}
    print(json.dumps(summary))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)
    sys.exit(1 if differ else 0)


if __name__ == "__main__":
    main()
