#!/usr/bin/env python
"""Generate tests/golden/dropin_calls.json by RUNNING THE REFERENCE's own orchestration code.

Needs a checkout of the reference server (its directory as the first argument):
    python scripts/gen_golden_dropin.py <path to willow-inference-server>

`chunkit`, `do_translate` and `do_whisper` are cut out of the reference's main.py with `ast` (main.py itself cannot be
imported without ctranslate2, librosa, aiortc, av) and executed unmodified with
  ctranslate2            := willow_inference_server_b200
  log_mel_spectrogram .. := the CPU log-mel oracle (the reference's wis.audio semantics)
and stubs for what stays outside the hot path (librosa, the HF tokenizer / processor, settings, the logger).  The model
is a recording engine: every call the reference makes on it is stored -- method, positional and keyword arguments
as given, feature windows as indices into the windows the reference computed, in order -- together with what
do_whisper / do_translate returned for the canned engine results.  tests/test_dropin_reference.py replays the record
against the shim's signatures (CPU) and on the real engine (GPU).
"""
import ast
import datetime
import json
import logging
import math
import os
import re
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import logmel as om  # noqa: E402
from tests.test_dropin_reference import FakeProcessor, canned_generate, canned_language, dims_table  # noqa: E402
from willow_inference_server_b200 import audio  # noqa: E402
import willow_inference_server_b200 as pkg  # noqa: E402


def namespace(main_py, model, audio_mod, pcm, dims):
    librosa = types.SimpleNamespace(load=lambda f, sr=16000, mono=True: (pcm, sr), get_duration=lambda y, sr: len(y) / float(sr))
    ns = {
        "datetime": datetime, "math": math, "re": re, "np": np, "librosa": librosa, "ctranslate2": pkg,
        "logger": logging.getLogger("dropin"), "settings": types.SimpleNamespace(language="en"),
        "models": types.SimpleNamespace(whisper_model_large=model, whisper_model_medium=model, whisper_model_small=model,
                                        whisper_model_base=model, whisper_model_tiny=model, whisper_processor=FakeProcessor(dims)),
        "chunk_iter": audio_mod.chunk_iter, "pad_or_trim": audio_mod.pad_or_trim,
        "log_mel_spectrogram": audio_mod.log_mel_spectrogram, "find_longest_common_sequence": audio_mod.find_longest_common_sequence,
        "beam_size": 1, "long_beam_size": 3, "long_beam_size_threshold": 12000, "support_chunking": True,
        "concurrent_gpu_chunks": 2,
    }
    tree = ast.parse(open(main_py).read())
    picked = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in {"chunkit", "do_translate", "do_whisper"}]
    assert len(picked) == 3
    exec(compile(ast.Module(body=picked, type_ignores=[]), main_py, "exec"), ns)
    return ns


class MelRecorder:
    """wis.audio surface on the CPU (the log-mel oracle); remembers every window it computed, in order."""

    def __init__(self):
        self.mels = []
        self.chunk_iter, self.find_longest_common_sequence = audio.chunk_iter, audio.find_longest_common_sequence
        self.pad_or_trim = om.pad_or_trim

    def log_mel_spectrogram(self, x):
        m = om.log_mel_spectrogram(x)
        self.mels.append(m)
        return types.SimpleNamespace(numpy=lambda: m)

    def window_of(self, w):
        hits = [i for i, m in enumerate(self.mels) if m.shape == w.shape and np.array_equal(m, w)]
        assert hits, "a feature window that the reference did not compute"
        return hits[0]


class RecordingEngine:
    def __init__(self, mels):
        self.mels, self.calls = mels, []

    def _enc(self, v):
        if isinstance(v, pkg.StorageView):
            a = np.asarray(v.array)
            return {"features": [self.mels.window_of(a[i]) for i in range(a.shape[0])]}
        if isinstance(v, (list, tuple)):
            return [self._enc(x) for x in v]
        if isinstance(v, (np.integer,)):
            return int(v)
        return v

    def _record(self, method, a, kw):
        self.calls.append({"method": method, "args": [self._enc(x) for x in a], "kwargs": {k: self._enc(v) for k, v in kw.items()}})

    def generate(self, *a, **kw):
        self._record("generate", a, kw)
        feats = a[0] if a else kw["features"]
        return canned_generate(feats.shape[0])

    def detect_language(self, *a, **kw):
        self._record("detect_language", a, kw)
        return canned_language()


def scenario(main_py, dims, n_samples, seed, do_whisper_args, translate=None, expect_error=None):
    mels = MelRecorder()
    eng = RecordingEngine(mels)
    ns = namespace(main_py, eng, mels, om.synth_utterance(n_samples, seed), dims)
    out = {"n_samples": n_samples, "seed": seed, "do_whisper_args": list(do_whisper_args)}
    if expect_error:
        try:
            ns["do_whisper"](*do_whisper_args)
        except Exception as e:  # noqa: BLE001
            out["raises"] = type(e).__name__
        return out
    lang, text, _ms, translation, _speedup, dur = ns["do_whisper"](*do_whisper_args)
    out.update(windows=len(mels.mels), calls=eng.calls, result={"lang": lang, "text": text, "translation": translation, "duration_ms": dur})
    if translate is not None:
        eng.calls = []
        tr = ns["do_translate"](eng, pkg.StorageView.from_array(mels.mels[0][None]), *translate)
        out["translate"] = {"args": list(translate), "calls": eng.calls, "result": tr}
    return out


def main():
    main_py = os.path.join(sys.argv[1], "main.py")
    dims = dims_table()
    rec = {
        "source": "chunkit / do_translate / do_whisper of the reference server's main.py, executed unmodified over the shim",
        "short": scenario(main_py, dims, 61440, 1, ("x.flac", "large", 5, "transcribe", False, "en")),
        "long": scenario(main_py, dims, 75 * 16000, 2, ("x.flac", "medium", 5, "transcribe", True, None), translate=(1, "<|de|>", 4)),
        "translate_flag": scenario(main_py, dims, 61440, 1, ("x.flac", "large", 5, "transcribe", False, "en", True), expect_error=True),
    }
    path = os.path.join(ROOT, "tests", "golden", "dropin_calls.json")
    with open(path, "w") as f:
        json.dump(rec, f, indent=1)
        f.write("\n")
    print("wrote", path)


if __name__ == "__main__":
    main()
