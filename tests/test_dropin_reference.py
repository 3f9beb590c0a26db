"""Drop-in test against the reference's OWN orchestration code (SURVEY.md section 7 step 2, section 8b).

`do_whisper`, `do_translate` and `chunkit` of the reference server's main.py (main.py:91-94, 514-547, 554-770) were run
unmodified over this package (`ctranslate2 := willow_inference_server_b200`, `wis.audio` := the log-mel oracle) with a
recording engine in place of the model; scripts/gen_golden_dropin.py stores every call they made on the engine in
tests/golden/dropin_calls.json -- method, positional vs keyword form, prompt ids, beam size, the windows of each call --
together with what do_whisper / do_translate returned for the canned engine results below.

  * CPU test: every recorded call binds to the signature of models.Whisper.generate / detect_language, and the record
    shows the reference behaviour the shim has to serve (one window at beam 5; detect_language first, 75 s -> 6 windows
    in 3 calls of 2 at the long-mode beam 3; the positional do_translate form).
  * GPU test: the recorded calls are replayed, exactly as the reference makes them, on the real engine; the token ids
    equal a direct wisb_generate on the same features.
"""
import inspect
import json
import os

import numpy as np
import pytest

PROMPT = [50258, 50259, 50359, 50363]


def dims_table():
    from willow_inference_server_b200 import weights as W

    d = W.WhisperDims()
    return {"sot": d.sot, "eot": d.eot, "transcribe": d.transcribe, "translate": d.translate, "no_timestamps": d.no_timestamps,
            "lang_first": d.lang_first, "n_vocab": d.n_vocab}


class FakeTokenizer:
    """Stands in for the HF tokenizer WIS loads (main.py:331-333): the four prompt tokens and the special-id list."""

    def __init__(self, dims):
        from willow_inference_server_b200.languages import LANGUAGE_CODES

        self.table = {"<|startoftranscript|>": dims["sot"], "<|transcribe|>": dims["transcribe"], "<|translate|>": dims["translate"],
                      "<|notimestamps|>": dims["no_timestamps"]}
        for i, c in enumerate(LANGUAGE_CODES):
            self.table[f"<|{c}|>"] = dims["lang_first"] + i
        self.all_special_ids = list(range(dims["eot"], dims["n_vocab"]))

    def convert_tokens_to_ids(self, toks):
        return [self.table[t] for t in toks]


class FakeProcessor:
    def __init__(self, dims):
        self.tokenizer = FakeTokenizer(dims)

    def decode(self, tokens):
        return " ".join(str(int(t)) for t in tokens)


def canned_generate(n):
    """What the recording engine answered to a generate call of n windows."""
    from willow_inference_server_b200 import models

    return [models.WhisperGenerationResult([[100 + i, 200 + i, 50257]]) for i in range(n)]


def canned_language():
    return [[("<|de|>", 0.9), ("<|en|>", 0.1)]]


def _record():
    with open(os.path.join(os.path.dirname(__file__), "golden", "dropin_calls.json")) as f:
        return json.load(f)


def _decode(v, windows):
    """A recorded argument -> the value the reference passed (feature windows rebuilt from `windows`)."""
    from willow_inference_server_b200 import models

    if isinstance(v, dict) and set(v) == {"features"}:
        return models.StorageView.from_array(np.ascontiguousarray(np.stack([windows[i] for i in v["features"]])))
    return v


def _bind(method, call, windows):
    from willow_inference_server_b200 import models

    args = [_decode(a, windows) for a in call["args"]]
    kwargs = {k: _decode(v, windows) for k, v in call["kwargs"].items()}
    bound = inspect.signature(getattr(models.Whisper, method)).bind(None, *args, **kwargs)
    bound.apply_defaults()
    return args, kwargs, bound.arguments


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_reference_do_whisper_drives_the_shim_api_on_cpu():
    rec = _record()
    d = dims_table()
    zeros = [np.zeros((80, 3000), np.float32)] * 8
    calls = rec["short"]["calls"] + rec["long"]["calls"] + rec["long"]["translate"]["calls"]
    for call in calls:  # every call the reference makes binds to the shim's signature, with what the shim accepts
        _, _, a = _bind(call["method"], call, zeros)
        assert a["features"].shape[1:] == [80, 3000]
        if call["method"] == "generate":
            assert len(a["prompts"]) == a["features"].shape[0] and all(len(p) == 4 for p in a["prompts"])
    # one short utterance: one window, beam 5, the English transcribe prompt
    short = rec["short"]
    assert short["windows"] == 1
    assert short["result"] == {"lang": "en", "text": "100 200 50257", "translation": None, "duration_ms": 3840}
    assert [(c["method"], _bind(c["method"], c, zeros)[2]["prompts"], _bind(c["method"], c, zeros)[2]["beam_size"]) for c in short["calls"]] == \
        [("generate", [PROMPT], 5)]
    # language detection + the long-audio path: 75 s -> 6 windows, two per engine call, beam 3 (long mode), LCS merge
    long = rec["long"]
    assert long["windows"] == 6 and long["result"]["lang"] == "de"
    assert long["calls"][0]["method"] == "detect_language" and long["calls"][0]["args"] == [{"features": [0]}]
    gen = [_bind("generate", c, zeros)[2] for c in long["calls"][1:]]
    assert [c["method"] for c in long["calls"][1:]] == ["generate"] * 3
    assert [g["features"].shape[0] for g in gen] == [2, 2, 2] and all(g["beam_size"] == 3 for g in gen)
    assert [w for c in long["calls"][1:] for w in c["args"][0]["features"]] == list(range(6))
    assert gen[0]["prompts"][0] == [d["sot"], d["lang_first"] + 2, d["transcribe"], d["no_timestamps"]]  # <|de|>
    # do_translate: positional generate(features, prompts, beam_size=...) with the <|translate|> prompt (main.py:535-537)
    tr = long["translate"]
    (c,) = tr["calls"]
    assert c["method"] == "generate" and len(c["args"]) == 2
    g = _bind("generate", c, zeros)[2]
    assert g["prompts"] == [[d["sot"], d["lang_first"] + 2, d["translate"], d["no_timestamps"]]] and g["beam_size"] == 4
    assert tr["result"] == "100 200 50257"
    # the latent reference bug is still the reference's: translate=True trips over len(int) (main.py:729, SURVEY section 2)
    assert rec["translate_flag"]["raises"] == "TypeError"


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_reference_do_whisper_over_the_real_engine():
    from oracle import logmel as om
    from tests.gpu_common import model_pair
    from willow_inference_server_b200 import audio, models

    rec = _record()
    dims, oracle, h = model_pair()
    model = models.Whisper(None, device="cuda", _handles=[h])
    pcm_short = om.synth_utterance(rec["short"]["n_samples"], 7)
    pcm_long = om.synth_utterance(rec["long"]["n_samples"], 8)
    short_windows = audio.log_mel_spectrogram(audio.pad_or_trim(pcm_short)).numpy()[None]
    long_windows, _ = audio.log_mel_chunks(pcm_long)
    assert long_windows.shape[0] == rec["long"]["windows"]
    replays = [(rec["short"]["calls"], short_windows), (rec["long"]["calls"], long_windows),
               (rec["long"]["translate"]["calls"], long_windows)]
    n_gen = 0
    for calls, windows in replays:
        for call in calls:
            args, kwargs, a = _bind(call["method"], call, windows)
            mel = a["features"].array
            got = getattr(model, call["method"])(*args, **kwargs)  # exactly the form the reference uses
            if call["method"] == "generate":
                want, _ = h.generate(mel, a["prompts"], beam_size=a["beam_size"])
                assert [r.sequences_ids[0] for r in got] == want
                assert all(len(w) > 0 for w in want)
                n_gen += 1
            else:
                _, probs = h.detect_language(mel)
                assert [[p for _, p in row] for row in got] == [[float(x) for x in row] for row in probs]
    assert n_gen == 5
