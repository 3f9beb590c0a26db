"""CPU tests of previous-text prompts (faster-whisper's <|startofprev|> context) in timestamp mode.

* ``get_prompt`` restates faster-whisper's ``WhisperModel.get_prompt``: [<|startofprev|>] + hotwords or the last 223
  previous tokens (timestamps included), then <|startoftranscript|>, language, task and, without timestamps,
  <|notimestamps|>.  ``models.Whisper.generate`` hands such prompts to the engine unchanged, in the timestamp mode the
  prompt asks for (CTranslate2's switch: no <|notimestamps|> anywhere).
* ``models.check_timestamp_prompt`` (the engine's acceptance rule restated) accepts any id before the last
  <|startoftranscript|> and refuses <|notimestamps|> and timestamps from it on.
* The timestamp oracle reads only generated tokens: a context that ends on a late timestamp does not move the first
  generated timestamp, and every transcript obeys the rules.
"""
import numpy as np
import pytest

from tests.gpu_common import mel_inputs
from tests.ts_oracle import TimestampOracle, check_invariants
from willow_inference_server_b200 import models, weights as W

SOT, SOT_PREV, NO_TS, EOT = 50258, 50361, 50363, 50257
TS0 = NO_TS + 1
SOT_SEQ = [SOT, 50259, 50359]          # <|startoftranscript|> <|en|> <|transcribe|>
MAX_LENGTH = 448


def get_prompt(previous_tokens, *, without_timestamps, hotwords=None):
    prompt = []
    if previous_tokens or hotwords:
        prompt.append(SOT_PREV)
        if hotwords:
            prompt.extend(hotwords)
        if previous_tokens:
            prompt.extend(previous_tokens[-(MAX_LENGTH // 2 - 1):])
    prompt.extend(SOT_SEQ)
    if without_timestamps:
        prompt.append(NO_TS)
    return prompt


def previous(n, seed=0):
    """n earlier-window tokens as faster-whisper keeps them: text ids with timestamp pairs between segments"""
    rng = np.random.default_rng(seed)
    out, t = [], TS0
    while len(out) < n:
        out.append(t)
        out.extend(int(x) for x in rng.integers(0, EOT, 3))
        t += int(rng.integers(10, 60))
        out.append(min(t, 51864))
    return out[:n]


PROMPTS = [get_prompt(previous(n, n), without_timestamps=wt) for n in (0, 8, 9, 60, 223, 300) for wt in (False, True)]
PROMPTS += [get_prompt([], without_timestamps=wt, hotwords=[440, 1029, 257]) for wt in (False, True)]   # initial_prompt


def test_previous_text_prompts_have_faster_whispers_shape():
    long = get_prompt(previous(300), without_timestamps=False)
    assert len(long) == 1 + 223 + 3 and long[0] == SOT_PREV and long[-3:] == SOT_SEQ
    assert any(t >= TS0 for t in long[1:-3])
    assert get_prompt([], without_timestamps=True) == SOT_SEQ + [NO_TS]


class Recorder:
    """one replica whose generate records the prompts and the timestamp mode it receives"""

    def __init__(self):
        self.calls = []

    def set_option(self, k, v):
        pass

    def dims(self):
        return {"d_model": 64, "n_vocab": 51865, "n_langs": 99, "n_mels": 80, "no_timestamps": NO_TS, "sot": SOT,
                "n_text_ctx": 448, "lang_first": 50259}

    def generate(self, mel, prompts, *args, B=None, timestamps=False, **kw):
        self.calls.append((np.asarray(prompts).tolist(), timestamps))
        n = len(prompts)
        return [[TS0]] * n, [0.0] * n


@pytest.mark.parametrize("prompt", PROMPTS, ids=lambda p: f"len{len(p)}{'-nots' if NO_TS in p else ''}")
def test_generate_passes_previous_text_unchanged(prompt):
    rec = Recorder()
    m = models.Whisper(None, device="cuda", _handles=[rec])
    feats = models.StorageView.from_array(np.zeros((2, 80, 3000), np.float32))
    m.generate(feats, [prompt, prompt], beam_size=5)
    assert rec.calls == [([prompt, prompt], NO_TS not in prompt)]


@pytest.mark.parametrize("prompt", [p for p in PROMPTS if NO_TS not in p])
def test_acceptance_rule_reads_from_the_last_sot(prompt):
    models.check_timestamp_prompt(prompt, SOT, NO_TS)
    for bad, msg in ((NO_TS, "notimestamps"), (TS0 + 3, "timestamp tokens")):
        with pytest.raises(ValueError, match=msg):
            models.check_timestamp_prompt(prompt + [bad], SOT, NO_TS)
    # a second sot sequence moves the checked range: the first one's context may then hold anything
    models.check_timestamp_prompt(prompt + [TS0 + 3] + SOT_SEQ, SOT, NO_TS)


def test_acceptance_rule_without_sot_checks_the_whole_prompt():
    models.check_timestamp_prompt([SOT_PREV, 11, 12], SOT, NO_TS)
    with pytest.raises(ValueError, match="timestamp tokens"):
        models.check_timestamp_prompt([SOT_PREV, TS0, 12], SOT, NO_TS)
    with pytest.raises(ValueError, match="timestamp tokens"):
        models.Whisper(None, device="cuda", _handles=[Recorder()]).generate(
            models.StorageView.from_array(np.zeros((1, 80, 3000), np.float32)), [SOT_SEQ + [TS0]])


def ts_oracle():
    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=2)
    tensors = W.synth_engine_tensors(dims, seed=11, eot_ramp=(8, 12.0), script=(4, 3.3, 1.67), ts_script=(2, 5, 8))
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    return dims, TimestampOracle.from_blob(buf)


def test_timestamp_oracle_applies_rules_to_generated_tokens_only():
    dims, oracle = ts_oracle()
    mel = mel_inputs(2)
    late = [SOT_PREV, 440, TS0 + 1400, 1029, TS0 + 1450] + SOT_SEQ   # context ends on <|29.00|>
    for beam in (1, 5):
        res = oracle.generate(mel, [late, late], beam_size=beam)
        for r in res:
            seq = r.sequences_ids[0]
            check_invariants(seq, dims)          # first generated token a timestamp <= <|1.00|>: context not read
