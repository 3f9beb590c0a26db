"""Repetition penalty and no-repeat n-gram blocking, host side: the oracle's processors against transformers (golden
tests/golden/history_processors_hf.npz), the comparator against injected defects, the loop test model, and the
argument checks of ``Whisper.generate`` and the batcher's keys (a fake engine stands in for the GPU)."""
import os

import numpy as np
import pytest
import torch

from tests.proc_oracle import PROC_DEFECTS, banned_ngram_tokens, history_processors
from tests.test_gpu_history_processors import LOOP, step_scenarios, ref_step
from willow_inference_server_b200 import models, weights as W
from willow_inference_server_b200.batcher import TranscribeBatcher
from willow_inference_server_b200.models import WhisperGenerationResult

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "history_processors_hf.npz")


def golden_rows():
    g = np.load(GOLDEN)
    for i in range(g["V"].shape[0]):
        V, gen = int(g["V"][i]), int(g["gen"][i])
        x = np.random.default_rng(int(g["seed"][i])).standard_normal(V, dtype=np.float32) * np.float32(3.0)
        k = g["set_idx"][i] >= 0
        x[g["set_idx"][i][k]] = g["set_val"][i][k]
        y = x.copy()
        k = g["out_idx"][i] >= 0
        y[g["out_idx"][i][k]] = g["out_val"][i][k]
        yield dict(V=V, p=float(g["p"][i]), n=int(g["n"][i]), hist=[int(t) for t in g["hist"][i][:gen]], x=x, y=y)


def oracle_row(row, defect=None):
    # p as stored (float32) is the value the engine computes with
    return history_processors(torch.from_numpy(row["x"][None].copy()), [row["hist"]], row["p"], row["n"], defect)[0].numpy()


def test_oracle_processors_match_hf_golden():
    rows = list(golden_rows())
    assert len(rows) >= 100 and {r["V"] for r in rows} == {51864, 51865, 51866}
    assert {r["p"] for r in rows} >= {np.float32(0.5), np.float32(1.1), np.float32(2.0)}
    assert {r["n"] for r in rows} >= {1, 2, 3, 4}
    for i, row in enumerate(rows):
        got = oracle_row(row)
        assert np.array_equal(got, row["y"]), (i, row["V"], row["p"], row["n"], row["hist"], np.flatnonzero(got != row["y"])[:8])


def test_golden_covers_the_cases():
    rows = list(golden_rows())
    pen = [r for r in rows if r["p"] != 1]
    vals = np.concatenate([r["x"][r["hist"]] for r in pen if r["hist"]])
    assert (vals < 0).any() and (vals == 0).any() and (vals > 0).any()
    assert any(len(set(r["hist"])) < len(r["hist"]) for r in pen)                         # duplicate ids
    assert any(max(r["hist"], default=0) > 50364 for r in rows)                            # timestamp ids
    ng = [r for r in rows if r["n"] > 0]
    assert any(len(r["hist"]) + 1 < r["n"] and r["hist"] for r in ng)                      # gen + 1 < n
    assert any(np.isneginf(r["y"]).any() for r in ng)
    assert any(len(r["hist"]) == 4 and len(set(r["hist"])) == 1 and r["n"] >= 2 and np.isneginf(r["y"]).any() for r in ng)


def test_ngram_rule_by_hand():
    assert banned_ngram_tokens([5, 6, 5], 2) == [6]
    assert banned_ngram_tokens([5, 5, 5, 5], 3) == [5, 5]
    assert banned_ngram_tokens([5, 6, 7], 1) == [5, 6, 7]
    assert banned_ngram_tokens([5], 3) == [] and banned_ngram_tokens([5, 6], 3) == []
    assert banned_ngram_tokens([5, 6, 5, 6], 0) == []


@pytest.mark.parametrize("defect", PROC_DEFECTS)
def test_comparator_rejects_injected_defects(defect):
    caught = 0
    if defect in ("compound", "divide_negative", "ngram_shift"):
        for row in golden_rows():
            caught += not np.array_equal(oracle_row(row, defect), row["y"])
    # the crafted search steps of the GPU test, with float64 candidates standing in for the device's
    for sc in step_scenarios():
        good = ref_step(sc)
        bad = ref_step(sc, defect=defect)
        caught += not np.array_equal(good[0], bad[0])
    assert caught >= 1, defect


def test_loop_model_is_byte_identical_without_the_option():
    dims = W.WhisperDims(d_model=64, n_heads=1, n_enc_layers=1, n_dec_layers=1)
    a = W.synth_state_dict(dims, seed=3, script=(4, 3.3, 1.67))
    b = W.synth_state_dict(dims, seed=3, script=(4, 3.3, 1.67), loop_pool=None)
    c = W.synth_state_dict(dims, seed=3, script=(4, 3.3, 1.67), loop_pool=LOOP)
    assert a.keys() == b.keys() and all(np.array_equal(a[k], b[k]) for k in a)
    changed = [k for k in a if not np.array_equal(a[k], c[k])]
    assert changed == ["model.decoder.embed_positions.weight"]
    with pytest.raises(ValueError):
        W.synth_state_dict(dims, seed=3, loop_pool=LOOP)


# ------------------------------------------------------------------------------------------------- Python surface
class FakeHandle:
    def __init__(self):
        self.calls = []

    def set_option(self, k, v):
        pass

    def dims(self):
        return {"n_vocab": 51865, "n_langs": 99, "n_mels": 80, "no_timestamps": 50363, "n_text_ctx": 448, "lang_first": 50259}

    def generate(self, mel, prompts, *args, **kw):
        self.calls.append(kw)
        return [[1, 2]] * mel.shape[0], [0.0] * mel.shape[0]


def test_generate_validates_the_processor_arguments():
    h = FakeHandle()
    m = models.Whisper(None, device="cuda", _handles=[h])
    feats = models.StorageView.from_array(np.zeros((1, 80, 3000), np.float32))
    P = [[50258, 50259, 50359, 50363]]
    for bad in (0, -1.0, float("nan"), float("inf"), True, "1.1", None):
        with pytest.raises(ValueError, match="repetition_penalty"):
            m.generate(feats, P, repetition_penalty=bad)
    for bad in (-1, 1.5, 2.0, True, "3", 449):
        with pytest.raises(ValueError, match="no_repeat_ngram_size"):
            m.generate(feats, P, no_repeat_ngram_size=bad)
    for kw in (dict(num_hypotheses=2), dict(sampling_topk=3), dict(suppress_blank=False), dict(asynchronous=True),
               dict(suppress_tokens=[5])):
        with pytest.raises(ValueError):
            m.generate(feats, P, **kw)
    assert not h.calls
    m.generate(feats, P, repetition_penalty=1.1, no_repeat_ngram_size=np.int64(3))
    m.generate(feats, P, repetition_penalty=2, no_repeat_ngram_size=448)
    m.generate(feats, P)
    got = [(c.get("repetition_penalty"), c.get("no_repeat_ngram_size")) for c in h.calls]
    assert got == [(1.1, 3), (2.0, 448), (None, None)]            # processors off: the call is unchanged
    assert all(type(c["repetition_penalty"]) is float and type(c["no_repeat_ngram_size"]) is int for c in h.calls[:2])


class FakeEngine:
    def __init__(self):
        self.calls = []

    def generate(self, features, prompts, **opts):
        self.calls.append((features.array.shape[0], dict(opts)))
        return [WhisperGenerationResult([[int(w[0, 0])]]) for w in features.array]


def test_batcher_keeps_different_processor_settings_apart():
    eng = FakeEngine()
    win = lambda tag: np.full((1, 80, 3000), tag, np.float32)  # noqa: E731
    settings = [dict(repetition_penalty=1.0), dict(repetition_penalty=1.2), dict(repetition_penalty=1.2),
                dict(no_repeat_ngram_size=3), dict(repetition_penalty=1.2, no_repeat_ngram_size=3)]
    with TranscribeBatcher(eng, max_batch=16, max_wait_ms=100) as b:
        futs = [b.submit(win(i), [50258, 50259, 50359, 50363], beam_size=5, **kw) for i, kw in enumerate(settings)]
        res = [f.result(timeout=10)[0].sequences_ids[0][0] for f in futs]
    assert res == list(range(len(settings)))
    keys = sorted((c[1].get("repetition_penalty", 1.0), c[1].get("no_repeat_ngram_size", 0), c[0]) for c in eng.calls)
    assert keys == [(1.0, 0, 1), (1.0, 3, 1), (1.2, 0, 2), (1.2, 3, 1)]
