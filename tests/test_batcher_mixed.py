"""Cross-request batcher with an engine that takes prompts and search options per window (host logic only), and
models.Whisper.generate's checks of per-window beam_size / patience / length_penalty (a stand-in handle, no GPU)."""
import threading

import numpy as np
import pytest

from willow_inference_server_b200 import models
from willow_inference_server_b200.batcher import TranscribeBatcher
from willow_inference_server_b200.models import WhisperGenerationResult

NO_TS = 50363
PROMPT = [50258, 50259, 50359, NO_TS]
OTHER_LANG = [50258, 50260, 50359, NO_TS]
TRANSLATE = [50258, 50259, 50358, NO_TS]
TS_PROMPT = [50258, 50259, 50359]


class MixingEngine:
    """A stand-in for models.Whisper: records each call, answers with (window tag, index, its prompt's language, its
    beam) so that mix-ups between requests show."""
    per_window_options = True
    dims = {"no_timestamps": NO_TS}

    def __init__(self, delay=0.05):
        self.calls = []
        self.delay = delay
        self.lock = threading.Lock()

    def generate(self, features, prompts, **opts):
        import time

        arr = features.array
        assert len(prompts) == arr.shape[0] and len({len(p) for p in prompts}) == 1
        with self.lock:
            self.calls.append((arr.shape[0], [list(p) for p in prompts], dict(opts), [int(w[0, 0]) for w in arr]))
        time.sleep(self.delay)
        beams = opts.get("beam_size", 5)
        beams = [beams] * len(prompts) if np.isscalar(beams) else list(beams)
        return [WhisperGenerationResult([[int(w[0, 0]), int(w[0, 1]), p[1], int(b)]]) for w, p, b in zip(arr, prompts, beams)]


def _window(tag, n=1):
    a = np.zeros((n, 80, 3000), np.float32)
    a[:, 0, 0] = tag
    a[:, 0, 1] = np.arange(n)
    return a


def _submit_all(b, reqs):
    """submit every (tag, n, prompt, options) request from its own thread at once -> futures by tag"""
    futs, threads = {}, []
    for tag, n, prompt, opts in reqs:
        t = threading.Thread(target=lambda tag=tag, n=n, prompt=prompt, opts=opts:
                             futs.__setitem__(tag, b.submit(_window(tag, n), prompt, **opts)))
        t.start()
        threads.append(t)
    for t in threads:
        t.join()
    return futs


def test_requests_differing_in_search_options_and_same_length_prompt_share_a_call():
    eng = MixingEngine()
    reqs = [(1, 2, PROMPT, dict(beam_size=1)),
            (2, 1, OTHER_LANG, dict(beam_size=3, patience=2.0)),
            (3, 1, TRANSLATE, dict(length_penalty=0.5, max_length=40)),
            (4, 1, PROMPT, {})]
    with TranscribeBatcher(eng, max_batch=16, max_wait_ms=50) as b:
        futs = _submit_all(b, reqs)
        res = {tag: futs[tag].result(timeout=5) for tag, *_ in reqs}
    assert len(eng.calls) == 1, eng.calls
    n, prompts, opts, order = eng.calls[0]
    assert n == 5
    for tag, k, prompt, o in reqs:
        assert [r.sequences_ids[0] for r in res[tag]] == [[tag, i, prompt[1], o.get("beam_size", 5)] for i in range(k)]
    # every window's own prompt and options, in the order of the windows (defaults for options a request left out)
    by_tag = {tag: (prompt, o) for tag, _, prompt, o in reqs}
    assert prompts == [by_tag[t][0] for t in order]
    assert list(opts["beam_size"]) == [by_tag[t][1].get("beam_size", 5) for t in order]
    assert np.allclose(opts["patience"], [by_tag[t][1].get("patience", 1.0) for t in order])
    assert np.allclose(opts["length_penalty"], [by_tag[t][1].get("length_penalty", 1.0) for t in order])
    assert list(opts["max_length"]) == [by_tag[t][1].get("max_length", 448) for t in order]


def test_equal_per_window_options_stay_scalars_and_unset_ones_stay_unset():
    eng = MixingEngine()
    with TranscribeBatcher(eng, max_batch=8, max_wait_ms=50) as b:
        futs = _submit_all(b, [(1, 1, PROMPT, dict(beam_size=3)), (2, 2, OTHER_LANG, dict(beam_size=3))])
        [f.result(timeout=5) for f in futs.values()]
    assert len(eng.calls) == 1
    _, _, opts, _ = eng.calls[0]
    assert opts["beam_size"] == 3 and "patience" not in opts and "length_penalty" not in opts


@pytest.mark.parametrize("other", [
    (TS_PROMPT, {}),                                     # timestamp mode (and another prompt length)
    (PROMPT[:3] + [50359, NO_TS], {}),                   # a 5-token prompt
    (PROMPT, dict(repetition_penalty=1.2)),              # history processors
    (PROMPT, dict(no_repeat_ngram_size=3)),
    (PROMPT, dict(suppress_tokens=[-1, 220])),           # suppress list
    (PROMPT, dict(max_initial_timestamp_index=10)),
])
def test_incompatible_requests_stay_apart(other):
    eng = MixingEngine(delay=0.02)
    prompt, opts = other
    with TranscribeBatcher(eng, max_batch=8, max_wait_ms=40) as b:
        futs = _submit_all(b, [(1, 1, PROMPT, dict(beam_size=1)), (2, 1, prompt, dict(beam_size=3, **opts))])
        r1, r2 = futs[1].result(timeout=5), futs[2].result(timeout=5)
    assert r1[0].sequences_ids[0] == [1, 0, PROMPT[1], 1] and r2[0].sequences_ids[0] == [2, 0, prompt[1], 3]
    assert len(eng.calls) == 2 and all(c[0] == 1 for c in eng.calls)


def test_same_length_timestamp_prompts_share_a_call():
    eng = MixingEngine()
    with TranscribeBatcher(eng, max_batch=8, max_wait_ms=50) as b:
        futs = _submit_all(b, [(1, 1, TS_PROMPT, dict(beam_size=1)), (2, 1, [50258, 50261, 50358], dict(beam_size=2))])
        [f.result(timeout=5) for f in futs.values()]
    assert len(eng.calls) == 1 and eng.calls[0][0] == 2


def test_padded_rows_are_bounded_by_real_rows():
    # 6 greedy windows + 1 at beam 8 would be 56 rows for 14 real ones: the beam-8 request gets a call of its own;
    # 2 greedy + 1 at beam 3 (9 rows for 5) share one
    eng = MixingEngine()
    with TranscribeBatcher(eng, max_batch=16, max_wait_ms=50) as b:
        futs = _submit_all(b, [(1, 6, PROMPT, dict(beam_size=1)), (2, 1, PROMPT, dict(beam_size=8))])
        r1, r2 = futs[1].result(timeout=5), futs[2].result(timeout=5)
    assert [r.sequences_ids[0][3] for r in r1] == [1] * 6 and r2[0].sequences_ids[0][3] == 8
    assert sorted(c[0] for c in eng.calls) == [1, 6], eng.calls
    eng = MixingEngine()
    with TranscribeBatcher(eng, max_batch=16, max_wait_ms=50) as b:
        futs = _submit_all(b, [(1, 2, PROMPT, dict(beam_size=1)), (2, 1, OTHER_LANG, dict(beam_size=3))])
        [f.result(timeout=5) for f in futs.values()]
    assert len(eng.calls) == 1 and eng.calls[0][0] == 3


class RefusingEngine(MixingEngine):
    """Refuses, as models.Whisper does, any call holding a window whose first feature value is 13 (a stand-in for an
    argument only the engine can check, such as a prompt token outside the vocabulary)."""

    def generate(self, features, prompts, **opts):
        if any(int(w[0, 0]) == 13 for w in features.array):
            with self.lock:
                self.calls.append((features.array.shape[0], None, dict(opts), [int(w[0, 0]) for w in features.array]))
            raise ValueError("prompt token outside the vocabulary")
        return super().generate(features, prompts, **opts)


@pytest.mark.parametrize("bad", [dict(beam_size=None), dict(beam_size=[1, 2]), dict(beam_size=9), dict(beam_size=0),
                                 dict(beam_size=2.0), dict(beam_size=True), dict(patience=0.0), dict(patience=np.inf),
                                 dict(patience=None), dict(length_penalty=np.nan), dict(length_penalty="1")])
def test_bad_search_options_fail_at_submit_and_the_batcher_keeps_serving(bad):
    eng = MixingEngine(delay=0.0)
    with TranscribeBatcher(eng, max_batch=8, max_wait_ms=10) as b:
        with pytest.raises(ValueError):
            b.submit(_window(1), PROMPT, **bad)
        assert b.submit(_window(2), OTHER_LANG, beam_size=1).result(timeout=5)[0].sequences_ids[0] == [2, 0, 50260, 1]
    assert [c[3] for c in eng.calls] == [[2]]


def test_a_refused_request_does_not_fail_the_requests_merged_with_it():
    eng = RefusingEngine(delay=0.02)
    with TranscribeBatcher(eng, max_batch=16, max_wait_ms=50) as b:
        futs = _submit_all(b, [(13, 1, PROMPT, dict(beam_size=1)), (2, 2, OTHER_LANG, dict(beam_size=3)),
                               (3, 1, TRANSLATE, {})])
        with pytest.raises(ValueError, match="vocabulary"):
            futs[13].result(timeout=5)
        assert [r.sequences_ids[0] for r in futs[2].result(timeout=5)] == [[2, 0, 50260, 3], [2, 1, 50260, 3]]
        assert futs[3].result(timeout=5)[0].sequences_ids[0] == [3, 0, 50259, 5]
        assert b.submit(_window(4), PROMPT, beam_size=1).result(timeout=5)[0].sequences_ids[0][0] == 4
    assert sorted(len(c[3]) for c in eng.calls)[-1] == 4  # they were merged first, then retried one by one


def test_handle_rejects_non_integer_beams():
    from willow_inference_server_b200 import _lib

    for bad in ([1.5, 2], [True, False], ["1", "2"]):
        with pytest.raises(ValueError):
            _lib.per_window(bad, 2, np.int32, "beam_size")
    with pytest.raises(ValueError):
        _lib.per_window(["1", "2"], 2, np.float32, "patience")
    assert _lib.per_window(5, 2, np.int32, "beam_size") is None
    assert _lib.per_window([1, 8], 2, np.int32, "beam_size").tolist() == [1, 8]
    assert _lib.per_window([1, 0.5], 2, np.float32, "patience").tolist() == [1.0, 0.5]


# ------------------------------------------------------------------------------------------------- models.Whisper
class StubHandle:
    """Records what models.Whisper hands the engine handle."""

    def __init__(self):
        self.calls = []

    def set_option(self, key, value):
        pass

    def dims(self):
        return {"n_vocab": 51865, "no_timestamps": NO_TS, "d_model": 128, "n_text_ctx": 448, "n_mels": 80, "lang_first": 50259,
                "n_langs": 99}

    def generate(self, mel, prompts, beam_size, patience, length_penalty, max_length, extra, **kw):
        self.calls.append((beam_size, patience, length_penalty, max_length))
        return [[7]] * mel.shape[0], [0.0] * mel.shape[0]


def test_whisper_generate_checks_per_window_options():
    h = StubHandle()
    m = models.Whisper(None, device="cuda", _handles=[h])
    feats = models.StorageView.from_array(np.zeros((3, 80, 3000), np.float32))
    prompts = [PROMPT, OTHER_LANG, TRANSLATE]
    for bad in (dict(beam_size=[1, 2]), dict(beam_size=[1, 2, 9]), dict(beam_size=[0, 1, 1]), dict(beam_size=[1.5, 1, 1]),
                dict(patience=[1.0, 0.0, 1.0]), dict(patience=[1.0, np.inf, 1.0]), dict(patience=[np.nan, 1, 1]),
                dict(patience=[1.0] * 4), dict(length_penalty=[1.0, np.nan, 1.0]), dict(length_penalty=[np.inf] * 3),
                dict(length_penalty=[[1.0] * 3]), dict(beam_size=["5", "5", "5"])):
        with pytest.raises(ValueError):
            m.generate(feats, prompts, **bad)
    assert not h.calls
    m.generate(feats, prompts, beam_size=[1, 3, 8], patience=[0.5, 1, 2], length_penalty=[1.0, 0.0, 0.6])
    beam, pat, lp, _ = h.calls[-1]
    assert list(beam) == [1, 3, 8] and list(pat) == [0.5, 1, 2] and list(lp) == [1.0, 0.0, 0.6]
    m.generate(feats, prompts, beam_size=2)       # scalars pass through unchanged
    assert h.calls[-1][:3] == (2, 1, 1)
    # prompts of different lengths or timestamp modes still cannot share a call
    with pytest.raises(ValueError):
        m.generate(feats, [PROMPT, TS_PROMPT, PROMPT], beam_size=[1, 2, 3])
    with pytest.raises(ValueError):
        m.generate(feats, [PROMPT, TS_PROMPT + [50000], PROMPT], beam_size=[1, 2, 3])
