"""CPU tests of the no-speech probability's host side: Whisper.generate hands each part of the windows a slice of one
array and reports each window's own value (features, host and device encoder outputs, beam and sampling calls, two
replicas), the prompt check, the calls Handle makes into the library, and the batcher merging requests that differ only
in return_no_speech_prob (fake handles and a recorder library; no GPU)."""
import ctypes
import threading

import numpy as np
import pytest

from willow_inference_server_b200 import _lib, models
from willow_inference_server_b200.batcher import TranscribeBatcher
from willow_inference_server_b200.models import StorageView, WhisperGenerationResult

D = 384
SOT = 50258


def prompt(w):
    """window w's prompt: its last token tags it"""
    return [SOT, 50259, 50359, 1000 + w]


def tag(p):
    return (int(p[-1]) - 1000) / 64 + 1 / 128


class FakeHandle:
    """a replica that fills no_speech_out with each window's tag (from its prompt)"""

    def __init__(self):
        self.calls = []

    def set_option(self, k, v):
        pass

    def dims(self):
        return {"d_model": D, "n_vocab": 51865, "n_langs": 99, "n_mels": 80, "no_timestamps": 50363, "n_text_ctx": 448,
                "lang_first": 50259, "sot": SOT}

    def load_encoder_output(self, enc, on_device=False, B=None, dtype=np.float16):
        pass

    def _fill(self, prompts, no_speech_out):
        self.calls.append(no_speech_out is not None)
        if no_speech_out is not None:
            assert no_speech_out.dtype == np.float32 and no_speech_out.shape == (len(prompts),)
            no_speech_out[:] = [tag(p) for p in prompts]

    def generate(self, mel, prompts, *args, B=None, no_speech_out=None, **kw):
        self._fill(prompts, no_speech_out)
        return [[7]] * len(prompts), [0.5] * len(prompts)

    def generate_sample(self, mel, prompts, n, *args, B=None, no_speech_out=None, **kw):
        self._fill(prompts, no_speech_out)
        return [[[7]] * n] * len(prompts), [[0.5] * n] * len(prompts)

    def encode(self, mel, out=None, on_device=False):
        return out


@pytest.fixture
def fake_buffers(monkeypatch):
    """_lib's device buffers as host arrays"""
    nxt = [0x1000]

    def alloc(device, nbytes):
        nxt[0] += 1 << 20
        return nxt[0]

    monkeypatch.setattr(_lib, "buffer_alloc", alloc)
    monkeypatch.setattr(_lib, "buffer_free", lambda addr: None)


def feats(n):
    return np.zeros((n, 80, 3000), np.float32)


SAMPLE = dict(beam_size=1, num_hypotheses=3, sampling_topk=0, sampling_temperature=0.5)


@pytest.mark.parametrize("replicas", [1, 2])
@pytest.mark.parametrize("sampling", [False, True])
def test_each_result_carries_its_windows_value(fake_buffers, replicas, sampling):
    hs = [FakeHandle() for _ in range(replicas)]
    m = models.Whisper(None, device="cuda", device_index=list(range(replicas)), _handles=hs)
    n = 5
    prompts = [prompt(w) for w in range(n)]
    kw = SAMPLE if sampling else {}
    sources = [StorageView.from_array(feats(n)), np.zeros((n, 1500, D), np.float16), m.encode(feats(n))]
    for src in sources:
        res = m.generate(src, prompts, return_no_speech_prob=True, **kw)
        assert [r.no_speech_prob for r in res] == [tag(p) for p in prompts]
        assert all(len(r.sequences_ids) == (3 if sampling else 1) for r in res)
        res = m.generate(src, prompts, **kw)
        assert [r.no_speech_prob for r in res] == [0.0] * n
    # features and host encoder outputs are split over both replicas; the handles saw the request only when asked
    assert all(h.calls for h in hs)
    assert sum(h.calls.count(True) for h in hs) == sum(h.calls.count(False) for h in hs)


def test_prompt_without_sot_refused_only_when_asked():
    h = FakeHandle()
    m = models.Whisper(None, device="cuda", _handles=[h])
    bad = [[50361, 400, 500, 600], prompt(1)]
    with pytest.raises(ValueError, match="startoftranscript"):
        m.generate(StorageView.from_array(feats(2)), bad, return_no_speech_prob=True)
    assert h.calls == []
    assert [r.no_speech_prob for r in m.generate(StorageView.from_array(feats(2)), bad)] == [0.0, 0.0]
    # a <|startoftranscript|> anywhere in the prompt will do (faster-whisper's previous-text prompts)
    ok = [[50361, 400, SOT, 50259], prompt(1)]
    assert m.generate(StorageView.from_array(feats(2)), ok, return_no_speech_prob=True)[1].no_speech_prob == tag(prompt(1))


class Recorder:
    """lib() that records the calls a Handle makes (the options initialiser is the library's own)"""

    def __init__(self, real):
        self.real, self.calls = real, []

    def wisb_generate_options_init(self, opt):
        return self.real.wisb_generate_options_init(opt)

    def wisb_set_option(self, h, key, value):
        self.calls.append(("set_option", key, value))
        return 0

    def wisb_generate(self, h, mel, B, prompts, prompt_len, opt, ids, stride, lens, scores):
        self.calls.append(("generate", B))
        return 0

    def wisb_get_no_speech_probs(self, h, B, out):
        self.calls.append(("get", B))
        np.ctypeslib.as_array((ctypes.c_float * B).from_address(out.value))[:] = 0.25
        return 0


@pytest.fixture
def recorder(monkeypatch):
    rec = Recorder(_lib.lib())
    monkeypatch.setattr(_lib, "lib", lambda: rec)
    return rec


def test_handle_calls_into_the_library(recorder):
    h = _lib.Handle(None)
    P2 = [prompt(0), prompt(1)]
    h.generate(None, P2, 5, B=2)
    h.generate_sample(None, P2, 2, 0, 1.0, np.asarray([1, 2], np.uint64), B=2)
    assert recorder.calls == [("generate", 2)] * 2
    recorder.calls.clear()
    for sample in (False, True):
        ns = np.zeros(2, np.float32)
        if sample:
            h.generate_sample(None, P2, 2, 0, 1.0, np.asarray([1, 2], np.uint64), B=2, no_speech_out=ns)
        else:
            h.generate(None, P2, 5, B=2, no_speech_out=ns)
        assert recorder.calls == [("set_option", b"no_speech_prob", 1), ("generate", 2), ("get", 2),
                                  ("set_option", b"no_speech_prob", 0)]
        assert ns.tolist() == [0.25, 0.25]
        recorder.calls.clear()
    for bad in (np.zeros(3, np.float32), np.zeros(2, np.float64), [0.0, 0.0], np.zeros(4, np.float32)[::2]):
        with pytest.raises(ValueError, match="no_speech_out"):
            h.generate(None, P2, 5, B=2, no_speech_out=bad)
    assert recorder.calls == []


def test_failed_generate_still_turns_the_option_off(recorder, monkeypatch):
    monkeypatch.setattr(recorder, "wisb_generate", lambda *a: recorder.calls.append(("generate",)) or 1)
    monkeypatch.setattr(recorder, "wisb_last_error", lambda: b"bad prompt", raising=False)
    h = _lib.Handle(None)
    with pytest.raises(ValueError, match="bad prompt"):
        h.generate(None, [prompt(0)], 5, B=1, no_speech_out=np.zeros(1, np.float32))
    assert recorder.calls == [("set_option", b"no_speech_prob", 1), ("generate",), ("set_option", b"no_speech_prob", 0)]


def test_one_lock_around_every_generate(recorder):
    """while a call that asks holds the handle, another call on it waits (option on ... off is never interleaved)"""
    h = _lib.Handle(None)
    entered, release = threading.Event(), threading.Event()
    real_get = recorder.wisb_get_no_speech_probs

    def slow_get(*a):
        entered.set()
        release.wait(5)
        return real_get(*a)

    recorder.wisb_get_no_speech_probs = slow_get
    t = threading.Thread(target=h.generate, args=(None, [prompt(0)], 5), kwargs=dict(B=1, no_speech_out=np.zeros(1, np.float32)))
    t.start()
    assert entered.wait(5)
    other = threading.Thread(target=h.generate, args=(None, [prompt(0)], 5), kwargs=dict(B=1))
    other.start()
    other.join(0.2)
    assert other.is_alive()
    release.set()
    t.join(5)
    other.join(5)
    assert recorder.calls == [("set_option", b"no_speech_prob", 1), ("generate", 1), ("get", 1),
                              ("set_option", b"no_speech_prob", 0), ("generate", 1)]


class FakeModel:
    """an engine that takes options per window; records its calls"""
    per_window_options = True
    n_mels = 80
    dims = {"no_timestamps": 50363}

    def __init__(self):
        self.calls = []

    def generate(self, features, prompts, **opts):
        self.calls.append(opts.get("return_no_speech_prob", False))
        asked = opts.get("return_no_speech_prob", False)
        return [WhisperGenerationResult([[7]], [], tag(p) if asked else 0.0) for p in prompts]


def test_batcher_merges_requests_that_differ_only_in_the_request():
    model = FakeModel()
    with TranscribeBatcher(model, max_batch=3, max_wait_ms=2000) as b:
        f1 = b.submit(feats(1), prompt(0), beam_size=5, return_no_speech_prob=True)
        f2 = b.submit(feats(2), prompt(1), beam_size=5)
        r1, r2 = f1.result(10), f2.result(10)
    assert model.calls == [True] and b.stats["engine_calls"] == 1
    assert [r.no_speech_prob for r in r1] == [tag(prompt(0))]
    assert [r.no_speech_prob for r in r2] == [0.0, 0.0]
    model = FakeModel()
    with TranscribeBatcher(model, max_batch=2, max_wait_ms=2000) as b:
        r = [b.submit(feats(1), prompt(w), beam_size=5) for w in range(2)]
        assert [x.result(10)[0].no_speech_prob for x in r] == [0.0, 0.0]
    assert model.calls == [False]
