"""Cross-request batcher (SURVEY 8f row 2): host logic only -- a fake engine stands in for models.Whisper."""
import asyncio
import threading
import time

import numpy as np
import pytest

from willow_inference_server_b200.batcher import TranscribeBatcher
from willow_inference_server_b200.models import WhisperGenerationResult

PROMPT = [50258, 50259, 50359, 50363]


class FakeEngine:
    """generate() answers with ids derived from each window's content, so mix-ups between requests are visible."""

    def __init__(self, delay=0.02, fail_on=None):
        self.calls = []
        self.delay = delay
        self.fail_on = fail_on
        self.lock = threading.Lock()

    def generate(self, features, prompts, **opts):
        arr = features.array
        with self.lock:
            self.calls.append((arr.shape[0], tuple(prompts[0]), dict(opts)))
        assert all(list(p) == list(prompts[0]) for p in prompts) and len(prompts) == arr.shape[0]
        time.sleep(self.delay)
        if self.fail_on is not None and any(int(w[0, 0]) == self.fail_on for w in arr):
            raise RuntimeError("engine failure")
        return [WhisperGenerationResult([[int(w[0, 0]), int(w[0, 1]), opts.get("beam_size", 5)]]) for w in arr]


def _window(tag, n=1):
    a = np.zeros((n, 80, 3000), np.float32)
    a[:, 0, 0] = tag
    a[:, 0, 1] = np.arange(n)
    return a


def test_concurrent_requests_share_engine_calls_and_keep_their_results():
    eng = FakeEngine(delay=0.05)
    with TranscribeBatcher(eng, max_batch=16, max_wait_ms=20) as b:
        futs = {}
        threads = []

        def client(tag, n):
            futs[tag] = b.submit(_window(tag, n), PROMPT, beam_size=5)

        for tag, n in [(1, 1), (2, 3), (3, 1), (4, 2), (5, 1), (6, 1)]:
            t = threading.Thread(target=client, args=(tag, n))
            t.start()
            threads.append(t)
        for t in threads:
            t.join()
        for tag, n in [(1, 1), (2, 3), (3, 1), (4, 2), (5, 1), (6, 1)]:
            res = futs[tag].result(timeout=5)
            assert [r.sequences_ids[0][:2] for r in res] == [[tag, i] for i in range(n)]
    assert sum(c[0] for c in eng.calls) == 9
    assert len(eng.calls) < 6, eng.calls            # coalesced
    assert b.stats["requests"] == 6 and b.stats["windows"] == 9 and b.stats["max_windows_per_call"] >= 2


def test_incompatible_requests_are_never_mixed_and_batches_respect_max_batch():
    eng = FakeEngine(delay=0.01)
    other = [50258, 50260, 50358, 50363]  # another language + translate
    with TranscribeBatcher(eng, max_batch=4, max_wait_ms=30) as b:
        fs = [b.submit(_window(i), PROMPT if i % 2 == 0 else other, beam_size=5 if i < 6 else 1) for i in range(10)]
        big = b.submit(_window(99, 7), PROMPT, beam_size=5)  # larger than max_batch: goes alone, not split
        for i, f in enumerate(fs):
            r = f.result(timeout=5)
            assert r[0].sequences_ids[0] == [i, 0, 5 if i < 6 else 1]
        assert [r.sequences_ids[0][1] for r in big.result(timeout=5)] == list(range(7))
    for n, prompt, opts in eng.calls:
        assert n <= 4 or n == 7
    # every call was homogeneous (checked inside FakeEngine.generate) and the three configurations all appeared
    assert {(c[1], c[2]["beam_size"]) for c in eng.calls} >= {(tuple(PROMPT), 5), (tuple(other), 5), (tuple(PROMPT), 1)}


def test_wait_budget_bounds_latency_of_a_lonely_request():
    eng = FakeEngine(delay=0.0)
    with TranscribeBatcher(eng, max_batch=64, max_wait_ms=30) as b:
        t0 = time.monotonic()
        b.submit(_window(1), PROMPT).result(timeout=5)
        dt = time.monotonic() - t0
    assert 0.02 <= dt < 1.0, dt  # waited for company about max_wait, not forever


def test_engine_errors_reach_every_waiter_of_the_batch_only():
    eng = FakeEngine(delay=0.02, fail_on=13)
    with TranscribeBatcher(eng, max_batch=8, max_wait_ms=30) as b:
        bad = [b.submit(_window(13), PROMPT), b.submit(_window(14), PROMPT)]
        for f in bad:
            with pytest.raises(RuntimeError, match="engine failure"):
                f.result(timeout=5)
        ok = b.submit(_window(15), PROMPT)  # the batcher keeps serving
        assert ok.result(timeout=5)[0].sequences_ids[0][0] == 15
    with pytest.raises(RuntimeError):
        b.submit(_window(1), PROMPT)  # closed
    with pytest.raises(ValueError):
        TranscribeBatcher(eng, max_batch=0)


def test_asyncio_face_and_queue_limit():
    eng = FakeEngine(delay=0.02)

    async def main():
        with TranscribeBatcher(eng, max_batch=32, max_wait_ms=20, max_queue_windows=40) as b:
            outs = await asyncio.gather(*[b.generate(_window(i, 2), [PROMPT, PROMPT], beam_size=3) for i in range(8)])
            assert [[r.sequences_ids[0][0] for r in o] for o in outs] == [[i, i] for i in range(8)]
            with pytest.raises(ValueError):
                b.submit(np.zeros((1, 80, 3000), np.float64), PROMPT)
            with pytest.raises(ValueError):
                b.submit(_window(1, 2), [PROMPT, PROMPT[::-1]])
            with pytest.raises(RuntimeError, match="full"):
                b.submit(_window(1, 41), PROMPT)

    asyncio.run(main())
    assert len(eng.calls) < 8


def test_requests_with_different_max_length_share_one_call():
    # the engine takes one length limit per window (wisb_generate_options.max_length_per_window), so max_length is not
    # part of the compatibility key
    eng = FakeEngine(delay=0.05)
    with TranscribeBatcher(eng, max_batch=16, max_wait_ms=30) as b:
        f1 = b.submit(_window(1, 2), PROMPT, beam_size=5, max_length=30)
        f2 = b.submit(_window(2, 1), PROMPT, beam_size=5, max_length=72)
        f3 = b.submit(_window(3, 1), PROMPT, beam_size=5)
        r1, r2, r3 = f1.result(timeout=5), f2.result(timeout=5), f3.result(timeout=5)
    assert [r.sequences_ids[0][0] for r in r1 + r2 + r3] == [1, 1, 2, 3]
    assert len(eng.calls) == 1 and eng.calls[0][0] == 4
    assert list(eng.calls[0][2]["max_length"]) == [30, 30, 72, 448]
    # equal limits stay a plain int (the CTranslate2 meaning)
    eng2 = FakeEngine()
    with TranscribeBatcher(eng2, max_batch=4, max_wait_ms=10) as b:
        b.submit(_window(1), PROMPT, beam_size=5, max_length=40).result(timeout=5)
    assert eng2.calls[0][2]["max_length"] == 40
