"""Cross-request dynamic batcher in front of ``models.Whisper`` (SURVEY.md section 8(f) row 2).

The reference serialises requests: ``do_whisper`` is called synchronously on the asyncio event-loop thread of a
single-worker gunicorn (main.py:1174-1215, 1243-1348; entrypoint.sh:19-21), two windows per engine call
(``concurrent_gpu_chunks``, main.py:91-94, 676-693).  The engine decodes every window of a call in ONE shared
decoder pass per generated token (rows = windows x beams up to the engine's row capacity, 320 by default = 64 windows at
beam 5; csrc/decoder_batch.cu): the 1.6 GB of decoder weights stream once per pass whatever the number of rows, finished
windows leave the pass, and requests with different ``max_length`` ride the same pass (per-window limits).  So
concurrent ``/api/asr`` and ``/api/willow`` requests should be coalesced (bench.py ``configs2`` measures 64 mixed-length
large-v2 windows at beam 5 in one call against one after the other).
This module is the piece a WIS maintainer puts between the endpoints and the engine:

    batcher = TranscribeBatcher(whisper_model, max_batch=64, max_wait_ms=2)
    results = await batcher.generate(features, prompt, beam_size=5)      # inside the FastAPI handlers
    results = batcher.submit(features, prompt, beam_size=5).result()      # from plain threads

Requests are compatible when they share the prompt and every generation option except ``max_length`` (same decoder
configuration; the length limits travel per window); a batch is closed when ``max_batch`` windows are collected or
``max_wait_ms`` after its oldest request arrived, whichever is first.  Latency note: every request of a batch is
answered when the whole batch has been decoded (the slowest window decides), so ``max_batch`` trades throughput against
the latency of short requests; ``max_batch`` above the engine's row capacity / beam only adds queueing.
The engine call runs on the batcher's own thread, so the event loop is never blocked (the C ABI releases the GIL).
"""
from __future__ import annotations

import asyncio
import collections
import threading
import time
from concurrent.futures import Future

import numpy as np

from .models import StorageView


class _Request:
    __slots__ = ("features", "n", "key", "prompt", "opts", "max_length", "future", "t_arrival")

    def __init__(self, features, prompt, opts):
        self.features = features
        self.n = int(features.shape[0])
        self.prompt = list(prompt)
        self.opts = dict(opts)
        self.max_length = int(self.opts.pop("max_length", 448))  # per request; merged per window by the worker
        self.key = (tuple(self.prompt), tuple(sorted((k, _freeze(v)) for k, v in self.opts.items())))
        self.future = Future()
        self.t_arrival = time.monotonic()


def _freeze(v):
    return tuple(v) if isinstance(v, (list, tuple)) else v


class TranscribeBatcher:
    def __init__(self, model, max_batch: int = 64, max_wait_ms: float = 2.0, max_queue_windows: int = 4096):
        if max_batch < 1:
            raise ValueError("max_batch must be >= 1")
        self._model = model
        self.max_batch = int(max_batch)
        self.max_wait = float(max_wait_ms) / 1e3
        self.max_queue_windows = int(max_queue_windows)
        self._queues = collections.OrderedDict()  # key -> deque of requests (FIFO per decoder configuration)
        self._queued_windows = 0
        self._cv = threading.Condition()
        self._closed = False
        self.stats = {"requests": 0, "windows": 0, "engine_calls": 0, "max_windows_per_call": 0}
        self._thread = threading.Thread(target=self._loop, name="wisb-batcher", daemon=True)
        self._thread.start()

    # ------------------------------------------------------------------------------------------------ producers
    def submit(self, features, prompt, **generate_options) -> Future:
        """features: float32 [n, 80, 3000] (or a StorageView); prompt: the n windows' common prompt ids.
        Returns a Future of the list of n results ``Whisper.generate`` would have returned for this request alone."""
        arr = features.array if isinstance(features, StorageView) else np.asarray(features)
        if arr.ndim != 3 or arr.dtype != np.float32:
            raise ValueError("features must be float32 [n, 80, 3000]")
        if prompt and isinstance(prompt[0], (list, tuple)):
            if any(list(p) != list(prompt[0]) for p in prompt) or len(prompt) != arr.shape[0]:
                raise ValueError("one request carries one prompt for all of its windows (as main.py:689 builds it)")
            prompt = prompt[0]
        req = _Request(np.ascontiguousarray(arr), prompt, generate_options)
        with self._cv:
            if self._closed:
                raise RuntimeError("batcher is closed")
            if self._queued_windows + req.n > self.max_queue_windows:
                raise RuntimeError("transcription queue is full")
            self._queues.setdefault(req.key, collections.deque()).append(req)
            self._queued_windows += req.n
            self.stats["requests"] += 1
            self._cv.notify()
        return req.future

    async def generate(self, features, prompt, **generate_options):
        """asyncio face of ``submit`` for the FastAPI handlers (main.py:1174, 1243)."""
        return await asyncio.wrap_future(self.submit(features, prompt, **generate_options))

    def close(self, timeout: float | None = None):
        """Stop accepting work, finish what is queued, join the worker."""
        with self._cv:
            self._closed = True
            self._cv.notify()
        self._thread.join(timeout)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # ------------------------------------------------------------------------------------------------ the worker
    def _oldest_key(self):
        best, t = None, None
        for k, q in self._queues.items():
            if q and (t is None or q[0].t_arrival < t):
                best, t = k, q[0].t_arrival
        return best

    def _take_batch(self):
        """Called with the lock held.  Blocks until a batch is due; returns its requests ([] once closed and drained)."""
        while True:
            key = self._oldest_key()
            if key is None:
                if self._closed:
                    return []
                self._cv.wait()
                continue
            q = self._queues[key]
            have = sum(r.n for r in q)
            deadline = q[0].t_arrival + self.max_wait
            now = time.monotonic()
            if have < self.max_batch and now < deadline and not self._closed:
                self._cv.wait(deadline - now)  # more compatible requests may still arrive
                continue
            batch, total = [], 0
            while q and (not batch or total + q[0].n <= self.max_batch):
                r = q.popleft()
                batch.append(r)
                total += r.n
            if not q:
                del self._queues[key]
            self._queued_windows -= total
            return batch

    def _loop(self):
        while True:
            with self._cv:
                batch = self._take_batch()
            if not batch:
                return
            live = [r for r in batch if r.future.set_running_or_notify_cancel()]
            if not live:
                continue
            n = sum(r.n for r in live)
            try:
                feats = live[0].features if len(live) == 1 else np.concatenate([r.features for r in live], axis=0)
                limits = [r.max_length for r in live for _ in range(r.n)]
                ml = limits[0] if len(set(limits)) == 1 else np.asarray(limits, np.int32)
                out = self._model.generate(StorageView.from_array(feats), [live[0].prompt] * n, max_length=ml, **live[0].opts)
                if len(out) != n:
                    raise RuntimeError(f"engine returned {len(out)} results for {n} windows")
            except BaseException as e:  # noqa: BLE001 -- every waiter must learn about it
                for r in live:
                    r.future.set_exception(e)
                continue
            self.stats["engine_calls"] += 1
            self.stats["windows"] += n
            self.stats["max_windows_per_call"] = max(self.stats["max_windows_per_call"], n)
            pos = 0
            for r in live:
                r.future.set_result(out[pos : pos + r.n])
                pos += r.n
