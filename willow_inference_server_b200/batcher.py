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

Requests are compatible when they share the prompt and every generation option except ``max_length`` and
``return_no_speech_prob`` (same decoder configuration; the length limits travel per window, and asking for the
no-speech probability changes no result).  With an engine that takes the search options per window
(``models.Whisper.per_window_options``) the rule is wider: prompts need only the same length and the same timestamp mode
(whether ``<|notimestamps|>`` is in them), and ``beam_size``, ``patience`` and ``length_penalty`` travel per window too,
so short commands at beam 1, dictation at beam 3 and requests in other languages or for translation share one call.
Every other option (``max_initial_timestamp_index``, ``suppress_tokens``, the history processors) must still match.
Sampling requests (``beam_size=1``, ``sampling_topk != 1``) share a call only with sampling requests of the same
``num_hypotheses``, ``sampling_topk``, ``sampling_temperature`` and search options, never with beam requests.  Each
gets its seed at ``submit`` (its own ``random_seed``, or a draw from the stream ``set_random_seed`` resets) and the
call takes one seed per window, so a merged request returns exactly what it returns alone with that seed.
Those three options are checked at ``submit`` (``ValueError`` there), and a call that the engine refuses as invalid
(``ValueError``) is retried request by request, so one client's bad request never fails the requests it was merged with.
Every window of such a call keeps as many decoder rows as the call's largest beam, so a batch keeps its padded rows at
most its real ones (windows x largest beam <= 2 x the sum of the beams), leaving the newest requests whose beams are
farthest from the oldest request's for the next batch: on an H100 (700 W power limit), 63 greedy windows and one at
beam 8 in one call (512 rows for 71 real ones) took 1.45x the time of two calls, while WIS's mix of beam 1 and beam 3
windows (168 rows for 88) took 0.94x (DESIGN.md section 6).  A batch is closed when ``max_batch`` windows are collected
or ``max_wait_ms`` after its oldest request arrived, whichever is first.  Latency note: every request of a batch is
answered when the whole batch has been decoded (the slowest window decides), so ``max_batch`` trades throughput against
the latency of short requests; ``max_batch`` above the engine's row capacity / beam only adds queueing.
The engine call runs on the batcher's own thread, so the event loop is never blocked (the C ABI releases the GIL).
"""
from __future__ import annotations

import asyncio
import collections
import dataclasses
import threading
import time
from concurrent.futures import Future

import numpy as np

from .models import StorageView, check_sampling_options, draw_seed, window_seeds


# search options an engine with per_window_options takes per window, with the defaults of CTranslate2's generate (which
# stand in for a request that does not set one when it shares a call with one that does)
PER_WINDOW_DEFAULTS = {"beam_size": 5, "patience": 1.0, "length_penalty": 1.0}


def _check_search_option(name, v):
    """A per-window search option as models.Whisper.generate accepts it: beam_size an int in [1, 8], patience a finite
    number > 0, length_penalty a finite number; anything else raises ValueError."""
    if name == "beam_size":
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or not 1 <= v <= 8:
            raise ValueError(f"beam_size must be an int in [1, 8], got {v!r}")
        return int(v)
    number = isinstance(v, (int, float, np.integer, np.floating)) and not isinstance(v, (bool, np.bool_))
    if not number or not np.isfinite(v) or (name == "patience" and v <= 0):
        raise ValueError(f"{name} must be a finite number{' > 0' if name == 'patience' else ''}, got {v!r}")
    return float(v)


class _Request:
    __slots__ = ("features", "n", "key", "prompt", "opts", "search", "max_length", "no_speech", "seed", "future",
                 "t_arrival")

    def __init__(self, features, prompt, opts, no_timestamps=None):
        """no_timestamps: the engine's <|notimestamps|> id when it takes prompts and search options per window, else
        None (then the prompt and every option but max_length are part of the key)"""
        self.features = features
        self.n = int(features.shape[0])
        self.prompt = list(prompt)
        self.opts = dict(opts)
        self.max_length = int(self.opts.pop("max_length", 448))  # per request; merged per window by the worker
        # a merged call asks for the no-speech probability when one of its requests does; the others get 0.0, what
        # CTranslate2 returns when it is not asked for
        self.no_speech = bool(self.opts.pop("return_no_speech_prob", False))
        self.search = {}
        prompt_key = tuple(self.prompt)
        # sampling: the request's seed, fixed now (its windows get seed + w); its search options stay in the key
        self.seed = None
        random_seed = self.opts.pop("random_seed", None)
        sampling = any(k in self.opts for k in ("num_hypotheses", "sampling_topk")) and check_sampling_options(
            self.opts.get("num_hypotheses", 1), self.opts.get("sampling_topk", 1), self.opts.get("sampling_temperature", 1),
            self.opts.get("beam_size", PER_WINDOW_DEFAULTS["beam_size"]), self.opts.get("patience", 1.0),
            self.opts.get("length_penalty", 1.0))
        if sampling:
            if random_seed is not None and (isinstance(random_seed, (bool, np.bool_)) or
                                            not isinstance(random_seed, (int, np.integer))):
                raise ValueError(f"random_seed of a request must be None or an int, got {random_seed!r}")
            self.seed = draw_seed() if random_seed is None else int(random_seed) % (1 << 64)
        if no_timestamps is not None:
            if not sampling:
                self.search = {k: _check_search_option(k, self.opts.pop(k)) for k in PER_WINDOW_DEFAULTS if k in self.opts}
            prompt_key = (len(self.prompt), no_timestamps in self.prompt)
        self.key = (prompt_key, tuple(sorted((k, _freeze(v)) for k, v in self.opts.items())))
        self.future = Future()
        self.t_arrival = time.monotonic()


def _freeze(v):
    return tuple(v) if isinstance(v, (list, tuple)) else v


class TranscribeBatcher:
    def __init__(self, model, max_batch: int = 64, max_wait_ms: float = 2.0, max_queue_windows: int = 4096):
        if max_batch < 1:
            raise ValueError("max_batch must be >= 1")
        self._model = model
        # features are checked at submit against the model's bin count (CTranslate2's Whisper.n_mels); an engine
        # without that property takes the 80-bin features of every Whisper model before large-v3
        self._n_mels = int(getattr(model, "n_mels", 80))
        # an engine that takes the prompt and the search options per window lets requests that differ in them share a
        # call; any other (CTranslate2's Whisper among them) gets calls with one prompt and one set of options
        self._no_ts = int(model.dims["no_timestamps"]) if getattr(model, "per_window_options", False) else None
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
        """features: float32 [n, n_mels, 3000] (or a StorageView), n_mels the model's (80, or 128 for the large-v3
        family); prompt: the n windows' common prompt ids.
        Returns a Future of the list of n results ``Whisper.generate`` would have returned for this request alone."""
        arr = features.array if isinstance(features, StorageView) else np.asarray(features)
        if arr.ndim != 3 or arr.dtype != np.float32 or tuple(arr.shape[1:]) != (self._n_mels, 3000):
            raise ValueError(f"features must be float32 [n, {self._n_mels}, 3000] for this model, got {arr.dtype} "
                             f"{tuple(arr.shape)}")
        if prompt and isinstance(prompt[0], (list, tuple)):
            if any(list(p) != list(prompt[0]) for p in prompt) or len(prompt) != arr.shape[0]:
                raise ValueError("one request carries one prompt for all of its windows (as main.py:689 builds it)")
            prompt = prompt[0]
        req = _Request(np.ascontiguousarray(arr), prompt, generate_options, self._no_ts)
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
            rest = []
            while not self._padding_ok(batch):
                # the newest of the requests whose beam is farthest from the oldest one's waits for the next batch
                b0 = self._beam(batch[0])
                far = max(range(1, len(batch)), key=lambda i: (abs(self._beam(batch[i]) - b0), i))
                rest.append(batch.pop(far))
                total -= rest[-1].n
            q.extendleft(sorted(rest, key=lambda r: r.t_arrival, reverse=True))
            if not q:
                del self._queues[key]
            self._queued_windows -= total
            return batch

    @staticmethod
    def _beam(r) -> int:
        return int(r.search.get("beam_size", PER_WINDOW_DEFAULTS["beam_size"]))

    def _padding_ok(self, reqs) -> bool:
        """padded rows <= real rows when these requests share a call (always true without per-window options)"""
        if self._no_ts is None:
            return True
        beams = [self._beam(r) for r in reqs]
        windows = sum(r.n for r in reqs)
        real = sum(r.n * b for r, b in zip(reqs, beams))
        return windows * max(beams) <= 2 * real

    def _loop(self):
        while True:
            with self._cv:
                batch = self._take_batch()
            if not batch:
                return
            live = [r for r in batch if r.future.set_running_or_notify_cancel()]
            if not live:
                continue
            try:
                self._answer(live)
            except ValueError as e:
                if len(live) == 1:
                    live[0].future.set_exception(e)
                    continue
                # the engine refused an argument of one of the requests (a prompt token, a length limit, ...): each
                # request alone, so that only the one it belongs to fails
                for r in live:
                    try:
                        self._answer([r])
                    except BaseException as e1:  # noqa: BLE001 -- the waiter must learn about it
                        r.future.set_exception(e1)
            except BaseException as e:  # noqa: BLE001 -- every waiter must learn about it
                for r in live:
                    r.future.set_exception(e)

    def _answer(self, live):
        """ONE engine call for the windows of these requests; sets their results (raises, setting none, on failure)."""
        n = sum(r.n for r in live)
        feats = live[0].features if len(live) == 1 else np.concatenate([r.features for r in live], axis=0)
        limits = [r.max_length for r in live for _ in range(r.n)]
        ml = limits[0] if len(set(limits)) == 1 else np.asarray(limits, np.int32)
        opts = dict(live[0].opts)
        for k, default in PER_WINDOW_DEFAULTS.items():  # (equal values stay a scalar: the CTranslate2 meaning)
            if any(k in r.search for r in live):
                vals = [r.search.get(k, default) for r in live for _ in range(r.n)]
                same = all(v == vals[0] for v in vals)
                opts[k] = vals[0] if same else np.asarray(vals, np.int32 if k == "beam_size" else np.float32)
        prompts = [r.prompt for r in live for _ in range(r.n)]
        if live[0].seed is not None:  # (a sampling batch: every request has its seed)
            opts["random_seed"] = np.concatenate([window_seeds(r.seed, r.n) for r in live])
        asked = any(r.no_speech for r in live)
        if asked:
            opts["return_no_speech_prob"] = True
        out = self._model.generate(StorageView.from_array(feats), prompts, max_length=ml, **opts)
        if len(out) != n:
            raise RuntimeError(f"engine returned {len(out)} results for {n} windows")
        self.stats["engine_calls"] += 1
        self.stats["windows"] += n
        self.stats["max_windows_per_call"] = max(self.stats["max_windows_per_call"], n)
        pos = 0
        for r in live:
            res = out[pos : pos + r.n]
            if asked and not r.no_speech:
                res = [dataclasses.replace(x, no_speech_prob=0.0) for x in res]
            r.future.set_result(res)
            pos += r.n
