"""Drop-in for the part of ``ctranslate2`` that WIS calls (main.py:39, 341-355, 454, 535-537, 638-640, 685-692).

    import willow_inference_server_b200 as ctranslate2
    model = ctranslate2.models.Whisper(path, device="cuda", compute_type=..., inter_threads=..., device_index=[0..N-1])
    feats = ctranslate2.StorageView.from_array(mel)            # float32 [n, 80, 3000]
    results = model.generate(feats, [prompt] * n, beam_size=5, return_scores=False)
    results[i].sequences_ids[0]                                # list[int]
    model.detect_language(feats)[0][0]                         # ("<|en|>", prob)
    enc = model.encode(feats)                                  # float16 [n, 1500, d_model], on the GPU (faster-whisper)
    model.generate(enc, [prompt] * n)                          # generate / detect_language / align take it for features

Same names, argument meaning and error behaviour (ValueError for bad shapes/arguments, RuntimeError for device
failures).  What differs by design: ``device`` must be "cuda" (no CPU fallback), ``compute_type`` is accepted and
ignored (one fp16-weights / fp32-accumulate path, no multi-backend dispatch), ``model_path`` points at a WISB200 weight
blob (file, or directory containing ``model.wisb``).  ``device_index=[...]`` builds one replica per GPU; a batch is
split across the replicas (weights are read once and copied to every GPU at load; bench.py does the same step with an
NCCL broadcast when launched under torchrun).
"""
from __future__ import annotations

import os
import threading
import zlib
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field

import numpy as np

from . import _lib
from .languages import LANGUAGE_CODES


class StorageView:
    """ctranslate2.StorageView stand-in.  Host form: a borrowed view of a host float32 array (features, main.py:638,685)
    or of a float16 / float32 encoder output.  Device form (Whisper.encode with to_cpu=False): a float16 encoder output in
    one device buffer of its own on GPU ``device_index``, freed with the view, whether or not the model still exists."""

    def __init__(self, array: np.ndarray):
        self.array = array
        self._buf = None         # device form: address of its wisb_buffer_alloc buffer (float16, C order)
        self._device_index = 0
        self._shape = None

    @classmethod
    def from_array(cls, array):
        a = np.asarray(array)
        if a.dtype not in (np.float32, np.float16):
            raise ValueError(f"StorageView.from_array: unsupported dtype {a.dtype} (float32 or float16 expected)")
        if not a.flags["C_CONTIGUOUS"]:
            raise ValueError("StorageView.from_array: the array must be C-contiguous")
        return cls(a)

    @classmethod
    def _empty_on_device(cls, device_index: int, shape):
        """an uninitialised float16 device view of `shape` on GPU `device_index`"""
        sv = cls(None)
        sv._buf = _lib.buffer_alloc(device_index, 2 * int(np.prod(shape)))
        sv._device_index = int(device_index)
        sv._shape = [int(v) for v in shape]
        return sv

    @property
    def shape(self):
        return list(self._shape) if self._buf is not None else list(self.array.shape)

    @property
    def device(self) -> str:
        return "cuda" if self._buf is not None else "cpu"

    @property
    def device_index(self) -> int:
        return self._device_index

    def to_device(self, device: str):
        """to_device("cpu"): a host StorageView of the same data and dtype (the view itself when it is one already)"""
        if device != "cpu":
            raise ValueError("StorageView.to_device: only 'cpu' is supported")
        if self._buf is None:
            return self
        return StorageView(_lib.buffer_to_host(self._buf, np.empty(self._shape, np.float16)))

    def __del__(self):
        if self._buf is not None:
            buf, self._buf = self._buf, None
            try:
                _lib.buffer_free(buf)
            except Exception:
                pass


@dataclass
class WhisperGenerationResult:
    sequences_ids: list
    scores: list = field(default_factory=list)
    no_speech_prob: float = 0.0

    @property
    def sequences(self):  # CT2 returns token strings here; WIS never reads them (main.py:707,713 use ids)
        return [[str(t) for t in seq] for seq in self.sequences_ids]


@dataclass
class WhisperAlignmentResult:
    alignments: list  # list[tuple[int, int]]: (text token index, encoder frame) along the DTW path
    text_token_probs: list  # list[float]


# The stream the seeds of sampling calls without `random_seed` are drawn from (one 64-bit seed per call).
_seed_lock = threading.Lock()
_seed_stream = np.random.default_rng()


def set_random_seed(seed: int):
    """ctranslate2.set_random_seed: restart the stream that seeds sampling calls made without ``random_seed``, so
    that a sequence of such calls repeats."""
    global _seed_stream
    if isinstance(seed, (bool, np.bool_)) or not isinstance(seed, (int, np.integer)):
        raise ValueError(f"the random seed must be an int, got {seed!r}")
    with _seed_lock:
        _seed_stream = np.random.default_rng(int(seed) % (1 << 64))


def draw_seed() -> int:
    """the next 64-bit call seed of the stream set_random_seed resets"""
    with _seed_lock:
        return int(_seed_stream.integers(0, 1 << 64, dtype=np.uint64, endpoint=False))


def _is_int(v) -> bool:
    return isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_))


def check_sampling_options(num_hypotheses, sampling_topk, sampling_temperature, beam_size, patience,
                           length_penalty) -> bool:
    """CTranslate2's switch: beam_size 1 with sampling_topk != 1 samples.  Returns whether these options sample, after
    checking them (ValueError): sampling_topk 0 (the whole vocabulary) or in [2, 16], sampling_temperature finite and
    > 0, num_hypotheses in [1, 8], scalar beam_size (1), patience and length_penalty.  num_hypotheses > 1 without
    sampling is refused; with sampling_topk 1 the temperature is ignored (greedy or beam search)."""
    if not _is_int(sampling_topk):
        raise ValueError(f"sampling_topk must be an int, got {sampling_topk!r}")
    if not _is_int(num_hypotheses) or not 1 <= num_hypotheses <= 8:
        raise ValueError(f"num_hypotheses must be an int in [1, 8], got {num_hypotheses!r}")
    if sampling_topk == 1:
        if num_hypotheses != 1:
            raise ValueError("num_hypotheses > 1 needs sampling (beam_size=1 and sampling_topk != 1)")
        return False
    if not all(np.isscalar(v) for v in (beam_size, patience, length_penalty)):
        raise ValueError("a sampling call takes beam_size, patience and length_penalty as scalars")
    if beam_size != 1:
        raise ValueError("sampling (sampling_topk != 1) needs beam_size=1")
    if not (sampling_topk == 0 or 2 <= sampling_topk <= 16):
        raise ValueError(f"sampling_topk must be 0 (the whole vocabulary), 1 or in [2, 16], got {sampling_topk}")
    number = lambda v: isinstance(v, (int, float, np.integer, np.floating)) and not isinstance(v, (bool, np.bool_))  # noqa: E731
    if not number(sampling_temperature) or not np.isfinite(sampling_temperature) or sampling_temperature <= 0:
        raise ValueError(f"sampling_temperature must be a finite number > 0, got {sampling_temperature!r}")
    if not number(length_penalty) or not np.isfinite(length_penalty):
        raise ValueError(f"length_penalty must be a finite number, got {length_penalty!r}")
    return True


def check_timestamp_prompt(prompt, sot: int, no_timestamps: int) -> None:
    """Raise ValueError unless `prompt` may start a timestamp-mode search (wisb_generate's rule, restated).

    The timestamp rules read only the generated tokens, so everything before the prompt's last <|startoftranscript|>
    (faster-whisper's <|startofprev|> context of earlier windows' output, timestamps included) may be any id.  From that
    token on (the whole prompt when it has none) <|notimestamps|> and timestamp ids are refused."""
    p = [int(t) for t in prompt]
    start = max((i for i, t in enumerate(p) if t == sot), default=0)
    for t in p[start:]:
        if t == no_timestamps:
            raise ValueError("timestamp decoding: the prompt must not contain <|notimestamps|>")
        if t > no_timestamps:
            raise ValueError("timestamp decoding: the prompt must not contain timestamp tokens")


def window_seeds(random_seed, n: int) -> np.ndarray:
    """The seed of each of the n windows of a sampling call: random_seed None (one call seed s drawn from the stream
    set_random_seed resets), an int s, or one int per window.  For a call seed s window w gets s + w mod 2^64, so a
    window's result depends on its seed alone, not on how calls are batched."""
    if random_seed is None:
        random_seed = draw_seed()
    if _is_int(random_seed):
        return np.arange(n, dtype=np.uint64) + np.uint64(int(random_seed) % (1 << 64))  # (wraps mod 2^64)
    vals = list(random_seed) if isinstance(random_seed, (list, tuple, np.ndarray)) else None
    if vals is None or len(vals) != n or not all(_is_int(v) for v in vals):
        raise ValueError("random_seed must be None, an int or one int per feature window")
    return np.asarray([int(v) % (1 << 64) for v in vals], np.uint64)


def get_supported_compute_types(device: str, device_index: int = 0):
    """main.py:454 only logs this.  One compute path exists: fp16 weights/activations, fp32 accumulation."""
    if device != "cuda":
        raise ValueError("willow_inference_server_b200 supports device='cuda' only")
    return {"float16"}


def _features_array(features, n_mels: int) -> np.ndarray:
    a = features.array if isinstance(features, StorageView) else np.asarray(features)
    if a.dtype != np.float32 or a.ndim != 3 or tuple(a.shape[1:]) != (n_mels, 3000):
        raise ValueError(f"features must be float32 [n, {n_mels}, 3000] for this model, got {a.dtype} {tuple(a.shape)}")
    return np.ascontiguousarray(a)


@dataclass
class _Input:
    """what a generate / detect_language / align call decodes: features, a host encoder output, or a device one"""
    n: int
    mel: np.ndarray = None   # float32 [n, n_mels, 3000]
    enc: np.ndarray = None   # float16 / float32 [n, 1500, d_model] in host memory
    dev: StorageView = None  # device form of a float16 [n, 1500, d_model] encoder output


class Whisper:
    # generate takes one prompt per window and beam_size / patience / length_penalty / max_length as one value per window:
    # batcher.TranscribeBatcher puts requests that differ in those into one call
    per_window_options = True

    def __init__(self, model_path, device: str = "cuda", *, device_index=0, compute_type: str = "default",
                 inter_threads: int = 1, intra_threads: int = 0, max_queued_batches: int = 0, files=None,
                 reuse_encoder=None, _handles=None, **_ignored):
        if device != "cuda":
            raise ValueError("willow_inference_server_b200.models.Whisper runs on device='cuda' only (no CPU fallback)")
        idx = [device_index] if isinstance(device_index, int) else list(device_index)
        if not idx:
            raise ValueError("device_index must name at least one GPU")
        self.device = device
        self.device_index = idx
        self.compute_type = "float16"
        if _handles is not None:
            self._handles = list(_handles)
        else:
            path = str(model_path)
            if os.path.isdir(path) and os.path.isfile(os.path.join(path, "model.wisb")):
                path = os.path.join(path, "model.wisb")
            if os.path.isfile(path):
                blob = np.fromfile(path, np.uint8)  # read once, copied to every replica
            elif os.path.isdir(path) and any(os.path.exists(os.path.join(path, f)) for f in
                                             ("model.bin", "model.safetensors", "model.safetensors.index.json",
                                              "pytorch_model.bin")):
                # a CTranslate2 directory as main.py:342 passes it, or an HF checkpoint: converted in memory
                from . import loaders, weights as _W

                dims, tensors = loaders.load_any(path)
                blob = np.zeros(_W.blob_nbytes(tensors), np.uint8)
                _W.write_blob_into(blob, dims, tensors)
            else:
                raise RuntimeError(f"Unable to open model '{path}' (expected model.wisb, a CTranslate2 model.bin "
                                   "or a Hugging Face Whisper checkpoint)")
            self._handles = [_lib.Handle.from_host(blob, d) for d in idx]
        # detect_language -> generate -> (translate) on the same window encode once (SURVEY 8f row 4); opt-in because a
        # caller that replays identical features on purpose (a benchmark) must not have work skipped behind its back
        if reuse_encoder is None:
            reuse_encoder = os.environ.get("WISB_ENCODER_CACHE", "0") not in ("", "0")
        self.reuse_encoder = bool(reuse_encoder)
        for h in self._handles:
            h.set_option("encoder_cache", 1 if self.reuse_encoder else 0)
        self._dims = self._handles[0].dims()
        self._pool = ThreadPoolExecutor(max_workers=len(self._handles)) if len(self._handles) > 1 else None
        self._rr = 0
        self._lock = threading.Lock()
        # loading an encoder output and the call that decodes it must not interleave with another such pair
        self._replica_locks = [threading.Lock() for _ in self._handles]

    # ----------------------------------------------------------------------------------------------------------
    @property
    def is_multilingual(self) -> bool:
        return self._dims["n_vocab"] >= 51865

    @property
    def num_languages(self) -> int:
        return self._dims["n_langs"]

    @property
    def n_mels(self) -> int:
        """log-mel bins the model's features must have: 80, or 128 for the large-v3 family"""
        return self._dims.get("n_mels", 80)  # (a stand-in handle that reports no bin count serves 80-bin features)

    @property
    def dims(self) -> dict:
        return dict(self._dims)

    def _split(self, n: int, mel=None):
        k = len(self._handles)
        if k > 1 and self.reuse_encoder and n <= 2 and mel is not None:
            # same features -> same replica, so the cached encoder output is found again
            return [(zlib.crc32(np.ascontiguousarray(mel[0, :, :64]).tobytes()) % k, 0, n)]
        if k == 1 or n == 1:
            with self._lock:
                i = self._rr % k
                self._rr += 1
            return [(i, 0, n)]
        per = -(-n // k)
        return [(i, s, min(n, s + per)) for i, s in enumerate(range(0, n, per))]

    def _run(self, jobs):
        if self._pool is None or len(jobs) == 1:
            return [fn() for fn in jobs]
        return [f.result() for f in [self._pool.submit(fn) for fn in jobs]]

    def _input(self, features) -> _Input:
        """CTranslate2's rule: an input [n, 1500, d_model] is an encoder output from encode(), anything else must be the
        model's features [n, n_mels, 3000]"""
        if isinstance(features, StorageView) and features.device == "cuda":
            shape = features.shape
        else:
            a = features.array if isinstance(features, StorageView) else np.asarray(features)
            shape = list(a.shape)
        if len(shape) != 3 or shape[1] != 1500:
            mel = _features_array(features, self.n_mels)
            return _Input(mel.shape[0], mel=mel)
        d = self._dims["d_model"]
        if isinstance(features, StorageView) and features.device == "cuda":
            if shape[2] != d:
                raise ValueError(f"an encoder output must be [n, 1500, {d}] for this model, got {tuple(shape)}")
            if features.device_index not in self.device_index:
                raise ValueError(f"the encoder output is on GPU {features.device_index}, where this model has no replica")
            return _Input(shape[0], dev=features)
        if a.dtype not in (np.float16, np.float32) or shape[2] != d:
            raise ValueError(f"an encoder output must be float16 or float32 [n, 1500, {d}] for this model, got {a.dtype} "
                             f"{tuple(shape)}")
        return _Input(shape[0], enc=np.ascontiguousarray(a))

    def _dispatch(self, src: _Input, fn):
        """fn(handle, mel, s, e) for each part [s, e) of the windows, on the replicas _split picks (features and host
        encoder outputs) or on the replica on the GPU of a device encoder output.  For an encoder output, mel is None and
        the part is loaded into the handle just before (the call then decodes it, passing B = e - s)."""
        if src.dev is not None:
            parts = [(self.device_index.index(src.dev.device_index), 0, src.n)]
        else:
            parts = self._split(src.n, src.mel)

        def job(i, s, e):
            h = self._handles[i]
            if src.mel is not None:
                return lambda: fn(h, src.mel[s:e], s, e)

            def run():
                with self._replica_locks[i]:
                    if src.dev is not None:
                        h.load_encoder_output(src.dev._buf, on_device=True, B=src.n, dtype=np.float16)
                    else:
                        h.load_encoder_output(src.enc[s:e])
                    return fn(h, None, s, e)
            return run

        return self._run([job(*pt) for pt in parts])

    def encode(self, features, to_cpu: bool = False) -> StorageView:
        """ctranslate2.models.Whisper.encode: features -> the encoder output, float16 [n, 1500, d_model], for
        detect_language, generate and align.  On the GPU of the replica that encoded it (one replica, round robin, runs
        the whole call), or with to_cpu=True in host memory (the replicas then split the windows as in generate)."""
        mel = _features_array(features, self.n_mels)
        n, d = mel.shape[0], self._dims["d_model"]
        if to_cpu:
            out = np.empty((n, 1500, d), np.float16)
            self._run([(lambda i=i, s=s, e=e: self._handles[i].encode(mel[s:e], out[s:e])) for i, s, e in self._split(n)])
            return StorageView(out)
        with self._lock:
            i = self._rr % len(self._handles)
            self._rr += 1
        sv = StorageView._empty_on_device(self.device_index[i], (n, 1500, d))
        self._handles[i].encode(mel, sv._buf, on_device=True)
        return sv

    def generate(self, features, prompts, *, asynchronous: bool = False, beam_size: int = 5, patience: float = 1,
                 num_hypotheses: int = 1, length_penalty: float = 1, repetition_penalty: float = 1,
                 no_repeat_ngram_size: int = 0, max_length: int = 448, return_scores: bool = False,
                 return_no_speech_prob: bool = False, max_initial_timestamp_index: int = 50,
                 suppress_blank: bool = True, suppress_tokens=(-1,), sampling_topk: int = 1,
                 sampling_temperature: float = 1, random_seed=None):
        """ctranslate2.models.Whisper.generate for the options WIS relies on (SURVEY.md section 8b defaults).  With
        beam_size=1 and sampling_topk != 1 it samples num_hypotheses hypotheses per window (``check_sampling_options``),
        returned best first; random_seed (an extension: None, an int or one int per window, ``window_seeds``) makes
        that reproducible.  return_no_speech_prob=True fills each result's no_speech_prob (one per window, sampling
        too): the probability of <|nospeech|> at the prompt's first <|startoftranscript|>, which every prompt must then
        contain."""
        src = self._input(features)
        n = src.n
        if len(prompts) != n:
            raise ValueError(f"expected {n} prompts (one per feature window), got {len(prompts)}")
        lens = {len(p) for p in prompts}
        if len(lens) != 1 or 0 in lens:
            raise ValueError("all prompts must be non-empty and of the same length")
        if isinstance(prompts[0][0], str):
            raise ValueError("prompts must be token ids (WIS builds them with convert_tokens_to_ids, main.py:656-663)")
        sampling = check_sampling_options(num_hypotheses, sampling_topk, sampling_temperature, beam_size, patience,
                                          length_penalty)
        # history processors on each hypothesis's generated tokens (csrc/search.cu)
        if isinstance(repetition_penalty, (bool, np.bool_)) or not isinstance(repetition_penalty, (int, float, np.number)) \
                or not np.isfinite(repetition_penalty) or repetition_penalty <= 0:
            raise ValueError("repetition_penalty must be a finite number > 0")
        if isinstance(no_repeat_ngram_size, (bool, np.bool_)) or not isinstance(no_repeat_ngram_size, (int, np.integer)) \
                or not 0 <= no_repeat_ngram_size <= self._dims.get("n_text_ctx", 448):
            raise ValueError("no_repeat_ngram_size must be an int in [0, n_text_ctx]")
        if not suppress_blank or -1 not in suppress_tokens or asynchronous:
            raise ValueError("suppress_blank=True, suppress_tokens containing -1 and asynchronous=False are required")
        # CTranslate2's rule: a prompt without <|notimestamps|> asks for timestamps (main.py:529, :661 say "Remove this
        # token to generate timestamps"); the returned ids then hold the timestamp tokens
        no_ts = self._dims["no_timestamps"]
        with_ts = {no_ts not in p for p in prompts}
        if len(with_ts) != 1:
            raise ValueError("the prompts of one call must all contain <|notimestamps|> or all omit it")
        timestamps = with_ts.pop()
        if timestamps:
            for q in prompts:
                check_timestamp_prompt(q, self._dims.get("sot", 50258), no_ts)  # (every Whisper vocabulary: 50258)
        if isinstance(max_initial_timestamp_index, bool) or int(max_initial_timestamp_index) != max_initial_timestamp_index \
                or max_initial_timestamp_index < 0:
            raise ValueError("max_initial_timestamp_index must be a non-negative int")
        extra = [int(t) for t in suppress_tokens if t >= 0]
        p = np.asarray(prompts, np.int32)
        # the no-speech probability of window w is read at its prompt's first <|startoftranscript|>; the handles fill
        # ns[s:e] for their windows (a stand-in handle that ignores no_speech_out leaves 0.0)
        ns = np.zeros(n, np.float32) if return_no_speech_prob else None
        if return_no_speech_prob and not (p == self._dims.get("sot", 50258)).any(axis=1).all():
            raise ValueError("return_no_speech_prob needs <|startoftranscript|> in every prompt")
        ns_out = lambda s, e: None if ns is None else ns[s:e]  # noqa: E731
        no_speech = lambda w: 0.0 if ns is None else float(ns[w])  # noqa: E731
        # extension over CTranslate2: `max_length` may be one int per window (requests with different limits coalesced
        # into one call by batcher.TranscribeBatcher); a plain int is the CTranslate2 meaning
        ml = None if np.isscalar(max_length) else np.asarray(max_length, np.int32)
        if ml is not None and ml.shape != (n,):
            raise ValueError("max_length must be an int or one int per feature window")
        # the same extension for the search options: each window searches with its own beam, patience and length
        # penalty, as it would in a call of its own (prompts already come per window)
        search = {"beam_size": beam_size, "patience": patience, "length_penalty": length_penalty}
        for name, v in search.items():
            if np.isscalar(v):
                continue
            a = np.asarray(v)
            kinds = "iu" if name == "beam_size" else "iuf"
            if a.shape != (n,) or a.dtype.kind not in kinds:
                raise ValueError(f"{name} must be a scalar or one {'int' if name == 'beam_size' else 'number'} per "
                                 "feature window")
            if name == "beam_size" and ((a < 1) | (a > 8)).any():
                raise ValueError("beam_size must be in [1, 8]")
            if name == "patience" and not (np.isfinite(a) & (a > 0)).all():
                raise ValueError("patience must be finite and > 0")
            if name == "length_penalty" and not np.isfinite(a).all():
                raise ValueError("length_penalty must be finite")
            search[name] = a
        window = lambda v, s, e: v if np.isscalar(v) else v[s:e]  # noqa: E731

        proc = {}
        if repetition_penalty != 1 or no_repeat_ngram_size != 0:
            proc = dict(repetition_penalty=float(repetition_penalty), no_repeat_ngram_size=int(no_repeat_ngram_size))

        if sampling:
            seeds = window_seeds(random_seed, n)

            def run_sample(h, mel, s, e):
                seqs, scores = h.generate_sample(mel, p[s:e], int(num_hypotheses), int(sampling_topk),
                                                 float(sampling_temperature), seeds[s:e], float(length_penalty),
                                                 max_length if ml is None else ml[s:e], extra, B=e - s,
                                                 timestamps=timestamps,
                                                 max_initial_timestamp_index=int(max_initial_timestamp_index),
                                                 no_speech_out=ns_out(s, e), **proc)
                return seqs, scores

            results = []
            for seqs, scores in self._dispatch(src, run_sample):
                for hyp, sc in zip(seqs, scores):
                    results.append(WhisperGenerationResult(hyp, list(sc) if return_scores else [],
                                                           no_speech(len(results))))
            return results

        def run(h, mel, s, e):
            return h.generate(mel, p[s:e], window(search["beam_size"], s, e), window(search["patience"], s, e),
                              window(search["length_penalty"], s, e), max_length if ml is None else ml[s:e],
                              extra, B=e - s, timestamps=timestamps,
                              max_initial_timestamp_index=int(max_initial_timestamp_index), no_speech_out=ns_out(s, e),
                              **proc)

        outs = self._dispatch(src, run)
        results = []
        for ids, scores in outs:
            for seq, sc in zip(ids, scores):
                results.append(WhisperGenerationResult([seq], [sc] if return_scores else [], no_speech(len(results))))
        return results

    def detect_language(self, features):
        src = self._input(features)
        out = []
        first = self._dims["lang_first"]
        for ids, probs in self._dispatch(src, lambda h, mel, s, e: h.detect_language(mel, B=e - s)):
            for row_ids, row_p in zip(ids, probs):
                out.append([(f"<|{LANGUAGE_CODES[int(t) - first]}|>" if int(t) - first < len(LANGUAGE_CODES) else f"<|{int(t)}|>",
                             float(pr)) for t, pr in zip(row_ids, row_p)])
        return out

    def align(self, features, start_sequence, text_tokens, num_frames, median_filter_width: int = 7):
        """ctranslate2.models.Whisper.align: per window, the DTW path from text tokens to encoder frames over the
        alignment heads' cross-attention, and each text token's probability.  The decoder is teacher-forced with
        start_sequence + [<|notimestamps|>] + text_tokens[b]; num_frames is an int or one int per window (feature frames,
        the path covers num_frames // 2 encoder frames).  Word grouping needs a tokenizer and stays with the caller."""
        src = self._input(features)
        n = src.n
        if len(text_tokens) != n:
            raise ValueError(f"expected {n} text token lists (one per feature window), got {len(text_tokens)}")
        if any(isinstance(t, str) for seq in text_tokens for t in seq) or any(isinstance(t, str) for t in start_sequence):
            raise ValueError("start_sequence and text_tokens must be token ids")
        if np.isscalar(num_frames):
            nf = np.full(n, int(num_frames), np.int64)
        else:
            nf = np.asarray(num_frames, np.int64)
            if nf.shape != (n,):
                raise ValueError("num_frames must be an int or one int per feature window")
        if (nf < 2).any() or (nf > 3000).any():
            raise ValueError("num_frames must be in [2, 3000]")
        text = [list(t) for t in text_tokens]
        start = list(start_sequence)

        results = []
        for paths, probs in self._dispatch(src, lambda h, mel, s, e: h.align(mel, start, text[s:e], nf[s:e],
                                                                              median_filter_width, B=e - s)):
            for p, pr in zip(paths, probs):
                results.append(WhisperAlignmentResult([(int(a), int(b)) for a, b in p], [float(v) for v in pr]))
        return results

    def timing(self, replica: int = 0) -> dict:
        return self._handles[replica].timing()

    def unload_model(self, to_cpu: bool = False):
        for h in self._handles:
            h.close()
