"""ctypes binding of libwisb200.so (include/wisb200.h).  No CPU fallback: a missing library or a missing CUDA
device is an error, never a silent downgrade."""
from __future__ import annotations

import ctypes as C
import os
import threading

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libwisb200.so")

N_DIMS = 20
DIM_NAMES = [
    "d_model", "n_heads", "n_enc_layers", "n_dec_layers", "n_vocab", "n_vocab_pad", "n_text_ctx", "n_mels",
    "n_audio_ctx", "sot", "eot", "transcribe", "translate", "no_timestamps", "sot_prev", "sot_lm", "no_speech",
    "blank", "lang_first", "n_langs",
]
PCM_F32, PCM_S16 = 0, 1
# GEMM epilogues (EpiMode in csrc/kernels.h)
EPI_F16, EPI_F16_GELU, EPI_RESID_F32, EPI_CONV2, EPI_CROSSKV, EPI_F32, EPI_QKV_VT, EPI_DEC_QKV = range(8)

_lib = None


class GenerateOptions(C.Structure):
    """ctypes mirror of wisb_generate_options (include/wisb200.h); the pointer fields take ptr(array) or None"""
    _fields_ = [("struct_size", C.c_uint32), ("beam_size", C.c_int32), ("patience", C.c_float),
                ("length_penalty", C.c_float), ("max_length", C.c_int32), ("timestamps", C.c_int32),
                ("max_initial_timestamp_index", C.c_int32), ("repetition_penalty", C.c_float),
                ("no_repeat_ngram_size", C.c_int32), ("num_hypotheses", C.c_int32), ("sampling_topk", C.c_int32),
                ("sampling_temperature", C.c_float), ("n_extra", C.c_int32), ("extra_suppress", C.c_void_p),
                ("max_length_per_window", C.c_void_p), ("beam_per_window", C.c_void_p),
                ("patience_per_window", C.c_void_p), ("length_penalty_per_window", C.c_void_p), ("seeds", C.c_void_p)]


_SIGS = {
    "wisb_abi_version": (C.c_int, []),
    "wisb_last_error": (C.c_char_p, []),
    "wisb_create": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]),
    "wisb_create_from_host": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_void_p)]),
    "wisb_create_from_device": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_void_p)]),
    "wisb_create_frontend": (C.c_int, [C.c_int, C.POINTER(C.c_void_p)]),
    "wisb_create_frontend_mels": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "wisb_destroy": (C.c_int, [C.c_void_p]),
    "wisb_get_dims": (C.c_int, [C.c_void_p, C.c_void_p]),
    "wisb_logmel": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]),
    "wisb_generate_options_init": (C.c_int, [C.POINTER(GenerateOptions)]),
    "wisb_generate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(GenerateOptions),
                                C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "wisb_detect_language": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "wisb_buffer_alloc": (C.c_int, [C.c_int, C.c_size_t, C.POINTER(C.c_void_p)]),
    "wisb_buffer_free": (C.c_int, [C.c_void_p]),
    "wisb_buffer_to_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "wisb_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]),
    "wisb_load_encoder_output": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]),
    "wisb_align": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                             C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "wisb_debug_align_capture": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                           C.c_int, C.c_void_p, C.c_void_p]),
    "wisb_debug_align_post": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                        C.c_void_p, C.c_void_p]),
    "wisb_get_timing": (C.c_int, [C.c_void_p, C.c_void_p]),
    "wisb_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int]),
    "wisb_get_no_speech_probs": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "wisb_debug_no_speech_probs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                             C.c_void_p]),
    "wisb_debug_gemm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                  C.c_void_p]),
    "wisb_debug_search_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wisb_debug_enc_attn": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "wisb_debug_dec_cross_attn": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wisb_debug_dec_prefill_cross_attn": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wisb_debug_dec_self_attn": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wisb_debug_dec_resid_ln": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_size_t,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wisb_debug_dec_embed_ln": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wisb_debug_dec_pass": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wisb_debug_dec_batch_pass": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p]),
    "wisb_debug_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]),
    "wisb_debug_enc_stem": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "wisb_debug_enc_ln": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "wisb_debug_enc_layer": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wisb_debug_forced_logits": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "wisb_flac_last_error": (C.c_char_p, []),
    "wisb_flac_info": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wisb_flac_decode": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_int64, C.c_void_p]),
}
EXPORTS = sorted(_SIGS)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `python willow_inference_server_b200/build.py`). There is no CPU / PyTorch fallback.")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(l, name)  # AttributeError here = the .so does not match include/wisb200.h
            fn.restype = res
            fn.argtypes = args
        if l.wisb_abi_version() != 2:
            raise ImportError("libwisb200.so ABI version mismatch")
        _lib = l
    return _lib


def check(rc: int):
    if rc == 0:
        return
    msg = lib().wisb_last_error().decode("utf-8", "replace")
    if rc == 1:
        raise ValueError(msg)
    raise RuntimeError(msg)


def ptr(a):
    if a is None:
        return None
    return a.ctypes.data_as(C.c_void_p)


def per_window(value, n: int, dtype, name: str):
    """A generate option given as a scalar (-> None) or as one value per window (-> a C-contiguous [n] array of dtype):
    integers for an int32 option, integers or floats for a float32 one; no silent truncation of a float to an int."""
    if np.isscalar(value):
        return None
    a = np.asarray(value)
    kinds = "iu" if np.dtype(dtype).kind in "iu" else "iuf"
    if a.shape != (n,) or a.dtype.kind not in kinds:
        raise ValueError(f"{name} must be a scalar or one {'int' if kinds == 'iu' else 'number'} per window ({n})")
    return np.ascontiguousarray(a, dtype)


class Handle:
    """Owns one wisb_handle (one model replica or one front end on one GPU)."""

    def __init__(self, raw, keepalive=None):
        self._h = raw
        self._keep = keepalive
        # held around every wisb_generate: a call that asks for the no-speech probability sets a handle option around
        # its wisb_generate, and no other call on this handle may run in between
        self._generate_lock = threading.Lock()

    @classmethod
    def from_path(cls, path: str, device: int = 0):
        h = C.c_void_p()
        check(lib().wisb_create(path.encode(), device, C.byref(h)))
        return cls(h)

    @classmethod
    def from_host(cls, blob: np.ndarray, device: int = 0):
        blob = np.ascontiguousarray(blob, np.uint8)
        h = C.c_void_p()
        check(lib().wisb_create_from_host(ptr(blob), blob.size, device, C.byref(h)))
        return cls(h)

    @classmethod
    def from_device(cls, dev_ptr: int, nbytes: int, device: int = 0, keepalive=None):
        h = C.c_void_p()
        check(lib().wisb_create_from_device(C.c_void_p(dev_ptr), nbytes, device, C.byref(h)))
        return cls(h, keepalive)

    @classmethod
    def frontend(cls, device: int = 0, n_mels: int = 80):
        """a handle without a model that computes n_mels-bin (80 or 128) log-mel features"""
        h = C.c_void_p()
        check(lib().wisb_create_frontend_mels(device, int(n_mels), C.byref(h)))
        return cls(h)

    def close(self):
        if self._h:
            lib().wisb_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ calls
    def dims(self) -> dict:
        out = np.zeros(N_DIMS, np.int32)
        check(lib().wisb_get_dims(self._h, ptr(out)))
        return dict(zip(DIM_NAMES, (int(v) for v in out)))

    @property
    def n_mels(self) -> int:
        """log-mel bins of this handle's features: 80, or 128 for the large-v3 family"""
        if getattr(self, "_n_mels", None) is None:
            self._n_mels = self.dims()["n_mels"]
        return self._n_mels

    def _check_features(self, mel):
        if mel.dtype != np.float32 or mel.ndim != 3 or mel.shape[1:] != (self.n_mels, 3000) or not mel.flags["C_CONTIGUOUS"]:
            raise ValueError(f"features must be a C-contiguous float32 array of shape [n, {self.n_mels}, 3000]")

    def set_option(self, key: str, value: int):
        check(lib().wisb_set_option(self._h, key.encode(), int(value)))

    def timing(self) -> dict:
        out = np.zeros(16, np.float32)
        check(lib().wisb_get_timing(self._h, ptr(out)))
        keys = ["logmel_ms", "h2d_ms", "encoder_ms", "cross_kv_ms", "decode_ms", "generate_ms", "decode_steps", "launches",
                "gemm_ms", "attn_ms", "ln_ms", "conv1_ms", "gemm_launches"]
        return dict(zip(keys, (float(v) for v in out)))

    def logmel(self, pcm, offsets, n_samples, *, to_host=True, keep=False, pcm_on_device=False, pcm_dtype=None, B=None):
        offsets = np.ascontiguousarray(offsets, np.int64)
        n_samples = np.ascontiguousarray(n_samples, np.int32)
        B = int(offsets.shape[0]) if B is None else B
        if pcm_on_device:
            p, dt = C.c_void_p(int(pcm)), pcm_dtype
        else:
            if pcm.dtype == np.int16:
                dt = PCM_S16
            elif pcm.dtype == np.float32:
                dt = PCM_F32
            else:
                raise ValueError("pcm must be float32 or int16")
            pcm = np.ascontiguousarray(pcm)
            p = ptr(pcm)
        out = np.empty((B, self.n_mels, 3000), np.float32) if to_host else None
        check(lib().wisb_logmel(self._h, p, dt, 1 if pcm_on_device else 0, ptr(offsets), ptr(n_samples), B, ptr(out),
                                1 if keep else 0))
        return out

    def generate(self, mel, prompts, beam_size=5, patience=1.0, length_penalty=1.0, max_length=448, extra_suppress=(),
                 B=None, timestamps=False, max_initial_timestamp_index=50, repetition_penalty=1.0, no_repeat_ngram_size=0,
                 no_speech_out=None):
        """-> (token ids per utterance, length-normalised scores).  no_speech_out: None, or a float32 [B] array the call
        fills with every window's no-speech probability (wisb_get_no_speech_probs; every prompt must then contain
        <|startoftranscript|>).  The options are those of wisb_generate_options:
        timestamps=True applies Whisper's timestamp rules to the generated tokens: the prompt may then hold any ids, timestamps
        included, before its last <|startoftranscript|> (a <|startofprev|> context), but neither <|notimestamps|> nor
        timestamp tokens from that token on (in the whole prompt when it has none); repetition_penalty != 1 or no_repeat_ngram_size > 0 switches on the history processors.
        beam_size, patience and length_penalty, like max_length, may each be one value per window."""
        ids, lens, scores = self._generate(
            mel, prompts, B, max_length, extra_suppress, 1, beam_size=beam_size, patience=patience,
            length_penalty=length_penalty, timestamps=1 if timestamps else 0,
            max_initial_timestamp_index=int(max_initial_timestamp_index), repetition_penalty=float(repetition_penalty),
            no_repeat_ngram_size=int(no_repeat_ngram_size), no_speech_out=no_speech_out)
        return [ids[b, : lens[b]].tolist() for b in range(len(lens))], scores.tolist()

    def generate_sample(self, mel, prompts, num_hypotheses, sampling_topk, sampling_temperature, seeds,
                        length_penalty=1.0, max_length=448, extra_suppress=(), B=None, timestamps=False,
                        max_initial_timestamp_index=50, repetition_penalty=1.0, no_repeat_ngram_size=0, no_speech_out=None):
        """num_hypotheses sampled hypotheses per window (sampling_topk != 1), window b seeded by seeds[b] (uint64) ->
        (per window the n token lists, per window the n scores), each window's sorted by score, descending.
        no_speech_out as in generate: one value per window."""
        n = int(num_hypotheses)
        ids, lens, scores = self._generate(
            mel, prompts, B, max_length, extra_suppress, n, beam_size=1, patience=1.0, length_penalty=length_penalty,
            num_hypotheses=n, sampling_topk=int(sampling_topk), sampling_temperature=float(sampling_temperature),
            seeds=seeds, timestamps=1 if timestamps else 0, max_initial_timestamp_index=int(max_initial_timestamp_index),
            repetition_penalty=float(repetition_penalty), no_repeat_ngram_size=int(no_repeat_ngram_size),
            no_speech_out=no_speech_out)
        seqs = [ids[i, : lens[i]].tolist() for i in range(len(lens))]
        return [seqs[b * n: (b + 1) * n] for b in range(len(lens) // n)], \
            [scores[b * n: (b + 1) * n].tolist() for b in range(len(lens) // n)]

    _PER_WINDOW = (("beam_size", "beam_per_window", np.int32), ("patience", "patience_per_window", np.float32),
                   ("length_penalty", "length_penalty_per_window", np.float32))

    def _generate(self, mel, prompts, B, max_length, extra_suppress, n, no_speech_out=None, **options):
        """The one wisb_generate call behind generate and generate_sample: checks the prompts, features, max_length (an
        int or one per window), seeds and per-window search options, sets `options` (arrays by address) over
        wisb_generate_options_init's defaults -> (ids int32 [B * n, stride], lens int32 [B * n], scores float32
        [B * n]), n entries per window.  With no_speech_out, option no_speech_prob is on for this call alone."""
        prompts = np.ascontiguousarray(prompts, np.int32)
        if prompts.ndim != 2:
            raise ValueError("prompts must be [B, prompt_len]")
        if mel is not None:
            self._check_features(mel)
            B = mel.shape[0]
        if B is None or prompts.shape[0] != B:
            raise ValueError("one prompt per feature window is required")
        if "seeds" in options:
            seeds = np.asarray(options["seeds"])
            if seeds.shape != (B,) or seeds.dtype != np.uint64:
                raise ValueError("seeds must be a uint64 array with one seed per window")
            options["seeds"] = np.ascontiguousarray(seeds)
        per_utt = None
        if not np.isscalar(max_length):  # one limit per utterance (requests coalesced by the batcher)
            per_utt = np.ascontiguousarray(max_length, np.int32)
            if per_utt.shape != (B,):
                raise ValueError("max_length must be an int or one int per utterance")
            max_length = int(per_utt.max())
        for name, field, dt in self._PER_WINDOW:
            options[field] = per_window(options[name], B, dt, name)
            # (a scalar given per window stands in as 1; the engine reads the array)
            options[name] = 1 if options[field] is not None else dt(options[name]).item()
        stride = max(1, int(max_length) // 2)
        ids = np.zeros((B * n, stride), np.int32)
        lens = np.zeros(B * n, np.int32)
        scores = np.zeros(B * n, np.float32)
        extra = np.ascontiguousarray(list(extra_suppress), np.int32)
        opt = GenerateOptions()
        check(lib().wisb_generate_options_init(C.byref(opt)))
        options.update(max_length=int(max_length), max_length_per_window=per_utt, n_extra=extra.size,
                       extra_suppress=extra if extra.size else None)
        for k, v in options.items():  # (the arrays stay referenced by `options` until the call returns)
            setattr(opt, k, ptr(v) if v is None or isinstance(v, np.ndarray) else v)
        if no_speech_out is not None and (not isinstance(no_speech_out, np.ndarray) or no_speech_out.dtype != np.float32
                                          or no_speech_out.shape != (B,) or not no_speech_out.flags["C_CONTIGUOUS"]
                                          or not no_speech_out.flags["WRITEABLE"]):
            raise ValueError("no_speech_out must be a writeable C-contiguous float32 array with one entry per window")
        with self._generate_lock:
            if no_speech_out is None:
                check(lib().wisb_generate(self._h, ptr(mel), B, ptr(prompts), prompts.shape[1], C.byref(opt), ptr(ids),
                                          stride, ptr(lens), ptr(scores)))
                return ids, lens, scores
            check(lib().wisb_set_option(self._h, b"no_speech_prob", 1))
            try:
                check(lib().wisb_generate(self._h, ptr(mel), B, ptr(prompts), prompts.shape[1], C.byref(opt), ptr(ids),
                                          stride, ptr(lens), ptr(scores)))
                check(lib().wisb_get_no_speech_probs(self._h, B, ptr(no_speech_out)))
            finally:
                check(lib().wisb_set_option(self._h, b"no_speech_prob", 0))
        return ids, lens, scores

    def detect_language(self, mel, B=None):
        if mel is not None:
            self._check_features(mel)
            B = mel.shape[0]
        nl = self.dims()["n_langs"]
        ids = np.zeros((B, nl), np.int32)
        probs = np.zeros((B, nl), np.float32)
        check(lib().wisb_detect_language(self._h, ptr(mel), B, ptr(ids), ptr(probs)))
        return ids, probs

    def encode(self, mel, out=None, on_device=False):
        """wisb_encode: features float32 [B, n_mels, 3000] (None: the features logmel kept, B = out's first dimension)
        -> encoder output float16 [B, 1500, d_model].  out: a C-contiguous float16 host array of that shape (None: a new
        one), or with on_device=True a device address (int) on this handle's GPU holding that many bytes."""
        if mel is not None:
            self._check_features(mel)
        d = self.dims()["d_model"]
        if on_device:
            if mel is None:
                raise ValueError("a device `out` needs the features (mel), which give the batch size")
            check(lib().wisb_encode(self._h, ptr(mel), mel.shape[0], C.c_void_p(int(out)), 1))
            return out
        if out is None:
            if mel is None:
                raise ValueError("encode(None) needs `out`, whose first dimension is the batch size")
            out = np.empty((mel.shape[0], 1500, d), np.float16)
        if not isinstance(out, np.ndarray) or out.dtype != np.float16 or out.ndim != 3 or out.shape[1:] != (1500, d) \
                or not out.flags["C_CONTIGUOUS"] or (mel is not None and out.shape[0] != mel.shape[0]):
            raise ValueError(f"out must be a C-contiguous float16 array [B, 1500, {d}]")
        check(lib().wisb_encode(self._h, ptr(mel), out.shape[0], ptr(out), 0))
        return out

    def load_encoder_output(self, enc, on_device=False, B=None, dtype=np.float16):
        """wisb_load_encoder_output: enc float16 or float32 [B, 1500, d_model], a host array, or with on_device=True a
        device address (int) on this handle's GPU (then B and dtype say what it holds).  Calls with mel=None, B=B then
        decode it."""
        d = self.dims()["d_model"]
        if on_device:
            dt = np.dtype(dtype)
            p = C.c_void_p(int(enc))
        else:
            enc = np.asarray(enc)
            if enc.ndim != 3 or enc.shape[1:] != (1500, d) or not enc.flags["C_CONTIGUOUS"]:
                raise ValueError(f"the encoder output must be a C-contiguous array [B, 1500, {d}]")
            dt, B, p = enc.dtype, enc.shape[0], ptr(enc)
        if dt not in (np.float16, np.float32):
            raise ValueError("the encoder output must be float16 or float32")
        check(lib().wisb_load_encoder_output(self._h, p, int(B), 0 if dt == np.float16 else 1, 1 if on_device else 0))

    def align(self, mel, start_sequence, text_tokens, num_frames, median_filter_width=7, B=None):
        """wisb_align -> (paths: list of int32 [len, 2] arrays of (text index, frame), token probs: list of float lists).
        num_frames: an int or one int per window."""
        if mel is not None:
            self._check_features(mel)
            B = mel.shape[0]
        if B is None or len(text_tokens) != B:
            raise ValueError("one text token list per feature window is required")
        start = np.ascontiguousarray(list(start_sequence), np.int32)
        lens = np.asarray([len(t) for t in text_tokens], np.int32)
        stride = max(1, int(lens.max()))
        text = np.zeros((B, stride), np.int32)
        for b, t in enumerate(text_tokens):
            text[b, : len(t)] = t
        nf = np.ascontiguousarray(np.broadcast_to(np.asarray(num_frames, np.int32), (B,)))
        path_stride = int((lens + nf // 2).max()) + 1  # the longest DTW path has n + F + 1 entries
        path = np.zeros((B, path_stride, 2), np.int32)
        plen = np.zeros(B, np.int32)
        probs = np.zeros((B, stride), np.float32)
        check(lib().wisb_align(self._h, ptr(mel), B, ptr(start), start.size, ptr(text), ptr(lens), stride, ptr(nf),
                               int(median_filter_width), ptr(path), path_stride, ptr(plen), ptr(probs)))
        return [path[b, : plen[b]].copy() for b in range(B)], [probs[b, : lens[b]].tolist() for b in range(B)]

    def align_timing(self) -> dict:
        """Stage timings of the last align call (ms; capture_ms needs option "profile")."""
        out = np.zeros(16, np.float32)
        check(lib().wisb_get_timing(self._h, ptr(out)))
        keys = {"h2d_ms": 1, "encoder_ms": 2, "passes_ms": 3, "filter_ms": 4, "align_ms": 5, "passes": 6, "launches": 7,
                "capture_ms": 13, "dtw_ms": 14}
        return {k: float(out[i]) for k, i in keys.items()}

    # ------------------------------------------------------------------ diagnostics (tests)
    def debug_align_capture(self, mel, start_sequence, text_tokens, num_frames, n_align_heads: int):
        """Raw captured probabilities of the model's `n_align_heads` alignment heads in wisb_align -> float32
        [B, A, n_max + 1, F_max] (zero where a window has no row / frame)."""
        B = mel.shape[0]
        start = np.ascontiguousarray(list(start_sequence), np.int32)
        lens = np.asarray([len(t) for t in text_tokens], np.int32)
        stride = max(1, int(lens.max()))
        text = np.zeros((B, stride), np.int32)
        for b, t in enumerate(text_tokens):
            text[b, : len(t)] = t
        nf = np.ascontiguousarray(np.broadcast_to(np.asarray(num_frames, np.int32), (B,)))
        has = lens > 0
        A = int(n_align_heads)
        n_max = int(lens[has].max()) if has.any() else 0
        f_max = int((nf[has] // 2).max()) if has.any() else 0
        cap = np.zeros((B, A, n_max + 1, f_max), np.float32)
        check(lib().wisb_debug_align_capture(self._h, ptr(np.ascontiguousarray(mel, np.float32)), B, ptr(start), start.size,
                                             ptr(text), ptr(lens), stride, ptr(nf), ptr(cap)))
        return cap

    def debug_align_post(self, weights, width: int = 7, dtw_only: bool = False):
        """wisb_debug_align_post on one window: weights float32 [A, R, F] (or the matrix [R, F] with dtw_only) ->
        (matrix float32 [R, F], path int32 [len, 2])."""
        w = np.ascontiguousarray(weights, np.float32)
        if dtw_only:
            w = w.reshape((1,) + w.shape[-2:])
        A, R, F = w.shape
        mat = np.zeros((R, F), np.float32)
        path = np.zeros((R + F, 2), np.int32)
        plen = np.zeros(1, np.int32)
        check(lib().wisb_debug_align_post(self._h, ptr(w), A, R, F, int(width), 1 if dtw_only else 0, ptr(mat), ptr(path),
                                          ptr(plen)))
        return mat, path[: plen[0]].copy()

    def debug_gemm(self, a16: np.ndarray, w16: np.ndarray, impl: int = 0, bn: int = 0, *, mode: int = EPI_F32,
                   planner: int = 0, bias=None, pos=None, out=None, aux=None, aux2=None, row_slot=None, row_pos=None,
                   a_wrap: int = 0, k_splits: int = 1, m_valid: int = 0, n_valid: int = 0, ldo: int = 0, d_model: int = 0,
                   n_heads: int = 0, batch: int = 0, kv_swizzle: int = 0, t_cap: int = 0, return_plan: bool = False):
        """One GEMM A . W^T through epilogue `mode` (EPI_*) -> `out` (or (out, plan) with return_plan).  out / aux / aux2
        are C-contiguous arrays updated in place: elements the epilogue does not write keep their values.  Without `out`
        (plain EPI_F32) a zero float32 [M, N] array is returned.  With a_wrap, a16 holds the physical [M + 1, a_wrap] rows.
        plan = {"bn", "mcast", "k_splits", "grid"} as launched."""
        a16 = np.ascontiguousarray(a16, np.float16)
        w16 = np.ascontiguousarray(w16, np.float16)
        N, K = w16.shape
        M = a16.shape[0] - (1 if a_wrap else 0)
        if a16.shape[1] != (a_wrap if a_wrap else K):
            raise ValueError("A and W disagree on K")
        if out is None:
            if mode != EPI_F32 or k_splits != 1 or planner == 2:
                raise ValueError("this epilogue needs an explicit out buffer")
            out = np.zeros((M, N), np.float32)
        for buf in (out, aux, aux2):
            if buf is not None and not buf.flags["C_CONTIGUOUS"]:
                raise ValueError("out / aux / aux2 must be C-contiguous")
        bias = None if bias is None else np.ascontiguousarray(bias, np.float32)
        pos = None if pos is None else np.ascontiguousarray(pos, np.float32)
        if bias is not None and bias.size != N:
            raise ValueError("bias must have N elements")
        if pos is not None and pos.size != 1500 * (ldo or N):
            raise ValueError("pos must be [1500, ldo]")
        slot = None if row_slot is None else np.ascontiguousarray(row_slot, np.int32)
        rpos = None if row_pos is None else np.ascontiguousarray(row_pos, np.int32)
        if (slot is not None and slot.size != M) or (rpos is not None and rpos.size != M):
            raise ValueError("row_slot / row_pos must have M entries")
        prm = np.asarray([M, N, K, impl, bn, planner, mode, a_wrap, k_splits, m_valid, n_valid, ldo, d_model, n_heads, batch,
                          kv_swizzle, t_cap], np.int32)
        plan = np.zeros(4, np.int32)
        nbytes = lambda b: 0 if b is None else b.nbytes  # noqa: E731
        check(lib().wisb_debug_gemm(self._h, ptr(prm), prm.size, ptr(a16), ptr(w16), ptr(bias), ptr(pos), ptr(slot), ptr(rpos),
                                    ptr(out), out.nbytes, ptr(aux), nbytes(aux), ptr(aux2), nbytes(aux2), ptr(plan)))
        if return_plan:
            return out, dict(zip(("bn", "mcast", "k_splits", "grid"), (int(v) for v in plan)))
        return out

    @staticmethod
    def search_state(n_utt: int, beam: int, max_new: int, t_max: int, sample: bool = False) -> dict:
        """A zeroed search state for debug_search_step_state (best_score -inf): name -> array, in the entry's order.
        sample: the layout of debug_search_step_sample (beam = the hypotheses; best_* per row)."""
        R = n_utt * beam
        H = R if sample else n_utt
        return {"st": np.zeros(5, np.int32), "flip": np.zeros(1, np.int32),   # DecState: pos, gen_step, n_done, all_done, ticket
                "seq": np.zeros((2, R, max_new), np.int32), "indir": np.zeros((2, R, t_max), np.int32),
                "tokens": np.zeros(R, np.int32), "row_pos": np.zeros(R, np.int32), "done": np.zeros(n_utt, np.int32),
                "n_hyp": np.zeros(n_utt, np.int32), "best_len": np.zeros(H, np.int32),
                "best_tokens": np.zeros((H, max_new), np.int32),
                "cum": np.zeros(R, np.float32), "best_score": np.full(H, -np.inf, np.float32)}

    _STATE_F = ("cum", "best_score")

    def debug_search_step(self, logits, hist, mask, *, beam: int, gen: int, eot: int, no_timestamps: int,
                          timestamps: bool, max_initial_timestamp_index: int = 50, cum=None, done=None,
                          repetition_penalty=None, no_repeat_ngram_size=None):
        """The candidates of one production search step on fresh hypotheses (max_hyp = beam, length penalty 1).
        logits float32 [n_utt*beam, V]; hist int [n_utt*beam, gen] the rows' generated tokens; mask uint8 [V] (bit 0
        every step, bit 1 at gen 0); cum [n_utt*beam] (None = 0); done [n_utt] finished utterances (None = none).
        -> (cand_idx int32 [n_utt, 2*beam] = beam*V + token, cand_score float32 [n_utt, 2*beam], row_lse float32
        [n_utt*beam]).  The whole search state: debug_search_step_state."""
        logits = np.ascontiguousarray(logits, np.float32)
        R = logits.shape[0]
        if R % beam:
            raise ValueError("logits rows must be n_utt * beam")
        n_utt = R // beam
        st = self.search_state(n_utt, beam, gen + 2, 1)
        st["st"][1] = gen
        if gen:
            st["seq"][0, :, :gen] = np.asarray(hist, np.int32).reshape(R, gen)
        if cum is not None:
            st["cum"][:] = np.asarray(cum, np.float32).reshape(R)
        if done is not None:
            st["done"][:] = np.asarray(done, np.int32).reshape(n_utt)
            st["st"][2] = int((st["done"] != 0).sum())
            if st["st"][2] == n_utt:
                raise ValueError("every utterance is finished")
        _, ci, cs, lse = self.debug_search_step_state(logits, mask, st, beam=beam, max_hyp=beam, eot=eot,
                                                      no_timestamps=no_timestamps, timestamps=timestamps,
                                                      max_initial_timestamp_index=max_initial_timestamp_index,
                                                      repetition_penalty=repetition_penalty,
                                                      no_repeat_ngram_size=no_repeat_ngram_size)
        return ci, cs, lse

    def debug_search_step_state(self, logits, mask, state, *, beam: int, max_hyp: int, eot: int, V: int = 0, no_timestamps: int = 0,
                          timestamps: bool = False, max_initial_timestamp_index: int = 50, length_penalty: float = 1.0,
                          max_new_u=None, prompt=None, shared_prefix: int = 0, repetition_penalty=None,
                          no_repeat_ngram_size=None, beam_u=None, max_hyp_u=None, length_penalty_u=None):
        """One production search step on caller state.  logits float32 [n_utt*beam, ldl] (only columns < V are read; V
        = ldl by default); mask uint8 [V] (bit 0 every step, bit 1 at the first generated step); state as made by
        search_state (its shapes give max_new and t_max); prompt int [n_utt, prompt_len]: run the search initialisation
        (with shared_prefix) first; repetition_penalty / no_repeat_ngram_size: the history processors (None: off);
        beam_u / max_hyp_u / length_penalty_u (all three, [n_utt] each): per-utterance search options, `beam` the row
        block of every utterance, max_hyp and length_penalty unused.
        -> (new state, cand_idx int32 [n_utt, 2*beam] = beam*V + token or -1, cand_score
        float32 [n_utt, 2*beam], row_lse float32 [n_utt*beam])."""
        out, ci, cs, lse = self._search_step(
            logits, mask, state, beam, max_hyp, 1, 1.0, None, (beam_u, max_hyp_u, length_penalty_u), eot=eot, V=V,
            no_timestamps=no_timestamps, timestamps=timestamps, max_initial_timestamp_index=max_initial_timestamp_index,
            length_penalty=length_penalty, max_new_u=max_new_u, prompt=prompt, shared_prefix=shared_prefix,
            repetition_penalty=repetition_penalty, no_repeat_ngram_size=no_repeat_ngram_size)
        return out, ci[:, : 2 * beam], cs[:, : 2 * beam], lse

    def debug_search_step_sample(self, logits, mask, state, seeds, *, n: int, sampling_topk: int,
                                 sampling_temperature: float, eot: int, V: int = 0, no_timestamps: int = 0,
                                 timestamps: bool = False, max_initial_timestamp_index: int = 50,
                                 length_penalty: float = 1.0, max_new_u=None, prompt=None, shared_prefix: int = 0,
                                 repetition_penalty=None, no_repeat_ngram_size=None):
        """One production sampling step on caller state.  As debug_search_step_state with n hypotheses per utterance,
        the state made by search_state(..., sample=True) and seeds uint64 [n_utt].
        -> (new state, sampled int32 [R] (-1 = none), key float32 [R], row_lse float32 [R])."""
        seeds = np.ascontiguousarray(np.asarray(seeds, np.uint64).ravel())
        out, ci, cs, lse = self._search_step(
            logits, mask, state, n, 1, int(sampling_topk), float(sampling_temperature), seeds, (None, None, None),
            eot=eot, V=V, no_timestamps=no_timestamps, timestamps=timestamps,
            max_initial_timestamp_index=max_initial_timestamp_index, length_penalty=length_penalty, max_new_u=max_new_u,
            prompt=prompt, shared_prefix=shared_prefix, repetition_penalty=repetition_penalty,
            no_repeat_ngram_size=no_repeat_ngram_size)
        # row k of utterance u drew the token in candidate slot k of u, with its Gumbel key as the score
        return out, ci[:, :n].reshape(-1), cs[:, :n].reshape(-1), lse

    def _search_step(self, logits, mask, state, rows: int, max_hyp: int, topk: int, temperature: float, seeds, per_utt,
                     *, eot, V, no_timestamps, timestamps, max_initial_timestamp_index, length_penalty, max_new_u,
                     prompt, shared_prefix, repetition_penalty, no_repeat_ngram_size):
        """wisb_debug_search_step with `rows` rows per utterance (sampling when topk != 1) and per_utt = (beam_u,
        max_hyp_u, length_penalty_u) -> (new state, cand_idx int32 [n_utt, 16], cand_score float32 [n_utt, 16],
        row_lse float32 [R])."""
        logits = np.ascontiguousarray(logits, np.float32)
        R, ldl = logits.shape
        V = V or ldl
        if R % rows:
            raise ValueError(f"logits rows must be n_utt * {rows}")
        n_utt = R // rows
        mask = np.ascontiguousarray(mask, np.uint8)
        if mask.shape != (V,):
            raise ValueError("mask must have V entries")
        if seeds is not None and seeds.shape != (n_utt,):
            raise ValueError("seeds must have n_utt entries")
        _, _, max_new = state["seq"].shape
        t_max = state["indir"].shape[2]
        want = self.search_state(n_utt, rows, max_new, t_max, sample=topk != 1)
        for k, v in want.items():
            if np.shape(state[k]) != v.shape:
                raise ValueError(f"state[{k!r}] must have shape {v.shape}")
        si = np.concatenate([np.asarray(state[k], np.int32).ravel() for k in want if k not in self._STATE_F])
        sf = np.concatenate([np.asarray(state[k], np.float32).ravel() for k in self._STATE_F])
        caps = None if max_new_u is None else np.ascontiguousarray(max_new_u, np.int32).reshape(n_utt)
        pr = None if prompt is None else np.ascontiguousarray(prompt, np.int32).reshape(n_utt, -1)
        init = 0 if pr is None else 1 + int(shared_prefix)
        prm = np.asarray([n_utt, rows, V, ldl, eot, no_timestamps, 1 if timestamps else 0, max_initial_timestamp_index,
                          max_new, max_hyp, t_max, init, 0 if pr is None else pr.shape[1], int(no_repeat_ngram_size or 0),
                          topk], np.int32)
        rp = 1.0 if repetition_penalty is None else repetition_penalty
        fprm = np.asarray([length_penalty, rp, temperature], np.float32)
        bu, hu, lu = (None if v is None else np.ascontiguousarray(v, dt).reshape(n_utt)
                      for v, dt in zip(per_utt, (np.int32, np.int32, np.float32)))
        ci = np.zeros((n_utt, 16), np.int32)
        cs = np.zeros((n_utt, 16), np.float32)
        lse = np.zeros(R, np.float32)
        check(lib().wisb_debug_search_step(self._h, ptr(prm), prm.size, ptr(fprm), fprm.size, ptr(logits), ptr(mask),
                                           ptr(caps), ptr(pr), ptr(bu), ptr(hu), ptr(lu), ptr(seeds), ptr(si), ptr(sf),
                                           ptr(ci), ptr(cs), ptr(lse)))
        out, oi, of = {}, 0, 0
        for k, v in want.items():
            if k in self._STATE_F:
                out[k], of = sf[of : of + v.size].reshape(v.shape).copy(), of + v.size
            else:
                out[k], oi = si[oi : oi + v.size].reshape(v.shape).copy(), oi + v.size
        return out, ci, cs, lse

    def debug_no_speech_probs(self, logits: np.ndarray, rows, n_vocab: int, no_speech: int, out=None) -> np.ndarray:
        """The no-speech reduction on caller data: logits float32 [n_rows, ldl], rows int [n] (< 0: out[u] kept) ->
        out float32 [n], out[u] = softmax(logits[rows[u], :n_vocab])[no_speech]."""
        logits = np.ascontiguousarray(logits, np.float32)
        rows = np.ascontiguousarray(rows, np.int32)
        out = np.zeros(rows.size, np.float32) if out is None else np.ascontiguousarray(out, np.float32).copy()
        check(lib().wisb_debug_no_speech_probs(self._h, ptr(logits), logits.shape[0], logits.shape[1], ptr(rows), rows.size,
                                               int(n_vocab), int(no_speech), ptr(out)))
        return out

    def debug_enc_attn(self, qkv16: np.ndarray, n_heads: int, impl: int = 0) -> np.ndarray:
        """Encoder self-attention on qkv fp16 [B, 1536, 3d] -> ctx fp16 [B, 1536, d]; impl 0 = wgmma (MN-major V),
        1 = wgmma (transposed Vt), 2 = SIMT check."""
        qkv16 = np.ascontiguousarray(qkv16, np.float16)
        B, T, three_d = qkv16.shape
        if T != 1536 or three_d % 3:
            raise ValueError("qkv must be [B, 1536, 3 d_model]")
        d = three_d // 3
        ctx = np.zeros((B, 1536, d), np.float16)
        check(lib().wisb_debug_enc_attn(self._h, ptr(qkv16), B, d, n_heads, impl, ptr(ctx)))
        return ctx

    # the batched decoder pass's own kernels (csrc/decoder_batch.cu) on caller data.  Output arrays are updated in place:
    # elements the kernel does not write keep their values.
    @staticmethod
    def _inout(a, dtype, shape, name):
        if not isinstance(a, np.ndarray) or a.dtype != dtype or a.shape != shape or not a.flags["C_CONTIGUOUS"]:
            raise ValueError(f"{name} must be a C-contiguous {np.dtype(dtype).name} array of shape {shape}")
        return a

    def debug_dec_cross_attn(self, q, ckv, ctx, *, layer: int, rows_per_utt: int, impl: int = 0, done=None):
        """Cross-attention: q float32 [n_utt * rows_per_utt, d] (unscaled), ckv float16 [n_layers, 2 (K, V), n_utt, H,
        1536, 64], ctx float16 [n_utt * rows_per_utt, d] in / out, done int [n_utt] or None.  impl 0 = wgmma, 1 = SIMT
        cluster kernel."""
        if not isinstance(ckv, np.ndarray) or ckv.dtype != np.float16 or ckv.ndim != 6 or ckv.shape[1] != 2 \
                or ckv.shape[4:] != (1536, 64) or not ckv.flags["C_CONTIGUOUS"]:
            raise ValueError("ckv must be a C-contiguous float16 array [n_layers, 2, n_utt, H, 1536, 64]")
        L, _, n_utt, H = ckv.shape[:4]
        shape = (n_utt * rows_per_utt, 64 * H)
        q = self._inout(np.ascontiguousarray(q, np.float32), np.float32, shape, "q")
        self._inout(ctx, np.float16, shape, "ctx")
        done = None if done is None else np.ascontiguousarray(np.asarray(done, np.int32).reshape(n_utt))
        prm = np.asarray([n_utt, rows_per_utt, H, L, layer, impl], np.int32)
        check(lib().wisb_debug_dec_cross_attn(self._h, ptr(prm), prm.size, ptr(q), ptr(ckv), ptr(done), ptr(ctx)))
        return ctx

    def debug_dec_prefill_cross_attn(self, q, ckv, ctx, *, layer: int, rows_per_utt: int, swizzled: bool = False):
        """Cross-attention of a wide prefill pass: q float32 [n_utt * rows_per_utt, d] (unscaled, rows_per_utt 1..448),
        ckv float16 [n_layers, 2 (K, V), n_utt, H, 1536, 64], in the persistent warp-MMA pass's chunk-swizzled layout when
        `swizzled`, ctx float16 [n_utt * rows_per_utt, d] in / out."""
        if not isinstance(ckv, np.ndarray) or ckv.dtype != np.float16 or ckv.ndim != 6 or ckv.shape[1] != 2 \
                or ckv.shape[4:] != (1536, 64) or not ckv.flags["C_CONTIGUOUS"]:
            raise ValueError("ckv must be a C-contiguous float16 array [n_layers, 2, n_utt, H, 1536, 64]")
        L, _, n_utt, H = ckv.shape[:4]
        shape = (n_utt * rows_per_utt, 64 * H)
        q = self._inout(np.ascontiguousarray(q, np.float32), np.float32, shape, "q")
        self._inout(ctx, np.float16, shape, "ctx")
        prm = np.asarray([n_utt, rows_per_utt, H, L, layer, 1 if swizzled else 0], np.int32)
        check(lib().wisb_debug_dec_prefill_cross_attn(self._h, ptr(prm), prm.size, ptr(q), ptr(ckv), ptr(ctx)))
        return ctx

    def debug_dec_self_attn(self, q, kcache, vcache, row_pos, row_slot, indir0, indir1, ctx, *, rows_per_utt: int,
                            flip: int, prefill: bool = False, done=None):
        """Self-attention over the cache: q float32 [R, d], kcache / vcache float16 [n_slots, t_cap, d], row_pos /
        row_slot int [R], indir0 / indir1 int [R, t_ind], ctx float16 [R, d] in / out, done int [R / rows_per_utt] or
        None; flip selects indir1."""
        q = np.ascontiguousarray(q, np.float32)
        R, d = q.shape
        n_slots, t_cap = kcache.shape[:2]
        self._inout(kcache, np.float16, (n_slots, t_cap, d), "kcache")
        self._inout(vcache, np.float16, (n_slots, t_cap, d), "vcache")
        self._inout(ctx, np.float16, (R, d), "ctx")
        if d % 64:
            raise ValueError("d must be 64 x heads")
        row_pos, row_slot = (np.ascontiguousarray(np.asarray(v, np.int32).reshape(R)) for v in (row_pos, row_slot))
        indir0, indir1 = (np.ascontiguousarray(v, np.int32) for v in (indir0, indir1))
        if indir0.ndim != 2 or indir0.shape[0] != R or indir1.shape != indir0.shape:
            raise ValueError("indir0 / indir1 must be [R, t_ind]")
        if R % rows_per_utt:
            raise ValueError("R must be a multiple of rows_per_utt")
        done = None if done is None else np.ascontiguousarray(np.asarray(done, np.int32).reshape(R // rows_per_utt))
        prm = np.asarray([R, d // 64, n_slots, t_cap, indir0.shape[1], rows_per_utt, int(prefill), int(flip)], np.int32)
        check(lib().wisb_debug_dec_self_attn(self._h, ptr(prm), prm.size, ptr(q), ptr(kcache), ptr(vcache), ptr(row_pos),
                                             ptr(row_slot), ptr(indir0), ptr(indir1), ptr(done), ptr(ctx)))
        return ctx

    def debug_dec_resid_ln(self, x, xn, part, bias, g, b, *, n_splits: int, split_stride: int, rows=None):
        """Split-K reduction + bias + residual + LayerNorm of the first `rows` rows (default all): x float32 [cap, d] and
        xn float16 [cap, d] in / out; part a C-contiguous float32 array holding slab s at flat offset s * split_stride;
        bias, g, b float32 [d]."""
        cap, d = x.shape
        R = cap if rows is None else int(rows)
        self._inout(x, np.float32, (cap, d), "x")
        self._inout(xn, np.float16, (cap, d), "xn")
        if not isinstance(part, np.ndarray) or part.dtype != np.float32 or not part.flags["C_CONTIGUOUS"]:
            raise ValueError("part must be a C-contiguous float32 array")
        vecs = [np.ascontiguousarray(np.asarray(v, np.float32).reshape(d)) for v in (bias, g, b)]
        check(lib().wisb_debug_dec_resid_ln(self._h, R, cap, d, int(n_splits), int(split_stride), ptr(part), part.size,
                                            *(ptr(v) for v in vecs), ptr(x), ptr(xn)))
        return x, xn

    def debug_dec_embed_ln(self, tokens, row_pos, tok_emb, pos_emb, g, b, x, xn):
        """Embedding + LayerNorm of R = len(tokens) rows: row_pos int [R], tok_emb float16 [n_vocab, d], pos_emb
        float32 [n_pos, d], g, b float32 [d]; x float32 [cap, d] and xn float16 [cap, d] in / out, cap >= R."""
        cap, d = x.shape
        R = len(tokens)
        self._inout(x, np.float32, (cap, d), "x")
        self._inout(xn, np.float16, (cap, d), "xn")
        tokens, row_pos = (np.ascontiguousarray(np.asarray(v, np.int32).reshape(R)) for v in (tokens, row_pos))
        tok_emb = np.ascontiguousarray(tok_emb, np.float16)
        pos_emb = np.ascontiguousarray(pos_emb, np.float32)
        if tok_emb.ndim != 2 or tok_emb.shape[1] != d or pos_emb.ndim != 2 or pos_emb.shape[1] != d:
            raise ValueError("tok_emb / pos_emb must be [rows, d]")
        vecs = [np.ascontiguousarray(np.asarray(v, np.float32).reshape(d)) for v in (g, b)]
        check(lib().wisb_debug_dec_embed_ln(self._h, R, cap, d, tok_emb.shape[0], pos_emb.shape[0], ptr(tokens), ptr(row_pos),
                                            ptr(tok_emb), ptr(pos_emb), *(ptr(v) for v in vecs), ptr(x), ptr(xn)))
        return x, xn

    def debug_dec_pass(self, impl: int, tokens, enc16, kcache, vcache, x, logits, *, n_utt: int, beam: int = 1,
                       pf_len: int = 0, pos: int = 0, flip: int = 0, indir0=None, indir1=None, with_logits: bool = True):
        """One persistent decoder pass (impl 1 warp-MMA, 0 SIMT) on caller state (wisb_debug_dec_pass).  tokens int
        [R] (R = n_utt * beam, or n_utt * pf_len for the one-pass prefill), enc16 float16 [n_utt, 1536, d], indir0 /
        indir1 int [R, 448] (decoding steps).  In / out: kcache / vcache float16 [L, 8, 448, d], x float32 [8, d],
        logits float32 [8, n_vocab_pad].  -> the cross K/V the pass read, float16 [L, 2, n_utt, H, 1536, 64]."""
        dm = self.dims()
        d, L, H = dm["d_model"], dm["n_dec_layers"], dm["n_heads"]
        self._inout(kcache, np.float16, (L, 8, 448, d), "kcache")
        self._inout(vcache, np.float16, (L, 8, 448, d), "vcache")
        self._inout(x, np.float32, (8, d), "x")
        self._inout(logits, np.float32, (8, dm["n_vocab_pad"]), "logits")
        enc16 = self._inout(np.ascontiguousarray(enc16, np.float16), np.float16, (n_utt, 1536, d), "enc16")
        R = n_utt * (pf_len if pf_len > 0 else beam)
        tokens = np.ascontiguousarray(np.asarray(tokens, np.int32).reshape(-1))
        if tokens.size != R:
            raise ValueError(f"tokens must have {R} entries")
        ind = [None, None]
        if pf_len == 0:
            if indir0 is None or indir1 is None:
                raise ValueError("a decoding step needs indir0 and indir1")
            ind = [self._inout(np.ascontiguousarray(v, np.int32), np.int32, (R, 448), n) for v, n in
                   ((indir0, "indir0"), (indir1, "indir1"))]
        ckv = np.zeros((L, 2, n_utt, H, 1536, 64), np.float16)
        prm = np.asarray([impl, n_utt, beam, pf_len, pos, flip, int(with_logits)], np.int32)
        check(lib().wisb_debug_dec_pass(self._h, ptr(prm), prm.size, ptr(tokens), ptr(ind[0]), ptr(ind[1]), ptr(enc16),
                                        ptr(ckv), ptr(kcache), ptr(vcache), ptr(x), ptr(logits)))
        return ckv

    BATCH_PLANS = ("qkv", "o", "cq", "co", "fc1", "fc2", "vocab")

    def debug_dec_batch_geometry(self, kind: int, n_utt: int, *, batch_rows: int = 1, t_need: int = 1,
                                 chunk_max: int = 1) -> dict:
        """The cache geometry a batched pass of this kind would run with now (wisb_debug_dec_batch_pass with no state;
        nothing is allocated) -> dict(slots, t_cap, layer_stride, rows_cap)."""
        prm = np.asarray([kind, n_utt, 1, 1, 1, 0, batch_rows, t_need, chunk_max, 0, 1 if kind == 0 else 0, 1, 0, 0, 0, 0],
                         np.int32)
        geom = np.zeros(4, np.int64)
        check(lib().wisb_debug_dec_batch_pass(self._h, ptr(prm), prm.size, None, None, None, None, None, None, None, None,
                                              None, None, ptr(geom), None))
        return dict(zip(("slots", "t_cap", "layer_stride", "rows_cap"), (int(v) for v in geom)))

    def debug_dec_batch_pass(self, kind: int, tokens, ckv, kcache, vcache, *, n_utt: int, rows_per_utt: int,
                             row_pos=None, indir0=None, indir1=None, flip: int = 0, done=None, slot_stride: int = 1,
                             p0: int = 0, batch_rows: int = 1, t_need: int = 1, chunk_max: int = 1,
                             with_logits: bool = False, cross_tc: int = 1, ckv_sw: int = 0, poison=None, x=None,
                             logits=None):
        """ONE batched decoder pass on caller state (wisb_debug_dec_batch_pass; kinds 0 step, 1 prefill, 2 / 3 wide
        prefill into the batched / persistent cache).  tokens int [R] (step) or the prompt matrix [n_utt, prompt_len];
        ckv float16 [L, 2, n_utt, H, 1536, 64]; kcache / vcache float16 [L, slots, t_cap, d] in / out, shaped from
        debug_dec_batch_geometry; poison None or the (slot, position) cell row-table padding points at.  x float32
        [>= R, d] and logits float32 [>= R, n_vocab_pad] (with logits) receive rows < R (logit columns < n_vocab); the
        rest keeps the caller's values (default: new zero arrays of R rows).
        -> dict(x, logits, plans, geom)."""
        dm = self.dims()
        d, L, H = dm["d_model"], dm["n_dec_layers"], dm["n_heads"]
        R = n_utt * rows_per_utt
        tokens = np.ascontiguousarray(np.asarray(tokens, np.int32))
        if kind == 0:
            if tokens.shape != (R,) or row_pos is None or indir0 is None or indir1 is None:
                raise ValueError("a step needs tokens [R], row_pos [R], indir0 and indir1 [R, 448]")
            row_pos = np.ascontiguousarray(np.asarray(row_pos, np.int32).reshape(R))
            ind = [self._inout(np.ascontiguousarray(v, np.int32), np.int32, (R, 448), n)
                   for v, n in ((indir0, "indir0"), (indir1, "indir1"))]
            prompt_len = 1
        else:
            if tokens.ndim != 2 or tokens.shape[0] != n_utt:
                raise ValueError("a prefill pass needs the prompt matrix [n_utt, prompt_len]")
            prompt_len = tokens.shape[1]
            ind = [None, None]
        done = None if done is None else np.ascontiguousarray(np.asarray(done, np.int32).reshape(n_utt))
        self._inout(ckv, np.float16, (L, 2, n_utt, H, 1536, 64), "ckv")
        geom = self.debug_dec_batch_geometry(kind, n_utt, batch_rows=batch_rows, t_need=t_need, chunk_max=chunk_max)
        shape = (L, geom["slots"], geom["t_cap"], d)
        self._inout(kcache, np.float16, shape, "kcache")
        self._inout(vcache, np.float16, shape, "vcache")
        x = np.zeros((R, d), np.float32) if x is None else x
        self._inout(x, np.float32, (max(R, x.shape[0]), d), "x")
        if with_logits:
            logits = np.zeros((R, dm["n_vocab_pad"]), np.float32) if logits is None else logits
            self._inout(logits, np.float32, (max(R, logits.shape[0]), dm["n_vocab_pad"]), "logits")
        else:
            logits = None
        ps, pp = poison if poison is not None else (0, 0)
        prm = np.asarray([kind, n_utt, rows_per_utt, slot_stride, prompt_len, p0, batch_rows, t_need, chunk_max, flip,
                          int(with_logits), cross_tc, ckv_sw, int(poison is not None), ps, pp], np.int32)
        g = np.zeros(4, np.int64)
        plan = np.zeros(28, np.int32)
        check(lib().wisb_debug_dec_batch_pass(self._h, ptr(prm), prm.size, ptr(tokens), ptr(row_pos), ptr(ind[0]),
                                              ptr(ind[1]), ptr(done), ptr(ckv), ptr(kcache), ptr(vcache), ptr(x),
                                              ptr(logits), ptr(g), ptr(plan)))
        plans = {k: tuple(int(v) for v in plan[4 * i: 4 * i + 4]) for i, k in enumerate(self.BATCH_PLANS)}
        return dict(x=x, logits=logits, plans=plans, geom=geom)

    def debug_encode(self, mel: np.ndarray, n_layers: int = -1) -> np.ndarray:
        mel = np.ascontiguousarray(mel, np.float32)
        out = np.zeros((mel.shape[0], 1500, self.dims()["d_model"]), np.float32)
        check(lib().wisb_debug_encode(self._h, ptr(mel), mel.shape[0], ptr(out), n_layers))
        return out

    # the encoder one stage at a time (wisb_debug_enc_*)
    def debug_enc_stem(self, mel: np.ndarray):
        """conv1 + conv2 on log-mel float32 [B, n_mels, 3000] -> (h1 float16 [B * 3072 + 8, d], x float32 [B, 1536, d])"""
        mel = np.ascontiguousarray(mel, np.float32)
        if mel.ndim != 3 or mel.shape[1:] != (self.n_mels, 3000):
            raise ValueError(f"mel must be [B, {self.n_mels}, 3000]")
        B, d = mel.shape[0], self.dims()["d_model"]
        h1 = np.zeros((B * 3072 + 8, d), np.float16)
        x = np.zeros((B, 1536, d), np.float32)
        check(lib().wisb_debug_enc_stem(self._h, ptr(mel), B, ptr(h1), ptr(x)))
        return h1, x

    def debug_enc_ln(self, x, g, b, y, *, pdl: bool = False):
        """The encoder LayerNorm of x float32 [rows, d] with g, b float32 [d] into y float16 [round_up(rows, 8), d] (in
        / out: rows >= `rows` keep their values)."""
        x = np.ascontiguousarray(x, np.float32)
        rows, d = x.shape
        self._inout(y, np.float16, ((rows + 7) // 8 * 8, d), "y")
        g, b = (np.ascontiguousarray(np.asarray(v, np.float32).reshape(d)) for v in (g, b))
        check(lib().wisb_debug_enc_ln(self._h, ptr(x), rows, d, ptr(g), ptr(b), int(bool(pdl)), ptr(y)))
        return y

    ENC_STAGES = (("xn1", np.float16, 1), ("qkv", np.float16, 3), ("vt", np.float16, 1), ("ctx", np.float16, 1),
                  ("x_o", np.float32, 1), ("xn2", np.float16, 1), ("fc1", np.float16, 4))

    def debug_enc_layer(self, layer: int, x_in, *, stages: bool = False):
        """Encoder layer `layer` on the residual x_in float32 [B, 1536, d] -> (x_out float32 [B, 1536, d], stages,
        plans).  stages (with stages=True, else None): the output of every launch, name -> array [B, 1536, width]
        (xn1, qkv, ctx, x_o after the o-projection, xn2, fc1), and vt [B, H, 64, 1536].  plans: {"qkv" | "o" | "fc1" |
        "fc2": (BN, multicast, K splits, grid)}."""
        dm = self.dims()
        d, H = dm["d_model"], dm["n_heads"]
        x_in = np.ascontiguousarray(x_in, np.float32)
        if x_in.ndim != 3 or x_in.shape[1:] != (1536, d):
            raise ValueError(f"x_in must be [B, 1536, {d}]")
        B = x_in.shape[0]
        md = B * 1536 * d
        x_out = np.zeros_like(x_in)
        buf = np.zeros(26 * md, np.uint8) if stages else None
        plan = np.zeros(16, np.int32)
        check(lib().wisb_debug_enc_layer(self._h, int(layer), B, ptr(x_in), ptr(x_out), ptr(buf), ptr(plan)))
        plans = {k: tuple(int(v) for v in plan[4 * i: 4 * i + 4]) for i, k in enumerate(("qkv", "o", "fc1", "fc2"))}
        if not stages:
            return x_out, None, plans
        out, at = {}, 0
        for name, dt, w in self.ENC_STAGES:
            n = np.dtype(dt).itemsize * w * md
            a = buf[at: at + n].view(dt)
            out[name] = a.reshape(B, H, 64, 1536) if name == "vt" else a.reshape(B, 1536, w * d)
            at += n
        return x_out, out, plans

    def debug_forced_logits(self, mel: np.ndarray, tokens) -> np.ndarray:
        mel = np.ascontiguousarray(mel, np.float32)
        tokens = np.ascontiguousarray(tokens, np.int32)
        out = np.zeros((tokens.shape[0], self.dims()["n_vocab"]), np.float32)
        check(lib().wisb_debug_forced_logits(self._h, ptr(mel), ptr(tokens), tokens.shape[0], ptr(out)))
        return out


def buffer_alloc(device: int, nbytes: int) -> int:
    """wisb_buffer_alloc: `nbytes` of device memory on GPU `device`, owned by no handle -> its address"""
    p = C.c_void_p()
    check(lib().wisb_buffer_alloc(int(device), int(nbytes), C.byref(p)))
    return p.value


def buffer_free(addr: int):
    check(lib().wisb_buffer_free(C.c_void_p(addr)))


def buffer_to_host(addr: int, out: np.ndarray):
    """the first out.nbytes bytes of buffer `addr` -> out (a C-contiguous host array)"""
    if not out.flags["C_CONTIGUOUS"]:
        raise ValueError("out must be C-contiguous")
    check(lib().wisb_buffer_to_host(C.c_void_p(addr), ptr(out), out.nbytes))
    return out


def flac_decode(data: bytes):
    """FLAC stream -> (int32 ndarray [n_frames, channels], sample_rate, bits_per_sample, md5 bytes).  Host code only."""
    l = lib()
    buf = np.frombuffer(data, np.uint8)
    sr, ch, bps, n = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int64()
    md5 = (C.c_uint8 * 16)()
    if l.wisb_flac_info(buf.ctypes.data, buf.size, C.byref(sr), C.byref(ch), C.byref(bps), C.byref(n), md5):
        raise ValueError("FLAC: " + l.wisb_flac_last_error().decode())
    # STREAMINFO is untrusted input: a frame is >= 9 bytes and carries <= 65535 samples per channel, so the stream
    # cannot hold more inter-channel samples than that, whatever the header claims (and 2^30 samples is the hard cap)
    bound = (buf.size // 9 + 1) * 65535
    if n.value < 0 or n.value > bound or n.value * max(ch.value, 1) > (1 << 30):
        raise ValueError(f"FLAC: STREAMINFO announces {n.value} samples, impossible for a {buf.size}-byte stream")
    out = np.zeros((n.value, ch.value), np.int32)
    got = C.c_int64()
    if l.wisb_flac_decode(buf.ctypes.data, buf.size, out.ctypes.data, n.value, C.byref(got)):
        raise ValueError("FLAC: " + l.wisb_flac_last_error().decode())
    return out[: got.value], sr.value, bps.value, bytes(md5)
