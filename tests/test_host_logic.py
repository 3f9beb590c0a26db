"""CPU tests of the host-side mirror of the reference interface and of the C-ABI surface (no GPU compute)."""
import ctypes
import json
import os
import re

import numpy as np
import pytest

import willow_inference_server_b200 as ct2
from willow_inference_server_b200 import _lib, audio, weights as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_chunk_iter_matches_reference_golden(golden_dir):
    g = json.load(open(os.path.join(golden_dir, "host_logic.json")))
    for n, table in g["chunk_iter"].items():
        x = np.zeros(int(n), np.float32)
        got = [[int(c.shape[0]), int(s[0]), int(s[1]), int(s[2])] for c, s in audio.chunk_iter(x)]
        assert got == table, n


def test_lcs_matches_reference_golden(golden_dir):
    g = json.load(open(os.path.join(golden_dir, "host_logic.json")))
    for case in g["lcs"]:
        class Tok:
            all_special_ids = case["special"]
        merged = audio.find_longest_common_sequence([(s, (0, 0, 0)) for s in case["in"]], Tok())
        assert [int(v) for v in merged] == case["out"]


def test_lcs_longer_second_window_does_not_raise():
    class Tok:
        all_special_ids = [50257]
    out = audio.find_longest_common_sequence([([1, 2], 0), ([1, 2, 3, 4, 5], 0)], Tok())
    assert out.tolist()[:2] == [1, 2] and out.tolist()[-1] == 5


def test_pad_or_trim():
    x = np.arange(10, dtype=np.float32)
    assert audio.pad_or_trim(x, 4).tolist() == [0, 1, 2, 3]
    assert audio.pad_or_trim(x, 12).tolist() == list(range(10)) + [0, 0]
    assert audio.pad_or_trim(np.zeros(5, np.float32)).shape == (480000,)


def test_c_abi_v2_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "wisb200.h")).read()
    declared = sorted(set(re.findall(r"\b(wisb_[a-z_0-9]+)\s*\(", hdr)))
    assert declared, "no declarations found"
    assert os.path.exists(_lib.LIB_PATH), "libwisb200.so is not built (run __graft_entry__.build())"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/wisb200.h but not exported"
    assert sorted(_lib.EXPORTS) == declared  # the ctypes table binds exactly the header
    assert _lib.lib().wisb_abi_version() == 2
    # ... with the same number of parameters per entry point as the C prototypes
    flat = re.sub(r"/\*.*?\*/", " ", hdr, flags=re.S)
    for name, params in re.findall(r"\b(wisb_[a-z_0-9]+)\s*\(([^)]*)\)\s*;", flat):
        params = params.strip()
        n = 0 if params in ("", "void") else params.count(",") + 1
        assert n == len(_lib._SIGS[name][1]), (name, n, len(_lib._SIGS[name][1]))


def test_storage_view_and_argument_errors():
    with pytest.raises(ValueError):
        ct2.StorageView.from_array(np.zeros((1, 80, 3000), np.float64))
    sv = ct2.StorageView.from_array(np.zeros((2, 80, 3000), np.float32))
    assert sv.shape == [2, 80, 3000]
    with pytest.raises(ValueError):
        ct2.models.Whisper("/nonexistent", device="cpu")
    with pytest.raises(ValueError):
        ct2.get_supported_compute_types("cpu")
    assert ct2.get_supported_compute_types("cuda") == {"float16"}


def test_blob_roundtrip(tmp_path):
    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=1, n_dec_layers=1)
    t = W.synth_engine_tensors(dims, seed=3)
    path = str(tmp_path / "model.wisb")
    n = W.write_blob(path, dims, t)
    assert n == os.path.getsize(path) and n % 256 == 0
    d2, t2 = W.read_blob(path)
    assert d2.d_model == 128 and d2.n_vocab == 51865 and d2.suppress_ids == sorted(set(dims.suppress_ids))
    assert set(t2) == set(t)
    for k in t:
        assert t2[k].dtype == t[k].dtype and np.array_equal(t2[k], t[k]), k
    assert t["dec.tok_emb"].shape == (51968, 128) and not t["dec.tok_emb"][51865:].any()
    assert t["dec.crosskv.w"].shape == (256, 128) and t["enc.conv2.w"].shape == (128, 384)


def test_no_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _lib.Handle.frontend(0)
    with pytest.raises(RuntimeError):
        audio.log_mel_spectrogram(np.zeros(16000, np.float32))


def test_chunk_table_is_chunk_iter_as_index_arithmetic(golden_dir):
    g = json.load(open(os.path.join(golden_dir, "host_logic.json")))
    totals = [int(n) for n in g["chunk_iter"]] + [1, 63999, 64001, 352000, 352001, 576000, 224000 * 3 + 5]
    for total in totals:
        x = np.arange(total, dtype=np.float32)
        want = [(int(c[0]), c.shape[0], s) for c, s in audio.chunk_iter(x)]
        offs, lens, strides = audio.chunk_table(total)
        assert [(int(o), int(n), st) for o, n, st in zip(offs, lens, strides)] == want, total


def test_transcribe_long_orchestration(monkeypatch):
    # windows -> one batched generate -> LCS merge, with a fake front end and a fake engine (host logic only)
    from willow_inference_server_b200.models import WhisperGenerationResult

    class Tok:
        all_special_ids = [50257, 50258]

    windows = [[1, 2, 3, 4, 5, 6, 50257], [4, 5, 6, 7, 8, 9], [8, 9, 10, 11]]
    calls = []

    class Engine:
        def generate(self, features, prompts, **kw):
            calls.append((features.array.shape[0], prompts, kw))
            start = int(features.array[0, 0, 0])
            return [WhisperGenerationResult([windows[start + i]]) for i in range(features.array.shape[0])]

    def fake_chunks(audio_, handle=None):
        mel = np.zeros((3, 80, 3000), np.float32)
        mel[:, 0, 0] = np.arange(3)
        return mel, [(352000, 0, 64000), (352000, 64000, 64000), (100000, 64000, 0)]

    monkeypatch.setattr(audio, "log_mel_chunks", fake_chunks)
    out = audio.transcribe_long(Engine(), np.zeros(800000, np.float32), [50258, 50259, 50359, 50363], Tok(), beam_size=3)
    assert out.tolist() == list(range(1, 12))                     # the SURVEY 8c(iii) stitching example
    assert len(calls) == 1 and calls[0][0] == 3 and calls[0][2] == {"beam_size": 3}
    calls.clear()
    out = audio.transcribe_long(Engine(), np.zeros(800000, np.float32), [50258], Tok(), max_windows_per_call=2)
    assert out.tolist() == list(range(1, 12)) and [c[0] for c in calls] == [2, 1]
    # <= 30 s: ONE zero-padded window and no windowing at all, as the reference does (main.py:587-617) -- 25 s of audio
    # would otherwise become two 22-s windows plus a stitch
    calls.clear()
    monkeypatch.setattr(audio, "log_mel_window", lambda a, handle=None: fake_chunks(a)[0][:1])
    monkeypatch.setattr(audio, "log_mel_chunks", lambda a, handle=None: (_ for _ in ()).throw(AssertionError("windowed a short utterance")))
    assert audio.transcribe_long(Engine(), np.zeros(400000, np.float32), [50258], Tok()).tolist() == [1, 2, 3, 4, 5, 6]
    assert [c[0] for c in calls] == [1]
