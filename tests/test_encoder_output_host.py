"""CPU tests of Whisper.encode and of encoder outputs passed to generate / detect_language / align: shape routing, the
ValueErrors, the replica each part runs on, StorageView's device form and the C ABI entries (fake handles; no GPU)."""
import ctypes
import os
import re

import numpy as np
import pytest

from willow_inference_server_b200 import _lib, models
from willow_inference_server_b200.batcher import TranscribeBatcher
from willow_inference_server_b200.models import StorageView

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 384
P = [50258, 50259, 50359, 50363]


class FakeHandle:
    """records what Whisper asks of one replica"""

    def __init__(self, d=D, n_mels=80):
        self.d, self.n_mels, self.calls = d, n_mels, []

    def set_option(self, k, v):
        pass

    def dims(self):
        return {"d_model": self.d, "n_vocab": 51865, "n_langs": 99, "n_mels": self.n_mels, "no_timestamps": 50363,
                "n_text_ctx": 448, "lang_first": 50259}

    def load_encoder_output(self, enc, on_device=False, B=None, dtype=np.float16):
        if on_device:
            self.calls.append(("load_device", enc, B, np.dtype(dtype).name))
        else:
            self.calls.append(("load", enc.shape[0], enc.dtype.name, float(enc.reshape(-1)[0])))

    def _rows(self, name, mel, B):
        self.calls.append((name, "mel" if mel is not None else None, mel.shape[0] if mel is not None else B))
        return mel.shape[0] if mel is not None else B

    def generate(self, mel, prompts, *args, B=None, **kw):
        n = self._rows("generate", mel, B)
        assert len(prompts) == n
        return [[7]] * n, [0.5] * n

    def detect_language(self, mel, B=None):
        n = self._rows("detect_language", mel, B)
        return np.tile(np.arange(50259, 50358, dtype=np.int32), (n, 1)), np.full((n, 99), 0.01, np.float32)

    def align(self, mel, start, text, num_frames, width=7, B=None):
        n = self._rows("align", mel, B)
        assert len(text) == n == len(num_frames)
        return [np.zeros((1, 2), np.int32)] * n, [[0.5]] * n

    def encode(self, mel, out=None, on_device=False):
        self.calls.append(("encode", mel.shape[0], on_device))
        if not on_device:
            out[...] = mel[:, :1, :1]  # window b's first feature, so the caller can tell which rows came back where
        return out


@pytest.fixture
def fake_buffers(monkeypatch):
    """_lib's device buffers as host arrays (address -> (device, bytes))"""
    mem, nxt = {}, [0x1000]

    def alloc(device, nbytes):
        addr = nxt[0]
        nxt[0] += 1 << 20
        mem[addr] = (device, np.arange(nbytes, dtype=np.uint8))
        return addr

    def free(addr):
        del mem[addr]

    def to_host(addr, out):
        out.view(np.uint8).reshape(-1)[:] = mem[addr][1][: out.nbytes]
        return out

    monkeypatch.setattr(_lib, "buffer_alloc", alloc)
    monkeypatch.setattr(_lib, "buffer_free", free)
    monkeypatch.setattr(_lib, "buffer_to_host", to_host)
    return mem


def feats(n, tag=0.0):
    a = np.zeros((n, 80, 3000), np.float32)
    a[:, 0, 0] = tag + np.arange(n)
    return a


def enc_out(n, dtype=np.float16, d=D):
    a = np.zeros((n, 1500, d), dtype)
    a[:, 0, 0] = np.arange(n)
    return a


# ------------------------------------------------------------------------------------------------ routing and errors
def test_shape_routing():
    h = FakeHandle()
    m = models.Whisper(None, device="cuda", _handles=[h])
    m.generate(StorageView.from_array(feats(2)), [P] * 2)
    assert h.calls == [("generate", "mel", 2)]
    for dt in (np.float16, np.float32):
        for x in (enc_out(3, dt), StorageView.from_array(enc_out(3, dt))):
            h.calls.clear()
            res = m.generate(x, [P] * 3, return_scores=True)
            assert [r.sequences_ids for r in res] == [[[7]]] * 3 and res[0].scores == [0.5]
            assert h.calls == [("load", 3, np.dtype(dt).name, 0.0), ("generate", None, 3)]
            h.calls.clear()
            assert len(m.detect_language(x)) == 3
            assert h.calls == [("load", 3, np.dtype(dt).name, 0.0), ("detect_language", None, 3)]
            h.calls.clear()
            assert len(m.align(x, P[:3], [[1, 2]] * 3, 3000)) == 3
            assert h.calls == [("load", 3, np.dtype(dt).name, 0.0), ("align", None, 3)]
    # the no-speech probability is still accepted and reported as 0.0
    assert m.generate(enc_out(1), [P], return_no_speech_prob=True)[0].no_speech_prob == 0.0


def test_value_errors(fake_buffers):
    h = FakeHandle()
    m = models.Whisper(None, device="cuda", _handles=[h])
    bad_enc = [np.zeros((1, 1500, D + 1), np.float16), np.zeros((1, 1500, 128), np.float32),
               np.zeros((1, 1500, D), np.float64), np.zeros((1, 1500, D), np.int16)]
    for x in bad_enc:
        for call in (lambda: m.generate(x, [P]), lambda: m.detect_language(x), lambda: m.align(x, P[:3], [[1]], 3000)):
            with pytest.raises(ValueError, match="encoder output"):
                call()
    for x in (np.zeros((1, 81, 3000), np.float32), np.zeros((1, 1499, D), np.float16), np.zeros((1, 80, 3000), np.float16),
              np.zeros((1, 80, 2999), np.float32), np.zeros((1500, D), np.float16)):
        with pytest.raises(ValueError, match=r"features must be float32 \[n, 80, 3000\]"):
            m.generate(x, [P])
    with pytest.raises(ValueError, match="prompts"):
        m.generate(enc_out(2), [P])
    with pytest.raises(ValueError, match="text token lists"):
        m.align(enc_out(2), P[:3], [[1]], 3000)
    # a device view on a GPU without a replica, or of another model width
    with pytest.raises(ValueError, match="no replica"):
        m.generate(StorageView._empty_on_device(1, (1, 1500, D)), [P])
    with pytest.raises(ValueError, match="encoder output"):
        m.detect_language(StorageView._empty_on_device(0, (1, 1500, 128)))
    assert not h.calls
    # a 128-bin model keeps naming 128 for features; encode takes features only
    v3 = models.Whisper(None, device="cuda", _handles=[FakeHandle(n_mels=128)])
    with pytest.raises(ValueError, match="128"):
        v3.generate(feats(1), [P])
    with pytest.raises(ValueError, match="features"):
        m.encode(enc_out(1))
    # StorageView: float16 accepted, float64 still refused; the batcher stays features-only
    assert StorageView.from_array(enc_out(1)).shape == [1, 1500, D]
    with pytest.raises(ValueError):
        StorageView.from_array(np.zeros((1, 1500, D), np.float64))
    with TranscribeBatcher(m, max_batch=4, max_wait_ms=1) as b:
        with pytest.raises(ValueError):
            b.submit(enc_out(1), P)


# ------------------------------------------------------------------------------------------------ replicas
def test_replica_choice(fake_buffers):
    h0, h1 = FakeHandle(), FakeHandle()
    m = models.Whisper(None, device="cuda", device_index=[0, 1], _handles=[h0, h1])
    # a host encoder output splits across the replicas like features
    m.generate(enc_out(4), [P] * 4)
    assert h0.calls == [("load", 2, "float16", 0.0), ("generate", None, 2)]
    assert h1.calls == [("load", 2, "float16", 2.0), ("generate", None, 2)]
    # ... and one window goes round robin
    for h in (h0, h1):
        h.calls.clear()
    m.detect_language(enc_out(1))
    m.detect_language(enc_out(1))
    assert len(h0.calls) == len(h1.calls) == 2
    # a device output runs whole on the replica on its GPU
    for h in (h0, h1):
        h.calls.clear()
    sv = StorageView._empty_on_device(1, (4, 1500, D))
    m.align(sv, P[:3], [[1]] * 4, 3000)
    assert h0.calls == [] and h1.calls == [("load_device", sv._buf, 4, "float16"), ("align", None, 4)]
    # with the encoder cache on, the crc routing applies to features only
    mc = models.Whisper(None, device="cuda", device_index=[0, 1], _handles=[h0, h1], reuse_encoder=True)
    for h in (h0, h1):
        h.calls.clear()
    for _ in range(2):
        mc.generate(feats(1, 5.0), [P])
    assert len(h0.calls) + len(h1.calls) == 2 and (h0.calls == [] or h1.calls == [])
    for h in (h0, h1):
        h.calls.clear()
    for _ in range(2):
        mc.generate(enc_out(1), [P])
    assert len(h0.calls) == len(h1.calls) == 2


def test_encode_replicas(fake_buffers):
    h0, h1 = FakeHandle(), FakeHandle()
    m = models.Whisper(None, device="cuda", device_index=[0, 1], _handles=[h0, h1])
    x = feats(4, 10.0)
    out = m.encode(StorageView.from_array(x), to_cpu=True)
    assert out.device == "cpu" and out.shape == [4, 1500, D] and out.array.dtype == np.float16
    assert out.array[:, 0, 0].tolist() == [10, 11, 12, 13]
    assert h0.calls == [("encode", 2, False)] and h1.calls == [("encode", 2, False)]
    # on the device: one replica runs the whole call, round robin
    for h in (h0, h1):
        h.calls.clear()
    a = m.encode(x)
    b = m.encode(x)
    assert (a.device, a.shape, b.device) == ("cuda", [4, 1500, D], "cuda")
    assert {a.device_index, b.device_index} == {0, 1}
    assert h0.calls == [("encode", 4, True)] and h1.calls == [("encode", 4, True)]
    assert len(fake_buffers) == 2
    del a, b
    assert not fake_buffers  # a view frees its buffer


def test_storage_view_to_device(fake_buffers):
    host = StorageView.from_array(enc_out(2))
    assert (host.device, host.device_index) == ("cpu", 0) and host.to_device("cpu") is host
    sv = StorageView._empty_on_device(1, (2, 1500, D))
    assert (sv.device, sv.device_index, sv.shape) == ("cuda", 1, [2, 1500, D])
    back = sv.to_device("cpu")
    assert back.device == "cpu" and back.shape == [2, 1500, D] and back.array.dtype == np.float16
    want = np.arange(2 * 1500 * D * 2, dtype=np.uint8).view(np.float16).reshape(2, 1500, D)
    assert np.array_equal(back.array.view(np.uint16), want.view(np.uint16))
    with pytest.raises(ValueError):
        sv.to_device("cuda")


# ------------------------------------------------------------------------------------------------ C ABI
def test_abi_table_has_the_encoder_output_entries():
    hdr = re.sub(r"/\*.*?\*/", " ", open(os.path.join(ROOT, "include", "wisb200.h")).read(), flags=re.S)
    protos = dict(re.findall(r"\b(wisb_[a-z_0-9]+)\s*\(([^)]*)\)\s*;", hdr))
    want = {"wisb_buffer_alloc": 3, "wisb_buffer_free": 1, "wisb_buffer_to_host": 3, "wisb_encode": 5,
            "wisb_load_encoder_output": 5}
    for name, n in want.items():
        assert protos[name].count(",") + 1 == n == len(_lib._SIGS[name][1]), name
        assert name in _lib.EXPORTS
    assert hasattr(ctypes.CDLL(_lib.LIB_PATH), "wisb_load_encoder_output")


def test_buffer_entries_refuse_foreign_pointers():
    lib = _lib.lib()
    assert lib.wisb_buffer_free(None) == 0
    bogus = ctypes.c_void_p(0xDEAD000)
    assert lib.wisb_buffer_free(bogus) == 1
    assert lib.wisb_buffer_to_host(bogus, None, 0) == 1
    with pytest.raises(ValueError, match="not a live"):
        _lib.buffer_free(0xDEAD000)
    import torch
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError):
            _lib.buffer_alloc(0, 1024)
