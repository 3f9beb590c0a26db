"""CPU tests of wisb_generate_options: the ctypes mirror's layout and defaults, and what Handle.generate /
Handle.generate_sample write into the struct for every kind of option (the engine is replaced by a recorder)."""
import ctypes
import os
import re

import numpy as np
import pytest

from willow_inference_server_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EOT = 50257
DEFAULTS = dict(beam_size=5, patience=1.0, length_penalty=1.0, max_length=448, timestamps=0,
                max_initial_timestamp_index=50, repetition_penalty=1.0, no_repeat_ngram_size=0, num_hypotheses=1,
                sampling_topk=1, sampling_temperature=1.0, n_extra=0, extra_suppress=None, max_length_per_window=None,
                beam_per_window=None, patience_per_window=None, length_penalty_per_window=None, seeds=None)
ARRAYS = {"extra_suppress": ctypes.c_int32, "max_length_per_window": ctypes.c_int32, "beam_per_window": ctypes.c_int32,
          "patience_per_window": ctypes.c_float, "length_penalty_per_window": ctypes.c_float, "seeds": ctypes.c_uint64}


def read_options(opt, B):
    """the fields of a GenerateOptions, arrays read back through their addresses as lists"""
    out = {}
    for name, _ in opt._fields_:
        v = getattr(opt, name)
        if name in ARRAYS and v is not None:
            n = opt.n_extra if name == "extra_suppress" else B
            v = [x.item() for x in np.ctypeslib.as_array((ARRAYS[name] * n).from_address(v))]
        out[name] = v
    return out


def test_layout_and_defaults():
    opt = _lib.GenerateOptions()
    assert _lib.lib().wisb_generate_options_init(ctypes.byref(opt)) == 0
    assert opt.struct_size == ctypes.sizeof(_lib.GenerateOptions)
    got = read_options(opt, 0)
    assert got.pop("struct_size") == opt.struct_size
    assert got == DEFAULTS
    assert _lib.lib().wisb_generate_options_init(None) == 1


class Recorder:
    """lib() whose wisb_generate records the options it receives (the initialiser is the library's own)"""

    def __init__(self, real):
        self.real, self.calls = real, []

    def wisb_generate_options_init(self, opt):
        return self.real.wisb_generate_options_init(opt)

    def wisb_generate(self, h, mel, B, prompts, prompt_len, opt, ids, stride, lens, scores):
        rec = read_options(opt._obj, B)
        assert rec.pop("struct_size") == ctypes.sizeof(_lib.GenerateOptions)
        self.calls.append(rec)
        return 0


@pytest.fixture
def recorder(monkeypatch):
    rec = Recorder(_lib.lib())
    monkeypatch.setattr(_lib, "lib", lambda: rec)
    return rec


def f32(x):
    return float(np.float32(x))


P2 = [[50258, 50259, 50359, 50363]] * 2
# Handle.generate's arguments -> the options the engine must see: what the entry point Handle.generate picked for
# that kind of option forwarded to the engine.  (Plain calls once went through an entry point that forwarded
# max_initial_timestamp_index 0; with timestamps off the engine does not read it.)
GENERATE_CASES = [
    # scalar options, bench.py's positional form
    ((None, P2, 5, 1.0, 1.0, 448, [EOT]), {}, dict(n_extra=1, extra_suppress=[EOT])),
    ((None, P2, 3, 2.0, 0.5, 200), {}, dict(beam_size=3, patience=2.0, length_penalty=0.5, max_length=200)),
    # per-window max_length
    ((None, P2, 1), dict(max_length=[100, 448]), dict(beam_size=1, max_length=448, max_length_per_window=[100, 448])),
    # timestamps, and an initial timestamp index off its default
    ((None, [[50258, 50259, 50359]] * 2, 5), dict(timestamps=True), dict(timestamps=1)),
    ((None, P2, 5), dict(max_initial_timestamp_index=7), dict(max_initial_timestamp_index=7)),
    ((None, [[50258, 50259, 50359]] * 2, 2), dict(timestamps=True, max_initial_timestamp_index=0),
     dict(beam_size=2, timestamps=1, max_initial_timestamp_index=0)),
    # the history processors
    ((None, P2, 5), dict(repetition_penalty=1.3, no_repeat_ngram_size=3),
     dict(repetition_penalty=f32(1.3), no_repeat_ngram_size=3)),
    ((None, P2, 5), dict(no_repeat_ngram_size=2, timestamps=False, max_length=[300, 20]),
     dict(no_repeat_ngram_size=2, max_length=300, max_length_per_window=[300, 20])),
    # per-window beam, patience and length penalty: a scalar given per window stands in as 1
    ((None, P2, [1, 5]), {}, dict(beam_size=1, beam_per_window=[1, 5])),
    ((None, P2, 4, [1.5, 2.0], 0.7), dict(repetition_penalty=1.1),
     dict(beam_size=4, patience=1.0, patience_per_window=[1.5, 2.0], length_penalty=f32(0.7),
          repetition_penalty=f32(1.1))),
    ((None, P2, [2, 3], 1.5, [0.25, 1.0]), dict(max_length=[64, 128], timestamps=False),
     dict(beam_size=1, beam_per_window=[2, 3], patience=1.5, length_penalty=1.0, length_penalty_per_window=[0.25, 1.0],
          max_length=128, max_length_per_window=[64, 128])),
]


@pytest.mark.parametrize("args, kw, want", GENERATE_CASES)
def test_generate_writes_the_options(recorder, args, kw, want):
    ids, scores = _lib.Handle(None).generate(*args, **kw, B=2)
    assert len(ids) == len(scores) == 2
    assert recorder.calls == [{**DEFAULTS, **want}]


def test_generate_sample_writes_the_options(recorder):
    seeds = np.asarray([7, 2 ** 64 - 1], np.uint64)
    ids, scores = _lib.Handle(None).generate_sample(None, P2, 3, 0, 0.7, seeds, 0.9, [100, 200], [EOT], B=2,
                                                    timestamps=False, repetition_penalty=1.2, no_repeat_ngram_size=4)
    assert len(ids) == len(scores) == 2 and all(len(i) == 3 for i in ids)
    want = dict(beam_size=1, patience=1.0, num_hypotheses=3, sampling_topk=0, sampling_temperature=f32(0.7),
                seeds=[7, 2 ** 64 - 1], length_penalty=f32(0.9), max_length=200, max_length_per_window=[100, 200],
                n_extra=1, extra_suppress=[EOT], repetition_penalty=f32(1.2), no_repeat_ngram_size=4)
    assert recorder.calls == [{**DEFAULTS, **want}]
    _lib.Handle(None).generate_sample(None, P2, 1, 5, 1.0, seeds, B=2)
    assert recorder.calls[1] == {**DEFAULTS, **dict(beam_size=1, sampling_topk=5, seeds=[7, 2 ** 64 - 1])}


def test_argument_errors_before_the_call(recorder):
    h = _lib.Handle(None)
    with pytest.raises(ValueError, match="one prompt per feature window"):
        h.generate(None, P2, 5, B=3)
    with pytest.raises(ValueError, match="beam_size"):
        h.generate(None, P2, [5, 5, 5], B=2)
    with pytest.raises(ValueError, match="max_length"):
        h.generate(None, P2, 5, max_length=[448], B=2)
    with pytest.raises(ValueError, match="seeds"):
        h.generate_sample(None, P2, 2, 0, 1.0, np.asarray([1], np.uint64), B=2)
    with pytest.raises(ValueError, match="seeds"):
        h.generate_sample(None, P2, 2, 0, 1.0, np.asarray([1, 2], np.int64), B=2)
    assert recorder.calls == []


def test_header_declares_one_generate_and_one_search_step():
    hdr = open(os.path.join(ROOT, "include", "wisb200.h")).read()
    declared = set(re.findall(r"\b(wisb_[a-z_0-9]+)\s*\(", hdr))
    assert sorted(n for n in declared if n.startswith("wisb_generate")) == ["wisb_generate", "wisb_generate_options_init"]
    assert [n for n in declared if n.startswith("wisb_debug_search_step")] == ["wisb_debug_search_step"]
