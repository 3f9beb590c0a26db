"""GPU: one generate call whose windows differ in beam size, patience, length penalty and prompt (other language or task
token, same length) -- ``wisb_generate`` with per-window options, what ``batcher.TranscribeBatcher`` sends when it
coalesces such requests.

On the peaked, timestamp-scripted synthetic model at a tiny width, every window of a mixed call must return what its solo
call returns and what the oracle (``tests.proc_oracle.ProcOracle``: the CTranslate2 search, the timestamp rules and the
history processors) returns with that window's own options, on every robust case: the oracle's transcript is unchanged
under logit noise of the documented tolerance and, at beam > 1, every step's decision gap exceeds DECISION_GAP.  Scores
are within the batch-versus-solo tolerance of tests/test_gpu_whisper.py.  Each decoder path is covered: the warp-MMA and
the SIMT persistent passes (windows x largest beam <= 8) and the batched pass (16 windows)."""
import functools

import numpy as np
import pytest

from tests.gpu_common import LOGIT_TOL, PROMPT, RAMP, SCRIPT, mel_inputs, robust_cases
from tests.proc_oracle import ProcOracle
from willow_inference_server_b200 import _lib, models, weights as W

pytestmark = pytest.mark.gpu
TS_SCRIPT = (2, 5, 8)
DECISION_GAP = LOGIT_TOL / 4
SCORE_TOL = 5e-2
# same length, other language and / or task token: none of them could share a call before
PROMPTS = [PROMPT, [50258, 50260, 50359, 50363], [50258, 50259, 50358, 50363], [50258, 50262, 50358, 50363]]
TS_PROMPTS = [p[:3] for p in PROMPTS]
PATIENCE = (1.0, 0.5, 2.0, 1.25)
LENGTH_PENALTY = (1.0, 0.6, 0.0, 1.3, 1.0)


@functools.lru_cache(maxsize=1)
def pair():
    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=2)
    tensors = W.synth_engine_tensors(dims, seed=11, eot_ramp=RAMP, script=SCRIPT, ts_script=TS_SCRIPT)
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    return dims, ProcOracle.from_blob(buf), _lib.Handle.from_host(buf, 0)


def options(n, beams, ts=False):
    """Per-window (prompts, beams, patience, length penalties) of n windows."""
    b = np.asarray([beams[i % len(beams)] for i in range(n)], np.int32)
    p = np.asarray([PATIENCE[i % len(PATIENCE)] for i in range(n)], np.float32)
    lp = np.asarray([LENGTH_PENALTY[i % len(LENGTH_PENALTY)] for i in range(n)], np.float32)
    prompts = np.asarray([(TS_PROMPTS if ts else PROMPTS)[i % len(PROMPTS)] for i in range(n)], np.int32)
    return prompts, b, p, lp


@functools.lru_cache(maxsize=None)
def oracle_window(i, prompt, beam, patience, lp, max_length, proc):
    """(oracle ids, score, robust) of window i alone with these options"""
    _, oracle, _ = pair()
    mel = mel_inputs(16)[i : i + 1]
    kw = dict(patience=patience, length_penalty=lp, max_length=max_length, **dict(proc))
    res, robust = robust_cases(oracle, mel, [list(prompt)], beam, n_probe=2, **kw)
    ok = bool(robust)
    if ok and beam > 1:
        trace = []
        oracle.generate(mel, [list(prompt)], beam_size=beam, trace=trace, **kw)
        ok = min(trace[0][:-1]) > DECISION_GAP
    return res[0].sequences_ids[0], res[0].scores[0], ok


def check_call(h, idx, prompts, beams, pats, lps, *, max_length=448, proc=(), got=None):
    """The mixed call on windows idx (or its result `got`) == each window's solo call and the oracle on robust cases.
    -> number of robust cases"""
    mel = np.ascontiguousarray(mel_inputs(16)[idx])
    ml = max_length if np.isscalar(max_length) else np.asarray(max_length, np.int32)
    proc = tuple(proc) + (("timestamps", len(prompts[0]) == 3),)   # (the handle takes the mode; the model reads the prompt)
    if got is None:
        got = h.generate(mel, prompts, beam_size=beams, patience=pats, length_penalty=lps, max_length=ml, **dict(proc))
    n_robust = 0
    for j, i in enumerate(idx):
        mlj = int(max_length if np.isscalar(max_length) else max_length[j])
        want, want_sc, robust = oracle_window(int(i), tuple(int(t) for t in prompts[j]), int(beams[j]), float(pats[j]),
                                              float(lps[j]), mlj, tuple(p for p in proc if p[0] != "timestamps"))
        if not robust:
            continue
        solo = h.generate(mel[j : j + 1], prompts[j : j + 1], beam_size=int(beams[j]), patience=float(pats[j]),
                          length_penalty=float(lps[j]), max_length=mlj, **dict(proc))
        for where, ids, sc in (("mixed", got[0][j], got[1][j]), ("solo", solo[0][0], solo[1][0])):
            assert ids == want, (where, j, int(beams[j]), float(pats[j]), float(lps[j]))
            assert abs(sc - want_sc) < SCORE_TOL, (where, j, sc, want_sc)
        n_robust += 1
    return n_robust


@pytest.mark.parametrize("path", ["warp_mma", "simt"])
def test_persistent_passes(path):
    # 4 windows x largest beam 2 = 8 rows: one persistent pass per step; two calls cover 8 windows
    dims, _, h = pair()
    h.set_option("mega_mma", 1 if path == "warp_mma" else 0)
    try:
        n_robust = 0
        for idx in (np.arange(0, 4), np.arange(4, 8)):
            prompts, b, p, lp = options(4, (1, 2, 2, 1))
            p, lp = p[::-1].copy(), np.roll(lp, int(idx[0]))
            n_robust += check_call(h, idx, prompts, b, p, lp)
        assert n_robust >= 4, n_robust
    finally:
        h.set_option("mega_mma", 1)


def test_batched_pass_beams_1_2_3_5_8():
    dims, _, h = pair()
    idx = np.arange(16)
    prompts, b, p, lp = options(16, (1, 2, 3, 5, 8))
    got = h.generate(np.ascontiguousarray(mel_inputs(16)), prompts, beam_size=b, patience=p, length_penalty=lp,
                     timestamps=False)
    assert h.timing()["decode_steps"] < 60    # one shared pass per step, not one loop per window
    assert check_call(h, idx, prompts, b, p, lp, got=got) >= 4


def test_timestamp_mode():
    dims, _, h = pair()
    prompts, b, p, lp = options(16, (2, 1, 5, 3), ts=True)
    assert check_call(h, np.arange(16), prompts, b, p, lp) >= 4
    prompts, b, p, lp = options(4, (1, 2, 2, 1), ts=True)      # and on the persistent pass
    check_call(h, np.arange(8, 12), prompts, b, p, lp)
    got = h.generate(np.ascontiguousarray(mel_inputs(16)[:4]), prompts, beam_size=b, patience=p, length_penalty=lp,
                     timestamps=True)
    assert all(ids and ids[0] > dims.no_timestamps for ids in got[0])   # every transcript opens with a timestamp


def test_history_processors_and_per_window_max_length():
    dims, _, h = pair()
    prompts, b, p, lp = options(16, (3, 1, 8, 2))
    limits = [24, 40, 448, 30, 60, 16, 448, 36] * 2
    n = check_call(h, np.arange(16), prompts, b, p, lp, max_length=limits,
                   proc=(("repetition_penalty", 1.3), ("no_repeat_ngram_size", 3)))
    assert n >= 4, n


def test_encoder_output_input_and_the_model_surface():
    # models.Whisper.generate with per-window options, on features and on an encode() output, equals the handle call
    dims, _, h = pair()
    m = models.Whisper(None, device="cuda", _handles=[h])
    mel = np.ascontiguousarray(mel_inputs(16)[:6])
    prompts, b, p, lp = options(6, (5, 1, 3))
    want = h.generate(mel, prompts, beam_size=b, patience=p, length_penalty=lp)
    kw = dict(beam_size=list(map(int, b)), patience=list(map(float, p)), length_penalty=lp, return_scores=True)
    for src in (models.StorageView.from_array(mel), m.encode(models.StorageView.from_array(mel)),
                m.encode(models.StorageView.from_array(mel), to_cpu=True)):
        out = m.generate(src, prompts.tolist(), **kw)
        assert [o.sequences_ids[0] for o in out] == want[0]
        assert np.allclose([o.scores[0] for o in out], want[1], atol=1e-6)


def test_equal_options_per_window_equal_the_scalar_call():
    # a per-window list whose values agree runs the scalar search: bit-identical tokens and scores
    dims, _, h = pair()
    mel = np.ascontiguousarray(mel_inputs(16)[:6])
    for beam, n in ((5, 6), (2, 3)):
        prompts = np.asarray([PROMPT] * n, np.int32)
        a = h.generate(mel[:n], prompts, beam_size=beam, patience=1.5, length_penalty=0.7)
        c = h.generate(mel[:n], prompts, beam_size=[beam] * n, patience=[1.5] * n, length_penalty=[0.7] * n)
        assert a == c, beam


def test_huge_patience_never_finishes_by_count():
    # beam x patience far beyond any hypothesis count (and beyond int range) ends a window only at its length limit or
    # when its beams die out, as a large finite patience does
    dims, _, h = pair()
    mel = np.ascontiguousarray(mel_inputs(16)[:2])
    prompts = np.asarray([PROMPT] * 2, np.int32)
    ref = h.generate(mel, prompts, beam_size=[2, 3], patience=[1000.0, 1000.0], max_length=40)
    assert h.generate(mel, prompts, beam_size=[2, 3], patience=[1e10, 3e38], max_length=40) == ref
    assert h.generate(mel[:1], prompts[:1], beam_size=2, patience=1e10, max_length=40) == \
        h.generate(mel[:1], prompts[:1], beam_size=2, patience=1000.0, max_length=40)


def test_bad_per_window_options():
    dims, _, h = pair()
    mel = np.ascontiguousarray(mel_inputs(16)[:2])
    prompts = np.asarray([PROMPT] * 2, np.int32)
    for bad in (dict(beam_size=[1, 9]), dict(beam_size=[0, 2]), dict(beam_size=[1, 2, 3]), dict(patience=[1.0, 0.0]),
                dict(patience=[np.inf, 1.0]), dict(patience=[np.nan, 1.0]), dict(length_penalty=[1.0, np.inf]),
                dict(length_penalty=[np.nan, 1.0]), dict(length_penalty=[1.0]), dict(beam_size=[1.5, 2])):
        with pytest.raises(ValueError):
            h.generate(mel, prompts, **bad)
