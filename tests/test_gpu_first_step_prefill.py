"""GPU: the first generated token read from the prompt prefill pass.

When every prompt position of every window of a call fits one prefill pass (persistent pass: windows x prompt length
<= 8 and a prompt of <= 8 tokens; batched pass: a prompt of at most the pass's positions per window), that pass also
computes the logits of the last prompt position, and the first search step reads window u's logits from its row
u * P + P - 1 instead of running a decoding pass of its own.

  * Pass level (Handle.debug_dec_pass, warp-MMA and SIMT, d = 128 and 1280): one prefill pass of P positions with
    logits against a prefill pass of P - 1 positions followed by a decoding step of B rows at position P - 1 whose
    indirection points at the window's prefix slot.  The merged row's logits equal every one of the step's B rows bit
    for bit, and so do the K/V cells at (slot u * B, position P - 1) in every layer.  Every cache cell neither run should
    read holds NaN.
  * End to end on the peaked synthetic model: greedy, beam 5, per-window beams (with dead rows), timestamps, the history
    processors and best-of-5 sampling, on the warp-MMA and SIMT persistent passes (NaN in every self-attention cache
    cell before the call) and on the batched pass (16 windows, after a call on other windows with another prompt length
    left unrelated finite values in its cache).  Scores are finite and the transcripts are the oracle's on its robust
    cases: a row that read a K/V cell of the last prompt position the merged pass did not write would show here."""
import functools

import numpy as np
import pytest

from tests.gpu_common import PROMPT, mel_inputs
from tests.test_gpu_dec_pass import NAN16, engine_model
from tests.test_gpu_mixed import TS_PROMPTS, check_call, pair
from tests.test_gpu_kernels import bits

pytestmark = pytest.mark.gpu

SHAPES = [(1, 4, 5), (2, 4, 4), (1, 8, 1), (2, 3, 2), (4, 2, 2), (2, 1, 3)]   # (windows, prompt length, beam)


def nan_cache(m):
    return np.full((m.L, 8, 448, m.d), NAN16, np.uint16).view(np.float16)


@functools.lru_cache(maxsize=None)
def pass_inputs(d, n_utt, P):
    rng = np.random.default_rng([7, d, n_utt, P])
    prompts = rng.integers(3, 51865, (n_utt, P)).astype(np.int32)
    prompts[0, 0] = 1   # a token row with a common offset (tests/test_gpu_dec_pass.py)
    enc = rng.standard_normal((n_utt, 1536, d)).astype(np.float16)
    return prompts, enc


@pytest.mark.parametrize("d", [128, 1280])
@pytest.mark.parametrize("impl", [1, 0])
def test_merged_prefill_pass_equals_prefix_pass_plus_step(d, impl):
    dims, m, h = engine_model(d, d // 64, 51865)
    Vp = dims.n_vocab_pad
    for n_utt, P, B in SHAPES:
        prompts, enc = pass_inputs(d, n_utt, P)
        x = np.zeros((8, d), np.float32)
        # merged: prompt positions 0 .. P - 1 of every window in one pass, with logits
        kc_m, vc_m, lg_m = nan_cache(m), nan_cache(m), np.zeros((8, Vp), np.float32)
        h.debug_dec_pass(impl, prompts.reshape(-1), enc, kc_m, vc_m, x.copy(), lg_m, n_utt=n_utt, beam=B, pf_len=P)
        # today's sequence: positions 0 .. P - 2 without logits, then a step of B rows per window at position P - 1
        kc_s, vc_s, lg_s = nan_cache(m), nan_cache(m), np.zeros((8, Vp), np.float32)
        if P > 1:
            h.debug_dec_pass(impl, prompts[:, : P - 1].reshape(-1), enc, kc_s, vc_s, x.copy(), lg_s, n_utt=n_utt,
                             beam=B, pf_len=P - 1, with_logits=False)
        ind = np.repeat(np.arange(n_utt) * B, B)[:, None].repeat(448, 1).astype(np.int32)
        h.debug_dec_pass(impl, np.repeat(prompts[:, P - 1], B), enc, kc_s, vc_s, x.copy(), lg_s, n_utt=n_utt, beam=B,
                         pos=P - 1, flip=0, indir0=ind, indir1=ind)
        tag = (d, impl, n_utt, P, B)
        for u in range(n_utt):
            merged = bits(lg_m[u * P + P - 1, : dims.n_vocab])
            assert np.isfinite(lg_m[u * P + P - 1, : dims.n_vocab]).all(), tag
            for k in range(B):
                assert np.array_equal(merged, bits(lg_s[u * B + k, : dims.n_vocab])), (tag, u, k)
            for got, want in ((kc_m, kc_s), (vc_m, vc_s)):
                cell_m, cell_s = got[:, u * B, P - 1], want[:, u * B, P - 1]
                assert np.isfinite(cell_m).all(), tag
                assert np.array_equal(bits(cell_m), bits(cell_s)), (tag, u)


# ------------------------------------------------------------------------------------------------ end to end
PROC = (("repetition_penalty", 1.3), ("no_repeat_ngram_size", 3))
# mode -> (beams cycled over the windows, timestamp prompts, processors)
MODES = {"greedy": ((1,), False, ()), "beam5": ((5,), False, ()), "mixed": ((1, 3, 2, 1), False, ()),
         "timestamps": ((2, 1, 3), True, ()), "history": ((3, 1, 2), False, PROC)}
PATHS = ["warp_mma", "simt", "batched16"]


def window_options(idx, beams, ts):
    src = TS_PROMPTS if ts else [PROMPT]
    prompts = np.asarray([src[i % len(src)] for i in idx], np.int32)
    b = np.asarray([beams[j % len(beams)] for j in range(len(idx))], np.int32)
    return prompts, b, np.ones(len(idx), np.float32), np.ones(len(idx), np.float32)


def poison(h, dims, path):
    """persistent pass: NaN in every self-attention cache cell (debug_dec_pass uploads the whole cache; its one-row
    prefill rewrites slot 0, position 0 only, which every call writes before reading).  Batched pass: a call on other
    windows with a 5-token prompt leaves unrelated finite K/V in its cache."""
    if path == "batched16":
        mel = np.ascontiguousarray(mel_inputs(16)[::-1])
        h.generate(mel, np.asarray([PROMPT + [440]] * 16, np.int32), beam_size=5, max_length=40)
        return
    L, d = dims.n_dec_layers, dims.d_model
    kc = np.full((L, 8, 448, d), NAN16, np.uint16).view(np.float16)
    h.debug_dec_pass(1, np.asarray([1], np.int32), np.zeros((1, 1536, d), np.float16), kc, kc.copy(),
                     np.zeros((8, d), np.float32), np.zeros((8, dims.n_vocab_pad), np.float32), n_utt=1, pf_len=1,
                     with_logits=False)


def calls(path, beams):
    """windows of each call: 16 on the batched pass; on the persistent pass 1 window, then 2 per call where their rows
    (windows x largest beam) and prompt positions fit 8"""
    if path == "batched16":
        return [np.arange(16)]
    n = 2 if 2 * max(beams) <= 8 else 1
    return [np.arange(0, 1)] + [np.arange(i, i + n) for i in range(1, 10, n)]


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("path", PATHS)
def test_first_step_from_the_prefill_pass(path, mode):
    dims, _, h = pair()
    beams, ts, proc = MODES[mode]
    h.set_option("mega_mma", 0 if path == "simt" else 1)
    try:
        n_robust = 0
        for idx in calls(path, beams):
            prompts, b, p, lp = window_options(idx, beams, ts)
            poison(h, dims, path)
            mel = np.ascontiguousarray(mel_inputs(16)[idx])
            got = h.generate(mel, prompts, beam_size=b, patience=p, length_penalty=lp, timestamps=ts, **dict(proc))
            assert np.isfinite(got[1]).all(), (path, mode, idx, got[1])
            n_robust += check_call(h, idx, prompts, b, p, lp, proc=proc, got=got)
        assert n_robust >= 2, (path, mode, n_robust)
    finally:
        h.set_option("mega_mma", 1)


@pytest.mark.parametrize("path", PATHS)
def test_first_step_from_the_prefill_pass_sampling(path):
    dims, _, h = pair()
    h.set_option("mega_mma", 0 if path == "simt" else 1)
    try:
        # best-of-5: 5 rows per window, every one live at the first step (1 window on the persistent pass)
        idx = np.arange(16) if path == "batched16" else np.arange(1)
        for topk in (0, 4):
            poison(h, dims, path)
            mel = np.ascontiguousarray(mel_inputs(16)[idx])
            prompts = np.asarray([PROMPT] * len(idx), np.int32)
            seeds = np.arange(100, 100 + len(idx), dtype=np.uint64)
            ids, scores = h.generate_sample(mel, prompts, 5, topk, 0.8, seeds, max_length=60)
            assert np.isfinite(np.asarray(scores)).all(), (path, topk, scores)
            assert all(len(s) > 0 for w in ids for s in w), (path, topk)
    finally:
        h.set_option("mega_mma", 1)
