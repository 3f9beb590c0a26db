"""GPU tests of the batched decoder pass (one pass over the decoder weights for every row of a batch of utterances;
csrc/decoder_batch.cu) -- the path main.py:676-693 takes when it feeds several windows per generate call,
and what BASELINE.json configs[2] / configs[3] (batch 64 / 512) measure.

  * teacher-forced logits of the batched pass vs the fp32 oracle (tolerance LOGIT_TOL), also with 2..8 positions as
    rows of one pass, for both cross-attention kernels
  * 16 utterances greedy with a 2- and a 4-token prompt: both cross-attention kernels equal the oracle on robust cases
  * B = 16, beam 5, mixed durations: every transcript identical to the B = 1 result (persistent SIMT pass) AND to the
    oracle on every robust case (tests/gpu_common.robust_cases)
  * per-utterance length limits in one shared pass == separate calls
  * row capacity smaller than the batch (groups) == one group
  * batch_rows = 1024 at beam 1: 520 windows in one shared pass equal the oracle on robust cases
"""
import numpy as np
import pytest

from tests.gpu_common import LOGIT_TOL, PROMPT, mel_inputs, model_pair, robust_cases
from willow_inference_server_b200 import models

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pair():
    return model_pair()


def test_batched_pass_forced_logits_match_oracle(pair):
    dims, oracle, h = pair
    mel = mel_inputs(4)[:1]
    toks = PROMPT + [100, 2000, 30000, 41000, 12, 50000, 7, 999, 4242]
    want = oracle.forced_logits(oracle.encode(mel)[0], toks).numpy()
    h.set_option("decoder_batch", 2)
    try:
        got = h.debug_forced_logits(mel, toks)
    finally:
        h.set_option("decoder_batch", 1)
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= LOGIT_TOL
    small = h.debug_forced_logits(mel, toks)  # the persistent SIMT pass on the same tokens
    assert np.abs(got - small).max() <= LOGIT_TOL


@pytest.mark.parametrize("beam", [5, 1])
def test_batch16_equals_single_and_oracle(pair, beam):
    dims, oracle, h = pair
    mel = mel_inputs(16)
    n = mel.shape[0]
    m = models.Whisper(None, device="cuda", _handles=[h])
    out = m.generate(models.StorageView.from_array(mel), [PROMPT] * n, beam_size=beam, return_scores=True)
    got = [o.sequences_ids[0] for o in out]
    assert m.timing()["decode_steps"] < 40  # ONE shared pass per step (about 20 passes), not 16 x 20
    res, robust = robust_cases(oracle, mel, [PROMPT] * n, beam, n_probe=2)
    assert len(robust) >= 10, f"only {len(robust)} of {n} oracle transcripts are robust decisions"
    for i in robust:
        assert got[i] == res[i].sequences_ids[0], (beam, i)
    # each utterance alone (<= 8 rows: the persistent SIMT pass) gives the same transcript as inside the batch
    for i in robust:
        solo = m.generate(models.StorageView.from_array(mel[i : i + 1]), [PROMPT], beam_size=beam)[0].sequences_ids[0]
        assert solo == got[i], (beam, i)
    assert len({tuple(g) for g in got}) >= 6
    # run-to-run determinism and batch-position invariance (utterance 3 moved to the front)
    again = [o.sequences_ids[0] for o in m.generate(models.StorageView.from_array(mel), [PROMPT] * n, beam_size=beam)]
    assert again == got
    perm = np.ascontiguousarray(np.concatenate([mel[3:4], mel[:3], mel[4:]]))
    moved = [o.sequences_ids[0] for o in m.generate(models.StorageView.from_array(perm), [PROMPT] * n, beam_size=beam)]
    assert moved[0] == got[3] and moved[1:4] == got[:3] and moved[4:] == got[4:]


def test_per_utterance_max_length_in_one_pass(pair):
    # requests with different length limits coalesced into ONE shared pass (max_length_per_window) decode exactly what
    # separate calls with those limits decode -- checked against the oracle on every robust case
    dims, oracle, h = pair
    mel = mel_inputs(6)
    limits = [16, 30, 60, 12, 24, 40]
    got, _ = h.generate(mel, [PROMPT] * 6, beam_size=5, max_length=np.asarray(limits, np.int32), extra_suppress=[dims.eot])
    n_checked = 0
    for i, ml in enumerate(limits):
        assert len(got[i]) == min(ml // 2, ml - 4)
        res, robust = robust_cases(oracle, mel[i : i + 1], [PROMPT], 5, n_probe=2, max_length=ml, suppress_tokens=(-1, dims.eot))
        if robust:
            assert got[i] == res[0].sequences_ids[0], i
            n_checked += 1
    assert n_checked >= 4
    # without the suppressed <|endoftext|>: hypotheses finish early, limits only cap the long ones
    got2, _ = h.generate(mel, [PROMPT] * 6, beam_size=5, max_length=np.asarray(limits, np.int32))
    assert all(len(g) <= min(ml // 2, ml - 4) for g, ml in zip(got2, limits))
    with pytest.raises(ValueError):
        h.generate(mel, [PROMPT] * 6, beam_size=5, max_length=np.asarray([16, 30], np.int32))
    # limits at the prompt length (no new token) and one above it (one token), beside a longer one: on the persistent
    # pass (beam 2: 6 rows) and on the batched pass (beam 5: 15 rows), like the same limits given alone
    for beam in (2, 5):
        ids, sc = h.generate(mel[:3], [PROMPT] * 3, beam_size=beam, max_length=np.asarray([4, 5, 16], np.int32))
        assert ids[0] == [] and sc[0] == 0.0, (beam, ids[0], sc[0])
        assert len(ids[1]) == 1 and ids[1] == h.generate(mel[1:2], [PROMPT], beam_size=beam, max_length=5)[0][0], beam
        assert ids[2] == h.generate(mel[2:3], [PROMPT], beam_size=beam, max_length=16)[0][0], beam
        assert h.generate(mel[:1], [PROMPT], beam_size=beam, max_length=4) == ([[]], [0.0])


def test_cross_attention_tensor_core_vs_simt(pair):
    # the wgmma cross-attention of the batched pass against the SIMT cluster kernel (two implementations of the same sum)
    dims, oracle, h = pair
    mel = mel_inputs(4)[:1]
    toks = PROMPT + [100, 2000, 30000, 41000, 12]
    h.set_option("decoder_batch", 2)
    try:
        a = h.debug_forced_logits(mel, toks)
        h.set_option("cross_tc", 0)
        b = h.debug_forced_logits(mel, toks)
    finally:
        h.set_option("cross_tc", 1)
        h.set_option("decoder_batch", 1)
    assert np.abs(a - b).max() < 2e-2
    mel6 = mel_inputs(6)
    ids_tc, _ = h.generate(mel6, [PROMPT] * 6, beam_size=5)
    h.set_option("cross_tc", 0)
    try:
        ids_simt, _ = h.generate(mel6, [PROMPT] * 6, beam_size=5)
    finally:
        h.set_option("cross_tc", 1)
    res, robust = robust_cases(oracle, mel6, [PROMPT] * 6, 5, n_probe=2)
    assert len(robust) >= 4
    for i in robust:
        assert ids_tc[i] == res[i].sequences_ids[0] == ids_simt[i], i


@pytest.mark.parametrize("cross_tc", [1, 0])
def test_multi_row_teacher_forcing_matches_oracle(pair, cross_tc):
    # 1..8 consecutive positions as rows of one pass (the way a prompt prefix is prefilled): every position's logits,
    # with the wgmma and with the SIMT cross-attention
    dims, oracle, h = pair
    mel = mel_inputs(4)[:1]
    toks = PROMPT + [100, 2000, 30000, 41000, 12, 50000, 7, 999]
    want = oracle.forced_logits(oracle.encode(mel)[0], toks).numpy()
    h.set_option("decoder_batch", 2)
    h.set_option("cross_tc", cross_tc)
    try:
        for chunk in (1, 2, 3, 5, 8):
            h.set_option("debug_chunk", chunk)
            err = np.abs(h.debug_forced_logits(mel, toks) - want).max(axis=1)
            assert err.shape == (len(toks),)
            assert np.all(err <= LOGIT_TOL), (chunk, err)
    finally:
        h.set_option("debug_chunk", 1)
        h.set_option("cross_tc", 1)
        h.set_option("decoder_batch", 1)


@pytest.mark.parametrize("prompt", [[50258, 50363], PROMPT])
def test_greedy16_both_cross_attention_kernels_match_oracle(pair, prompt):
    # 16 utterances, greedy: with a 2-token prompt the prefix pass has one row per utterance too
    dims, oracle, h = pair
    mel = mel_inputs(16)
    prompts = [prompt] * 16
    res, robust = robust_cases(oracle, mel, prompts, 1, n_probe=2, max_length=24)
    assert len(robust) >= 10, f"only {len(robust)} of 16 oracle transcripts are robust decisions"
    for tc in (1, 0):
        h.set_option("cross_tc", tc)
        try:
            ids, _ = h.generate(mel, np.asarray(prompts, np.int32), beam_size=1, max_length=24)
        finally:
            h.set_option("cross_tc", 1)
        for i in robust:
            assert ids[i] == res[i].sequences_ids[0], (tc, i)


def test_greedy_pass_above_512_utterances(pair):
    # batch_rows = 1024 at beam 1 puts 520 windows into ONE shared pass (one row each): the cross-attention takes up to
    # 1024 utterances per launch.  Every copy of a robust window equals the oracle; copies of a window are identical.
    dims, oracle, h = pair
    mel16 = mel_inputs(16)
    res, robust = robust_cases(oracle, mel16, [PROMPT] * 16, 1, n_probe=2, max_length=24)
    assert len(robust) >= 10, f"only {len(robust)} of 16 oracle transcripts are robust decisions"
    n = 520
    mel = np.ascontiguousarray(np.tile(mel16, (n // 16 + 1, 1, 1))[:n])
    h.set_option("batch_rows", 1024)
    try:
        ids, _ = h.generate(mel, np.asarray([PROMPT] * n, np.int32), beam_size=1, max_length=24)
    finally:
        h.set_option("batch_rows", 320)
    for i in range(n):
        assert ids[i] == ids[i % 16], i
    for i in robust:
        assert ids[i] == res[i].sequences_ids[0], i


def test_row_capacity_groups(pair):
    dims, oracle, h = pair
    mel = mel_inputs(6)
    want, _ = h.generate(mel, [PROMPT] * 6, beam_size=5)
    h.set_option("batch_rows", 20)  # 4 utterances x 5 beams per shared pass -> two groups
    try:
        got, _ = h.generate(mel, [PROMPT] * 6, beam_size=5)
    finally:
        h.set_option("batch_rows", 320)
    assert got == want
    # graphs and eager launches, with and without programmatic dependent launch, agree
    for key, val in (("use_graphs", 0), ("batch_pdl", 0)):
        h.set_option(key, val)
        try:
            again, _ = h.generate(mel, [PROMPT] * 6, beam_size=5)
        finally:
            h.set_option(key, 1)
        assert again == want, key
