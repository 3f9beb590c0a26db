"""GPU: timestamp decoding (a prompt without <|notimestamps|>).

* ``wisb_debug_search_step`` runs ONE production search step on crafted rows; its candidates must be the oracle's
  processors + timestamp rules + log-softmax + top-2*beam exactly (ids), scores within 1e-5.
* End to end on the timestamp-scripted test model (``weights.synth_state_dict(ts_script=...)``), 3-token prompt, against
  ``tests.ts_oracle.TimestampOracle`` on its robust cases: every decoder path, every utterance equal to its solo run.
* With timestamps off, ``max_initial_timestamp_index`` changes nothing: bit for bit, launch count included.
"""
import functools
import threading

import numpy as np
import pytest
import torch

from tests.gpu_common import LOGIT_TOL, PROMPT, mel_inputs, model_pair, robust_cases
from tests.ts_oracle import TimestampOracle, apply_timestamp_rules, check_invariants
from willow_inference_server_b200 import _lib, audio, models, weights as W

pytestmark = pytest.mark.gpu
TS_PROMPT = [50258, 50259, 50359]
SCRIPT, RAMP, TS_SCRIPT = (4, 3.3, 1.67), (8, 12.0), (2, 5, 8)
GEOMETRIES = [(51865, 50257, 50363), (51864, 50256, 50362), (51866, 50257, 50364)]
STEP = 2.0 ** -11   # logit grid


# ----------------------------------------------------------------------------------------------------- one search step
@pytest.fixture(scope="module")
def frontend():
    return _lib.Handle.frontend(0)


def ref_step(logits, hists, mask, gen, beam, cum, eot, no_ts, ts, max_init):
    """The oracle's processors -> (candidate ids [n_utt, 2 beam], scores, row lse) in float64."""
    x = torch.from_numpy(logits.astype(np.float64))
    m = torch.from_numpy(mask)
    x[:, (m & 1).bool()] = float("-inf")
    if gen == 0:
        x[:, (m & 2).bool()] = float("-inf")
    if ts:
        x = apply_timestamp_rules(x, hists, gen, no_timestamps=no_ts, eot=eot, max_initial_timestamp_index=max_init)
    lse = torch.logsumexp(x, -1)
    V = x.shape[1]
    total = (x - lse[:, None] + torch.from_numpy(cum.astype(np.float64))[:, None]) / (gen + 1)
    ids, scores = [], []
    for u in range(x.shape[0] // beam):
        flat = total[u * beam : (u + 1) * beam].reshape(-1)
        if gen == 0:
            flat = flat.clone()
            flat[V:] = float("-inf")
        order = torch.argsort(-flat, stable=True)[: 2 * beam]
        ok = torch.isfinite(flat[order])
        ids.append([int(i) if k else -1 for i, k in zip(order, ok)])
        scores.append([float(s) for s in flat[order]])
    return np.asarray(ids), np.asarray(scores), lse.numpy()


def grid_logits(rng, R, V):
    return np.stack([(rng.permutation(V) - V / 2) * STEP for _ in range(R)]).astype(np.float32)


def set_margin(row, hist, gen, mask, eot, no_ts, margin):
    """Shift the row's timestamp logits (by grid steps) so that rule 5's margin lse(ts) - max(text) is ~margin."""
    x = torch.from_numpy(row[None].astype(np.float64))
    x[:, torch.from_numpy(mask & 1).bool()] = float("-inf")
    y = apply_timestamp_rules(x, [hist], gen, no_timestamps=no_ts, eot=eot, disable=(5,))[0]
    now = float(torch.logsumexp(y[no_ts + 1:], 0) - y[: no_ts + 1].max())
    row[no_ts + 1:] += np.float32(round((margin - now) / STEP) * STEP)


def scenarios(V, eot, no_ts, rng):
    T = lambda i: no_ts + 1 + i  # noqa: E731
    # (gen, beam, per-row histories, done, margins per row or None, extra suppressed ids, max_init)
    yield 0, 2, [[], []] * 2, None, None, [], 50
    yield 0, 1, [[]] * 3, None, None, [T(1), T(2)], 3
    yield 0, 1, [[]], None, None, [], 3000
    yield 1, 2, [[T(3)], [T(5)], [T(0)], [T(50)]], None, None, [], 50
    yield 3, 2, [[T(0), 500, T(20)], [T(0), 500, 600],          # 3b / rule 4 at <= t, one utterance
                 [500, 600, T(40)], [T(0), T(7), 700],           # 3b without an earlier timestamp / after a pair
                 [T(0), 500, 600], [T(0), 500, 600]], [0, 0, 1], None, [], 50   # a finished (frozen) utterance
    yield 2, 2, [[T(3), 500], [T(3), 500], [500, 600], [500, 600]], None, [1e-3, -1e-3, 1e-3, -1e-3], [], 50
    yield 2, 1, [[500, T(0)], [500, 600], [T(2), T(9)]], None, None, [], 50   # the text / timestamp chunk boundary
    yield 4, 3, [[T(0), 9, T(30), T(30)], [T(0), 9, 10, 11], [T(0), 9, 10, T(60)]], None, None, \
        [T(k) for k in range(28, 70)], 50                       # extra-suppress list full of timestamps
    yield 5, 8, [[T(0), 100 + k, 200, T(10 + k), T(10 + k)] for k in range(8)], None, None, [], 50


@pytest.mark.parametrize("geom", range(3))
def test_search_step_matches_oracle(frontend, geom):
    V, eot, no_ts = GEOMETRIES[geom]
    rng = np.random.default_rng(7 + geom)
    base_mask = np.zeros(V, np.uint8)
    base_mask[W.WhisperDims().suppress_ids] |= 1
    base_mask[[220, eot]] |= 2
    n_checked = 0
    for sc in scenarios(V, eot, no_ts, rng):
        gen, beam, hists, done, margins, extra, max_init = sc
        R = len(hists)
        mask = base_mask.copy()
        mask[extra] |= 1
        logits = grid_logits(rng, R, V)
        if sc[2] and sc[2][0] == [500, no_ts + 1]:               # boundary rows: the best ids sit next to ts_begin
            logits[:, no_ts - 1] = 20.0
            logits[:, no_ts + 2] = 20.0 - STEP
            logits[:, no_ts + 1] = 20.0 - 2 * STEP
        if margins:
            for r, mg in enumerate(margins):
                set_margin(logits[r], hists[r], gen, mask, eot, no_ts, mg)
        cum = (rng.standard_normal(R) * 2 - 3).astype(np.float32) if gen else np.zeros(R, np.float32)
        for ts in (1, 0):
            ci, cs, lse = frontend.debug_search_step(logits, hists, mask, beam=beam, gen=gen, eot=eot, no_timestamps=no_ts,
                                                     timestamps=ts, max_initial_timestamp_index=max_init, cum=cum,
                                                     done=done)
            wi, ws, wl = ref_step(logits, hists, mask, gen, beam, cum, eot, no_ts, ts, max_init)
            assert np.array_equal(ci, wi), (geom, sc[:3], ts, ci, wi)
            fin = wi >= 0
            assert np.abs(cs[fin] - ws[fin]).max() <= 1e-5, (geom, sc[:3], ts)
            assert np.abs(lse - wl).max() <= 2e-5, (geom, sc[:3], ts)
            n_checked += 1
    assert n_checked == 18


def test_search_step_rule5_margins_decide(frontend):
    # the +-1e-3 rows really sit on both sides of rule 5: text candidates exist exactly in the negative-margin rows
    V, eot, no_ts = GEOMETRIES[0]
    rng = np.random.default_rng(3)
    mask = np.zeros(V, np.uint8)
    for mg, want_text in ((1e-3, False), (-1e-3, True), (2e-3, False), (-2e-3, True)):
        row = grid_logits(rng, 1, V)
        set_margin(row[0], [500, 600], 2, mask, eot, no_ts, mg)
        ci, _, _ = frontend.debug_search_step(row, [[500, 600]], mask, beam=1, gen=2, eot=eot, no_timestamps=no_ts,
                                              timestamps=True)
        assert (ci[0] < no_ts).any() == want_text, (mg, ci)


# ----------------------------------------------------------------------------------------------------- end to end
@functools.lru_cache(maxsize=1)
def ts_pair():
    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=2)
    tensors = W.synth_engine_tensors(dims, seed=11, eot_ramp=RAMP, script=SCRIPT, ts_script=TS_SCRIPT)
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    return dims, TimestampOracle.from_blob(buf), _lib.Handle.from_host(buf, 0)


N_UTT = 16


DECISION_GAP = LOGIT_TOL / 4


@functools.lru_cache(maxsize=4)
def oracle_cases(beam):
    dims, oracle, h = ts_pair()
    mel = mel_inputs(N_UTT)
    res, robust = robust_cases(oracle, mel, [TS_PROMPT] * N_UTT, beam)
    if beam > 1:
        # Two beam candidates that share a prefix differ in a few logits only, so iid logit noise rarely reorders them:
        # the probe called a case robust whose top-beam boundary was 3e-3 apart in cumulative log-prob, and the fp16
        # warp-MMA pass (logits within 0.05 of the oracle all along) resolved it the other way.  A case also needs every
        # step's decision-relevant gap (WhisperOracle._beam_margin) above DECISION_GAP.
        trace = []
        oracle.generate(mel, [TS_PROMPT] * N_UTT, beam_size=beam, trace=trace)
        robust = [i for i in robust if min(trace[i][:-1]) > DECISION_GAP]
    return mel, res, robust


def check_against_oracle(ids, scores, res, robust, beam, where):
    dims = ts_pair()[0]
    for i in robust:
        assert ids[i] == res[i].sequences_ids[0], (where, beam, i)
        if beam > 1 and scores is not None:
            assert abs(scores[i] - res[i].scores[0]) < 5e-2, (where, beam, i)
    for s in ids:
        check_invariants(s, dims)


@pytest.mark.parametrize("beam", [1, 2, 5])
def test_enough_robust_cases_with_segments(beam):
    dims = ts_pair()[0]
    mel, res, robust = oracle_cases(beam)
    assert len(robust) >= 3, f"only {len(robust)} of {N_UTT} oracle transcripts are robust"
    assert min(check_invariants(res[i].sequences_ids[0], dims) for i in robust) >= 2


@pytest.mark.parametrize("beam", [1, 2, 5])
@pytest.mark.parametrize("path", ["mega_mma", "mega_simt", "batched_small"])
def test_small_rows_paths_match_oracle(beam, path):
    dims, oracle, h = ts_pair()
    mel, res, robust = oracle_cases(beam)
    opts = {"mega_mma": {}, "mega_simt": {"mega_mma": 0}, "batched_small": {"decoder_batch": 2}}[path]
    P = np.array([TS_PROMPT], np.int32)
    for k, v in opts.items():
        h.set_option(k, v)
    try:
        solo, solo_sc = [], []
        for i in range(N_UTT):
            ids, sc = h.generate(mel[i : i + 1], P, beam, timestamps=True)
            solo.append(ids[0])
            solo_sc.append(sc[0])
        check_against_oracle(solo, solo_sc, res, robust, beam, path)
        group = max(1, 8 // beam)                             # <= 8 rows: one pass (4 x 2 prompt rows: one-pass prefill)
        for g0 in range(0, N_UTT, group):
            ids, _ = h.generate(mel[g0 : g0 + group], np.repeat(P, len(mel[g0 : g0 + group]), 0), beam, timestamps=True)
            assert ids == solo[g0 : g0 + group], (path, beam, g0)
    finally:
        for k in opts:
            h.set_option(k, 1)


@pytest.mark.parametrize("beam", [1, 2, 5])
def test_batched_pass_16_utterances(beam):
    dims, oracle, h = ts_pair()
    mel, res, robust = oracle_cases(beam)
    mel16 = mel                                               # 16 utterances in one call: the batched pass
    ids, sc = h.generate(mel16, np.repeat(np.array([TS_PROMPT], np.int32), 16, 0), beam, timestamps=True)
    check_against_oracle(ids, sc, res, robust, beam, "batched")
    h.set_option("decoder_batch", 2)                          # solo runs on the same (batched) pass
    try:
        solo = [h.generate(mel[i : i + 1], np.array([TS_PROMPT], np.int32), beam, timestamps=True)[0][0] for i in range(N_UTT)]
    finally:
        h.set_option("decoder_batch", 1)
    assert ids == solo
    h.set_option("use_graphs", 0)
    try:
        eager, _ = h.generate(mel16, np.repeat(np.array([TS_PROMPT], np.int32), 16, 0), beam, timestamps=True)
    finally:
        h.set_option("use_graphs", 1)
    assert eager == ids


def test_max_initial_timestamp_index_on_the_device():
    dims, oracle, h = ts_pair()
    mel = mel_inputs(N_UTT)
    P = np.repeat(np.array([TS_PROMPT], np.int32), N_UTT, 0)
    ts0 = dims.no_timestamps + 1
    first = {}
    for mi in (0, 5, 1000):
        res, robust = robust_cases(oracle, mel, P.tolist(), 1, n_probe=2, max_initial_timestamp_index=mi)
        assert len(robust) >= 3, mi
        ids, _ = h.generate(mel, P, 1, timestamps=True, max_initial_timestamp_index=mi)
        for i in robust:
            assert ids[i] == res[i].sequences_ids[0], (mi, i)
        assert all(s[0] <= ts0 + mi for s in ids)
        first[mi] = [s[0] for s in ids]
        ids5, _ = h.generate(mel[:2], P[:2], 5, timestamps=True, max_initial_timestamp_index=mi)
        assert all(ts0 <= s[0] <= ts0 + mi for s in ids5)
    assert set(first[0]) == {ts0}
    # the script lifts index 60 above index 8 at the first step: without the clamp some transcripts start later
    assert any(s > ts0 + 50 for s in first[1000])


def test_timestamps_off_is_generate_ex_bit_for_bit():
    dims, oracle, h = model_pair()
    mel = mel_inputs(6)
    for n, beam in ((1, 5), (2, 1), (6, 5)):                  # persistent pass and batched pass
        P = np.repeat(np.array([PROMPT], np.int32), n, 0)
        a_ids, a_sc = h.generate(mel[:n], P, beam)                                   # the default index, 50
        a_t = h.timing()
        b_ids, b_sc = h.generate(mel[:n], P, beam, max_initial_timestamp_index=7)    # timestamps still off
        b_t = h.timing()
        assert a_ids == b_ids and np.array_equal(np.float32(a_sc), np.float32(b_sc))
        assert a_t["launches"] == b_t["launches"] and a_t["decode_steps"] == b_t["decode_steps"]


def test_timestamp_argument_errors():
    dims, oracle, h = ts_pair()
    mel = mel_inputs(2)[:1]
    with pytest.raises(ValueError, match="notimestamps"):
        h.generate(mel, np.array([TS_PROMPT + [dims.no_timestamps]], np.int32), 1, timestamps=True)
    with pytest.raises(ValueError, match="timestamp tokens"):
        h.generate(mel, np.array([TS_PROMPT + [dims.no_timestamps + 3]], np.int32), 1, timestamps=True)
    with pytest.raises(ValueError, match="max_initial"):
        h.generate(mel, np.array([TS_PROMPT], np.int32), 1, timestamps=True, max_initial_timestamp_index=-1)
    m = models.Whisper(None, device="cuda", _handles=[h])
    out = m.generate(models.StorageView.from_array(mel), [TS_PROMPT], beam_size=1)   # the public switch
    assert out[0].sequences_ids[0] == h.generate(mel, np.array([TS_PROMPT], np.int32), 1, timestamps=True)[0][0]


def test_batcher_keeps_timestamp_and_plain_requests_apart():
    from willow_inference_server_b200.batcher import TranscribeBatcher

    dims, oracle, h = ts_pair()
    mel = mel_inputs(4)
    m = models.Whisper(None, device="cuda", _handles=[h])
    plain = TS_PROMPT + [dims.no_timestamps]
    want_ts = [r.sequences_ids[0] for r in m.generate(models.StorageView.from_array(mel), [TS_PROMPT] * 4, beam_size=2)]
    want_pl = [r.sequences_ids[0] for r in m.generate(models.StorageView.from_array(mel), [plain] * 4, beam_size=2)]
    assert all(s[0] > dims.no_timestamps for s in want_ts) and want_ts != want_pl
    with TranscribeBatcher(m, max_batch=8, max_wait_ms=50) as b:
        futs = {}
        jobs = [(i, p) for i in range(4) for p in ("ts", "plain")]
        ts = [threading.Thread(target=lambda i=i, p=p: futs.__setitem__(
            (i, p), b.submit(mel[i : i + 1], TS_PROMPT if p == "ts" else plain, beam_size=2))) for i, p in jobs]
        [t.start() for t in ts]
        [t.join() for t in ts]
        for i in range(4):
            assert futs[(i, "ts")].result(timeout=120)[0].sequences_ids[0] == want_ts[i]
            assert futs[(i, "plain")].result(timeout=120)[0].sequences_ids[0] == want_pl[i]


def _synth(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.float64) / 16000.0
    return (0.3 * np.sin(2 * np.pi * (200.0 + 300.0 * t) * t) + 0.05 * rng.standard_normal(n)).astype(np.float32)


def test_full_size_small_and_batched_paths_agree():
    # large-v2 dims, beam 5, 3-token prompt: the persistent pass alone and the batched pass inside a batch (peaked
    # timestamp-scripted weights, so that the two passes' different fp16 roundings cannot flip a decision)
    dims = W.WhisperDims.for_size("large-v2")
    tensors = W.synth_engine_tensors(dims, seed=0, eot_ramp=RAMP, script=SCRIPT, ts_script=TS_SCRIPT)
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    del tensors
    h = _lib.Handle.from_host(buf, 0)
    del buf
    try:
        mel = audio.log_mel_batch([_synth(61440, 1), _synth(160000, 2), _synth(480000, 3)], h)
        P = np.array([TS_PROMPT], np.int32)
        batch, _ = h.generate(mel, np.repeat(P, 3, 0), 5, max_length=64, timestamps=True)     # 15 rows: batched pass
        for i in range(3):
            solo, _ = h.generate(mel[i : i + 1], P, 5, max_length=64, timestamps=True)        # 5 rows: persistent pass
            assert solo[0] == batch[i], i
        ts0 = dims.no_timestamps + 1
        for s in batch:
            check_invariants(s, dims)
    finally:
        h.close()
