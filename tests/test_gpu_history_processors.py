"""GPU: repetition penalty and no-repeat n-gram blocking in the device token search.

* One production search step at a time (``wisb_debug_search_step`` with the processors): the candidate ids and the
  whole integer state must equal the oracle step (``tests.proc_oracle.process_rows`` -> log-softmax -> top 2*beam in
  float64 -> ``tests.test_gpu_search.expected_step``), cum within CUM_ULPS.  Crafted cases cover random beam histories,
  both vocabulary splits, the three vocabularies, beams 1 / 5 / 8, gen 0, 1, n - 1, n and 447, a banned arg-max, ids
  the penalty pushes across a chunk's top-k boundary and rule 5 flipped by the penalty.
* Multi-step chains from the search initialisation end where the oracle loop ends wherever every decision gap is clear.
* End to end on the loop test model (``weights.synth_state_dict(loop_pool=...)``): tokens equal to ``ProcOracle`` on
  its robust cases on every decoder pass, in one timestamp case and in a multi-utterance call; with n set no returned
  sequence holds an n-gram twice; either processor changes most transcripts.
"""
import ctypes
import functools
import zlib

import numpy as np
import pytest
import torch

from oracle.whisper_ref import beam_search, length_norm
from tests.gpu_common import LOGIT_TOL, PROMPT, RAMP, SCRIPT, mel_inputs, robust_cases
from tests.proc_oracle import ProcOracle, process_rows
from tests.test_gpu_search import GEOMETRIES, LDL, NEG, base_mask, check_candidates, compare, expected_step
from tests.ts_oracle import apply_timestamp_rules, check_invariants
from willow_inference_server_b200 import _lib, models, weights as W

LOOP = 4                      # the loop model's pool of scripted tokens
TS_PROMPT = [50258, 50259, 50359]
TS_SCRIPT = (2, 5, 8)
STEP = 2.0 ** -11
PROMPT_LAST = 7777            # a text id standing in for the last prompt token (the prompt_history defect counts it)


# ----------------------------------------------------------------------------------------------------- one search step
def masked(x, mask, gen):
    """the suppress masks on float64 logits"""
    x = x.double()
    m = torch.from_numpy(mask)
    x[:, (m & 1).bool()] = NEG
    if gen == 0:
        x[:, (m & 2).bool()] = NEG
    return x


def ref_step(sc, defect=None):
    """float64 candidates (ids [n_utt, 2 beam], scores, totals) of the oracle's processed logits for scenario sc."""
    V, eot, no_ts, beam, gen = sc["V"], sc["eot"], sc["no_ts"], sc["beam"], sc["gen"]
    rules = None
    if sc["ts"]:
        rules = lambda x, h, g: apply_timestamp_rules(x, h, g, no_timestamps=no_ts, eot=eot,  # noqa: E731
                                                      max_initial_timestamp_index=sc["max_init"])
    x = process_rows(torch.from_numpy(sc["logits"][:, :V].copy()), sc["hists"], gen,
                     masks=lambda y, g: masked(y, sc["mask"], g), rules=rules, repetition_penalty=sc["p"],
                     no_repeat_ngram_size=sc["n"], prompt=[PROMPT_LAST], defect=defect).double()
    logp = x - torch.logsumexp(x, -1, keepdim=True)
    total = (logp + torch.from_numpy(sc["cum"].astype(np.float64))[:, None]) / length_norm(gen, 1.0)
    ids, scores = [], []
    for u in range(len(sc["hists"]) // beam):
        flat = total[u * beam: (u + 1) * beam].reshape(-1)
        valid = torch.isfinite(logp[u * beam: (u + 1) * beam]).reshape(-1)
        if gen == 0:
            valid[V:] = False
        idx = torch.nonzero(valid).flatten()
        order = idx[torch.argsort(-flat[idx], stable=True)[: 2 * beam]].tolist()
        pad = 2 * beam - len(order)
        ids.append(order + [-1] * pad)
        scores.append([float(flat[i]) for i in order] + [NEG] * pad)
    return np.asarray(ids), np.asarray(scores), total


def grid_row(rng, V, lo=-12.0):
    """distinct logits on a 2^-11 grid in [lo, lo + V * 2^-11)"""
    return (lo + rng.permutation(V) * STEP).astype(np.float32)


def scenario(name, geom, beam, gen, hists, logits, *, p, n, ts=0, rng, max_init=50, n_utt=1):
    V, eot, no_ts = GEOMETRIES[geom]
    R = n_utt * beam
    x = np.full((R, LDL), np.nan, np.float32)
    x[:, :V] = logits
    cum = (rng.standard_normal(R) - 3).astype(np.float32) if gen else np.zeros(R, np.float32)
    return dict(name=name, V=V, eot=eot, no_ts=no_ts, beam=beam, gen=gen, hists=[list(h) for h in hists], logits=x,
                mask=base_mask(V, eot), ts=ts, p=p, n=n, cum=cum, max_init=max_init)


def loopy_hist(rng, gen, pool):
    return [int(pool[i]) for i in rng.integers(0, len(pool), gen)]


def step_scenarios():
    rng = np.random.default_rng(21)
    settings = [(1.1, 3), (2.0, 0), (1.0, 2), (0.5, 1), (1.3, 4)]
    k = 0
    for geom in range(3):
        V, eot, no_ts = GEOMETRIES[geom]
        T = lambda i: no_ts + 1 + i  # noqa: E731
        for ts in (0, 1):
            for beam in (1, 5, 8):
                p, n = settings[k % len(settings)]
                k += 1
                pool = [1000, 2345, 17, 40000, 777, 31000]
                gens = sorted({0, 1, max(n - 1, 0), n, 6})
                for gen in gens:
                    hists = []
                    for r in range(beam):
                        h = loopy_hist(rng, gen, pool)
                        if ts and gen >= 2 and r % 2:
                            h[0] = T(r)                                   # timestamps inside the history
                        hists.append(h)
                    x = np.stack([grid_row(rng, V) for _ in range(beam)])
                    if ts:                                                # rule 5 sometimes one way, sometimes the other
                        x[:, no_ts + 1:] -= np.float32(rng.uniform(2.0, 6.0))
                    for r, h in enumerate(hists):                         # history ids near the top, both signs (off grid)
                        for j, t in enumerate(sorted(set(h))):
                            x[r, t] = np.float32((12.5 if j % 2 == 0 else -0.75) - j * 0.125 + 2.0 ** -12)
                    yield scenario(f"random g{geom} ts{ts} b{beam} gen{gen}", geom, beam, gen, hists, x, p=p, n=n,
                                   ts=ts, rng=rng)
        # gen 447 (the longest history a row can hold): a loop of 6 tokens, every processor
        hists = [[pool[(t + r) % 6] for t in range(447)] for r, pool in enumerate([[11, 22, 33, 44, 55, 66]] * 5)]
        x = np.stack([grid_row(rng, V) for _ in range(5)])
        x[:, [11, 22, 33, 44, 55, 66, 77]] = np.float32(12.0)
        yield scenario(f"gen447 g{geom}", geom, 5, 447, hists, x, p=1.2, n=3, rng=rng)
        # a banned id that would be the arg-max (hist a b a: n = 2 bans b)
        a, b = 3000, 4000
        x = grid_row(rng, V)[None].copy()
        x[0, b] = np.float32(20.0)
        yield scenario(f"banned_argmax g{geom}", geom, 1, 3, [[a, b, a]], x, p=1.0, n=2, rng=rng)
        # ids the penalty pushes across one chunk's top-k boundary: 2 beam + 1 ids of one chunk at the top, the best in
        # the history; p = 2 drops it below the boundary and the next id enters
        for ts in (0, 1):
            beam = 5
            c0 = 5000
            x = np.stack([grid_row(rng, V) for _ in range(beam)])
            ids = [c0 + 3 * j for j in range(2 * beam + 1)]
            x[0, ids] = np.float32(16.0) - np.arange(2 * beam + 1, dtype=np.float32) * np.float32(0.25)  # row 0 only
            x[:, no_ts + 1:] -= np.float32(20.0)                          # rule 5 keeps the text
            hists = [[ids[0], 9000]] * beam
            sc = scenario(f"chunk_boundary g{geom} ts{ts}", geom, beam, 2, hists, x, p=2.0, n=0, ts=ts, rng=rng)
            sc["cum"][:] = -1.5                                           # row 0 holds the 2 beam best
            yield sc
        # the last prompt token is no history: its logit stays the best
        x = grid_row(rng, V)[None].copy()
        x[0, PROMPT_LAST] = np.float32(15.0)
        yield scenario(f"prompt_token g{geom}", geom, 1, 2, [[3000, 4000]], x, p=2.0, n=2, rng=rng)
        # rule 5 flipped by the penalty: the best text token (10) in the history halves below the timestamps'
        # log-sum-exp (1 + log 1501 + ...); without the penalty text stays on
        for p in (1.0, 2.0):
            x = (-8.0 + rng.permutation(V) * STEP * 2 ** -6).astype(np.float32)[None].copy()
            x[0, no_ts + 1:] = (1.0 + rng.permutation(V - no_ts - 1) * STEP).astype(np.float32)
            x[0, 6000] = np.float32(10.0)
            yield scenario(f"rule5 p{p} g{geom}", geom, 1, 1, [[6000]], x, p=p, n=0, ts=1, rng=rng)


@pytest.fixture(scope="module")
def h():
    return _lib.Handle.frontend(0)


def device_step(h, sc):
    beam, gen, R = sc["beam"], sc["gen"], len(sc["hists"])
    n_utt = R // beam
    t_max = min(gen + 6, 448)
    pos = min(gen + 3, t_max - 1)
    st = h.search_state(n_utt, beam, min(max(gen + 2, 4), 448), t_max)
    rng = np.random.default_rng(gen)
    st["st"][:2] = (pos, gen)
    st["flip"][0] = gen & 1
    st["seq"][:] = rng.integers(0, 50000, st["seq"].shape)      # the other ping-pong buffer holds junk
    for r, hist in enumerate(sc["hists"]):
        st["seq"][gen & 1, r, :gen] = hist
    st["indir"][:] = rng.integers(0, R, st["indir"].shape)
    st["row_pos"][:] = pos
    st["cum"][:] = sc["cum"]
    got, ci, cs, _ = h.debug_search_step_state(sc["logits"], sc["mask"], st, beam=beam, max_hyp=beam, eot=sc["eot"],
                                               V=sc["V"], no_timestamps=sc["no_ts"], timestamps=bool(sc["ts"]),
                                               max_initial_timestamp_index=sc["max_init"],
                                               repetition_penalty=sc["p"], no_repeat_ngram_size=sc["n"])
    return st, got, ci, cs


@pytest.mark.gpu
def test_search_steps_match_the_oracle_step(h):
    n = 0
    seen = set()
    for sc in step_scenarios():
        st, got, ci, cs = device_step(h, sc)
        wi, ws, total = ref_step(sc)
        where = (sc["name"], sc["p"], sc["n"])
        check_candidates(ci, cs, wi, ws, total, sc["beam"], where)
        compare(got, expected_step(st, ci, cs, beam=sc["beam"], V=sc["V"], eot=sc["eot"], max_hyp=sc["beam"], lp=1.0),
                where)
        seen.add(sc["name"].split()[0])
        n += 1
        if sc["name"].startswith("banned_argmax"):
            assert 4000 not in ci % sc["V"] and ci[0, 0] >= 0, where
        if sc["name"].startswith("prompt_token"):
            assert ci[0, 0] == PROMPT_LAST, where
        if sc["name"].startswith("chunk_boundary"):
            cand = set((ci[ci >= 0] % sc["V"]).tolist())
            assert 5000 not in cand and 5000 + 3 * 10 in cand, where
    assert n >= 90 and seen == {"random", "gen447", "banned_argmax", "chunk_boundary", "prompt_token", "rule5"}, (n, seen)


@pytest.mark.gpu
def test_rule5_is_flipped_by_the_penalty(h):
    text = {}
    for sc in step_scenarios():
        if sc["name"].startswith("rule5"):
            _, _, ci, _ = device_step(h, sc)
            text[(sc["name"].split()[-1], sc["p"])] = bool((ci[ci >= 0] % sc["V"] < sc["no_ts"]).any())
    for g in ("g0", "g1", "g2"):
        assert text[(g, 1.0)] and not text[(g, 2.0)], text


@pytest.mark.gpu
def test_processors_off_is_the_default_step(h):
    # (1, 0) through the n_prm == 15 form is the 13-parameter step bit for bit
    for sc in list(step_scenarios())[:12]:
        sc = dict(sc, p=1.0, n=0)
        st, got, ci, cs = device_step(h, sc)                 # explicit (1, 0): the 15-parameter form
        beam = sc["beam"]
        got2, ci2, cs2, _ = h.debug_search_step_state(sc["logits"], sc["mask"], st, beam=beam, max_hyp=beam,
                                                      eot=sc["eot"], V=sc["V"], no_timestamps=sc["no_ts"],
                                                      timestamps=bool(sc["ts"]))
        assert np.array_equal(ci, ci2) and np.array_equal(cs, cs2)
        for k in got:
            assert np.array_equal(got[k], got2[k]), k


# ------------------------------------------------------------------------------------------------------------- chains
CHAIN_POOL = [1000, 2345, 777, 31000, 40000]


def chain_logits(hist, seed, V, eot, gen):
    """raw logits of a row with generated tokens `hist`: seeded by the history, a few pool tokens on top (so that the
    chains repeat), eot ramped up with the step"""
    key = zlib.crc32(np.asarray([seed] + list(hist), np.int64).tobytes())
    rng = np.random.default_rng(key)
    x = (rng.standard_normal(V) * 2.0).astype(np.float32)
    x[CHAIN_POOL] = (7.0 + 1.5 * rng.standard_normal(len(CHAIN_POOL))).astype(np.float32)
    x[eot] = np.float32(-4.0 + 1.1 * gen + rng.standard_normal())
    return x


def run_chain(h, seed, beam, ts, p, n, max_new=12):
    V, eot, no_ts = GEOMETRIES[0]
    mask = base_mask(V, eot)
    st = h.search_state(1, beam, max_new, 3 + max_new)
    prompt = np.asarray([TS_PROMPT], np.int32)
    kw = dict(timestamps=bool(ts), no_timestamps=no_ts, max_initial_timestamp_index=6, repetition_penalty=p,
              no_repeat_ngram_size=n)
    s, reordered = 0, False
    while True:
        cur = int(st["flip"][0])
        hists = [list(st["seq"][cur, r, :s]) for r in range(beam)]
        x = np.full((beam, LDL), np.nan, np.float32)
        for r in range(beam):
            x[r, :V] = chain_logits(hists[r], seed, V, eot, s)
        got, ci, cs, _ = h.debug_search_step_state(x, mask, st, beam=beam, max_hyp=beam, eot=eot, V=V,
                                                   prompt=prompt if s == 0 else None, shared_prefix=1, **kw)
        if s == 0:
            init = h.search_state(1, beam, max_new, 3 + max_new)
            init["st"][0] = 2
            init["tokens"][:] = TS_PROMPT[-1]
            init["row_pos"][:] = 2
            init["indir"][:] = 0
            st = init
        compare(got, expected_step(st, ci, cs, beam=beam, V=V, eot=eot, max_hyp=beam, lp=1.0), (seed, beam, ts, s))
        nxt = int(got["flip"][0])
        parents = [int(got["indir"][nxt, r, 2 + s]) for r in range(beam)]
        reordered |= s > 0 and parents != list(range(beam)) and bool(np.isfinite(got["cum"]).all())
        st = got
        s += 1
        if st["st"][3]:
            break

    def logits_fn(step, tokens, parents):
        if step == 0:
            logits_fn.hist = [[] for _ in range(beam)]
        else:
            logits_fn.hist = [logits_fn.hist[q] + [t] for q, t in zip(parents, tokens)]
        return torch.from_numpy(np.stack([chain_logits(hh, seed, V, eot, step) for hh in logits_fn.hist]))

    rules = None
    if ts:
        rules = lambda y, hh, g: apply_timestamp_rules(y, hh, g, no_timestamps=no_ts, eot=eot,  # noqa: E731
                                                       max_initial_timestamp_index=6)

    def process(logits, hists, step):
        return process_rows(logits, hists, step, masks=lambda y, g: masked(y, mask, g), rules=rules,
                            repetition_penalty=p, no_repeat_ngram_size=n).float()

    trace = []
    want = beam_search(logits_fn, process, beam=beam, V=V, eot=eot, max_new=max_new, max_hyp=beam, length_penalty=1.0,
                       trace=trace)
    return st, want, min(trace), reordered


@pytest.mark.gpu
@pytest.mark.parametrize("beam", [1, 5, 8])
@pytest.mark.parametrize("ts", [0, 1])
def test_chains_end_where_the_oracle_loop_ends(h, beam, ts):
    clear, reordered = 0, 0
    for seed, (p, n) in enumerate([(1.3, 0), (1.0, 2), (1.2, 3), (2.0, 1)]):
        st, want, gap, re = run_chain(h, seed, beam, ts, p, n)
        reordered += re
        if gap > 1e-4:
            assert st["n_hyp"][0] == len(want.hyps), (seed, beam, ts)
            assert list(st["best_tokens"][0, : st["best_len"][0]]) == want.best_tokens, (seed, beam, ts)
            assert abs(st["best_score"][0] - want.best_score) <= 1e-4, (seed, beam, ts)
            clear += 1
    assert clear >= 2, clear
    assert beam == 1 or reordered >= 1


# ----------------------------------------------------------------------------------------------------- end to end
N_UTT = 16
SETTINGS = [(1.2, 0), (2.0, 0), (1.0, 2), (1.0, 3), (1.2, 3)]
DECISION_GAP = LOGIT_TOL / 4
# Robust cases of 16 per (beam, setting) have a floor a little under the count measured with the CPU oracle.  With the
# penalty alone or with (1.2, 3), no beam-5 case survives the noise probe and the decision-gap filter on this model (the
# penalty pulls the scripted alternatives' scores together): there only the n-gram property is checked.
FLOOR = {(1, (1.2, 0)): 2, (1, (2.0, 0)): 1, (1, (1.0, 2)): 4, (1, (1.0, 3)): 6, (1, (1.2, 3)): 3,
         (5, (1.2, 0)): 0, (5, (2.0, 0)): 0, (5, (1.0, 2)): 1, (5, (1.0, 3)): 3, (5, (1.2, 3)): 0}


@functools.lru_cache(maxsize=2)
def loop_pair(ts=False):
    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=2)
    tensors = W.synth_engine_tensors(dims, seed=11, eot_ramp=RAMP, script=SCRIPT, loop_pool=LOOP,
                                     ts_script=TS_SCRIPT if ts else None)
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    return dims, ProcOracle.from_blob(buf), _lib.Handle.from_host(buf, 0)


@functools.lru_cache(maxsize=16)
def oracle_cases(beam, p, n, ts=False):
    dims, oracle, _ = loop_pair(ts)
    mel = mel_inputs(N_UTT)
    prompt = TS_PROMPT if ts else PROMPT
    kw = dict(repetition_penalty=p, no_repeat_ngram_size=n)
    res, robust = robust_cases(oracle, mel, [prompt] * N_UTT, beam, **kw)
    # every step's decision gap too, greedy included: the penalty moves logits by whole fractions of themselves, and one
    # greedy case that survived the noise probe went the other way on the batched pass
    trace = []
    oracle.generate(mel, [prompt] * N_UTT, beam_size=beam, trace=trace, **kw)
    robust = [i for i in robust if min(trace[i][:-1]) > DECISION_GAP]
    return mel, res, robust


def has_repeated_ngram(seq, n):
    grams = [tuple(seq[i: i + n]) for i in range(len(seq) - n + 1)]
    return len(grams) != len(set(grams))


@pytest.mark.gpu
@pytest.mark.parametrize("setting", SETTINGS)
@pytest.mark.parametrize("beam", [1, 5])
@pytest.mark.parametrize("path", ["mega_mma", "mega_simt", "batched_small"])
def test_loop_model_matches_oracle(path, beam, setting):
    p, n = setting
    dims, oracle, h = loop_pair()
    mel, res, robust = oracle_cases(beam, p, n)
    assert len(robust) >= FLOOR[(beam, setting)], f"only {len(robust)} of {N_UTT} oracle transcripts are robust"
    opts = {"mega_mma": {}, "mega_simt": {"mega_mma": 0}, "batched_small": {"decoder_batch": 2}}[path]
    for k, v in opts.items():
        h.set_option(k, v)
    try:
        P = np.array([PROMPT], np.int32)
        ids = [h.generate(mel[i: i + 1], P, beam, repetition_penalty=p, no_repeat_ngram_size=n)[0][0]
               for i in range(N_UTT)]
    finally:
        for k in opts:
            h.set_option(k, 1)
    for i in robust:
        assert ids[i] == res[i].sequences_ids[0], (path, beam, setting, i)
    if n:
        assert not any(has_repeated_ngram(s, n) for s in ids), (path, beam, setting)


@pytest.mark.gpu
@pytest.mark.parametrize("beam", [1, 5])
def test_processors_change_most_transcripts(beam):
    dims, oracle, h = loop_pair()
    mel = mel_inputs(N_UTT)
    P = np.repeat(np.array([PROMPT], np.int32), N_UTT, 0)
    base, _ = h.generate(mel, P, beam)
    assert sum(has_repeated_ngram(s, 2) for s in base) > N_UTT // 2      # the loop model loops
    _, _, robust = oracle_cases(beam, 1.0, 0)
    assert len(robust) >= 3
    for p, n in SETTINGS:
        ids, _ = h.generate(mel, P, beam, repetition_penalty=p, no_repeat_ngram_size=n)
        assert sum(ids[i] != base[i] for i in robust) > len(robust) // 2, (beam, p, n)


@pytest.mark.gpu
@pytest.mark.parametrize("beam", [1, 5])
def test_timestamp_mode(beam):
    dims, oracle, h = loop_pair(ts=True)
    p, n = 1.2, 3
    mel, res, robust = oracle_cases(beam, p, n, ts=True)
    assert len(robust) >= (6 if beam == 1 else 1)
    P = np.array([TS_PROMPT], np.int32)
    ids = [h.generate(mel[i: i + 1], P, beam, timestamps=True, repetition_penalty=p, no_repeat_ngram_size=n)[0][0]
           for i in range(N_UTT)]
    for i in robust:
        assert ids[i] == res[i].sequences_ids[0], (beam, i)
    for s in ids:
        check_invariants(s, dims)
        assert not has_repeated_ngram(s, n)
    m = models.Whisper(None, device="cuda", _handles=[h])                # the public surface
    out = m.generate(models.StorageView.from_array(mel[:2]), [TS_PROMPT] * 2, beam_size=beam, repetition_penalty=p,
                     no_repeat_ngram_size=n)
    assert [o.sequences_ids[0] for o in out] == ids[:2]


@pytest.mark.gpu
def test_multi_utterance_call_matches_solo_runs():
    dims, oracle, h = loop_pair()
    beam, (p, n) = 5, (1.0, 3)
    mel, res, robust = oracle_cases(beam, p, n)
    assert len(robust) >= 3
    P = np.repeat(np.array([PROMPT], np.int32), N_UTT, 0)
    ids, sc = h.generate(mel, P, beam, repetition_penalty=p, no_repeat_ngram_size=n)       # 80 rows: batched pass
    for i in robust:
        assert ids[i] == res[i].sequences_ids[0], i
    h.set_option("decoder_batch", 2)
    try:
        solo = [h.generate(mel[i: i + 1], P[:1], beam, repetition_penalty=p, no_repeat_ngram_size=n)[0][0]
                for i in range(N_UTT)]
    finally:
        h.set_option("decoder_batch", 1)
    assert ids == solo
    # a cached step graph never serves another processor setting
    plain, _ = h.generate(mel, P, beam)
    again, _ = h.generate(mel, P, beam, repetition_penalty=p, no_repeat_ngram_size=n)
    assert again == ids and plain != ids
    h.set_option("use_graphs", 0)
    try:
        eager, _ = h.generate(mel, P, beam, repetition_penalty=p, no_repeat_ngram_size=n)
    finally:
        h.set_option("use_graphs", 1)
    assert eager == ids


@pytest.mark.gpu
def test_options_from_init_and_from_python_bit_for_bit():
    dims, oracle, h = loop_pair()
    mel = mel_inputs(6)
    lib = _lib.lib()
    for nb, beam in ((1, 5), (2, 1), (6, 5)):                         # persistent pass and batched pass
        P = np.ascontiguousarray(np.repeat(np.array([PROMPT], np.int32), nb, 0))
        out = []
        for explicit in (False, True):
            ids = np.zeros((nb, 224), np.int32)
            lens = np.zeros(nb, np.int32)
            scores = np.zeros(nb, np.float32)
            m = np.ascontiguousarray(mel[:nb])
            if explicit:  # every field written from Python, processors off: what the ctypes mirror hands the engine
                opt = _lib.GenerateOptions(
                    struct_size=ctypes.sizeof(_lib.GenerateOptions), beam_size=beam, patience=1.0, length_penalty=1.0,
                    max_length=448, timestamps=0, max_initial_timestamp_index=50, repetition_penalty=1.0,
                    no_repeat_ngram_size=0, num_hypotheses=1, sampling_topk=1, sampling_temperature=1.0, n_extra=0,
                    extra_suppress=None, max_length_per_window=None, beam_per_window=None, patience_per_window=None,
                    length_penalty_per_window=None, seeds=None)
            else:         # wisb_generate_options_init's defaults
                opt = _lib.GenerateOptions()
                _lib.check(lib.wisb_generate_options_init(ctypes.byref(opt)))
                opt.beam_size, opt.max_length = beam, 448
            _lib.check(lib.wisb_generate(h._h, _lib.ptr(m), nb, _lib.ptr(P), P.shape[1], ctypes.byref(opt), _lib.ptr(ids),
                                         224, _lib.ptr(lens), _lib.ptr(scores)))
            out.append((ids.copy(), lens.copy(), scores.copy(), h.timing()["launches"]))
        for a, b in zip(*out):
            assert np.array_equal(a, b)


@pytest.mark.gpu
def test_options_struct_is_checked():
    dims, oracle, h = loop_pair()
    m = np.ascontiguousarray(mel_inputs(2)[:1])
    P = np.array([PROMPT], np.int32)
    ids, lens, scores = np.zeros((1, 224), np.int32), np.zeros(1, np.int32), np.zeros(1, np.float32)
    lib = _lib.lib()

    def run(**fields):
        opt = _lib.GenerateOptions()
        _lib.check(lib.wisb_generate_options_init(ctypes.byref(opt)))
        for k, v in fields.items():
            setattr(opt, k, v)
        rc = lib.wisb_generate(h._h, _lib.ptr(m), 1, _lib.ptr(P), P.shape[1], ctypes.byref(opt), _lib.ptr(ids), 224,
                               _lib.ptr(lens), _lib.ptr(scores))
        return rc, lib.wisb_last_error().decode()

    assert run(beam_size=1)[0] == 0
    for fields, msg in ((dict(struct_size=ctypes.sizeof(_lib.GenerateOptions) - 8), "struct_size"),
                        (dict(num_hypotheses=2), "num_hypotheses"),
                        (dict(sampling_topk=0, num_hypotheses=2), "beam_size must be 1")):
        rc, err = run(**fields)
        assert rc == 1 and msg in err, (fields, err)
    assert lib.wisb_generate(h._h, _lib.ptr(m), 1, _lib.ptr(P), P.shape[1], None, _lib.ptr(ids), 224, _lib.ptr(lens),
                             _lib.ptr(scores)) == 1


@pytest.mark.gpu
def test_argument_errors():
    dims, oracle, h = loop_pair()
    mel = mel_inputs(2)[:1]
    P = np.array([PROMPT], np.int32)
    for p, n in ((0.0, 0), (-1.0, 0), (float("nan"), 0), (float("inf"), 0), (1.0, -1), (1.0, 449)):
        with pytest.raises(ValueError):
            h.generate(mel, P, 1, repetition_penalty=p, no_repeat_ngram_size=n)
