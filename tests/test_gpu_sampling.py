"""GPU: sampling with num_hypotheses (``wisb_generate`` with ``sampling_topk != 1``), one step at a time and end to end.

One step (``wisb_debug_search_step`` sampling) on caller state is compared with the oracle's draw on the same processed
logits (``tests.sampling_oracle.check_draws``): the sampled id wherever the float64 key gap beats the fp32 bound (at
least 99 % of the rows), keys, cum within 4 ulps, and the whole integer state exactly.  Many seeds on identical logits
check the device generator's frequencies against softmax(l_S / T) on their own.  End to end, on the peaked synthetic
model, sampled transcripts equal the oracle's (``tests.sampling_oracle.SampleOracle``) with the same seeds on the robust
cases, on the warp-MMA, SIMT and batched passes, and a window's hypotheses depend on its seed alone."""
import functools

import numpy as np
import pytest
import torch
from scipy import stats

from tests.gpu_common import LOGIT_TOL, PROMPT, RAMP, SCRIPT, mel_inputs, robust_cases
from tests.proc_oracle import history_processors
from tests.sampling_oracle import SampleOracle, check_draws, distribution, fp32_norm, step_draws, ulps
from tests.test_gpu_search import GEOMETRIES, LDL, base_mask
from tests.ts_oracle import apply_timestamp_rules, check_invariants
from willow_inference_server_b200 import _lib, models, weights as W
from willow_inference_server_b200.batcher import TranscribeBatcher

pytestmark = pytest.mark.gpu
INT_KEYS = ("st", "flip", "seq", "indir", "tokens", "row_pos", "done", "n_hyp", "best_len", "best_tokens")
NEG = float("-inf")


@pytest.fixture(scope="module")
def h():
    return _lib.Handle.frontend(0)


# ------------------------------------------------------------------------------------------------------ one step
def processed32(x, mask, hists, gen, V, eot, no_ts, ts, max_init, rp, ngram):
    """the engine's processed logits (each processor one fp32 operation; rule 5 decided in float64 as the oracle does)"""
    t = torch.from_numpy(np.ascontiguousarray(x[:, :V]))
    if rp != 1.0 or ngram:
        t = history_processors(t, hists, rp, ngram)
    m = torch.from_numpy(mask)
    t[:, (m & 1).bool()] = NEG
    if gen == 0:
        t[:, (m & 2).bool()] = NEG
    if ts:
        t = apply_timestamp_rules(t, hists, gen, no_timestamps=no_ts, eot=eot, max_initial_timestamp_index=max_init)
    return t.numpy().astype(np.float32)


def sample_state(h, n_utt, n, *, gen, V, no_ts, rng, max_new=None, ts_hist=False):
    R = n_utt * n
    pos = gen + 3
    max_new = max_new or gen + 4
    st = h.search_state(n_utt, n, max_new, pos + 3, sample=True)
    st["st"][:2] = (pos, gen)
    st["flip"][0] = gen & 1
    st["seq"][:] = rng.integers(1000, 1400, st["seq"].shape)        # repeats: the history processors bite
    if ts_hist:
        ts = rng.random(st["seq"].shape) < 0.3
        st["seq"][ts] = rng.integers(no_ts + 1, V, int(ts.sum()))
    st["indir"][:] = rng.integers(0, R, st["indir"].shape)
    st["tokens"][:] = rng.integers(0, 50000, R)
    st["row_pos"][:] = pos
    st["cum"][:] = rng.uniform(-6, -1, R).astype(np.float32)
    return st


def expected_state(st, choice, x32, lse, *, n, eot, lp, caps):
    """the device state after one step from the rows' chosen tokens (-1 = none)"""
    out = {k: v.copy() for k, v in st.items()}
    pos, gen, _, all_done, _ = (int(v) for v in st["st"])
    if all_done:
        return out
    n_utt = len(st["done"])
    max_new = st["seq"].shape[2]
    cur = int(st["flip"][0])
    nxt = cur ^ 1
    norm = fp32_norm(gen, lp)
    for u in range(n_utt):
        cap = int(caps[u]) if caps is not None else max_new
        any_cont = False
        for r in range(u * n, (u + 1) * n):
            out["seq"][nxt, r, :gen] = st["seq"][cur, r, :gen]
            out["indir"][nxt, r, :pos] = st["indir"][cur, r, :pos]
            out["indir"][nxt, r, pos] = r
            tok = int(choice[r])
            if gen < max_new:
                out["seq"][nxt, r, gen] = tok if tok >= 0 else eot
            cont = False
            if tok >= 0:
                c = np.float32(np.float32(x32[r, tok] - lse[r]) + np.float32(st["cum"][r]))
                if tok == eot or gen + 1 >= cap:
                    out["best_tokens"][r, :gen] = st["seq"][cur, r, :gen]
                    if tok != eot:
                        out["best_tokens"][r, gen] = tok
                    out["best_len"][r] = gen + (tok != eot)
                    out["best_score"][r] = np.float32(c / norm)
                else:
                    cont = True
                    out["cum"][r] = c
            out["tokens"][r] = tok if cont else eot
            if not cont:
                out["cum"][r] = NEG
            any_cont |= cont
        if not st["done"][u] and not any_cont:
            out["done"][u] = 1
            out["st"][2] += 1
    out["st"][0] += 1
    out["st"][1] += 1
    out["st"][3] = int(out["st"][2] == n_utt)
    out["flip"][0] = nxt
    out["row_pos"] += 1
    return out


def run_step(h, *, V, eot, no_ts, n, n_utt, topk, T, gen, ts=False, rp=1.0, ngram=0, frozen=(), dead=(), caps=None,
             eot_rows=(), lp=1.0, seed=0, init=False, scale=2.0):
    rng = np.random.default_rng(seed)
    R = n_utt * n
    st = sample_state(h, n_utt, n, gen=gen, V=V, no_ts=no_ts, rng=rng, ts_hist=ts)
    x = np.full((R, LDL), np.nan, np.float32)
    x[:, :V] = rng.standard_normal((R, V)).astype(np.float32) * np.float32(scale)
    for r in eot_rows:
        x[r, eot] = 40.0
    for u in frozen:
        st["done"][u] = 1
        st["cum"][u * n:(u + 1) * n] = NEG
    st["st"][2] = int(st["done"].sum())
    for r in dead:
        st["cum"][r] = NEG
    mask = base_mask(V, eot)
    seeds = rng.integers(0, 1 << 64, n_utt, dtype=np.uint64)
    kw = dict(n=n, sampling_topk=topk, sampling_temperature=T, eot=eot, V=V, no_timestamps=no_ts, timestamps=ts,
              max_initial_timestamp_index=7, length_penalty=lp, max_new_u=caps)
    if rp != 1.0 or ngram:
        kw.update(repetition_penalty=rp, no_repeat_ngram_size=ngram)
    prompt = None
    if init:
        prompt = np.tile(np.asarray([50258, 50259, 50359], np.int32), (n_utt, 1))
        kw.update(prompt=prompt, shared_prefix=1)
        st = h.search_state(n_utt, n, st["seq"].shape[2], st["indir"].shape[2], sample=True)
    got, sampled, key, lse = h.debug_search_step_sample(x, mask, st, seeds, **kw)
    if init:  # the state search_init leaves, which the step then starts from
        st = h.search_state(n_utt, n, st["seq"].shape[2], st["indir"].shape[2], sample=True)
        st["st"][0] = 2
        st["indir"][:] = (np.arange(R) // n * n)[None, :, None]
        st["tokens"][:] = 50359
        st["row_pos"][:] = 2
        gen = 0
    cur = int(st["flip"][0])
    hists = [list(hh[:gen]) for hh in st["seq"][cur]]
    x32 = processed32(x, mask, hists, gen, V, eot, no_ts, ts, 7, rp, ngram)
    cap = caps if caps is not None else [st["seq"].shape[2]] * n_utt
    live = [not st["done"][r // n] and st["cum"][r] != NEG and gen < cap[r // n] for r in range(R)]
    for r in range(R):
        if live[r]:
            fin = x32[r][np.isfinite(x32[r])].astype(np.float64)
            want = np.logaddexp.reduce(fin) if fin.size else NEG
            assert abs(lse[r] - want) <= 1e-5 * max(1.0, abs(want)), (r, lse[r], want)
    draws = step_draws(x32, lse, st["cum"], temperature=T, topk=topk, seeds=seeds, n=n, gen=gen, live=live)
    dev_cum = np.asarray([got["cum"][r] if np.isfinite(got["cum"][r]) or d is None else d.cum
                          for r, d in enumerate(draws)], np.float32)
    info = check_draws(sampled, key, dev_cum, draws, where=(V, topk, T, n, gen, ts))
    want = expected_state(st, sampled, x32, lse, n=n, eot=eot, lp=lp, caps=caps)
    for k in INT_KEYS:
        assert np.array_equal(got[k], want[k]), (k, np.argwhere(got[k] != want[k])[:4])
    for k in ("cum", "best_score"):
        assert all(ulps(g, w) <= 4 for g, w in zip(got[k], want[k])), k
    return info, got


@pytest.mark.parametrize("geom", GEOMETRIES)
@pytest.mark.parametrize("topk", [0, 2, 5, 16])
def test_one_step_against_the_oracle(h, geom, topk):
    V, eot, no_ts = geom
    for T in (0.2, 1.0, 1.5):
        for n in (1, 5, 8):
            n_utt = max(2, 24 // n)
            run_step(h, V=V, eot=eot, no_ts=no_ts, n=n, n_utt=n_utt, topk=topk, T=T, gen=3, seed=int(T * 10) + n,
                     frozen=(1,), dead=(0,) if n > 1 else (), eot_rows=range(2 * n, 3 * n, 2))


@pytest.mark.parametrize("topk", [0, 5])
def test_timestamps_history_processors_and_caps(h, topk):
    V, eot, no_ts = GEOMETRIES[0]
    for gen in (0, 1, 4):
        run_step(h, V=V, eot=eot, no_ts=no_ts, n=5, n_utt=6, topk=topk, T=1.0, gen=gen, ts=True, seed=gen)
        run_step(h, V=V, eot=eot, no_ts=no_ts, n=5, n_utt=6, topk=topk, T=1.0, gen=gen, rp=1.3, ngram=2, seed=gen + 9)
    # the last step of window 0 (cap gen + 1), window 1 capped earlier, the others free; a cap of 0 / 1 at gen 0
    info, got = run_step(h, V=V, eot=eot, no_ts=no_ts, n=5, n_utt=4, topk=topk, T=1.0, gen=3, caps=[4, 3, 7, 7], lp=0.7)
    assert got["done"][0] == 1 and got["done"][1] == 1 and (got["best_len"][:5] == 4).all()
    info, got = run_step(h, V=V, eot=eot, no_ts=no_ts, n=8, n_utt=3, topk=topk, T=1.0, gen=0, caps=[0, 1, 4])
    assert list(got["done"]) == [1, 1, 0] and (got["best_len"][:8] == 0).all() and (got["best_len"][8:16] == 1).all()


def test_search_init_then_first_step(h):
    V, eot, no_ts = GEOMETRIES[0]
    info, got = run_step(h, V=V, eot=eot, no_ts=no_ts, n=8, n_utt=4, topk=0, T=1.0, gen=0, init=True)
    assert info["rows"] == 32                                         # every row is live at gen 0


@pytest.mark.parametrize("shape", [(1024, 1), (128, 8)])
def test_many_rows(h, shape):
    V, eot, no_ts = GEOMETRIES[1]
    n_utt, n = shape
    run_step(h, V=V, eot=eot, no_ts=no_ts, n=n, n_utt=n_utt, topk=5, T=1.0, gen=2, frozen=(3, 7), seed=4)


@pytest.mark.parametrize("topk", [0, 5])
def test_device_frequencies_pass_chi_square(h, topk):
    """128 windows x 8 hypotheses per launch on identical logits, each window its own seed: 16384 draws over eight
    launches at two generated-token indices."""
    V, eot, T = 48, 47, 0.7
    rng = np.random.default_rng(11)
    row = rng.standard_normal(V).astype(np.float32)
    row[[5, 9]] = -np.inf
    n_utt, n = 128, 8
    x = np.tile(row, (n_utt * n, 1))
    mask = np.zeros(V, np.uint8)
    counts = np.zeros(V)
    for gen in (0, 5, 0, 5, 0, 5, 0, 5):
        st = h.search_state(n_utt, n, 8, 10, sample=True)
        st["st"][:2] = (gen + 2, gen)
        st["flip"][0] = gen & 1
        st["row_pos"][:] = gen + 2
        seeds = rng.integers(0, 1 << 64, n_utt, dtype=np.uint64)
        _, sampled, _, _ = h.debug_search_step_sample(x, mask, st, seeds, n=n, sampling_topk=topk, sampling_temperature=T,
                                                      eot=eot)
        np.add.at(counts, sampled, 1)
    p = distribution(row, T, topk)
    assert counts.sum() == 8 * n_utt * n and (counts[p == 0] == 0).all()
    S = p > 0
    _, pv = stats.chisquare(counts[S], counts.sum() * p[S])
    assert pv > 1e-4, (pv, counts[S], p[S])


# ------------------------------------------------------------------------------------------------------ end to end
TS_SCRIPT = (2, 5, 8)
TS_PROMPT = PROMPT[:3]
N, TOPK, TEMP = 2, 5, 0.2     # (near-greedy draws: most cases survive the noise probe)


@functools.lru_cache(maxsize=1)
def pair():
    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=2)
    tensors = W.synth_engine_tensors(dims, seed=11, eot_ramp=RAMP, script=SCRIPT, ts_script=TS_SCRIPT)
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    return dims, SampleOracle.from_blob(buf), _lib.Handle.from_host(buf, 0)


SKW = dict(num_hypotheses=N, sampling_topk=TOPK, sampling_temperature=TEMP)


@functools.lru_cache(maxsize=None)
def oracle_window(i, seed, prompt=tuple(PROMPT), proc=()):
    """(oracle result, robust) of window i alone with this seed: unchanged under one logit-noise probe and every draw's
    key gap above LOGIT_TOL / T"""
    _, oracle, _ = pair()
    mel = mel_inputs(16)[i: i + 1]
    kw = dict(SKW, random_seed=seed, **dict(proc))
    res, robust = robust_cases(oracle, mel, [list(prompt)], 1, n_probe=1, **kw)
    ok = bool(robust)
    if ok:
        trace = []
        oracle.generate(mel, [list(prompt)], beam_size=1, trace=trace, **kw)
        ok = min((d.gap for d in trace[0] if d is not None), default=np.inf) > LOGIT_TOL / TEMP
    return res[0], ok


def engine(h, mel, prompts, seeds, **kw):
    return h.generate_sample(mel, prompts, N, TOPK, TEMP, np.asarray(seeds, np.uint64), **kw)


@pytest.mark.parametrize("path", ["mma", "simt", "batched"])
def test_transcripts_match_the_oracle(path):
    _, _, h = pair()
    mel = mel_inputs(16)
    seeds = [1000 + 17 * i for i in range(16)]
    h.set_option("mega_mma", 0 if path == "simt" else 1)
    try:
        if path == "batched":
            seqs, scores = engine(h, mel, np.asarray([PROMPT] * 16, np.int32), seeds)
            idx = range(16)
        else:   # 5 rows: the persistent pass takes one window per call
            idx = range(6)
            outs = [engine(h, mel[i: i + 1], np.asarray([PROMPT], np.int32), seeds[i: i + 1]) for i in idx]
            seqs, scores = [o[0][0] for o in outs], [o[1][0] for o in outs]
    finally:
        h.set_option("mega_mma", 1)
    robust = 0
    for j, i in enumerate(idx):
        want, ok = oracle_window(i, seeds[i])
        assert scores[j] == sorted(scores[j], reverse=True)
        if not ok:
            continue
        robust += 1
        assert seqs[j] == want.sequences_ids, (path, i)
        assert np.allclose(scores[j], want.scores, atol=5e-2), (path, i, scores[j], want.scores)
    assert robust >= (2 if path == "batched" else 1), (path, robust)


def test_a_window_depends_on_its_seed_alone():
    """16-window call == each window alone (both on the batched pass, same plans) == the batcher == an encode() output,
    bit for bit; the same seed repeats; another seed differs."""
    _, _, h = pair()
    mel = mel_inputs(16)
    seeds = np.arange(16, dtype=np.uint64) + np.uint64((1 << 64) - 8)     # (wraps past 2^64 - 1)
    P16 = np.asarray([PROMPT] * 16, np.int32)
    h.set_option("decoder_batch", 2)
    try:
        full = engine(h, mel, P16, seeds)
        again = engine(h, mel, P16, seeds)
        assert full == again
        for i in (0, 5, 15):
            solo = engine(h, mel[i: i + 1], P16[:1], seeds[i: i + 1])
            assert solo[0][0] == full[0][i] and solo[1][0] == full[1][i], i
        other = engine(h, mel, P16, seeds + np.uint64(1))
        assert other[0] != full[0]
        m = models.Whisper(None, device="cuda", _handles=[h])
        with TranscribeBatcher(m, max_batch=16, max_wait_ms=200) as b:
            futs = [b.submit(mel[i: i + 4], PROMPT, beam_size=1, return_scores=True, random_seed=int(seeds[i]), **SKW)
                    for i in range(0, 16, 4)]
            res = [r for f in futs for r in f.result(timeout=600)]
        # request j's windows get seeds[4 j] + w = seeds[4 j + w]
        assert [r.sequences_ids for r in res] == full[0] and [r.scores for r in res] == full[1]
        enc = m.encode(models.StorageView.from_array(mel))
        r_enc = m.generate(enc, [PROMPT] * 16, beam_size=1, return_scores=True, random_seed=[int(s) for s in seeds],
                           **SKW)
        assert [r.sequences_ids for r in r_enc] == full[0] and [r.scores for r in r_enc] == full[1]
    finally:
        h.set_option("decoder_batch", 1)


def test_timestamps_and_no_repeat_ngram():
    dims, _, h = pair()
    mel = mel_inputs(16)
    seqs, scores = engine(h, mel, np.asarray([TS_PROMPT] * 16, np.int32), range(16), timestamps=True)
    for hyps in seqs:
        for s in hyps:
            if s:
                check_invariants(s, dims)
    seqs, _ = engine(h, mel, np.asarray([PROMPT] * 16, np.int32), range(16), no_repeat_ngram_size=2)
    for hyps in seqs:
        for s in hyps:
            grams = [tuple(s[i: i + 2]) for i in range(len(s) - 1)]
            assert len(grams) == len(set(grams)), s
    assert all(sc == sorted(sc, reverse=True) for sc in scores)


def test_faster_whisper_fallback_call():
    _, _, h = pair()
    m = models.Whisper(None, device="cuda", _handles=[h])
    enc = m.encode(models.StorageView.from_array(mel_inputs(1)))
    res = m.generate(enc, [PROMPT], beam_size=1, num_hypotheses=5, sampling_topk=0, sampling_temperature=0.2,
                     length_penalty=1, max_length=448, return_scores=True, return_no_speech_prob=True,
                     suppress_blank=True, suppress_tokens=[-1], max_initial_timestamp_index=50)
    assert len(res) == 1 and len(res[0].sequences_ids) == 5 and len(res[0].scores) == 5
    assert res[0].scores == sorted(res[0].scores, reverse=True) and all(np.isfinite(res[0].scores))
