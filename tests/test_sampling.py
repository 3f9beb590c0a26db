"""Sampling without a GPU: the Philox generator, the oracle's distribution against transformers, the comparator the
GPU step tests use, and the argument rules of models.Whisper.generate, Handle.generate_sample and the batcher."""
import os

import numpy as np
import pytest
from scipy import stats

from tests.sampling_oracle import (SAMPLE_DEFECTS, candidates, check_draws, distribution, gumbel, philox4x32_10,
                                   sample_row, step_draws)
from willow_inference_server_b200 import models, set_random_seed
from willow_inference_server_b200.batcher import TranscribeBatcher
from willow_inference_server_b200.models import WhisperGenerationResult

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "sampling_warpers_hf.npz")
P = [50258, 50259, 50359, 50363]


def test_philox_known_answers():
    # Random123's kat_vectors for philox4x32_10
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
              (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in cases:
        got = tuple(int(w) for w in philox4x32_10([np.uint32(c) for c in ctr], key))
        assert got == want, [hex(w) for w in got]


def test_distribution_matches_transformers_warpers():
    g = np.load(GOLDEN)
    for i, V in enumerate(g["V"]):
        x = g["logits"][i, :V]
        for a, t in enumerate(g["temps"]):
            for b, k in enumerate(g["topks"]):
                want = g["probs"][i, a, b, :V]
                got = distribution(x, float(t), int(k))
                assert np.abs(got - want).max() <= 1e-6, (i, t, k)


@pytest.mark.parametrize("topk", [0, 5])
@pytest.mark.parametrize("temperature", [0.5, 1.5])
def test_gumbel_max_frequencies_pass_chi_square(topk, temperature):
    """2^16 draws (hypotheses 0..7 x steps 0..8191 of one seed) of one row against softmax(l_S / T)."""
    x = np.random.default_rng(3).standard_normal(24).astype(np.float32)
    x[[3, 11]] = -np.inf
    p = distribution(x, temperature, topk)
    S = candidates(x, topk)
    a = (x[S] / np.float32(temperature)).astype(np.float64)
    counts = np.zeros(x.size)
    gens = np.arange(8192)[:, None]
    for k in range(8):
        np.add.at(counts, S[np.argmax(a + gumbel(77, k, gens, S[None, :]), axis=1)], 1)
    assert counts.sum() == 1 << 16 and (counts[p == 0] == 0).all()
    _, pv = stats.chisquare(counts[S], (1 << 16) * p[S])
    assert pv > 1e-4, (pv, counts[S], p[S])


def test_ties_go_to_the_lowest_id():
    x = np.full(30, -np.inf, np.float32)
    x[[4, 9, 17, 21, 25]] = [3.0, 1.0, 1.0, 1.0, 2.0]
    assert list(candidates(x, 3)) == [4, 9, 25]                   # of the tied 9 / 17 / 21 only 9 is a candidate
    assert list(candidates(x, 3, "topk_ties_high")) == [4, 21, 25]
    # equal keys: the lowest id wins (a row of equal logits at gen / k where two noises coincide does not exist in
    # practice, so check the rule on the argmax the oracle uses)
    assert int(np.argmax(np.asarray([1.0, 2.0, 2.0]))) == 1


def crafted_step(V=300, n_utt=48, n=4, gen=3, topk=0, temperature=1.0, seed=5):
    """Processed logits for the comparator: every window's rows share their logits (so hypotheses must differ), the
    first third of the windows hold large logits (|l / T| >= 2^12, where the key must be exact), ties at the top-k
    boundary in the rest."""
    rng = np.random.default_rng(seed)
    R = n_utt * n
    x = np.full((R, V), -np.inf, np.float32)
    for u in range(n_utt):
        row = rng.standard_normal(V).astype(np.float32)
        row[rng.choice(V, V // 5, replace=False)] = -np.inf
        if u < n_utt // 3:
            row = (row * np.float32(0.01) + np.float32(6000.0) * np.float32(temperature)).astype(np.float32)
            row[~np.isfinite(row)] = -np.inf
        elif topk:
            top = np.sort(row[np.isfinite(row)])[::-1]
            fin = np.nonzero(np.isfinite(row))[0]
            row[fin[:4]] = top[topk - 1]                           # several ids tied with the k-th value
        x[u * n:(u + 1) * n] = row
    lse = np.asarray([np.logaddexp.reduce(r[np.isfinite(r)].astype(np.float64)) for r in x], np.float32)
    cum = np.full(R, -2.5, np.float32)
    seeds = rng.integers(0, 1 << 63, n_utt, dtype=np.uint64)
    return x, lse, cum, seeds


def as_device(draws):
    sampled = np.asarray([d.tok if d else -1 for d in draws], np.int32)
    key = np.asarray([np.float32(d.key) if d else -np.inf for d in draws], np.float32)
    cum = np.asarray([d.cum if d else -np.inf for d in draws], np.float32)
    return sampled, key, cum


@pytest.mark.parametrize("topk", [0, 5])
def test_comparator_accepts_the_oracle_itself(topk):
    x, lse, cum, seeds = crafted_step(topk=topk, temperature=1.5)
    d = step_draws(x, lse, cum, temperature=1.5, topk=topk, seeds=seeds, n=4, gen=3)
    info = check_draws(*as_device(d), d, min_qualify=0.9)
    assert info["large"] > 50 and info["qualify"] > 100


@pytest.mark.parametrize("defect", SAMPLE_DEFECTS)
def test_comparator_rejects_injected_defects(defect):
    topk = 5
    x, lse, cum, seeds = crafted_step(topk=topk, temperature=1.5)
    want = step_draws(x, lse, cum, temperature=1.5, topk=topk, seeds=seeds, n=4, gen=3)
    bad = step_draws(x, lse, cum, temperature=1.5, topk=topk, seeds=seeds, n=4, gen=3, defect=defect)
    with pytest.raises(AssertionError):
        check_draws(*as_device(bad), want, min_qualify=0.9)


def test_empty_candidate_set_draws_nothing():
    x = np.full(10, -np.inf, np.float32)
    assert sample_row(x, np.float32(0), np.float32(0), 1.0, 0, 1, 0, 0) is None


# ------------------------------------------------------------------------------------------------ Python-side rules
class FakeHandle:
    def __init__(self):
        self.calls, self.samples = [], []

    def dims(self):
        return {"d_model": 384, "n_vocab": 51865, "no_timestamps": 50363, "n_text_ctx": 448, "lang_first": 50259,
                "n_langs": 99, "n_mels": 80}

    def set_option(self, *a):
        pass

    def generate(self, mel, prompts, *args, **kw):
        self.calls.append((args, kw))
        return [[1, 2]] * mel.shape[0], [0.0] * mel.shape[0]

    def generate_sample(self, mel, prompts, n, topk, temperature, seeds, *args, **kw):
        self.samples.append(dict(n=n, topk=topk, temperature=temperature, seeds=[int(s) for s in seeds], args=args,
                                 kw=kw))
        return [[[k] for k in range(n)] for _ in range(mel.shape[0])], [[-0.1 * k for k in range(n)]] * mel.shape[0]


def feats(n=1):
    return models.StorageView.from_array(np.zeros((n, 80, 3000), np.float32))


def test_generate_validates_the_sampling_options():
    h = FakeHandle()
    m = models.Whisper(None, device="cuda", _handles=[h])
    bad = [dict(num_hypotheses=2), dict(num_hypotheses=2, beam_size=1),             # n > 1 needs sampling
           dict(sampling_topk=3),                                                     # beam 5 with sampling
           dict(beam_size=1, sampling_topk=17), dict(beam_size=1, sampling_topk=-1),
           dict(beam_size=1, sampling_topk=True), dict(beam_size=1, sampling_topk=2.0),
           dict(beam_size=1, sampling_topk=0, sampling_temperature=0),
           dict(beam_size=1, sampling_topk=0, sampling_temperature=float("nan")),
           dict(beam_size=1, sampling_topk=0, sampling_temperature=float("inf")),
           dict(beam_size=1, sampling_topk=0, num_hypotheses=9), dict(beam_size=1, sampling_topk=0, num_hypotheses=0),
           dict(beam_size=[1], sampling_topk=0), dict(beam_size=1, patience=[1.0], sampling_topk=0),
           dict(beam_size=1, sampling_topk=0, random_seed="1"), dict(beam_size=1, sampling_topk=0, random_seed=[1, 2])]
    for kw in bad:
        with pytest.raises(ValueError):
            m.generate(feats(), [P], **kw)
    assert not h.calls and not h.samples


def test_greedy_and_beam_calls_reach_handle_generate_unchanged():
    h = FakeHandle()
    m = models.Whisper(None, device="cuda", _handles=[h])
    m.generate(feats(), [P], beam_size=5)
    m.generate(feats(), [P], beam_size=1, sampling_topk=1, sampling_temperature=0.7, random_seed=3)
    m.generate(feats(), [P], beam_size=1)
    assert not h.samples
    assert h.calls[1] == h.calls[2] and h.calls[0][0][0] == 5        # the temperature is ignored at topk 1


def test_sampling_results_and_seeds():
    h = FakeHandle()
    m = models.Whisper(None, device="cuda", _handles=[h])
    fw = dict(beam_size=1, num_hypotheses=5, sampling_topk=0, sampling_temperature=0.2, length_penalty=1,
              max_length=448, return_scores=True, return_no_speech_prob=True, suppress_blank=True,
              suppress_tokens=[-1], max_initial_timestamp_index=50)
    r = m.generate(feats(), [P], **fw)
    assert len(r) == 1 and len(r[0].sequences_ids) == 5 and len(r[0].scores) == 5 and r[0].no_speech_prob == 0.0
    s = h.samples[-1]
    assert (s["n"], s["topk"], s["temperature"]) == (5, 0, 0.2)
    m.generate(feats(3), [P] * 3, **fw, random_seed=(1 << 64) - 2)
    assert h.samples[-1]["seeds"] == [(1 << 64) - 2, (1 << 64) - 1, 0]
    m.generate(feats(2), [P] * 2, **fw, random_seed=[7, 3])
    assert h.samples[-1]["seeds"] == [7, 3]
    set_random_seed(42)
    m.generate(feats(2), [P] * 2, **fw)
    first = h.samples[-1]["seeds"]
    set_random_seed(42)
    m.generate(feats(2), [P] * 2, **fw)
    assert h.samples[-1]["seeds"] == first and first[1] == (first[0] + 1) % (1 << 64)
    r = m.generate(feats(), [P], **dict(fw, return_scores=False))
    assert r[0].scores == []


def test_seeds_spread_across_replicas():
    hs = [FakeHandle(), FakeHandle()]
    m = models.Whisper(None, device="cuda", device_index=[0, 1], _handles=hs)
    m.generate(feats(4), [P] * 4, beam_size=1, num_hypotheses=2, sampling_topk=0, random_seed=100)
    assert [s for h in hs for c in h.samples for s in c["seeds"]] == [100, 101, 102, 103]


class FakeEngine:
    per_window_options = True
    dims = {"no_timestamps": 50363}

    def __init__(self):
        self.calls = []

    def generate(self, features, prompts, **opts):
        self.calls.append((features.array.shape[0], dict(opts)))
        n = opts.get("num_hypotheses", 1)
        seeds = opts.get("random_seed")
        return [WhisperGenerationResult([[int(w[0, 0]), -1 if seeds is None else int(seeds[i])]] * n)
                for i, w in enumerate(features.array)]


def test_batcher_keeps_sampling_apart_and_passes_each_requests_seeds():
    eng = FakeEngine()
    win = lambda tag, n=1: np.full((n, 80, 3000), tag, np.float32)  # noqa: E731
    smp = dict(beam_size=1, num_hypotheses=5, sampling_topk=0, sampling_temperature=0.2)
    with TranscribeBatcher(eng, max_batch=16, max_wait_ms=200) as b:
        futs = [b.submit(win(0), P, beam_size=5),
                b.submit(win(1, 2), P, **smp, random_seed=10),
                b.submit(win(2), P, beam_size=1),
                b.submit(win(3, 3), P, **smp, random_seed=(1 << 64) - 1),
                b.submit(win(4), P, **dict(smp, sampling_temperature=0.4), random_seed=1),
                b.submit(win(5), P, **smp)]
        res = [f.result(timeout=10) for f in futs]
    seeds = [[r.sequences_ids[0][1] for r in rs] for rs in res]
    assert seeds[1] == [10, 11] and seeds[3] == [(1 << 64) - 1, 0, 1] and seeds[4] == [1]
    assert seeds[0] == [-1] and seeds[2] == [-1]                     # beam requests: no seeds
    assert all(len(r.sequences_ids) == 5 for r in res[1] + res[3] + res[4] + res[5])
    for n, opts in eng.calls:
        sampling = opts.get("sampling_topk", 1) != 1
        assert sampling == ("random_seed" in opts)
        if sampling:
            assert opts["beam_size"] == 1 and len(opts["random_seed"]) == n
    # requests 1, 3 and 5 share a call; 4 (another temperature) and the beam requests do not join it
    assert sorted(n for n, o in eng.calls if o.get("sampling_temperature") == 0.2) == [6]


def test_batcher_refuses_bad_sampling_options_at_submit():
    eng = FakeEngine()
    with TranscribeBatcher(eng, max_batch=16, max_wait_ms=1) as b:
        for kw in (dict(sampling_topk=3), dict(beam_size=1, sampling_topk=20), dict(num_hypotheses=3),
                   dict(beam_size=1, sampling_topk=0, sampling_temperature=-1.0),
                   dict(beam_size=1, sampling_topk=0, random_seed=1.5)):
            with pytest.raises(ValueError):
                b.submit(np.zeros((1, 80, 3000), np.float32), P, **kw)
    assert not eng.calls
