"""Sampling with num_hypotheses on top of the fp32 oracle (TEST INFRASTRUCTURE ONLY).

Restates the engine's sampling search (csrc/search.cu header comment, DESIGN.md section 5): beam_size 1 with
sampling_topk != 1 draws num_hypotheses independent hypotheses per window, each row from softmax(l_S / T) over the
processed logits l by the Gumbel-max trick with noise from Philox4x32-10 keyed by the window's seed.
  * ``philox4x32_10``: the Random123 generator (Salmon et al., SC'11), checked against its known-answer vectors;
  * ``gumbel(seed, k, gen, v)``: the noise of token v for hypothesis k at generated-token index gen, in float64;
  * ``sample_row``: one row's draw (candidates, keys, the untempered log-prob); ``sample_search``: the loop for one
    window with the same ``logits_fn`` / ``process`` contract as ``oracle.whisper_ref.beam_search``;
  * ``SampleOracle``: ``tests.proc_oracle.ProcOracle`` (timestamp rules and history processors) with
    ``generate(..., num_hypotheses, sampling_topk, sampling_temperature, random_seed)``.
The distribution it samples is pinned to transformers' TemperatureLogitsWarper -> TopKLogitsWarper -> softmax by
``tests/golden/sampling_warpers_hf.npz`` (``scripts/gen_golden_sampling_hf.py``).  ``SAMPLE_DEFECTS`` are the wrong
variants the comparator tests inject.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from oracle.whisper_ref import GenerationResult, length_norm
from tests.proc_oracle import ProcOracle

NEG_INF = float("-inf")
# T applied as a multiply by 1/T, one log in the Gumbel transform, k or gen missing from the counter, the score taken
# from the tempered log-prob, top-k ties to the highest id
SAMPLE_DEFECTS = ("t_multiply", "single_log", "no_k", "no_gen", "tempered_score", "topk_ties_high")

_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85


def philox4x32_10(ctr, key):
    """ctr: 4 uint32 arrays (broadcastable), key: 2 uint32 values -> the 4 output words (uint32 arrays)."""
    c = [np.asarray(x, np.uint64) & 0xFFFFFFFF for x in ctr]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    m = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(_M0) * c[0]
        p1 = np.uint64(_M1) * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0)) & m, p1 & m, ((p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1)) & m,
             p0 & m]
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return [x.astype(np.uint32) for x in c]


def uniform(seed: int, k, gen, v) -> np.ndarray:
    """(k, gen, v broadcast) u = ((x >> 9) + 0.5) * 2^-23 of word 0 for counter (v, gen, k, 0), key (lo32(seed), hi32(seed)): in (0, 1)."""
    v, gen, k = np.broadcast_arrays(*(np.asarray(a, np.uint64) for a in (v, gen, k)))
    x = philox4x32_10((v, gen, k, np.zeros_like(v)),
                      (int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF))[0]
    return ((x >> np.uint32(9)).astype(np.float64) + 0.5) * 2.0 ** -23


def gumbel(seed: int, k: int, gen: int, v, defect=None) -> np.ndarray:
    """float64 Gumbel noise -log(-log u) of tokens v (one log with the "single_log" defect)."""
    u = uniform(seed, 0 if defect == "no_k" else k, 0 if defect == "no_gen" else gen, v)
    return -np.log(u) if defect == "single_log" else -np.log(-np.log(u))


def candidates(l32: np.ndarray, topk: int, defect=None) -> np.ndarray:
    """The candidate ids S of a row's processed logits (ascending): every finite one (topk 0) or the topk largest,
    ties to the lowest id (the highest with the "topk_ties_high" defect)."""
    fin = np.nonzero(np.isfinite(l32))[0]
    if topk == 0 or fin.size <= topk:
        return fin
    tie = -fin if defect == "topk_ties_high" else fin
    order = np.lexsort((tie, -l32[fin].astype(np.float64)))
    return np.sort(fin[order[:topk]])


@dataclass
class Draw:
    tok: int          # sampled id
    key: float        # its key fp32(l / T) + g (float64 sum)
    a: float          # fp32(l / T)
    g: float          # its noise
    gap: float        # key - the runner-up's key (inf without a runner-up)
    g2: float         # the runner-up's noise (0 without one)
    runner: int       # the runner-up's id (-1 without one)
    cum: float        # fp32 (l - lse) + cum
    logit: float      # l


def sample_row(l32, lse32, cum32, temperature, topk, seed, k, gen, defect=None):
    """One row's draw from processed fp32 logits l32 [V] (-inf = off) with the row's fp32 lse -> Draw, or None when no
    token can be sampled."""
    S = candidates(l32, topk, defect)
    if S.size == 0:
        return None
    T = np.float32(temperature)
    if defect == "t_multiply":
        a = (l32[S] * np.float32(np.float32(1.0) / T)).astype(np.float32)
    else:
        a = (l32[S] / T).astype(np.float32)
    g = gumbel(seed, k, gen, S, defect)
    key = a.astype(np.float64) + g
    i = int(np.argmax(key))        # first of equal keys: the lowest id (S ascending)
    j = -1
    if S.size > 1:
        rest = key.copy()
        rest[i] = -np.inf
        j = int(np.argmax(rest))
    v = int(S[i])
    if defect == "tempered_score":
        t = torch.from_numpy(l32.astype(np.float32)) / float(T)
        lp = np.float32(float(torch.log_softmax(t, -1)[v]))
    else:
        lp = np.float32(np.float32(l32[v]) - np.float32(lse32))
    return Draw(v, float(key[i]), float(a[i]), float(g[i]), float(key[i] - key[j]) if j >= 0 else np.inf,
                float(g[j]) if j >= 0 else 0.0, int(S[j]) if j >= 0 else -1, float(np.float32(lp + np.float32(cum32))),
                float(l32[v]))


def key_bound(key: float, g1: float, g2: float) -> float:
    """Largest change of the engine's fp32 key difference against float64: the fp32 noise (logf is within 1 ulp, twice
    composed: relative 2^-22 on -log u and 2^-22 on the result) and the rounding of both fp32 sums."""
    ulp = np.spacing(np.float32(abs(key) + abs(g1) + abs(g2) + 1.0))
    return float(2.0 ** -19 * (2.0 + abs(g1) + abs(g2)) + 2.0 * ulp)


def fp32_norm(gen: int, lp: float) -> np.float32:
    return np.float32(length_norm(gen, float(np.float32(lp))))


def sample_search(logits_fn, process, *, n: int, V: int, eot: int, max_new: int, temperature: float, topk: int,
                  seed: int, length_penalty: float = 1.0, trace=None, defect=None):
    """One window's n hypotheses -> [(score, tokens)] per hypothesis index k (not sorted).  logits_fn(s, tokens) -> raw
    logits [n, V] of step s (or [1, V] at s = 0: every row holds the prompt), row k fed tokens[k]; process(logits, hists,
    s) -> processed logits.  trace, if a list, receives every draw's Draw."""
    if max_new <= 0:
        return [(0.0, [])] * n
    seqs, cum, alive = [[] for _ in range(n)], [np.float32(0.0)] * n, [True] * n
    hyps = [(NEG_INF, [])] * n
    tokens = None
    for s in range(max_new):
        logits = logits_fn(s, tokens)
        if logits.shape[0] == 1:
            logits = logits.expand(n, -1)
        x = process(logits, seqs, s).float()
        lse = torch.logsumexp(x, -1).numpy().astype(np.float32)
        x32 = x.numpy().astype(np.float32)
        norm = fp32_norm(s, length_penalty)
        tokens = []
        for k in range(n):
            if not alive[k]:
                tokens.append(eot)
                continue
            d = sample_row(x32[k], lse[k], cum[k], temperature, topk, seed, k, s, defect)
            if trace is not None:
                trace.append(d)
            if d is None:
                alive[k] = False
                tokens.append(eot)
                continue
            if d.tok == eot or s + 1 == max_new:
                hyps[k] = (float(np.float32(np.float32(d.cum) / norm)), seqs[k] + ([] if d.tok == eot else [d.tok]))
                alive[k] = False
                tokens.append(eot)
            else:
                seqs[k] = seqs[k] + [d.tok]
                cum[k] = np.float32(d.cum)
                tokens.append(d.tok)
        if not any(alive):
            break
    return hyps


def ranked(hyps):
    """hypotheses sorted by score, descending, ties to the lower hypothesis index"""
    order = sorted(range(len(hyps)), key=lambda k: -hyps[k][0])
    return [hyps[k] for k in order]


class SampleOracle(ProcOracle):
    """ProcOracle with sampling: generate(..., num_hypotheses, sampling_topk, sampling_temperature, random_seed) returns
    num_hypotheses sequences and scores per window, best first.  random_seed: an int s (window w gets s + w mod 2^64)
    or one seed per window."""

    def generate(self, features, prompts, beam_size: int = 1, num_hypotheses: int = 1, sampling_topk: int = 1,
                 sampling_temperature: float = 1.0, random_seed=0, length_penalty: float = 1.0, max_length: int = 448,
                 trace=None, enc=None, logit_noise=None, sample_defect=None, **kw):
        if sampling_topk == 1:
            return super().generate(features, prompts, beam_size=beam_size, length_penalty=length_penalty,
                                    max_length=max_length, trace=trace, enc=enc, logit_noise=logit_noise, **kw)
        assert beam_size == 1
        n = len(prompts)
        seeds = ([(int(random_seed) + w) % (1 << 64) for w in range(n)] if np.isscalar(random_seed)
                 else [int(s) % (1 << 64) for s in random_seed])
        # the processors of ProcOracle / TimestampOracle, set up as their generate would
        self.max_initial_timestamp_index = kw.pop("max_initial_timestamp_index", 50)
        self.disable = ()
        self.repetition_penalty = kw.pop("repetition_penalty", 1.0)
        self.no_repeat_ngram_size = kw.pop("no_repeat_ngram_size", 0)
        self.proc_defect = None
        extra = [t for t in kw.pop("suppress_tokens", (-1,)) if t >= 0]
        self.logit_noise = None
        if logit_noise is not None:
            g = torch.Generator()
            g.manual_seed(int(logit_noise[1]))
            self.logit_noise = (float(logit_noise[0]), g)
        try:
            if enc is None:
                enc = self.encode(features)
            out = []
            for b, prompt in enumerate(prompts):
                tr = [] if trace is not None else None
                hyps = self._sample(enc[b], list(prompt), num_hypotheses, sampling_topk, sampling_temperature, seeds[b],
                                    length_penalty, max_length, extra, tr, sample_defect)
                if trace is not None:
                    trace.append(tr)
                r = ranked(hyps)
                out.append(GenerationResult([t for _, t in r], [s for s, _ in r]))
            return out
        finally:
            self.logit_noise = None
            self.repetition_penalty, self.no_repeat_ngram_size = 1.0, 0

    @torch.no_grad()
    def _sample(self, enc_row, prompt, n, topk, temperature, seed, length_penalty, max_length, extra, trace, defect):
        ckv = self.cross_kv(enc_row)
        cache = self._prefill(prompt, ckv)
        start = len(prompt) - 1

        def logits_fn(s, tokens):
            nonlocal cache
            if s == 0:
                logits, cache = self.decode_rows([prompt[-1]], start, cache, ckv)
                cache = [(k_.expand(n, -1, -1).contiguous(), v_.expand(n, -1, -1).contiguous()) for k_, v_ in cache]
                return logits
            logits, cache = self.decode_rows(tokens, start + s, cache, ckv)
            return logits

        return sample_search(logits_fn, self._processors(prompt, extra), n=n, V=self.dims.n_vocab, eot=self.dims.eot,
                             max_new=self.max_new_tokens(len(prompt), max_length), temperature=temperature, topk=topk,
                             seed=seed, length_penalty=length_penalty, trace=trace, defect=defect)


def distribution(l32, temperature, topk) -> np.ndarray:
    """float64 probabilities [V] the engine samples from: softmax(fp32(l / T)) over the candidates, 0 elsewhere."""
    S = candidates(l32, topk)
    p = np.zeros(l32.shape[0], np.float64)
    a = (l32[S] / np.float32(temperature)).astype(np.float32).astype(np.float64)
    e = np.exp(a - a.max())
    p[S] = e / e.sum()
    return p


def step_draws(x32, lse32, cum32, *, temperature, topk, seeds, n, gen, live=None, defect=None):
    """Every row's Draw (or None) of one step: x32 [R, V] processed fp32 logits, lse32 / cum32 [R], seeds [n_utt], row r
    = hypothesis r mod n of window r // n; live [R] (None = all) -- the others get None."""
    out = []
    for r in range(x32.shape[0]):
        if live is not None and not live[r]:
            out.append(None)
            continue
        out.append(sample_row(x32[r], lse32[r], cum32[r], temperature, topk, int(seeds[r // n]), r % n, gen, defect))
    return out


def ulps(a, b) -> int:
    a, b = np.float32(a), np.float32(b)
    if a == b:
        return 0
    if not (np.isfinite(a) and np.isfinite(b)):
        return 1 << 30
    ia, ib = (int(np.array(x, np.float32).view(np.int32)) for x in (a, b))
    ia = ia if ia >= 0 else -(ia & 0x7fffffff)
    ib = ib if ib >= 0 else -(ib & 0x7fffffff)
    return abs(ia - ib)


def check_draws(sampled, key, cum, draws, *, min_qualify=0.99, where="") -> dict:
    """Compare one step of the engine (sampled id, key and new cum per row; -1 / anything / anything where it drew
    nothing) with the oracle's draws.  Rows whose float64 gap beats key_bound must draw the oracle's token (and at least
    min_qualify of the drawing rows must qualify); a row inside a near-tie must draw the oracle's token or its runner-up.
    Where the tokens agree: the key within key_bound of float64, the new cum within 4 ulps, and where |fp32(l / T)| >=
    2^12 (its ulp dwarfs the noise's rounding) the key must be exactly fp32(fp32(l / T) + fp32(g)) in >= 99 % of the
    rows.  -> {"rows", "qualify", "large", "large_exact"}; AssertionError on a difference."""
    rows = qual = large = exact = 0
    for r, d in enumerate(draws):
        if d is None:
            assert sampled[r] == -1, (where, r, sampled[r])
            continue
        rows += 1
        b = key_bound(d.key, d.g, d.g2)
        if d.gap > b:
            qual += 1
            assert sampled[r] == d.tok, (where, "token", r, int(sampled[r]), d.tok, d.gap)
        else:
            assert sampled[r] in (d.tok, d.runner), (where, "near-tie token", r, int(sampled[r]), d.tok, d.runner)
        if sampled[r] != d.tok:
            continue
        assert abs(float(key[r]) - d.key) <= key_bound(d.key, d.g, 0.0), (where, "key", r, float(key[r]), d.key)
        assert ulps(cum[r], d.cum) <= 4, (where, "cum", r, float(cum[r]), d.cum)
        if abs(d.a) >= 2.0 ** 12:
            large += 1
            exact += int(np.float32(key[r]) == np.float32(np.float32(d.a) + np.float32(d.g)))
    assert qual >= min_qualify * rows, (where, "too few rows qualify", qual, rows)
    assert exact >= 0.99 * large, (where, "large keys not exact", exact, large)
    return {"rows": rows, "qualify": qual, "large": large, "large_exact": exact}
