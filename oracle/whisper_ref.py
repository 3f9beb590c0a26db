"""Oracle: fp32 CPU restatement of the Whisper model call behind ``ctranslate2.models.Whisper``.

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.

What it restates (reference call sites; the arithmetic itself lives in the
un-vendored dependency ctranslate2==4.1.0, requirements.txt:22):
  * ``Whisper.generate(features, prompts, beam_size=, return_scores=False)``
        main.py:687-692 (positional form :535-537)
  * ``Whisper.detect_language(features)``          main.py:638-640
  * result use ``results[i].sequences_ids[0]``     main.py:707,713

Model arithmetic follows the Whisper architecture as implemented in
[HF] transformers/models/whisper/modeling_whisper.py (conv stem :567-568,:619-620;
sinusoid table :55; attention scaling / k_proj without bias :267,:279,:310;
encoder layer :361-415; decoder layer :417-508; tied output projection :966-971)
and is PINNED against that independent implementation in
``tests/test_oracle_whisper.py`` (golden ``tests/golden/whisper_hf_tiny.npz``).

Decoding follows the published CTranslate2 4.1.0 algorithm (src/decoding.cc
``GreedySearch`` / ``BeamSearch``, src/models/whisper.cc) as summarised in
SURVEY.md section 8a rows A11-A14:
  - prompt[:-1] is forwarded once to fill the self-attention cache, decoding
    starts from the last prompt token;
  - max generated tokens = min(max_length // 2, max_length - len(prompt)), max_length 448;
  - logits processors: ``suppress_ids`` every step, ``suppress_ids_begin``
    ({blank, eot}) at the first generated step; timestamp rules are off because
    the WIS prompt contains <|notimestamps|> (main.py:661);
  - greedy (beam_size 1): arg-max (lowest id on ties), stop at eot, eot excluded;
  - beam search: log-softmax, cumulative scores, length-normalised by
    (step+1)^length_penalty, top 2*beam of beam*V, the first ``beam`` candidates
    that end in eot become finished hypotheses and are replaced by the next
    non-eot candidates, an utterance finishes once round(beam*patience)
    hypotheses exist (length_penalty != 0 disables the early exit) or at the last
    step, best normalised score wins (num_hypotheses=1).
**PARITY UNPINNED for the decoding rules**: no CTranslate2 binary, source or
golden transcript ships with the reference server.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
import torch
import torch.nn.functional as F

from willow_inference_server_b200.weights import WhisperDims, read_blob

NEG_INF = float("-inf")


@dataclass
class GenerationResult:
    sequences_ids: list  # list[list[int]] (num_hypotheses = 1)
    scores: list  # list[float]


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).float()


# ------------------------------------------------------------------------------------------------------------ search
def max_hypotheses(beam: int, patience: float) -> int:
    """Finished hypotheses that end an utterance's search: beam * patience rounded half up, in fp32 as the engine
    computes it, and at least 1.  UNPINNED: CTranslate2 is C++ and presumably rounds with std::round (half away from
    zero, the same for positive values); Python's round() would round half to even (beam 5 x patience 0.5 -> 2)."""
    return max(1, int(np.float32(beam) * np.float32(patience) + np.float32(0.5)))


def length_norm(gen: int, length_penalty: float) -> float:
    """Divisor of the cumulative log-prob at generated-token index ``gen``."""
    return math.pow(gen + 1, length_penalty) if length_penalty != 0 else 1.0


@dataclass
class BeamState:
    """One utterance's search state between two steps, as the engine keeps it.  Every list over rows has ``beam``
    entries.  A row whose candidate does not exist is dead: it feeds eot, its cum is -inf and it never becomes a
    hypothesis."""
    seqs: list                                  # generated tokens of every row
    cum: list                                   # cumulative log-prob of every row (fp32 values)
    tokens: list = None                         # token every row feeds next (None before the first step)
    parents: list = None                        # row of the previous step every row continues
    hyps: list = field(default_factory=list)    # (normalised score, tokens) of every finished hypothesis, in order
    best: int = -1                              # index into hyps of the best one, -1 = none
    finished: bool = False
    picks: list = None                          # candidate rank every row took at the last step

    @property
    def best_score(self) -> float:
        return self.hyps[self.best][0] if self.best >= 0 else NEG_INF

    @property
    def best_tokens(self) -> list:
        return self.hyps[self.best][1] if self.best >= 0 else []


BEAM_STEP_DEFECTS = ("secondary_from_0", "best_ge", "is_last_early", "invalid_hyps")


def beam_step(state: BeamState, cand_ids, cand_scores, *, V: int, eot: int, gen: int, cap: int, max_hyp: int,
              norm: float, defect=None) -> BeamState:
    """The bookkeeping of one step of one utterance.

    cand_ids: the 2 * beam candidates, best first, as flat ids row * V + token, -1 where no candidate exists;
    cand_scores: their normalised scores (fp32 values).  gen: index of the token being generated; cap: the utterance's
    limit on generated tokens (gen + 1 == cap is its last step, and with gen >= cap it finishes with no hypothesis);
    norm: the step's length normalisation.  Rules: each of the first ``beam`` candidates that exists and ends in eot (or
    any, at the last step) becomes a hypothesis, the first best one wins ties, and its row continues with the next
    unused non-eot candidate after rank beam - 1 (or keeps its own candidate when none is left); a row without a
    candidate is dead; the new cum is the fp32 product score * norm.  ``defect`` (comparator tests only) injects one
    of BEAM_STEP_DEFECTS."""
    beam, n_cand = len(state.seqs), len(cand_ids)
    is_last = gen + (2 if defect == "is_last_early" else 1) >= cap
    capped = gen >= cap
    hyps, best = list(state.hyps), state.best
    best_score = state.best_score
    picks = []
    secondary = 0 if defect == "secondary_from_0" else beam
    for k in range(beam):
        pick = k
        idx = cand_ids[k]
        tok = idx % V if idx >= 0 else eot
        if not capped and (idx >= 0 or defect == "invalid_hyps") and (tok == eot or is_last):
            row = idx // V if idx >= 0 else k
            hyps.append((cand_scores[k], state.seqs[row] + ([] if tok == eot else [tok])))
            if cand_scores[k] > best_score or (defect == "best_ge" and cand_scores[k] == best_score):
                best, best_score = len(hyps) - 1, cand_scores[k]
            for j in range(secondary, n_cand):
                if cand_ids[j] >= 0 and cand_ids[j] % V != eot:
                    pick, secondary = j, j + 1
                    break
        picks.append(pick)
    seqs, cum, tokens, parents = [], [], [], []
    for k, j in enumerate(picks):
        idx = cand_ids[j]
        parent, tok = (idx // V, idx % V) if idx >= 0 else (k, eot)
        seqs.append(state.seqs[parent] + [tok])
        cum.append(float(np.float32(cand_scores[j]) * np.float32(norm)) if idx >= 0 else NEG_INF)
        tokens.append(tok)
        parents.append(parent)
    return BeamState(seqs, cum, tokens, parents, hyps, best, is_last or len(hyps) >= max_hyp, picks)


def beam_candidates(logp: torch.Tensor, cum: torch.Tensor, norm: float, n_cand: int, first: bool):
    """logp [rows, V] processed log-probs, cum [rows] (fp32) -> (flat ids, scores) of the n_cand best
    (logp + cum) / norm, ties to the lowest flat id.  Only row 0 counts at the first step (every row holds the prompt);
    a token whose processed logit is -inf is no candidate, and missing candidates are id -1 with score -inf."""
    V = logp.shape[1]
    flat = ((logp + cum[:, None]) / norm).reshape(-1)
    valid = torch.isfinite(logp).reshape(-1)
    if first:
        valid[V:] = False
    idx = torch.nonzero(valid).flatten()
    order = idx[torch.argsort(-flat[idx], stable=True)[:n_cand]]
    pad = n_cand - order.numel()
    return order.tolist() + [-1] * pad, flat[order].tolist() + [NEG_INF] * pad


def beam_search(logits_fn, process, *, beam: int, V: int, eot: int, max_new: int, max_hyp: int, length_penalty: float,
                trace=None) -> BeamState:
    """The search loop around ``beam_step`` for one utterance.

    logits_fn(s, tokens, parents) -> raw logits of step s: [1, V] or [beam, V] at s = 0 (every row holds the prompt),
    [beam, V] after, row k fed tokens[k] and continuing row parents[k] of the previous step.  process(logits, hists, s)
    -> processed logits (hists: the rows' generated tokens).  trace, if a list, receives every step's smallest
    decision-relevant gap (``beam_margin``)."""
    st = BeamState([[] for _ in range(beam)], [0.0] * beam)
    rows = beam
    for s in range(max_new):
        logits = logits_fn(s, st.tokens, None if st.parents is None else ([0] * beam if rows == 1 else st.parents))
        rows = logits.shape[0]
        logp = torch.log_softmax(process(logits, st.seqs[:rows], s), dim=-1)
        norm = length_norm(s, length_penalty)
        ids, scores = beam_candidates(logp, torch.tensor(st.cum[:rows], dtype=torch.float32), norm, 2 * beam, s == 0)
        st = beam_step(st, ids, scores, V=V, eot=eot, gen=s, cap=max_new, max_hyp=max_hyp, norm=norm)
        if trace is not None:
            toks = [i % V if i >= 0 else -1 for i in ids]
            trace.append(beam_margin(scores, toks, st.picks, beam, eot, norm, st.finished, s + 1 == max_new))
        if st.finished:
            break
    return st


def beam_margin(cs, cand_tok, nxt, beam, eot, norm, finishing, is_last):
    """Smallest DECISION-RELEVANT gap of one beam-search step, in cumulative log-prob units (normalised gap x norm).

    A step decides (a) which candidates form the top-``beam`` set -- those ending in eot (all of them at the last
    step) become hypotheses -- and (b) which later non-eot candidates replace them as alive beams.  The order of two
    alive non-eot candidates inside the used set changes nothing (it only permutes rows), so only two boundaries
    count: rank beam-1 vs rank beam, and the last used candidate vs the next one that could be used instead.  When
    the search ends at this step the alive set no longer matters, only the hypothesis set does."""
    gaps = []

    def gap(a, b):
        if b < len(cs) and math.isfinite(cs[a]):
            gaps.append((cs[a] - cs[b]) if math.isfinite(cs[b]) else 1e9)

    a, b = beam - 1, beam
    both_plain = cand_tok[a] != eot and cand_tok[b] != eot
    if finishing:
        if is_last or not both_plain:
            gap(a, b)
    else:
        if not (both_plain and b in nxt):
            gap(a, b)
        m = max(nxt)
        if m >= beam:
            c = next((j for j in range(m + 1, len(cs)) if cand_tok[j] != eot), None)
            if c is not None:
                gap(m, c)
            elif m + 1 < len(cs):
                gap(m, len(cs) - 1)  # the real competitor is below the candidate list: a lower bound of the gap
            else:
                gaps.append(0.0)     # cannot tell how close the next candidate was
    return (min(gaps) if gaps else 1e9) * norm


class WhisperOracle:
    def __init__(self, dims: WhisperDims, tensors: dict):
        self.dims = dims
        self.w = {k: _t(v) for k, v in tensors.items() if not k.startswith("meta.")}
        d = dims.d_model
        self.conv1_w = self.w["enc.conv1.w"].view(d, 3, dims.n_mels).permute(0, 2, 1).contiguous()
        self.conv2_w = self.w["enc.conv2.w"].view(d, 3, d).permute(0, 2, 1).contiguous()
        self.emb = self.w["dec.tok_emb"][: dims.n_vocab]
        self.suppress = torch.tensor(sorted(set(dims.suppress_ids)), dtype=torch.long)
        self.suppress_begin = torch.tensor(list(dims.suppress_ids_begin), dtype=torch.long)
        self.logit_noise = None
        # True: cross K/V and every appended self-attention K/V row are rounded through fp16, the two storage roundings
        # of the engine's SIMT decoder pass (its activations stay fp32), so that pass can be checked to a tight bound
        self.kv_fp16 = False
        self._call_search = (1.0, 1.0)   # (patience, length penalty) of the generate call in progress

    @classmethod
    def from_blob(cls, src):
        dims, tensors = read_blob(src)
        return cls(dims, tensors)

    # ------------------------------------------------------------------ blocks
    def _ln(self, x, name):
        return F.layer_norm(x, (x.shape[-1],), self.w[name + ".g"], self.w[name + ".b"], 1e-5)

    def _mha(self, q, k, v):
        """q [N,Tq,d], k/v [N,Tk,d] -> [N,Tq,d]; softmax(q k^T / 8) v per 64-wide head."""
        n, tq, d = q.shape
        h = self.dims.n_heads
        qh = q.view(n, tq, h, 64).transpose(1, 2)
        kh = k.view(n, -1, h, 64).transpose(1, 2)
        vh = v.view(n, -1, h, 64).transpose(1, 2)
        s = torch.matmul(qh, kh.transpose(-1, -2)) * 0.125
        p = torch.softmax(s, dim=-1)
        return torch.matmul(p, vh).transpose(1, 2).reshape(n, tq, d)

    # ----------------------------------------------------------------- encoder
    def conv_stem(self, mel: torch.Tensor) -> torch.Tensor:
        x = F.gelu(F.conv1d(mel, self.conv1_w, self.w["enc.conv1.b"], padding=1))
        x = F.gelu(F.conv1d(x, self.conv2_w, self.w["enc.conv2.b"], stride=2, padding=1))
        return x.permute(0, 2, 1) + self.w["enc.pos"]

    def encoder_layer(self, x, i):
        p = f"enc.{i}."
        d = self.dims.d_model
        xn = self._ln(x, p + "ln1")
        qkv = F.linear(xn, self.w[p + "qkv.w"], self.w[p + "qkv.b"])
        a = self._mha(qkv[..., :d], qkv[..., d : 2 * d], qkv[..., 2 * d :])
        x = x + F.linear(a, self.w[p + "o.w"], self.w[p + "o.b"])
        xn = self._ln(x, p + "ln2")
        hdn = F.gelu(F.linear(xn, self.w[p + "fc1.w"], self.w[p + "fc1.b"]))
        return x + F.linear(hdn, self.w[p + "fc2.w"], self.w[p + "fc2.b"])

    @torch.no_grad()
    def encode(self, mel, n_layers: int | None = None, final_ln: bool = True) -> torch.Tensor:
        """mel float32 [B,80,3000] -> [B,1500,d]."""
        mel = torch.as_tensor(np.asarray(mel), dtype=torch.float32)
        x = self.conv_stem(mel)
        nl = self.dims.n_enc_layers if n_layers is None else n_layers
        for i in range(nl):
            x = self.encoder_layer(x, i)
        return self._ln(x, "enc.ln_post") if final_ln else x

    # ----------------------------------------------------------------- decoder
    def _kv_store(self, t: torch.Tensor) -> torch.Tensor:
        return t.half().float() if self.kv_fp16 else t

    @torch.no_grad()
    def cross_kv(self, enc: torch.Tensor):
        """enc [1500,d] -> list over layers of (K [1500,d], V [1500,d])."""
        d = self.dims.d_model
        kv = self._kv_store(F.linear(enc, self.w["dec.crosskv.w"], self.w["dec.crosskv.b"]))
        return [(kv[:, i * 2 * d : i * 2 * d + d], kv[:, i * 2 * d + d : (i + 1) * 2 * d])
                for i in range(self.dims.n_dec_layers)]

    @torch.no_grad()
    def decode_rows(self, tokens, pos: int, cache, ckv):
        """One decoder step for R rows of one utterance.

        tokens [R] ints at position ``pos``; cache: list over layers of
        (K [R,pos,d], V [R,pos,d]) or None at pos 0; returns (logits [R,V], new cache).
        """
        d = self.dims.d_model
        tok = torch.as_tensor(tokens, dtype=torch.long)
        x = self.emb[tok] + self.w["dec.pos"][pos]
        r = x.shape[0]
        new_cache = []
        for i in range(self.dims.n_dec_layers):
            p = f"dec.{i}."
            xn = self._ln(x, p + "ln1")
            qkv = F.linear(xn, self.w[p + "qkv.w"], self.w[p + "qkv.b"])
            k_new, v_new = self._kv_store(qkv[:, d : 2 * d]).unsqueeze(1), self._kv_store(qkv[:, 2 * d :]).unsqueeze(1)
            if cache is not None:
                k_all = torch.cat([cache[i][0], k_new], 1)
                v_all = torch.cat([cache[i][1], v_new], 1)
            else:
                k_all, v_all = k_new, v_new
            new_cache.append((k_all, v_all))
            a = self._mha(qkv[:, :d].unsqueeze(1), k_all, v_all)[:, 0]
            x = x + F.linear(a, self.w[p + "o.w"], self.w[p + "o.b"])
            xn = self._ln(x, p + "ln2")
            q = F.linear(xn, self.w[p + "cq.w"], self.w[p + "cq.b"]).unsqueeze(1)
            ck, cv = ckv[i]
            a = self._mha(q, ck.unsqueeze(0).expand(r, -1, -1), cv.unsqueeze(0).expand(r, -1, -1))[:, 0]
            x = x + F.linear(a, self.w[p + "co.w"], self.w[p + "co.b"])
            xn = self._ln(x, p + "ln3")
            hdn = F.gelu(F.linear(xn, self.w[p + "fc1.w"], self.w[p + "fc1.b"]))
            x = x + F.linear(hdn, self.w[p + "fc2.w"], self.w[p + "fc2.b"])
        x = self._ln(x, "dec.ln")
        return F.linear(x, self.emb), new_cache

    def _process(self, logits, gen_step: int, extra_suppress=None):
        """CT2 logits processors for the WIS call (suppress_tokens=[-1], suppress_blank=True)."""
        logits = logits.clone()
        if self.logit_noise is not None:  # robustness probe (tests): see ``generate(logit_noise=...)``
            sigma, gen = self.logit_noise
            logits += sigma * torch.randn(logits.shape, generator=gen)
        logits[:, self.suppress] = NEG_INF
        if extra_suppress is not None and len(extra_suppress):
            logits[:, torch.as_tensor(list(extra_suppress), dtype=torch.long)] = NEG_INF
        if gen_step == 0:
            logits[:, self.suppress_begin] = NEG_INF
        return logits

    @staticmethod
    def max_new_tokens(prompt_len: int, max_length: int = 448) -> int:
        return max(0, min(max_length // 2, max_length - prompt_len))

    def _prefill(self, prompt, ckv):
        cache = None
        for pos, t in enumerate(prompt[:-1]):
            _, cache = self.decode_rows([t], pos, cache, ckv)
        return cache

    @torch.no_grad()
    def forced_logits(self, enc_row: torch.Tensor, tokens) -> torch.Tensor:
        """Teacher-forced raw logits [len(tokens), V] (no processors)."""
        ckv = self.cross_kv(enc_row)
        cache, out = None, []
        for pos, t in enumerate(tokens):
            lg, cache = self.decode_rows([t], pos, cache, ckv)
            out.append(lg[0])
        return torch.stack(out)

    # ------------------------------------------------------------------ search
    def _processors(self, prompt, extra_suppress):
        """-> process(logits, hists, gen): the logits processors of one utterance's search (hists: the rows' generated
        tokens; the timestamp oracle adds its rules here)."""
        return lambda logits, hists, gen: self._process(logits, gen, extra_suppress)

    # The two per-utterance entry points (a subclass may override either); both run the one search loop.
    @torch.no_grad()
    def _greedy(self, enc_row, prompt, max_length, extra_suppress, trace):
        """beam 1: the beam procedure with 2 candidates (greedy arg-max decoding), at the call's patience and length
        penalty as the engine runs it."""
        patience, length_penalty = self._call_search
        return self._search(enc_row, prompt, 1, max_length, patience, length_penalty, extra_suppress, trace)

    @torch.no_grad()
    def _beam(self, enc_row, prompt, beam, max_length, patience, length_penalty, extra_suppress, trace):
        return self._search(enc_row, prompt, beam, max_length, patience, length_penalty, extra_suppress, trace)

    _beam_margin = staticmethod(beam_margin)

    @torch.no_grad()
    def _search(self, enc_row, prompt, beam, max_length, patience, length_penalty, extra_suppress, trace):
        """One utterance through ``beam_search``."""
        ckv = self.cross_kv(enc_row)
        cache = self._prefill(prompt, ckv)
        start = len(prompt) - 1

        def logits_fn(s, tokens, parents):
            nonlocal cache
            if s == 0:
                tokens = [prompt[-1]]
            else:
                pidx = torch.tensor(parents, dtype=torch.long)
                cache = [(k_[pidx], v_[pidx]) for k_, v_ in cache]
            logits, cache = self.decode_rows(tokens, start + s, cache, ckv)
            return logits

        st = beam_search(logits_fn, self._processors(prompt, extra_suppress), beam=beam, V=self.dims.n_vocab,
                         eot=self.dims.eot, max_new=self.max_new_tokens(len(prompt), max_length),
                         max_hyp=max_hypotheses(beam, patience), length_penalty=length_penalty, trace=trace)
        if not st.hyps:
            return GenerationResult([[]], [0.0])
        if trace is not None:  # last entry: gap between the two best finished hypotheses (normalised scores)
            hs = sorted((h_[0] for h_ in st.hyps), reverse=True)
            trace.append(("final", hs[0] - hs[1] if len(hs) > 1 else 1e9))
        return GenerationResult([st.best_tokens], [st.best_score])

    @torch.no_grad()
    def generate(self, features, prompts, beam_size: int = 5, patience: float = 1.0, length_penalty: float = 1.0,
                 max_length: int = 448, suppress_tokens=(-1,), return_scores: bool = False, trace=None,
                 enc=None, logit_noise=None):
        """features float32 [B,80,3000]; prompts list[list[int]] -> list[GenerationResult].

        ``logit_noise=(sigma, seed)`` adds seeded Gaussian noise of that size to every raw logit of every step: the
        tests use it to find out whether a transcript is a ROBUST decision of the reference algorithm (unchanged under
        perturbations of the size of the documented fp16-vs-fp32 logit tolerance) or hangs on a near-tie."""
        self.logit_noise = None
        self._call_search = (patience, length_penalty)
        if logit_noise is not None:
            g = torch.Generator()
            g.manual_seed(int(logit_noise[1]))
            self.logit_noise = (float(logit_noise[0]), g)
        try:
            return self._generate(features, prompts, beam_size, patience, length_penalty, max_length, suppress_tokens,
                                  trace, enc)
        finally:
            self.logit_noise = None
            self._call_search = (1.0, 1.0)

    def _generate(self, features, prompts, beam_size, patience, length_penalty, max_length, suppress_tokens, trace, enc):
        extra = [t for t in suppress_tokens if t >= 0]
        if -1 not in suppress_tokens:
            raise NotImplementedError("oracle restates the WIS call, which always keeps suppress_tokens=[-1]")
        if enc is None:
            enc = self.encode(features)
        res = []
        for b, prompt in enumerate(prompts):
            tr = [] if trace is not None else None
            if beam_size == 1:
                r = self._greedy(enc[b], list(prompt), max_length, extra, tr)
            else:
                r = self._beam(enc[b], list(prompt), beam_size, max_length, patience, length_penalty, extra, tr)
            if trace is not None:
                trace.append(tr)
            res.append(r)
        return res

    @torch.no_grad()
    def detect_language(self, features, enc=None):
        """-> per utterance, list of (lang token id, probability) sorted by probability desc."""
        if enc is None:
            enc = self.encode(features)
        lang = torch.tensor(self.dims.lang_ids, dtype=torch.long)
        out = []
        for b in range(enc.shape[0]):
            logits, _ = self.decode_rows([self.dims.sot], 0, None, self.cross_kv(enc[b]))
            p = torch.softmax(logits[0, lang], -1)
            order = torch.argsort(-p, stable=True)
            out.append([(int(lang[i]), float(p[i])) for i in order])
        return out
