"""Whisper's timestamp rules on top of the fp32 oracle (TEST INFRASTRUCTURE ONLY).

``apply_timestamp_rules`` restates openai/whisper's ``ApplyTimestampRules`` as transformers implements it in
``WhisperTimeStampLogitsProcessor`` (pinned against that class by ``tests/golden/timestamp_rules_hf.npz``, written by
``scripts/gen_golden_timestamp_rules_hf.py``).  ``TimestampOracle`` is ``oracle.whisper_ref.WhisperOracle`` with the
rules applied after the logit-noise probe and the suppress masks whenever the prompt lacks <|notimestamps|>
(CTranslate2's switch), in greedy and in beam search alike.  Every rule can be switched off (``disable``) so the tests
can show that each one changes something.

Rules (ts_begin = no_timestamps + 1, gen = index of the token being generated, hist = the row's generated tokens):
  1. <|notimestamps|> is off.
  2. gen == 0: every id < ts_begin is off, and every timestamp > ts_begin + max_initial_timestamp_index.
  3. last token a timestamp: if the one before it is one too (or gen == 1) timestamps are off (3a), else ids < eot (3b).
  4. timestamps below the row's last timestamp t are off; t itself too unless 3b holds.
  5. if logsumexp(processed timestamp logits) > max(processed text logits), every id < ts_begin is off.
"""
from __future__ import annotations

import math

import torch

from oracle.whisper_ref import GenerationResult, WhisperOracle

NEG_INF = float("-inf")
RULES = (1, 2, 3, 4, 5)


def apply_timestamp_rules(logits: torch.Tensor, hists, gen: int, *, no_timestamps: int, eot: int,
                          max_initial_timestamp_index: int = 50, disable=()) -> torch.Tensor:
    """logits [R, V] (already through the suppress masks); hists: R token lists of length gen."""
    out = logits.clone()
    ts_begin = no_timestamps + 1
    if 1 not in disable:
        out[:, no_timestamps] = NEG_INF
    for k, seq in enumerate(hists):
        seq = list(seq)
        last_ts = len(seq) >= 1 and seq[-1] >= ts_begin
        pen_ts = len(seq) < 2 or seq[-2] >= ts_begin
        if 3 not in disable and last_ts:
            if pen_ts:
                out[k, ts_begin:] = NEG_INF
            else:
                out[k, :eot] = NEG_INF
        stamps = [t for t in seq if t >= ts_begin]
        if 4 not in disable and stamps:
            lo = stamps[-1] if (last_ts and not pen_ts) else stamps[-1] + 1
            out[k, ts_begin:lo] = NEG_INF
    if gen == 0 and 2 not in disable:
        out[:, :ts_begin] = NEG_INF
        out[:, ts_begin + max_initial_timestamp_index + 1:] = NEG_INF
    if 5 not in disable:
        for k in range(out.shape[0]):
            row = out[k].double()
            if torch.logsumexp(row[ts_begin:], 0) > row[:ts_begin].max():
                out[k, :ts_begin] = NEG_INF
    return out


class TimestampOracle(WhisperOracle):
    """WhisperOracle with timestamp decoding for prompts without <|notimestamps|>."""

    max_initial_timestamp_index = 50
    disable = ()

    def generate(self, features, prompts, beam_size: int = 5, max_initial_timestamp_index: int = 50, disable=(), **kw):
        self.max_initial_timestamp_index = max_initial_timestamp_index
        self.disable = tuple(disable)
        return super().generate(features, prompts, beam_size=beam_size, **kw)

    def _rules(self, logits, hists, gen):
        return apply_timestamp_rules(logits, hists, gen, no_timestamps=self.dims.no_timestamps, eot=self.dims.eot,
                                     max_initial_timestamp_index=self.max_initial_timestamp_index, disable=self.disable)

    def _wants_ts(self, prompt):
        return self.dims.no_timestamps not in prompt

    @torch.no_grad()
    def _greedy(self, enc_row, prompt, max_length, extra_suppress, trace):
        if not self._wants_ts(prompt):
            return super()._greedy(enc_row, prompt, max_length, extra_suppress, trace)
        ckv = self.cross_kv(enc_row)
        cache = self._prefill(prompt, ckv)
        start = len(prompt) - 1
        last = prompt[-1]
        out, cum = [], 0.0
        for s in range(self.max_new_tokens(len(prompt), max_length)):
            logits, cache = self.decode_rows([last], start + s, cache, ckv)
            logits = self._rules(self._process(logits, s, extra_suppress), [out], s)
            tok = int(torch.argmax(logits[0]))
            cum += float(torch.log_softmax(logits[0], -1)[tok])
            if tok == self.dims.eot:
                break
            out.append(tok)
            last = tok
        return GenerationResult([out], [cum])

    @torch.no_grad()
    def _beam(self, enc_row, prompt, beam, max_length, patience, length_penalty, extra_suppress, trace):
        if not self._wants_ts(prompt):
            return super()._beam(enc_row, prompt, beam, max_length, patience, length_penalty, extra_suppress, trace)
        V, eot = self.dims.n_vocab, self.dims.eot
        ckv = self.cross_kv(enc_row)
        cache = self._prefill(prompt, ckv)
        start = len(prompt) - 1
        n_cand = 2 * beam
        max_hyp = int(round(beam * patience))
        max_new = self.max_new_tokens(len(prompt), max_length)
        alive_tokens = [[]]
        alive_scores = torch.zeros(1)
        last = [prompt[-1]]
        hyps = []
        for s in range(max_new):
            is_last = s + 1 == max_new
            logits, cache = self.decode_rows(last, start + s, cache, ckv)
            logp = torch.log_softmax(self._rules(self._process(logits, s, extra_suppress), alive_tokens, s), dim=-1)
            norm = math.pow(s + 1, length_penalty) if length_penalty != 0 else 1.0
            flat = ((logp + alive_scores[:, None]) / norm).reshape(-1)
            order = torch.argsort(-flat, stable=True)[:n_cand]
            cand_scores = flat[order]
            cand_beam = (order // V).tolist()
            cand_tok = (order % V).tolist()
            nxt = []
            secondary = beam
            for k in range(beam):
                pick = k
                if cand_tok[k] == eot or is_last:
                    toks = alive_tokens[cand_beam[k]] + ([] if cand_tok[k] == eot else [cand_tok[k]])
                    hyps.append((float(cand_scores[k]), toks))
                    for j in range(secondary, n_cand):
                        if cand_tok[j] != eot:
                            pick = j
                            secondary = j + 1
                            break
                nxt.append(pick)
            if trace is not None:  # the step's smallest decision-relevant gap (WhisperOracle._beam_margin)
                trace.append(self._beam_margin(cand_scores.tolist(), cand_tok, nxt, beam, eot, norm,
                                               is_last or len(hyps) >= max_hyp, is_last))
            if is_last or len(hyps) >= max_hyp:
                break
            parents = [cand_beam[j] for j in nxt]
            alive_tokens = [alive_tokens[cand_beam[j]] + [cand_tok[j]] for j in nxt]
            alive_scores = torch.stack([cand_scores[j] for j in nxt]) * norm
            last = [cand_tok[j] for j in nxt]
            pidx = torch.tensor(parents, dtype=torch.long)
            cache = [(k_[pidx], v_[pidx]) for k_, v_ in cache]
        if not hyps:
            return GenerationResult([[]], [0.0])
        if trace is not None:  # last entry: gap between the two best finished hypotheses (normalised scores)
            hs = sorted((h_[0] for h_ in hyps), reverse=True)
            trace.append(("final", hs[0] - hs[1] if len(hs) > 1 else 1e9))
        best = max(range(len(hyps)), key=lambda i: (hyps[i][0], -i))
        return GenerationResult([hyps[best][1]], [hyps[best][0]])


def check_invariants(seq, dims, max_initial_timestamp_index: int = 50):
    """Assert what every timestamp transcript satisfies; returns the number of segments (closed timestamp pairs)."""
    ts_begin = dims.no_timestamps + 1
    assert dims.no_timestamps not in seq and dims.eot not in seq
    assert seq and ts_begin <= seq[0] <= ts_begin + max_initial_timestamp_index, seq[:3]
    stamps = [t for t in seq if t >= ts_begin]
    assert stamps == sorted(stamps), "timestamps decrease"
    # runs of timestamps: a pair (closing + opening) between text, a single one only at the very start or end
    runs, i = [], 0
    while i < len(seq):
        if seq[i] >= ts_begin:
            j = i
            while j < len(seq) and seq[j] >= ts_begin:
                j += 1
            runs.append((i, j - i))
            i = j
        else:
            i += 1
    for start, n in runs:
        if start == 0:
            assert n == 1, "the first timestamp is followed by text"
        elif start + n == len(seq):
            assert n in (1, 2), "more than two timestamps in a row"
        else:
            assert n == 2, "timestamps come in pairs"
    return sum(1 for start, n in runs if start > 0)
