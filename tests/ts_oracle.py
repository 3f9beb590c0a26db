"""Whisper's timestamp rules on top of the fp32 oracle (TEST INFRASTRUCTURE ONLY).

``apply_timestamp_rules`` restates openai/whisper's ``ApplyTimestampRules`` as transformers implements it in
``WhisperTimeStampLogitsProcessor`` (pinned against that class by ``tests/golden/timestamp_rules_hf.npz``, written by
``scripts/gen_golden_timestamp_rules_hf.py``).  ``TimestampOracle`` is ``oracle.whisper_ref.WhisperOracle`` with the
rules applied after the logit-noise probe and the suppress masks whenever the prompt lacks <|notimestamps|>
(CTranslate2's switch), in greedy and in beam search alike: it supplies only the rules to
``oracle.whisper_ref.beam_search``, the one search loop.  Every rule can be switched off (``disable``) so the tests
can show that each one changes something.

Rules (ts_begin = no_timestamps + 1, gen = index of the token being generated, hist = the row's generated tokens):
  1. <|notimestamps|> is off.
  2. gen == 0: every id < ts_begin is off, and every timestamp > ts_begin + max_initial_timestamp_index.
  3. last token a timestamp: if the one before it is one too (or gen == 1) timestamps are off (3a), else ids < eot (3b).
  4. timestamps below the row's last timestamp t are off; t itself too unless 3b holds.
  5. if logsumexp(processed timestamp logits) > max(processed text logits), every id < ts_begin is off.
"""
from __future__ import annotations

import torch

from oracle.whisper_ref import WhisperOracle

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

    def _processors(self, prompt, extra_suppress):
        base = super()._processors(prompt, extra_suppress)
        if not self._wants_ts(prompt):
            return base
        return lambda logits, hists, gen: self._rules(base(logits, hists, gen), hists, gen)


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
