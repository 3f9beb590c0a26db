"""The history processors -- repetition penalty and no-repeat n-gram blocking -- on top of the fp32 oracle (TEST
INFRASTRUCTURE ONLY).

``history_processors`` restates transformers' ``RepetitionPenaltyLogitsProcessor`` and ``NoRepeatNGramLogitsProcessor``
with ``input_ids`` = the row's generated tokens (pinned against those classes by
``tests/golden/history_processors_hf.npz``, written by ``scripts/gen_golden_history_processors_hf.py``).
``ProcOracle`` is ``tests.ts_oracle.TimestampOracle`` with the processors applied after the logit-noise probe and
before the suppress masks; in timestamp mode the rules follow, so rule 5 sees the penalised logits.  At the defaults
(1, 0) it is the timestamp oracle unchanged.

Semantics (hist = the row's generated tokens, timestamps included, prompt excluded; gen = len(hist)):
  * repetition_penalty p: every distinct id in hist gets l < 0 ? l * p : l / p (one fp32 operation, once per id);
  * no_repeat_ngram_size n: if gen + 1 >= n, every hist[i + n - 1] with hist[i .. i + n - 2] == hist[gen - n + 1 ..
    gen - 1], 0 <= i <= gen - n, is -inf.
``PROC_DEFECTS`` are the wrong variants the comparator tests inject.
"""
from __future__ import annotations

import torch

from oracle.whisper_ref import WhisperOracle
from tests.ts_oracle import TimestampOracle

NEG_INF = float("-inf")
# penalty compounded per occurrence, negative logits divided, n-gram suffix shifted back by one, the last prompt token
# counted as history, the processors applied after the timestamp rules
PROC_DEFECTS = ("compound", "divide_negative", "ngram_shift", "prompt_history", "after_ts_rules")


def banned_ngram_tokens(hist, n: int, defect=None) -> list:
    """Ids the n-gram rule bans for a row with generated tokens `hist`."""
    g = len(hist)
    if n <= 0 or g + 1 < n:
        return []
    lo = g - n + 1 - (1 if defect == "ngram_shift" else 0)
    suffix = list(hist[max(lo, 0): max(lo, 0) + n - 1])
    return [hist[i + n - 1] for i in range(g - n + 1) if list(hist[i: i + n - 1]) == suffix]


def history_processors(logits: torch.Tensor, hists, repetition_penalty: float = 1.0, no_repeat_ngram_size: int = 0,
                       defect=None) -> torch.Tensor:
    """logits [R, V] (any float dtype; the penalty is one operation in that dtype with p rounded to fp32, as the
    engine computes it); hists: R token lists."""
    out = logits.clone()
    p = torch.tensor(float(torch.tensor(repetition_penalty, dtype=torch.float32)), dtype=out.dtype)
    for k, hist in enumerate(hists):
        hist = [int(t) for t in hist]
        if repetition_penalty != 1 and hist:
            ids = hist if defect == "compound" else sorted(set(hist))
            for t in ids:
                v = out[k, t]
                out[k, t] = v / p if (defect == "divide_negative" or not v < 0) else v * p
        ban = banned_ngram_tokens(hist, no_repeat_ngram_size, defect)
        if ban:
            out[k, torch.tensor(ban, dtype=torch.long)] = NEG_INF
    return out


def process_rows(logits: torch.Tensor, hists, gen: int, *, masks, rules=None, repetition_penalty: float = 1.0,
                 no_repeat_ngram_size: int = 0, prompt=(), defect=None) -> torch.Tensor:
    """One step's processed logits in the engine's order: the history processors, masks(x, gen) (the suppress masks),
    then rules(x, hists, gen) (timestamp mode, or None).  ``defect`` (comparator tests only) injects one of
    PROC_DEFECTS."""
    h = [list(prompt[-1:]) + list(s) for s in hists] if defect == "prompt_history" else hists
    x = logits
    if defect != "after_ts_rules":
        x = history_processors(x, h, repetition_penalty, no_repeat_ngram_size, defect)
    x = masks(x, gen)
    if rules is not None:
        x = rules(x, hists, gen)
    if defect == "after_ts_rules":
        x = history_processors(x, h, repetition_penalty, no_repeat_ngram_size)
    return x


class ProcOracle(TimestampOracle):
    """TimestampOracle with the history processors (both modes: a prompt with <|notimestamps|> gets no rules)."""

    repetition_penalty = 1.0
    no_repeat_ngram_size = 0
    proc_defect = None

    def generate(self, features, prompts, beam_size: int = 5, repetition_penalty: float = 1.0,
                 no_repeat_ngram_size: int = 0, proc_defect=None, **kw):
        self.repetition_penalty, self.no_repeat_ngram_size, self.proc_defect = \
            repetition_penalty, no_repeat_ngram_size, proc_defect
        try:
            return super().generate(features, prompts, beam_size=beam_size, **kw)
        finally:
            self.repetition_penalty, self.no_repeat_ngram_size, self.proc_defect = 1.0, 0, None

    def _masks(self, logits, gen, extra_suppress):
        """WhisperOracle's suppress masks without the noise probe (which the processors' step applied first)."""
        noise, self.logit_noise = self.logit_noise, None
        try:
            return WhisperOracle._process(self, logits, gen, extra_suppress)
        finally:
            self.logit_noise = noise

    def _processors(self, prompt, extra_suppress):
        p, n = self.repetition_penalty, self.no_repeat_ngram_size
        if p == 1 and n == 0:
            return super()._processors(prompt, extra_suppress)
        rules = self._rules if self._wants_ts(prompt) else None

        def process(logits, hists, gen):
            x = logits.clone()
            if self.logit_noise is not None:
                sigma, g = self.logit_noise
                x += sigma * torch.randn(x.shape, generator=g)
            return process_rows(x, hists, gen, masks=lambda y, s: self._masks(y, s, extra_suppress), rules=rules,
                                repetition_penalty=p, no_repeat_ngram_size=n, prompt=prompt, defect=self.proc_defect)

        return process
