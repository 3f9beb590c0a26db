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
from dataclasses import dataclass

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
    @torch.no_grad()
    def _greedy(self, enc_row, prompt, max_length, extra_suppress, trace):
        ckv = self.cross_kv(enc_row)
        cache = self._prefill(prompt, ckv)
        start = len(prompt) - 1
        last = prompt[-1]
        out, cum = [], 0.0
        for s in range(self.max_new_tokens(len(prompt), max_length)):
            logits, cache = self.decode_rows([last], start + s, cache, ckv)
            logits = self._process(logits, s, extra_suppress)
            tok = int(torch.argmax(logits[0]))  # first (lowest id) maximum
            if trace is not None:
                top2 = torch.topk(logits[0], 2).values
                trace.append(float(top2[0] - top2[1]))
            cum += float(torch.log_softmax(logits[0], -1)[tok])
            if tok == self.dims.eot:
                break
            out.append(tok)
            last = tok
        return GenerationResult([out], [cum])

    @torch.no_grad()
    def _beam(self, enc_row, prompt, beam, max_length, patience, length_penalty, extra_suppress, trace):
        V = self.dims.n_vocab
        eot = self.dims.eot
        ckv = self.cross_kv(enc_row)
        cache = self._prefill(prompt, ckv)
        start = len(prompt) - 1
        n_cand = 2 * beam
        max_hyp = int(round(beam * patience))
        max_new = self.max_new_tokens(len(prompt), max_length)
        alive_tokens = [[]]  # generated tokens per alive beam
        alive_scores = torch.zeros(1)
        last = [prompt[-1]]
        hyps = []  # (normalised score, tokens)
        for s in range(max_new):
            is_last = s + 1 == max_new
            logits, cache = self.decode_rows(last, start + s, cache, ckv)
            logp = torch.log_softmax(self._process(logits, s, extra_suppress), dim=-1)
            total = logp + alive_scores[:, None]  # [rows, V] cumulative
            norm = math.pow(s + 1, length_penalty) if length_penalty != 0 else 1.0
            flat = (total / norm).reshape(-1)
            # descending, ties -> lowest flat index (stable sort on the negated values)
            order = torch.argsort(-flat, stable=True)[:n_cand]
            cand_scores = flat[order]
            cand_beam = (order // V).tolist()
            cand_tok = (order % V).tolist()
            nxt = []  # indices into the candidate list that stay alive
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
            if trace is not None:
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
        best = max(range(len(hyps)), key=lambda i: (hyps[i][0], -i))  # first best on ties
        return GenerationResult([hyps[best][1]], [hyps[best][0]])

    @staticmethod
    def _beam_margin(cs, cand_tok, nxt, beam, eot, norm, finishing, is_last):
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

    @torch.no_grad()
    def generate(self, features, prompts, beam_size: int = 5, patience: float = 1.0, length_penalty: float = 1.0,
                 max_length: int = 448, suppress_tokens=(-1,), return_scores: bool = False, trace=None,
                 enc=None, logit_noise=None):
        """features float32 [B,80,3000]; prompts list[list[int]] -> list[GenerationResult].

        ``logit_noise=(sigma, seed)`` adds seeded Gaussian noise of that size to every raw logit of every step: the
        tests use it to find out whether a transcript is a ROBUST decision of the reference algorithm (unchanged under
        perturbations of the size of the documented fp16-vs-fp32 logit tolerance) or hangs on a near-tie."""
        self.logit_noise = None
        if logit_noise is not None:
            g = torch.Generator()
            g.manual_seed(int(logit_noise[1]))
            self.logit_noise = (float(logit_noise[0]), g)
        try:
            return self._generate(features, prompts, beam_size, patience, length_penalty, max_length, suppress_tokens,
                                  trace, enc)
        finally:
            self.logit_noise = None

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
