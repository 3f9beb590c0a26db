"""CPU restatement of ``Whisper.align`` on top of the fp32 oracle (tests only).

Steps (openai/whisper ``find_alignment``, with the filter and DTW pinned to transformers
``models/whisper/generation_whisper.py``: ``_extract_token_timestamps``, ``_median_filter``, ``_dynamic_time_warping``;
``tests/test_align_rules.py`` checks them against ``tests/golden/alignment_hf.npz``):
  1. the decoder is teacher-forced with start_sequence + [<|notimestamps|>] + text;
  2. rows r = 0..n are positions S + r;
  3. weights = the alignment heads' fp32 cross-attention softmax over all 1500 frames, cut to F = num_frames // 2
     (no re-softmax after the cut, as transformers);
  4. standardise over rows (population std), median filter along frames (reflect padding; identity when
     F <= width // 2), mean over heads;
  5. DTW on -matrix with an fp32 cost;
  6. text_token_probs[i] = softmax over ids [0, eot) of row i's logits, at text[i].
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F


def default_heads(dims):
    if dims.alignment_heads:
        return [tuple(h) for h in dims.alignment_heads]
    L = dims.n_dec_layers
    return [(l, h) for l in range(L // 2, L) for h in range(dims.n_heads)]


@torch.no_grad()
def forced_capture(oracle, enc_row: torch.Tensor, tokens, heads):
    """Teacher-forced decoder over the whole token list -> (logits [T, V], probs [A, T, 1500]) with probs the fp32
    cross-attention softmax of each (layer, head) in ``heads``.  Runs the oracle's own step-by-step decoder
    (``decode_rows``) and records, at each cross-attention call, the softmax of the same scores ``_mha`` forms."""
    H = oracle.dims.n_heads
    ckv = oracle.cross_kv(enc_row)
    step = []  # this position's cross-attention probabilities, one [H, 1500] per layer in call order
    mha = oracle._mha

    def recording_mha(q, k, v):
        if k.shape[1] == enc_row.shape[0]:  # cross-attention: keys are the encoder frames
            n = q.shape[0]
            qh = q.view(n, -1, H, 64).transpose(1, 2)
            kh = k.view(n, -1, H, 64).transpose(1, 2)
            step.append(torch.softmax(torch.matmul(qh, kh.transpose(-1, -2)) * 0.125, dim=-1)[0, :, 0])
        return mha(q, k, v)

    oracle._mha = recording_mha
    try:
        cache, logits, probs = None, [], []
        for pos, t in enumerate(tokens):
            step.clear()
            lg, cache = oracle.decode_rows([t], pos, cache, ckv)
            logits.append(lg[0])
            probs.append(torch.stack([step[l][h] for l, h in heads]))
    finally:
        del oracle._mha
    return torch.stack(logits), torch.stack(probs, 1)


def standardise(weights: torch.Tensor) -> torch.Tensor:
    """[A, R, F]: per head and frame over the rows, population std (transformers _extract_token_timestamps)."""
    std = torch.std(weights, dim=-2, keepdim=True, unbiased=False)
    mean = torch.mean(weights, dim=-2, keepdim=True)
    return (weights - mean) / std


def median_filter(x: torch.Tensor, width: int) -> torch.Tensor:
    """transformers _median_filter: reflect padding, identity when the last dimension is <= width // 2."""
    pad = width // 2
    if x.shape[-1] <= pad:
        return x
    xp = F.pad(x[None], (pad, pad, 0, 0), mode="reflect")[0]
    return xp.unfold(-1, width, 1).sort()[0][..., pad]


def filter_matrix(weights, width: int) -> torch.Tensor:
    """[A, R, F] captured probabilities (already cut to F frames) -> matrix [R, F]."""
    w = torch.as_tensor(np.asarray(weights), dtype=torch.float32)
    return median_filter(standardise(w), width).mean(dim=0)


def dtw(matrix) -> np.ndarray:
    """transformers _dynamic_time_warping(-matrix), fp32 cost -> path int [len, 2] of (text index, time index)."""
    m = -np.asarray(matrix, np.float32)
    n, f = m.shape
    cost = np.full((n + 1, f + 1), np.inf, np.float32)
    trace = -np.ones((n + 1, f + 1), np.float32)
    cost[0, 0] = 0
    for j in range(1, f + 1):
        for i in range(1, n + 1):
            c0, c1, c2 = cost[i - 1, j - 1], cost[i - 1, j], cost[i, j - 1]
            if c0 < c1 and c0 < c2:
                c, t = c0, 0
            elif c1 < c0 and c1 < c2:
                c, t = c1, 1
            else:
                c, t = c2, 2
            cost[i, j] = np.float32(m[i - 1, j - 1] + c)
            trace[i, j] = t
    i, j = n, f
    trace[0, :] = 2
    trace[:, 0] = 1
    out = []
    while i > 0 or j > 0:
        out.append((i - 1, j - 1))
        t = trace[i, j]
        if t == 0:
            i, j = i - 1, j - 1
        elif t == 1:
            i -= 1
        else:
            j -= 1
    return np.asarray(out[::-1], np.int64).reshape(-1, 2)


def capture_window(oracle, enc_row, start_sequence, text, num_frames, heads=None):
    """Steps 1-3 and 6 for one window -> (weights [A, n + 1, F], token probs [n])."""
    dims = oracle.dims
    heads = default_heads(dims) if heads is None else heads
    S, n = len(start_sequence), len(text)
    tokens = list(start_sequence) + [dims.no_timestamps] + list(text)
    logits, probs = forced_capture(oracle, enc_row, tokens, heads)
    weights = probs[:, S:S + n + 1, : num_frames // 2]
    lg = logits[S:S + n, : dims.eot]
    tp = torch.softmax(lg, -1)[torch.arange(n), torch.as_tensor(text, dtype=torch.long)] if n else torch.zeros(0)
    return weights.numpy(), tp.numpy()


def align_window(oracle, enc_row, start_sequence, text, num_frames, width=7, heads=None):
    """-> (path [len, 2], token probs [n], matrix [n + 1, F], weights [A, n + 1, F])."""
    weights, tp = capture_window(oracle, enc_row, start_sequence, text, num_frames, heads)
    if len(text) == 0:
        return np.zeros((0, 2), np.int64), tp, None, weights
    mat = filter_matrix(weights, width).numpy()
    return dtw(mat), tp, mat, weights
