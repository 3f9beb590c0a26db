"""CPU: the alignment oracle's post-processing (tests/align_oracle.py) against transformers' own code
(tests/golden/alignment_hf.npz, scripts/gen_golden_alignment_hf.py), the teeth of that comparison, and the
alignment_heads plumbing of the loaders and the weight blob."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import align_oracle as AO
from willow_inference_server_b200 import loaders, weights as W

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "alignment_hf.npz")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLDEN))


def _cases(g):
    k = 0
    while f"w{k}" in g:
        yield g[f"w{k}"], int(g[f"width{k}"]), g[f"mat{k}"], g[f"path{k}"]
        k += 1


def _agrees(g, filt=AO.filter_matrix, dtw=AO.dtw):
    """True when every golden case is reproduced: matrices to 1e-6, paths exactly."""
    for w, width, mat, path in _cases(g):
        m = filt(w, width)
        m = m.numpy() if isinstance(m, torch.Tensor) else m
        if m.shape != mat.shape or not np.allclose(m, mat, rtol=0, atol=1e-6, equal_nan=True):
            return False
        p = dtw(m)
        if p.shape != path.shape or (p != path).any():
            return False
    k = 0
    while f"tie_mat{k}" in g:
        p = dtw(g[f"tie_mat{k}"])
        if p.shape != g[f"tie_path{k}"].shape or (p != g[f"tie_path{k}"]).any():
            return False
        k += 1
    return True


def test_oracle_matches_transformers(gold):
    assert _agrees(gold)


def test_golden_paths_are_not_trivial(gold):
    # a straight diagonal would let a broken tie rule pass
    assert any(len(np.unique(p[:, 0])) > 2 and (np.diff(p[:, 0]) == 0).any() for _, _, _, p in _cases(gold))


# ---- each injected defect must make the comparison fail
def _filter_unbiased(w, width):
    w = torch.as_tensor(np.asarray(w))
    x = (w - w.mean(-2, keepdim=True)) / torch.std(w, dim=-2, keepdim=True, unbiased=True)
    return AO.median_filter(x, width).mean(0)


def _filter_zero_pad(w, width):
    x = AO.standardise(torch.as_tensor(np.asarray(w)))
    pad = width // 2
    if x.shape[-1] <= pad:
        return x.mean(0)
    xp = F.pad(x, (pad, pad), mode="constant", value=0.0)
    return xp.unfold(-1, width, 1).sort()[0][..., pad].mean(0)


def _filter_mean_first(w, width):
    x = AO.standardise(torch.as_tensor(np.asarray(w))).mean(0, keepdim=True)
    return AO.median_filter(x, width)[0]


def _filter_resoftmax(w, width):
    w = torch.as_tensor(np.asarray(w))
    return AO.filter_matrix((w / w.sum(-1, keepdim=True)).numpy(), width)


def _dtw_swapped_ties(matrix):
    m = -np.asarray(matrix, np.float32)
    n, f = m.shape
    cost = np.full((n + 1, f + 1), np.inf, np.float32)
    trace = np.zeros((n + 1, f + 1), np.int8)
    cost[0, 0] = 0
    for j in range(1, f + 1):
        for i in range(1, n + 1):
            c0, c1, c2 = cost[i - 1, j - 1], cost[i - 1, j], cost[i, j - 1]
            if c0 < c1 and c0 < c2:
                c, t = c0, 0
            elif c2 < c0 and c2 < c1:  # left tested before up: ties between them go up
                c, t = c2, 2
            else:
                c, t = c1, 1
            cost[i, j] = np.float32(m[i - 1, j - 1] + c)
            trace[i, j] = t
    trace[0, :] = 2
    trace[:, 0] = 1
    i, j, out = n, f, []
    while i > 0 or j > 0:
        out.append((i - 1, j - 1))
        t = trace[i, j]
        i, j = (i - 1, j - 1) if t == 0 else ((i - 1, j) if t == 1 else (i, j - 1))
    return np.asarray(out[::-1]).reshape(-1, 2)


@pytest.mark.parametrize("defect", ["unbiased_std", "zero_padding", "swapped_ties", "mean_before_median", "resoftmax"])
def test_defect_is_detected(gold, defect):
    kw = {"unbiased_std": {"filt": _filter_unbiased}, "zero_padding": {"filt": _filter_zero_pad},
          "swapped_ties": {"dtw": _dtw_swapped_ties}, "mean_before_median": {"filt": _filter_mean_first},
          "resoftmax": {"filt": _filter_resoftmax}}[defect]
    assert not _agrees(gold, **kw)


# ---- alignment heads in loaders and blob
def test_hf_generation_config_heads():
    cfg = {"encoder_layers": 4, "decoder_layers": 4, "d_model": 384, "encoder_attention_heads": 6,
           "decoder_attention_heads": 6, "vocab_size": 51865}
    dims = loaders.dims_from_hf_config(cfg, {"alignment_heads": [[2, 2], [3, 0], [3, 5]]})
    assert dims.alignment_heads == [[2, 2], [3, 0], [3, 5]]
    assert loaders.dims_from_hf_config(cfg, {}).alignment_heads is None


def test_ct2_config_heads(tmp_path, monkeypatch):
    import json

    (tmp_path / "config.json").write_text(json.dumps({"alignment_heads": [[1, 1], [3, 0]]}))

    def fake_bin(path):
        emb = np.zeros((51865, 128), np.float32)
        v = {"decoder/embeddings/weight": emb, "decoder/position_encodings/encodings": np.zeros((448, 128), np.float32)}
        for side in ("encoder", "decoder"):
            for i in range(4):
                v[f"{side}/layer_{i}/x"] = np.zeros(1, np.float32)
        return "WhisperSpec", 1, v, {}

    def fake_sd(variables, aliases, dims):
        return W.synth_state_dict(dims, seed=0)

    monkeypatch.setattr(loaders, "read_ct2_model_bin", fake_bin)
    monkeypatch.setattr(loaders, "ct2_to_hf_state_dict", fake_sd)
    dims, tensors = loaders.load_ct2_dir(str(tmp_path))
    assert dims.alignment_heads == [[1, 1], [3, 0]]
    assert tensors["meta.alignment_heads"].tolist() == [[1, 1], [3, 0]]


def test_blob_heads_round_trip_and_default_unchanged():
    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=2)
    plain = W.synth_engine_tensors(dims, seed=3)
    assert "meta.alignment_heads" not in plain
    buf = np.zeros(W.blob_nbytes(plain), np.uint8)
    W.write_blob_into(buf, dims, plain)
    d2, _ = W.read_blob(buf)
    assert d2.alignment_heads is None
    named = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=2, alignment_heads=[[1, 0], [0, 1]])
    t = W.synth_engine_tensors(named, seed=3)
    assert all(np.array_equal(t[k], plain[k]) for k in plain)
    buf = np.zeros(W.blob_nbytes(t), np.uint8)
    W.write_blob_into(buf, named, t)
    d3, t3 = W.read_blob(buf)
    assert d3.alignment_heads == [[1, 0], [0, 1]] and t3["meta.alignment_heads"].dtype == np.int32
    with pytest.raises(ValueError):
        W.pack_state_dict(W.synth_state_dict(named, seed=3),
                          W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=2, alignment_heads=[[2, 0]]))


def test_oracle_capture_rows_and_probs():
    """The oracle's capture: rows are softmax distributions over 1500 frames before the cut, the token probabilities are
    the restricted softmax, and the teacher-forced logits agree with the oracle's own step-by-step decoder."""
    from oracle.whisper_ref import WhisperOracle

    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=2)
    oracle = WhisperOracle(dims, W.synth_engine_tensors(dims, seed=5))
    enc = torch.randn(1500, 128, generator=torch.Generator().manual_seed(1))
    start = [dims.sot, dims.lang_first, dims.transcribe]
    text = [400, 401, 977, 1200]
    toks = start + [dims.no_timestamps] + text
    logits, probs = AO.forced_capture(oracle, enc, toks, AO.default_heads(dims))
    assert probs.shape == (2, len(toks), 1500)
    assert torch.allclose(probs.sum(-1), torch.ones(()), atol=1e-5)
    ref = oracle.forced_logits(enc, toks)
    assert torch.allclose(logits, ref, atol=1e-3, rtol=1e-4)
    w, tp = AO.capture_window(oracle, enc, start, text, 1000)
    assert w.shape == (2, len(text) + 1, 500)
    lp = torch.log_softmax(ref[3:3 + len(text), : dims.eot], -1)[torch.arange(len(text)), torch.tensor(text)]
    assert np.allclose(np.log(tp), lp.numpy(), atol=1e-4)


def test_oracle_capture_matches_transformers(gold):
    """The oracle's capture (head indexing, 1/8 scale, softmax over all 1500 frames, no renormalisation) against the
    cross-attention probabilities transformers returns with output_attentions=True, on the alignment-scripted model."""
    from oracle import logmel as om
    from oracle.whisper_ref import WhisperOracle

    heads = [[2, 1], [3, 0], [3, 1]]
    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=4, alignment_heads=heads)
    oracle = WhisperOracle(dims, W.synth_engine_tensors(dims, seed=11, align_script=(30.0, 250.0, 3000.0)))
    enc = oracle.encode(om.log_mel_batch([om.synth_utterance(61440, 1234)]))
    _, probs = AO.forced_capture(oracle, enc[0], [int(t) for t in gold["cap_tokens"]], AO.default_heads(dims))
    assert np.abs(probs[:, :, gold["cap_frames"]].numpy() - gold["cap_probs"]).max() < 1e-5
    assert np.abs(probs.argmax(-1).numpy() - gold["cap_argmax"]).max() <= 2  # (a peak's top is a few frames wide)
    # the script's peaks move monotonically with the decoder position: the paths it produces are not trivial
    assert (np.diff(gold["cap_argmax"], axis=1) > 0).all()


def test_align_script_default_off():
    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=2)
    a, b = W.synth_state_dict(dims, seed=4), W.synth_state_dict(dims, seed=4, align_script=None)
    assert all(np.array_equal(a[k], b[k]) for k in a)
