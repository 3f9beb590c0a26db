"""Write tests/golden/alignment_hf.npz: Whisper.align's post-processing run through transformers' own code.

Crafted weight stacks [A, R, F] go through the standardisation of WhisperGenerationMixin._extract_token_timestamps
(population std over the rows), ``_median_filter`` and the head mean; the result goes through
``_dynamic_time_warping(-matrix.double())``, as transformers calls it.  Integer-valued matrices with exact cost ties are
run through the DTW alone.  The cross-attention probabilities that transformers' WhisperForConditionalGeneration
returns with ``output_attentions=True`` for a seeded tiny model with alignment heads (``weights.synth_state_dict(
align_script=...)``), teacher-forced on start + <|notimestamps|> + text, pin the oracle's capture (head indexing, scale,
softmax over all 1500 frames).  tests/test_align_rules.py compares tests/align_oracle.py with these arrays.

    python scripts/gen_golden_alignment_hf.py      # needs transformers; runs on the CPU in seconds
"""
import os

import sys

import numpy as np
import torch
from transformers import WhisperConfig, WhisperForConditionalGeneration
from transformers.models.whisper.generation_whisper import _dynamic_time_warping, _median_filter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import logmel as om  # noqa: E402
from willow_inference_server_b200 import weights as W  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "alignment_hf.npz")

# (A, R, F, width): widths 1/3/7/9, F <= width // 2 (identity filter), F = 1, R = 2
CASES = [(3, 6, 40, 7), (2, 5, 33, 1), (4, 7, 25, 3), (2, 9, 50, 9), (3, 6, 3, 7), (2, 4, 1, 3), (2, 2, 17, 7),
         (1, 3, 4, 9)]


def hf_filter(w: torch.Tensor, width: int) -> torch.Tensor:
    std = torch.std(w, dim=-2, keepdim=True, unbiased=False)
    mean = torch.mean(w, dim=-2, keepdim=True)
    w = (w - mean) / std
    return _median_filter(w, width).mean(dim=0)


# tiny model with named alignment heads and the alignment script (the GPU tests use the same recipe)
CAP_CFG = dict(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=4)
CAP_HEADS = [[2, 1], [3, 0], [3, 1]]
CAP_SEED, CAP_SCRIPT = 11, (30.0, 250.0, 3000.0)
CAP_TOKENS = [50258, 50259, 50359, 50363, 400, 9000, 123, 30000, 777, 5150, 20000, 41000, 300, 12345]
CAP_FRAMES = np.arange(0, 1500, 15)


def hf_capture():
    dims = W.WhisperDims(**CAP_CFG, alignment_heads=CAP_HEADS)
    sd = W.synth_state_dict(dims, seed=CAP_SEED, align_script=CAP_SCRIPT)
    cfg = WhisperConfig(
        vocab_size=dims.n_vocab, num_mel_bins=80, d_model=dims.d_model,
        encoder_layers=dims.n_enc_layers, encoder_attention_heads=dims.n_heads, encoder_ffn_dim=4 * dims.d_model,
        decoder_layers=dims.n_dec_layers, decoder_attention_heads=dims.n_heads, decoder_ffn_dim=4 * dims.d_model,
        max_source_positions=1500, max_target_positions=448, activation_function="gelu",
        pad_token_id=50257, bos_token_id=50257, eos_token_id=50257, decoder_start_token_id=50258,
    )
    model = WhisperForConditionalGeneration(cfg).eval()
    model.config._attn_implementation = "eager"  # attention probabilities are returned by the eager path only
    tsd = {k: torch.from_numpy(v) for k, v in sd.items()}
    tsd["proj_out.weight"] = tsd["model.decoder.embed_tokens.weight"]
    model.load_state_dict(tsd, strict=False)
    mel = torch.from_numpy(om.log_mel_batch([om.synth_utterance(61440, 1234)]))
    with torch.no_grad():
        o = model(input_features=mel, decoder_input_ids=torch.tensor([CAP_TOKENS]), output_attentions=True)
    cross = torch.stack([o.cross_attentions[l][0, h] for l, h in CAP_HEADS])  # [A, T, 1500]
    return {"cap_tokens": np.asarray(CAP_TOKENS, np.int32), "cap_frames": CAP_FRAMES.astype(np.int32),
            "cap_probs": cross[:, :, CAP_FRAMES].numpy(), "cap_argmax": cross.argmax(-1).numpy().astype(np.int32)}


def main():
    rng = np.random.default_rng(20261015)
    out = {}
    for k, (A, R, F, width) in enumerate(CASES):
        # rows with a drifting peak, so the path is not a straight line; the softmax runs over F + 12 frames and is cut
        # to F afterwards without renormalising, as the engine's capture is
        logits = rng.standard_normal((A, R, F + 12)).astype(np.float32)
        for r in range(R):
            logits[:, r, :] -= 0.05 * (np.arange(F + 12) - (r + 0.5) * F / R) ** 2 / max(F / R, 1.0)
        w = torch.softmax(torch.from_numpy(logits), -1)[..., :F].contiguous()
        mat = hf_filter(w, width)
        ti, tj = _dynamic_time_warping(-mat.cpu().double().numpy())
        out[f"w{k}"] = w.numpy()
        out[f"width{k}"] = np.int32(width)
        out[f"mat{k}"] = mat.numpy()
        out[f"path{k}"] = np.stack([ti, tj], 1).astype(np.int32)
    # DTW alone on integer-valued matrices: every cost is exact, so ties between predecessors happen and the tie order
    # decides the path
    for k, (R, F) in enumerate([(5, 9), (8, 8), (3, 12), (6, 20)]):
        m = rng.integers(0, 3, (R, F)).astype(np.float32)
        ti, tj = _dynamic_time_warping(-torch.from_numpy(m).double().numpy())
        out[f"tie_mat{k}"] = m
        out[f"tie_path{k}"] = np.stack([ti, tj], 1).astype(np.int32)
    out.update(hf_capture())
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
