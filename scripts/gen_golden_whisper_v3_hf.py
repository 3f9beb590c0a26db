#!/usr/bin/env python
"""Generate tests/golden/whisper_v3_hf.npz with HF transformers' Whisper on a large-v3-shaped model: 128 mel bins,
the 51866-token vocabulary and an encoder deeper than the decoder (4 / 2 layers, small d).

    python scripts/gen_golden_whisper_v3_hf.py

The seeded synthetic weights (willow_inference_server_b200.weights.synth_state_dict) are loaded into
``WhisperForConditionalGeneration``; we record its encoder output and teacher-forced logits (as whisper_hf_tiny.npz
does for the 80-bin family).  Tests regenerate the weights and inputs from the seeds stored here."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from transformers import WhisperConfig, WhisperForConditionalGeneration  # noqa: E402

from oracle import logmel as om  # noqa: E402
from willow_inference_server_b200 import weights as W  # noqa: E402

CFG = dict(d_model=128, n_heads=2, n_enc_layers=4, n_dec_layers=2, n_mels=128, n_vocab=51866)
SEED = 13
EOT_RAMP = (10, 8.0)
PROMPT = [50258, 50259, 50360, 50364]  # sot, <|en|>, <|transcribe|>, <|notimestamps|> of the 51866 vocabulary
FORCED = PROMPT + [100, 2000, 30000, 41000, 12, 50000, 7, 999]


def main():
    dims = W.WhisperDims(**CFG)
    sd = W.synth_state_dict(dims, seed=SEED, eot_ramp=EOT_RAMP)
    cfg = WhisperConfig(
        vocab_size=dims.n_vocab, num_mel_bins=dims.n_mels, d_model=dims.d_model,
        encoder_layers=dims.n_enc_layers, encoder_attention_heads=dims.n_heads, encoder_ffn_dim=4 * dims.d_model,
        decoder_layers=dims.n_dec_layers, decoder_attention_heads=dims.n_heads, decoder_ffn_dim=4 * dims.d_model,
        max_source_positions=1500, max_target_positions=448, activation_function="gelu",
        pad_token_id=50257, bos_token_id=50257, eos_token_id=50257, decoder_start_token_id=50258,
    )
    model = WhisperForConditionalGeneration(cfg).eval()
    tsd = {k: torch.from_numpy(v) for k, v in sd.items()}
    tsd["proj_out.weight"] = tsd["model.decoder.embed_tokens.weight"]
    print(model.load_state_dict(tsd, strict=False))
    filters = om.slaney_mel_filterbank(n_mels=128)
    mel = om.log_mel_batch([om.synth_utterance(61440, 1234), om.synth_utterance(160000, 5)], filters)
    feats = torch.from_numpy(mel)
    with torch.no_grad():
        enc = model.model.encoder(feats).last_hidden_state  # [2,1500,d]
        logits = model(input_features=feats[:1], decoder_input_ids=torch.tensor([FORCED])).logits[0]
    vocab_idx = np.unique(np.concatenate([np.arange(0, dims.n_vocab, 97), np.arange(50250, dims.n_vocab, 3)]))
    np.savez_compressed(
        os.path.join(ROOT, "tests", "golden", "whisper_v3_hf.npz"),
        cfg=np.array([CFG[k] for k in ("d_model", "n_heads", "n_enc_layers", "n_dec_layers", "n_mels", "n_vocab")]),
        seed=np.int64(SEED), eot_ramp=np.array(EOT_RAMP, np.float64), forced=np.array(FORCED),
        enc_sub=enc[:, ::25].numpy(), vocab_idx=vocab_idx, logits_sub=logits[:, vocab_idx].numpy(),
    )


if __name__ == "__main__":
    main()
