"""CPU: the large-v3 family's host side -- the 128-bin filterbank and log-mel oracle against transformers, the oracle on a
v3-shaped model against HF Whisper (tests/golden/*128*, whisper_v3_hf.npz, from scripts/gen_golden_logmel128_hf.py and
scripts/gen_golden_whisper_v3_hf.py), the 51866-token vocabulary layout through every loader, and the bin-count rule."""
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import logmel as om
from oracle.whisper_ref import WhisperOracle
from willow_inference_server_b200 import loaders, weights as W
from willow_inference_server_b200.languages import LANGUAGE_CODES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "willow_inference_server_b200", "csrc")
MEL128_SHA256 = "e399c2d72d2f7375e503c296d8453cefcc0c1e47a9c1a0a09e0d70f59c820f20"
# the 51866-token vocabulary: 100 languages (<|yue|> = 50358) move every later special id up by one
V3_IDS = dict(sot=50258, eot=50257, lang_first=50259, n_langs=100, translate=50359, transcribe=50360, sot_lm=50361,
              sot_prev=50362, no_speech=50363, no_timestamps=50364)
V2_IDS = dict(sot=50258, eot=50257, lang_first=50259, n_langs=99, translate=50358, transcribe=50359, sot_lm=50360,
              sot_prev=50361, no_speech=50362, no_timestamps=50363)


def _ids(dims):
    return {k: getattr(dims, k) for k in V3_IDS}


def _parse_table(path, n):
    """the generated __constant__ table -> dense float32 [n, 201]"""
    txt = open(path).read()
    body = lambda name: txt.split(name, 1)[1].split("{", 1)[1].split("};", 1)[0]  # noqa: E731
    pre = "kMel" if n == 80 else "kMel128"
    starts = [int(v) for v in body(f"{pre}Start[").split(",")]
    lens = [int(v) for v in body(f"{pre}Len[").split(",")]
    rows = [r.split("}")[0] for r in body(f"{pre}W[").split("{")[1:]]
    w = np.zeros((n, 201), np.float32)
    for m, (s, ln, r) in enumerate(zip(starts, lens, rows)):
        w[m, s:s + ln] = np.array([float(v.strip().rstrip("f")) for v in r.split(",")[:ln]], np.float32)
    return w


# ------------------------------------------------------------------------------------------------- filterbank tables
def test_80_bin_table_is_the_reference_asset_and_unchanged():
    w = _parse_table(os.path.join(CSRC, "mel_filters_table.inc"), 80)
    assert om.mel_filters_sha256(w + np.float32(0)) == om.MEL_FILTERS_SHA256
    # byte-identical to what the generator has always written (pinned by content hash of the file)
    txt = open(os.path.join(CSRC, "mel_filters_table.inc"), "rb").read()
    assert b"sha256(raw f32 [80,201]) = " + om.MEL_FILTERS_SHA256.encode() in txt
    assert b"kMel128" not in txt


def test_128_bin_table_matches_transformers_and_is_pinned(golden_dir):
    w = _parse_table(os.path.join(CSRC, "mel_filters_table128.inc"), 128)
    assert om.mel_filters_sha256(w + np.float32(0)) == MEL128_SHA256
    assert om.mel_filters_sha256(om.slaney_mel_filterbank(n_mels=128)) == MEL128_SHA256
    hf = np.load(os.path.join(golden_dir, "logmel128_hf.npz"))["filters"].astype(np.float64)
    assert hf.shape == (128, 201) and np.abs(w.astype(np.float64) - hf).max() < 1e-8
    nz = (w != 0).sum(1)
    assert int(nz.sum()) == 394 and nz.min() >= 1 and nz.max() <= 16  # MEL_MAXNZ


def test_generator_reproduces_both_tables(tmp_path):
    # the generator writes into the tree: run it on a copy and compare bytes
    import shutil

    for sub in ("oracle", "scripts"):
        shutil.copytree(os.path.join(ROOT, sub), tmp_path / sub)
    os.makedirs(tmp_path / "willow_inference_server_b200" / "csrc")
    subprocess.run([sys.executable, str(tmp_path / "scripts" / "gen_mel_table.py")], check=True, capture_output=True)
    for f in ("mel_filters_table.inc", "mel_filters_table128.inc"):
        a = open(tmp_path / "willow_inference_server_b200" / "csrc" / f, "rb").read()
        b = open(os.path.join(CSRC, f), "rb").read()
        assert hashlib.sha256(a).digest() == hashlib.sha256(b).digest(), f


# ------------------------------------------------------------------------------------------------- oracle vs HF
def test_oracle_logmel_128_matches_transformers(golden_dir):
    g = np.load(os.path.join(golden_dir, "logmel128_hf.npz"))
    f = om.slaney_mel_filterbank(n_mels=128)
    names = [k[:-2] for k in g.files if k.endswith("_n")]
    assert len(names) == 4
    for name in names:
        n, seed = (int(v) for v in g[name + "_n"])
        mel = om.log_mel_spectrogram(om.pad_or_trim(om.synth_utterance(n, seed)), f)
        assert mel.shape == (128, 3000)
        assert np.abs(mel[:, ::16] - g[name + "_sub"]).max() < 1e-4, name


@pytest.fixture(scope="module")
def v3(golden_dir):
    g = np.load(os.path.join(golden_dir, "whisper_v3_hf.npz"))
    d, h, le, ld, nm, nv = (int(v) for v in g["cfg"])
    dims = W.WhisperDims(d_model=d, n_heads=h, n_enc_layers=le, n_dec_layers=ld, n_mels=nm, n_vocab=nv)
    tensors = W.synth_engine_tensors(dims, seed=int(g["seed"]), eot_ramp=(int(g["eot_ramp"][0]), float(g["eot_ramp"][1])))
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    o = WhisperOracle.from_blob(buf)
    mel = om.log_mel_batch([om.synth_utterance(61440, 1234), om.synth_utterance(160000, 5)],
                           om.slaney_mel_filterbank(n_mels=128))
    return g, o, mel, o.encode(mel)


def test_v3_blob_round_trip(v3):
    g, o, mel, enc = v3
    assert (o.dims.n_mels, o.dims.n_vocab, o.dims.n_enc_layers, o.dims.n_dec_layers) == (128, 51866, 4, 2)
    assert _ids(o.dims) == V3_IDS and mel.shape == (2, 128, 3000)


def test_v3_encoder_matches_hf(v3):
    g, o, mel, enc = v3
    assert enc.shape == (2, 1500, o.dims.d_model)
    assert np.abs(enc[:, ::25].numpy() - g["enc_sub"]).max() < 2e-5


def test_v3_forced_logits_match_hf(v3):
    g, o, mel, enc = v3
    lg = o.forced_logits(enc[0], [int(t) for t in g["forced"]])
    assert lg.shape[1] == 51866
    assert np.abs(lg[:, g["vocab_idx"]].numpy() - g["logits_sub"]).max() < 1e-4


# ------------------------------------------------------------------------------------------------- vocabulary layout
def test_vocab_layout_of_both_multilingual_vocabularies():
    v2, v3 = W.vocab_layout(51865), W.vocab_layout(51866)
    assert {k: v2[k] for k in V2_IDS} == V2_IDS and {k: v3[k] for k in V3_IDS} == V3_IDS
    # 51865: exactly the list the project has always shipped
    assert v2["suppress_ids"] == W.NON_SPEECH_TOKENS_MULTI and W.WhisperDims().suppress_ids == W.NON_SPEECH_TOKENS_MULTI
    assert 50363 in v3["suppress_ids"] and 50358 not in v3["suppress_ids"]  # <|nospeech|> off, <|yue|> live
    assert [t for t in v3["suppress_ids"] if t < 50257] == [t for t in v2["suppress_ids"] if t < 50257]
    assert v3["suppress_ids"][-6:] == [50258, 50359, 50360, 50361, 50362, 50363]
    assert v3["suppress_ids_begin"] == [220, 50257]
    assert _ids(W.WhisperDims(n_vocab=51866)) == V3_IDS and _ids(W.WhisperDims()) == V2_IDS
    # an id given explicitly wins over the layout
    assert W.WhisperDims(n_vocab=51866, no_timestamps=50000).no_timestamps == 50000


def test_for_size_knows_the_v3_family():
    for name, (le, ld) in {"large-v3": (32, 32), "large-v3-turbo": (32, 4), "distil-large-v3": (32, 2)}.items():
        d = W.WhisperDims.for_size(name)
        assert (d.d_model, d.n_heads, d.n_enc_layers, d.n_dec_layers, d.n_mels, d.n_vocab) == (1280, 20, le, ld, 128, 51866)
        assert _ids(d) == V3_IDS
        d.validate()
    d = W.WhisperDims.for_size("large-v2")
    assert (d.n_enc_layers, d.n_dec_layers, d.n_mels, d.n_vocab) == (32, 32, 80, 51865) and _ids(d) == V2_IDS


def test_language_table_has_yue_100th():
    assert len(LANGUAGE_CODES) == 100 and LANGUAGE_CODES[99] == "yue"
    assert V3_IDS["lang_first"] + LANGUAGE_CODES.index("yue") == 50358


def test_n_mels_other_than_80_or_128_is_rejected():
    for n in (96, 0, 64, 256):
        with pytest.raises(ValueError):
            W.WhisperDims(n_mels=n).validate()
        with pytest.raises(ValueError):
            loaders.dims_from_hf_config(dict(_v3_config(), num_mel_bins=n))
    W.WhisperDims(n_mels=128).validate()
    W.WhisperDims(n_mels=80).validate()


# ------------------------------------------------------------------------------------------------- loaders
def _v3_config():
    return dict(d_model=128, encoder_layers=4, decoder_layers=2, encoder_attention_heads=2, decoder_attention_heads=2,
                vocab_size=51866, num_mel_bins=128, max_target_positions=448, max_source_positions=1500,
                decoder_start_token_id=50258, eos_token_id=50257)


def _v3_generation_config():
    """the generation_config.json layout of openai/whisper-large-v3 (ids of the 51866-token vocabulary)"""
    lang = {f"<|{c}|>": 50259 + i for i, c in enumerate(LANGUAGE_CODES)}
    sup = [t for t in W.NON_SPEECH_TOKENS_MULTI if t < 50257] + [50258, 50359, 50360, 50361, 50362, 50363]
    return dict(lang_to_id=lang, task_to_id={"translate": 50359, "transcribe": 50360}, no_timestamps_token_id=50364,
                prev_sot_token_id=50362, suppress_tokens=sup, begin_suppress_tokens=[220, 50257],
                alignment_heads=[[1, 0], [1, 1]], decoder_start_token_id=50258)


@pytest.mark.parametrize("with_gen", [True, False])
def test_hf_directory_of_a_v3_model(tmp_path, with_gen):
    torch = pytest.importorskip("torch")
    tr = pytest.importorskip("transformers")
    c = _v3_config()
    cfg = tr.WhisperConfig(d_model=c["d_model"], encoder_layers=4, decoder_layers=2, encoder_attention_heads=2,
                           decoder_attention_heads=2, encoder_ffn_dim=512, decoder_ffn_dim=512, vocab_size=51866,
                           num_mel_bins=128, decoder_start_token_id=50258, eos_token_id=50257, bos_token_id=50257,
                           pad_token_id=50257)
    torch.manual_seed(4)
    model = tr.WhisperForConditionalGeneration(cfg).eval()
    d = str(tmp_path / "hf")
    model.save_pretrained(d)
    gen_path = os.path.join(d, "generation_config.json")
    if with_gen:
        json.dump(_v3_generation_config(), open(gen_path, "w"))
    elif os.path.exists(gen_path):
        os.remove(gen_path)  # ids derived from the vocabulary size alone
    dims, tensors = loaders.load_hf_dir(d)
    assert (dims.n_mels, dims.n_vocab, dims.n_enc_layers, dims.n_dec_layers) == (128, 51866, 4, 2)
    assert _ids(dims) == V3_IDS
    assert 50363 in dims.suppress_ids and 50358 not in dims.suppress_ids
    assert dims.alignment_heads == ([[1, 0], [1, 1]] if with_gen else None)
    assert tensors["enc.conv1.w"].shape == (128, 384)
    # the blob keeps it all
    out = loaders.convert(d, str(tmp_path / "wisb"))
    d2, _ = W.read_blob(out)
    assert (d2.n_mels, d2.n_vocab) == (128, 51866) and _ids(d2) == V3_IDS
    assert d2.suppress_ids == sorted(set(dims.suppress_ids))


def test_ct2_directory_keeps_128_mels(tmp_path):
    from tests.test_loaders import _ct2_variables, _write_ct2

    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=4, n_dec_layers=2, n_mels=128, n_vocab=51866)
    sd = {k: np.asarray(v, np.float32) for k, v in W.synth_state_dict(dims, seed=6).items()}
    d = tmp_path / "ct2"
    os.makedirs(d)
    _write_ct2(str(d / "model.bin"), _ct2_variables(sd, dims, False), {"decoder/projection/weight": "decoder/embeddings/weight"})
    json.dump({"suppress_ids": W.vocab_layout(51866)["suppress_ids"], "suppress_ids_begin": [220, 50257],
               "lang_ids": list(range(50259, 50359))}, open(d / "config.json", "w"))
    d2, tensors = loaders.load_any(str(d))
    assert (d2.n_mels, d2.n_vocab, d2.n_enc_layers, d2.n_dec_layers) == (128, 51866, 4, 2)
    assert _ids(d2) == V3_IDS and 50363 in d2.suppress_ids
    want = W.pack_state_dict(sd, d2)
    assert tensors["enc.conv1.w"].shape == (128, 384) and np.array_equal(tensors["enc.conv1.w"], want["enc.conv1.w"])
    out = loaders.convert(str(d), str(tmp_path / "wisb"))
    assert W.read_blob(out)[0].n_mels == 128
