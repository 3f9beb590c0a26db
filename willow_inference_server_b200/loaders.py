"""Checkpoint readers: Hugging Face Whisper directories and CTranslate2 model directories -> ``model.wisb``.

SURVEY.md section 8(f) row 3b.  The reference loads CTranslate2 directories ``models/tovera-wis-whisper-<size>/``
(main.py:341-443; fetched by utils.sh:99-108, 265-269); those hold ``model.bin`` +
``config.json`` (suppress_ids, suppress_ids_begin, lang_ids) produced by ``ct2-transformers-converter`` from the HF
checkpoints.  Neither a checkpoint nor the ``ctranslate2`` package exists in the build image, so:

* ``load_hf_dir`` is validated against ``transformers`` itself (tests/test_loaders.py builds a random
  ``WhisperForConditionalGeneration``, saves it with ``save_pretrained`` and reads it back through this module);
* ``read_ct2_model_bin`` / ``load_ct2_dir`` restate the CTranslate2 4.1 container
  (python/ctranslate2/specs/model_spec.py ``_serialize``, binary version 6) and the variable naming of
  specs/whisper_spec.py + transformer_spec.py FROM THE PUBLISHED SOURCE AS REMEMBERED -- **unpinned**: no ``model.bin`` is
  available to check against; the test only proves writer/reader self-consistency and the int8 de-quantisation rule.

Both produce the engine tensors of ``weights.pack_state_dict``; ``convert`` writes the flat blob the C ABI loads.
"""
from __future__ import annotations

import json
import os
import struct

import numpy as np

from . import weights as W

# ----------------------------------------------------------------------------------------------------------- Hugging Face


def dims_from_hf_config(cfg: dict, gen_cfg: dict | None = None) -> W.WhisperDims:
    """HF ``config.json`` (+ optional ``generation_config.json``) -> WhisperDims.  [HF] configuration_whisper.py."""
    gen_cfg = gen_cfg or {}
    if cfg.get("encoder_layers") is None or cfg.get("d_model") is None:
        raise ValueError("not a Whisper config.json (encoder_layers / d_model missing)")
    n_vocab = int(cfg["vocab_size"])
    dims = W.WhisperDims(
        d_model=int(cfg["d_model"]), n_heads=int(cfg["encoder_attention_heads"]),
        n_enc_layers=int(cfg["encoder_layers"]), n_dec_layers=int(cfg["decoder_layers"]), n_vocab=n_vocab,
        n_text_ctx=int(cfg.get("max_target_positions", 448)), n_mels=int(cfg.get("num_mel_bins", 80)),
        n_audio_ctx=int(cfg.get("max_source_positions", 1500)),
        sot=int(cfg.get("decoder_start_token_id", 50258)), eot=int(cfg.get("eos_token_id", 50257)))
    if int(cfg["decoder_attention_heads"]) != dims.n_heads:
        raise ValueError("encoder and decoder head counts differ")
    # multilingual vocabularies (51865 / 51866) carry the language + task tokens; English-only ones (51864) do not
    multilingual = n_vocab >= 51865
    if not multilingual:
        raise ValueError("English-only Whisper checkpoints (vocab 51864) are not supported: WIS ships multilingual models")
    task = gen_cfg.get("task_to_id") or {}
    dims.transcribe = int(task.get("transcribe", dims.transcribe))
    dims.translate = int(task.get("translate", dims.translate))
    lang = gen_cfg.get("lang_to_id") or {}
    if lang:
        ids = sorted(int(v) for v in lang.values())
        if ids != list(range(ids[0], ids[0] + len(ids))):
            raise ValueError("language ids are not contiguous")
        dims.lang_first, dims.n_langs = ids[0], len(ids)
    if "no_timestamps_token_id" in gen_cfg:
        dims.no_timestamps = int(gen_cfg["no_timestamps_token_id"])
    sup = gen_cfg.get("suppress_tokens", cfg.get("suppress_tokens"))
    if sup:
        # CTranslate2's converter stores HF suppress_tokens as config.json:suppress_ids (SURVEY 8a row A11)
        dims.suppress_ids = sorted(set(int(v) for v in sup) | {dims.sot, dims.translate, dims.transcribe})
    beg = gen_cfg.get("begin_suppress_tokens", cfg.get("begin_suppress_tokens"))
    if beg:
        dims.suppress_ids_begin = [int(v) for v in beg]
    dims.validate()
    return dims


def _read_safetensors(path: str) -> dict:
    """Minimal safetensors reader (8-byte header length, JSON table, raw little-endian data) -> {name: ndarray}."""
    dt = {"F32": np.float32, "F16": np.float16, "I64": np.int64, "I32": np.int32, "U8": np.uint8, "BF16": None}
    with open(path, "rb") as f:
        (n,) = struct.unpack("<Q", f.read(8))
        table = json.loads(f.read(n))
        base = 8 + n
        out = {}
        for name, e in table.items():
            if name == "__metadata__":
                continue
            lo, hi = e["data_offsets"]
            f.seek(base + lo)
            raw = f.read(hi - lo)
            if e["dtype"] == "BF16":  # widen: bf16 is the upper half of an fp32
                a = (np.frombuffer(raw, np.uint16).astype(np.uint32) << 16).view(np.float32)
            else:
                a = np.frombuffer(raw, dt[e["dtype"]])
            out[name] = a.reshape(e["shape"])
    return out


def _hf_state_dict(path: str) -> dict:
    st = os.path.join(path, "model.safetensors")
    if os.path.exists(st):
        sd = _read_safetensors(st)
    else:
        idx = os.path.join(path, "model.safetensors.index.json")
        if os.path.exists(idx):
            sd = {}
            for shard in sorted(set(json.load(open(idx))["weight_map"].values())):
                sd.update(_read_safetensors(os.path.join(path, shard)))
        else:
            pt = os.path.join(path, "pytorch_model.bin")
            if not os.path.exists(pt):
                raise FileNotFoundError(f"{path}: no model.safetensors / pytorch_model.bin")
            import torch

            sd = {k: v.float().numpy() for k, v in torch.load(pt, map_location="cpu", weights_only=True).items()}
    # checkpoints saved from WhisperForConditionalGeneration carry the "model." prefix, bare WhisperModel ones do not
    if not any(k.startswith("model.") for k in sd):
        sd = {"model." + k: v for k, v in sd.items()}
    if "model.encoder.embed_positions.weight" not in sd:
        raise ValueError("checkpoint has no encoder positional table")
    return sd


def load_hf_dir(path: str):
    """HF Whisper directory (config.json [+ generation_config.json] + weights) -> (WhisperDims, engine tensors)."""
    cfg = json.load(open(os.path.join(path, "config.json")))
    g = os.path.join(path, "generation_config.json")
    dims = dims_from_hf_config(cfg, json.load(open(g)) if os.path.exists(g) else None)
    return dims, W.pack_state_dict(_hf_state_dict(path), dims)


# ----------------------------------------------------------------------------------------------------------- CTranslate2
CT2_DTYPES = {0: np.float32, 1: np.int8, 2: np.int16, 3: np.int32, 4: np.float16, 5: None}  # 5 = bfloat16


def read_ct2_model_bin(path: str):
    """CTranslate2 ``model.bin`` -> (spec_name, revision, {name: ndarray}, {alias: name}).  UNPINNED (module docstring).

    Layout restated (little endian): u32 binary_version; string spec_name; u32 spec_revision; u32 n_variables;
    per variable {string name; u8 rank; u32 dims[rank]; u8 dtype_id; u32 n_bytes; data}; u32 n_aliases;
    per alias {string alias; string target}.  A string is u16 length (including the trailing NUL) + bytes.
    Binary versions < 5 stored {u8 item_size; u32 n_items} instead of {dtype_id, n_bytes}.
    """
    with open(path, "rb") as f:
        buf = f.read()
    pos = 0

    def take(fmt):
        nonlocal pos
        v = struct.unpack_from("<" + fmt, buf, pos)
        pos += struct.calcsize("<" + fmt)
        return v[0] if len(v) == 1 else v

    def string():
        nonlocal pos
        n = take("H")
        s = buf[pos : pos + n - 1].decode("utf-8")
        pos += n
        return s

    version = take("I")
    if not 2 <= version <= 6:
        raise ValueError(f"unsupported CTranslate2 binary version {version}")
    spec = string()
    revision = take("I")
    n_vars = take("I")
    variables = {}
    for _ in range(n_vars):
        name = string()
        rank = take("B")
        shape = [take("I") for _ in range(rank)]
        if version >= 5:
            dtype_id = take("B")
            n_bytes = take("I")
            if dtype_id not in CT2_DTYPES:
                raise ValueError(f"{name}: unknown dtype id {dtype_id}")
            raw = buf[pos : pos + n_bytes]
            if CT2_DTYPES[dtype_id] is None:
                a = (np.frombuffer(raw, np.uint16).astype(np.uint32) << 16).view(np.float32)
            else:
                a = np.frombuffer(raw, CT2_DTYPES[dtype_id])
        else:
            item, n_items = take("B"), take("I")
            n_bytes = item * n_items
            a = np.frombuffer(buf[pos : pos + n_bytes], {4: np.float32, 2: np.int16, 1: np.int8}[item])
        pos += n_bytes
        variables[name] = a.reshape(shape)
    aliases = {}
    if pos < len(buf):
        for _ in range(take("I")):
            a = string()
            aliases[a] = string()
    return spec, revision, variables, aliases


def ct2_to_hf_state_dict(variables: dict, aliases: dict, dims: W.WhisperDims) -> dict:
    """CTranslate2 WhisperSpec variables -> HF-named fp32 state dict (de-quantising int8/int16 weights:
    w = q / weight_scale[row], the rule of CTranslate2's ``quantize`` -- scale = 127 / max|row|)."""
    v = dict(variables)
    for a, t in aliases.items():
        v[a] = v[t]

    def dense(prefix):
        w = v[prefix + "/weight"]
        if w.dtype in (np.int8, np.int16):
            w = w.astype(np.float32) / np.asarray(v[prefix + "/weight_scale"], np.float32).reshape(-1, 1)
        return np.asarray(w, np.float32), (np.asarray(v[prefix + "/bias"], np.float32) if prefix + "/bias" in v else None)

    d = dims.d_model
    sd = {}

    def ln(dst, src):
        sd[dst + ".weight"] = np.asarray(v[src + "/gamma"], np.float32)
        sd[dst + ".bias"] = np.asarray(v[src + "/beta"], np.float32)

    def conv(dst, src):
        w = v[src + "/weight"]
        if w.dtype in (np.int8, np.int16):
            w = w.astype(np.float32) / np.asarray(v[src + "/weight_scale"], np.float32).reshape(-1, 1, 1)
        sd[dst + ".weight"] = np.asarray(w, np.float32)
        sd[dst + ".bias"] = np.asarray(v[src + "/bias"], np.float32)

    def self_attn(dst, src):
        w, b = dense(src + "/linear_0")  # fused [3d, d]
        for j, nm in enumerate(("q_proj", "k_proj", "v_proj")):
            sd[f"{dst}.{nm}.weight"] = w[j * d : (j + 1) * d]
            if nm != "k_proj":
                sd[f"{dst}.{nm}.bias"] = b[j * d : (j + 1) * d]
        w, b = dense(src + "/linear_1")
        sd[dst + ".out_proj.weight"], sd[dst + ".out_proj.bias"] = w, b

    def ffn(dst, src):
        ln(dst + ".final_layer_norm", src + "/layer_norm")
        sd[dst + ".fc1.weight"], sd[dst + ".fc1.bias"] = dense(src + "/linear_0")
        sd[dst + ".fc2.weight"], sd[dst + ".fc2.bias"] = dense(src + "/linear_1")

    conv("model.encoder.conv1", "encoder/conv1")
    conv("model.encoder.conv2", "encoder/conv2")
    sd["model.encoder.embed_positions.weight"] = np.asarray(v["encoder/position_encodings/encodings"], np.float32)
    ln("model.encoder.layer_norm", "encoder/layer_norm")
    for i in range(dims.n_enc_layers):
        s, t = f"encoder/layer_{i}", f"model.encoder.layers.{i}"
        ln(t + ".self_attn_layer_norm", s + "/self_attention/layer_norm")
        self_attn(t + ".self_attn", s + "/self_attention")
        ffn(t, s + "/ffn")
    sd["model.decoder.embed_tokens.weight"] = dense("decoder/embeddings")[0]
    sd["model.decoder.embed_positions.weight"] = np.asarray(v["decoder/position_encodings/encodings"], np.float32)
    ln("model.decoder.layer_norm", "decoder/layer_norm")
    for i in range(dims.n_dec_layers):
        s, t = f"decoder/layer_{i}", f"model.decoder.layers.{i}"
        ln(t + ".self_attn_layer_norm", s + "/self_attention/layer_norm")
        self_attn(t + ".self_attn", s + "/self_attention")
        ln(t + ".encoder_attn_layer_norm", s + "/attention/layer_norm")
        w, b = dense(s + "/attention/linear_0")  # query
        sd[t + ".encoder_attn.q_proj.weight"], sd[t + ".encoder_attn.q_proj.bias"] = w, b
        w, b = dense(s + "/attention/linear_1")  # fused key/value [2d, d]
        sd[t + ".encoder_attn.k_proj.weight"], sd[t + ".encoder_attn.v_proj.weight"] = w[:d], w[d:]
        sd[t + ".encoder_attn.v_proj.bias"] = b[d:]
        w, b = dense(s + "/attention/linear_2")
        sd[t + ".encoder_attn.out_proj.weight"], sd[t + ".encoder_attn.out_proj.bias"] = w, b
        ffn(t, s + "/ffn")
    return sd


def load_ct2_dir(path: str):
    """CTranslate2 Whisper directory (model.bin + config.json) -> (WhisperDims, engine tensors).  UNPINNED."""
    spec, _rev, variables, aliases = read_ct2_model_bin(os.path.join(path, "model.bin"))
    if "Whisper" not in spec:
        raise ValueError(f"model.bin holds a {spec!r}, not a Whisper model")
    emb = variables.get("decoder/embeddings/weight", variables.get(aliases.get("decoder/embeddings/weight", ""), None))
    d = int(emb.shape[1])
    n_layers = lambda side: 1 + max(int(k.split("/")[1][6:]) for k in variables if k.startswith(side + "/layer_") and
                                    k.split("/")[1][6:].isdigit())  # noqa: E731
    dims = W.WhisperDims(d_model=d, n_heads=d // 64, n_enc_layers=n_layers("encoder"), n_dec_layers=n_layers("decoder"),
                         n_vocab=int(emb.shape[0]), n_text_ctx=int(variables["decoder/position_encodings/encodings"].shape[0]))
    cfg_path = os.path.join(path, "config.json")
    if os.path.exists(cfg_path):
        cfg = json.load(open(cfg_path))
        if cfg.get("suppress_ids"):
            dims.suppress_ids = [int(x) for x in cfg["suppress_ids"]]
        if cfg.get("suppress_ids_begin"):
            dims.suppress_ids_begin = [int(x) for x in cfg["suppress_ids_begin"]]
        if cfg.get("lang_ids"):
            ids = sorted(int(x) for x in cfg["lang_ids"])
            dims.lang_first, dims.n_langs = ids[0], len(ids)
    dims.validate()
    return dims, W.pack_state_dict(ct2_to_hf_state_dict(variables, aliases, dims), dims)


# ----------------------------------------------------------------------------------------------------------- front door
def load_any(path: str):
    """Directory holding model.wisb, an HF checkpoint or a CTranslate2 model -> (WhisperDims, engine tensors)."""
    if os.path.isfile(path):
        return W.read_blob(path)
    if os.path.exists(os.path.join(path, "model.wisb")):
        return W.read_blob(os.path.join(path, "model.wisb"))
    if os.path.exists(os.path.join(path, "model.bin")):
        return load_ct2_dir(path)
    return load_hf_dir(path)


def convert(src: str, dst_dir: str) -> str:
    """Write ``dst_dir/model.wisb`` from an HF or CTranslate2 directory; returns the blob path."""
    dims, tensors = load_any(src)
    os.makedirs(dst_dir, exist_ok=True)
    out = os.path.join(dst_dir, "model.wisb")
    W.write_blob(out, dims, tensors)
    return out


if __name__ == "__main__":
    import sys

    if len(sys.argv) != 3:
        raise SystemExit("usage: python -m willow_inference_server_b200.loaders <hf-or-ct2-dir> <out-dir>")
    print(convert(sys.argv[1], sys.argv[2]))
