"""The encoder one stage at a time, against the float64 reference of tests/enc_oracle.py that rounds where the chain
stores.  Handle.debug_enc_stem / debug_enc_ln / debug_enc_layer run the functions the encoder itself runs
(enc_stem_run, layernorm_f32_to_f16_run, enc_layer_run in csrc/engine.cu) on caller data.

  * one synthetic model per Whisper width, d = 384, 512, 768, 1024, 1280 (6 .. 20 heads), 2 encoder layers
  * stem at 1 and 3 windows: conv1 against float64 within a derived bound, conv2 + positions from the device's own h1
    within tol_gemm, and h1's zero rows and x's padding rows exactly 0, also after a larger call on other content
  * LayerNorm at every d = 128 .. 1536 (multiples of 128), 1, 7, 9 and 4608 rows, with and without programmatic
    dependent launch, Gaussian, constant and offset rows, the rest of the kernel's last 8-row block untouched
  * a layer stage by stage at 1, 2 and 3 windows, both V layouts of the attention, layers 0 and 1: each launch against
    float64 from the device's own input to it; residual rows with per-window offsets, outlier channels at +-100 in
    every fifth row, rows offset 16 times their spread and padding rows at +-1e4 (valid rows bit-identical to a run with
    zero padding rows); attention far from uniform on these weights
  * the layer end to end against the all-float64 chain; the snapshotted run, the production sequence with and without
    programmatic dependent launch and a repeat bit-identical; every window of a call bit-identical to its solo run
  * the whole encoder (stem, 2 layers, ln_post) against float64, with PDL on and off bit-identical and the SIMT
    attention (option attn_ref) under both V layouts

The tests without the gpu mark check the comparators: each rejects a reference with a known defect."""
import functools

import numpy as np
import pytest

from tests import enc_oracle as O
from tests.test_gpu_decoder_kernels import check_ln_out, ln_params, ln_ref, ln_rows, ln_tol, within
from tests.test_gpu_kernels import attn_tol, bits, note_ratio, sentinel, tol_gemm, worst_ratio
from willow_inference_server_b200 import weights as W

WIDTHS = [(384, 6), (512, 8), (768, 12), (1024, 16), (1280, 20)]
LN_GROUP = 3  # the encoder's LayerNorm adds each float4 left to right (ln_tol)
SENT16 = np.uint16(0x7E5A)
OFFSET_ROWS = (5, 777, 1499)  # rows offset 16 times their spread in the layer inputs
# Rows with the +-100 outlier channels.  In every row they would dominate LayerNorm's variance and leave every query and
# key the same two channels: attention then spreads almost uniformly (median peak 0.006 at d = 384), where a key or head
# mix-up would hardly show.
OUTLIER_EVERY = 5
# Layer and whole-encoder tolerances, fractions of each reference row's rms, chosen from measurement (H100 80GB HBM3,
# 700 W): see DESIGN section 5 for the measured worst per width.
RTOL_LAYER = 3e-3  # measured worst 1.4e-3 (d = 768)
RTOL_ENC = 1.5e-2  # measured worst 7.7e-3 (d = 768)
MIN_PEAK = 0.05  # median largest attention probability of a valid query row and head: far from uniform (1 / 1500)


@functools.lru_cache(maxsize=5)
def blob(d, H):
    dims = W.WhisperDims(d_model=d, n_heads=H, n_enc_layers=2, n_dec_layers=1)
    t = W.synth_engine_tensors(dims, seed=d)
    buf = np.zeros(W.blob_nbytes(t), np.uint8)
    W.write_blob_into(buf, dims, t)
    return buf


@functools.lru_cache(maxsize=5)
def model(d, H):
    from willow_inference_server_b200 import _lib

    buf = blob(d, H)
    return O.Model(buf), _lib.Handle.from_host(buf, 0)


@pytest.fixture(scope="module")
def fe():
    from willow_inference_server_b200 import _lib

    return _lib.Handle.frontend(0)


# ------------------------------------------------------------------------------------------------ inputs
def mel_case(B, seed):
    """log-mel windows [B, 80, 3000]: uniform between each window's floor and maximum (2 apart, as Whisper's clamp
    leaves them), stretches at the floor and at the maximum, and first / last frames of their own"""
    rng = np.random.default_rng([seed, B])
    mel = np.empty((B, 80, 3000), np.float32)
    for b in range(B):
        top = 1.0 + 0.15 * b + 0.05 * seed
        m = rng.uniform(top - 2, top, (80, 3000))
        m[:, 400 + 50 * b: 700 + 50 * b] = top - 2
        m[:, 1800 - 50 * b: 2100 - 50 * b] = top
        m[:, 0] = np.linspace(top - 2, top, 80)
        m[:, -1] = np.linspace(top, top - 1.5, 80)
        mel[b] = m
    return mel


def enc_ln_rows(rng, R, d):
    """ln_rows (Gaussian, constant rows 1 and 2, rows 3 and 8 offset 100 times their spread) with row 4 offset 250
    times its spread, cut to R rows"""
    x = ln_rows(rng, max(R, 9), d)
    x[4] = 250.0 + rng.standard_normal(d)
    return x[:R]


def layer_input(d, B, seed=0, pad=1e4):
    """residual [B, 1536, d]: Gaussian rows around a per-window offset pattern; in every OUTLIER_EVERY-th row channels 3
    and d / 2 + 7 at +100 / -100; rows OFFSET_ROWS offset 16 times their spread; padding rows 1500..1535 at +-pad"""
    rng = np.random.default_rng([d, B, seed])
    x = rng.standard_normal((B, O.T_PAD, d)) + 0.5 * rng.standard_normal((B, 1, d))
    x[:, ::OUTLIER_EVERY, 3], x[:, ::OUTLIER_EVERY, d // 2 + 7] = 100.0, -100.0
    x[:, list(OFFSET_ROWS)] += 16.0
    x[:, O.T_ENC:] = pad * rng.choice([-1.0, 1.0], (B, O.T_PAD - O.T_ENC, d))
    return x.astype(np.float32)


def sample_rows(rng, B, extra=(0, 1, 1499, 1500, 1535), n_random=12, hi=O.T_ENC):
    """query rows [B, n] per window: `extra` (and OFFSET_ROWS) plus n_random others below hi"""
    fixed = sorted(set(extra) | set(OFFSET_ROWS))
    out = []
    for _ in range(B):
        pool = np.setdiff1d(np.arange(hi), fixed)
        out.append(np.sort(np.concatenate([fixed, rng.choice(pool, n_random, replace=False)])))
    return np.stack(out)


class options:
    """handle options for a block, restored to the encoder defaults afterwards"""

    DEFAULTS = {"enc_pdl": 1, "attn_v_mn_major": 1, "attn_ref": 0}

    def __init__(self, h, **kw):
        self.h, self.kw = h, kw

    def __enter__(self):
        for k, v in self.kw.items():
            self.h.set_option(k, v)

    def __exit__(self, *exc):
        for k in self.kw:
            self.h.set_option(k, self.DEFAULTS[k])


# ------------------------------------------------------------------------------------------------ stem
def check_stem(m, mel, h1, x, tag, rng):
    B, d = mel.shape[0], m.d
    pre, S = O.conv1(m, mel)
    ref = O.gelu(pre)
    win = h1[: B * O.H1_ROWS].reshape(B, O.H1_ROWS, d)
    got = win[:, 1: 1 + O.N_FRAMES]
    tol = O.conv1_tol(pre, S, ref)
    note_ratio(f"conv1 d {d}", worst_ratio(got, ref, tol))
    assert within(got, ref, tol), tag
    assert np.all(bits(win[:, 0]) == 0) and np.all(bits(win[:, 1 + O.N_FRAMES:]) == 0), tag
    rows = sample_rows(rng, B, extra=(0, 1, 2, 749, 1497, 1498, 1499), n_random=64)
    acc, r, ref2 = O.conv2(m, h1, B, rows)
    got2 = O.gather(x, rows)
    tol2 = tol_gemm(3 * d, r, ref2, "conv2", acc)
    note_ratio(f"conv2 + pos d {d}", worst_ratio(got2, ref2, tol2))
    assert within(got2, ref2, tol2), tag
    assert np.all(bits(x[:, O.T_ENC:]) == 0), tag


@pytest.mark.gpu
@pytest.mark.parametrize("d,H", WIDTHS)
def test_stem_matches_fp64(d, H):
    m, h = model(d, H)
    rng = np.random.default_rng(d)
    for B, seed in ((3, 0), (1, 1)):  # the 1-window call follows a larger one on other content
        mel = mel_case(B, seed)
        h1, x = h.debug_enc_stem(mel)
        check_stem(m, mel, h1, x, (d, B), rng)


# ------------------------------------------------------------------------------------------------ LayerNorm
@pytest.mark.gpu
@pytest.mark.parametrize("d", list(range(128, 1537, 128)))
def test_layernorm_matches_fp64(fe, d):
    rng = np.random.default_rng(d)
    g, b = ln_params(rng, d)
    for rows in (1, 7, 9, 3 * O.T_PAD):
        x = enc_ln_rows(rng, rows, d).astype(np.float32)
        for pdl in (False, True):
            y = sentinel(((rows + 7) // 8 * 8, d), np.float16)
            fe.debug_enc_ln(x, g, b, y, pdl=pdl)
            check_ln_out(x, y[:rows], g, b, (d, rows, pdl), LN_GROUP, "encoder LayerNorm (fp16 out)")
            assert np.all(bits(y[rows:]) == SENT16), (d, rows, pdl)


# ------------------------------------------------------------------------------------------------ one layer
def check_stages(m, i, x_in, st, x_out, rows, vmn, tag):
    """every launch of the layer against float64 from the device's own input to it"""
    p, d, H = f"enc.{i}.", m.d, m.H
    name = f"encoder layer d {d}"
    f = m.f
    check_ln_out(x_in.reshape(-1, d), st["xn1"].reshape(-1, d), f(p + "ln1.g"), f(p + "ln1.b"), tag, LN_GROUP, f"{name} LN1")
    qkv = st["qkv"] if vmn else O.qkv_with_v(st["qkv"], st["vt"])
    acc, r = O.linear(O.gather(st["xn1"], rows), f(p + "qkv.w"), f(p + "qkv.b"))
    tol = tol_gemm(d, r, acc, "f16")
    got = O.gather(qkv, rows)
    note_ratio(f"{name} qkv", worst_ratio(got, acc, tol))
    assert within(got, acc, tol), tag
    ref, pmax = O.attention(qkv, H, rows)
    tol = attn_tol(qkv, H, ref)
    got = O.gather(st["ctx"], rows)
    note_ratio(f"{name} attention", worst_ratio(got, ref, tol))
    assert within(got, ref, tol), tag
    peak = float(np.median(pmax[rows < O.T_ENC]))
    note_ratio(f"{name} median peak attention probability (>= {MIN_PEAK})", peak)
    assert peak >= MIN_PEAK, (tag, peak)
    # residual GEMMs: x += acc + bias rounds acc + bias once more (2^-24 of it) before the residual add
    for stage, src, w, b, out, res in (("o-proj", "ctx", "o.w", "o.b", st["x_o"], x_in),
                                       ("fc2", "fc1", "fc2.w", "fc2.b", x_out, st["x_o"])):
        acc, r = O.linear(O.gather(st[src], rows), f(p + w), f(p + b))
        ref = O.gather(res, rows) + acc
        tol = tol_gemm(st[src].shape[-1], r, ref, "f32") + O.U * np.abs(acc)
        got = O.gather(out, rows)
        note_ratio(f"{name} {stage}", worst_ratio(got, ref, tol))
        assert within(got, ref, tol), (tag, stage)
        if stage == "o-proj":
            check_ln_out(st["x_o"].reshape(-1, d), st["xn2"].reshape(-1, d), f(p + "ln2.g"), f(p + "ln2.b"), tag, LN_GROUP,
                         f"{name} LN2")
            acc, r = O.linear(O.gather(st["xn2"], rows), f(p + "fc1.w"), f(p + "fc1.b"))
            ref = O.gelu(acc)
            tol = tol_gemm(d, r, ref, "gelu16", acc)
            got = O.gather(st["fc1"], rows)
            note_ratio(f"{name} fc1", worst_ratio(got, ref, tol))
            assert within(got, ref, tol), tag


LAYER_CASES = [(1, 1, 0), (2, 0, 1), (3, 1, 1), (3, 0, 0)]  # (windows, attn_v_mn_major, layer)


@pytest.mark.gpu
@pytest.mark.parametrize("B,vmn,layer", LAYER_CASES)
@pytest.mark.parametrize("d,H", WIDTHS)
def test_layer_stage_by_stage(d, H, B, vmn, layer):
    m, h = model(d, H)
    tag = (d, B, vmn, layer)
    x_in = layer_input(d, B)
    rows = sample_rows(np.random.default_rng([d, B, layer]), B)
    with options(h, attn_v_mn_major=vmn):
        x_out, st, plans = h.debug_enc_layer(layer, x_in, stages=True)
        check_stages(m, layer, x_in, st, x_out, rows, vmn, tag)
        # the all-float64 chain from the residual
        ref = O.layer(m, layer, x_in.astype(np.float64), rows)
        note_ratio(f"encoder layer d {d} end to end: max |error| / row rms", O.row_ratio(O.gather(x_out, rows), ref, 1.0))
        assert O.row_ratio(O.gather(x_out, rows), ref, RTOL_LAYER) <= 1, tag
        # the production sequence (no snapshots) under PDL off / on, and a repeat: bit for bit
        for pdl in (0, 1, 1):
            with options(h, enc_pdl=pdl):
                again, _, _ = h.debug_enc_layer(layer, x_in)
            assert np.array_equal(bits(again), bits(x_out)), (tag, pdl)
        # padding rows only ever reach padding rows
        x0 = x_in.copy()
        x0[:, O.T_ENC:] = 0
        out0, _, _ = h.debug_enc_layer(layer, x0)
        assert np.array_equal(bits(out0[:, :O.T_ENC]), bits(x_out[:, :O.T_ENC])), tag
        # every window as its own call
        if B > 1:
            for b in range(B):
                solo, _, solo_plans = h.debug_enc_layer(layer, x_in[b: b + 1])
                print(f"d {d} window {b} of {B}: plans {plans}, solo {solo_plans}")
                assert np.array_equal(bits(solo[0]), bits(x_out[b])), (tag, b, plans, solo_plans)


# ------------------------------------------------------------------------------------------------ whole encoder
@pytest.mark.gpu
@pytest.mark.parametrize("d,H", WIDTHS)
def test_encoder_matches_fp64(d, H):
    m, h = model(d, H)
    mel = mel_case(2, 3)
    rows = sample_rows(np.random.default_rng(d), 2, extra=(0, 1, 5, 777, 1498, 1499), n_random=24)
    ref = O.encoder(m, mel, rows)
    outs = {}
    for pdl, vmn, simt in ((1, 1, 0), (0, 1, 0), (1, 0, 0), (0, 0, 0), (1, 1, 1), (1, 0, 1)):
        with options(h, enc_pdl=pdl, attn_v_mn_major=vmn, attn_ref=simt):
            outs[pdl, vmn, simt] = h.debug_encode(mel)
    for vmn in (1, 0):
        assert np.array_equal(bits(outs[1, vmn, 0]), bits(outs[0, vmn, 0])), (d, vmn)
    for key, out in outs.items():
        got = O.gather(out, rows)
        what = f"encoder d {d}, {'SIMT' if key[2] else 'wgmma'} attention"
        r = O.row_ratio(got, ref, 1.0)
        note_ratio(f"{what}: max |error| / row rms", r)
        assert r <= RTOL_ENC, (d, key, r)


# ------------------------------------------------------------------------------------------------ arguments
@pytest.mark.gpu
def test_debug_entries_reject_bad_arguments_and_grow(fe):
    from willow_inference_server_b200 import _lib

    m, _ = model(384, 6)
    h = _lib.Handle.from_host(blob(384, 6), 0)  # a fresh handle: nothing encoded yet
    x1 = layer_input(384, 1)
    for layer in (-1, 2):
        with pytest.raises(ValueError):
            h.debug_enc_layer(layer, x1)
    with pytest.raises(ValueError):
        h.debug_enc_layer(0, x1[:0])
    with pytest.raises(ValueError):
        h.debug_enc_stem(mel_case(1, 0)[:0])
    with pytest.raises(ValueError):
        fe.debug_enc_stem(mel_case(1, 0))  # a handle without a model
    g, b = ln_params(np.random.default_rng(0), 384)
    with pytest.raises(ValueError):
        fe.debug_enc_ln(np.zeros((0, 384), np.float32), g, b, np.zeros((0, 384), np.float16))
    for d in (320, 1664):
        with pytest.raises(ValueError):
            fe.debug_enc_ln(np.zeros((8, d), np.float32), *np.ones((2, d), np.float32), np.zeros((8, d), np.float16))
    # 1 window, then 3 (the buffers are reallocated), then 1 again on other content
    rng = np.random.default_rng(1)
    for B, seed in ((1, 4), (3, 5), (1, 6)):
        mel = mel_case(B, seed)
        h1, x = h.debug_enc_stem(mel)
        check_stem(m, mel, h1, x, ("grow", B), rng)
    out, _, _ = h.debug_enc_layer(1, layer_input(384, 3))
    assert np.all(np.isfinite(out))
    h.close()


# ------------------------------------------------------------------------------------------------ comparator power (CPU)
@functools.lru_cache(maxsize=1)
def cpu_model():
    return O.Model(blob(384, 6))


def test_stem_comparators_reject_injected_defects():
    m = cpu_model()
    mel = mel_case(1, 0)
    pre, S = O.conv1(m, mel)
    ref = O.gelu(pre)
    tol = O.conv1_tol(pre, S, ref)
    assert within(ref.astype(np.float16), ref, tol)
    for defect in ("taps_reversed", "no_left_pad"):
        bad = O.gelu(O.conv1(m, mel, defect)[0]).astype(np.float16)
        assert not within(bad, ref, tol), defect
    h1 = O.h1_layout(ref.astype(np.float16))
    rows = sample_rows(np.random.default_rng(0), 1, extra=(0, 1, 2, 1498, 1499), n_random=64)
    acc, r, ref2 = O.conv2(m, h1, 1, rows)
    tol2 = tol_gemm(3 * m.d, r, ref2, "conv2", acc)
    assert within(ref2.astype(np.float32), ref2, tol2)
    bad = O.conv2(m, h1, 1, rows, "pos_shift")[2].astype(np.float32)
    assert not within(bad, ref2, tol2)
    assert not np.all(bits(O.stem_padding(m, 1, "pos_padding").astype(np.float32)) == 0)
    assert np.all(bits(O.stem_padding(m, 1).astype(np.float32)) == 0)


def test_layernorm_comparator_rejects_one_pass_variance():
    rng = np.random.default_rng(3)
    for d in (384, 1280):
        g, b = ln_params(rng, d)
        x = enc_ln_rows(rng, 9, d).astype(np.float32)
        ref = ln_ref(x) * g + b
        tol = ln_tol(x, g, b, ref, LN_GROUP)
        assert within(ref.astype(np.float16), ref, tol)
        one = O.layer_norm(x, g, b, one_pass=True).astype(np.float16)
        assert not within(one[[3, 4, 8]], ref[[3, 4, 8]], tol[[3, 4, 8]]), d


def cpu_layer_case(B=2, layer=0):
    """the reference chain's own stage values on a layer input at d = 384: (model, x, xn1, qkv, rows)"""
    m = cpu_model()
    p = f"enc.{layer}."
    x = layer_input(m.d, B).astype(np.float64)
    xn = O.r16(O.layer_norm(x, m.f(p + "ln1.g"), m.f(p + "ln1.b")))
    qkv = O.r16(xn @ m.f(p + "qkv.w").T + m.f(p + "qkv.b")).astype(np.float16)
    rows = sample_rows(np.random.default_rng(7), B)
    return m, x, xn, qkv, rows


def test_attention_comparator_rejects_injected_defects():
    m, x, xn, qkv, rows = cpu_layer_case()
    ref, pmax = O.attention(qkv, m.H, rows)
    assert np.median(pmax[rows < O.T_ENC]) >= MIN_PEAK
    tol = attn_tol(qkv, m.H, ref)
    assert within(ref.astype(np.float16), ref, tol)
    for kw in (dict(scale=m.d ** -0.5), dict(n_keys=O.T_PAD), dict(window_shift=1)):
        bad = O.attention(qkv, m.H, rows, **kw)[0].astype(np.float16)
        assert not within(bad, ref, tol), kw


def test_layer_comparators_reject_injected_defects():
    """o-projection bias dropped: rejected by the o-proj stage bound and by the end-to-end layer tolerance; the window
    and mask defects by the layer tolerance too.  tanh-GELU in fc1 is reported against the fc1 stage bound."""
    m, x, xn, qkv, rows = cpu_layer_case()
    p = "enc.0."
    ctx = O.r16(O.attention(qkv, m.H, rows)[0])
    acc, r = O.linear(ctx, m.f(p + "o.w"), m.f(p + "o.b"))
    ref = O.gather(x, rows) + acc
    tol = tol_gemm(m.d, r, ref, "f32") + O.U * np.abs(acc)
    assert within(ref.astype(np.float32), ref, tol)
    bad = O.gather(x, rows) + O.linear(ctx, m.f(p + "o.w"), 0)[0]
    assert not within(bad.astype(np.float32), ref, tol)
    full = O.layer(m, 0, x, rows)
    for defect, kw in (("o_bias", None), (None, dict(window_shift=1)), (None, dict(n_keys=O.T_PAD)),
                       (None, dict(scale=m.d ** -0.5))):
        assert O.row_ratio(O.layer(m, 0, x, rows, defect, kw), full, RTOL_LAYER) > 1, (defect, kw)
    # fc1 with tanh-GELU against the erf-GELU stage bound
    y = O.gather(x, rows) + ctx @ m.f(p + "o.w").T + m.f(p + "o.b")
    xn2 = O.r16(O.layer_norm(y, m.f(p + "ln2.g"), m.f(p + "ln2.b")))
    acc, r = O.linear(xn2, m.f(p + "fc1.w"), m.f(p + "fc1.b"))
    ref = O.gelu(acc)
    tol = tol_gemm(m.d, r, ref, "gelu16", acc)
    assert within(ref.astype(np.float16), ref, tol)
    ratio = worst_ratio(O.gelu_tanh(acc).astype(np.float16), ref, tol)
    print(f"tanh-GELU at the fc1 stage bound: worst error / tolerance {ratio:.3g}")
    assert ratio > 1  # rejected
