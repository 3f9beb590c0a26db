"""float64 reference of the Whisper encoder, one stage at a time, from the blob's fp16 weights (weights.read_blob).

Stages, as the encoder runs them (csrc/engine.cu enc_stem_run / enc_layer_run):
  stem   conv1 (k = 3, padding 1) + erf-GELU into h1 fp16 [B * 3072 + 8, d] (conv1_gelu_kernel: window b's frame f at
         row b * 3072 + 1 + f, every other row zero), then conv2 (stride 2) as a GEMM over h1 with the EPI_CONV2
         epilogue: x = gelu(acc + bias) + pos for rows t < 1500 of each 1536-row window, exactly 0 from row 1500 on
  layer  xn = fp16(LN1(x)); qkv = fp16(xn Wqkv^T + b); ctx = fp16(softmax(q k^T / 8 over keys < 1500) v) per head;
         x += ctx Wo^T + bo; xn = fp16(LN2(x)); h = fp16(gelu(xn W1^T + b1)); x += h W2^T + b2

Everything is computed in float64; the only roundings are the chain's fp16 stores (h1, xn, qkv, ctx, h).  The residual
x, float32 on the device, stays float64 here.  Every stage function takes its input as an argument, so a test can feed
it the device's own input to that stage and check one kernel alone; `layer` chains them from a residual.  Rows are
(window, t) pairs: a stage evaluates only the query rows it is given (`rows`, per window), the attention always reads
every key of the window.

`defect` arguments inject known bugs for the comparator tests: conv1 "taps_reversed" (tap k read as 2 - k),
"no_left_pad" (frame -1 read as frame 0); conv2 "pos_shift" (pos of row t + 1), "pos_padding" (pos added to the padding
rows); attention scale (1 / sqrt(d) instead of 1/8), n_keys = 1536 (padding keys unmasked), window_shift = 1 (window b
reads window b + 1's keys and values); layer "o_bias" (o-projection bias dropped), "gelu_tanh" (tanh GELU in fc1),
"ln_one_pass" (E[x^2] - mean^2 variance in fp32)."""
import numpy as np
from scipy.special import erf

from willow_inference_server_b200 import weights as W

T_ENC, T_PAD, H1_ROWS, N_MELS, N_FRAMES = 1500, 1536, 3072, 80, 3000
U = 2.0 ** -24


def r16(v):
    return np.asarray(v, np.float64).astype(np.float16).astype(np.float64)


def gelu(v):
    return 0.5 * v * (1 + erf(v / np.sqrt(2)))


def gelu_tanh(v):
    return 0.5 * v * (1 + np.tanh(np.sqrt(2 / np.pi) * (v + 0.044715 * v ** 3)))


class Model:
    """the blob's encoder tensors (views), converted to float64 on use"""

    def __init__(self, blob):
        self.dims, self.t = W.read_blob(blob)
        self.d, self.H, self.L = self.dims.d_model, self.dims.n_heads, self.dims.n_enc_layers

    def f(self, name):
        return np.asarray(self.t[name], np.float64)


# ------------------------------------------------------------------------------------------------ stem
def conv1(m, mel, defect=None):
    """-> (pre, S): pre-activation acc + bias [B, 3000, d] and S = sum |a w| + |bias| (the bound's scale) of conv1 on
    log-mel [B, 80, 3000], weights in the engine's layout [d][k * 80 + ci]"""
    mel = np.asarray(mel, np.float64)
    B, d = mel.shape[0], m.d
    w = m.f("enc.conv1.w").reshape(d, 3, N_MELS)
    bias = m.f("enc.conv1.b")
    xp = np.zeros((B, N_MELS, N_FRAMES + 2))
    xp[:, :, 1: N_FRAMES + 1] = mel
    if defect == "no_left_pad":
        xp[:, :, 0] = mel[:, :, 0]
    taps = (2, 1, 0) if defect == "taps_reversed" else (0, 1, 2)
    pre = np.broadcast_to(bias, (B, N_FRAMES, d)).copy()
    S = np.broadcast_to(np.abs(bias), (B, N_FRAMES, d)).copy()
    for k in range(3):
        a = xp[:, :, k: k + N_FRAMES].transpose(0, 2, 1)
        wk = w[:, taps[k], :]
        pre += a @ wk.T
        S += np.abs(a) @ np.abs(wk).T
    return pre, S


def conv1_tol(pre, S, ref):
    """Bound on |fp16(gelu_erf(acc + bias)) - float64| for conv1_gelu_kernel: acc is 240 sequential fp32 FMAs, each
    rounding once a partial sum bounded by S, and the bias add one more rounding: within 241 2^-24 S.  GELU's slope is at
    most 1.13.  fp32 gelu_erf = 0.5 x (1 + erff(x 0.7071...)) adds erff's 2 ulp of 1 times |x| / 2 (2^-23 |x|), the
    rounded argument through erf's slope (0.8 2^-24 x^2) and three roundings of products and sums (3 2^-24 |x|).  The fp16
    store adds half an ulp: 2^-11 |ref| + 2^-25."""
    a = np.abs(pre)
    err = 1.13 * 241 * U * S + 2.0 ** -23 * a + 3 * U * a + 0.8 * U * a * a
    return (1 + 2.0 ** -11) * err + 2.0 ** -11 * np.abs(ref) + 2.0 ** -25


def h1_layout(frames16):
    """conv1 output frames [B, 3000, d] -> the engine's h1 rows [B * 3072 + 8, d] (zero rows 0 and 3001..3071 of each
    window and the tail)"""
    B, _, d = frames16.shape
    h1 = np.zeros((B * H1_ROWS + 8, d), np.float16)
    for b in range(B):
        h1[b * H1_ROWS + 1: b * H1_ROWS + 1 + N_FRAMES] = frames16[b]
    return h1


def conv2(m, h1, B, rows, defect=None):
    """-> (acc, r, ref) for rows [B, n] (t < 1500) of conv2 + pos over the engine's h1 rows: acc = A W2^T + b2 with A
    row t = h1 rows 2t, 2t + 1, 2t + 2 of its window, r the root-sum-square of the products, ref = gelu(acc) + pos[t]"""
    d = m.d
    w2 = m.f("enc.conv2.w")
    pos = m.f("enc.pos")
    if defect == "pos_shift":
        pos = np.concatenate([pos[1:], pos[-1:]])
    rows = np.asarray(rows)
    A = np.empty(rows.shape + (3 * d,))
    for b in range(B):
        base = b * H1_ROWS + 2 * rows[b]
        A[b] = np.concatenate([h1[base + k] for k in range(3)], axis=-1).astype(np.float64)
    acc = A @ w2.T + m.f("enc.conv2.b")
    r = np.sqrt((A * A) @ (w2 * w2).T)
    return acc, r, gelu(acc) + pos[rows]


def stem_padding(m, B, defect=None):
    """x rows 1500..1535 of each window [B, 36, d]: exactly 0 (defect "pos_padding": pos[t - 1500] added)"""
    out = np.zeros((B, T_PAD - T_ENC, m.d))
    if defect == "pos_padding":
        out += m.f("enc.pos")[: T_PAD - T_ENC]
    return out


def stem(m, mel):
    """the whole stem in float64 with h1 rounded to fp16: x [B, 1536, d]"""
    B = mel.shape[0]
    pre, _ = conv1(m, mel)
    h1 = h1_layout(gelu(pre).astype(np.float16))
    x = np.zeros((B, T_PAD, m.d))
    _, _, x[:, :T_ENC] = conv2(m, h1, B, np.tile(np.arange(T_ENC), (B, 1)))
    return x


# ------------------------------------------------------------------------------------------------ layer stages
def layer_norm(x, g, b, one_pass=False):
    x = np.asarray(x, np.float64)
    if one_pass:  # (defect) fp32 E[x^2] - mean^2
        x32 = x.astype(np.float32)
        n = np.float32(x.shape[-1])
        mean = x32.sum(-1, keepdims=True, dtype=np.float32) / n
        var = np.maximum((x32 * x32).sum(-1, keepdims=True, dtype=np.float32) / n - mean * mean, 0)
        return (x - mean.astype(np.float64)) / np.sqrt(var.astype(np.float64) + 1e-5) * g + b
    mean = x.mean(-1, keepdims=True)
    c = x - mean
    return c / np.sqrt((c * c).mean(-1, keepdims=True) + 1e-5) * g + b


def linear(a, w, bias):
    """-> (a w^T + bias, root-sum-square of the products) of the float64 rows a [..., K]"""
    a = np.asarray(a, np.float64)
    return a @ w.T + bias, np.sqrt((a * a) @ (w * w).T)


def gather(a, rows):
    """rows [B, n] of each window of a [B, 1536, ...]"""
    return np.take_along_axis(np.asarray(a), np.asarray(rows)[:, :, None], axis=1)


def qkv_with_v(qkv, vt):
    """qkv [B, 1536, 3d] with its V columns taken from the transposed Vt layout [B, H, 64, 1536] (attn_v_mn_major 0:
    the epilogue writes V only there)"""
    B, _, three_d = qkv.shape
    d = three_d // 3
    out = np.array(qkv)
    out[:, :, 2 * d:] = np.asarray(vt).transpose(0, 3, 1, 2).reshape(B, T_PAD, d)
    return out


def attention(qkv, H, rows, scale=0.125, n_keys=T_ENC, window_shift=0):
    """float64 softmax(q k^T scale over keys < n_keys) v of the fp16 qkv [B, 1536, 3d] for query rows [B, n] ->
    (ctx [B, n, d], the largest probability of every (row, head) [B, n, H])"""
    B, _, three_d = qkv.shape
    d = three_d // 3
    rows = np.asarray(rows)
    out = np.empty(rows.shape + (d,))
    pmax = np.empty(rows.shape + (H,))
    for b in range(B):
        kb = (b + window_shift) % B
        q = qkv[b, rows[b]].astype(np.float64)
        kv = qkv[kb, :n_keys].astype(np.float64)
        for h in range(H):
            c = slice(64 * h, 64 * h + 64)
            s = q[:, c] @ kv[:, d + 64 * h: d + 64 * h + 64].T * scale
            p = np.exp(s - s.max(axis=1, keepdims=True))
            out[b, :, c] = p @ kv[:, 2 * d + 64 * h: 2 * d + 64 * h + 64] / p.sum(axis=1, keepdims=True)
            pmax[b, :, h] = p.max(axis=1) / p.sum(axis=1)
    return out, pmax


def layer(m, i, x, rows, defect=None, attn_kw=None):
    """the whole layer from the residual x [B, 1536, d] in float64 with the chain's fp16 stores -> x_out at rows [B, n]
    (every row's K and V is formed; the query-side stages run on `rows` only)"""
    p = f"enc.{i}."
    d = m.d
    one = defect == "ln_one_pass"
    xn = r16(layer_norm(x, m.f(p + "ln1.g"), m.f(p + "ln1.b"), one))
    wqkv, bqkv = m.f(p + "qkv.w"), m.f(p + "qkv.b")
    qkv = np.empty(x.shape[:2] + (3 * d,))
    qkv[..., d:] = r16(xn @ wqkv[d:].T + bqkv[d:])
    xr = gather(xn, rows)
    q = r16(xr @ wqkv[:d].T + bqkv[:d])
    for b in range(x.shape[0]):
        qkv[b, rows[b], :d] = q[b]
    ctx, _ = attention(qkv, m.H, rows, **(attn_kw or {}))
    ctx = r16(ctx)
    y = gather(x, rows) + ctx @ m.f(p + "o.w").T + (0 if defect == "o_bias" else m.f(p + "o.b"))
    xn2 = r16(layer_norm(y, m.f(p + "ln2.g"), m.f(p + "ln2.b"), one))
    act = gelu_tanh if defect == "gelu_tanh" else gelu
    hh = r16(act(xn2 @ m.f(p + "fc1.w").T + m.f(p + "fc1.b")))
    return y + hh @ m.f(p + "fc2.w").T + m.f(p + "fc2.b")


def encoder(m, mel, rows, n_layers=None):
    """stem, every layer (the last one on `rows` only, the others on all rows) and ln_post, fp16 output rows [B, n, d]"""
    nl = m.L if n_layers is None else n_layers
    x = stem(m, mel)
    B = x.shape[0]
    every = np.tile(np.arange(T_PAD), (B, 1))
    for i in range(nl):
        x = layer(m, i, x, rows if i == nl - 1 else every)
    if nl == 0:
        x = gather(x, rows)
    return r16(layer_norm(x, m.f("enc.ln_post.g"), m.f("enc.ln_post.b")))


# ------------------------------------------------------------------------------------------------ tolerance
def row_ratio(got, ref, rtol):
    """worst |got - ref| / (rtol x the rms of the reference row) over rows [..., d] (inf where NaN)"""
    ref = np.asarray(ref, np.float64)
    tol = rtol * np.sqrt(np.mean(ref * ref, axis=-1, keepdims=True))
    with np.errstate(invalid="ignore"):
        q = np.abs(np.asarray(got, np.float64) - ref) / tol
    return float(np.max(np.where(np.isnan(q), np.inf, q)))
