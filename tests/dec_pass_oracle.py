"""float64 reference of ONE persistent decoder pass (csrc/decoder_mega.cu), rounding where the pass rounds.

impl 1 is the warp-MMA pass (dec_pass_mma_kernel), impl 0 the SIMT pass (dec_pass_kernel).  Everything is computed in
float64; the only roundings applied are the storage roundings of the pass being checked (decoder_mega.cu line numbers):

  both passes   K / V appended to the self-attention cache as fp16 (:487, :1464); the cross K/V is fp16 input
  warp-MMA      LayerNorm-GEMV input fp16(x * g_next) (publish_resid :1063, embedding :1822); queries fp16(q / 8)
                (:1459, :1609); P rounded to fp16 for P.V while the normaliser sums the unrounded P, relative to the running
                maximum of the warp's 32-key blocks (self :1214-1234, cross :1672-1691); attention output and fc1's
                GELU output as fp16 exchange images (:114, :1454)

The LayerNorm is folded in both passes: rstd * (W . a - mean * s2) + biasf with s2 = sum_k g_k W_nk and biasf = bias +
sum_k b_k W_nk (ln_fold_kernel), a = x * g (SIMT, fp32) or fp16(x * g) (warp-MMA).  The reference takes the row
statistics exactly from its own residual (option one_pass: fp32 E[x^2] - mean^2, the kernels' formula).  With
mirror=False the warp-MMA roundings are not applied: the plain model, identical to the SIMT pass's reference.

Tolerances (`tol`) are per pass, a fraction of the rms of each row (residual row, logit row, written K/V cell), plus
one fp16 step of the element for the K/V cells the pass stores (a value within fp32 noise of a rounding midpoint may
land on either side):
  SIMT       RTOL_SIMT = 2e-3.  fp32 arithmetic alone moves a row by ~1e-6 of its rms; what remains is the fp16 K/V the
             pass itself stores -- a one-step flip of an own-position key or value (2^-10 relative) reaches the residual
             through that key's attention weight.  Measured worst on an H100: 0.35 of the tolerance (logits), 0.26
             (residual).  The warp-MMA roundings move rows by ~1e-2 of their rms, several times this tolerance: the SIMT
             comparator tells the passes apart (test_simt_comparator_tells_the_passes_apart).
  warp-MMA   RTOL_MMA = 4e-2 against the rounding-aware reference, RTOL_PLAIN = 6e-2 against the plain model.  With
             attention this peaked (scores of tens at the dominating keys) a flip of one fp16 rounding moves the
             weights by more than the rounding itself, so the mirrored reference is not closer to the kernel than the
             plain model: measured worst 0.52 of RTOL_MMA (2.1e-2 of the rms, logits, d = 1280) and 0.40 of RTOL_PLAIN
             (2.4e-2, d = 128).  Both are far below what any injected defect costs (comparator tests).
"""
import numpy as np
from scipy.special import erf

T_ENC, T_PAD, T_MAX, SLOTS, GRID = 1500, 1536, 448, 8, 132


# ------------------------------------------------------------------------------------------------ geometry (mirrors)
def cross_geom(n_utt, H, grid=GRID):
    """decoder_mega.cu cross_geom: S key splits per (utterance, head), KS keys per split (whole 32-key blocks)."""
    s = min(max(grid // (n_utt * H), -(-T_ENC // 288)), 16)
    ks = (-(-T_ENC // s) + 31) // 32 * 32
    return s, ks


def empty_splits(n_utt, H, grid=GRID):
    """splits of a head that hold no key < 1500"""
    s, ks = cross_geom(n_utt, H, grid)
    return [j for j in range(s) if j * ks >= T_ENC]


def cta_cols(N, b, impl, grid=GRID):
    """columns [lo, hi) CTA b owns in a GEMV phase: warp-MMA mma_geom (N / grid each, the first N % grid one more);
    SIMT cta_cols (ceil(N / grid) each)"""
    if impl == 1:
        base, rem = divmod(N, grid)
        lo = b * base + min(b, rem)
        return lo, lo + base + (1 if b < rem else 0)
    per = -(-N // grid)
    lo = min(N, b * per)
    return lo, min(N, lo + per)


# ------------------------------------------------------------------------------------------------ fp16 rounding
def r16(v):
    return np.asarray(v, np.float64).astype(np.float16).astype(np.float64)


# ------------------------------------------------------------------------------------------------ model
class Model:
    """float64 weights of the engine tensors (weights.pack_state_dict names)"""

    def __init__(self, tensors, dims):
        self.d, self.H, self.L, self.V = dims.d_model, dims.n_heads, dims.n_dec_layers, dims.n_vocab
        f = lambda n: np.asarray(tensors[n], np.float64)  # noqa: E731
        self.tok = np.asarray(tensors["dec.tok_emb"], np.float16)
        self.pos = f("dec.pos")
        self.layers = []
        for i in range(self.L):
            p = f"dec.{i}."
            ly = {k: f(p + k) for k in ("ln1.g", "ln1.b", "qkv.w", "qkv.b", "o.w", "o.b", "ln2.g", "ln2.b", "cq.w", "cq.b",
                                        "co.w", "co.b", "ln3.g", "ln3.b", "fc1.w", "fc1.b", "fc2.w", "fc2.b")}
            self.layers.append(ly)
        self.lng, self.lnb = f("dec.ln.g"), f("dec.ln.b")
        self.E = self.tok[: self.V].astype(np.float64)


def ln_fold(impl, x, g, b, W, bias, mirror, drop_share=None, one_pass=False):
    """LN(x) W^T + bias as the passes fold it (consume_gemv :455-463, consume_gemv_mma :1433-1437, consume_cross_fused
    :1606-1608).  drop_share (a defect): CTA drop_share's columns left out of the row statistics; one_pass: the
    statistics as the kernels form them, fp32 sum and sum of squares, var = E[x^2] - mean^2."""
    K = x.shape[1]
    a = x * g
    if impl == 1 and mirror:
        a = r16(a)
    xs = x
    if drop_share is not None:
        lo, hi = cta_cols(K, drop_share, impl)
        xs = x.copy()
        xs[:, lo:hi] = 0.0
    if one_pass:
        x32 = xs.astype(np.float32)
        mean = (x32.sum(1, keepdims=True, dtype=np.float32) / np.float32(K)).astype(np.float64)
        e2 = ((x32 * x32).sum(1, keepdims=True, dtype=np.float32) / np.float32(K)).astype(np.float32)
        var = np.maximum(e2 - np.float32(mean) * np.float32(mean), 0).astype(np.float64)
    else:
        mean = xs.sum(1, keepdims=True) / K
        var = ((xs - mean) ** 2).sum(1, keepdims=True) / K
    rstd = 1 / np.sqrt(var + 1e-5)
    s2 = W @ g
    bf = W @ b + (0 if bias is None else bias)
    return rstd * (a @ W.T - mean * s2) + bf


def gelu(v):
    return 0.5 * v * (1 + erf(v / np.sqrt(2)))


# ------------------------------------------------------------------------------------------------ attention
def attend(s, V, blocks, p16, phantom=0):
    """One (row, head): o = sum_t w16_t V_t / sum_t w_t with w_t = exp(s_t - M), w16_t = fp16(exp(s_t - m_t)) exp(m_t - M)
    (p16: P rounded relative to m_t, the running maximum of the key's 32-key walk; `blocks` = (walk id, block order) of
    every key, the walk's running maximum is taken over its blocks up to this one).  phantom (a defect): empty key
    splits merged as keys of the row's maximum score and value 0."""
    M = s.max()
    w = np.exp(s - M)
    if p16:
        walk, order = blocks
        bm = np.full((walk.max() + 1, order.max() + 1), -np.inf)
        np.maximum.at(bm, (walk, order), s)
        mrun = np.maximum.accumulate(bm, axis=1)[walk, order]
        w16 = r16(np.exp(s - mrun)) * np.exp(mrun - M)
    else:
        w16 = w
    return w16 @ V / (w.sum() + phantom)


def self_keys(case, r, pos, defect):
    """(slots, positions) row r attends to: t <= pos through indir (own slot at t = pos; prefill: own slot always)"""
    if case["pf_len"] > 0:
        last = case["pf_len"] - 1 if defect == "prefill_later" else pos
        t = np.arange(last + 1)
        return np.full(t.size, case["slot"][r]), t
    t = np.arange(pos if defect == "keys_lt_pos" else pos + 1)
    sl = case["indir"][r, t].astype(np.int64)
    if defect == "own_slot":
        sl[:] = case["slot"][r]
    sl[t == pos] = case["slot"][r]
    return sl, t


# ------------------------------------------------------------------------------------------------ the pass
def run_pass(m, case, impl, *, mirror=True, defect=None, one_pass=False, with_logits=True):
    """-> dict(x [R, d], logits [R, V], kc / vc [L, 8, 448, d] (float64, NaN kept), written [(layer, slot, pos)]).
    case: tokens [R], pos [R], slot [R], pf_len, n_utt, beam (rows per utterance in the cross-attention: pf_len in a
    prefill), indir [R, 448] (the current ping-pong buffer), kc / vc float16 [L, 8, 448, d], ckv float16 [L, 2, n_utt, H,
    1536, 64].  defect (comparator tests): "drop_cols" (one CTA's column slice of layer 0's fc2 never added),
    "drop_share" (one CTA's LayerNorm share left out of every statistic), "keys_lt_pos", "own_slot", "prefill_later",
    "unmask_padding", "empty_nan", "empty_weight"."""
    d, H = m.d, m.H
    p16 = impl == 1 and mirror
    R = len(case["tokens"])
    tok, pos, slot = case["tokens"], case["pos"], case["slot"]
    n_utt, rpu = case["n_utt"], case["beam"]
    x = m.tok[tok].astype(np.float64) + m.pos[pos]
    kc = case["kc"].astype(np.float64)
    vc = case["vc"].astype(np.float64)
    S, KS = cross_geom(n_utt, H)
    n_keys = T_PAD if defect == "unmask_padding" else T_ENC
    n_empty = len(empty_splits(n_utt, H))
    # the cross-attention walk of key t: split t // KS, warp (t % KS // 32) % 7, block order (t % KS // 32) // 7
    tk = np.arange(n_keys)
    loc_blk = (tk % KS) // 32
    cblocks = ((tk // KS) * 7 + loc_blk % 7, loc_blk // 7)
    lnf = lambda x_, g, b, W, bias: ln_fold(impl, x_, g, b, W, bias, mirror,  # noqa: E731
                                           7 if defect == "drop_share" else None, one_pass)
    for li, ly in enumerate(m.layers):
        # ---- LN1 + QKV: q, and K / V appended at (slot, pos) of every row
        v = lnf(x, ly["ln1.g"], ly["ln1.b"], ly["qkv.w"], ly["qkv.b"])
        q = r16(v[:, :d] * 0.125) if p16 else v[:, :d] * 0.125
        for r in range(R):
            kc[li, slot[r], pos[r]] = r16(v[r, d:2 * d])
            vc[li, slot[r], pos[r]] = r16(v[r, 2 * d:])
        # ---- self-attention
        ctx = np.zeros((R, d))
        for r in range(R):
            sl, t = self_keys(case, r, pos[r], defect)
            if t.size == 0:
                ctx[r] = np.nan
                continue
            blocks = (np.zeros(t.size, np.int64), t // 32)
            for h in range(H):
                c = slice(64 * h, 64 * h + 64)
                ctx[r, c] = attend(kc[li, sl, t, c] @ q[r, c], vc[li, sl, t, c], blocks, p16)
        if p16:
            ctx = r16(ctx)
        x = x + ctx @ ly["o.w"].T + ly["o.b"]
        # ---- LN2 + cross-query + cross-attention over the fp16 cross K / V
        q = lnf(x, ly["ln2.g"], ly["ln2.b"], ly["cq.w"], ly["cq.b"]) * 0.125
        if p16:
            q = r16(q)
        ctx = np.zeros((R, d))
        ph = n_empty if defect == "empty_weight" else 0
        for u in range(n_utt):
            for h in range(H):
                c = slice(64 * h, 64 * h + 64)
                Kh = case["ckv"][li, 0, u, h, :n_keys].astype(np.float64)
                Vh = case["ckv"][li, 1, u, h, :n_keys].astype(np.float64)
                for k in range(rpu):
                    r = u * rpu + k
                    ctx[r, c] = attend(Kh @ q[r, c], Vh, cblocks, p16, ph)
                    if defect == "empty_nan" and n_empty:
                        ctx[r, c] = np.nan
        if p16:
            ctx = r16(ctx)
        x = x + ctx @ ly["co.w"].T + ly["co.b"]
        # ---- LN3 + fc1 + GELU, fc2
        hg = gelu(lnf(x, ly["ln3.g"], ly["ln3.b"], ly["fc1.w"], ly["fc1.b"]))
        if p16:
            hg = r16(hg)
        y = hg @ ly["fc2.w"].T + ly["fc2.b"]
        if defect == "drop_cols" and li == 0:
            lo, hi = cta_cols(d, 7, impl)
            y[:, lo:hi] = 0.0
        x = x + y
    out = dict(x=x, kc=kc, vc=vc, written=[(li, int(slot[r]), int(pos[r])) for li in range(m.L) for r in range(R)])
    if with_logits:
        out["logits"] = lnf(x, m.lng, m.lnb, m.E, None)
    return out


RTOL_SIMT, RTOL_MMA, RTOL_PLAIN = 2e-3, 4e-2, 6e-2  # of a row's rms (see the module docstring)


def step16(v):
    """fp16 spacing at |v| (the larger one at a power of two; 2^-24 in the subnormal range)"""
    a = np.abs(np.asarray(v, np.float64))
    with np.errstate(divide="ignore"):
        e = np.floor(np.log2(np.maximum(a, 2.0 ** -30)))
    return np.maximum(2.0 ** (e - 10), 2.0 ** -24)


def tol(ref_rows, rtol, stored16=False):
    """tolerance per element: rtol times the rms of its row, plus one fp16 step of the element for values the pass
    stores as fp16 (the written K/V cells)"""
    r = np.asarray(ref_rows, np.float64)
    t = rtol * np.sqrt(np.mean(r * r, axis=-1, keepdims=True))
    return t + step16(r) if stored16 else t


def ratios(got, ref, rtol):
    """worst |got - ref| / tol of the residual, the logits and the written K/V cells (inf where NaN): got is the kernel's
    output (x [>= R, d], logits [>= R, >= V], kc / vc) or another reference"""
    R = ref["x"].shape[0]

    def worst(g, r, t):
        with np.errstate(invalid="ignore"):
            q = np.abs(np.asarray(g, np.float64) - r) / t
        return float(np.max(np.where(np.isnan(q), np.inf, q))) if q.size else 0.0

    out = {"x": worst(got["x"][:R], ref["x"], tol(ref["x"], rtol))}
    if "logits" in ref and "logits" in got:
        V = ref["logits"].shape[1]
        out["logits"] = worst(got["logits"][:R, :V], ref["logits"], tol(ref["logits"], rtol))
    cells = tuple(np.asarray(ref["written"]).T)
    out["kv"] = max(worst(got[f][cells], ref[f][cells], tol(ref[f][cells], rtol, True)) for f in ("kc", "vc"))
    return out


def rejects(ref, bad, rtol):
    """True when `bad` (a defective reference) leaves the tolerance of `ref` somewhere (NaN counts as outside)"""
    return max(ratios(bad, ref, rtol).values()) > 1
