"""float64 reference of ONE batched decoder pass (csrc/decoder_batch.cu batch_pass_run), rounding where the pass rounds.

The batched pass is a chain of wgmma GEMMs and small kernels; unlike the persistent pass it does not fold the LayerNorm.
The only roundings applied (mirror=True) are the pass's own storage roundings:

  LayerNorm      xn = fp16(LN(x) g + b) before every GEMM, statistics exact (row_layernorm_store :31 takes the mean, then
                 the centred sum of squares, in fp32: no cancellation).  Embedding x = fp16 tok_emb + fp32 pos.
  QKV epilogue   q fp32, unscaled; K / V stored fp16 at (row_slot, row_pos) (gemm_tc.cu EPI_DEC_QKV).
  self-attn      fp32 q against the fp16 cache, scores x 0.125, exact softmax, ctx fp16 (bd_self_attn_kernel :133).  A
                 prefill row reads its own slot at every t <= pos; a step row reads slot indir[t] for t < pos, its own at pos.
  o / co / fc2   fp32 split-K partials added to bias + residual (exact sums here).
  cross-query    fp32 with bias.
  cross-attn     "tc" (bd_cross_attn_tc_kernel): q16 = fp16(q / 8), P16 = fp16(exp(s - M)) with M the exact row maximum
                 over the 1500 keys, normaliser = sum of P16; "px" (bd_prefill_cross_attn_kernel, wide passes and > 8
                 rows per window): the same but P16 relative to the running maximum over the 128-key tiles seen so far,
                 rescaled to the final maximum; "simt" (bd_cross_attn_kernel<NB>): exact q / 8, exact softmax.  ctx fp16
                 over keys < 1500.
  fc1            fp16(gelu_erf(.)).
  logits         fp16 xn (final LayerNorm) . fp16 tok_emb^T in fp32: no bias.

With mirror=False none of these is applied but the fp16 K / V the cache holds: the plain float64 model.

Tolerances (dec_pass_oracle.tol): a fraction of the rms of each row (residual row, logit row, written K / V cell) plus one
fp16 step of the element for the K / V the pass stores.
  RTOL_BATCH = 4e-2 against the rounding-aware reference.  The pass and the reference differ by fp32 accumulation order
      and __expf against exp (~1e-6 of a row) and by which side of an fp16 midpoint a stored value lands (q16, P16, xn,
      ctx, the GELU output and K / V): a flipped fp16 rounding of one dominating attention key or value moves a row by up
      to its attention weight times 2^-11 of the value, and the row's later LayerNorms amplify it by the gain of two
      layers.  Measured worst on an H100: 0.79 of the bound (residual, d = 128), 0.68 (logits, d = 384), 0.31 (K / V).
  RTOL_PLAIN = 1.2e-1 against the plain model: the fp16 roundings themselves move rows by ~1e-2 of their rms and, with
      attention this peaked (scores of a few units, QK_GAIN), by more on the rare row whose dominating weights shift:
      measured 8.6e-2 of the rms on one residual row of a 1024-row step at d = 128 (0.72 of this bound), where the
      persistent pass's 6e-2 would have failed.
Both are far below what any injected defect costs (tests/test_gpu_batch_pass.py, tests without the gpu mark).
"""
import numpy as np

from tests import dec_pass_oracle as O
from tests.dec_pass_oracle import T_ENC, T_PAD, gelu, r16

RTOL_BATCH, RTOL_PLAIN = 4e-2, 1.2e-1  # of a row's rms (see the module docstring)
CROSS_IMPLS = ("tc", "simt", "px")


# ------------------------------------------------------------------------------------------------ geometry (mirrors)
def dec_plan(M, N, K, allow_split):
    """(BN, K splits) engine.cu plan_dec_gemm picks for a decoder GEMM planned at M capacity rows"""
    mt = M // 128
    bn = 256
    while bn > 64 and (N % bn != 0 or mt * (N // bn) < 120):
        bn //= 2
    splits = 1
    if allow_split:
        kb = K // 64
        while mt * (N // bn) * splits < 120 and splits < 8 and kb % (splits * 2) == 0 and kb // (splits * 2) >= 4:
            splits *= 2
    return bn, splits


def layer_plans(M, d):
    """plan_batch_layers' GEMMs at capacity M: name -> (BN, K splits)"""
    return {"qkv": dec_plan(M, 3 * d, d, False), "o": dec_plan(M, d, d, True), "cq": dec_plan(M, d, d, False),
            "co": dec_plan(M, d, d, True), "fc1": dec_plan(M, 4 * d, d, False), "fc2": dec_plan(M, d, 4 * d, True)}


def cross_nb(rows_per_utt):
    """the bd_cross_attn_kernel<NB> instance the SIMT cross-attention launches"""
    return 1 if rows_per_utt == 1 else 5 if rows_per_utt <= 5 else 8


def unswizzle(ckv):
    """the persistent warp-MMA pass's chunk-swizzled cross K/V (16-byte chunk c of key t at c ^ (t & 7)) -> linear (the
    permutation is its own inverse)"""
    x = ckv.view(np.uint16).reshape(ckv.shape[:-1] + (8, 8))
    idx = np.arange(8)[None, :] ^ (np.arange(T_PAD)[:, None] & 7)
    idx = np.broadcast_to(idx[..., None], x.shape)
    return np.ascontiguousarray(np.take_along_axis(x, idx, axis=-2).reshape(ckv.shape)).view(np.float16)


# ------------------------------------------------------------------------------------------------ pieces
def layernorm(x, g, b, mirror):
    mean = x.mean(1, keepdims=True)
    var = ((x - mean) ** 2).mean(1, keepdims=True)
    y = (x - mean) / np.sqrt(var + 1e-5) * g + b
    return r16(y) if mirror else y


def cross_attend(q, K, V, impl, mirror):
    """q [rows, H, 64] (unscaled), K / V [H, keys, 64] -> ctx [rows, H, 64]"""
    if impl == "simt" or not mirror:
        s = np.einsum("rhd,htd->rht", q * 0.125, K)
        w = np.exp(s - s.max(-1, keepdims=True))
        return np.einsum("rht,htd->rhd", w, V) / w.sum(-1)[..., None]
    s = np.einsum("rhd,htd->rht", r16(q * 0.125), K)
    M = s.max(-1, keepdims=True)
    if impl == "tc":
        p = r16(np.exp(s - M))
        return np.einsum("rht,htd->rhd", p, V) / p.sum(-1)[..., None]
    # px: P16 relative to the running maximum over the 128-key tiles, rescaled to the final one
    n = s.shape[-1]
    nt = -(-n // 128)
    tile_max = np.full(s.shape[:-1] + (nt,), -np.inf)
    for j in range(nt):
        tile_max[..., j] = s[..., 128 * j: 128 * j + 128].max(-1)
    run = np.maximum.accumulate(tile_max, axis=-1)
    mrun = np.repeat(run, 128, axis=-1)[..., :n]
    p = r16(np.exp(s - mrun)) * np.exp(mrun - M)
    return np.einsum("rht,htd->rhd", p, V) / p.sum(-1)[..., None]


# ------------------------------------------------------------------------------------------------ the pass
def run_batch_pass(m, case, *, mirror=True, defect=None, logit_rows=()):
    """-> dict(x [R, d], logits [len(logit_rows), V], kw / vw [L, R, d] the K / V row r writes in each layer (wrow
    [slots, t_cap] maps a cell to its row, kc_in / vc_in the caller's caches, not copied), written [(layer, slot, pos)]
    every cell the pass writes, checked [(layer, slot, pos)] the cells whose values are defined (rows of live windows),
    live [R] bool).
    case: tokens [R], pos [R], slot [R], prefill (bool), n_utt, rpu (rows per window), indir [R, 448] (step: the current
    ping-pong buffer), done [n_utt] bool or None, kc / vc float16 [L, slots, t_cap, d], ckv float16 [L, 2, n_utt, H, 1536,
    64] in the layout the pass reads, ckv_sw (chunk-swizzled), cross ("tc" / "simt" / "px"), splits (fc2's K splits),
    beam (prefill: slot stride), chunk0 (first position of the last chunk, for "chunk_blind").
    defect (comparator tests): "drop_slab" (layer 0's last fc2 split-K slab never added), "next_gain" (the LayerNorm
    after layer 0 with layer 0's own ln1 gain), "chunk_blind" (rows at positions >= chunk0 cannot see the K/V of earlier
    positions), "slot_u" (prefill rows in slot u instead of u * beam), "keys_lt_pos", "unmask_padding",
    "swizzle_ignored", "neighbour_ckv" (window u reads window u + 1's cross K/V), "dead_not_skipped" (the cross-attention
    walks the first n_live windows whatever their state: live windows past them get no output)."""
    d, H, L = m.d, m.H, m.L
    R = len(case["tokens"])
    tok, pos = np.asarray(case["tokens"]), np.asarray(case["pos"])
    slot = np.asarray(case["slot"]).copy()
    n_utt, rpu = case["n_utt"], case["rpu"]
    win = np.arange(R) // rpu
    if defect == "slot_u" and case["prefill"]:
        slot = win.copy()
    done = np.zeros(n_utt, bool) if case.get("done") is None else np.asarray(case["done"], bool)
    live = ~done[win]
    ckv = case["ckv"]
    if case.get("ckv_sw") and defect != "swizzle_ignored":
        ckv = unswizzle(ckv)
    n_keys = T_PAD if defect == "unmask_padding" else T_ENC
    impl = case["cross"]
    x = m.tok[tok].astype(np.float64) + m.pos[pos]
    # the caches stay the caller's fp16 arrays (read only): what this pass writes lives in kw / vw, row r's K / V of
    # layer li at kw[li, r], found through wrow[slot, pos] (-1: not written by this pass)
    kc_in, vc_in = case["kc"], case["vc"]
    kw, vw = np.zeros((L, R, d)), np.zeros((L, R, d))
    wrow = np.full(kc_in.shape[1:3], -1, np.int64)
    wrow[slot, pos] = np.arange(R)
    ln = lambda v, g, b: layernorm(v, g, b, mirror)  # noqa: E731
    xn = ln(x, m.layers[0]["ln1.g"], m.layers[0]["ln1.b"])
    for li, ly in enumerate(m.layers):
        # ---- QKV: q fp32, K / V stored fp16 at (slot, pos) of every row
        v = xn @ ly["qkv.w"].T + ly["qkv.b"]
        q = v[:, :d]
        kw[li], vw[li] = r16(v[:, d:2 * d]), r16(v[:, 2 * d:])
        # ---- self-attention
        ctx = np.zeros((R, d))
        for r in range(R):
            if not live[r]:
                ctx[r] = np.nan
                continue
            p = int(pos[r])
            last = p if defect == "keys_lt_pos" else p + 1
            t = np.arange(last)
            if case["prefill"]:
                sl = np.full(t.size, slot[r])
                if defect == "chunk_blind" and p >= case["chunk0"]:
                    t = t[t >= case["chunk0"]]
                    sl = sl[: t.size]
            else:
                sl = case["indir"][r, t].astype(np.int64)
                sl[t == p] = slot[r]
            if t.size == 0:
                ctx[r] = np.nan
                continue
            Kt, Vt = kc_in[li, sl, t].astype(np.float64), vc_in[li, sl, t].astype(np.float64)
            own = wrow[sl, t]
            Kt[own >= 0], Vt[own >= 0] = kw[li, own[own >= 0]], vw[li, own[own >= 0]]
            Kt, Vt = Kt.reshape(t.size, H, 64), Vt.reshape(t.size, H, 64)
            s = np.einsum("thd,hd->ht", Kt, q[r].reshape(H, 64)) * 0.125
            w = np.exp(s - s.max(-1, keepdims=True))
            ctx[r] = (np.einsum("ht,thd->hd", w, Vt) / w.sum(-1)[:, None]).reshape(d)
        if mirror:
            ctx = r16(ctx)
        x = x + ctx @ ly["o.w"].T + ly["o.b"]
        xn = ln(x, ly["ln2.g"], ly["ln2.b"])
        # ---- cross-query, cross-attention over the window's fp16 cross K / V
        q = xn @ ly["cq.w"].T + ly["cq.b"]
        ctx = np.full((R, d), np.nan)
        live_w = [u for u in range(n_utt) if not done[u]]
        run_w = list(range(len(live_w))) if defect == "dead_not_skipped" else live_w
        for u in run_w:
            if done[u]:
                continue
            src = (u + 1) % n_utt if defect == "neighbour_ckv" else u
            K = ckv[li, 0, src, :, :n_keys].astype(np.float64)
            V = ckv[li, 1, src, :, :n_keys].astype(np.float64)
            rows = slice(u * rpu, u * rpu + rpu)
            ctx[rows] = cross_attend(q[rows].reshape(rpu, H, 64), K, V, impl, mirror).reshape(rpu, d)
        if mirror:
            ctx = r16(ctx)
        x = x + ctx @ ly["co.w"].T + ly["co.b"]
        xn = ln(x, ly["ln3.g"], ly["ln3.b"])
        # ---- MLP
        hg = gelu(xn @ ly["fc1.w"].T + ly["fc1.b"])
        if mirror:
            hg = r16(hg)
        if defect == "drop_slab" and li == 0:
            k = 4 * d // case["splits"]
            hg = hg.copy()
            hg[:, 4 * d - k:] = 0.0
        x = x + hg @ ly["fc2.w"].T + ly["fc2.b"]
        if li + 1 < L:
            g = ly["ln1.g"] if defect == "next_gain" and li == 0 else m.layers[li + 1]["ln1.g"]
            xn = ln(x, g, m.layers[li + 1]["ln1.b"])
        else:
            xn = ln(x, m.lng, m.lnb)
    written = [(li, int(slot[r]), int(pos[r])) for li in range(L) for r in range(R)]
    checked = [(li, int(slot[r]), int(pos[r])) for li in range(L) for r in range(R) if live[r]]
    out = dict(x=x, kw=kw, vw=vw, wrow=wrow, kc_in=kc_in, vc_in=vc_in, written=written, checked=checked, live=live)
    rows = np.asarray(logit_rows, np.int64)
    out["logits"] = xn[rows] @ m.E.T if rows.size else np.zeros((0, m.V))
    return out


def kv_at(out, f, cells):
    """K (f "kc") or V ("vc") at cells [(layer, slot, pos)] as float64 [n, d]: of the kernel's caches, or of a reference
    (what it wrote, else the cache it started from)"""
    li, sl, t = (np.asarray(v, np.int64) for v in zip(*cells))
    if "wrow" not in out:
        return np.asarray(out[f][li, sl, t], np.float64)
    val = out[f + "_in"][li, sl, t].astype(np.float64)
    r = out["wrow"][sl, t]
    val[r >= 0] = out["kw" if f == "kc" else "vw"][li[r >= 0], r[r >= 0]]
    return val


def ratios(got, ref, rtol, logit_rows=()):
    """worst |got - ref| / tol (dec_pass_oracle.ratios) over the rows of live windows, the logit rows `logit_rows`
    (a reference holds exactly those) and the K / V cells of live rows: got is the kernel's output (x [R, d], logits
    [R, >= V], kc / vc) or another reference"""
    live = ref["live"]
    lr = np.asarray(logit_rows, np.int64)
    keep = live[lr] if lr.size else np.zeros(0, bool)
    V = ref["logits"].shape[1]
    cells = ref["checked"]
    n = len(cells)
    g = dict(x=np.asarray(got["x"])[live])
    r = dict(x=ref["x"][live], written=[(i,) for i in range(max(n, 1))])
    for f in ("kc", "vc"):  # (compact [n, d] arrays: O.ratios indexes them by written = [(i,)])
        g[f] = kv_at(got, f, cells) if n else np.zeros((1, 1))
        r[f] = kv_at(ref, f, cells) if n else np.zeros((1, 1))
    if keep.any():
        lg = np.asarray(got["logits"])
        g["logits"] = lg[keep] if "live" in got else lg[lr[keep], :V]  # (another reference holds the logit rows only)
        r["logits"] = ref["logits"][keep]
    return O.ratios(g, r, rtol)


def rejects(ref, bad, rtol, logit_rows=()):
    """True when `bad` (a defective reference) leaves the tolerance of `ref` somewhere (NaN counts as outside)"""
    return max(ratios(bad, ref, rtol, logit_rows).values()) > 1
