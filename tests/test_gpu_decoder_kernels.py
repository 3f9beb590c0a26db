"""Kernel-level parity of the batched decoder pass's own kernels (csrc/decoder_batch.cu), each launched through the
launcher the pass itself uses (Handle.debug_dec_*) on crafted data and compared with a reference computed here:

  * cross-attention, wgmma and SIMT: float64 softmax(q/8 . K^T over keys < 1500) . V for every (utterance, head), at
    1..8 rows per utterance, 2..20 heads, fewer / as many / many more items than the 132 SMs (up to the configs[2]
    shape 64 x 20 and the 1024-utterance limit), with finished utterances interleaved, against cross_tol
  * self-attention over the beam-indirected cache: float64 over t <= pos with every unaddressed cache cell NaN, at
    positions 0 .. 447, against the same bound
  * residual + LayerNorm and embedding + LayerNorm: the fp32 residual stream bit for bit against numpy float32 in the
    kernel's summation order, xn against float64 LayerNorm within ln_tol

The tests without the gpu mark check the comparators themselves: each must reject a reference with a known defect."""
import numpy as np
import pytest

from tests.test_gpu_kernels import bits, note_ratio, sentinel
from willow_inference_server_b200 import _lib

T_PAD, T_ENC = 1536, 1500
NAN16 = np.uint16(0x7E00)
SENT16 = np.uint16(0x7E5A)
SENT32 = np.uint32(0x7FC0DEAD)
U23 = 2.0 ** -23
MAX_UTT = 1024  # BD_CROSS_MAX_UTT (csrc/decoder.cuh)


@pytest.fixture(scope="module")
def h():
    return _lib.Handle.frontend(0)


def within(got, ref, tol):
    """every element finite and within tol (NaN anywhere fails)"""
    return bool(np.all(np.abs(got.astype(np.float64) - ref) <= tol))


def ratio(got, ref, tol):
    return float(np.max(np.abs(got.astype(np.float64) - ref) / tol))


# ------------------------------------------------------------------------------------------------ softmax error bound
def softmax_tol(s, sabs, v, ref, *, score_ulps, p16, n_acc):
    """Bound on |kernel - float64| for attention rows o = sum_t p_t v_t / sum_t p_t, p_t = exp(s_t - max s).

    s [n, T] float64 scores of the attended keys, sabs [n, T] = sum_i |q_i k_ti| / 8, v [n or 1, T, 64], ref [n, 64].
    A relative error e_t on each weight moves o by sum_t p_t e_t (v_t - o) / sum_t p_t (1 + e_t), at most
    max|e| . dev / (1 - max|e|) with dev = sum_t p_t |v_t - o| / sum_t p_t.  The weight errors are
      * the fp32 score: each score within score_ulps 2^-23 sabs (products and partial sums rounded; the tensor core may
        truncate), which changes a weight relative to the maximum's by twice that;
      * the exponential: exp2f / __expf (2 ulp) of an argument whose fp32 rounding and log2(e) scaling cost 2^-23 |s|
        per evaluation; a generous 2^-22 (16 + 6 max|s|) covers the online rescales of the SIMT kernel too;
      * p16 (wgmma): P rounded to fp16 before the P.V product, 2^-11 relative, while the normaliser sums the same
        rounded P (the kernel documents this), so only the weights move; P below 2^-14 is subnormal in fp16 and may move
        by 2^-25 absolute instead.
    The fp32 accumulations of P.V and of the normaliser add n_acc 2^-23 sum_t p_t |v_t| / sum_t p_t, and the fp16
    output half an ulp: 2^-11 |ref| + 2^-25."""
    m = s.max(axis=1, keepdims=True)
    p = np.exp(s - m)
    l = p.sum(axis=1)
    dv = np.abs(v - ref[:, None, :])
    dev = np.einsum("nt,ntd->nd", p, dv) / l[:, None]
    eps = 2 * score_ulps * U23 * sabs.max(axis=1) + 2.0 ** -22 * (16 + 6 * np.abs(s).max(axis=1))
    if p16:
        eps = eps + 2.0 ** -11
    tol = (eps / (1 - eps))[:, None] * dev
    if p16:
        tol = tol + 2.0 ** -25 * np.einsum("nt,ntd->nd", (p < 2.0 ** -14).astype(np.float64), dv) / l[:, None]
    tol = tol + n_acc * U23 * np.einsum("nt,ntd->nd", p, np.abs(v)) / l[:, None]
    return tol + 2.0 ** -11 * np.abs(ref) + 2.0 ** -25


def softmax_ref(s, v):
    p = np.exp(s - s.max(axis=1, keepdims=True))
    return np.einsum("nt,ntd->nd", p, v) / p.sum(axis=1)[:, None]


# ------------------------------------------------------------------------------------------------ cross-attention
def cross_case(kind, n_utt, H, rpu, *, tier="exact", n_layers=2, layer=1, seed=0):
    """-> (q float32 [n_utt rpu, 64 H], ckv float16 [n_layers, 2, n_utt, H, 1536, 64]).  The other layers are NaN, so a
    read of the wrong layer poisons the result.  Scores have std ~3; every (utterance, head) item has its own V offset,
    so mix-ups cannot cancel; the padding keys 1500..1535 hold large, distinct V in every case.

    tier "exact": q = 8 x fp16 values, so q/8 is the same fp16 number in both kernels; "gauss": unrounded fp32 q."""
    rng = np.random.default_rng([seed, n_utt, H, rpu, ["late", "early", "uniform", "padding", "onehot", "rowpeak",
                                                       "gauss"].index(kind)])
    ckv = np.full((n_layers, 2, n_utt, H, T_PAD, 64), NAN16, np.uint16).view(np.float16)
    K = rng.standard_normal((n_utt, H, T_PAD, 64), dtype=np.float32) * np.float32(1.73)
    V = rng.standard_normal((n_utt, H, T_PAD, 64), dtype=np.float32)
    V += (0.01 * (np.arange(n_utt * H) % 97)).reshape(n_utt, H, 1, 1).astype(np.float32)
    V[:, :, T_ENC:] = 1000.0 + 7.0 * np.arange(T_PAD - T_ENC)[:, None] + np.arange(64)
    q = rng.standard_normal((n_utt, rpu, H, 64)) * 1.73
    if kind == "late":       # every row's maximum in the last, partially masked key tile 1408..1499
        q[..., 0], K[:, :, 1408:T_ENC, 0] = 16.0, 16.0
    elif kind == "early":    # maximum in the first tile
        q[..., 0], K[:, :, :128, 0] = 16.0, 20.0
    elif kind == "uniform":  # all scores 0: the mean of V over exactly 1500 keys
        q[:] = 0
    elif kind == "padding":  # the padding keys would take every row's whole weight: only the mask keeps them out
        q[..., 0], K[:, :, T_ENC:, 0] = 16.0, 60.0
        K[:, :, :T_ENC, 0] *= 0.1
    elif kind == "onehot":   # one key 40 above all others: P = exp(-40) rounds to 0, the peak's P to exactly 1.0
        q[..., 0], K[:, :, 777, 0] = 24.0, 16.0
        K[:, :, :T_ENC, 1:] *= 0.1
        K[:, :, np.r_[0:777, 778:T_ENC], 0] = 0.2
    elif kind == "rowpeak":  # row k of each utterance peaks at its own key, 173 k + 11: a row / column mix-up shows
        for k in range(rpu):
            q[:, k, :, k + 1] = 12.0
            K[:, :, 173 * k + 11, k + 1] = 16.0
    if tier == "exact":
        q = 8.0 * (q / 8.0).astype(np.float16).astype(np.float64)
    ckv[layer, 0], ckv[layer, 1] = K, V
    return np.ascontiguousarray(q.reshape(n_utt * rpu, H * 64), np.float32), ckv


def cross_ref(q, ckv, rpu, *, layer=1, impl=0, n_keys=T_ENC, scale=0.125, scale_head=None, swap_rows=False,
              utt_shift=0, items=None):
    """float64 reference and bound per (utterance, head): (ref, tol) [n_utt rpu, d], NaN rows for items not listed.
    impl 0 (wgmma) attends with fp16(q/8), impl 1 (SIMT) with the exact q/8.  Defects for the comparator tests:
    n_keys (mask), scale (all heads) / scale_head (that head only), swap_rows (rows 0 and 1 of every utterance), utt_shift
    (K/V of utterance u + shift)."""
    n_utt, H = ckv.shape[2], ckv.shape[3]
    ref = np.full(q.shape, np.nan)
    tol = np.full(q.shape, np.nan)
    items = [(u, hd) for u in range(n_utt) for hd in range(H)] if items is None else items
    for u, hd in items:
        uk = (u + utt_shift) % n_utt
        Kh = ckv[layer, 0, uk, hd, :n_keys].astype(np.float64)
        Vh = ckv[layer, 1, uk, hd, :n_keys].astype(np.float64)
        rows = np.arange(u * rpu, (u + 1) * rpu)
        cs = slice(hd * 64, hd * 64 + 64)
        sc = scale if scale_head is None or hd == scale_head else 0.125
        qs = q[rows, cs].astype(np.float64) * sc
        if impl == 0:
            qs = qs.astype(np.float16).astype(np.float64)
        if swap_rows and rpu > 1:
            qs[[0, 1]] = qs[[1, 0]]
        s = qs @ Kh.T
        o = softmax_ref(s, Vh[None])
        ref[rows, cs] = o
        tol[rows, cs] = softmax_tol(s, np.abs(qs) @ np.abs(Kh).T, Vh[None], o, score_ulps=8, p16=impl == 0, n_acc=128)
    return ref, tol


def done_mask(pattern, n_utt):
    d = np.zeros(n_utt, np.int32)
    if pattern == "every_other":
        d[1::2] = 1
    elif pattern == "all_but_last":
        d[:-1] = 1
    elif pattern == "first_last":
        d[[0, -1]] = 1
    return None if pattern == "none" else d


def run_cross(h, q, ckv, rpu, impl, done=None, layer=1):
    ctx = sentinel(q.shape, np.float16)
    return h.debug_dec_cross_attn(q, ckv, ctx, layer=layer, rows_per_utt=rpu, impl=impl, done=done)


def check_cross(h, tag, q, ckv, rpu, *, done=None, layer=1, exact_q=False):
    """Both kernels against their reference; rows of finished utterances keep the sentinel bit for bit; the kernels
    agree with each other within the sum of their bounds plus the gap between their references (none with exact_q,
    where fp16(q/8) = q/8 and one reference serves both); the wgmma kernel is bit-identical run to run."""
    n_utt, H = ckv.shape[2], ckv.shape[3]
    live = [u for u in range(n_utt) if done is None or not done[u]]
    items = [(u, hd) for u in live for hd in range(H)]
    rows = np.concatenate([np.arange(u * rpu, (u + 1) * rpu) for u in live])
    dead = np.setdiff1d(np.arange(n_utt * rpu), rows)
    outs, refs, tols = {}, {}, {}
    for impl in (0, 1):
        got = run_cross(h, q, ckv, rpu, impl, done, layer)
        ref, tol = cross_ref(q, ckv, rpu, layer=layer, impl=impl, items=items)
        note_ratio(f"decoder cross-attention impl {impl}", ratio(got[rows], ref[rows], tol[rows]))
        assert within(got[rows], ref[rows], tol[rows]), (tag, impl)
        assert np.all(bits(got[dead]) == SENT16), (tag, impl)
        outs[impl], refs[impl], tols[impl] = got, ref[rows], tol[rows]
    if exact_q:
        assert np.array_equal(refs[0], refs[1]), tag
    gap = np.abs(refs[0] - refs[1])
    assert within(outs[0][rows], outs[1][rows].astype(np.float64), tols[0] + tols[1] + gap), tag
    assert np.array_equal(bits(run_cross(h, q, ckv, rpu, 0, done, layer)), bits(outs[0])), tag


CROSS_KINDS = ["late", "early", "uniform", "padding", "onehot", "rowpeak"]


@pytest.mark.gpu
@pytest.mark.parametrize("tier", ["exact", "gauss"])
@pytest.mark.parametrize("kind", CROSS_KINDS)
def test_cross_attention_score_shapes(h, kind, tier):
    """24 utterances x 6 heads = 144 items (> 132 SMs: some CTAs take two), 5 rows per utterance, layer 1 of 2."""
    rpu = 5
    q, ckv = cross_case(kind, 24, 6, rpu, tier=tier)
    check_cross(h, (kind, tier), q, ckv, rpu, exact_q=tier == "exact")


# (rows per utterance, heads, utterances, finished pattern): items n_utt x H below, equal to and well above 132
CROSS_GEOMETRY = [
    (1, 2, 4, "none"),
    (2, 6, 22, "every_other"),
    (3, 20, 7, "first_last"),
    (5, 6, 22, "none"),
    (7, 2, 100, "all_but_last"),
    (8, 20, 13, "none"),
    (1, 20, 64, "every_other"),
    (5, 20, 64, "none"),  # configs[2]: 64 windows x beam 5 of large-v2, 1280 items (~10 per CTA)
]


@pytest.mark.gpu
@pytest.mark.parametrize("rpu,H,n_utt,done", CROSS_GEOMETRY)
def test_cross_attention_geometry(h, rpu, H, n_utt, done):
    q, ckv = cross_case("rowpeak" if rpu > 1 else "gauss", n_utt, H, rpu, tier="gauss")
    check_cross(h, (rpu, H, n_utt, done), q, ckv, rpu, done=done_mask(done, n_utt))


@pytest.mark.gpu
def test_cross_attention_utterance_limit(h):
    """1024 utterances (the largest row capacity at one row each) in one launch, both kernels; 1025 is refused before
    anything is launched."""
    q, ckv = cross_case("gauss", MAX_UTT, 1, 1, tier="gauss", n_layers=1, layer=0)
    done = np.zeros(MAX_UTT, np.int32)
    done[3::7] = 1
    check_cross(h, "limit", q, ckv, 1, done=done, layer=0)
    check_cross(h, "limit, no done", q, ckv, 1, layer=0)
    big = np.zeros((1, 2, MAX_UTT + 1, 1, T_PAD, 64), np.float16)
    for impl in (0, 1):
        with pytest.raises(ValueError, match="utterances"):
            run_cross(h, np.zeros((MAX_UTT + 1, 64), np.float32), big, 1, impl, layer=0)


@pytest.mark.gpu
def test_cross_attention_rejects_bad_arguments(h):
    q, ckv = cross_case("gauss", 2, 2, 1, tier="gauss")
    for kw in (dict(layer=2), dict(layer=-1), dict(impl=2)):
        args = dict(layer=1, rows_per_utt=1, impl=0) | kw
        with pytest.raises(ValueError):
            h.debug_dec_cross_attn(q, ckv, sentinel(q.shape, np.float16), **args)
    q9, ckv9 = cross_case("gauss", 1, 2, 9, tier="gauss")
    with pytest.raises(ValueError):
        run_cross(h, q9, ckv9, 9, 0)


# ------------------------------------------------------------------------------------------------ self-attention
SA_POS = [0, 1, 31, 32, 33, 63, 64, 447]
T_IND = 448


def self_case(*, rpu=8, n_utt=3, prefill_p0=None, seed=0):
    """-> dict of the kernel's inputs, H = 6 (not a multiple of the 4 warps of a CTA).  Decode rows (prefill_p0 None):
    utterance u's rows sit at SA_POS (rotated by u), each row in its own slot; indir0 / indir1 hold different random
    slots at every position.  Prefill rows: utterance u's rpu rows are positions p0 .. p0 + rpu - 1, all in slot u.
    Every cache cell a correct kernel reads (under either flip) holds distinct data; every other cell is NaN."""
    rng = np.random.default_rng([seed, rpu, n_utt, 0 if prefill_p0 is None else 1 + prefill_p0])
    H, d = 6, 384
    R = n_utt * rpu
    n_slots = R + 3
    if prefill_p0 is None:
        pos = np.concatenate([np.roll(SA_POS, u)[:rpu] for u in range(n_utt)]).astype(np.int32)
        slot = np.arange(R, dtype=np.int32)
    else:
        pos = np.tile(prefill_p0 + np.arange(rpu), n_utt).astype(np.int32)
        slot = np.repeat(np.arange(n_utt), rpu).astype(np.int32)
    ind0 = rng.integers(0, n_slots, (R, T_IND)).astype(np.int32)
    ind1 = ((ind0 + rng.integers(1, n_slots, (R, T_IND))) % n_slots).astype(np.int32)
    kc = np.full((n_slots, T_IND, d), NAN16, np.uint16).view(np.float16)
    vc = kc.copy()
    for r in range(R):
        t = np.arange(pos[r] + 1)
        cells = [(np.full(t.size, slot[r]), t)] if prefill_p0 is not None else [
            (ind0[r, : pos[r]], t[:-1]), (ind1[r, : pos[r]], t[:-1]), (slot[r:r + 1], t[-1:])]
        for sl, tt in cells:
            kc[sl, tt] = (rng.standard_normal((tt.size, d)) * 1.73).astype(np.float16)
            vc[sl, tt] = (rng.standard_normal((tt.size, d)) + 0.1 * (r % 7)).astype(np.float16)
    q = (rng.standard_normal((R, d)) * 1.73).astype(np.float32)
    return dict(q=q, kc=kc, vc=vc, pos=pos, slot=slot, ind=(ind0, ind1), rpu=rpu, H=H, d=d, R=R,
                prefill=prefill_p0 is not None)


def self_ref(c, flip, *, ignore_flip=False, own_from_indir=False, window=0, scale=0.125, rows=None):
    """float64 reference and bound [R, d] over t <= pos (NaN rows for rows not listed).  Defects for the comparator
    tests: ignore_flip (always indir0), own_from_indir (indir[pos] instead of the own slot), window (+-1 positions),
    scale."""
    R, H = c["R"], c["H"]
    ref, tol = np.full((R, c["d"]), np.nan), np.full((R, c["d"]), np.nan)
    ind = c["ind"][0 if ignore_flip else flip]
    for r in range(R) if rows is None else rows:
        p = int(c["pos"][r])
        t = np.arange(p + 1 + window)
        if t.size == 0:
            continue
        tt = np.minimum(t, T_IND - 1)
        sl = ind[r, tt].copy()
        own = (t == p) if not c["prefill"] else np.ones(t.size, bool)
        if not own_from_indir:
            sl[own] = c["slot"][r]
        for hd in range(H):
            cs = slice(hd * 64, hd * 64 + 64)
            Kh = c["kc"][sl, tt, cs].astype(np.float64)
            Vh = c["vc"][sl, tt, cs].astype(np.float64)
            qh = c["q"][r, cs].astype(np.float64)
            s = (Kh @ qh * scale)[None]
            o = softmax_ref(s, Vh[None])
            ref[r, cs] = o[0]
            tol[r, cs] = softmax_tol(s, (np.abs(Kh) @ np.abs(qh) * 0.125)[None], Vh[None], o, score_ulps=20, p16=False,
                                     n_acc=2 * T_IND)[0]
    return ref, tol


def run_self(h, c, flip, done=None):
    ctx = sentinel((c["R"], c["d"]), np.float16)
    return h.debug_dec_self_attn(c["q"], c["kc"], c["vc"], c["pos"], c["slot"], c["ind"][0], c["ind"][1], ctx,
                                 rows_per_utt=c["rpu"], flip=flip, prefill=c["prefill"], done=done)


@pytest.mark.gpu
@pytest.mark.parametrize("flip", [0, 1])
@pytest.mark.parametrize("finished", [False, True])
def test_self_attention_matches_fp64(h, flip, finished):
    """Rows at positions 0, 1, 31, 32, 33, 63, 64 and 447 of 3 utterances; with `finished`, utterance 1's rows must
    keep the sentinel."""
    c = self_case()
    done = np.asarray([0, 1, 0], np.int32) if finished else None
    got = run_self(h, c, flip, done)
    live = np.asarray([r for r in range(c["R"]) if not (finished and r // c["rpu"] == 1)])
    ref, tol = self_ref(c, flip, rows=live)
    note_ratio("decoder self-attention", ratio(got[live], ref[live], tol[live]))
    assert within(got[live], ref[live], tol[live]), (flip, finished)
    if finished:
        assert np.all(bits(got[8:16]) == SENT16)
    assert np.array_equal(bits(run_self(h, c, flip, done)), bits(got))


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", range(1, 9))
def test_self_attention_prefill_chunks(h, chunk):
    """Prefill: `chunk` consecutive positions of each utterance as rows of one pass, all in the utterance's slot."""
    c = self_case(rpu=chunk, prefill_p0=29)
    got = run_self(h, c, 1)
    ref, tol = self_ref(c, 1)
    note_ratio("decoder self-attention", ratio(got, ref, tol))
    assert within(got, ref, tol), chunk


@pytest.mark.gpu
def test_self_attention_rejects_bad_indices(h):
    c = self_case(rpu=2, n_utt=1)
    n_slots = c["kc"].shape[0]
    for key, bad in (("slot", n_slots), ("slot", -1), ("pos", T_IND), ("ind0", n_slots), ("ind1", -1)):
        cc = dict(c, slot=c["slot"].copy(), pos=c["pos"].copy(), ind=(c["ind"][0].copy(), c["ind"][1].copy()))
        if key in ("slot", "pos"):
            cc[key][1] = bad
        else:
            cc["ind"][int(key[-1])][0, 5] = bad
        with pytest.raises(ValueError):
            run_self(h, cc, 0)
    pos = c["pos"].copy()
    pos[1] = 64  # < t_ind, but a cache of 64 positions has no position 64
    with pytest.raises(ValueError):
        run_self(h, dict(c, pos=pos, kc=c["kc"][:, :64].copy(), vc=c["vc"][:, :64].copy()), 0)


# ------------------------------------------------------------------------------------------------ LayerNorm kernels
LN_D = [384, 512, 768, 1024, 1280, 1536]


def ln_ref(x):
    x = x.astype(np.float64)
    mean = x.mean(axis=1, keepdims=True)
    c = x - mean
    return c / np.sqrt((c * c).mean(axis=1, keepdims=True) + 1e-5)


def ln_tol(x, g, b, ref, group=2):
    """Bound on |fp16 LN(x) - float64| for the kernel's fp32 two-pass statistics (one warp per row).
    Each lane sums its d / 32 values as d / 128 float4 groups ((x + y) + (z + w), `group` = 2 levels; the encoder's
    kernel adds them left to right, 3 levels) and a 5-level butterfly adds the lanes: depth D = d / 128 + 5 + group
    roundings, so the mean is within D 2^-24 mean|x| (+ 2^-24 |mean| for the division).
    The centred sum of squares is within (D + 3) 2^-24 of its value, plus d dmean^2 from the mean's error; rsqrtf adds 2
    ulp; so rstd is within e_r = (D + 5) 2^-25 + dmean^2 / (2 (var + eps)) + 2^-22 relative.  The output
    (x - mean) rstd g + b then errs by |g| rstd dmean + |y0| e_r + 4 2^-24 (|y0| + |b|) with y0 = (x - mean) rstd g,
    and the fp16 store adds half an ulp: 2^-11 |ref| + 2^-25."""
    x = x.astype(np.float64)
    d = x.shape[1]
    D = d // 128 + 5 + group
    mean = x.mean(axis=1, keepdims=True)
    var = ((x - mean) ** 2).mean(axis=1, keepdims=True)
    rstd = 1 / np.sqrt(var + 1e-5)
    dmean = D * 2.0 ** -24 * np.abs(x).mean(axis=1, keepdims=True) + 2.0 ** -24 * np.abs(mean)
    e_r = (D + 5) * 2.0 ** -25 + dmean ** 2 / (2 * (var + 1e-5)) + 2.0 ** -22
    y0 = np.abs((x - mean) * rstd * g)
    err = np.abs(g) * rstd * dmean + y0 * e_r + 4 * 2.0 ** -24 * (y0 + np.abs(b))
    return (1 + 2.0 ** -10) * err + 2.0 ** -11 * np.abs(ref) + 2.0 ** -25


def ln_fp32(x, g, b, one_pass=False):
    """The kernel's LayerNorm emulated in numpy float32, lane by lane (the comparator tests): two-pass statistics, or
    with one_pass the E[x^2] - mean^2 variance."""
    x = np.asarray(x, np.float32)
    R, d = x.shape
    f = np.float32
    v = x.reshape(R, d // 128, 32, 4)  # [row, iter, lane, 4]

    def lane_sum(a):  # per-lane ((a0 + a1) + (a2 + a3)) accumulated over the iterations, then the xor butterfly
        s = np.zeros((R, 32), np.float32)
        for i in range(a.shape[1]):
            s = s + ((a[:, i, :, 0] + a[:, i, :, 1]) + (a[:, i, :, 2] + a[:, i, :, 3]))
        for o in (16, 8, 4, 2, 1):
            s = s + s[:, np.arange(32) ^ o]
        return s[:, :1]

    mean = lane_sum(v) / f(d)
    if one_pass:
        var = lane_sum(v * v) / f(d) - mean * mean
    else:
        c = v - mean[:, :, None, None]
        var = lane_sum(c * c) / f(d)
    rstd = f(1) / np.sqrt(var + f(1e-5))
    return ((x - mean) * rstd * np.asarray(g, np.float32) + np.asarray(b, np.float32)).astype(np.float16)


def ln_rows(rng, R, d):
    """Residual rows: Gaussian, then two constant rows (values whose partial sums are exact: xn must be b exactly) and
    two rows with a common offset 100x their spread (where a one-pass variance loses its digits)."""
    x = rng.standard_normal((R, d))
    x[1], x[2] = 0.75, -3.5
    x[3] = 100.0 + rng.standard_normal(d)
    x[R - 1] = -250.0 + 2.5 * rng.standard_normal(d)
    return x


def ln_params(rng, d):
    g = (1 + 0.3 * rng.standard_normal(d)).astype(np.float32)
    b = (rng.integers(-64, 65, d) / 64).astype(np.float32)  # fp16-exact: constant rows must give b exactly
    return g, b


def check_ln_out(x_new, xn, g, b, tag, group=2, name="decoder LayerNorm (fp16 out)"):
    ref = ln_ref(x_new) * g + b
    tol = ln_tol(x_new, g, b, ref, group)
    note_ratio(name, ratio(xn, ref, tol))
    assert within(xn, ref, tol), tag
    const = np.all(x_new == x_new[:, :1], axis=1)
    assert np.array_equal(bits(xn[const]), bits(np.broadcast_to(b.astype(np.float16), xn[const].shape))), tag


def resid_case(d, ns, R, seed=0):
    rng = np.random.default_rng([d, ns, R, seed])
    bias = (rng.integers(-32, 33, d) / 64).astype(np.float32)
    target = ln_rows(rng, R, d)
    parts = (rng.standard_normal((ns, R, d)) * 0.3).astype(np.float32)
    parts[:, [1, 2]] = 0
    x = (target - bias).astype(np.float32)  # exact for the constant rows: x + bias gives the constant back
    stride = R * d + 4 * (3 + d // 128)     # slabs further apart than R d, NaN in between
    part = np.full((ns - 1) * stride + R * d + 4 * 5, np.nan, np.float32)
    for s in range(ns):
        part[s * stride: s * stride + R * d] = parts[s].reshape(-1)
    g, b = ln_params(rng, d)
    return dict(x=x, parts=parts, part=part, stride=stride, bias=bias, g=g, b=b, R=R)


def resid_expected(c, drop_last=False):
    """x + (((bias + p0) + p1) + ...) in float32, the kernel's documented order"""
    acc = np.broadcast_to(c["bias"], c["x"].shape).copy()
    for s in range(c["parts"].shape[0] - (1 if drop_last else 0)):
        acc = acc + c["parts"][s]
    return c["x"] + acc


@pytest.mark.gpu
@pytest.mark.parametrize("ns", [1, 2, 4, 8])
@pytest.mark.parametrize("d", LN_D)
def test_resid_layernorm(h, d, ns):
    """x bit-exact against float32 in the kernel's order, xn within ln_tol; R = 37 or 39 (the last CTA of 4 rows is
    partial) and rows R.. of the buffers keep the sentinel."""
    R = 37 if ns % 4 else 39
    c = resid_case(d, ns, R)
    cap = R + 5
    x = sentinel((cap, d), np.float32)
    x[:R] = c["x"]
    xn = sentinel((cap, d), np.float16)
    h.debug_dec_resid_ln(x, xn, c["part"], c["bias"], c["g"], c["b"], n_splits=ns, split_stride=c["stride"], rows=R)
    want = resid_expected(c)
    assert np.array_equal(bits(x[:R]), bits(want)), (d, ns)
    assert np.all(bits(x[R:]) == SENT32) and np.all(bits(xn[R:]) == SENT16)
    check_ln_out(want, xn[:R], c["g"], c["b"], (d, ns))


@pytest.mark.gpu
@pytest.mark.parametrize("d", LN_D)
def test_embed_layernorm(h, d):
    """x = float32(fp16 tok_emb[token]) + pos_emb[pos] bit for bit, xn within ln_tol; tokens 0 and n_vocab - 1,
    positions 0 and 447; R = 4 k + 1 with rows R.. keeping the sentinel."""
    rng = np.random.default_rng(d)
    n_vocab, n_pos, R = 4099, 448, 33
    emb = (rng.standard_normal((n_vocab, d)) * 0.5).astype(np.float16)
    pos_emb = (rng.standard_normal((n_pos, d)) * 0.5).astype(np.float32)
    tokens = rng.integers(0, n_vocab, R).astype(np.int32)
    rows = rng.integers(0, n_pos, R).astype(np.int32)
    tokens[:8], rows[:8] = [0, n_vocab - 1, 5, 6, 7, 11, 12, 13], [447, 0, 7, 8, 9, 20, 21, 22]
    # rows 5 and 6: constant sums (0.75 and -3.5 from fp16-exact halves), row 7 offset 100x its spread
    for r, cst in ((5, 0.75), (6, -3.5)):
        emb[tokens[r]] = 0.5
        pos_emb[rows[r]] = cst - 0.5
    emb[tokens[7]] = 96.0
    pos_emb[rows[7]] = 4.0 + rng.standard_normal(d).astype(np.float32)
    g, b = ln_params(rng, d)
    cap = R + 3
    x = sentinel((cap, d), np.float32)
    xn = sentinel((cap, d), np.float16)
    h.debug_dec_embed_ln(tokens, rows, emb, pos_emb, g, b, x, xn)
    want = emb[tokens].astype(np.float32) + pos_emb[rows]
    assert np.array_equal(bits(x[:R]), bits(want)), d
    assert np.all(bits(x[R:]) == SENT32) and np.all(bits(xn[R:]) == SENT16)
    check_ln_out(want, xn[:R], g, b, d)


@pytest.mark.gpu
def test_layernorm_entries_reject_bad_arguments(h):
    c = resid_case(384, 2, 5)
    x, xn = c["x"].copy(), np.zeros((5, 384), np.float16)
    for kw in (dict(n_splits=3), dict(split_stride=5 * 384 - 4), dict(split_stride=c["stride"] + 2),
               dict(split_stride=c["stride"] * 2)):
        args = dict(n_splits=2, split_stride=c["stride"]) | kw
        with pytest.raises(ValueError):
            h.debug_dec_resid_ln(x, xn, c["part"], c["bias"], c["g"], c["b"], **args)
    x2, xn2 = np.zeros((4, 320), np.float32), np.zeros((4, 320), np.float16)  # d not a multiple of 128
    with pytest.raises(ValueError):
        h.debug_dec_resid_ln(x2, xn2, np.zeros(4 * 320, np.float32), *np.ones((3, 320), np.float32), n_splits=1,
                             split_stride=0)
    emb, pe, g, b = np.zeros((10, 384), np.float16), np.zeros((4, 384), np.float32), *ln_params(np.random.default_rng(0), 384)
    for tok, pos in (([10], [0]), ([-1], [0]), ([0], [4])):
        with pytest.raises(ValueError):
            h.debug_dec_embed_ln(tok, pos, emb, pe, g, b, np.zeros((1, 384), np.float32), np.zeros((1, 384), np.float16))


# ------------------------------------------------------------------------------------------------ comparator power (CPU)
def test_cross_comparator_rejects_injected_defects():
    rpu = 3
    for kind, defect in (("late", dict(n_keys=1408)), ("padding", dict(n_keys=1501)), ("uniform", dict(n_keys=1501)),
                         ("gauss", dict(scale_head=1, scale=128 ** -0.5)), ("early", dict(scale=128 ** -0.5)),
                         ("rowpeak", dict(swap_rows=True)), ("uniform", dict(utt_shift=1)),
                         ("gauss", dict(utt_shift=1))):
        q, ckv = cross_case(kind, 2, 2, rpu, tier="gauss", n_layers=1, layer=0)
        for impl in (0, 1):
            ref, tol = cross_ref(q, ckv, rpu, layer=0, impl=impl)
            assert within(ref.astype(np.float16), ref, tol), (kind, impl)
            bad, _ = cross_ref(q, ckv, rpu, layer=0, impl=impl, **defect)
            assert not within(bad.astype(np.float16), ref, tol), (kind, defect, impl)
    # the shapes are what they claim: late / early peaks, the one-hot P exactly 1 and 0
    q, ckv = cross_case("late", 1, 2, rpu, n_layers=1, layer=0)
    s = q[:, :64].astype(np.float64) / 8 @ ckv[0, 0, 0, 0, :T_ENC].astype(np.float64).T
    assert np.all(s.argmax(axis=1) >= 1408)
    q, ckv = cross_case("onehot", 1, 2, rpu, n_layers=1, layer=0)
    s = q[:, :64].astype(np.float64) / 8 @ ckv[0, 0, 0, 0, :T_ENC].astype(np.float64).T
    p = np.exp(s - s.max(axis=1, keepdims=True)).astype(np.float16)
    assert np.all(p[:, 777] == 1) and np.all(np.delete(p, 777, axis=1) == 0)


def test_self_comparator_rejects_injected_defects():
    c = self_case()
    ref, tol = self_ref(c, 1)
    assert within(ref.astype(np.float16), ref, tol)
    for defect in (dict(ignore_flip=True), dict(own_from_indir=True), dict(window=1), dict(window=-1),
                   dict(scale=384 ** -0.5)):
        bad, _ = self_ref(c, 1, **defect)
        assert not within(bad.astype(np.float16), ref, tol), defect
    # beyond NaN poisoning, a defect on finite data must fail the bound too: the own-slot cell read at t < pos
    bad, _ = self_ref(c, 1, window=-1)
    live = np.isfinite(bad).all(axis=1)
    assert live.any() and not within(bad[live].astype(np.float16), ref[live], tol[live])
    cp = self_case(rpu=4, prefill_p0=29)
    ref, tol = self_ref(cp, 1)
    assert within(ref.astype(np.float16), ref, tol)
    bad, _ = self_ref(dict(cp, prefill=False), 1)
    assert not within(bad.astype(np.float16), ref, tol)


@pytest.mark.parametrize("d", LN_D)
def test_layernorm_comparator_rejects_injected_defects(d):
    rng = np.random.default_rng(d)
    g, b = ln_params(rng, d)
    x = ln_rows(rng, 9, d).astype(np.float32)
    ref = ln_ref(x) * g + b
    tol = ln_tol(x, g, b, ref)
    assert within(ref.astype(np.float16), ref, tol)
    assert within(ln_fp32(x, g, b), ref, tol)  # the kernel's arithmetic, emulated lane by lane, passes
    one = ln_fp32(x, g, b, one_pass=True)     # ... with E[x^2] - mean^2 it fails on the offset rows 3 and 8
    assert within(one[:3], ref[:3], tol[:3]) and not within(one[[3, 8]], ref[[3, 8]], tol[[3, 8]])
    bad = (ln_ref(x[:, :-1]) * g[:-1] + b[:-1]).astype(np.float16)  # one element short of the row
    assert not within(bad, ref[:, :-1], tol[:, :-1])
    live = [0, 3, 4, 5, 6, 7, 8]  # (the constant rows have no unbiased std)
    xl = x[live].astype(np.float64)
    unbiased = ((xl - xl.mean(1, keepdims=True)) / xl.std(1, ddof=1, keepdims=True) * g + b).astype(np.float16)
    assert not within(unbiased, ref[live], tol[live])
    # the residual's summation order is pinned bit for bit: dropping the last slab is caught
    c = resid_case(d, 4, 9)
    assert not np.array_equal(bits(resid_expected(c, drop_last=True)), bits(resid_expected(c)))
