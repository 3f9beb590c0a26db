"""Kernel-level parity of the wgmma GEMM epilogues (csrc/gemm_tc.cu) and of the encoder self-attention
(csrc/encoder.cu), each against a reference computed here in float64 from seeded data.

  * exact tier: operands in {-3..3} and biases in multiples of 1/4 keep every fp32 accumulation exact (|sum| < 2^24),
    so each epilogue must store np.float16 / np.float32 of the exact value bit for bit (both round to nearest even),
    and every element it must not touch keeps the sentinel it was filled with: rows >= m_valid, columns >= n_valid,
    cache cells not addressed, other heads / layers / split slabs
  * transcendental tier: F16_GELU and CONV2 against float64 gelu_erf of the exact pre-activation
  * census: Gaussian operands at model scale through every plan the encoder and decoder planners choose for
    d_model 384..1280, against the statistical bound tol_gemm
  * attention: softmax(Q K^T / 8 over keys < 1500) V in float64 for all 1536 query rows of every window and head

The tests without the gpu mark check the comparators themselves: each must reject a reference with a known defect."""
import numpy as np
import pytest
from scipy.special import erf

from willow_inference_server_b200 import _lib
from willow_inference_server_b200._lib import (EPI_CONV2, EPI_CROSSKV, EPI_DEC_QKV, EPI_F16, EPI_F16_GELU, EPI_F32,
                                               EPI_QKV_VT, EPI_RESID_F32)

T_PAD, T_ENC = 1536, 1500
SENT16 = np.uint16(0x7E5A)        # quiet-NaN bit patterns that no epilogue writes
SENT32 = np.uint32(0x7FC0DEAD)
U32 = 2.0 ** -24                  # unit roundoff of fp32 (round to nearest)
BNS = (64, 128, 160, 256)


@pytest.fixture(scope="module")
def h():
    return _lib.Handle.frontend(0)


def gelu64(x):
    return 0.5 * x * (1.0 + erf(x / np.sqrt(2.0)))


def sentinel(shape, dtype):
    if dtype == np.float16:
        return np.full(shape, SENT16, np.uint16).view(np.float16)
    return np.full(shape, SENT32, np.uint32).view(np.float32)


def bits(a):
    return a.view(np.uint16 if a.dtype == np.float16 else np.uint32)


# ------------------------------------------------------------------------------------------------ GEMM references
def logical_a(a, K, a_wrap, rows=None):
    """float64 rows of A as the kernel reads it: with a_wrap, logical row r = [physical row r | first K - a_wrap
    values of physical row r + 1]."""
    n = a.shape[0] - (1 if a_wrap else 0)
    rows = np.arange(n) if rows is None else np.asarray(rows)
    if not a_wrap:
        return a[rows].astype(np.float64)
    return np.concatenate([a[rows], a[rows + 1, : K - a_wrap]], axis=1).astype(np.float64)


def chunked_product(A, w, square=False):
    """A @ w^T in float64 (of w squared with `square`), over bounded slices of the large cross-K/V weights."""
    out = np.empty((A.shape[0], w.shape[0]))
    for n0 in range(0, w.shape[0], 8192):
        W = w[n0: n0 + 8192].astype(np.float64)
        out[:, n0: n0 + 8192] = A @ (W * W if square else W).T
    return out


def gemm_ref(a, w, bias=None, a_wrap=0, rows=None, drop_kblock=None, k_range=None):
    """float64 A . W^T (+ bias) of the fp16 operands, for `rows` of A (all by default)."""
    A = logical_a(a, w.shape[1], a_wrap, rows)
    if drop_kblock is not None:  # defect injection: one 64-wide K block missing
        A[:, 64 * drop_kblock: 64 * drop_kblock + 64] = 0
    if k_range is not None:
        A, w = A[:, k_range[0]: k_range[1]], w[:, k_range[0]: k_range[1]]
    out = chunked_product(A, w)
    if bias is not None:
        out += bias.astype(np.float64)
    return out


def targets(mode, rows, ncols, p, swap_heads=False, no_swizzle=False):
    """Where the epilogue stores element (row, col) for rows x [0, ncols): {buffer: (mask [R, ncols], flat index)}."""
    r = np.asarray(rows, np.int64)[:, None]
    c = np.arange(ncols, dtype=np.int64)[None, :]
    shape = (r.shape[0], ncols)
    ones = np.ones(shape, bool)
    ldo = p["ldo"]
    if mode in (EPI_F16, EPI_F16_GELU, EPI_RESID_F32, EPI_CONV2, EPI_F32):
        return {"out": (ones, np.broadcast_to(r * ldo + c, shape))}
    d, H = p["d_model"], p["n_heads"]
    b, t = r // T_PAD, r % T_PAD

    def head_of(cc):
        hd = cc // 64
        if swap_heads:  # defect injection: heads 0 and 1 exchanged
            hd = np.where(hd == 0, 1, np.where(hd == 1, 0, hd))
        return hd

    if mode == EPI_CROSSKV:
        layer, kv, cc = c // (2 * d), (c % (2 * d)) // d, c % d
        e = np.broadcast_to(cc % 64, shape)
        if p["kv_swizzle"] and not no_swizzle:  # 16-byte chunk j of key t's 128-byte row sits at chunk j ^ (t & 7)
            e = ((e // 8) ^ (t & 7)) * 8 + e % 8
        idx = ((((layer * 2 + kv) * p["batch"] + b) * H + head_of(cc)) * T_PAD + t) * 64 + e
        return {"out": (ones, np.broadcast_to(idx, shape))}
    if mode == EPI_QKV_VT:
        q = np.broadcast_to(c < 2 * d, shape)
        cv = np.maximum(c - 2 * d, 0)
        vt = ((b * H + head_of(cv)) * 64 + cv % 64) * T_PAD + t
        return {"out": (q, np.broadcast_to(r * ldo + c, shape)), "aux": (~q, np.broadcast_to(vt, shape))}
    if mode == EPI_DEC_QKV:
        q = np.broadcast_to(c < d, shape)
        is_v = np.broadcast_to(c >= 2 * d, shape)
        at = (p["row_slot"][r] * p["t_cap"] + p["row_pos"][r]) * d + (c - np.where(c >= 2 * d, 2 * d, d))
        at = np.broadcast_to(at, shape)
        return {"out": (q, np.broadcast_to(r * ldo + c, shape)), "aux": (~q & ~is_v, at), "aux2": (is_v, at)}
    raise ValueError(mode)


def epilogue_values(mode, acc, rows, p, init_out=None):
    """float64 value the epilogue stores for each (row, col) of acc (= A.W^T + bias)."""
    ncols = acc.shape[1]
    if mode == EPI_F16_GELU:
        return gelu64(acc)
    if mode == EPI_RESID_F32:  # out += acc + bias, in fp32: exact for integers
        idx = np.asarray(rows)[:, None] * p["ldo"] + np.arange(ncols)[None, :]
        return init_out.reshape(-1)[idx].astype(np.float64) + acc
    if mode == EPI_CONV2:
        t = np.asarray(rows)[:, None] % T_PAD
        pos = p["pos"].reshape(T_ENC, p["ldo"])[np.minimum(t, T_ENC - 1), np.arange(ncols)[None, :]]
        return np.where(t < T_ENC, gelu64(acc) + pos, 0.0)
    return acc


def expected_buffers(mode, acc, rows, p, init, **mutations):
    """init buffers with every epilogue store applied (values rounded to the buffer's type)."""
    want = {k: v.copy() for k, v in init.items()}
    vals = epilogue_values(mode, acc, rows, p, init.get("out"))
    for name, (mask, idx) in targets(mode, rows, acc.shape[1], p, **mutations).items():
        flat = want[name].reshape(-1)
        flat[idx[mask]] = vals[mask].astype(flat.dtype)
    return want


def exact_mismatches(got, want):
    """-> list of (buffer, mismatching elements, first flat index); empty when every bit agrees."""
    bad = []
    for name in want:
        ne = np.flatnonzero(bits(got[name]).reshape(-1) != bits(want[name]).reshape(-1))
        if ne.size:
            bad.append((name, int(ne.size), int(ne[0])))
    return bad


def tol_gemm(K, r, ref, kind, acc=None):
    """Statistical bound on |kernel - float64| for one output whose K products have root-sum-square r.

    Each of the K / 16 wgmma k-steps adds 16 exact fp16 x fp16 products into the fp32 accumulator and rounds (the
    tensor core may truncate: error <= 2^-23 of the operands' magnitude).  The partial sums of Gaussian products are a
    random walk of scale r; bounding their maximum by 8 r (exceeded with probability ~1e-14 per output) and the
    products of one step by sqrt(16) r gives |acc err| <= 2^-23 r (8 K / 16 + sqrt(K)).  Output rounding adds half an
    ulp: 2^-11 |ref| for fp16, 2^-23 |ref| for fp32 after the bias / residual add.  GELU multiplies the accumulator
    error by at most 1.13 and fp32 erff adds <= 2 ulp of 1 times |x| / 2."""
    acc_err = 2.0 ** -23 * r * (K / 2.0 + np.sqrt(K))
    if kind in ("gelu16", "conv2"):
        acc_err = 1.13 * acc_err + 2.0 ** -23 * np.abs(acc)
    if kind in ("f16", "gelu16"):  # round(ref + e) is within |e| + 2^-11 |ref + e| of ref
        return (1 + 2.0 ** -11) * acc_err + 2.0 ** -11 * np.abs(ref) + 2.0 ** -25
    return (1 + 2.0 ** -23) * acc_err + 2.0 ** -23 * np.abs(ref) + 2.0 ** -40


def worst_ratio(got, ref, tol):
    return float(np.max(np.abs(got.astype(np.float64) - ref) / tol))


RATIOS = {}


def note_ratio(name, ratio):
    RATIOS[name] = max(RATIOS.get(name, 0.0), ratio)
    print(f"worst error / tolerance, {name}: {RATIOS[name]:.3g}")


# ------------------------------------------------------------------------------------------------ exact-tier cases
# (d_model, n_heads, layers) per (bn, ragged) for the epilogues whose N is fixed by the model: ragged = N is not a
# multiple of BN (partial last tile).  N = 3 d (QKV) and N = layers * 2 d (cross K/V) are multiples of 64, and the
# cross-K/V widths here of 128, so those have no ragged case at BN 64 (and 128).
QKV_D = {(64, False): 128, (128, False): 128, (160, False): 320, (256, False): 256,
         (128, True): 192, (160, True): 192, (256, True): 192}
CKV_D = {(64, False): (128, 1), (128, False): (128, 1), (160, False): (128, 5), (256, False): (192, 2),
         (160, True): (192, 1), (256, True): (192, 1)}
EXACT_MODES = ["f32", "f32_bias", "f16", "resid", "split4", "crosskv", "crosskv_swizzled", "qkv_vt", "dec_qkv"]
MODE_OF = {"f32": EPI_F32, "f32_bias": EPI_F32, "f16": EPI_F16, "resid": EPI_RESID_F32, "split4": EPI_F32,
           "crosskv": EPI_CROSSKV, "crosskv_swizzled": EPI_CROSSKV, "qkv_vt": EPI_QKV_VT, "dec_qkv": EPI_DEC_QKV}


def int_operands(rng, M_rows, N, K):
    a = rng.integers(-3, 4, (M_rows, K)).astype(np.float16)
    w = rng.integers(-3, 4, (N, K)).astype(np.float16)
    bias = (rng.integers(-32, 33, N) / 4.0).astype(np.float32)
    return a, w, bias


def exact_case(name, bn, variant, seed=0):
    """-> dict(mode, a, w, bias, params, init buffers, gemm kwargs, rows) or None when the shape cannot exist."""
    ragged = variant == "ragged"
    rng = np.random.default_rng([EXACT_MODES.index(name), bn, ("mcast", "single", "ragged").index(variant), seed])
    mode = MODE_OF[name]
    p = dict(ldo=0, d_model=0, n_heads=0, batch=0, kv_swizzle=0, t_cap=0)
    kw = {}
    if mode in (EPI_CROSSKV, EPI_QKV_VT):
        key = (bn, ragged)
        if key not in (CKV_D if mode == EPI_CROSSKV else QKV_D):
            return None
        if mode == EPI_CROSSKV:
            d, L = CKV_D[key]
            N = L * 2 * d
        else:
            d = QKV_D[key]
            N = 3 * d
        M, K = 2 * T_PAD, 128
        p.update(d_model=d, n_heads=d // 64, batch=2, kv_swizzle=int(name == "crosskv_swizzled"))
        m_valid, n_valid = (M - 37, N - 32) if ragged else (M, N)
    elif mode == EPI_DEC_QKV:
        if (bn, ragged) not in QKV_D:
            return None
        d = QKV_D[(bn, ragged)]
        M, N, K = 256, 3 * d, 128
        m_valid, n_valid = (156, N - 32) if ragged else (M - 37, N)
        # distinct cache cells in shuffled order; rows >= m_valid point at the reserved last slot
        n_slots, t_cap = 48, 8
        cells = rng.permutation(n_slots * t_cap)[:m_valid]
        slot = np.full(M, n_slots, np.int32)
        pos = (np.arange(M) % t_cap).astype(np.int32)
        slot[:m_valid], pos[:m_valid] = cells // t_cap, cells % t_cap
        p.update(d_model=d, t_cap=t_cap, row_slot=slot, row_pos=pos)
        kw.update(row_slot=slot, row_pos=pos)
    else:
        M, K = 256, (512 if name == "split4" else 192)
        N = 2 * bn - 32 if ragged else 2 * bn
        m_valid, n_valid = (156, N - 64) if ragged else (M - 37, N)
    p["ldo"] = N
    a, w, bias = int_operands(rng, M, N, K)
    if name in ("f32", "split4"):
        bias = None
    ks = 4 if name == "split4" else 1
    init = {}
    if mode == EPI_RESID_F32:
        init["out"] = rng.integers(-100, 101, (M, N)).astype(np.float32)
    elif mode == EPI_F32:
        init["out"] = sentinel((8 if ks > 1 else 1, M, N), np.float32)
    elif mode == EPI_DEC_QKV:
        init["out"] = sentinel((M, N), np.float32)
        init["aux"] = sentinel(((n_slots + 1) * t_cap, d), np.float16)
        init["aux2"] = sentinel(((n_slots + 1) * t_cap, d), np.float16)
    elif mode == EPI_CROSSKV:
        init["out"] = sentinel((N // (2 * d), 2, 2, d // 64, T_PAD, 64), np.float16)
    elif mode == EPI_QKV_VT:
        init["out"] = sentinel((M, N), np.float16)
        init["aux"] = sentinel((2, d // 64, 64, T_PAD), np.float16)
    else:
        init["out"] = sentinel((M, N), np.float16)
    kw.update(mode=mode, bias=bias, k_splits=ks, m_valid=m_valid, n_valid=n_valid, ldo=N,
              **{k: p[k] for k in ("d_model", "n_heads", "batch", "kv_swizzle", "t_cap")})
    return dict(name=name, mode=mode, a=a, w=w, bias=bias, p=p, init=init, kw=kw, M=M, N=N, K=K, ks=ks,
                rows=np.arange(m_valid), n_valid=n_valid)


def exact_expected(c, drop_kblock=None, bias_shift=False, **mutations):
    bias = c["bias"]
    if bias_shift:  # defect injection: bias read one 32-column chunk off
        bias = np.roll(bias, 32)
    nv = c["n_valid"]
    if c["ks"] > 1:  # split-K: slab s holds the exact partial over K blocks [s K / ks, (s + 1) K / ks)
        want = {"out": c["init"]["out"].copy()}
        step = c["K"] // c["ks"]
        for s in range(c["ks"]):
            part = gemm_ref(c["a"], c["w"], bias, rows=c["rows"], drop_kblock=drop_kblock,
                            k_range=(s * step, (s + 1) * step))[:, :nv]
            want["out"][s, c["rows"], :nv] = part.astype(np.float32)
        return want
    acc = gemm_ref(c["a"], c["w"], bias, rows=c["rows"], drop_kblock=drop_kblock)[:, :nv]
    return expected_buffers(c["mode"], acc, c["rows"], c["p"], c["init"], **mutations)


def run_case(h, c, bn):
    bufs = {k: v.copy() for k, v in c["init"].items()}
    kw = dict(c["kw"])
    _, plan = h.debug_gemm(c["a"], c["w"], 0, bn, out=bufs["out"], aux=bufs.get("aux"), aux2=bufs.get("aux2"),
                           return_plan=True, **kw)
    return bufs, plan


def exact_params():
    out = []
    for name in EXACT_MODES:
        for bn in BNS:
            for variant in ("mcast", "single", "ragged"):
                if exact_case(name, bn, variant) is not None:
                    out.append((name, bn, variant))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name,bn,variant", exact_params())
def test_gemm_epilogue_exact(h, name, bn, variant):
    c = exact_case(name, bn, variant)
    got, plan = run_case(h, c, -bn if variant == "single" else bn)
    want_mcast = int(variant == "mcast")  # ragged: a partial last N tile rules the 2-CTA clusters out
    assert (plan["bn"], plan["mcast"], plan["k_splits"]) == (bn, want_mcast, c["ks"]), plan
    bad = exact_mismatches(got, exact_expected(c))
    assert not bad, (plan, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,want", [
    (128, 384, 1536, (64, 0, 4)),   # fc2 of a 384-wide decoder at 128 rows
    (128, 512, 2048, (64, 0, 8)),   # fc2 of a 512-wide decoder at 128 rows
    (256, 384, 1536, (64, 1, 4)),   # ... at 256 rows: 2-CTA clusters and split-K together
    (256, 768, 3072, (64, 1, 8)),
])
def test_decoder_planner_split_slabs_exact(h, M, N, K, want):
    """The decoder planner's split-K partials: each slab is the exact partial of its K range, the slabs it does not use
    keep the sentinel, and the slabs summed in slab order give the exact product."""
    rng = np.random.default_rng(M + N + K)
    a, w, _ = int_operands(rng, M, N, K)
    m_valid = M - 5
    out = sentinel((8, M, N), np.float32)
    _, plan = h.debug_gemm(a, w, planner=2, out=out, m_valid=m_valid, return_plan=True)
    assert (plan["bn"], plan["mcast"], plan["k_splits"]) == want, plan
    ks, step = plan["k_splits"], K // plan["k_splits"]
    want_out = sentinel((8, M, N), np.float32)
    for s in range(ks):
        want_out[s, :m_valid] = gemm_ref(a, w, rows=np.arange(m_valid), k_range=(s * step, (s + 1) * step))
    assert not exact_mismatches({"out": out}, {"out": want_out})
    total = np.zeros((m_valid, N), np.float32)
    for s in range(ks):
        total += out[s, :m_valid]
    assert np.array_equal(total, gemm_ref(a, w, rows=np.arange(m_valid)).astype(np.float32))


# ------------------------------------------------------------------------------------------------ transcendental tier
@pytest.mark.gpu
@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("mcast", [True, False])
def test_gemm_f16_gelu_within_one_ulp(h, bn, mcast):
    """fc1: fp16 gelu_erf(acc + bias) within 1 fp16 ulp of float64 gelu of the exact pre-activation, plus the fp32
    erff's absolute error near -1 (2 ulp of 1 times |x| / 2), which the output rounding may not absorb."""
    rng = np.random.default_rng(bn)
    M, N, K = 256, 2 * bn, 128
    a, w, bias = int_operands(rng, M, N, K)
    a = (a / 4).astype(np.float16)  # pre-activations in quarter steps, std ~11: much of it on the curved part of GELU
    out = sentinel((M, N), np.float16)
    m_valid = M - 37
    _, plan = h.debug_gemm(a, w, 0, bn if mcast else -bn, mode=EPI_F16_GELU, bias=bias, out=out, m_valid=m_valid,
                           return_plan=True)
    assert (plan["bn"], plan["mcast"]) == (bn, int(mcast))
    x = gemm_ref(a, w, bias)[:m_valid]
    ref = gelu64(x)
    ulp = np.spacing(np.abs(ref.astype(np.float16))).astype(np.float64)
    tol = ulp + 2.0 ** -23 * np.abs(x)
    note_ratio("F16_GELU (fp16 ulp)", worst_ratio(out[:m_valid], ref, tol))
    assert np.all(np.abs(out[:m_valid].astype(np.float64) - ref) <= tol)
    assert np.all(bits(out[m_valid:]) == SENT16)


def conv1_shaped(rng, B, d):
    """conv1 output rows as the engine lays them out: per window one zero row, 3000 frames, zero tail (3072 rows of
    d), viewed by conv2 as B * 1536 + 1 rows of 2 d."""
    h1 = np.zeros((B * 2 * T_PAD + 2, d), np.float16)
    for b in range(B):
        h1[b * 2 * T_PAD + 1: b * 2 * T_PAD + 3001] = rng.integers(-3, 4, (3000, d))
    return h1.reshape(B * T_PAD + 1, 2 * d)


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [0, *BNS])
def test_gemm_conv2_epilogue(h, bn):
    """conv2 as a GEMM over the overlapping-row view (a_wrap = 2 d): fp32 gelu(acc + bias) + pos within a few fp32 ulp
    of float64, and rows 1500..1535 of every window exactly 0."""
    rng = np.random.default_rng(7 + bn)
    B, d = 2, 320
    M, K = B * T_PAD, 3 * d
    a = conv1_shaped(rng, B, d)
    w = rng.integers(-3, 4, (d, K)).astype(np.float16)
    w = (w / 8).astype(np.float16)
    bias = (rng.integers(-32, 33, d) / 4.0).astype(np.float32)
    pos = rng.standard_normal((T_ENC, d)).astype(np.float32)
    out = sentinel((M, d), np.float32)
    _, plan = h.debug_gemm(a, w, 0, bn, mode=EPI_CONV2, bias=bias, pos=pos, out=out, a_wrap=2 * d, return_plan=True)
    assert plan["mcast"] == 0 and (bn == 0 or plan["bn"] == bn), plan
    x = gemm_ref(a, w, bias, a_wrap=2 * d)
    t = np.arange(M) % T_PAD
    valid = t < T_ENC
    g, p = gelu64(x[valid]), np.tile(pos, (B, 1))
    ref = g + p
    tol = 4 * np.spacing((np.abs(g) + np.abs(p)).astype(np.float32)).astype(np.float64) + 2.0 ** -23 * np.abs(x[valid])
    note_ratio("CONV2 (fp32 ulp)", worst_ratio(out[valid], ref, tol))
    assert np.all(np.abs(out[valid].astype(np.float64) - ref) <= tol)
    assert np.all(bits(out[~valid]) == 0)  # +0.0 exactly


# ------------------------------------------------------------------------------------------------ production census
ENC_LAYERS = {384: 4, 512: 6, 768: 12, 1024: 24, 1280: 32}  # decoder layers of the Whisper models with this width
N_VOCAB_PAD = 51968
CENSUS = set()


def census_rows(M, m_valid, rng, windows):
    rows = {0, 63, 64, 127, 128, m_valid - 1}
    if windows:
        for b in range(M // T_PAD):
            rows |= {b * T_PAD + T_ENC - 1, b * T_PAD + T_PAD - 1}
    rows |= set(rng.choice(m_valid, 8, replace=False).tolist())
    return np.asarray(sorted(r for r in rows if r < m_valid))


def census_one(h, rng, tag, a, w, bias, mode, M, planner=0, a_wrap=0, m_valid=0, **p):
    """Run one production GEMM on Gaussian data and compare the sampled rows (all columns) with float64."""
    N, K = w.shape
    m_valid = m_valid or M
    ldo = p.pop("ldo", N)
    pp = dict(ldo=ldo, d_model=p.get("d_model", 0), n_heads=p.get("n_heads", 0), batch=p.get("batch", 0),
              kv_swizzle=0, t_cap=p.get("t_cap", 0), row_slot=p.get("row_slot"), row_pos=p.get("row_pos"),
              pos=p.get("pos"))
    bufs = {}
    if mode == EPI_CROSSKV:
        bufs["out"] = np.empty(N * p["batch"] * T_PAD, np.float16)
    elif mode == EPI_DEC_QKV:
        cap = (M + 1) * p["t_cap"] * p["d_model"]
        bufs.update(out=np.empty((M, ldo), np.float32), aux=np.empty(cap, np.float16), aux2=np.empty(cap, np.float16))
    elif planner == 2:
        bufs["out"] = np.empty((8, M, N), np.float32)
    elif mode == EPI_RESID_F32:
        bufs["out"] = rng.standard_normal((M, ldo)).astype(np.float32)
    else:
        bufs["out"] = np.empty((M, ldo), np.float16 if mode in (EPI_F16, EPI_F16_GELU) else np.float32)
    init_out = bufs["out"].copy() if mode == EPI_RESID_F32 else None
    _, plan = h.debug_gemm(a, w, 0, 0, mode=mode, planner=planner, bias=bias, out=bufs["out"], aux=bufs.get("aux"),
                           aux2=bufs.get("aux2"), a_wrap=a_wrap, m_valid=m_valid, ldo=ldo, return_plan=True,
                           **{k: v for k, v in p.items() if k in ("d_model", "n_heads", "batch", "t_cap", "pos",
                                                                   "row_slot", "row_pos")})
    CENSUS.add((plan["bn"], plan["mcast"], plan["k_splits"]))
    rows = census_rows(M, m_valid, rng, windows=planner == 0)
    acc = gemm_ref(a, w, bias, a_wrap=a_wrap, rows=rows)
    r = np.sqrt(chunked_product(logical_a(a, K, a_wrap, rows) ** 2, w, square=True))
    if planner == 2:  # split-K slabs, summed in slab order as the consumer kernel does
        got = np.zeros((rows.size, N), np.float32)
        for s in range(plan["k_splits"]):
            got += bufs["out"][s, rows]
        tol = tol_gemm(K, r, acc, "f32") + plan["k_splits"] * 2.0 ** -23 * r
        note_ratio("census F32 split-K", worst_ratio(got, acc, tol))
        assert np.all(np.abs(got - acc) <= tol), (tag, plan)
        return
    kind = {EPI_F16_GELU: "gelu16", EPI_CONV2: "conv2"}.get(mode, "f16" if mode in (EPI_F16, EPI_CROSSKV, EPI_QKV_VT) else "f32")
    ref = epilogue_values(mode, acc, rows, pp, init_out)
    tol = tol_gemm(K, r, ref, kind, acc)
    if mode == EPI_DEC_QKV:  # q columns fp32, K / V columns fp16
        tol = np.where(np.arange(N) < p["d_model"], tol, tol_gemm(K, r, ref, "f16"))
    got = np.empty_like(ref)
    for name, (mask, idx) in targets(mode, rows, N, pp).items():
        got[mask] = bufs[name].reshape(-1)[idx[mask]].astype(np.float64)
    if mode == EPI_CONV2:
        tol = np.where(ref == 0, 0.0, tol)
    note_ratio(f"census mode {mode}", worst_ratio(got, ref, np.maximum(tol, 1e-300)))
    assert np.all(np.abs(got - ref) <= tol), (tag, plan)


@pytest.mark.gpu
@pytest.mark.parametrize("d", sorted(ENC_LAYERS))
def test_production_shape_census(h, d):
    """Every encoder GEMM at 1..3 windows and every batched-decoder GEMM at 128..640 rows of a d-wide model, Gaussian
    operands at model scale (unit activations, weights / sqrt(K)), against float64 on sampled rows."""
    rng = np.random.default_rng(d)
    H, L = d // 64, ENC_LAYERS[d]

    def g(*shape, scale=1.0):
        return (rng.standard_normal(shape, dtype=np.float32) * scale).astype(np.float16)

    def wts(N, K):
        return g(N, K, scale=K ** -0.5), (rng.standard_normal(N) * 0.5).astype(np.float32)

    enc_w = {"conv2": wts(d, 3 * d), "qkv": wts(3 * d, d), "o": wts(d, d), "fc1": wts(4 * d, d), "fc2": wts(d, 4 * d),
             "ckv": wts(L * 2 * d, d)}
    pos = rng.standard_normal((T_ENC, d)).astype(np.float32)
    for B in (1, 2, 3):
        M = B * T_PAD
        a_d, a_4d = g(M, d), g(M, 4 * d)
        h1 = g(M + 1, 2 * d)
        census_one(h, rng, ("conv2", d, B), h1, *enc_w["conv2"], EPI_CONV2, M, a_wrap=2 * d, pos=pos)
        census_one(h, rng, ("qkv", d, B), a_d, *enc_w["qkv"], EPI_F16, M)
        census_one(h, rng, ("o", d, B), a_d, *enc_w["o"], EPI_RESID_F32, M)
        census_one(h, rng, ("fc1", d, B), a_d, *enc_w["fc1"], EPI_F16_GELU, M)
        census_one(h, rng, ("fc2", d, B), a_4d, *enc_w["fc2"], EPI_RESID_F32, M)
        census_one(h, rng, ("ckv", d, B), a_d, *enc_w["ckv"], EPI_CROSSKV, M, d_model=d, n_heads=H, batch=B)
    dec_w = {k: wts(*nk) for k, nk in dict(qkv=(3 * d, d), o=(d, d), cq=(d, d), co=(d, d), fc1=(4 * d, d),
                                           fc2=(d, 4 * d), voc=(N_VOCAB_PAD, d)).items()}
    for M in (128, 256, 384, 640):
        m_valid = M - 5  # live rows below the row capacity
        a_d, a_4d = g(M, d), g(M, 4 * d)
        t_cap = 2
        cells = rng.permutation(M * t_cap)[:m_valid]
        slot = np.full(M, M, np.int32)
        rpos = np.zeros(M, np.int32)
        slot[:m_valid], rpos[:m_valid] = cells // t_cap, cells % t_cap
        census_one(h, rng, ("dqkv", d, M), a_d, *dec_w["qkv"], EPI_DEC_QKV, M, planner=1, m_valid=m_valid, d_model=d,
                   t_cap=t_cap, row_slot=slot, row_pos=rpos)
        census_one(h, rng, ("do", d, M), a_d, dec_w["o"][0], None, EPI_F32, M, planner=2, m_valid=m_valid)
        census_one(h, rng, ("dcq", d, M), a_d, *dec_w["cq"], EPI_F32, M, planner=1, m_valid=m_valid)
        census_one(h, rng, ("dco", d, M), a_d, dec_w["co"][0], None, EPI_F32, M, planner=2, m_valid=m_valid)
        census_one(h, rng, ("dfc1", d, M), a_d, *dec_w["fc1"], EPI_F16_GELU, M, planner=1, m_valid=m_valid)
        census_one(h, rng, ("dfc2", d, M), a_4d, dec_w["fc2"][0], None, EPI_F32, M, planner=2, m_valid=m_valid)
        census_one(h, rng, ("dvoc", d, M), a_d, dec_w["voc"][0], None, EPI_F32, M, planner=1, m_valid=m_valid)
    print(f"census after d_model {d}: (BN, mcast, k_splits) =", sorted(CENSUS))
    if d == max(ENC_LAYERS):
        # the configurations the planners are known to pick for Whisper tiny..large: 1-window encoder tiles, the
        # wave-quantised 160-wide tile, BN 64 decoder GEMMs with split-K 2/4/8, alone and on 2-CTA clusters
        need = {(128, 0, 1), (128, 1, 1), (160, 1, 1), (256, 0, 1), (256, 1, 1), (64, 0, 1), (64, 0, 2), (64, 0, 4),
                (64, 0, 8), (64, 1, 1), (64, 1, 2), (64, 1, 4), (64, 1, 8)}
        assert need <= CENSUS, need - CENSUS


# ------------------------------------------------------------------------------------------------ encoder attention
def attn_case(kind, B, H, seed=0):
    """qkv fp16 [B, 1536, 3d].  Every (window, head) has its own V offset, so mix-ups cannot cancel."""
    rng = np.random.default_rng(seed + 100 * H + B)
    d = 64 * H
    q = rng.standard_normal((B, T_PAD, H, 64)) * 20 ** 0.5  # score std ~20 (x 1/8 over 64 products)
    k = rng.standard_normal((B, T_PAD, H, 64)) * 20 ** 0.5
    v = rng.standard_normal((B, T_PAD, H, 64)) + 2 + 0.37 * np.arange(B * H).reshape(B, 1, H, 1)
    # padding keys hold large, distinct V in every case: any weight leaking past the mask shows
    v[:, T_ENC:] = 1000.0 + 7.0 * np.arange(T_PAD - T_ENC)[:, None, None] + np.arange(64)
    if kind == "late":     # every row's maximum in the last, partially masked key block 1408..1499
        q[..., 0], k[:, 1408:T_ENC, :, 0] = 28.0, 28.0
    elif kind == "early":  # maximum in the first block; later blocks negligible after the rescale
        q[..., 0], k[:, :128, :, 0] = 28.0, 36.0
    elif kind == "uniform":  # all scores 0: the mean of V over exactly 1500 keys
        q[:] = 0
    elif kind == "padding":  # padding keys would take all the weight of every row: only the mask keeps them out
        q, k = q * 0.3, k * 0.3
        q[..., 0], k[:, T_ENC:, :, 0] = 28.0, 60.0
    qkv = np.concatenate([x.reshape(B, T_PAD, d) for x in (q, k, v)], axis=2)
    return qkv.astype(np.float16)


def attn_ref(qkv, H, n_keys=T_ENC, scale=0.125):
    """float64 softmax(Q K^T * scale over keys < n_keys) V of the fp16 inputs, all 1536 query rows."""
    B, _, three_d = qkv.shape
    d = three_d // 3
    out = np.empty((B, T_PAD, d))
    for b in range(B):
        for hd in range(H):
            cs = slice(hd * 64, hd * 64 + 64)
            qh = qkv[b, :, cs].astype(np.float64)
            kh = qkv[b, :n_keys, d:][:, cs].astype(np.float64)
            vh = qkv[b, :n_keys, 2 * d:][:, cs].astype(np.float64)
            s = qh @ kh.T * scale
            p = np.exp(s - s.max(axis=1, keepdims=True))
            out[b, :, cs] = (p @ vh) / p.sum(axis=1, keepdims=True)
    return out


def attn_tol(qkv, H, ref):
    """P is rounded to fp16 (relative 2^-11) in the P.V product while the normaliser sums the unrounded P: together at
    most 2^-10 max|V| of the head's valid keys; the fp16 output adds half an ulp, 2^-11 |ref|."""
    B, _, three_d = qkv.shape
    d = three_d // 3
    vmax = np.abs(qkv[:, :T_ENC, 2 * d:].astype(np.float64)).reshape(B, T_ENC, H, 64).max(axis=(1, 3))
    return 2.0 ** -10 * np.repeat(vmax, 64, axis=1)[:, None, :] + 2.0 ** -11 * np.abs(ref)


ATTN_KINDS = ["late", "early", "uniform", "padding"]


@pytest.mark.gpu
@pytest.mark.parametrize("H", [6, 20])
@pytest.mark.parametrize("kind", ATTN_KINDS)
def test_encoder_attention_matches_fp64(h, kind, H):
    qkv = attn_case(kind, 3, H)
    ref = attn_ref(qkv, H)
    tol = attn_tol(qkv, H, ref)
    outs = [h.debug_enc_attn(qkv, H, impl) for impl in (0, 1, 2)]
    for impl, got in enumerate(outs):
        assert np.all(np.isfinite(got)), impl
        note_ratio(f"attention impl {impl}", worst_ratio(got, ref, tol))
        assert np.all(np.abs(got.astype(np.float64) - ref) <= tol), (kind, H, impl)
    for i, j in ((0, 1), (0, 2), (1, 2)):
        assert np.all(np.abs(outs[i].astype(np.float64) - outs[j]) <= tol), (kind, H, i, j)
    assert np.array_equal(bits(h.debug_enc_attn(qkv, H, 0)), bits(outs[0]))  # run to run


# ------------------------------------------------------------------------------------------------ comparator power (CPU)
GEMM_DEFECTS = {
    "drop_kblock": dict(drop_kblock=1),
    "bias_shift": dict(bias_shift=True),
    "swap_heads": dict(swap_heads=True),
    "no_swizzle": dict(no_swizzle=True),
}


@pytest.mark.parametrize("name", EXACT_MODES)
def test_exact_comparator_rejects_injected_defects(name):
    c = exact_case(name, 128, "mcast")
    good = exact_expected(c)
    assert not exact_mismatches(good, exact_expected(c))
    defects = ["drop_kblock"]
    if c["bias"] is not None:
        defects.append("bias_shift")
    if c["mode"] in (EPI_CROSSKV, EPI_QKV_VT):
        defects.append("swap_heads")
    if c["kw"]["kv_swizzle"]:
        defects.append("no_swizzle")
    for defect in defects:
        assert exact_mismatches(exact_expected(c, **GEMM_DEFECTS[defect]), good), (name, defect)


def test_census_tolerance_rejects_injected_defects():
    rng = np.random.default_rng(5)
    M, N, K = 256, 384, 1280
    a = rng.standard_normal((M, K)).astype(np.float16)
    w = (rng.standard_normal((N, K)) / K ** 0.5).astype(np.float16)
    bias = (rng.standard_normal(N) * 0.5).astype(np.float32)
    rows = np.arange(0, M, 7)
    ref = gemm_ref(a, w, bias, rows=rows)
    r = np.sqrt((a[rows].astype(np.float64) ** 2) @ (w.astype(np.float64) ** 2).T)
    for kind, cast in (("f32", np.float32), ("f16", np.float16)):
        tol = tol_gemm(K, r, ref, kind)
        assert worst_ratio(ref.astype(cast), ref, tol) <= 1.0
        bad_k = gemm_ref(a, w, bias, rows=rows, drop_kblock=K // 64 - 1).astype(cast)
        bad_b = gemm_ref(a, w, np.roll(bias, 32), rows=rows).astype(cast)
        assert worst_ratio(bad_k, ref, tol) > 1.0 and worst_ratio(bad_b, ref, tol) > 1.0, kind


def test_attention_comparator_rejects_injected_defects():
    B, H = 1, 2
    d = 64 * H
    for kind, defects in (("late", dict(n_keys=1408)), ("padding", dict(n_keys=1501)),
                          ("uniform", dict(n_keys=1501)), ("late", dict(scale=d ** -0.5)),
                          ("early", dict(scale=d ** -0.5))):
        qkv = attn_case(kind, B, H)
        ref = attn_ref(qkv, H)
        tol = attn_tol(qkv, H, ref)
        assert worst_ratio(ref.astype(np.float16), ref, tol) <= 1.0
        bad = attn_ref(qkv, H, **defects).astype(np.float16)
        assert worst_ratio(bad, ref, tol) > 1.0, (kind, defects)
    # the late case really puts every row's maximum into the last, partially masked block
    qkv = attn_case("late", B, H)
    for hd in range(H):
        cs = slice(hd * 64, hd * 64 + 64)
        s = qkv[0, :, cs].astype(np.float64) @ qkv[0, :T_ENC, d:][:, cs].astype(np.float64).T
        assert np.all(s.argmax(axis=1) >= 1408)


def test_conv2_gemm_reference_matches_conv1d_on_oracle_weights():
    """conv2 as the GEMM computes it (overlapping-row view of conv1's output, tap-major weights [d, 3 d]) equals
    torch conv1d(stride 2, padding 1) with the oracle's weights, for every valid row of every window."""
    import torch
    import torch.nn.functional as F

    from oracle.whisper_ref import WhisperOracle
    from willow_inference_server_b200 import weights as W

    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=1, n_dec_layers=1)
    oracle = WhisperOracle(dims, W.synth_engine_tensors(dims, seed=3))
    d, B = dims.d_model, 2
    rng = np.random.default_rng(9)
    a = conv1_shaped(rng, B, d)
    w = oracle.w["enc.conv2.w"].numpy().astype(np.float16)
    bias = oracle.w["enc.conv2.b"].numpy()
    got = gemm_ref(a, w, bias, a_wrap=2 * d).reshape(B, T_PAD, d)[:, :T_ENC]
    x = a.reshape(-1, d)[: B * 2 * T_PAD].reshape(B, 2 * T_PAD, d)[:, 1:3001]  # the 3000 conv1 frames per window
    ref = F.conv1d(torch.from_numpy(x.astype(np.float64)).permute(0, 2, 1),
                   oracle.conv2_w.to(torch.float16).to(torch.float64), torch.from_numpy(bias.astype(np.float64)),
                   stride=2, padding=1).permute(0, 2, 1).numpy()
    assert ref.shape == got.shape
    assert np.abs(got - ref).max() <= 1e-9 * max(1.0, np.abs(ref).max())
