"""One persistent decoder pass (csrc/decoder_mega.cu) at a time, on caller state, against the float64 reference of
tests/dec_pass_oracle.py that rounds where the pass rounds (Handle.debug_dec_pass launches it exactly as decoding does).

  * every Whisper width, d = 128 .. 1280 for both passes and 1536 for the SIMT pass (its only production use), 2 decoder
    layers, a 51865-word vocabulary (51864 and 51866 at one width each: a ragged last vocabulary slice)
  * every row count 1 .. 8 (the pass is compiled for 2, 5 and 8 rows: the others run padded), beam layouts up to 1 x 8,
    positions 0, 1, 31, 32, 33, 255 and 447 with random beam-reorder histories and NaN in every cache cell a row must not
    read, and every (utterances x heads) product whose last cross-attention key split is empty
  * the one-pass prompt prefill (rows = utterances x prompt positions, each reading K/V other rows of the pass wrote)
  * encoder rows with a dominating key in the first split and in the last partial split, and padding rows 1500..1535
    large enough to take all the weight if the mask failed; residual rows with a common offset of 4 and 16 times their
    spread (tokens 1 and 2)

Checked: residual x, logits and the K/V cells the pass writes within the derived bound; every other cache cell and every
output cell outside [R] x [V] bit for bit unchanged; the same call twice bit-identical; the warp-MMA pass against the
plain float64 model (no warp-MMA roundings) within the looser bound that records what those roundings cost.  The tests
without the gpu mark show that each comparator rejects references with known defects."""
import functools

import numpy as np
import pytest

from tests import dec_pass_oracle as O
from tests.test_gpu_kernels import bits, note_ratio, sentinel
from willow_inference_server_b200 import weights as W

NAN16 = np.uint16(0x7E00)
SENT16 = np.uint16(0x7E5A)
SENT32 = np.uint32(0x7FC0DEAD)
OFFSETS = {1: 4.0, 2: 16.0}  # token -> common offset of its residual row, in units of the row's spread
QK_GAIN = 0.6  # attention scores of a few units (the default 2.5 makes them tens: every weight error is then exponentiated)


def build_model(d, H, n_vocab=51865, seed=5):
    """(dims, tensors): 2 decoder layers, 1 encoder layer; token rows 1 and 2 carry a common offset of 4 and 16 times
    the spread of an embedded row (token + position embedding, std sqrt(2) 4 / sqrt(d) in weights.synth_state_dict)"""
    dims = W.WhisperDims(d_model=d, n_heads=H, n_enc_layers=1, n_dec_layers=2, n_vocab=n_vocab)
    t = W.synth_engine_tensors(dims, seed=seed, qk_gain=QK_GAIN)
    spread = np.sqrt(2.0) * 4.0 / np.sqrt(d)
    emb = t["dec.tok_emb"].astype(np.float32)
    for tok, k in OFFSETS.items():
        emb[tok] += np.float32(k * spread)
    t["dec.tok_emb"] = emb.astype(np.float16)
    return dims, t


@functools.lru_cache(maxsize=1)
def engine_model(d, H, n_vocab):
    from willow_inference_server_b200 import _lib

    dims, t = build_model(d, H, n_vocab)
    buf = np.zeros(W.blob_nbytes(t), np.uint8)
    W.write_blob_into(buf, dims, t)
    return dims, O.Model(t, dims), _lib.Handle.from_host(buf, 0)


# ------------------------------------------------------------------------------------------------ cases
def make_case(m, n_utt, beam, pos, *, pf_len=0, flip=1, seed=0):
    """Inputs of one pass.  Decoding: row r = u * beam + k at position pos in slot r; indir0 / indir1 hold different
    random beam-reorder histories (each entry one of the utterance's beam slots); the cells (indir[flip][r, t], t), t <
    pos, hold K ~ N(0, 1), V ~ N(0, 4) in every layer, every other cell is NaN.  Prefill: rows u * pf_len + p at
    position p, all in slot u * beam, the whole cache NaN.  Token of row 0 / 1: the offset rows (tokens 1 / 2)."""
    rng = np.random.default_rng([seed, m.d, n_utt, beam, pos, pf_len])
    L, d = m.L, m.d
    R = n_utt * (pf_len or beam)
    tokens = rng.integers(3, m.V, R).astype(np.int32)
    tokens[: min(R, 2)] = [1, 2][: min(R, 2)]
    kc = np.full((L, 8, 448, d), NAN16, np.uint16).view(np.float16)
    vc = kc.copy()
    if pf_len:
        rpos = np.tile(np.arange(pf_len), n_utt).astype(np.int32)
        slot = np.repeat(np.arange(n_utt) * beam, pf_len).astype(np.int32)
        ind = None
    else:
        rpos = np.full(R, pos, np.int32)
        slot = np.arange(R, dtype=np.int32)
        base = (np.arange(R) // beam * beam)[:, None]
        ind = [(base + rng.integers(0, beam, (R, 448))).astype(np.int32) for _ in range(2)]
        r_idx = np.repeat(np.arange(R), pos)
        t_idx = np.tile(np.arange(pos), R)
        cells = (ind[flip][r_idx, t_idx], t_idx)
        for li in range(L):
            kc[li][cells] = (0.5 * rng.standard_normal((r_idx.size, d))).astype(np.float16)
            vc[li][cells] = (2 * rng.standard_normal((r_idx.size, d))).astype(np.float16)
    enc = rng.standard_normal((n_utt, O.T_PAD, d)).astype(np.float32)
    s, ks = O.cross_geom(n_utt, m.H)
    last = min(O.T_ENC - 1, ((O.T_ENC - 1) // ks) * ks + 5)  # in the last split that holds keys (partial)
    enc[:, 37] *= 6      # dominates where its score is positive: first split
    enc[:, last] *= 6    # ... and the last, partially filled split
    enc[:, O.T_ENC:] *= 12  # padding rows: would take the weight wherever unmasked
    return dict(tokens=tokens, pos=rpos, slot=slot, pf_len=pf_len, n_utt=n_utt, beam=pf_len or beam, slot_beam=beam,
                indir=None if ind is None else ind[flip], ind=ind, flip=flip, kc=kc, vc=vc, enc=enc.astype(np.float16))


def run_gpu(h, dims, c, impl):
    x = sentinel((8, dims.d_model), np.float32)
    lg = sentinel((8, dims.n_vocab_pad), np.float32)
    kc, vc = c["kc"].copy(), c["vc"].copy()
    ind = c["ind"] or (None, None)
    ckv = h.debug_dec_pass(impl, c["tokens"], c["enc"], kc, vc, x, lg, n_utt=c["n_utt"], beam=c["slot_beam"],
                           pf_len=c["pf_len"], pos=int(c["pos"][0]) if not c["pf_len"] else 0, flip=c["flip"],
                           indir0=ind[0], indir1=ind[1])
    return dict(x=x, logits=lg, kc=kc, vc=vc, ckv=ckv)


RTOL = {0: O.RTOL_SIMT, 1: O.RTOL_MMA}


def check_pass(h, dims, m, c, impl, tag, *, repeat=False):
    """the kernel against its rounding-aware reference (and the warp-MMA pass against the plain model); sentinels
    outside [R] x [V] and every cache cell the pass does not write bit for bit unchanged; optionally a repeat bit-identical"""
    R, V = len(c["tokens"]), dims.n_vocab
    got = run_gpu(h, dims, c, impl)
    ref = O.run_pass(m, dict(c, ckv=got["ckv"]), impl)
    name = f"decoder pass impl {impl} d {dims.d_model}"
    r = O.ratios(got, ref, RTOL[impl])
    for k, v in r.items():
        note_ratio(f"{name} {k}", v)
    assert max(r.values()) <= 1, (tag, r)
    assert np.all(bits(got["x"][R:]) == SENT32) and np.all(bits(got["logits"][R:]) == SENT32), tag
    assert np.all(bits(got["logits"][:, V:]) == SENT32), tag
    wmask = np.zeros(c["kc"].shape[:3], bool)
    wmask[tuple(np.asarray(ref["written"]).T)] = True
    for f in ("kc", "vc"):
        assert np.array_equal(bits(got[f][~wmask]), bits(c[f][~wmask])), (tag, f)
    if impl == 1:  # the plain model (no warp-MMA roundings), within the looser tolerance
        plain = O.run_pass(m, dict(c, ckv=got["ckv"]), impl, mirror=False)
        rp = O.ratios(got, plain, O.RTOL_PLAIN)
        note_ratio(f"{name} vs plain float64", max(rp.values()))
        assert max(rp.values()) <= 1, (tag, rp)
        off = np.isin(c["tokens"], list(OFFSETS))
        lg = got["logits"][:R, :V]
        for rows, what in ((off, "offset rows"), (~off, "other rows")):
            if rows.any():
                err = np.abs(lg[rows] - plain["logits"][rows]).max(axis=1)
                rms = np.sqrt(np.mean(plain["logits"][rows] ** 2, axis=1))
                note_ratio(f"warp-MMA vs plain float64 d {dims.d_model}, {what}: max |logit error| / logit rms",
                           float((err / rms).max()))
    if repeat:
        again = run_gpu(h, dims, c, impl)
        for f in ("x", "logits", "kc", "vc"):
            assert np.array_equal(bits(again[f]), bits(got[f])), (tag, f)


# ------------------------------------------------------------------------------------------------ parameter sets
# (d, H): (n_utt, beam, pos) decoding layouts; every R 1..8 at the ends of the width range
FULL = [(1, 1, 0), (1, 2, 1), (3, 1, 31), (2, 2, 32), (1, 5, 33), (2, 3, 255), (7, 1, 447), (4, 2, 1), (1, 8, 447)]
LAYOUTS = {
    (128, 2): FULL + [(5, 1, 64), (6, 1, 2)],  # n_utt x H = 10, 12, 14: empty last key split
    (384, 6): [(2, 2, 32), (1, 1, 447), (3, 1, 255), (1, 6, 33)],  # 2 x 6 = 12: empty split
    (512, 8): [(1, 1, 31), (2, 2, 447), (1, 8, 0)],
    (768, 12): [(1, 1, 32), (1, 2, 255), (1, 7, 447)],  # whisper-small, one utterance: 12 heads, an empty split
    (1024, 16): [(1, 4, 33), (2, 1, 447), (1, 8, 1)],
    (1280, 20): FULL,  # 2 utterances: S = 6 with several tasks per CTA
    (1536, 24): [(1, 1, 0), (2, 3, 447), (1, 8, 32), (4, 2, 255)],  # SIMT only: fc2's K = 6144 streams chunk-major
}
VOCAB = {(512, 8): 51864, (1024, 16): 51866}
PREFILL = [(1, 1, 1), (2, 2, 2), (1, 3, 1), (2, 4, 2), (1, 5, 1), (1, 6, 1), (1, 7, 1), (1, 8, 1), (4, 2, 2)]  # (n_utt, pf_len, beam)
PREFILL_D = {(128, 2), (1280, 20)}


def cases():
    """width-major, so that each width's model is built once"""
    out = []
    for (d, H), lays in LAYOUTS.items():
        for impl in ((0,) if d > 1280 else (1, 0)):
            out += [pytest.param(d, H, impl, lay, 0, id=f"d{d}-impl{impl}-u{lay[0]}b{lay[1]}p{lay[2]}") for lay in lays]
            if (d, H) in PREFILL_D:
                out += [pytest.param(d, H, impl, (u, b, 0), pf, id=f"d{d}-impl{impl}-prefill-u{u}pf{pf}b{b}")
                        for u, pf, b in PREFILL]
    return out


def test_parameter_sets_cover_the_cross_geometries():
    """the layouts reach what the module docstring claims: every n_utt x H with an empty last split at some width
    (10, 12, 14), whisper-small one utterance, and S = 6 with more tasks than CTAs (large-v2, 2 utterances)"""
    empty = {(u, H) for (d, H), lays in LAYOUTS.items() for u, _, _ in lays if O.empty_splits(u, H)}
    assert {u * H for u, H in empty} >= {10, 12, 14}
    assert (1, 12) in empty and (2, 6) in empty
    s, ks = O.cross_geom(2, 20)
    assert s == 6 and 2 * 20 * s > O.GRID and any(u == 2 for u, _, _ in LAYOUTS[(1280, 20)])
    assert O.cross_geom(1, 12) == (11, 160) and O.empty_splits(1, 12) == [10]
    rows = {u * b for lays in LAYOUTS.values() for u, b, _ in lays}
    assert rows >= set(range(1, 9))
    assert {p for lays in LAYOUTS.values() for _, _, p in lays} >= {0, 1, 31, 32, 33, 255, 447}
    assert {pf for _, pf, _ in PREFILL} == set(range(1, 9)) and all(u * pf <= 8 and u * b <= 8 for u, pf, b in PREFILL)


# ------------------------------------------------------------------------------------------------ GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("d,H,impl,lay,pf_len", cases())
def test_decoder_pass_matches_fp64(d, H, impl, lay, pf_len):
    dims, m, h = engine_model(d, H, VOCAB.get((d, H), 51865))
    n_utt, beam, pos = lay
    c = make_case(m, n_utt, beam, pos, pf_len=pf_len, flip=(pos + n_utt) % 2)
    check_pass(h, dims, m, c, impl, (d, impl, lay, pf_len), repeat=lay == LAYOUTS[(d, H)][0] and not pf_len)


@pytest.mark.gpu
def test_decoder_pass_rejects_bad_arguments():
    """(the d = 1536 model, the last one the test above builds: the warp-MMA pass is refused there too)"""
    dims, m, h = engine_model(1536, 24, 51865)
    c = make_case(m, 1, 2, 5)

    def call(impl=0, tokens=None, n_utt=1, beam=2, pf_len=0, pos=5, ind=None):
        x = sentinel((8, dims.d_model), np.float32)
        lg = sentinel((8, dims.n_vocab_pad), np.float32)
        R = n_utt * (pf_len or beam)
        tok = np.resize(c["tokens"], R) if tokens is None else tokens
        i0, i1 = ind or (np.resize(c["ind"][0], (R, 448)), np.resize(c["ind"][1], (R, 448)))
        enc = np.resize(c["enc"], (n_utt, 1536, dims.d_model))
        h.debug_dec_pass(impl, tok, enc, c["kc"].copy(), c["vc"].copy(), x, lg, n_utt=n_utt, beam=beam, pf_len=pf_len,
                         pos=pos, flip=c["flip"], indir0=i0, indir1=i1)
        return x

    assert np.all(np.isfinite(call()[:2]))
    bad_ind = c["ind"][0].copy()
    bad_ind[1, 3] = 8
    for kw in (dict(impl=1), dict(impl=2), dict(n_utt=3, beam=3), dict(pos=448), dict(pos=-1),
               dict(tokens=np.asarray([0, dims.n_vocab])), dict(tokens=np.asarray([-1, 0])), dict(ind=(bad_ind, c["ind"][1])),
               dict(n_utt=1, pf_len=9, beam=1), dict(n_utt=3, pf_len=3, beam=1), dict(n_utt=2, pf_len=2, beam=5)):
        with pytest.raises(ValueError):
            call(**kw)


# ------------------------------------------------------------------------------------------------ comparator power (CPU)
@functools.lru_cache(maxsize=1)
def small_model():
    dims, t = build_model(128, 2)
    return dims, O.Model(t, dims)


def synth_ckv(m, c, seed=0):
    """cross K/V from the case's encoder rows as the cross-K/V GEMM forms them (fp16 of the float64 product)"""
    rng = np.random.default_rng(seed)
    n_utt, H, L = c["n_utt"], m.H, m.L
    enc = c["enc"].astype(np.float64)
    ckv = np.zeros((L, 2, n_utt, H, O.T_PAD, 64), np.float16)
    for li in range(L):
        for j in range(2):
            w = rng.standard_normal((m.d, m.d)) * 2.5 / np.sqrt(m.d)
            kv = (enc @ w.T).reshape(n_utt, O.T_PAD, H, 64).transpose(0, 2, 1, 3)
            ckv[li, j] = kv.astype(np.float16)
    return ckv


def cpu_case(n_utt, beam, pos, pf_len=0):
    dims, m = small_model()
    c = make_case(m, n_utt, beam, pos, pf_len=pf_len, flip=1)
    c["ckv"] = synth_ckv(m, c)
    return m, c


@pytest.mark.parametrize("impl", [1, 0])
def test_comparator_rejects_injected_defects(impl):
    rtol = RTOL[impl]
    for n_utt, beam, pos, pf_len, defects in (
            (2, 2, 33, 0, ["drop_cols", "drop_share", "keys_lt_pos", "own_slot", "unmask_padding"]),
            (5, 1, 40, 0, ["empty_nan", "empty_weight", "keys_lt_pos"]),  # 5 x 2 heads: the last key split is empty
            (1, 1, 0, 0, ["keys_lt_pos"]),
            (2, 2, 0, 4, ["prefill_later", "drop_share"])):
        m, c = cpu_case(n_utt, beam, pos, pf_len)
        ref = O.run_pass(m, c, impl)
        assert not O.rejects(ref, ref, rtol)
        for defect in defects:
            assert O.rejects(ref, O.run_pass(m, c, impl, defect=defect), rtol), (impl, defect)


@pytest.mark.parametrize("pos", [33, 447])
def test_simt_comparator_tells_the_passes_apart(pos):
    """the SIMT comparator rejects a reference with the warp-MMA pass's fp16 roundings (a SIMT pass that rounded its
    activations would fail), while the warp-MMA comparator accepts the plain model as within what those roundings cost"""
    m, c = cpu_case(2, 2, pos)
    simt = O.run_pass(m, c, 0)
    mma = O.run_pass(m, c, 1)
    r = O.ratios(mma, simt, O.RTOL_SIMT)
    print(f"warp-MMA roundings / SIMT tolerance at pos {pos}: {r}")
    assert max(r["x"], r["logits"]) > 3
    assert not O.rejects(mma, O.run_pass(m, c, 1, mirror=False), O.RTOL_PLAIN)


def test_one_pass_variance_on_offset_rows():
    """The kernels' fp32 E[x^2] - mean^2 statistics against exact ones, on rows with a common offset of 4 and 16 times
    their spread (rows 0 and 1): within the SIMT tolerance, so the one-pass formula costs less than the pass's own
    fp16 K/V stores at these offsets.  At 1000 times the spread it fails (the formula's limit, kept visible)."""
    m, c = cpu_case(2, 2, 33)
    exact = O.run_pass(m, c, 0)
    r = O.ratios(O.run_pass(m, c, 0, one_pass=True), exact, O.RTOL_SIMT)
    print(f"one-pass fp32 variance / SIMT tolerance: {r}")
    assert max(r.values()) <= 1
    x = exact["x"][:1]
    far = x - x.mean() + 1000 * x.std()
    g, b = np.ones(m.d), np.zeros(m.d)
    W = np.eye(m.d)
    a = O.ln_fold(0, far, g, b, W, None, True)
    one = O.ln_fold(0, far, g, b, W, None, True, one_pass=True)
    assert np.abs(one - a).max() > O.RTOL_SIMT * np.sqrt(np.mean(a * a))
