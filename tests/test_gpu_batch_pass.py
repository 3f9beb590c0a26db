"""One batched decoder pass (csrc/decoder_batch.cu batch_pass_run) at a time, on caller state, against the float64
reference of tests/batch_pass_oracle.py that rounds where the pass rounds.  Handle.debug_dec_batch_pass launches the pass
exactly as its production caller does: workspaces and GEMM plans from ensure_batch / ensure_prefill, arguments from the
engine's own builders, prefill row tables from prefill_rows_run.

  * decoding steps of 8 .. 1024 rows (8 is the decoder_batch = 2 path, 320 the batch-64 config, 1024 the largest row
    capacity), 1, 2, 5, 6 and 8 rows per window (every bd_cross_attn_kernel<NB> instance), both cross-attention kernels,
    positions 0, 1, 31, 32, 33, 255, 447 and t_cap - 1 of a cache shorter than 448, random beam-reorder histories with
    NaN in every cache cell a row must not read, finished windows between live ones
  * batched prefill: the merged first-step pass with logits (16 windows x 4 positions, 3 x 8) and a narrow prefill of two
    chained 8-position passes
  * wide prefill chained pass by pass on the same caches against ONE reference run over the whole prompt (so every
    chunk boundary is checked): the batched cache at d = 1280 (16 x 127 in chunks of 64 + 63, 1 x 226, 3 x 447 in one
    1341-row pass, a ragged 4-pass split), the persistent pass's cache at d = 128 and 1280 with the cross K/V chunk-
    swizzled and linear; then the first decoding step on top with the indirection search_init builds for fed = P - 1
  * widths d = 128 .. 1280, 2 decoder layers, a 51866-word vocabulary at d = 512

Checked: residual rows of live windows, logits (the first and last row of every 128-row tile and each window's last
prompt row) and the K/V cells the pass writes within the bound, against the rounding-aware reference and, more loosely,
the plain float64 model; every cache cell the pass does not write bit for bit unchanged; a run with every workspace row
>= R poisoned with NaN and the row-table padding pointed at an unused cache cell bit-identical to the clean run (and that
cell unchanged); one repeat per width bit-identical; the GEMM plans the pass launched equal to the planner rule mirrored
in the reference.  The tests without the gpu mark show that each comparator rejects references with known defects and
that the parameter sets reach every split-K factor, tile width, tile remainder and cross-attention instance."""
import functools
import hashlib

import numpy as np
import pytest

from tests import batch_pass_oracle as B
from tests import dec_pass_oracle as O
from tests.test_gpu_dec_pass import NAN16, build_model, engine_model
from tests.test_gpu_kernels import bits, note_ratio
from tests.test_gpu_prev_text import swizzle
from willow_inference_server_b200 import _lib
from willow_inference_server_b200 import weights as W

PLAN_NAMES = ("qkv", "o", "cq", "co", "fc1", "fc2")
SENT32 = np.uint32(0x7FC0DEAD)


def round_up(v, k):
    return -(-v // k) * k


# ------------------------------------------------------------------------------------------------ inputs
def synth_ckv(m, n_utt, seed):
    """cross K/V [L, 2, n_utt, H, 1536, 64] fp16 as the cross-K/V GEMM forms them from encoder rows with a dominating
    row in the first and in the last 128-key tile, and padding rows 1500..1535 large enough to take all the weight if the
    mask failed"""
    rng = np.random.default_rng([seed, m.d, n_utt])
    enc = rng.standard_normal((n_utt, O.T_PAD, m.d), dtype=np.float32)
    enc[:, 37] *= 6
    enc[:, 1490] *= 6
    enc[:, O.T_ENC:] *= 12
    ckv = np.zeros((m.L, 2, n_utt, m.H, O.T_PAD, 64), np.float16)
    for li in range(m.L):
        for j in range(2):
            w = (rng.standard_normal((m.d, m.d), dtype=np.float32) * np.float32(2.5 / np.sqrt(m.d)))
            ckv[li, j] = (enc @ w.T).reshape(n_utt, O.T_PAD, m.H, 64).transpose(0, 2, 1, 3).astype(np.float16)
    return ckv


def nan_cache(m, geom):
    return np.full((m.L, geom["slots"], geom["t_cap"], m.d), NAN16, np.uint16).view(np.float16)


def poison_cell(geom, written):
    """a cache cell of the last slot that the pass does not write (row-table padding exists only when the workspaces
    hold more rows than the pass: the last slot then belongs to no row and nothing reads it)"""
    used = {(s, p) for _, s, p in written}
    s = geom["slots"] - 1
    return next((s, p) for p in range(min(geom["t_cap"], 448) - 1, -1, -1) if (s, p) not in used)


def tile_rows(R):
    """the first and last row of every 128-row tile"""
    return sorted({r for t in range(0, R, 128) for r in (t, min(t + 127, R - 1))})


# ------------------------------------------------------------------------------------------------ checks
def check(m, got, c, ref, tag, logit_rows=(), plain=None):
    name = f"batched pass d {m.d}"
    r = B.ratios(got, ref, B.RTOL_BATCH, logit_rows)
    for k, v in r.items():
        note_ratio(f"{name} {k}", v)
    assert max(r.values()) <= 1, (tag, r)
    if plain is not None:
        rp = B.ratios(got, plain, B.RTOL_PLAIN, logit_rows)
        note_ratio(f"{name} vs plain float64", max(rp.values()))
        assert max(rp.values()) <= 1, (tag, rp)
    wmask = np.zeros(c["kc"].shape[:3], bool)
    wmask[tuple(np.asarray(ref["written"]).T)] = True
    for f in ("kc", "vc"):
        assert np.array_equal(bits(got[f][~wmask]), bits(c[f][~wmask])), (tag, f)


def same_bits(a, b, tag):
    """bit-identical outputs (caches may be given by their digest)"""
    for f in ("x", "logits", "kc", "vc"):
        if a.get(f) is not None:
            if isinstance(a[f], bytes):
                assert a[f] == digest(b[f]), (tag, f)
            else:
                assert np.array_equal(bits(a[f]), bits(b[f])), (tag, f)


def digest(a):
    return a if isinstance(a, bytes) else hashlib.sha256(np.ascontiguousarray(a).view(np.uint8)).digest()


def with_digests(got):
    """got with its caches replaced by their digests (the caches are the largest host arrays of a case)"""
    return dict(got, kc=digest(got["kc"]), vc=digest(got["vc"]))


def sentinel_outputs(R, d, n_vocab_pad, with_logits=True):
    """x [R + 2, d] and logits [R + 2, n_vocab_pad] (None without logits) filled with a NaN pattern the pass never
    writes"""
    x = np.full((R + 2, d), SENT32, np.uint32).view(np.float32)
    return x, np.full((R + 2, n_vocab_pad), SENT32, np.uint32).view(np.float32) if with_logits else None


def check_sentinels(x, logits, R, V):
    """rows >= R and logit columns >= n_vocab of the caller's arrays untouched"""
    assert np.all(bits(x[R:]) == SENT32)
    if logits is not None:
        assert np.all(bits(logits[R:]) == SENT32) and np.all(bits(logits[:R, V:]) == SENT32)


def fresh_handle(d, H, n_vocab=51865):
    """a handle whose batched workspaces have never been sized"""
    dims, t = build_model(d, H, n_vocab)
    buf = np.zeros(W.blob_nbytes(t), np.uint8)
    W.write_blob_into(buf, dims, t)
    return dims, O.Model(t, dims), _lib.Handle.from_host(buf, 0)


def run_chain(h, kind, passes, kc, vc, **kw):
    """passes [(p0, rows_per_utt)] chained on the same caches -> (x of every pass, the last plans)"""
    xs = []
    out = None
    dm = h.dims()
    for p0, ch in passes:
        R = kw["n_utt"] * ch
        with_logits = kw.get("with_logits", False)
        x, lg = sentinel_outputs(R, dm["d_model"], dm["n_vocab_pad"], with_logits)
        out = h.debug_dec_batch_pass(kind, kw["prompt"], kw["ckv"], kc, vc, n_utt=kw["n_utt"], rows_per_utt=ch, p0=p0,
                                     slot_stride=kw["beam"], batch_rows=kw.get("batch_rows", 1),
                                     t_need=kw.get("t_need", 1), chunk_max=kw.get("chunk_max", 1),
                                     with_logits=with_logits, cross_tc=kw.get("cross_tc", 1),
                                     ckv_sw=kw.get("ckv_sw", 0), poison=kw.get("poison"), x=x, logits=lg)
        check_sentinels(x, lg, R, dm["n_vocab"])
        xs.append(dict(out, x=x[:R], logits=lg[:R] if with_logits else None))
    return xs, out


def assemble(xs, passes, n_utt, n_pos, field="x"):
    """chunk outputs (rows u * ch + i at position p0 + i) -> window-major rows u * n_pos + p"""
    width = xs[0][field].shape[1]
    out = np.full((n_utt * n_pos, width), np.nan, np.float64)
    for o, (p0, ch) in zip(xs, passes):
        a = o[field].reshape(n_utt, ch, width)
        for u in range(n_utt):
            out[u * n_pos + p0: u * n_pos + p0 + ch] = a[u]
    return out


def assert_plans(plans, geom, d):
    want = B.layer_plans(geom["rows_cap"], d)
    for k in PLAN_NAMES:
        assert (plans[k][0], plans[k][2]) == want[k], (k, plans[k], want[k])


# ------------------------------------------------------------------------------------------------ parameter sets
# decoding steps: (d, H) -> [(n_utt, beam, pos, cross_tc, dead windows)], in the order one handle runs them (the batched
# workspaces only grow).  pos: one position for every row, a tuple of per-window positions, or LAST: the last position
# of a 64-position cache, on a handle of its own so that the cache is that short
LAST = "last"
STEPS = {
    (128, 2): [(4, 2, LAST, 1, False), (9, 1, 0, 1, False), (5, 2, 1, 0, False), (8, 5, 31, 0, True),
               (16, 5, 32, 1, True), (127, 1, 33, 0, False), (16, 8, 255, 0, False), (20, 6, 100, 0, True),
               (6, 2, (447, 0, 1, 31, 32, 255), 0, True), (129, 1, 447, 1, False), (64, 5, 447, 1, True),
               (128, 8, 255, 1, False)],
    (384, 6): [(3, 2, 33, 1, False), (10, 6, 255, 0, True)],
    (512, 8): [(2, 5, 32, 0, False), (20, 2, 447, 1, True)],
    (768, 12): [(64, 5, 255, 1, True)],
    (1024, 16): [(8, 1, 1, 0, False), (1, 8, 447, 1, False)],
    (1280, 20): [(3, 3, 33, 1, False), (5, 3, (255, 0, 33, 100, 1), 1, False), (40, 1, 255, 0, True),
                 (43, 3, 1, 1, True)],
}
VOCAB = {(512, 8): 51866}
# batched prefill (kind 1): (d, H, n_utt, prompt_len, beam, passes [(p0, chunk)], with_logits, cross_tc)
PREFILL = [(128, 2, 16, 4, 5, [(0, 4)], True, 1), (128, 2, 3, 8, 1, [(0, 8)], True, 0),
           (128, 2, 2, 17, 4, [(0, 8), (8, 8)], False, 0),
           (1280, 20, 16, 4, 5, [(0, 4)], True, 1), (1280, 20, 3, 8, 1, [(0, 8)], True, 1),
           (1280, 20, 2, 17, 4, [(0, 8), (8, 8)], False, 1)]
# wide prefill: (kind, d, H, n_utt, prompt_len, beam, chunks, ckv_sw, step on top)
# (in the order one handle runs them: the wide workspaces only grow, and the first case plans fc1 with BN 128)
WIDE = [(2, 1280, 20, 8, 101, 2, [40, 40, 15, 5], 0, True),  # a ragged 4-pass split
        (2, 1280, 20, 16, 128, 5, [64, 63], 0, True),     # DESIGN section 6: 16 windows x 128-token prompts
        (2, 1280, 20, 1, 227, 1, [226], 0, True),
        (2, 1280, 20, 3, 448, 1, [447], 0, False),        # one 1341-row pass
        (3, 128, 2, 1, 227, 1, [226], 0, False), (3, 128, 2, 1, 227, 1, [226], 1, False),
        (3, 128, 2, 2, 60, 4, [20, 20, 19], 0, False), (3, 128, 2, 2, 60, 4, [20, 20, 19], 1, False),
        (3, 1280, 20, 1, 227, 1, [226], 1, False), (3, 1280, 20, 2, 60, 4, [20, 20, 19], 1, False),
        (3, 1280, 20, 2, 60, 4, [20, 20, 19], 0, False)]


def step_params():
    def pid(p):
        return "-".join(map(str, p)) if isinstance(p, tuple) else p
    return [pytest.param(d, H, lay, id=f"d{d}-u{lay[0]}b{lay[1]}p{pid(lay[2])}-tc{lay[3]}{'-dead' if lay[4] else ''}")
            for (d, H), lays in STEPS.items() for lay in lays]


def positions(pos):
    """the positions a STEPS entry names (LAST: 63)"""
    return {63} if pos == LAST else set(pos) if isinstance(pos, tuple) else {pos}


def passes_of(chunks):
    out, p0 = [], 0
    for ch in chunks:
        out.append((p0, ch))
        p0 += ch
    return out


# ------------------------------------------------------------------------------------------------ coverage (CPU)
def test_parameter_sets_cover_the_plans_tiles_and_kernels():
    """the parameter sets reach what the module docstring claims, with the capacities the workspaces grow to in the
    order the tests run (planner rule mirrored from engine.cu plan_dec_gemm)"""
    splits, bns, rows = set(), set(), set()

    def add(cap, d):
        for bn, s in B.layer_plans(cap, d).values():
            splits.add(s)
            bns.add(bn)
    for (d, H), lays in STEPS.items():
        cap = 0
        for u, b, p, tc, dead in lays:
            cap = max(cap, round_up(u * b, 128))
            add(cap, d)
            rows.add(u * b)
    cap, last_d = 0, None
    for kind, d, H, n_utt, P, beam, chunks, sw, step in WIDE:
        cap = max(cap if d == last_d else 0, round_up(n_utt * max(chunks), 128))
        last_d = d
        add(cap, d)
    assert splits >= {1, 2, 4, 8} and bns >= {64, 128}, (splits, bns)
    assert {r % 128 for r in rows if r > 128} - {0} and any(r % 128 == 0 for r in rows), rows
    assert rows >= {8, 9, 10, 40, 80, 127, 128, 129, 320, 1024}
    simt_rpu = {b for lays in STEPS.values() for _, b, _, tc, _ in lays if tc == 0}
    assert {B.cross_nb(b) for b in simt_rpu} == {1, 5, 8} and {1, 2, 5, 6, 8} <= {b for lays in STEPS.values()
                                                                                    for _, b, _, _, _ in lays}
    assert set().union(*(positions(p) for lays in STEPS.values() for _, _, p, _, _ in lays)) >= {0, 1, 31, 32, 33, 255, 447}
    assert any(isinstance(p, tuple) and len(set(p)) > 1 for lays in STEPS.values() for _, _, p, _, _ in lays)
    assert any(d == 1280 and n == 16 and P == 128 and ch == [64, 63] for _, d, _, n, P, _, ch, _, _ in WIDE)
    assert {(k, sw) for k, _, _, _, _, _, _, sw, _ in WIDE} == {(2, 0), (3, 0), (3, 1)}


# ------------------------------------------------------------------------------------------------ GPU tests
REPEATED = set()  # widths whose first case has run twice


@pytest.mark.gpu
@pytest.mark.parametrize("d,H,lay", step_params())
def test_batched_step_matches_fp64(d, H, lay):
    n_utt, beam, pos, tc, dead = lay
    R = n_utt * beam
    if pos == LAST:
        dims, m, h = fresh_handle(d, H, VOCAB.get((d, H), 51865))
        geom = h.debug_dec_batch_geometry(0, n_utt, batch_rows=R, t_need=64)
        assert geom["t_cap"] == 64
        pos = geom["t_cap"] - 1
    else:
        dims, m, h = engine_model(d, H, VOCAB.get((d, H), 51865))
    rpos = np.repeat(np.resize(np.asarray(pos, np.int64), n_utt), beam)  # per-window positions
    t_need = int(rpos.max()) + 1
    geom = h.debug_dec_batch_geometry(0, n_utt, batch_rows=R, t_need=t_need)
    seed = [d, n_utt, beam, *np.atleast_1d(pos)]
    rng = np.random.default_rng(seed)
    flip = (int(rpos.max()) + n_utt) % 2
    tokens = rng.integers(3, m.V, R).astype(np.int32)
    tokens[: min(R, 2)] = [1, 2][: min(R, 2)]
    base = (np.arange(R) // beam * beam)[:, None]
    ind = [(base + rng.integers(0, beam, (R, 448))).astype(np.int32) for _ in range(2)]
    r_idx = np.repeat(np.arange(R), rpos)
    t_idx = np.concatenate([np.arange(p) for p in rpos])
    cells = (ind[flip][r_idx, t_idx], t_idx)

    def caches():
        """the step's input caches (fresh arrays, the same every call): K ~ N(0, 1/4), V ~ N(0, 4) in the cells (indir[r,
        t], t), t < row_pos[r], NaN everywhere else"""
        g = np.random.default_rng(seed + [1])
        kc, vc = nan_cache(m, geom), nan_cache(m, geom)
        for li in range(m.L):
            kc[li][cells] = (0.5 * g.standard_normal((r_idx.size, d))).astype(np.float16)
            vc[li][cells] = (2 * g.standard_normal((r_idx.size, d))).astype(np.float16)
        return kc, vc
    done = (np.arange(n_utt) % 3 == 1).astype(np.int32) if dead else None
    ckv = synth_ckv(m, n_utt, seed=int(rpos.max()))
    kc, vc = caches()
    c = dict(tokens=tokens, pos=rpos, slot=np.arange(R), prefill=False, n_utt=n_utt, rpu=beam, indir=ind[flip], done=done,
             kc=kc, vc=vc, ckv=ckv, cross="tc" if tc else "simt")
    lrows = [r for r in tile_rows(R) if done is None or not done[r // beam]]
    ref = B.run_batch_pass(m, c, logit_rows=lrows)
    plain = B.run_batch_pass(m, c, mirror=False, logit_rows=lrows)

    def run(poison=None):
        k2, v2 = caches()
        x, lg = sentinel_outputs(R, d, dims.n_vocab_pad)
        o = h.debug_dec_batch_pass(0, tokens, ckv, k2, v2, n_utt=n_utt, rows_per_utt=beam, row_pos=rpos, indir0=ind[0],
                                   indir1=ind[1], flip=flip, done=done, batch_rows=R, t_need=t_need, with_logits=True,
                                   cross_tc=tc, poison=poison, x=x, logits=lg)
        check_sentinels(x, lg, R, dims.n_vocab)
        return dict(o, x=x[:R], logits=lg[:R], kc=k2, vc=v2)
    got = run()
    assert got["geom"] == geom
    assert_plans(got["plans"], geom, d)
    assert got["plans"]["vocab"][0] == B.dec_plan(geom["rows_cap"], dims.n_vocab_pad, d, False)[0]
    check(m, got, c, ref, (d, lay), lrows, plain)
    cell = poison_cell(geom, ref["written"])  # (in the last slot, at a position no row reads)
    got = with_digests(got)
    del c, ref, plain, kc, vc
    same_bits(got, run(poison=cell), (d, lay, "poison"))
    if d not in REPEATED:
        REPEATED.add(d)
        same_bits(got, run(), (d, lay, "repeat"))


@pytest.mark.gpu
@pytest.mark.parametrize("case", PREFILL, ids=lambda c: f"d{c[0]}-u{c[2]}P{c[3]}b{c[4]}-{len(c[5])}pass-tc{c[7]}")
def test_batched_prefill_matches_fp64(case):
    d, H, n_utt, P, beam, passes, with_logits, tc = case
    dims, m, h = engine_model(d, H, 51865)
    rng = np.random.default_rng([d, n_utt, P, beam])
    prompt = rng.integers(3, m.V, (n_utt, P)).astype(np.int32)
    prompt[0, :2] = [1, 2]
    n_pos = passes[-1][0] + passes[-1][1]
    batch_rows = n_utt * beam
    geom = h.debug_dec_batch_geometry(1, n_utt, batch_rows=batch_rows, t_need=P + 8)
    kc, vc = nan_cache(m, geom), nan_cache(m, geom)
    ckv = synth_ckv(m, n_utt, seed=P)
    c = dict(tokens=prompt[:, :n_pos].reshape(-1), pos=np.tile(np.arange(n_pos), n_utt),
             slot=np.repeat(np.arange(n_utt) * beam, n_pos), prefill=True, n_utt=n_utt, rpu=n_pos, kc=kc, vc=vc, ckv=ckv,
             cross="tc" if tc else "simt")
    lrows = [u * n_pos + n_pos - 1 for u in range(n_utt)] if with_logits else []
    ref = B.run_batch_pass(m, c, logit_rows=lrows)
    plain = B.run_batch_pass(m, c, mirror=False, logit_rows=lrows)

    def run(poison=None):
        k2, v2 = nan_cache(m, geom), nan_cache(m, geom)
        xs, last = run_chain(h, 1, passes, k2, v2, prompt=prompt, ckv=ckv, n_utt=n_utt, beam=beam, batch_rows=batch_rows,
                             t_need=P + 8, with_logits=with_logits, cross_tc=tc, poison=poison)
        got = dict(x=assemble(xs, passes, n_utt, n_pos), kc=k2, vc=v2, plans=last["plans"], geom=last["geom"])
        if with_logits:
            got["logits"] = assemble(xs, passes, n_utt, n_pos, "logits")
        return got
    got = run()
    assert_plans(got["plans"], got["geom"], d)
    check(m, got, c, ref, case, lrows, plain)
    cell = poison_cell(got["geom"], ref["written"])
    got = with_digests(got)
    del c, ref, plain, kc, vc
    same_bits(got, run(poison=cell), (case, "poison"))


@pytest.mark.gpu
@pytest.mark.parametrize("case", WIDE, ids=lambda c: f"kind{c[0]}-d{c[1]}-u{c[3]}P{c[4]}b{c[5]}-{'+'.join(map(str, c[6]))}"
                                                     f"-sw{c[7]}{'-step' if c[8] else ''}")
def test_wide_prefill_chain_matches_one_fp64_run(case):
    kind, d, H, n_utt, P, beam, chunks, sw, step = case
    dims, m, h = engine_model(d, H, 51865)
    rng = np.random.default_rng([d, n_utt, P, beam, len(chunks)])
    prompt = rng.integers(3, m.V, (n_utt, P)).astype(np.int32)
    prompt[0, :2] = [1, 2]
    n_pos = P - 1
    passes = passes_of(chunks)
    assert passes[-1][0] + passes[-1][1] == n_pos
    kw = dict(batch_rows=n_utt * beam, t_need=min(448, P + 96), chunk_max=max(chunks))
    geom = h.debug_dec_batch_geometry(kind, n_utt, **kw)
    kc, vc = nan_cache(m, geom), nan_cache(m, geom)
    ckv = synth_ckv(m, n_utt, seed=P)
    ckv_in = swizzle(ckv) if sw else ckv
    c = dict(tokens=prompt[:, :n_pos].reshape(-1), pos=np.tile(np.arange(n_pos), n_utt),
             slot=np.repeat(np.arange(n_utt) * beam, n_pos), prefill=True, n_utt=n_utt, rpu=n_pos, kc=kc, vc=vc, ckv=ckv,
             cross="px")
    ref = B.run_batch_pass(m, c)
    plain = B.run_batch_pass(m, c, mirror=False)

    def run(poison=None):
        k2, v2 = nan_cache(m, geom), nan_cache(m, geom)
        xs, last = run_chain(h, kind, passes, k2, v2, prompt=prompt, ckv=ckv_in, n_utt=n_utt, beam=beam, ckv_sw=sw,
                             poison=poison, **kw)
        return dict(x=assemble(xs, passes, n_utt, n_pos), kc=k2, vc=v2, plans=last["plans"], geom=last["geom"])
    got = run()
    assert got["geom"]["rows_cap"] >= round_up(n_utt * max(chunks), 128)
    assert_plans(got["plans"], got["geom"], d)
    check(m, got, c, ref, case, (), plain)
    cell = poison_cell(geom, ref["written"])
    del c, ref, plain, kc, vc
    if step:
        step_on_top(h, dims, m, ckv, prompt, beam, got, kw["t_need"], geom, case)
    got = with_digests(got)
    same_bits(got, run(poison=cell), (case, "poison"))


def step_on_top(h, dims, m, ckv, prompt, beam, got, t_need, geom, case):
    n_utt, P = prompt.shape
    n_pos = P - 1
    # the first decoding step on top: rows u * beam + k at position P - 1, every earlier position from slot u * beam
    R = n_utt * beam
    sgeom = h.debug_dec_batch_geometry(0, n_utt, batch_rows=R, t_need=t_need)
    assert all(sgeom[k] == geom[k] for k in ("slots", "t_cap", "layer_stride"))
    ind = np.repeat(np.arange(n_utt) * beam, beam)[:, None] + np.zeros((1, 448), np.int64)
    ind = ind.astype(np.int32)
    tokens = np.repeat(prompt[:, P - 1], beam).astype(np.int32)
    sc = dict(tokens=tokens, pos=np.full(R, n_pos), slot=np.arange(R), prefill=False, n_utt=n_utt, rpu=beam, indir=ind,
              kc=got["kc"], vc=got["vc"], ckv=ckv, cross="tc")
    lrows = tile_rows(R)
    sref = B.run_batch_pass(m, sc, logit_rows=lrows)
    k2, v2 = got["kc"].copy(), got["vc"].copy()
    x, lg = sentinel_outputs(R, m.d, dims.n_vocab_pad)
    o = h.debug_dec_batch_pass(0, tokens, ckv, k2, v2, n_utt=n_utt, rows_per_utt=beam, row_pos=np.full(R, n_pos),
                               indir0=ind, indir1=ind, batch_rows=R, t_need=t_need, with_logits=True, x=x, logits=lg)
    check_sentinels(x, lg, R, dims.n_vocab)
    check(m, dict(o, x=x[:R], logits=lg[:R], kc=k2, vc=v2), sc, sref, (case, "step"), lrows,
          B.run_batch_pass(m, sc, mirror=False, logit_rows=lrows))


@pytest.mark.gpu
def test_batched_pass_rejects_bad_arguments():
    """every index is checked against the geometry before anything is sized or launched: a refused call leaves the
    caller's caches and outputs and the handle's workspaces as they were (a fresh d = 128 handle: a 32-position cache)"""
    dims, m, h = fresh_handle(128, 2)
    n_utt, beam, pos = 2, 2, 5
    R = n_utt * beam
    geom = h.debug_dec_batch_geometry(0, n_utt, batch_rows=R, t_need=32)
    assert geom["t_cap"] == 32 and geom["slots"] == 128
    ckv = np.zeros((m.L, 2, n_utt, m.H, O.T_PAD, 64), np.float16)
    ind = np.zeros((R, 448), np.int32)
    prompt = np.full((n_utt, 60), 3, np.int32)
    kc0 = np.zeros((m.L, geom["slots"], geom["t_cap"], m.d), np.float16)

    def call(kind, tokens, **kw):
        kc, vc = kc0.copy(), kc0.copy()
        rows = n_utt * kw["rows_per_utt"]
        kw.setdefault("with_logits", kind == 0)
        x, lg = sentinel_outputs(rows, m.d, dims.n_vocab_pad, kw["with_logits"])
        out = h.debug_dec_batch_pass(kind, tokens, ckv, kc, vc, n_utt=n_utt, t_need=32, x=x, logits=lg, **kw)
        check_sentinels(x, lg, rows, dims.n_vocab)
        return out

    def step(**kw):
        a = dict(tokens=np.full(R, 3, np.int32), row_pos=np.full(R, pos), indir0=ind, indir1=ind, rows_per_utt=beam,
                 batch_rows=R)
        a.update(kw)
        return call(0, a.pop("tokens"), **a)

    assert np.all(np.isfinite(step()["x"][:R]))

    def refused(kind, tokens, **kw):
        kc, vc = kc0.copy(), kc0.copy()
        x = np.full((R + 2, m.d), SENT32, np.uint32).view(np.float32)
        kw.setdefault("with_logits", kind == 0)
        lg = np.full((R + 2, dims.n_vocab_pad), SENT32, np.uint32).view(np.float32) if kw["with_logits"] else None
        with pytest.raises(ValueError):
            h.debug_dec_batch_pass(kind, tokens, ckv, kc, vc, n_utt=kw.pop("n_utt", n_utt), t_need=kw.pop("t_need", 32),
                                   x=x, logits=lg, **kw)
        assert np.array_equal(bits(kc), bits(kc0)) and np.array_equal(bits(vc), bits(kc0))
        assert np.all(bits(x) == SENT32) and (lg is None or np.all(bits(lg) == SENT32))
        assert h.debug_dec_batch_geometry(0, n_utt, batch_rows=R, t_need=32) == geom  # nothing grew

    bad_ind = ind.copy()
    bad_ind[1, 2] = geom["slots"]
    base = dict(row_pos=np.full(R, pos), indir0=ind, indir1=ind, rows_per_utt=beam, batch_rows=R)
    tok = np.full(R, 3, np.int32)
    for kw in (dict(tokens=np.asarray([0, 1, 2, dims.n_vocab], np.int32)), dict(tokens=np.asarray([-1, 1, 2, 3], np.int32)),
               dict(row_pos=np.full(R, geom["t_cap"])), dict(row_pos=np.full(R, -1)), dict(indir0=bad_ind),
               dict(with_logits=False), dict(ckv_sw=1), dict(cross_tc=2), dict(poison=(R - 1, pos)),
               dict(poison=(0, geom["t_cap"]))):
        a = dict(base, **kw)
        refused(0, a.pop("tokens", tok), **a)
    for kind, kw in ((1, dict(rows_per_utt=9)), (1, dict(rows_per_utt=8, p0=53)),
                     (1, dict(rows_per_utt=4, slot_stride=geom["slots"])),
                     (1, dict(rows_per_utt=4, with_logits=True, cross_tc=0, ckv_sw=1)),
                     # prefill positions at or beyond the cache's 32 positions (inside the prompt and n_text_ctx)
                     (1, dict(rows_per_utt=4, p0=30)), (1, dict(rows_per_utt=8, p0=32, slot_stride=64)),
                     (2, dict(rows_per_utt=20, p0=20, chunk_max=20)), (2, dict(rows_per_utt=33, chunk_max=40)),
                     (2, dict(rows_per_utt=10, chunk_max=8)), (4, dict(rows_per_utt=1))):
        refused(kind, prompt, batch_rows=R, **kw)
    refused(1, prompt, n_utt=1, rows_per_utt=4, p0=0, batch_rows=R, t_need=449)
    with pytest.raises(ValueError):
        h.debug_dec_batch_geometry(0, 1025, batch_rows=1025, t_need=64)
    # the same positions inside a cache that holds them: accepted
    call(1, prompt, rows_per_utt=4, p0=28, batch_rows=R)


# ------------------------------------------------------------------------------------------------ comparator power (CPU)
@functools.lru_cache(maxsize=1)
def small_model():
    dims, t = build_model(128, 2)
    return O.Model(t, dims)


def cpu_step_case(cross, n_utt=4, beam=2, pos=33, dead=True):
    m = small_model()
    R = n_utt * beam
    rng = np.random.default_rng([n_utt, beam, pos])
    tokens = rng.integers(3, m.V, R)
    tokens[:2] = [1, 2]
    ind = (np.arange(R) // beam * beam)[:, None] + rng.integers(0, beam, (R, 448))
    kc = np.full((m.L, 128, 64, m.d), NAN16, np.uint16).view(np.float16)
    vc = kc.copy()
    r_idx, t_idx = np.repeat(np.arange(R), pos), np.tile(np.arange(pos), R)
    for li in range(m.L):
        kc[li][ind[r_idx, t_idx], t_idx] = (0.5 * rng.standard_normal((r_idx.size, m.d))).astype(np.float16)
        vc[li][ind[r_idx, t_idx], t_idx] = (2 * rng.standard_normal((r_idx.size, m.d))).astype(np.float16)
    done = np.asarray([0, 1, 0, 0][:n_utt]) if dead else None
    return m, dict(tokens=tokens, pos=np.full(R, pos), slot=np.arange(R), prefill=False, n_utt=n_utt, rpu=beam,
                   indir=ind, done=done, kc=kc, vc=vc, ckv=synth_ckv(m, n_utt, 1), cross=cross,
                   splits=B.layer_plans(128, m.d)["fc2"][1])


def cpu_prefill_case(sw, n_utt=2, n_pos=20, beam=3):
    m = small_model()
    rng = np.random.default_rng([n_utt, n_pos, beam])
    tokens = rng.integers(3, m.V, n_utt * n_pos)
    kc = np.full((m.L, 8, 448, m.d), NAN16, np.uint16).view(np.float16)
    ckv = synth_ckv(m, n_utt, 2)
    return m, dict(tokens=tokens, pos=np.tile(np.arange(n_pos), n_utt), slot=np.repeat(np.arange(n_utt) * beam, n_pos),
                   prefill=True, n_utt=n_utt, rpu=n_pos, kc=kc, vc=kc.copy(), ckv=swizzle(ckv) if sw else ckv,
                   ckv_sw=sw, cross="px", chunk0=10, splits=2)


@pytest.mark.parametrize("mirror", [True, False])
@pytest.mark.parametrize("cross", ["tc", "simt"])
def test_step_comparator_rejects_injected_defects(cross, mirror):
    m, c = cpu_step_case(cross)
    assert c["splits"] == 2
    rtol = B.RTOL_BATCH if mirror else B.RTOL_PLAIN
    lrows = [0, 7]
    ref = B.run_batch_pass(m, c, mirror=mirror, logit_rows=lrows)
    assert not B.rejects(ref, ref, rtol, lrows)
    assert not B.rejects(ref, B.run_batch_pass(m, c, mirror=not mirror, logit_rows=lrows), B.RTOL_PLAIN, lrows)
    for defect in ("drop_slab", "next_gain", "keys_lt_pos", "unmask_padding", "neighbour_ckv", "dead_not_skipped"):
        bad = B.run_batch_pass(m, c, mirror=mirror, defect=defect, logit_rows=lrows)
        assert B.rejects(ref, bad, rtol, lrows), (cross, mirror, defect)


@pytest.mark.parametrize("mirror", [True, False])
@pytest.mark.parametrize("sw", [0, 1])
def test_prefill_comparator_rejects_injected_defects(sw, mirror):
    m, c = cpu_prefill_case(sw)
    rtol = B.RTOL_BATCH if mirror else B.RTOL_PLAIN
    ref = B.run_batch_pass(m, c, mirror=mirror)
    assert not B.rejects(ref, ref, rtol)
    defects = ["chunk_blind", "slot_u", "keys_lt_pos", "unmask_padding", "neighbour_ckv", "drop_slab", "next_gain"]
    for defect in defects + (["swizzle_ignored"] if sw else []):
        assert B.rejects(ref, B.run_batch_pass(m, c, mirror=mirror, defect=defect), rtol), (sw, mirror, defect)


def test_cross_attention_roundings_against_the_plain_softmax():
    """the three cross-attention mirrors agree with the exact softmax to half of RTOL_BATCH, and the px
    mirror's running-maximum P16 differs from the tc mirror's exact-maximum P16 (they are not the same model)"""
    rng = np.random.default_rng(0)
    q = rng.standard_normal((6, 2, 64)) * 3
    K = B.r16(rng.standard_normal((2, 1500, 64)))
    V = B.r16(rng.standard_normal((2, 1500, 64)) * 2)
    K[:, 1400] *= 4
    exact = B.cross_attend(q, K, V, "simt", True)
    out = {i: B.cross_attend(q, K, V, i, True) for i in B.CROSS_IMPLS}
    rms = np.sqrt(np.mean(exact ** 2))
    for i, v in out.items():
        assert np.abs(v - exact).max() < 0.5 * B.RTOL_BATCH * rms, i
    assert not np.array_equal(out["tc"], out["px"])
