"""The device token search (search.cu) one step at a time, with its whole state in and out.

``wisb_debug_search_step`` (``Handle.debug_search_step_state``) runs ONE production step -- processors, top-k partials,
candidate merge, bookkeeping and step advance -- on caller state and returns all of it.  ``expected_step`` maps the
oracle's one bookkeeping step (``oracle.whisper_ref.beam_step``, the step every oracle search runs) onto the device
state, given the device's own candidate list:
  * integers (seq / indir ping-pong, tokens, done, n_hyp, best hypothesis, DecState, flip, row_pos) must be equal;
  * cum and best_score must be the fp32 product score * norm within CUM_ULPS (powf is not correctly rounded);
  * the candidate list itself is checked against float64 (``ref_candidates``) wherever float64 has no near-tie.
Multi-step chains run on the host with logits that are a seeded function of each row's history, and must end where the
oracle's search loop ends wherever every step's decision gap is clear.  The tests without the gpu mark show that the
comparator rejects oracle steps with known defects."""
import zlib

import numpy as np
import pytest
import torch

from oracle.whisper_ref import (BEAM_STEP_DEFECTS, BeamState, beam_search, beam_step, length_norm, max_hypotheses)
from tests.ts_oracle import apply_timestamp_rules
from willow_inference_server_b200 import _lib, weights as W

GEOMETRIES = [(51865, 50257, 50363), (51864, 50256, 50362), (51866, 50257, 50364)]   # V, eot, no_timestamps
LDL = 51968
CUM_ULPS = 4          # cum / best_score vs the fp32 product score * norm (measured worst: DESIGN.md section 5)
DEFECTS = BEAM_STEP_DEFECTS + ("indir_own", "indir_inclusive")
INT_KEYS = ("st", "flip", "seq", "indir", "tokens", "row_pos", "done", "n_hyp", "best_len", "best_tokens")


# ----------------------------------------------------------------------------------------------------------- reference
def fp32_norm(gen, lp):
    return float(np.float32(length_norm(gen, lp)))


def expected_step(st, ci, cs, *, beam, V, eot, max_hyp, lp, caps=None, defect=None):
    """The device state after one step, from state `st` and the candidate list (ci, cs) [n_utt, 2 beam]."""
    out = {k: v.copy() for k, v in st.items()}
    pos, gen, _, all_done, _ = (int(x) for x in st["st"])
    if all_done:
        return out
    n_utt = len(st["done"])
    max_new = st["seq"].shape[2]
    cur = int(st["flip"][0])
    nxt = cur ^ 1
    norm = fp32_norm(gen, lp)
    for u in range(n_utt):
        rows = range(u * beam, (u + 1) * beam)
        if st["done"][u]:
            for r in rows:
                out["seq"][nxt, r] = st["seq"][cur, r]
                out["indir"][nxt, r] = st["indir"][cur, r]
                out["indir"][nxt, r, pos] = r
            continue
        n_hyp, best = int(st["n_hyp"][u]), float(st["best_score"][u])
        hyps = [(NEG, [])] * n_hyp
        if best > NEG and n_hyp:
            hyps[0] = (best, list(st["best_tokens"][u, : st["best_len"][u]]))
        prev = BeamState([list(st["seq"][cur, r, :gen]) for r in rows], [float(st["cum"][r]) for r in rows],
                         hyps=hyps, best=0 if best > NEG and n_hyp else -1)
        cap = int(caps[u]) if caps is not None else max_new
        new = beam_step(prev, [int(i) for i in ci[u]], [float(s) for s in cs[u]], V=V, eot=eot, gen=gen, cap=cap,
                        max_hyp=max_hyp, norm=norm, defect=defect if defect in BEAM_STEP_DEFECTS else None)
        out["n_hyp"][u] = len(new.hyps)
        out["best_score"][u] = new.best_score
        if new.best != prev.best:
            toks = new.best_tokens
            out["best_tokens"][u, : len(toks)] = toks
            out["best_len"][u] = len(toks)
        for k, r in enumerate(rows):
            pr = u * beam + new.parents[k]
            out["seq"][nxt, r, : gen + 1] = new.seqs[k][:max_new]
            if defect == "indir_inclusive":
                out["indir"][nxt, r, : pos + 1] = st["indir"][cur, pr, : pos + 1]
            else:
                out["indir"][nxt, r, :pos] = st["indir"][cur, pr, :pos]
                out["indir"][nxt, r, pos] = r if defect == "indir_own" else pr
            out["tokens"][r] = new.tokens[k]
            out["cum"][r] = new.cum[k]
        if new.finished:
            out["done"][u] = 1
            out["st"][2] += 1
    out["st"][0] += 1
    out["st"][1] += 1
    out["st"][3] = int(out["st"][2] == n_utt)
    out["flip"][0] = nxt
    out["row_pos"] += 1
    return out


NEG = float("-inf")


def ulps(a, b):
    """|a - b| in fp32 ulps (equal infinities: 0)."""
    a, b = np.float32(a), np.float32(b)
    if a == b:
        return 0
    if not (np.isfinite(a) and np.isfinite(b)):
        return 1 << 30
    ia, ib = (int(np.array(x, np.float32).view(np.int32)) for x in (a, b))
    ia = ia if ia >= 0 else -(ia & 0x7fffffff)
    ib = ib if ib >= 0 else -(ib & 0x7fffffff)
    return abs(ia - ib)


def compare(got, want, where=""):
    """-> worst ulps of cum / best_score; raises AssertionError on any other difference."""
    for k in INT_KEYS:
        assert np.array_equal(got[k], want[k]), (where, k, np.argwhere(got[k] != want[k])[:4])
    worst = 0
    for k in ("cum", "best_score"):
        for g, w in zip(got[k], want[k]):
            d = ulps(g, w)
            assert d <= CUM_ULPS, (where, k, g, w, d)
            worst = max(worst, d)
    return worst


def processed(logits, mask, hists, gen, V, eot, no_ts, ts, max_init):
    x = torch.from_numpy(np.asarray(logits[:, :V], np.float64))
    m = torch.from_numpy(mask)
    x[:, (m & 1).bool()] = NEG
    if gen == 0:
        x[:, (m & 2).bool()] = NEG
    if ts:
        x = apply_timestamp_rules(x, hists, gen, no_timestamps=no_ts, eot=eot, max_initial_timestamp_index=max_init)
    return x


def ref_candidates(logits, mask, st, *, beam, V, eot, no_ts=0, ts=0, max_init=50, lp=1.0):
    """float64 candidates [n_utt, 2 beam] (ids, -1 = none; scores) of the rows' processed logits."""
    gen, cur = int(st["st"][1]), int(st["flip"][0])
    hists = [list(h[:gen]) for h in st["seq"][cur]]
    x = processed(logits, mask, hists, gen, V, eot, no_ts, ts, max_init)
    logp = x - torch.logsumexp(x, -1, keepdim=True)
    total = (logp + torch.from_numpy(st["cum"].astype(np.float64))[:, None]) / length_norm(gen, lp)
    ids, scores = [], []
    for u in range(len(st["done"])):
        flat = total[u * beam : (u + 1) * beam].reshape(-1)
        valid = torch.isfinite(logp[u * beam : (u + 1) * beam]).reshape(-1)
        if gen == 0:
            valid[V:] = False
        idx = torch.nonzero(valid).flatten()
        order = idx[torch.argsort(-flat[idx], stable=True)[: 2 * beam]].tolist()
        pad = 2 * beam - len(order)
        ids.append(order + [-1] * pad)
        scores.append([float(flat[i]) for i in order] + [NEG] * pad)
    return np.asarray(ids), np.asarray(scores), total


def check_candidates(ci, cs, wi, ws, total, beam, where):
    """Device candidates vs float64: the same ids except inside float64 near-ties, scores within 1e-5."""
    for u in range(len(ci)):
        for j in range(2 * beam):
            if wi[u, j] < 0:
                assert ci[u, j] == -1, (where, u, j)
                continue
            assert ci[u, j] >= 0, (where, u, j)
            if ci[u, j] != wi[u, j]:
                got64 = float(total[u * beam : (u + 1) * beam].reshape(-1)[ci[u, j]])
                assert abs(got64 - ws[u, j]) <= 2e-6 * max(1.0, abs(ws[u, j])), (where, u, j, ci[u, j], wi[u, j])
            if np.isfinite(ws[u, j]):
                assert abs(cs[u, j] - ws[u, j]) <= 1e-5 * max(1.0, abs(ws[u, j])), (where, u, j)
            else:
                assert cs[u, j] == ws[u, j], (where, u, j)


# ------------------------------------------------------------------------------------------------------ crafted steps
def base_mask(V, eot):
    m = np.zeros(V, np.uint8)
    m[W.WhisperDims().suppress_ids] |= 1
    m[[220, eot]] |= 2
    return m


def new_state(h, n_utt, beam, *, gen, pos=None, max_new=None, t_max=None, rng=None, cum=None, V=51865):
    """A mid-search state: random histories (tokens < 50000), random indirection slots in every cell (the cells at and
    after pos too, so that a copy of the wrong range shows), cum given or equal for all rows."""
    rng = rng or np.random.default_rng(0)
    pos = gen + 3 if pos is None else pos
    max_new = max_new or gen + 4
    t_max = t_max or pos + 3
    R = n_utt * beam
    st = h.search_state(n_utt, beam, max_new, t_max)
    st["st"][:2] = (pos, gen)
    st["flip"][0] = gen & 1
    st["seq"][:] = rng.integers(0, 50000, st["seq"].shape)
    st["indir"][:] = rng.integers(0, R, st["indir"].shape)
    st["tokens"][:] = rng.integers(0, 50000, R)
    st["row_pos"][:] = pos
    st["cum"][:] = -1.5 if cum is None else cum
    return st


def rank_logits(V, R, ranks, ldl=LDL, base=0.0):
    """Logits [R, ldl] (NaN padding) with `ranks` = [(row, token), ...] set to decreasing values above `base`: with
    equal cum and a vocabulary-wide base mass dominating every row's lse, the candidate list follows `ranks`."""
    x = np.full((R, ldl), np.nan, np.float32)
    x[:, :V] = base
    for j, (r, t) in enumerate(ranks):
        x[r, t] = base + 4.0 - 0.25 * j
    return x


TEXT = [t for t in range(1000, 40000, 37) if t not in set(W.WhisperDims().suppress_ids)]   # plain text tokens


def free_token(at):
    """The first text token >= at that no processor suppresses."""
    return next(t for t in range(at, at + 1000) if t not in set(W.WhisperDims().suppress_ids))


TIES = [free_token(100), free_token(200), free_token(1700), free_token(30000), free_token(45000)]


def crafted(h, V, eot):
    """(name, beam, state, logits, mask, step kwargs) of the crafted single steps."""
    mask = base_mask(V, eot)
    rng = np.random.default_rng(5)
    T = TEXT.__getitem__
    for beam in (2, 4, 8):
        R = beam
        # eot at rank 0 / at rank beam - 1 / at several ranks / only below rank beam
        layouts = {
            "eot_rank0": [(0, eot)] + [(k % R, T(k)) for k in range(1, 2 * beam)],
            "eot_rank_last": [(k % R, T(k)) for k in range(beam - 1)] + [(1 % R, eot)] +
                             [(k % R, T(k)) for k in range(beam, 2 * beam)],
            "eot_several": [(k, eot) if k % 2 == 0 else (k, T(k)) for k in range(beam)] +
                           [(k % R, T(k + 50)) for k in range(beam)],
            "eot_below_beam": [(k % R, T(k)) for k in range(beam)] + [(0, eot)] +
                              [(k % R, T(k + 50)) for k in range(beam - 1)],
        }
        for name, ranks in layouts.items():
            st = new_state(h, 1, beam, gen=3, rng=rng, V=V)
            yield name, beam, st, rank_logits(V, R, ranks), mask, {}
        # is_last with and without eot (max_new = gen + 1), and secondary picks running out of non-eot candidates
        st = new_state(h, 1, beam, gen=3, max_new=4, rng=rng, V=V)
        yield "is_last_eot", beam, st, rank_logits(V, R, layouts["eot_several"]), mask, {}
        st = new_state(h, 1, beam, gen=3, max_new=4, rng=rng, V=V)
        yield "is_last_plain", beam, st, rank_logits(V, R, layouts["eot_rank_last"]), mask, {}
        st = new_state(h, 1, beam, gen=3, max_new=5, rng=rng, V=V)    # the step before the last
        yield "before_last", beam, st, rank_logits(V, R, layouts["eot_rank_last"]), mask, {}
        ranks = [(k, T(k)) for k in range(beam)] + [(k, eot) for k in range(beam)]
        st = new_state(h, 1, beam, gen=3, max_new=4, rng=rng, V=V)
        yield "secondary_runs_out", beam, st, rank_logits(V, R, ranks), mask, {}
        # fewer finite candidates than 2 beam: one unmasked token per row (gen > 0), three at gen 0
        m1 = mask.copy()
        m1[:] |= 1
        m1[eot] = 0
        st = new_state(h, 1, beam, gen=2, rng=rng, V=V)
        st["cum"][:] = -np.arange(beam, dtype=np.float32)
        yield "few_candidates", beam, st, rank_logits(V, R, []), m1, {}
        m3 = mask.copy()
        m3[:] |= 1
        m3[T(2)] = 0
        st = new_state(h, 1, beam, gen=0, pos=3, rng=rng, V=V)
        st["cum"][:] = 0
        yield "few_candidates_gen0", beam, st, rank_logits(V, R, [(0, T(2))]), m3, {}
        # hypothesis score ties: two identical rows with equal cum end in eot at ranks 0 and 1, first one wins
        st = new_state(h, 1, beam, gen=3, rng=rng, V=V)
        x = rank_logits(V, R, [(0, eot)] + [(0, T(k)) for k in range(1, 2 * beam)])
        x[1] = x[0]
        yield "hyp_tie", beam, st, x, mask, {}
    # exact logit ties inside a chunk, across chunks and across beams with equal cum (identical rows)
    for beam in (1, 3):
        st = new_state(h, 2, beam, gen=2, rng=rng, V=V)
        x = rank_logits(V, 2 * beam, [])
        x[:, TIES] = 3.0                                 # the first two in one chunk, the others in other chunks
        yield "logit_ties", beam, st, x, mask, {}
    # timestamp mode, gen 0: max_initial_timestamp_index 3 leaves 4 candidates for 10 (beam 5)
    st = new_state(h, 2, 5, gen=0, pos=2, rng=rng, V=V)
    st["cum"][:] = 0
    yield "ts_gen0_few", 5, st, rank_logits(V, 10, []), mask, dict(timestamps=True, max_initial_timestamp_index=3)


def run_step(h, st, x, mask, *, beam, V, eot, no_ts, patience=1.0, lp=1.0, caps=None, **kw):
    max_hyp = max_hypotheses(beam, patience)
    got, ci, cs, lse = h.debug_search_step_state(x, mask, st, beam=beam, max_hyp=max_hyp, eot=eot, V=V, no_timestamps=no_ts,
                                           length_penalty=lp, max_new_u=caps, **kw)
    want = expected_step(st, ci, cs, beam=beam, V=V, eot=eot, max_hyp=max_hyp, lp=lp, caps=caps)
    return got, want, ci, cs


@pytest.fixture(scope="module")
def h():
    return _lib.Handle.frontend(0)


@pytest.mark.gpu
@pytest.mark.parametrize("geom", range(3))
def test_crafted_steps(h, geom):
    V, eot, no_ts = GEOMETRIES[geom]
    n = 0
    for name, beam, st, x, mask, kw in crafted(h, V, eot):
        ts = kw.get("timestamps", False)
        got, want, ci, cs = run_step(h, st, x, mask, beam=beam, V=V, eot=eot, no_ts=no_ts, **kw)
        compare(got, want, (geom, name, beam))
        wi, ws, total = ref_candidates(x, mask, st, beam=beam, V=V, eot=eot, no_ts=no_ts, ts=ts,
                                       max_init=kw.get("max_initial_timestamp_index", 50))
        check_candidates(ci, cs, wi, ws, total, beam, (geom, name, beam))
        # what each layout is for
        if name == "hyp_tie":
            assert ci[0, 0] == eot and ci[0, 1] == V + eot and cs[0, 0] == cs[0, 1]
            assert got["n_hyp"][0] == 2 and list(got["best_tokens"][0, :3]) == list(st["seq"][st["flip"][0], 0, :3])
        if name.startswith("few_candidates") or name == "ts_gen0_few":
            assert (ci == -1).any(), name
        if name in ("few_candidates_gen0", "ts_gen0_few"):
            assert np.isneginf(got["cum"]).any() and (got["tokens"][np.isneginf(got["cum"])] == eot).all(), name
        if name == "few_candidates":
            assert got["n_hyp"][0] == beam and (got["tokens"] == eot).all()
        if name == "secondary_runs_out":
            assert got["n_hyp"][0] == beam and got["done"][0] == 1
        if name == "logit_ties":
            # equal scores: lowest flat id first, so row 0's ties come before the equal ones of row 1
            assert list(ci[0]) == (TIES[:2] if beam == 1 else TIES + [V + TIES[0]])
        n += 1
    assert n == 3 * 11 + 2 + 1


@pytest.mark.gpu
def test_hypothesis_tie_with_the_current_best(h):
    # a new hypothesis whose score equals the recorded best does not replace it (strict >: the first one wins)
    V, eot, no_ts = GEOMETRIES[0]
    mask = base_mask(V, eot)
    st = new_state(h, 1, 2, gen=3, V=V)
    x = rank_logits(V, 2, [(0, eot), (1, 900), (0, 901), (1, 902)])
    _, ci, cs, _ = h.debug_search_step_state(x, mask, st, beam=2, max_hyp=3, eot=eot, V=V)
    st["n_hyp"][0] = 1
    st["best_score"][0] = cs[0, 0]
    st["best_len"][0] = 2
    st["best_tokens"][0, :2] = (77, 78)
    got, want, _, _ = run_step(h, st, x, mask, beam=2, V=V, eot=eot, no_ts=no_ts, patience=1.5)
    compare(got, want, "tie")
    assert got["n_hyp"][0] == 2 and got["best_len"][0] == 2 and list(got["best_tokens"][0, :2]) == [77, 78]


@pytest.mark.gpu
@pytest.mark.parametrize("patience", [0.5, 1.0, 1.25, 2.0])
@pytest.mark.parametrize("lp", [0.0, 0.6, 1.0, 1.5])
def test_patience_and_length_penalty(h, patience, lp):
    # max_hyp = round-half-up(beam * patience); with max_hyp - 1 hypotheses recorded, one more finishes the utterance
    V, eot, no_ts = GEOMETRIES[0]
    mask = base_mask(V, eot)
    rng = np.random.default_rng(int(patience * 8 + lp * 10))
    for beam in (2, 5):
        max_hyp = max_hypotheses(beam, patience)
        for have in (max_hyp - 1, max(0, max_hyp - 2)):
            st = new_state(h, 3, beam, gen=4, rng=rng, V=V)
            st["n_hyp"][:] = have
            st["best_score"][:] = -0.9 if have else -np.inf
            st["best_len"][:] = 3 if have else 0
            x = np.concatenate([rank_logits(V, beam, [(0, eot)] + [(k % beam, TEXT[k]) for k in range(1, 2 * beam)])
                                for _ in range(3)])
            got, want, ci, cs = run_step(h, st, x, mask, beam=beam, V=V, eot=eot, no_ts=no_ts, patience=patience, lp=lp)
            compare(got, want, (patience, lp, beam, have))
            assert list(got["done"]) == [int(have + 1 >= max_hyp)] * 3


@pytest.mark.gpu
def test_per_utterance_caps(h):
    # caps 0, 1 and max_new at the first step: 0 finishes with no hypothesis, 1 turns every top candidate into one
    V, eot, no_ts = GEOMETRIES[0]
    mask = base_mask(V, eot)
    for beam in (1, 3):
        st = new_state(h, 4, beam, gen=0, pos=3, max_new=6, V=V)
        st["cum"][:] = 0
        x = np.concatenate([rank_logits(V, beam, [(0, TEXT[k]) for k in range(2 * beam)]) for _ in range(4)])
        caps = [0, 1, 6, 0]
        got, want, _, _ = run_step(h, st, x, mask, beam=beam, V=V, eot=eot, no_ts=no_ts, caps=caps)
        compare(got, want, ("caps", beam))
        assert list(got["done"]) == [1, 1, 0, 1] and list(got["n_hyp"]) == [0, beam, 0, 0]
        assert list(got["best_len"]) == [0, 1, 0, 0] and got["st"][3] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("n_utt,beam", [(1, 1), (64, 4), (1024, 1), (128, 8)])
def test_frozen_utterances_and_the_finishing_step(h, n_utt, beam):
    # frozen utterances between live ones are carried over bit for bit (indir[pos] = r); the step that finishes the
    # last utterance still advances pos / gen_step / flip / row_pos, sets all_done and leaves the ticket at 0
    V, eot, no_ts = GEOMETRIES[0]
    mask = base_mask(V, eot)
    rng = np.random.default_rng(n_utt + beam)
    R = n_utt * beam
    for last in (False, True):
        st = new_state(h, n_utt, beam, gen=5, max_new=6 if last else 9, rng=rng, V=V)
        st["done"][1::2] = 1
        st["st"][2] = int(st["done"].sum())
        x = rank_logits(V, R, [])
        x[:, :V] = rng.standard_normal((R, V)).astype(np.float32)
        got, want, ci, cs = run_step(h, st, x, mask, beam=beam, V=V, eot=eot, no_ts=no_ts)
        compare(got, want, (n_utt, beam, last))
        assert got["st"][4] == 0 and (got["st"][3] == 1 or not last)
        assert got["st"][0] == st["st"][0] + 1 and got["flip"][0] == st["flip"][0] ^ 1
        # a step on a finished search changes nothing at all
        if last:
            again, _, _, _ = h.debug_search_step_state(x, mask, got, beam=beam, max_hyp=beam, eot=eot, V=V)
            for k in got:
                assert np.array_equal(again[k], got[k]), k


@pytest.mark.gpu
def test_search_init_then_first_step(h):
    # the step straight after search initialisation from a prompt, with and without a shared prefix
    V, eot, no_ts = GEOMETRIES[0]
    mask = base_mask(V, eot)
    rng = np.random.default_rng(9)
    for shared in (0, 1):
        for n_utt, beam in ((3, 5), (2, 8), (5, 1)):
            prompt = rng.integers(0, 50000, (n_utt, 4))
            st = h.search_state(n_utt, beam, 10, 20)
            st["indir"][:] = 7 % (n_utt * beam)
            x = rank_logits(V, n_utt * beam, [])
            x[:, :V] = rng.standard_normal((n_utt * beam, V)).astype(np.float32)
            got, ci, cs, _ = h.debug_search_step_state(x, mask, st, beam=beam, max_hyp=beam, eot=eot, V=V, prompt=prompt,
                                                 shared_prefix=shared)
            init = h.search_state(n_utt, beam, 10, 20)
            init["st"][0] = 3 if shared else 0
            init["tokens"][:] = np.repeat(prompt[:, 3 if shared else 0], beam)
            init["row_pos"][:] = init["st"][0]
            slot = np.arange(n_utt * beam) // beam * beam if shared else np.arange(n_utt * beam)
            init["indir"][:] = slot[None, :, None]
            want = expected_step(init, ci, cs, beam=beam, V=V, eot=eot, max_hyp=beam, lp=1.0)
            compare(got, want, (shared, n_utt, beam))
            wi, ws, total = ref_candidates(x, mask, init, beam=beam, V=V, eot=eot)
            check_candidates(ci, cs, wi, ws, total, beam, (shared, n_utt, beam))


@pytest.mark.gpu
def test_repeat_is_bit_identical(h):
    V, eot, no_ts = GEOMETRIES[0]
    mask = base_mask(V, eot)
    rng = np.random.default_rng(4)
    st = new_state(h, 128, 8, gen=3, rng=rng, V=V)
    st["cum"][:] = rng.standard_normal(1024).astype(np.float32) - 3
    x = rank_logits(V, 1024, [])
    x[:, :V] = rng.standard_normal((1024, V)).astype(np.float32)
    a = h.debug_search_step_state(x, mask, st, beam=8, max_hyp=8, eot=eot, V=V)
    b = h.debug_search_step_state(x, mask, st, beam=8, max_hyp=8, eot=eot, V=V)
    for k in a[0]:
        assert np.array_equal(a[0][k], b[0][k]), k
    for p, q in zip(a[1:], b[1:]):
        assert np.array_equal(p, q)


# ------------------------------------------------------------------------------------------------------------- chains
def chain_logits(hist, seed, V, eot, no_ts, gen):
    """The raw logits of a row with generated tokens `hist`: seeded by the history, eot ramped up with the step."""
    key = zlib.crc32(np.asarray([seed] + list(hist), np.int64).tobytes())
    rng = np.random.default_rng(key)
    x = (rng.standard_normal(V) * 2.0).astype(np.float32)
    x[eot] = np.float32(-4.0 + 1.1 * gen + rng.standard_normal())
    x[no_ts + 1 :] -= np.float32(1.0)
    return x


def run_chain(h, seed, beam, ts, V, eot, no_ts, max_new=14):
    """Device steps from search initialisation to the end, each step checked against expected_step and every live
    row's indirection checked as a semantic property.  -> (device state, oracle BeamState, smallest decision gap)."""
    mask = base_mask(V, eot)
    R = beam
    st = h.search_state(1, beam, max_new, 3 + max_new)
    prompt = np.asarray([[50258, 50259, 50359]], np.int32)
    kw = dict(timestamps=bool(ts), no_timestamps=no_ts, max_initial_timestamp_index=6)
    H = []              # H[t][q]: the generated tokens of row q at step t
    s = 0
    while True:
        cur = int(st["flip"][0])
        hists = [list(st["seq"][cur, r, :s]) for r in range(R)]
        x = np.full((R, LDL), np.nan, np.float32)
        for r in range(R):
            x[r, :V] = chain_logits(hists[r], seed, V, eot, no_ts, s)
        H.append(hists)
        got, ci, cs, _ = h.debug_search_step_state(x, mask, st, beam=beam, max_hyp=beam, eot=eot, V=V,
                                             prompt=prompt if s == 0 else None, shared_prefix=1, **kw)
        if s == 0:
            init = h.search_state(1, beam, max_new, 3 + max_new)
            init["st"][0] = 2
            init["tokens"][:] = 50359
            init["row_pos"][:] = 2
            init["indir"][:] = 0
            st = init
        compare(got, expected_step(st, ci, cs, beam=beam, V=V, eot=eot, max_hyp=beam, lp=1.0), (seed, beam, ts, s))
        # indirection: slot indir[r][2 + t] fed row r's own ancestor at step t (the same generated prefix)
        nxt = int(got["flip"][0])
        for r in range(R):
            if not np.isfinite(got["cum"][r]):
                continue
            hr = list(got["seq"][nxt, r, : s + 1])
            for t in range(s + 1):
                q = int(got["indir"][nxt, r, 2 + t])
                assert H[t][q] == hr[:t], (seed, beam, ts, s, r, t)
            assert (got["indir"][nxt, r, :2] == 0).all()
        st = got
        s += 1
        if st["st"][3]:
            break

    def logits_fn(step, tokens, parents):
        if step == 0:
            logits_fn.hist = [[] for _ in range(beam)]
        else:
            logits_fn.hist = [logits_fn.hist[p] + [t] for p, t in zip(parents, tokens)]
        return torch.from_numpy(np.stack([chain_logits(hh, seed, V, eot, no_ts, step) for hh in logits_fn.hist]))

    def process(logits, hists, step):
        x = processed(logits.numpy()[:, :V], mask, hists, step, V, eot, no_ts, ts, 6)
        return x.float()

    trace = []
    want = beam_search(logits_fn, process, beam=beam, V=V, eot=eot, max_new=max_new, max_hyp=beam, length_penalty=1.0,
                       trace=trace)
    return st, want, min(trace)


@pytest.mark.gpu
@pytest.mark.parametrize("beam", [1, 2, 5, 8])
@pytest.mark.parametrize("ts", [0, 1])
def test_chains_end_where_the_oracle_loop_ends(h, beam, ts):
    V, eot, no_ts = GEOMETRIES[0]
    clear = 0
    for seed in range(4):
        st, want, gap = run_chain(h, seed, beam, ts, V, eot, no_ts)
        if gap > 1e-4:
            assert st["n_hyp"][0] == len(want.hyps), (seed, beam, ts)
            assert list(st["best_tokens"][0, : st["best_len"][0]]) == want.best_tokens, (seed, beam, ts)
            assert abs(st["best_score"][0] - want.best_score) <= 1e-4, (seed, beam, ts)
            clear += 1
    assert clear >= 2, clear


# --------------------------------------------------------------------------------------------- the comparator (no GPU)
@pytest.mark.parametrize("defect", DEFECTS)
def test_comparator_rejects_injected_defects(defect):
    # the crafted steps, with float64 candidates standing in for the device's, separate the oracle step from each
    # defective one somewhere
    V, eot, no_ts = GEOMETRIES[0]
    caught = 0
    for name, beam, st, x, mask, kw in crafted(_lib.Handle, V, eot):
        ts = kw.get("timestamps", False)
        wi, ws, _ = ref_candidates(x, mask, st, beam=beam, V=V, eot=eot, no_ts=no_ts, ts=ts,
                                   max_init=kw.get("max_initial_timestamp_index", 50))
        cs = ws.astype(np.float32)
        good = expected_step(st, wi, cs, beam=beam, V=V, eot=eot, max_hyp=beam, lp=1.0)
        bad = expected_step(st, wi, cs, beam=beam, V=V, eot=eot, max_hyp=beam, lp=1.0, defect=defect)
        try:
            compare(bad, good)
        except AssertionError:
            caught += 1
    assert caught >= 1, defect


def test_oracle_step_rules():
    # the rules the oracle step pins (engine side: search.cu, wisb_generate with timestamps)
    assert [max_hypotheses(5, 0.5), max_hypotheses(2, 1.25), max_hypotheses(5, 2.0), max_hypotheses(1, 0.1)] == [3, 3, 10, 1]
    V, eot = 100, 99
    st = BeamState([[1], [2]], [-1.0, -2.0])
    # a missing candidate: the row is dead (eot, -inf) and never a hypothesis, even at the last step
    new = beam_step(st, [5, 106, -1, -1], [-0.5, -0.7, NEG, NEG], V=V, eot=eot, gen=1, cap=2, max_hyp=5, norm=2.0)
    assert len(new.hyps) == 2 and new.finished
    new = beam_step(st, [5, -1, -1, -1], [-0.5, NEG, NEG, NEG], V=V, eot=eot, gen=1, cap=9, max_hyp=5, norm=2.0)
    assert new.tokens == [5, eot] and new.cum[1] == NEG and new.parents == [0, 1] and not new.hyps
    # a cap of 0 new tokens: finished at once, no hypothesis
    new = beam_step(st, [5, 106, 7, 8], [-0.5, -0.7, -0.8, -0.9], V=V, eot=eot, gen=0, cap=0, max_hyp=5, norm=1.0)
    assert new.finished and not new.hyps
