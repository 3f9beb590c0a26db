"""The device token search one step at a time with a beam, patience and length penalty of each utterance's own
(``wisb_debug_search_step`` with beam_u / max_hyp_u / length_penalty_u, the search of ``wisb_generate`` with per-window
options).

Every utterance keeps a block of B rows (B = the largest beam of the call) and searches its first b_u of them.  The step
must equal, utterance by utterance, the oracle's ``beam_step`` at that utterance's own beam, max_hyp and length penalty
(integers exact, cum / best_score within the 4-ulp bound of tests/test_gpu_search.py), its candidate list must match
float64 wherever float64 has no near-tie, and the surplus rows must stay dead: cum -inf, token eot, never in the
candidate list, never a hypothesis."""
import numpy as np
import pytest

from oracle.whisper_ref import BeamState, beam_step, max_hypotheses
from tests.test_gpu_search import (GEOMETRIES, NEG, TEXT, base_mask, check_candidates, compare, fp32_norm, new_state,
                                   rank_logits, ref_candidates)
from willow_inference_server_b200 import _lib

pytestmark = pytest.mark.gpu


def expected_mixed(st, ci, cs, *, B, beams, hyps, lps, V, eot, caps=None):
    """The device state after one step: oracle beam_step per utterance at its own (beam, max_hyp, length penalty) on
    its first beams[u] rows; the other rows carried over dead (eot, cum -inf, own slot at pos)."""
    out = {k: v.copy() for k, v in st.items()}
    pos, gen, _, all_done, _ = (int(x) for x in st["st"])
    if all_done:
        return out
    n_utt = len(st["done"])
    max_new = st["seq"].shape[2]
    cur = int(st["flip"][0])
    nxt = cur ^ 1
    for u in range(n_utt):
        if st["done"][u]:
            for r in range(u * B, (u + 1) * B):
                out["seq"][nxt, r] = st["seq"][cur, r]
                out["indir"][nxt, r] = st["indir"][cur, r]
                out["indir"][nxt, r, pos] = r
            continue
        b = int(beams[u])
        rows = range(u * B, u * B + b)
        n_hyp, best = int(st["n_hyp"][u]), float(st["best_score"][u])
        hyps_ = [(NEG, [])] * n_hyp
        if best > NEG and n_hyp:
            hyps_[0] = (best, list(st["best_tokens"][u, : st["best_len"][u]]))
        prev = BeamState([list(st["seq"][cur, r, :gen]) for r in rows], [float(st["cum"][r]) for r in rows],
                         hyps=hyps_, best=0 if best > NEG and n_hyp else -1)
        cap = int(caps[u]) if caps is not None else max_new
        new = beam_step(prev, [int(i) for i in ci[u, : 2 * b]], [float(s) for s in cs[u, : 2 * b]], V=V, eot=eot, gen=gen,
                        cap=cap, max_hyp=int(hyps[u]), norm=fp32_norm(gen, float(np.float32(lps[u]))))
        out["n_hyp"][u] = len(new.hyps)
        out["best_score"][u] = new.best_score
        if new.best != prev.best:
            toks = new.best_tokens
            out["best_tokens"][u, : len(toks)] = toks
            out["best_len"][u] = len(toks)
        for k, r in enumerate(rows):
            pr = u * B + new.parents[k]
            out["seq"][nxt, r, : gen + 1] = new.seqs[k][:max_new]
            out["indir"][nxt, r, :pos] = st["indir"][cur, pr, :pos]
            out["indir"][nxt, r, pos] = pr
            out["tokens"][r] = new.tokens[k]
            out["cum"][r] = new.cum[k]
        for r in range(u * B + b, (u + 1) * B):
            out["seq"][nxt, r, :gen] = st["seq"][cur, r, :gen]
            if gen < max_new:
                out["seq"][nxt, r, gen] = eot
            out["indir"][nxt, r, :pos] = st["indir"][cur, r, :pos]
            out["indir"][nxt, r, pos] = r
            out["tokens"][r] = eot
            out["cum"][r] = NEG
        if new.finished:
            out["done"][u] = 1
            out["st"][2] += 1
    out["st"][0] += 1
    out["st"][1] += 1
    out["st"][3] = int(out["st"][2] == n_utt)
    out["flip"][0] = nxt
    out["row_pos"] += 1
    return out


def check_dead_and_candidates(st, got, ci, cs, x, mask, *, B, beams, lps, V, eot, no_ts=0, ts=False, max_init=50,
                              proc=None, where="", ref_every=1):
    """Surplus rows dead, candidate lists of live utterances == float64 (near-ties aside; every ref_every-th utterance),
    padding entries none."""
    for u, b in enumerate(beams):
        b = int(b)
        dead = slice(u * B + b, (u + 1) * B)
        if not st["done"][u]:
            assert (got["tokens"][dead] == eot).all() and np.isneginf(got["cum"][dead]).all(), (where, u)
        valid = ci[u] >= 0
        assert (ci[u, 2 * b :] == -1).all() and np.isneginf(cs[u, 2 * b :]).all(), (where, u, ci[u])
        assert (ci[u][valid] // V < b).all(), (where, u, ci[u])      # never a candidate from a dead row
        if st["done"][u] or proc or u % ref_every:
            continue
        rows = slice(u * B, u * B + b)
        sub = {"st": st["st"], "flip": st["flip"], "seq": st["seq"][:, rows], "cum": st["cum"][rows],
               "done": np.zeros(1, np.int32)}
        wi, ws, total = ref_candidates(x[rows], mask, sub, beam=b, V=V, eot=eot, no_ts=no_ts, ts=ts, max_init=max_init,
                                       lp=float(np.float32(lps[u])))
        check_candidates(ci[u : u + 1], cs[u : u + 1], wi, ws, total, b, (where, u))


def run_mixed(h, st, x, mask, *, B, beams, patience, lps, V, eot, no_ts, caps=None, check_ref=True, **kw):
    beams = np.asarray(beams, np.int32)
    hyps = np.asarray([max_hypotheses(int(b), float(p)) for b, p in zip(beams, patience)], np.int32)
    lps = np.asarray(lps, np.float32)
    got, ci, cs, lse = h.debug_search_step_state(x, mask, st, beam=B, max_hyp=1, eot=eot, V=V, no_timestamps=no_ts,
                                                 max_new_u=caps, beam_u=beams, max_hyp_u=hyps, length_penalty_u=lps, **kw)
    want = expected_mixed(st, ci, cs, B=B, beams=beams, hyps=hyps, lps=lps, V=V, eot=eot, caps=caps)
    if check_ref:
        check_dead_and_candidates(st, got, ci, cs, x, mask, B=B, beams=beams, lps=lps, V=V, eot=eot, no_ts=no_ts,
                                  ts=kw.get("timestamps", False), max_init=kw.get("max_initial_timestamp_index", 50),
                                  proc=kw.get("repetition_penalty") or kw.get("no_repeat_ngram_size"))
    return got, want, ci, cs


def dead_state(st, B, beams, eot):
    """A mid-search state whose surplus rows are what search_init and every later step leave there."""
    for u, b in enumerate(beams):
        st["cum"][u * B + b : (u + 1) * B] = NEG
        st["tokens"][u * B + b : (u + 1) * B] = eot
    return st


def layout(kind, b, eot, u):
    """(row within the utterance, token) ranks of one utterance's candidates: eot at rank 0, at rank b - 1, at several
    ranks, or only below rank b"""
    T = lambda k: TEXT[(k + 7 * u) % len(TEXT)]  # noqa: E731
    if kind == 0:
        return [(0, eot)] + [(k % b, T(k)) for k in range(1, 2 * b)]
    if kind == 1:
        return [(k % b, T(k)) for k in range(b - 1)] + [(1 % b, eot)] + [(k % b, T(k)) for k in range(b, 2 * b)]
    if kind == 2:
        return [(k, eot) if k % 2 == 0 else (k, T(k)) for k in range(b)] + [(k % b, T(k + 50)) for k in range(b)]
    return [(k % b, T(k)) for k in range(b)] + [(0, eot)] + [(k % b, T(k + 50)) for k in range(b - 1)]


def mixed_logits(V, B, beams, kinds, eot):
    """Logits [n_utt * B, LDL]: each utterance's searched rows ranked by layout(kind); its dead rows get the largest
    logits of all (a merge that read them would pick them)."""
    x = rank_logits(V, len(beams) * B, [])
    for u, (b, kind) in enumerate(zip(beams, kinds)):
        blk = rank_logits(V, b, layout(kind, b, eot, u))
        x[u * B : u * B + b] = blk
        if b < B:
            x[u * B + b : (u + 1) * B, :V] = 0.0
            x[u * B + b : (u + 1) * B, TEXT[3]] = 9.0
            x[u * B + b : (u + 1) * B, eot] = 8.5
    return x


@pytest.fixture(scope="module")
def h():
    return _lib.Handle.frontend(0)


BEAM_SETS = [(1, 8), (8, 1, 1, 8), (1, 2, 3, 4, 5, 6, 7, 8), (3, 5, 2), (1, 1, 1, 1)]   # (the last at B = 8: all b = 1)


@pytest.mark.parametrize("geom", range(3))
def test_mixed_beams_eot_ranks_and_last_step(h, geom):
    V, eot, no_ts = GEOMETRIES[geom]
    mask = base_mask(V, eot)
    rng = np.random.default_rng(geom)
    n = 0
    for beams in BEAM_SETS:
        B = 8 if beams == (1, 1, 1, 1) else max(beams)
        for kind in range(4):
            kinds = [(kind + u) % 4 for u in range(len(beams))]
            for max_new in (9, 4):              # mid-search and the last step (gen 3 = max_new - 1)
                st = dead_state(new_state(h, len(beams), B, gen=3, max_new=max_new, rng=rng, V=V), B, beams, eot)
                patience = [1.0] * len(beams)
                lps = [(0.0, 0.6, 1.0, 1.5)[u % 4] for u in range(len(beams))]
                x = mixed_logits(V, B, beams, kinds, eot)
                got, want, ci, cs = run_mixed(h, st, x, mask, B=B, beams=beams, patience=patience, lps=lps, V=V, eot=eot,
                                              no_ts=no_ts)
                compare(got, want, (geom, beams, kind, max_new))
                if max_new == 4:
                    assert got["done"].all(), (beams, kind)
                n += 1
    assert n == len(BEAM_SETS) * 8


def test_fewer_candidates_than_2b(h):
    # only <|endoftext|> unmasked: each searched row has one candidate, so the list ends in none (-1) entries; the dead
    # rows, whose eot is as finite as any, must not fill them
    V, eot, no_ts = GEOMETRIES[0]
    mask = base_mask(V, eot)
    mask[:] |= 1
    mask[eot] = 0
    rng = np.random.default_rng(6)
    for beams in ((1, 8), (2, 5, 1), (1, 1, 1, 1)):
        B = 8 if beams == (1, 1, 1, 1) else max(beams)
        st = dead_state(new_state(h, len(beams), B, gen=2, rng=rng, V=V), B, beams, eot)
        x = rank_logits(V, len(beams) * B, [])
        x[:, :V] = rng.standard_normal((len(beams) * B, V)).astype(np.float32)
        got, want, ci, _ = run_mixed(h, st, x, mask, B=B, beams=beams, patience=[2.0] * len(beams),
                                     lps=[1.0] * len(beams), V=V, eot=eot, no_ts=no_ts)
        compare(got, want, ("few", beams))
        for u, b in enumerate(beams):
            assert (ci[u, :b] % V == eot).all() and (ci[u, b:] == -1).all(), (beams, u, ci[u])


def test_patience_gives_every_max_hyp(h):
    # max_hyp from 1 to 2 b (patience 0.1 .. 2): with max_hyp - 1 hypotheses recorded, one more finishes the utterance
    V, eot, no_ts = GEOMETRIES[0]
    mask = base_mask(V, eot)
    rng = np.random.default_rng(3)
    beams = (1, 2, 3, 5, 8)
    B = 8
    for patience in (0.1, 0.5, 1.0, 1.25, 2.0):
        hyps = [max_hypotheses(b, patience) for b in beams]
        for lag in (1, 2):
            st = dead_state(new_state(h, len(beams), B, gen=4, rng=rng, V=V), B, beams, eot)
            have = [max(0, m - lag) for m in hyps]
            st["n_hyp"][:] = have
            st["best_score"][:] = [-0.9 if k else NEG for k in have]
            st["best_len"][:] = [3 if k else 0 for k in have]
            x = mixed_logits(V, B, beams, [0] * len(beams), eot)
            got, want, _, _ = run_mixed(h, st, x, mask, B=B, beams=beams, patience=[patience] * len(beams),
                                        lps=[1.0] * len(beams), V=V, eot=eot, no_ts=no_ts)
            compare(got, want, (patience, lag))
            assert list(got["done"]) == [int(k + 1 >= m) for k, m in zip(have, hyps)], (patience, lag)
    for b in beams:   # every beam from max_hyp 1 to 2 b
        got_range = [max_hypotheses(b, p) for p in (0.1, 0.5, 1.0, 1.25, 2.0)]
        assert min(got_range) == 1 and max(got_range) == 2 * b


def test_per_window_patience_and_length_penalty_in_one_call(h):
    # the same beam for every utterance, patience and length penalty different per utterance
    V, eot, no_ts = GEOMETRIES[0]
    mask = base_mask(V, eot)
    rng = np.random.default_rng(8)
    beams = (4, 4, 4, 4)
    patience = (0.5, 1.0, 1.5, 2.0)
    lps = (0.0, 0.5, 1.0, 2.0)
    st = dead_state(new_state(h, 4, 4, gen=6, rng=rng, V=V), 4, beams, eot)
    st["cum"][:] = rng.uniform(-9, -2, 16).astype(np.float32)
    st["n_hyp"][:] = [1, 3, 5, 7]
    st["best_score"][:] = -0.9
    st["best_len"][:] = 2
    x = rank_logits(V, 16, [])
    x[:, :V] = rng.standard_normal((16, V)).astype(np.float32)
    x[:, eot] += 3.0
    got, want, _, _ = run_mixed(h, st, x, mask, B=4, beams=beams, patience=patience, lps=lps, V=V, eot=eot, no_ts=no_ts)
    compare(got, want, "patience_lp")


def test_search_init_makes_surplus_rows_dead(h):
    V, eot, no_ts = GEOMETRIES[0]
    mask = base_mask(V, eot)
    rng = np.random.default_rng(9)
    for shared in (0, 1):
        for beams in ((1, 8), (2, 1, 3), (1, 1, 1)):
            B = 8 if beams == (1, 1, 1) else max(beams)
            n_utt, R = len(beams), len(beams) * B
            prompt = rng.integers(0, 50000, (n_utt, 4))
            st = h.search_state(n_utt, B, 10, 20)
            x = rank_logits(V, R, [])
            x[:, :V] = rng.standard_normal((R, V)).astype(np.float32)
            got, ci, cs, _ = h.debug_search_step_state(
                x, mask, st, beam=B, max_hyp=1, eot=eot, V=V, prompt=prompt, shared_prefix=shared,
                beam_u=np.asarray(beams), max_hyp_u=np.asarray(beams), length_penalty_u=np.ones(n_utt, np.float32))
            init = h.search_state(n_utt, B, 10, 20)
            init["st"][0] = 3 if shared else 0
            init["tokens"][:] = np.repeat(prompt[:, 3 if shared else 0], B)
            init["row_pos"][:] = init["st"][0]
            slot = np.arange(R) // B * B if shared else np.arange(R)
            init["indir"][:] = slot[None, :, None]
            dead_state(init, B, beams, eot)
            want = expected_mixed(init, ci, cs, B=B, beams=beams, hyps=beams, lps=[1.0] * n_utt, V=V, eot=eot)
            compare(got, want, (shared, beams))
            check_dead_and_candidates(init, got, ci, cs, x, mask, B=B, beams=beams, lps=[1.0] * n_utt, V=V, eot=eot,
                                      where=(shared, beams))


def test_timestamp_mode(h):
    # gen 0 with a low max_initial_timestamp_index (fewer candidates than 2 b), then a mid-search step
    V, eot, no_ts = GEOMETRIES[0]
    mask = base_mask(V, eot)
    rng = np.random.default_rng(11)
    beams = (1, 5, 3, 8)
    B = 8
    kw = dict(timestamps=True, max_initial_timestamp_index=3)
    st = dead_state(new_state(h, 4, B, gen=0, pos=2, rng=rng, V=V), B, beams, eot)
    st["cum"][[u * B + k for u, b in enumerate(beams) for k in range(b)]] = 0
    x = rank_logits(V, 4 * B, [])
    x[:, :V] = rng.standard_normal((4 * B, V)).astype(np.float32)
    got, want, ci, _ = run_mixed(h, st, x, mask, B=B, beams=beams, patience=[1.0] * 4, lps=[1.0, 0.5, 0.0, 1.2], V=V,
                                 eot=eot, no_ts=no_ts, **kw)
    compare(got, want, "ts_gen0")
    assert (ci[1] == -1).any()   # 4 timestamps for 10 candidates
    # a mid-search step: histories end in text, a lone timestamp and a timestamp pair
    st = dead_state(new_state(h, 4, B, gen=4, rng=rng, V=V), B, beams, eot)
    cur = int(st["flip"][0])
    st["seq"][cur, :, :4] = [1000, 1001, 1002, 1003]
    st["seq"][cur, 8:16, 3] = no_ts + 20
    st["seq"][cur, 16:24, 2:4] = no_ts + 20
    st["cum"][:] = np.where(np.isneginf(st["cum"]), NEG, -2.0)
    x = rank_logits(V, 4 * B, [])
    x[:, :V] = rng.standard_normal((4 * B, V)).astype(np.float32)
    x[:, no_ts + 1 :] += 1.5
    got, want, _, _ = run_mixed(h, st, x, mask, B=B, beams=beams, patience=[1.0, 2.0, 0.5, 1.0], lps=[1.0] * 4, V=V,
                                eot=eot, no_ts=no_ts, **kw)
    compare(got, want, "ts_mid")


def test_history_processors_and_caps(h):
    V, eot, no_ts = GEOMETRIES[0]
    mask = base_mask(V, eot)
    rng = np.random.default_rng(12)
    beams = (2, 1, 6, 3)
    B = 6
    st = dead_state(new_state(h, 4, B, gen=5, max_new=9, rng=rng, V=V), B, beams, eot)
    cur = int(st["flip"][0])
    st["seq"][cur, :, :5] = rng.integers(1000, 1010, (4 * B, 5))
    x = rank_logits(V, 4 * B, [])
    x[:, :V] = rng.standard_normal((4 * B, V)).astype(np.float32)
    x[:, 1000:1010] += 4.0   # the history tokens lead before the processors act
    got, want, ci, _ = run_mixed(h, st, x, mask, B=B, beams=beams, patience=[1.0] * 4, lps=[1.0] * 4, V=V, eot=eot,
                                 no_ts=no_ts, repetition_penalty=1.7, no_repeat_ngram_size=2)
    compare(got, want, "processors")
    # per-utterance caps 0, 1 and max_new at the first step
    st = dead_state(new_state(h, 4, B, gen=0, pos=3, max_new=6, V=V), B, beams, eot)
    st["cum"][[u * B + k for u, b in enumerate(beams) for k in range(b)]] = 0
    x = mixed_logits(V, B, beams, [3, 3, 3, 3], eot)
    caps = [0, 1, 6, 1]
    got, want, _, _ = run_mixed(h, st, x, mask, B=B, beams=beams, patience=[1.0] * 4, lps=[1.0] * 4, V=V, eot=eot,
                                no_ts=no_ts, caps=caps)
    compare(got, want, "caps")
    assert list(got["done"]) == [1, 1, 0, 1] and list(got["n_hyp"]) == [0, 1, 0, 3]


@pytest.mark.parametrize("B", [8, 2])
def test_1024_rows_with_frozen_utterances(h, B):
    V, eot, no_ts = GEOMETRIES[0]
    mask = base_mask(V, eot)
    rng = np.random.default_rng(B)
    n_utt = 1024 // B
    beams = rng.integers(1, B + 1, n_utt)
    beams[:2] = (1, B)
    st = dead_state(new_state(h, n_utt, B, gen=5, max_new=9, rng=rng, V=V), B, beams, eot)
    st["done"][3::4] = 1
    st["st"][2] = int(st["done"].sum())
    live = np.isfinite(st["cum"])
    st["cum"][live] = rng.uniform(-6, -1, int(live.sum())).astype(np.float32)
    x = rank_logits(V, 1024, [])
    x[:, :V] = rng.standard_normal((1024, V)).astype(np.float32)
    patience = rng.choice([0.5, 1.0, 2.0], n_utt)
    lps = rng.choice([0.0, 1.0, 0.7], n_utt)
    got, want, ci, cs = run_mixed(h, st, x, mask, B=B, beams=beams, patience=patience, lps=lps, V=V, eot=eot,
                                  no_ts=no_ts, check_ref=False)
    compare(got, want, ("1024", B))
    check_dead_and_candidates(st, got, ci, cs, x, mask, B=B, beams=beams, lps=lps, V=V, eot=eot, where=("1024", B),
                              ref_every=max(1, n_utt // 16))


def test_one_beam_for_all_equals_the_scalar_search(h):
    # every utterance at the same beam B, patience and length penalty: the per-utterance search is the scalar one
    V, eot, no_ts = GEOMETRIES[0]
    mask = base_mask(V, eot)
    rng = np.random.default_rng(21)
    for B in (1, 5, 8):
        st = new_state(h, 6, B, gen=3, rng=rng, V=V)
        st["cum"][:] = rng.uniform(-5, -1, 6 * B).astype(np.float32)
        x = rank_logits(V, 6 * B, [])
        x[:, :V] = rng.standard_normal((6 * B, V)).astype(np.float32)
        x[:, eot] += 2.5
        a = h.debug_search_step_state(x, mask, st, beam=B, max_hyp=B, eot=eot, V=V, length_penalty=0.8)
        b = h.debug_search_step_state(x, mask, st, beam=B, max_hyp=1, eot=eot, V=V, beam_u=[B] * 6, max_hyp_u=[B] * 6,
                                      length_penalty_u=[0.8] * 6)
        for k in a[0]:
            assert np.array_equal(a[0][k], b[0][k]), (B, k)
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3])


def test_bad_per_utterance_arguments(h):
    V, eot, _ = GEOMETRIES[0]
    mask = base_mask(V, eot)
    st = new_state(h, 2, 4, gen=2, V=V)
    x = rank_logits(V, 8, [])
    ok = dict(beam_u=[4, 2], max_hyp_u=[4, 2], length_penalty_u=[1.0, 1.0])
    h.debug_search_step_state(x, mask, st, beam=4, max_hyp=1, eot=eot, V=V, **ok)
    for bad in (dict(beam_u=[5, 2]), dict(beam_u=[0, 2]), dict(max_hyp_u=[0, 2]),
                dict(length_penalty_u=[np.inf, 1.0]), dict(length_penalty_u=[1.0, np.nan])):
        with pytest.raises(ValueError):
            h.debug_search_step_state(x, mask, st, beam=4, max_hyp=1, eot=eot, V=V, **{**ok, **bad})
    with pytest.raises(ValueError):  # all three or none
        h.debug_search_step_state(x, mask, st, beam=4, max_hyp=1, eot=eot, V=V, beam_u=[4, 2], max_hyp_u=[4, 2])
