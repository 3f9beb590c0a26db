"""GPU: the no-speech probability of every window (wisb_get_no_speech_probs, Whisper.generate's no_speech_prob).

  * Kernel: the reduction on caller rows (Handle.debug_no_speech_probs) against float64 at V = 51864, 51865 and 51866,
    with NaN in every padding column: spreads of +-1e4, -inf entries, the no-speech logit as the maximum, an all-equal
    row (1 / V), skipped windows.
  * End to end against the oracle: softmax in float64 of WhisperOracle.forced_logits(enc, prompt[:s + 1])[s] at
    <|nospeech|>, s = the prompt's first <|startoftranscript|>, within |d log p| <= 2 LOGIT_TOL.  On the peaked tiny
    model and on a variant whose <|nospeech|> embedding row copies the oracle's most likely token at the SOT position
    (p large; <|nospeech|> is suppressed and never an input, so decoding is unchanged).  Every prefill mode: fused,
    the one-pass prefix with logits, the wide prefill with the gather, one pass per position, the 8-position batched
    chunks, s = P - 1 read from the first step's pass, windows with different s in one call, on the warp-MMA, SIMT and
    batched passes, with greedy, beam 5, per-window beams, timestamps and best-of-5 sampling, max_length leaving 0 new
    tokens, and more windows than one group.
  * Each such call returns ids, lengths and scores bit-identical to the call without the request, with equal
    decode_steps.
  * faster-whisper's sequence: Whisper.encode -> generate(enc, return_no_speech_prob=True) gives the features call's
    values, and permuting the windows permutes them."""
import functools

import numpy as np
import pytest

from oracle.whisper_ref import WhisperOracle
from tests.gpu_common import LOGIT_TOL, PROMPT, RAMP, SCRIPT, mel_inputs
from willow_inference_server_b200 import _lib, models, weights as W

pytestmark = pytest.mark.gpu

SOT, SOT_PREV, LANG, TASK = 50258, 50361, 50259, 50359
TS_SCRIPT = (2, 5, 8)


# ------------------------------------------------------------------------------------------------ kernel
def ref_no_speech(row, ns):
    x = row.astype(np.float64)
    m = x.max()
    return float(np.exp(x[ns] - m) / np.exp(x - m).sum())


@pytest.mark.parametrize("V", [51864, 51865, 51866])
def test_reduction_kernel_against_float64(V):
    _, _, h = model(False)
    ldl = -(-V // 128) * 128
    ns = 50362
    rng = np.random.default_rng(V)
    rows = [rng.standard_normal(V) * 4]
    wide = rng.uniform(-1e4, 1e4, V)
    wide[ns] = wide.max() - 5.0
    rows.append(wide)
    rows.append(rng.uniform(-1e4, 1e4, V))
    inf = rng.standard_normal(V) * 3
    inf[rng.choice(V, 500, replace=False)] = -np.inf
    inf[ns] = 1.0
    rows.append(inf)
    top = rng.standard_normal(V)
    top[ns] = top.max() + 0.5
    rows.append(top)
    rows.append(np.full(V, 3.25))
    low = rng.standard_normal(V) * 2
    low[ns] = -40.0
    rows.append(low)
    lg = np.full((len(rows), ldl), np.nan, np.float32)
    for i, r in enumerate(rows):
        lg[i, :V] = r
    order = np.asarray([3, 0, 5, 1, -1, 6, 2, 4, -1], np.int32)
    sentinel = np.full(order.size, 7.5, np.float32)
    got = h.debug_no_speech_probs(lg, order, V, ns, out=sentinel)
    for u, r in enumerate(order):
        if r < 0:
            assert got[u] == 7.5, (V, u)
            continue
        want = ref_no_speech(lg[r, :V], ns)
        if want > 1e-30:
            assert abs(got[u] - want) <= 1e-5 * want, (V, u, r, got[u], want)
        else:
            assert got[u] <= 1e-29, (V, u, r, got[u], want)
    assert abs(got[2] - 1.0 / V) <= 1e-5 / V


# ------------------------------------------------------------------------------------------------ models
@functools.lru_cache(maxsize=2)
def model(variant):
    """(dims, oracle, handle) of the peaked tiny model; variant: <|nospeech|>'s embedding row copies the oracle's most
    likely token at the SOT position of window 0"""
    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=2)
    tensors = W.synth_engine_tensors(dims, seed=11, eot_ramp=RAMP, script=SCRIPT, ts_script=TS_SCRIPT)
    if variant:
        _, base, _ = model(False)
        top = int(base.forced_logits(base.encode(mel_inputs(16)[:1])[0], [SOT])[0].argmax())
        emb = tensors["dec.tok_emb"].copy()
        emb[dims.no_speech] = emb[top]
        tensors = dict(tensors)
        tensors["dec.tok_emb"] = emb
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    return dims, WhisperOracle.from_blob(buf), _lib.Handle.from_host(buf, 0)


@functools.lru_cache(maxsize=None)
def encoded(variant, w):
    _, oracle, _ = model(variant)
    return oracle.encode(mel_inputs(16)[w : w + 1])[0]


@functools.lru_cache(maxsize=None)
def oracle_log_p(variant, w, prompt):
    dims, oracle, _ = model(variant)
    s = prompt.index(SOT)
    lg = oracle.forced_logits(encoded(variant, w), list(prompt[: s + 1]))[s].double().numpy()
    m = lg.max()
    return float(lg[dims.no_speech] - m - np.log(np.exp(lg - m).sum()))


def make_prompt(s, P, seed):
    """P tokens whose first <|startoftranscript|> is at s: [<|startofprev|>, text ...] before it, then language and task
    (and text) after it"""
    rng = np.random.default_rng(seed)
    p = [int(t) for t in rng.integers(400, 9000, P)]
    if s > 0:
        p[0] = SOT_PREV
    p[s] = SOT
    for i, t in enumerate((LANG, TASK)):
        if s + 1 + i < P:
            p[s + 1 + i] = t
    return p


# case -> (windows' first-sot positions, prompt length, beams, timestamps, sampling)
CASES = {
    "fused_beam5": ([0], 4, [5], False, False),
    "prefix_2x5_greedy": ([2, 2], 5, [1], False, False),
    "sot_last_3x3": ([2, 2, 2], 3, [1], False, False),
    "mixed_s_beams": ([11, 13, 2], 14, [2, 1, 2], False, False),
    "long_beam5": ([224], 227, [5], False, False),
    "timestamps": ([0, 0], 3, [2, 1], True, False),
    "sample_best_of_5": ([0], 4, [5], False, True),
    "sample_long": ([11], 14, [5], False, True),
}
PATHS = ["warp_mma", "simt", "batched"]


def set_path(h, path, wide):
    h.set_option("mega_mma", 0 if path == "simt" else 1)
    h.set_option("decoder_batch", 2 if path == "batched" else 1)
    h.set_option("wide_prefill", wide)


def reset(h):
    for k, v in (("mega_mma", 1), ("decoder_batch", 1), ("wide_prefill", 1), ("batch_rows", 320)):
        h.set_option(k, v)


def f32bits(x):
    return np.asarray(x, np.float32).view(np.uint32).tolist()


def call(h, mel, prompts, beams, ts, sampling, max_length, ns=None):
    """-> (ids, score bits, decode_steps)"""
    if sampling:
        seeds = np.arange(40, 40 + len(prompts), dtype=np.uint64)
        ids, scores = h.generate_sample(mel, prompts, beams[0], 0, 0.8, seeds, max_length=max_length, timestamps=ts,
                                        no_speech_out=ns)
        return ids, [f32bits(s) for s in scores], h.timing()["decode_steps"]
    b = beams[0] if len(set(beams)) == 1 else np.asarray(beams, np.int32)
    ids, scores = h.generate(mel, prompts, b, max_length=max_length, timestamps=ts, no_speech_out=ns)
    return ids, f32bits(scores), h.timing()["decode_steps"]


def check(variant, h, windows, prompts, beams, *, ts=False, sampling=False, max_length=448, tag=()):
    """the call with and without the request: identical results and passes; the values against the oracle"""
    mel = np.ascontiguousarray(mel_inputs(16)[windows])
    p = np.asarray(prompts, np.int32)
    plain = call(h, mel, p, beams, ts, sampling, max_length)
    ns = np.full(len(windows), -1.0, np.float32)
    asked = call(h, mel, p, beams, ts, sampling, max_length, ns)
    assert plain == asked, tag
    for i, w in enumerate(windows):
        want = oracle_log_p(variant, int(w), tuple(int(t) for t in prompts[i]))
        assert ns[i] > 0 and abs(np.log(ns[i]) - want) <= 2 * LOGIT_TOL, (tag, i, float(ns[i]), np.exp(want))
    return ns


@pytest.mark.parametrize("variant", [False, True])
@pytest.mark.parametrize("wide", [1, 0])
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("case", list(CASES))
def test_end_to_end_against_the_oracle(case, path, wide, variant):
    sots, P, beams, ts, sampling = CASES[case]
    if wide == 0 and P - 1 <= 8:
        pytest.skip("the prompt never reaches the wide prefill")
    if P > 100 and path != "warp_mma" and wide == 0:
        pytest.skip("one pass per position of a 227-token prompt: covered on the warp-MMA pass")
    _, _, h = model(variant)
    n = len(sots)
    prompts = [make_prompt(s, P, 7 * u + s) for u, s in enumerate(sots)]
    beams = [beams[u % len(beams)] for u in range(n)]
    set_path(h, path, wide)
    try:
        windows = np.arange(n) + 3
        check(variant, h, windows, prompts, beams, ts=ts, sampling=sampling, tag=(case, path, wide))
        # max_length leaving 0 new tokens: every window still gets its value; then one window capped at 0 among others
        check(variant, h, windows, prompts, beams, ts=ts, sampling=sampling, max_length=P, tag=(case, path, wide, 0))
        if n > 1 and not sampling:
            mls = [P] + [P + 20] * (n - 1)
            check(variant, h, windows, prompts, beams, ts=ts, max_length=np.asarray(mls), tag=(case, path, wide, "ml"))
    finally:
        reset(h)


@pytest.mark.parametrize("variant", [False, True])
@pytest.mark.parametrize("wide", [1, 0])
def test_batched_16_windows_and_several_groups(wide, variant):
    _, _, h = model(variant)
    windows = np.arange(16)
    sots = [(0, 11, 13, 2)[u % 4] for u in range(16)]
    prompts = [make_prompt(s, 14, 3 * u + s) for u, s in enumerate(sots)]
    h.set_option("wide_prefill", wide)
    try:
        for rows in (320, 16):  # 16 rows at beam 5: groups of 3 windows
            h.set_option("batch_rows", rows)
            check(variant, h, windows, prompts, [5] * 16, tag=(wide, rows))
            check(variant, h, windows, [PROMPT] * 16, [5] * 16, tag=(wide, rows, "fused"))
            check(variant, h, windows, [PROMPT] * 16, [1] * 16, sampling=True, tag=(wide, rows, "sample"))
    finally:
        reset(h)


def test_faster_whisper_sequence():
    _, _, h = model(True)
    m = models.Whisper(None, device="cuda", _handles=[h])
    feats = models.StorageView.from_array(np.ascontiguousarray(mel_inputs(16)[:4]))
    prompts = [make_prompt(s, 14, 11 + s) for s in (11, 0, 13, 5)]
    kw = dict(beam_size=5, return_scores=True, return_no_speech_prob=True)
    from_feats = m.generate(feats, prompts, **kw)
    enc = m.encode(feats)
    from_enc = m.generate(enc, prompts, **kw)
    a = np.asarray([r.no_speech_prob for r in from_feats])
    b = np.asarray([r.no_speech_prob for r in from_enc])
    assert (a > 0).all()
    np.testing.assert_allclose(b, a, rtol=1e-5)
    assert [r.sequences_ids for r in from_enc] == [r.sequences_ids for r in from_feats]
    host = m.generate(m.encode(feats, to_cpu=True), prompts, **kw)
    np.testing.assert_allclose([r.no_speech_prob for r in host], a, rtol=1e-5)
    perm = [2, 0, 3, 1]
    mel_p = models.StorageView.from_array(np.ascontiguousarray(mel_inputs(16)[:4][perm]))
    permuted = m.generate(m.encode(mel_p), [prompts[i] for i in perm], **kw)
    np.testing.assert_allclose([r.no_speech_prob for r in permuted], a[perm], rtol=1e-5)
    # sampling: one value per window
    sampled = m.generate(enc, prompts, beam_size=1, num_hypotheses=5, sampling_topk=0, sampling_temperature=0.7,
                         return_no_speech_prob=True, random_seed=5)
    np.testing.assert_allclose([r.no_speech_prob for r in sampled], a, rtol=1e-5)
    # without the request: 0.0, and no prompt check
    assert all(r.no_speech_prob == 0.0 for r in m.generate(enc, prompts, beam_size=5))
    with pytest.raises(ValueError, match="startoftranscript"):
        m.generate(enc, [[SOT_PREV, 400, 500, 600]] * 4, return_no_speech_prob=True)


def test_c_abi_refusals():
    _, _, h = model(False)
    mel = np.ascontiguousarray(mel_inputs(16)[:2])
    ns = np.zeros(2, np.float32)
    with pytest.raises(ValueError, match="startoftranscript"):
        h.generate(mel, np.asarray([PROMPT, [SOT_PREV, 400, 500, 600]], np.int32), 1, no_speech_out=ns)
    # that failed call leaves nothing to read, and neither does a call without the option
    assert _lib.lib().wisb_get_no_speech_probs(h._h, 2, _lib.ptr(ns)) == 1
    h.generate(mel, np.asarray([PROMPT] * 2, np.int32), 1)
    assert _lib.lib().wisb_get_no_speech_probs(h._h, 2, _lib.ptr(ns)) == 1
    h.generate(mel, np.asarray([PROMPT] * 2, np.int32), 1, no_speech_out=ns)
    assert (ns > 0).all()
    assert _lib.lib().wisb_get_no_speech_probs(h._h, 3, _lib.ptr(np.zeros(3, np.float32))) == 1  # another B
    out = np.zeros(2, np.float32)
    assert _lib.lib().wisb_get_no_speech_probs(h._h, 2, _lib.ptr(out)) == 0 and np.array_equal(out, ns)
    # without the request a prompt without <|startoftranscript|> decodes as before
    h.generate(mel, np.asarray([[SOT_PREV, 400, 500, 600]] * 2, np.int32), 1, max_length=10)
