"""Previous-text prompts: faster-whisper's <|startofprev|> context, timestamps included, and its wide prefill.

* The wide prefill's cross-attention kernel (Handle.debug_dec_prefill_cross_attn) against float64
  softmax(fp16(q/8) . K^T over keys < 1500) . V within tests.test_gpu_decoder_kernels' bound, at 1..447 rows per
  utterance, in both cross-K/V layouts, with NaN in every padding key and every other layer and sentinels in the ctx
  rows it must not write; bit-identical on a repeat.  The CPU tests show that the comparator rejects injected defects.
* End to end on the timestamp-scripted synthetic model: prompts with a timestamped previous-text context decode in
  timestamp mode (and with <|notimestamps|> without), equal to the oracle on its robust cases on every decoder path;
  wide_prefill 1 against 0 gives the same tokens in ceil((prompt_len - 1) / chunk) prefill passes.
* Full-size synthetic large-v2: a 227-token prompt, one generated token, wide against narrow prefill.
* Prompts of <= 9 tokens: wide_prefill changes nothing, launches and decode steps included.
"""
import math

import numpy as np
import pytest

from tests.gpu_common import LOGIT_TOL, PROMPT, mel_inputs, model_pair, robust_cases
from tests.test_gpu_decoder_kernels import SENT16, T_ENC, T_PAD, cross_case, cross_ref, ratio, within
from tests.test_gpu_kernels import bits, note_ratio, sentinel
from tests.test_prev_text_host import SOT_PREV, previous
from tests.ts_oracle import check_invariants
from willow_inference_server_b200 import _lib, weights as W

NAN16 = np.uint16(0x7E00)


# ------------------------------------------------------------------------------------------------ kernel
def swizzle(ckv):
    """the persistent warp-MMA pass's layout: 16-byte chunk c of key t's 128-byte row stored at chunk c ^ (t & 7)"""
    x = ckv.view(np.uint16).reshape(ckv.shape[:-1] + (8, 8))
    idx = np.arange(8)[None, :] ^ (np.arange(T_PAD)[:, None] & 7)           # position p holds chunk p ^ (t & 7)
    idx = np.broadcast_to(idx[..., None], x.shape)
    return np.ascontiguousarray(np.take_along_axis(x, idx, axis=-2).reshape(ckv.shape)).view(np.float16)


def prefill_case(n_utt, H, rpu, seed=0, kind="gauss"):
    q, ckv = cross_case(kind, n_utt, H, rpu, tier="gauss", seed=seed)
    ckv[:, :, :, :, T_ENC:] = NAN16.view(np.float16)                       # padding keys: NaN in K and V
    return q, ckv


GEOMS = [(1, 2, 16), (8, 6, 3), (9, 20, 3), (63, 2, 3), (64, 6, 1), (65, 2, 16), (226, 20, 1), (447, 6, 1),
         (447, 2, 3)]


@pytest.fixture(scope="module")
def fe():
    return _lib.Handle.frontend(0)


@pytest.mark.gpu
@pytest.mark.parametrize("swz", [0, 1])
@pytest.mark.parametrize("rpu,H,n_utt", GEOMS)
def test_prefill_cross_attention_matches_fp64(fe, rpu, H, n_utt, swz):
    q, ckv = prefill_case(n_utt, H, rpu, seed=rpu)
    dev = swizzle(ckv) if swz else ckv
    ref, tol = cross_ref(q, ckv, rpu, impl=0)
    rows = np.arange(n_utt * rpu)
    ctx = sentinel((n_utt * rpu + 5, H * 64), np.float16)                  # 5 rows past the last: must stay untouched
    got = fe.debug_dec_prefill_cross_attn(q, dev, ctx[: n_utt * rpu], layer=1, rows_per_utt=rpu, swizzled=bool(swz))
    note_ratio("prefill cross-attention", ratio(got[rows], ref, tol))
    assert within(got[rows], ref, tol), (rpu, H, n_utt, swz)
    assert np.all(bits(ctx[n_utt * rpu:]) == SENT16)
    again = fe.debug_dec_prefill_cross_attn(q, dev, sentinel(got.shape, np.float16), layer=1, rows_per_utt=rpu,
                                            swizzled=bool(swz))
    assert np.array_equal(bits(again), bits(got))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["late", "early", "uniform", "padding", "onehot"])
def test_prefill_cross_attention_score_shapes(fe, kind):
    q, ckv = prefill_case(2, 2, 70, kind=kind)
    ref, tol = cross_ref(q, ckv, 70, impl=0)
    got = fe.debug_dec_prefill_cross_attn(q, ckv, sentinel(q.shape, np.float16), layer=1, rows_per_utt=70)
    note_ratio("prefill cross-attention", ratio(got, ref, tol))
    assert within(got, ref, tol), kind


@pytest.mark.gpu
def test_prefill_cross_attention_rejects_bad_arguments(fe):
    q, ckv = prefill_case(1, 2, 9)
    for kw in (dict(rows_per_utt=449), dict(rows_per_utt=0), dict(layer=2), dict(layer=-1)):
        args = dict(layer=1, rows_per_utt=9) | kw
        qq = np.zeros((args["rows_per_utt"], 128), np.float32)
        with pytest.raises(ValueError):
            fe.debug_dec_prefill_cross_attn(qq, ckv, sentinel(qq.shape, np.float16), **args)
    with pytest.raises(ValueError):                                        # the <= 8-row entry still refuses 9 rows
        fe.debug_dec_cross_attn(q, ckv, sentinel(q.shape, np.float16), layer=1, rows_per_utt=9)


def test_prefill_comparator_rejects_injected_defects():
    n_utt, H, rpu = 1, 2, 130
    q, ckv = cross_case("padding", n_utt, H, rpu, tier="gauss", seed=3)     # finite padding that would win unmasked
    ref, tol = cross_ref(q, ckv, rpu, impl=0)
    perfect = ref.astype(np.float16)
    assert within(perfect, ref, tol)
    defects = {
        "keys >= 1500 unmasked": cross_ref(q, ckv, rpu, impl=0, n_keys=T_PAD),
        "swizzle ignored": cross_ref(q, swizzle(ckv), rpu, impl=0),
        "scale applied twice": cross_ref(q, ckv, rpu, impl=0, scale=0.125 / 8),
        "last key tile dropped": cross_ref(q, ckv, rpu, impl=0, n_keys=11 * 128),
    }
    qn = q.copy()
    qn[64:128] = q[0:64]                                                    # tile 1 reads tile 0's queries
    defects["tile reads its neighbour's queries"] = cross_ref(qn, ckv, rpu, impl=0)
    for name, (bad, bad_tol) in defects.items():
        assert not within(perfect, bad, bad_tol), name


# ------------------------------------------------------------------------------------------------ end to end
TS_PROMPT = [50258, 50259, 50359]


def fw_prompt(n_prev, no_ts, seed=0):
    return [SOT_PREV] + previous(n_prev, seed) + TS_PROMPT + ([50363] if no_ts else [])


def ts_setup():
    from tests.test_gpu_timestamps import ts_pair
    return ts_pair()


def robust(oracle, mel, prompt, beam):
    res, rob = robust_cases(oracle, mel, [prompt] * len(mel), beam)
    if beam > 1:
        trace = []
        oracle.generate(mel, [prompt] * len(mel), beam_size=beam, trace=trace)
        rob = [i for i in rob if min(trace[i][:-1]) > LOGIT_TOL / 4]
    return res, rob


def run(h, mel, prompt, beam, ts, max_length=448, **opts):
    for k, v in opts.items():
        h.set_option(k, v)
    try:
        ids, sc = h.generate(mel, np.repeat(np.array([prompt], np.int32), len(mel), 0), beam, max_length=max_length,
                             timestamps=ts)
        return ids, sc, h.timing()
    finally:
        for k, v in opts.items():
            h.set_option(k, {"wide_prefill": 1, "mega_mma": 1, "decoder_batch": 1}[k])


@pytest.mark.gpu
@pytest.mark.parametrize("no_ts", [False, True])
@pytest.mark.parametrize("beam", [1, 5])
@pytest.mark.parametrize("path", ["mega_mma", "mega_simt", "batched_small", "batched16"])
def test_previous_text_end_to_end(path, beam, no_ts):
    dims, oracle, h = ts_setup()
    n = 16 if path == "batched16" else 6
    mel = mel_inputs(16)[:n]
    prompt = fw_prompt(60, no_ts, seed=beam)
    P = len(prompt)
    res, rob = robust(oracle, mel, prompt, beam)
    assert len(rob) >= 2, f"only {len(rob)} robust cases"
    opts = {"mega_mma": {}, "mega_simt": {"mega_mma": 0}, "batched_small": {"decoder_batch": 2}, "batched16": {}}[path]
    if path == "batched16":
        calls = [(mel, list(range(n)))]
        chunks = (min(8, 128 // n), min(P - 1, max(min(8, 128 // n), 1024 // n)))    # 16 x 5 rows: 128-row workspace
    else:
        calls = [(mel[i : i + 1], [i]) for i in range(n)]
        chunks = (8 if path == "batched_small" else 1, P - 1)
    for x, idx in calls:
        wide = run(h, x, prompt, beam, not no_ts, **opts)
        narrow = run(h, x, prompt, beam, not no_ts, wide_prefill=0, **opts)
        for j, i in enumerate(idx):
            if i in rob:
                assert wide[0][j] == res[i].sequences_ids[0], (path, beam, i)
                assert narrow[0][j] == wide[0][j], (path, beam, i)
                if beam > 1:
                    assert abs(wide[1][j] - res[i].scores[0]) < 5e-2
            if not no_ts:
                check_invariants(wide[0][j], dims)
        if wide[0] == narrow[0]:
            n_narrow, n_wide = math.ceil((P - 1) / chunks[0]), math.ceil((P - 1) / chunks[1])
            assert wide[2]["decode_steps"] - n_wide == narrow[2]["decode_steps"] - n_narrow, (path, wide[2], narrow[2])


@pytest.mark.gpu
def test_short_prompts_unchanged_by_wide_prefill():
    dims, oracle, h = model_pair()
    mel = mel_inputs(16)
    for prompt in (PROMPT, [SOT_PREV, 440, 1029, 257, 11, 50258, 50259, 50359, 50363]):       # 4 and 9 tokens
        for n, beam, opts in ((1, 5, {}), (1, 5, {"mega_mma": 0}), (1, 5, {"decoder_batch": 2}), (16, 5, {}),
                              (2, 1, {})):
            a = run(h, mel[:n], prompt, beam, False, **opts)
            b = run(h, mel[:n], prompt, beam, False, wide_prefill=0, **opts)
            assert a[0] == b[0] and np.array_equal(np.float32(a[1]), np.float32(b[1])), (len(prompt), n, opts)
            assert a[2]["launches"] == b[2]["launches"] and a[2]["decode_steps"] == b[2]["decode_steps"]


@pytest.mark.gpu
def test_full_size_227_token_prompt():
    dims = W.WhisperDims.for_size("large-v2")
    tensors = W.synth_engine_tensors(dims, seed=0)
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    del tensors
    h = _lib.Handle.from_host(buf, 0)
    mel = mel_inputs(1)
    rng = np.random.default_rng(5)
    prompt = [SOT_PREV] + [int(t) for t in rng.integers(0, 50257, 222)] + PROMPT
    assert len(prompt) == 227
    wide = run(h, mel, prompt, 5, False, max_length=228)                   # min(228 / 2, 228 - 227): one new token
    narrow = run(h, mel, prompt, 5, False, max_length=228, wide_prefill=0)
    assert len(wide[0][0]) == 1 and wide[0] == narrow[0]
    assert abs(wide[1][0] - narrow[1][0]) <= 2.5e-1
    assert wide[2]["decode_steps"] == 2 and narrow[2]["decode_steps"] == 227
