"""GPU parity: the CUDA Whisper path through the C ABI vs the fp32 oracle on seeded synthetic weights.

Tolerances (north_star: token-id exact under greedy, text-exact under beam=5):
  * encoder output (after the final LayerNorm, O(1) values): fp16 tensor-core inputs, fp32 accumulation -> <= 3e-2 abs
  * teacher-forced logits (std ~4): <= 6e-2 abs
  * token ids: EXACT on every case whose oracle transcript is a robust decision (tests/gpu_common.robust_cases); the
    tests also require that most cases are robust, so the comparison cannot become vacuous
"""
import numpy as np
import pytest
import torch

from oracle.whisper_ref import WhisperOracle
from tests.gpu_common import LOGIT_TOL, PROMPT, make_blob, mel_inputs, model_pair, robust_cases
from willow_inference_server_b200 import _lib, models

pytestmark = pytest.mark.gpu
ENC_TOL = 3e-2
SIMT_SIGMA = 1e-2   # robustness probe of the SIMT-pass transcripts: a few times the SIMT-vs-kv_fp16-oracle logit bound


@pytest.fixture(scope="module")
def pair():
    return model_pair()


def test_encoder_matches_oracle(pair):
    dims, oracle, h = pair
    mel = mel_inputs(4)[:3]
    want = oracle.encode(mel).numpy()
    for vmn in (1, 0):  # both V-operand layouts of the attention kernel
        h.set_option("attn_v_mn_major", vmn)
        got = h.debug_encode(mel)
        err = np.abs(got - want).max()
        assert err <= ENC_TOL, (vmn, err)
    h.set_option("attn_v_mn_major", 1)


def test_encoder_layer_by_layer(pair):
    dims, oracle, h = pair
    mel = mel_inputs(4)[:1]
    for nl in (0, 1, 2):
        want = oracle.encode(mel, n_layers=nl).numpy()
        got = h.debug_encode(mel, n_layers=nl)
        assert np.abs(got - want).max() <= ENC_TOL, nl


def test_attention_tensor_core_vs_simt(pair):
    dims, oracle, h = pair
    mel = mel_inputs(4)[:2]
    a = h.debug_encode(mel)
    h.set_option("attn_ref", 1)
    b = h.debug_encode(mel)
    h.set_option("attn_ref", 0)
    assert np.abs(a - b).max() <= 1e-2


def test_forced_logits_match_oracle(pair):
    dims, oracle, h = pair
    mel = mel_inputs(4)[:1]
    toks = PROMPT + [100, 2000, 30000, 41000, 12, 50000, 7, 999, 4242]
    want = oracle.forced_logits(oracle.encode(mel)[0], toks).numpy()
    got = h.debug_forced_logits(mel, toks)
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= LOGIT_TOL


@pytest.mark.parametrize("beam", [1, 5, 2])
def test_generate_matches_oracle(pair, beam):
    dims, oracle, h = pair
    mel = mel_inputs(6)
    n = mel.shape[0]
    res, robust = robust_cases(oracle, mel, [PROMPT] * n, beam)
    assert len(robust) >= 4, f"only {len(robust)} of {n} oracle transcripts are robust decisions"
    m = models.Whisper(None, device="cuda", _handles=[h])
    out = m.generate(models.StorageView.from_array(mel), [PROMPT] * n, beam_size=beam, return_scores=True)
    for i in robust:  # exact token parity, no tolerated mismatch; the length-normalised score at every beam size
        assert out[i].sequences_ids[0] == res[i].sequences_ids[0], (beam, i)
        assert abs(out[i].scores[0] - res[i].scores[0]) < 5e-2, (beam, i)
    assert len({tuple(res[i].sequences_ids[0]) for i in robust}) >= 3  # the transcripts depend on the audio
    for o in out:
        assert dims.eot not in o.sequences_ids[0]
        assert not set(o.sequences_ids[0]) & set(dims.suppress_ids)


SEARCH_CONFIGS = [(5, 0.5, 1.0), (5, 2.0, 1.0), (2, 1.25, 1.0), (5, 1.0, 0.0), (2, 1.0, 0.6)]   # beam, patience, lp


@pytest.mark.parametrize("beam,patience,lp", SEARCH_CONFIGS)
def test_patience_and_length_penalty_match_oracle(pair, beam, patience, lp):
    # max_hyp = beam * patience rounded half up (5 x 0.5 -> 3, 2 x 1.25 -> 3) and the length penalty, on the batched
    # pass (6 utterances: 12 or 30 rows) and on the <= 8-row persistent pass (one utterance per call)
    dims, oracle, h = pair
    mel = mel_inputs(6)
    n = mel.shape[0]
    kw = dict(patience=patience, length_penalty=lp)
    res, robust = robust_cases(oracle, mel, [PROMPT] * n, beam, **kw)
    kw["beam_size"] = beam
    assert len(robust) >= 3, f"only {len(robust)} of {n} oracle transcripts are robust decisions"
    batched = h.generate(mel, [PROMPT] * n, **kw)
    solo = [h.generate(mel[i : i + 1], [PROMPT], **kw) for i in range(n)]
    for i in robust:
        for where, ids, sc in (("batched", batched[0][i], batched[1][i]), ("solo", solo[i][0][0], solo[i][1][0])):
            assert ids == res[i].sequences_ids[0], (where, beam, patience, lp, i)
            assert abs(sc - res[i].scores[0]) < 5e-2, (where, beam, patience, lp, i)


def test_search_settings_do_not_share_a_graph(pair):
    # back-to-back batched calls that differ only in patience or length penalty each decode what they decode alone
    dims = pair[0]
    mel = mel_inputs(6)
    calls = [dict(patience=1.0, length_penalty=1.0), dict(patience=2.0, length_penalty=1.0),
             dict(patience=2.0, length_penalty=0.0), dict(patience=1.0, length_penalty=1.0)]
    h = _lib.Handle.from_host(make_blob(dims), 0)
    try:
        mixed = [h.generate(mel, [PROMPT] * 6, beam_size=5, **c) for c in calls]
    finally:
        h.close()
    for c, got in zip(calls, mixed):
        alone = _lib.Handle.from_host(make_blob(dims), 0)
        try:
            want = alone.generate(mel, [PROMPT] * 6, beam_size=5, **c)
        finally:
            alone.close()
        assert got[0] == want[0] and np.array_equal(np.float32(got[1]), np.float32(want[1])), c
    assert mixed[0] == mixed[3] and mixed[2][1] != mixed[1][1]   # the length penalty really changed the call


def test_graphs_and_eager_agree(pair):
    dims, oracle, h = pair
    mel = mel_inputs(4)[:2]
    a, _ = h.generate(mel, [PROMPT] * 2, beam_size=5)
    h.set_option("use_graphs", 0)
    b, _ = h.generate(mel, [PROMPT] * 2, beam_size=5)
    h.set_option("use_graphs", 1)
    assert a == b


def test_persistent_passes_vs_oracles(pair):
    # the two decoder implementations for <= 8 rows: the warp-MMA persistent pass (default; fp16 B operands) and the SIMT
    # persistent pass, whose activations are fp32 and whose only roundings are the fp16 cross K/V and self-attention
    # cache.  The SIMT pass is checked tightly against an oracle that rounds at exactly those two points (kv_fp16), fed
    # the engine's own encoder output; the MMA pass against the plain oracle and the SIMT pass.  The calls have <= 8 rows
    # (4 utterances x beam 2, 1 x beam 5), so every transcript comes from a persistent pass.
    dims, oracle, h = pair
    oracle16 = WhisperOracle.from_blob(make_blob(dims))
    oracle16.kv_fp16 = True
    mel = mel_inputs(4)
    toks = PROMPT + [100, 2000, 30000, 41000, 12]
    calls = [(4, 2), (1, 5)]
    want = oracle.forced_logits(oracle.encode(mel[:1])[0], toks).numpy()
    a = h.debug_forced_logits(mel[:1], toks)
    ids_a = [h.generate(mel[:n], [PROMPT] * n, beam_size=beam)[0] for n, beam in calls]
    h.set_option("mega_mma", 0)
    try:
        s_ = h.debug_forced_logits(mel[:1], toks)
        ids_s = [h.generate(mel[:n], [PROMPT] * n, beam_size=beam)[0] for n, beam in calls]
    finally:
        h.set_option("mega_mma", 1)
    enc = {n: torch.from_numpy(h.debug_encode(mel[:n])) for n, _ in calls}
    want16 = oracle16.forced_logits(enc[1][0], toks).numpy()
    # SIMT pass vs the kv_fp16 oracle: summation order and rare fp16 rounding-boundary flips of K/V only (measured worst
    # 3.9e-4 on an H100 80GB HBM3 at a 700 W power limit; against the plain oracle the same logits differ by 1.7e-2)
    assert np.abs(s_ - want16).max() <= 2e-3
    assert np.abs(a - want).max() <= LOGIT_TOL     # tensor-core pass vs the oracle
    assert np.abs(a - s_).max() <= LOGIT_TOL
    n16 = n_plain = 0
    for (n, beam), got_a, got_s in zip(calls, ids_a, ids_s):
        res16, robust16 = robust_cases(oracle16, mel[:n], [PROMPT] * n, beam, enc=enc[n], sigma=SIMT_SIGMA)
        for i in robust16:
            assert got_s[i] == res16[i].sequences_ids[0], (n, beam, i)
        res, robust = robust_cases(oracle, mel[:n], [PROMPT] * n, beam)
        for i in robust:
            assert got_a[i] == got_s[i] == res[i].sequences_ids[0], (n, beam, i)
        n16 += len(robust16)
        n_plain += len(robust)
    assert n16 >= 4 and n_plain >= 3, (n16, n_plain)   # of 5 cases


@pytest.mark.parametrize("n_utt,beam", [(2, 3), (4, 2), (8, 1), (3, 2)])
def test_small_path_several_utterances_per_pass(pair, n_utt, beam):
    # <= 8 rows: several utterances x beams inside ONE persistent pass (the warp-MMA pass and the SIMT pass alike): every
    # utterance decodes exactly as it does alone, and as the oracle says on its robust cases
    dims, oracle, h = pair
    mel = mel_inputs(8)[:n_utt]
    res, robust = robust_cases(oracle, mel, [PROMPT] * n_utt, beam)
    for mma in (1, 0):
        h.set_option("mega_mma", mma)
        try:
            ids, _ = h.generate(mel, [PROMPT] * n_utt, beam_size=beam)
            solo = [h.generate(mel[i : i + 1], [PROMPT], beam_size=beam)[0][0] for i in range(n_utt)]
        finally:
            h.set_option("mega_mma", 1)
        assert ids == solo, (mma, n_utt, beam)
        for i in robust:
            assert ids[i] == res[i].sequences_ids[0], (mma, n_utt, beam, i)


def test_max_length_and_suppress(pair):
    dims, oracle, h = pair
    mel = mel_inputs(4)[:1]
    for beam in (1, 3):
        ids, _ = h.generate(mel, [PROMPT], beam_size=beam, max_length=24, extra_suppress=[dims.eot])
        assert len(ids[0]) == 12
        want, robust = robust_cases(oracle, mel, [PROMPT], beam, max_length=24, suppress_tokens=(-1, dims.eot))
        assert len(want[0].sequences_ids[0]) == 12
        if robust:
            assert ids[0] == want[0].sequences_ids[0]
    ids, _ = h.generate(mel, [PROMPT], beam_size=1)  # mask restored: <|endoftext|> ends the transcript again
    assert ids[0] == h.generate(mel, [PROMPT], beam_size=1, extra_suppress=[])[0][0]
    assert ids[0] != h.generate(mel, [PROMPT], beam_size=1, extra_suppress=[dims.eot])[0][0]


def test_detect_language(pair):
    dims, oracle, h = pair
    mel = mel_inputs(4)[:2]
    m = models.Whisper(None, device="cuda", _handles=[h])
    got = m.detect_language(models.StorageView.from_array(mel))
    want = oracle.detect_language(mel)
    from willow_inference_server_b200.languages import LANGUAGE_CODES

    for g, w in zip(got, want):
        assert len(g) == 99 and g[0][0].startswith("<|")
        assert abs(sum(p for _, p in g) - 1) < 1e-4
        # the detected language (WIS reads results[0][0], main.py:640) and the next two are the oracle's
        want_top = [f"<|{LANGUAGE_CODES[t - dims.lang_first]}|>" for t, _ in w[:3]]
        assert [t for t, _ in g[:3]] == want_top
        for (_, pg), (_, pw) in zip(g[:3], w[:3]):
            assert abs(pg - pw) < 2e-2


def test_argument_errors(pair):
    dims, oracle, h = pair
    mel = mel_inputs(4)[:1]
    m = models.Whisper(None, device="cuda", _handles=[h])
    with pytest.raises(ValueError):
        m.generate(mel[:, :40], [PROMPT])
    with pytest.raises(ValueError):
        m.generate(mel, [PROMPT, PROMPT])
    with pytest.raises(ValueError):
        m.generate(mel, [PROMPT], beam_size=9)
    with pytest.raises(ValueError):
        m.generate(mel, [[50258, 60000, 50359, 50363]])
    with pytest.raises(ValueError):
        h.generate(mel, np.array([PROMPT], np.int32), max_length=1000)
    with pytest.raises(ValueError):
        h.set_option("decoder_mega", 0)   # an option that no longer exists


def test_wider_model_batch(pair):
    # d=256, 4 heads, 3 layers: exercises multi-head indexing, BN=256 tiles and a 7-utterance batch (35 rows: the
    # batched decoder pass)
    dims, oracle, h = model_pair(256, 4, 3, 7)
    mel = np.concatenate([mel_inputs(6)[:4], mel_inputs(6)[:3]])
    want = oracle.encode(mel[:2]).numpy()
    assert np.abs(h.debug_encode(mel[:2]) - want).max() <= ENC_TOL
    res, robust = robust_cases(oracle, mel, [PROMPT] * 7, 5)
    assert len(robust) >= 5
    got, _ = h.generate(mel, [PROMPT] * 7, beam_size=5)
    for i in robust:
        assert got[i] == res[i].sequences_ids[0], i
    assert got[0] == got[4] and got[1] == got[5]  # same audio -> same transcript regardless of batch position


def test_encoder_cache_detect_then_generate(pair):
    # SURVEY 8f row 4: detect_language -> generate -> translate on one window encode once when the cache is switched on
    dims, oracle, h = pair
    mel = mel_inputs(4)[:1].copy()
    plain = models.Whisper(None, device="cuda", _handles=[h])
    want = plain.generate(models.StorageView.from_array(mel), [PROMPT], beam_size=5)[0].sequences_ids[0]
    ores, orobust = robust_cases(oracle, mel, [PROMPT], 5)
    if orobust:
        assert want == ores[0].sequences_ids[0]  # checked against the oracle, not only against the engine itself
    want_lang = plain.detect_language(models.StorageView.from_array(mel))
    assert [t for t, _ in want_lang[0]][0] == "<|%s|>" % __import__("willow_inference_server_b200.languages", fromlist=["x"]).LANGUAGE_CODES[
        oracle.detect_language(mel)[0][0][0] - dims.lang_first]
    m = models.Whisper(None, device="cuda", _handles=[h], reuse_encoder=True)
    try:
        langs = m.detect_language(models.StorageView.from_array(mel))
        assert [t for t, _ in langs[0]] == [t for t, _ in want_lang[0]]
        got = m.generate(models.StorageView.from_array(mel), [PROMPT], beam_size=5)[0].sequences_ids[0]
        t_reuse = m.timing()
        assert got == want
        assert t_reuse["encoder_ms"] < 0.05 and t_reuse["cross_kv_ms"] < 0.05, t_reuse   # nothing was re-encoded
        translate = [PROMPT[0], PROMPT[1], dims.translate, PROMPT[3]]
        tr = m.generate(models.StorageView.from_array(mel), [translate], beam_size=5)[0].sequences_ids[0]
        assert m.timing()["encoder_ms"] < 0.05
        assert tr == plain.generate(models.StorageView.from_array(mel), [translate], beam_size=5)[0].sequences_ids[0]
        m2 = models.Whisper(None, device="cuda", _handles=[h], reuse_encoder=True)
        mel2 = mel.copy()
        mel2[0, 3, 100] += 0.5                                   # one changed feature: the cache must miss
        other = m2.generate(models.StorageView.from_array(mel2), [PROMPT], beam_size=5)[0].sequences_ids[0]
        assert m2.timing()["encoder_ms"] > 0.05
        again = m2.generate(models.StorageView.from_array(mel), [PROMPT], beam_size=5)[0].sequences_ids[0]
        assert again == want and m2.timing()["encoder_ms"] > 0.05   # different features in between: re-encoded
    finally:
        h.set_option("encoder_cache", 0)


def test_encoder_cache_needs_one_group(pair):
    # a cache that holds two windows encoded as one batch must not serve a call that decodes them in two groups: each
    # group would read the cross K/V at the offsets of a batch of one, and the second group would read the first window's
    dims = pair[0]
    mel = np.ascontiguousarray(mel_inputs(4)[:2])
    prompts = np.asarray([PROMPT] * 2, np.int32)
    plain = _lib.Handle.from_host(make_blob(dims), 0)
    plain.set_option("batch_rows", 8)
    want = plain.generate(mel, prompts, beam_size=5)
    h = _lib.Handle.from_host(make_blob(dims), 0)
    h.set_option("encoder_cache", 1)
    h.generate(mel, prompts, beam_size=5)  # 10 rows, one group of 2 windows: the cache now holds both
    h.set_option("batch_rows", 8)          # 8 // 5 = 1 window per group
    assert h.generate(mel, prompts, beam_size=5) == want
    assert h.timing()["launches"] == plain.timing()["launches"]  # both groups were encoded again


def test_encoder_cache_layout_rerun(pair):
    # detect_language leaves the cross K/V chunk-swizzled (<= 8 rows: the warp-MMA persistent pass); a generate at beam 5
    # on the same 2 windows (10 rows: the batched pass) reads it linear and reruns only the cross-K/V GEMM
    dims = pair[0]
    mel = np.ascontiguousarray(mel_inputs(4)[:2])
    prompts = np.asarray([PROMPT] * 2, np.int32)
    plain = _lib.Handle.from_host(make_blob(dims), 0)
    want = plain.generate(mel, prompts, beam_size=5)
    t_plain = plain.timing()
    h = _lib.Handle.from_host(make_blob(dims), 0)
    h.set_option("encoder_cache", 1)
    h.detect_language(mel)
    got = h.generate(mel, prompts, beam_size=5)
    t = h.timing()
    assert got == want
    assert t["decode_steps"] == t_plain["decode_steps"]
    # no encoder: conv1, conv2, 7 per layer, ln_post are gone; the cross-K/V GEMM reran once (linear layout)
    assert t["launches"] == t_plain["launches"] - (3 + 7 * dims.n_enc_layers)


def test_batcher_over_the_real_engine(pair):
    import threading

    from willow_inference_server_b200.batcher import TranscribeBatcher

    dims, oracle, h = pair
    mel = mel_inputs(4)
    m = models.Whisper(None, device="cuda", _handles=[h])
    want = [r.sequences_ids[0] for r in m.generate(models.StorageView.from_array(mel), [PROMPT] * 4, beam_size=5)]
    with TranscribeBatcher(m, max_batch=8, max_wait_ms=50) as b:
        futs = [None] * 4
        ts = [threading.Thread(target=lambda i=i: futs.__setitem__(i, b.submit(mel[i : i + 1], PROMPT, beam_size=5))) for i in range(4)]
        [t.start() for t in ts]
        [t.join() for t in ts]
        got = [f.result(timeout=60)[0].sequences_ids[0] for f in futs]
    assert got == want                       # batch-position invariance makes the coalesced call equal to the direct one
    assert b.stats["engine_calls"] < 4


def test_two_replicas_in_one_process():
    # the reference's multi-GPU mode: ONE process, ctranslate2-style device_index=[0..N-1] replicas (main.py:295,346);
    # every kernel's function attributes must be configured on every device, not once per process
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs in one process")
    from willow_inference_server_b200 import _lib, weights as W

    dims, oracle, h0 = model_pair()
    from tests.gpu_common import make_blob

    h1 = _lib.Handle.from_host(make_blob(dims), 1)
    mel = mel_inputs(4)
    one = models.Whisper(None, device="cuda", _handles=[h0])
    want = [r.sequences_ids[0] for r in one.generate(models.StorageView.from_array(mel), [PROMPT] * 4, beam_size=5)]
    two = models.Whisper(None, device="cuda", device_index=[0, 1], _handles=[h0, h1])
    for _ in range(2):
        got = [r.sequences_ids[0] for r in two.generate(models.StorageView.from_array(mel), [PROMPT] * 4, beam_size=5)]
        assert got == want
    # replica 1 alone on 5 rows, through both persistent decoder passes, and the front end on the second device
    for mma in (1, 0):
        h1.set_option("mega_mma", mma)
        solo = models.Whisper(None, device="cuda", device_index=[1], _handles=[h1])
        assert [r.sequences_ids[0] for r in solo.generate(models.StorageView.from_array(mel[:1]), [PROMPT], beam_size=5)] == want[:1]
    h1.set_option("mega_mma", 1)
    langs = two.detect_language(models.StorageView.from_array(mel[:2]))
    assert [t for t, _ in langs[0]][:3] == [t for t, _ in one.detect_language(models.StorageView.from_array(mel[:1]))[0]][:3]
    pcm = np.zeros(16000, np.float32)
    assert np.array_equal(h1.logmel(pcm, [0], [16000]), h0.logmel(pcm, [0], [16000]))
    h1.close()
