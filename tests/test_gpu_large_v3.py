"""GPU: the large-v3 family -- 128-bin log-mel, the 128-bin conv stem, the 51866-token vocabulary (100 languages) and
decoders shallower than their encoders, against the oracle.

* Log-mel at 128 bins within 1e-4 of the oracle: f32 and s16 input, the 16 mixed durations, input over 30 s, 1 sample,
  all zeros; through log_mel_spectrogram, log_mel_batch and log_mel_chunks (75 s); features kept on the device by a v3
  model handle decode like the same features from the host; an 80-bin front end is bit-identical before and after a
  128-bin one ran in the same process.
* Stem at 128 bins (wisb_debug_enc_stem), 1 and 3 windows, d = 384 and 1280: conv1 against float64 within a bound
  derived for 384 sequential fp32 FMAs, conv2 + positions within the GEMM bound, zero rows exact.
* End to end on synthetic 128-mel, 51866-token models, (encoder, decoder) layers (2, 2), (4, 2), (4, 1): greedy and
  beam 5 on the warp-MMA and SIMT persistent passes and the batched pass (16 utterances x beam 5), tokens equal to the
  oracle on its robust cases; timestamp decoding with the v3 ids; detect_language with 100 entries; align on (4, 2);
  the encoder cache; 80-bin features refused.
* Full size: synthetic large-v3-turbo (d 1280, 32 / 4 layers) against the fp32 oracle, the bars of
  test_gpu_fullsize.test_large_v2_numeric_parity_against_the_oracle."""
import functools

import numpy as np
import pytest
import torch

from oracle import logmel as om
from oracle.whisper_ref import WhisperOracle
from tests import enc_oracle as O
from tests.gpu_common import DURATIONS, LOGIT_TOL, RAMP, SCRIPT, make_blob, robust_cases
from tests.test_gpu_align import row_of_frame, windows
from tests.test_gpu_kernels import bits, note_ratio, tol_gemm, worst_ratio
from willow_inference_server_b200 import _lib, audio, models, weights as W
from willow_inference_server_b200.languages import LANGUAGE_CODES

pytestmark = pytest.mark.gpu
TOL = 1e-4
PROMPT3 = [50258, 50259, 50360, 50364]  # sot, <|en|>, <|transcribe|>, <|notimestamps|> of the 51866 vocabulary
TS_PROMPT3 = PROMPT3[:3]
FILTERS = om.slaney_mel_filterbank(n_mels=128)
U = 2.0 ** -24


def oracle_mel(pcm_list):
    return om.log_mel_batch(pcm_list, FILTERS)


@functools.lru_cache(maxsize=1)
def fe128():
    return _lib.Handle.frontend(0, 128)


@functools.lru_cache(maxsize=1)
def v3_inputs(n=16):
    pcm = [om.synth_utterance(m, 100 + i) for i, m in enumerate(DURATIONS[:n])]
    return pcm, oracle_mel(pcm)


def v3_dims(le, ld, d=128, H=2, **kw):
    return W.WhisperDims(d_model=d, n_heads=H, n_enc_layers=le, n_dec_layers=ld, n_mels=128, n_vocab=51866, **kw)


@functools.lru_cache(maxsize=3)
def v3_pair(le, ld):
    dims = v3_dims(le, ld)
    buf = make_blob(dims)
    return dims, WhisperOracle.from_blob(buf), _lib.Handle.from_host(buf, 0)


# ------------------------------------------------------------------------------------------------ log-mel
def test_logmel128_mixed_batch_f32_and_s16():
    rng = np.random.default_rng(3)
    pcm = [om.synth_utterance(m, 100 + i) for i, m in enumerate(DURATIONS)]
    pcm += [om.synth_utterance(560000, 7), np.array([0.25], np.float32), np.zeros(480000, np.float32),
            (0.5 * rng.standard_normal(480000)).astype(np.float32)]
    mel = audio.log_mel_batch(pcm, n_mels=128)
    assert mel.shape == (len(pcm), 128, 3000) and mel.dtype == np.float32
    ref = oracle_mel(pcm)
    for i in range(len(pcm)):
        assert np.abs(mel[i] - ref[i]).max() <= TOL, i
    s16 = [np.clip(np.round(p * 32768.0), -32768, 32767).astype(np.int16) for p in pcm[:6]]
    got = audio.log_mel_batch(s16, fe128())
    ref16 = oracle_mel([p.astype(np.float32) / 32768.0 for p in s16])
    assert np.abs(got - ref16).max() <= TOL


def test_logmel128_surfaces_and_80_bin_front_end_unchanged():
    pcm = om.synth_utterance(61440, 1234)
    before = audio.log_mel_spectrogram(pcm).numpy()          # the 80-bin front end first
    a = audio.log_mel_spectrogram(audio.pad_or_trim(pcm), n_mels=128).numpy()
    assert a.shape == (128, 3000)
    assert np.abs(a - om.log_mel_spectrogram(om.pad_or_trim(pcm), FILTERS)).max() <= TOL
    assert np.array_equal(a, audio.log_mel_spectrogram(pcm, 128).numpy())
    after = audio.log_mel_spectrogram(pcm).numpy()           # 80 bins again, after the 128-bin tables were uploaded
    assert after.shape == (80, 3000) and np.array_equal(before, after)
    fe80 = _lib.Handle.frontend(0)
    assert np.array_equal(audio.log_mel_batch([pcm], fe80)[0], before)
    for bad in (96, 64, 0):
        with pytest.raises(AssertionError):
            audio.log_mel_spectrogram(pcm, n_mels=bad)
        with pytest.raises(ValueError):
            _lib.Handle.frontend(0, bad)
    with pytest.raises(ValueError):
        audio.log_mel_batch([pcm], fe128(), n_mels=80)
    # long audio: every chunk_iter window framed from the one PCM buffer
    rng = np.random.default_rng(5)
    x = (0.3 * np.sin(np.arange(75 * 16000) * 0.05) + 0.05 * rng.standard_normal(75 * 16000)).astype(np.float32)
    mel, strides = audio.log_mel_chunks(x, n_mels=128)
    want = [(om.log_mel_spectrogram(om.pad_or_trim(c), FILTERS), s) for c, s in audio.chunk_iter(x)]
    assert mel.shape == (6, 128, 3000) and strides == [s for _, s in want]
    for i, (w, _) in enumerate(want):
        assert np.abs(mel[i] - w).max() <= TOL, i
    assert audio.log_mel_chunks(np.zeros(0, np.float32), fe128())[0].shape == (0, 128, 3000)
    assert audio.log_mel_window(x, n_mels=128).shape == (1, 128, 3000)


def test_device_kept_features_decode_like_host_features():
    dims, oracle, h = v3_pair(2, 2)
    pcm, _ = v3_inputs()
    mel = audio.log_mel_batch(pcm[:3], h)                    # a model handle frames with its model's 128 bins
    assert mel.shape == (3, 128, 3000)
    P = np.array([PROMPT3] * 3, np.int32)
    want, _ = h.generate(mel, P, 5)
    n = np.array([p.shape[0] for p in pcm[:3]], np.int32)
    off = np.concatenate([[0], np.cumsum(n[:-1])]).astype(np.int64)
    h.logmel(np.concatenate(pcm[:3]), off, n, to_host=False, keep=True)
    got, _ = h.generate(None, P, 5, B=3)
    assert got == want and all(len(s) > 0 for s in want)


# ------------------------------------------------------------------------------------------------ stem
def conv1_128(m, mel):
    """-> (pre, S) of conv1 on log-mel [B, 128, 3000] in float64 (weights [d][k * 128 + ci])"""
    mel = np.asarray(mel, np.float64)
    B, nm, d = mel.shape[0], mel.shape[1], m.d
    w = m.f("enc.conv1.w").reshape(d, 3, nm)
    bias = m.f("enc.conv1.b")
    xp = np.zeros((B, nm, O.N_FRAMES + 2))
    xp[:, :, 1: O.N_FRAMES + 1] = mel
    pre = np.broadcast_to(bias, (B, O.N_FRAMES, d)).copy()
    S = np.broadcast_to(np.abs(bias), (B, O.N_FRAMES, d)).copy()
    for k in range(3):
        a = xp[:, :, k: k + O.N_FRAMES].transpose(0, 2, 1)
        pre += a @ w[:, k, :].T
        S += np.abs(a) @ np.abs(w[:, k, :]).T
    return pre, S


def conv1_tol_128(pre, S, ref):
    """enc_oracle.conv1_tol for K = 384: 384 sequential fp32 FMAs and the bias add round a partial sum bounded by S
    (385 2^-24 S), GELU's slope <= 1.13, fp32 erff's 2 ulp of 1 times |x| / 2, the rounded argument through erf's slope
    and three roundings, and half an fp16 ulp for the store."""
    a = np.abs(pre)
    err = 1.13 * 385 * U * S + 2.0 ** -23 * a + 3 * U * a + 0.8 * U * a * a
    return (1 + 2.0 ** -11) * err + 2.0 ** -11 * np.abs(ref) + 2.0 ** -25


def mel128_case(B, seed):
    rng = np.random.default_rng([seed, B, 128])
    mel = np.empty((B, 128, 3000), np.float32)
    for b in range(B):
        top = 1.0 + 0.15 * b + 0.05 * seed
        m = rng.uniform(top - 2, top, (128, 3000))
        m[:, 400 + 50 * b: 700 + 50 * b] = top - 2
        m[:, 0] = np.linspace(top - 2, top, 128)
        m[:, -1] = np.linspace(top, top - 1.5, 128)
        mel[b] = m
    return mel


@functools.lru_cache(maxsize=2)
def stem_model(d, H):
    dims = v3_dims(1, 1, d, H)
    t = W.synth_engine_tensors(dims, seed=d)
    buf = np.zeros(W.blob_nbytes(t), np.uint8)
    W.write_blob_into(buf, dims, t)
    return O.Model(buf), _lib.Handle.from_host(buf, 0)


@pytest.mark.parametrize("d,H", [(384, 6), (1280, 20)])
def test_stem_128_matches_fp64(d, H):
    m, h = stem_model(d, H)
    rng = np.random.default_rng(d)
    for B, seed in ((3, 0), (1, 1)):
        mel = mel128_case(B, seed)
        h1, x = h.debug_enc_stem(mel)
        pre, S = conv1_128(m, mel)
        ref = O.gelu(pre)
        win = h1[: B * O.H1_ROWS].reshape(B, O.H1_ROWS, d)
        got = win[:, 1: 1 + O.N_FRAMES]
        tol = conv1_tol_128(pre, S, ref)
        note_ratio(f"conv1 128 bins d {d}", worst_ratio(got, ref, tol))
        assert (np.abs(got.astype(np.float64) - ref) <= tol).all(), (d, B)
        assert np.all(bits(win[:, 0]) == 0) and np.all(bits(win[:, 1 + O.N_FRAMES:]) == 0)
        rows = np.stack([np.sort(np.concatenate([[0, 1, 2, 749, 1497, 1498, 1499],
                                                 rng.choice(np.arange(3, 1497), 64, replace=False)])) for _ in range(B)])
        acc, r, ref2 = O.conv2(m, h1, B, rows)
        got2 = O.gather(x, rows)
        tol2 = tol_gemm(3 * d, r, ref2, "conv2", acc)
        note_ratio(f"conv2 + pos 128 bins d {d}", worst_ratio(got2, ref2, tol2))
        assert (np.abs(got2.astype(np.float64) - ref2) <= tol2).all(), (d, B)
        assert np.all(bits(x[:, O.T_ENC:]) == 0)
    with pytest.raises(ValueError):
        h.debug_enc_stem(mel128_case(1, 0)[:, :80])


# ------------------------------------------------------------------------------------------------ end to end
SHAPES = [(2, 2), (4, 2), (4, 1)]


# A case counts when its transcript survives the logit-noise probe AND every step's decision-relevant gap
# (WhisperOracle's trace) is above DECISION_GAP: iid noise rarely reorders two candidates that share a prefix, and one
# such case, 0.01 apart, resolved the other way on the warp-MMA pass.
DECISION_GAP = {1: LOGIT_TOL, 5: LOGIT_TOL / 4}
# cases of 16 that must qualify: measured 8-13 greedy, 2-6 at beam 5 (fewest on the 4 / 1-layer model: with 4 scripted
# alternatives per position the 5th and 6th beam candidates are often close); the beam-5 cases are also compared in
# test_batched_pass_16_utterances_beam5
MIN_ROBUST = {1: 8, 5: 2}


@functools.lru_cache(maxsize=6)
def oracle_cases(le, ld, beam):
    dims, oracle, h = v3_pair(le, ld)
    _, mel = v3_inputs()
    enc = oracle.encode(mel)
    res, robust = robust_cases(oracle, mel, [PROMPT3] * 16, beam, enc=enc)
    trace = []
    oracle.generate(mel, [PROMPT3] * 16, beam_size=beam, enc=enc, trace=trace)
    return mel, res, [i for i in robust if min(trace[i][:-1]) > DECISION_GAP[beam]]


@pytest.mark.parametrize("le,ld", SHAPES)
@pytest.mark.parametrize("beam", [1, 5])
def test_small_row_passes_match_oracle(le, ld, beam):
    dims, oracle, h = v3_pair(le, ld)
    mel, res, robust = oracle_cases(le, ld, beam)
    print(f"({le}, {ld}) beam {beam}: {len(robust)} of 16 oracle transcripts robust")
    assert len(robust) >= MIN_ROBUST[beam], f"only {len(robust)} of 16 oracle transcripts are robust"
    P = np.array([PROMPT3], np.int32)
    for mma in (1, 0):
        h.set_option("mega_mma", mma)
        try:
            group = max(1, 8 // beam)  # <= 8 rows: one persistent pass
            ids = []
            for g0 in range(0, 16, group):
                part = mel[g0: g0 + group]
                ids += h.generate(np.ascontiguousarray(part), np.repeat(P, len(part), 0), beam)[0]
        finally:
            h.set_option("mega_mma", 1)
        for i in robust:
            assert ids[i] == res[i].sequences_ids[0], (mma, beam, i)
        assert all(dims.eot not in s and not set(s) & set(dims.suppress_ids) for s in ids)


@pytest.mark.parametrize("le,ld", SHAPES)
def test_batched_pass_16_utterances_beam5(le, ld):
    dims, oracle, h = v3_pair(le, ld)
    mel, res, robust = oracle_cases(le, ld, 5)
    ids, _ = h.generate(mel, np.repeat(np.array([PROMPT3], np.int32), 16, 0), 5)  # 80 rows: the batched pass
    for i in robust:
        assert ids[i] == res[i].sequences_ids[0], i


def test_timestamps_with_v3_ids():
    from tests.ts_oracle import TimestampOracle, check_invariants

    dims = v3_dims(2, 2)  # test_gpu_timestamps' model with the 51866 vocabulary's ids
    tensors = W.synth_engine_tensors(dims, seed=11, eot_ramp=RAMP, script=SCRIPT, ts_script=(2, 5, 8))
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    oracle, h = TimestampOracle.from_blob(buf), _lib.Handle.from_host(buf, 0)
    _, mel = v3_inputs()
    for beam in (1, 5):
        res, robust = robust_cases(oracle, mel, [TS_PROMPT3] * 16, beam)
        if beam > 1:  # the test_gpu_timestamps gap criterion: every step's decision-relevant gap above LOGIT_TOL / 4
            trace = []
            oracle.generate(mel, [TS_PROMPT3] * 16, beam_size=beam, trace=trace)
            robust = [i for i in robust if min(trace[i][:-1]) > LOGIT_TOL / 4]
        # (measured: 8 greedy cases and 1 at beam 5 qualify; every one of the 16 engine transcripts is checked against
        # the timestamp rules below whatever its robustness)
        assert len(robust) >= {1: 3, 5: 1}[beam], (beam, len(robust))
        segments = [check_invariants(res[i].sequences_ids[0], dims) for i in robust]
        print(f"timestamps beam {beam}: {len(robust)} robust cases, segments {segments}")
        assert min(segments) >= 1 and (beam > 1 or max(segments) >= 2)  # greedy: the pair and non-decreasing rules act
        ids, _ = h.generate(mel, np.repeat(np.array([TS_PROMPT3], np.int32), 16, 0), beam, timestamps=True)
        solo = [h.generate(mel[i: i + 1], np.array([TS_PROMPT3], np.int32), beam, timestamps=True)[0][0] for i in range(16)]
        for i in robust:
            assert ids[i] == res[i].sequences_ids[0] == solo[i], (beam, i)
        for s in ids:
            check_invariants(s, dims)
        assert any(t > dims.no_timestamps for s in ids for t in s)


def test_detect_language_100_entries():
    dims, oracle, h = v3_pair(4, 2)
    _, mel = v3_inputs()
    m = models.Whisper(None, device="cuda", _handles=[h])
    assert m.n_mels == 128 and m.num_languages == 100
    got = m.detect_language(models.StorageView.from_array(mel[:4]))
    want = oracle.detect_language(mel[:4])
    for b in range(4):
        assert len(got[b]) == 100 and abs(sum(p for _, p in got[b]) - 1.0) < 1e-3
        assert [t for t, _ in got[b][:3]] == [f"<|{LANGUAGE_CODES[t - dims.lang_first]}|>" for t, _ in want[b][:3]], b
        assert "<|yue|>" in {t for t, _ in got[b]}


def test_align_on_the_4_2_model():
    from tests import align_oracle as AO

    heads = [[1, 0], [1, 1]]
    dims = v3_dims(4, 2, alignment_heads=heads)
    tensors = W.synth_engine_tensors(dims, seed=11, align_script=(30.0, 250.0, 3000.0))
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    oracle, h = WhisperOracle.from_blob(buf), _lib.Handle.from_host(buf, 0)
    _, mel = v3_inputs()
    enc = oracle.encode(mel)
    texts, frames = windows()  # test_gpu_align's 16 windows: mixed text lengths and num_frames
    paths, probs = h.align(mel, TS_PROMPT3, texts, frames, 7)
    robust, n_text = 0, 0
    for b in range(16):
        if not texts[b]:
            assert paths[b].shape == (0, 2)
            continue
        n_text += 1
        weights, tp = AO.capture_window(oracle, enc[b], TS_PROMPT3, texts[b], frames[b])
        assert np.abs(np.log(np.asarray(probs[b])) - np.log(tp)).max() <= 2 * LOGIT_TOL
        want = AO.dtw(AO.filter_matrix(weights, 7).numpy())
        g = torch.Generator().manual_seed(b)
        stable = all(np.array_equal(AO.dtw(AO.filter_matrix(
            weights * np.exp(0.05 * torch.randn(weights.shape, generator=g).numpy()), 7).numpy()), want) for _ in range(3))
        if stable:
            robust += 1
            assert np.array_equal(paths[b], want), b
        F = frames[b] // 2
        assert np.mean(row_of_frame(paths[b], F) == row_of_frame(want, F)) >= 0.98, b
        p = paths[b]
        assert tuple(p[0]) == (0, 0) and tuple(p[-1]) == (len(texts[b]), F - 1)
    assert robust * 5 >= n_text


def test_encoder_cache_sequence_and_feature_shape():
    dims, oracle, h = v3_pair(2, 2)
    _, mel = v3_inputs()
    one = np.ascontiguousarray(mel[:1])
    P = np.array([PROMPT3], np.int32)
    translate = np.array([[50258, 50259, dims.translate, dims.no_timestamps]], np.int32)
    plain = [h.detect_language(one)[0].tolist(), h.generate(one, P, 5)[0], h.generate(one, translate, 5)[0]]
    enc_ms = h.timing()["encoder_ms"]  # (option off: the translate call encoded again)
    cached = _lib.Handle.from_host(make_blob(dims), 0)
    cached.set_option("encoder_cache", 1)
    got = [cached.detect_language(one)[0].tolist(), cached.generate(one, P, 5)[0], cached.generate(one, translate, 5)[0]]
    assert got == plain
    assert cached.timing()["encoder_ms"] < 0.5 * enc_ms  # the translate call reused the encoder output
    m = models.Whisper(None, device="cuda", _handles=[h])
    mel80 = om.log_mel_batch([om.synth_utterance(61440, 1)])
    with pytest.raises(ValueError, match="128"):
        m.generate(models.StorageView.from_array(mel80), [PROMPT3])
    with pytest.raises(ValueError, match="128"):
        m.detect_language(models.StorageView.from_array(mel80))
    with pytest.raises(ValueError):
        h.generate(mel80, P, 5)
    from willow_inference_server_b200.batcher import TranscribeBatcher

    with TranscribeBatcher(m, max_batch=4, max_wait_ms=1) as b:
        with pytest.raises(ValueError, match="128"):
            b.submit(mel80, PROMPT3)
        assert b.submit(one, PROMPT3, beam_size=5).result(timeout=60)[0].sequences_ids[0] == plain[1][0]


# ------------------------------------------------------------------------------------------------ full size
def test_large_v3_turbo_numeric_parity_against_the_oracle():
    """Synthetic large-v3-turbo (d 1280, 32 encoder / 4 decoder layers, 128 mels, 51866 tokens) against the fp32 oracle:
    encoder output <= 6e-2 abs, teacher-forced logits of the warp-MMA and batched passes <= 2.5e-1, a beam-5 decode equal
    to the oracle's robust transcript alone and as one row of a batch of 3."""
    dims = W.WhisperDims.for_size("large-v3-turbo")
    tensors = W.synth_engine_tensors(dims, seed=3, eot_ramp=RAMP, script=SCRIPT)
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    h = _lib.Handle.from_host(buf, 0)
    del buf
    oracle = WhisperOracle(dims, tensors)
    del tensors
    mel = oracle_mel([om.synth_utterance(61440, 21), om.synth_utterance(160000, 22), om.synth_utterance(100000, 23)])
    enc = oracle.encode(mel)
    enc_err = float(np.abs(h.debug_encode(mel[:2]) - enc[:2].numpy()).max())
    toks = PROMPT3 + [1000, 2000, 30000, 41000, 12, 50000]
    want = oracle.forced_logits(enc[0], toks).numpy()
    got_mma = h.debug_forced_logits(mel[:1], toks)
    h.set_option("decoder_batch", 2)
    got_b = h.debug_forced_logits(mel[:1], toks)
    h.set_option("decoder_batch", 1)
    err_mma, err_b = (float(np.abs(g - want).max()) for g in (got_mma, got_b))
    print(f"large-v3-turbo: encoder max abs err {enc_err:.4f}; logits err {err_mma:.4f} (warp-MMA pass) {err_b:.4f} "
          f"(batched pass); logit range [{want.min():.1f}, {want.max():.1f}]")
    assert enc_err <= 6e-2 and err_mma <= 2.5e-1 and err_b <= 2.5e-1
    base = oracle.generate(mel, [PROMPT3] * 3, beam_size=5, enc=enc)
    probe = oracle.generate(mel, [PROMPT3] * 3, beam_size=5, enc=enc, logit_noise=(LOGIT_TOL, 77))
    robust = [i for i in range(3) if base[i].sequences_ids == probe[i].sequences_ids]
    assert robust, "no full-size oracle transcript is a robust decision"
    m = models.Whisper(None, device="cuda", _handles=[h])
    out = [m.generate(models.StorageView.from_array(mel[i: i + 1]), [PROMPT3], beam_size=5, return_scores=True)[0]
           for i in range(3)]
    outb = m.generate(models.StorageView.from_array(mel), [PROMPT3] * 3, beam_size=5)
    for i in robust:
        assert out[i].sequences_ids[0] == base[i].sequences_ids[0], i
        assert 5 <= len(out[i].sequences_ids[0]) < 40
        assert abs(out[i].scores[0] - base[i].scores[0]) < 5e-2
        assert outb[i].sequences_ids[0] == base[i].sequences_ids[0], i
    h.close()
