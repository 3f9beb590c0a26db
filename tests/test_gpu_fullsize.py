"""GPU tests at BASELINE.json's full model size (whisper-large-v2 dims, seeded synthetic weights) through size-independent
properties -- the fp32 oracle needs ~9 s per utterance at this size, so exact parity at full size is checked once per run
by bench.py (`tokens_identical_to_cpu_oracle`) and here we check what does not need the oracle."""
import threading

import numpy as np
import pytest

from willow_inference_server_b200 import _lib, audio, models, weights as W

pytestmark = pytest.mark.gpu
PROMPT = [50258, 50259, 50359, 50363]


def _synth(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.float64) / 16000.0
    return (0.3 * np.sin(2 * np.pi * (200.0 + 300.0 * t) * t) + 0.05 * rng.standard_normal(n)).astype(np.float32)


@pytest.fixture(scope="module")
def large():
    dims = W.WhisperDims.for_size("large-v2")
    tensors = W.synth_engine_tensors(dims, seed=0)
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    del tensors
    h = _lib.Handle.from_host(buf, 0)
    return dims, h


def test_mixed_duration_batch_properties(large):
    dims, h = large
    # configs[2]-style ragged batch: 3.84 s / 10 s / 30 s utterances, two of them repeated at other batch positions
    pcm = [_synth(61440, 1), _synth(160000, 2), _synth(480000, 3), _synth(61440, 1), _synth(160000, 2)]
    mel = audio.log_mel_batch(pcm, h)
    assert mel.shape == (5, 80, 3000) and np.isfinite(mel).all()
    assert np.array_equal(mel[0], mel[3]) and np.array_equal(mel[1], mel[4])
    m = models.Whisper(None, device="cuda", _handles=[h])
    feats = models.StorageView.from_array(mel)
    out = m.generate(feats, [PROMPT] * 5, beam_size=5, max_length=24, return_scores=True)
    ids = [o.sequences_ids[0] for o in out]
    assert ids[0] == ids[3] and ids[1] == ids[4]            # batch-position invariance
    assert all(0 < len(s) <= 12 for s in ids)               # max_length // 2
    assert all(dims.eot not in s and not set(s) & set(dims.suppress_ids) for s in ids)
    again = [o.sequences_ids[0] for o in m.generate(feats, [PROMPT] * 5, beam_size=5, max_length=24)]
    assert again == ids                                      # run-to-run determinism (no atomics in the arithmetic)
    # one utterance at a time == inside the batch
    solo = m.generate(models.StorageView.from_array(mel[2:3]), [PROMPT], beam_size=5, max_length=24)
    assert solo[0].sequences_ids[0] == ids[2]
    # greedy and beam agree on the first token whenever the beam result starts with the greedy arg-max path's token
    g = m.generate(feats, [PROMPT] * 5, beam_size=1, max_length=24)
    assert all(len(o.sequences_ids[0]) <= 12 for o in g)
    # persistent pass kernel vs per-op chain at full size
    h.set_option("decoder_mega", 0)
    chain = [o.sequences_ids[0] for o in m.generate(feats, [PROMPT] * 5, beam_size=5, max_length=24)]
    h.set_option("decoder_mega", 1)
    assert chain == ids
    langs = m.detect_language(models.StorageView.from_array(mel[:2]))
    assert len(langs) == 2 and abs(sum(p for _, p in langs[0]) - 1.0) < 1e-3


def test_small_path_batches_equal_solo_runs_at_full_size(large):
    # large-v2, <= 8 rows in one persistent pass: with 20 heads and several utterances the fused cross-attention phase gives
    # most CTAs more than one (utterance, head, key split) task -- every utterance must still decode exactly as it does alone
    dims, h = large
    mel = audio.log_mel_batch([_synth(61440, 1), _synth(160000, 2), _synth(100000, 5), _synth(61440, 7), _synth(30000, 9)], h)
    P = np.array([PROMPT], np.int32)
    for n_utt, beam in ((5, 1), (2, 3), (4, 2)):
        ids, _ = h.generate(mel[:n_utt], np.repeat(P, n_utt, 0), beam, max_length=20)
        solo = [h.generate(mel[i : i + 1], P, beam, max_length=20)[0][0] for i in range(n_utt)]
        assert ids == solo, (n_utt, beam)
        assert all(0 < len(s) <= 10 for s in ids)
    h.set_option("mega_mma", 0)  # the SIMT pass agrees on greedy decoding of the same batch
    try:
        simt, _ = h.generate(mel[:5], np.repeat(P, 5, 0), 1, max_length=20)
    finally:
        h.set_option("mega_mma", 1)
    mma, _ = h.generate(mel[:5], np.repeat(P, 5, 0), 1, max_length=20)
    assert sum(a == b for a, b in zip(simt, mma)) >= 4  # (fp16 vs fp32 activations: a near-tie may flip one transcript)


def test_handles_coexist_and_threads(large):
    dims, h = large
    small_dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=2)
    from tests.gpu_common import make_blob

    hs = _lib.Handle.from_host(make_blob(small_dims), 0)  # a second model size next to the large one (WIS keeps five, main.py:319-326)
    mel = audio.log_mel_batch([_synth(61440, 1)])
    want_small, _ = hs.generate(mel, np.array([PROMPT], np.int32), 5)
    want_large, _ = h.generate(mel, np.array([PROMPT], np.int32), 5, max_length=16)
    results, errors = {}, []

    def work(name, handle, kw):
        try:
            for _ in range(3):
                results[name], _ = handle.generate(mel, np.array([PROMPT], np.int32), 5, **kw)
        except Exception as e:  # pragma: no cover
            errors.append(e)

    ths = [threading.Thread(target=work, args=("s1", hs, {})), threading.Thread(target=work, args=("s2", hs, {})),
           threading.Thread(target=work, args=("l", h, {"max_length": 16}))]
    [t_.start() for t_ in ths]
    [t_.join() for t_ in ths]
    assert not errors
    assert results["s1"] == want_small and results["s2"] == want_small and results["l"] == want_large
    hs.close()


def test_large_v2_numeric_parity_against_the_oracle():
    """Full-size (d_model 1280, 32 + 32 layers) numeric parity: encoder output, teacher-forced logits and a beam-5 decode
    whose hypotheses finish on their own (<|endoftext|> NOT suppressed), against the fp32 oracle on the same weights.
    Tolerances (fp16 tensor-core operands, fp32 accumulation, 32 layers deep): encoder output <= 6e-2 abs (values O(1)),
    logits <= 2.5e-1 abs on logits that span about +-60 (peaked model), tokens exact when the oracle's transcript is a
    robust decision."""
    from oracle import logmel as om
    from oracle.whisper_ref import WhisperOracle
    from tests.gpu_common import LOGIT_TOL, RAMP, SCRIPT

    dims = W.WhisperDims.for_size("large-v2")
    tensors = W.synth_engine_tensors(dims, seed=3, eot_ramp=RAMP, script=SCRIPT)
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    h = _lib.Handle.from_host(buf, 0)
    del buf
    oracle = WhisperOracle(dims, tensors)
    del tensors
    pcm = [_synth(61440, 21), _synth(160000, 22)]
    mel = om.log_mel_batch(pcm)
    enc = oracle.encode(mel)
    got_enc = h.debug_encode(mel)
    enc_err = float(np.abs(got_enc - enc.numpy()).max())
    toks = PROMPT + [1000, 2000, 30000, 41000, 12, 50000]
    want = oracle.forced_logits(enc[0], toks).numpy()
    got = h.debug_forced_logits(mel[:1], toks)           # persistent SIMT pass (fp32 activations)
    h.set_option("decoder_batch", 2)
    got_b = h.debug_forced_logits(mel[:1], toks)         # batched pass (fp16 GEMM operands, wgmma)
    h.set_option("decoder_batch", 1)
    err, err_b = float(np.abs(got - want).max()), float(np.abs(got_b - want).max())
    print(f"large-v2: encoder max abs err {enc_err:.4f}; logits err {err:.4f} (SIMT pass) {err_b:.4f} (batched pass); "
          f"logit range [{want.min():.1f}, {want.max():.1f}]")
    assert enc_err <= 6e-2
    assert err <= 2.5e-1 and err_b <= 2.5e-1
    # beam-5 decode, hypotheses finish through the <|endoftext|> ramp (finished pool, early stop, length normalisation)
    base = oracle.generate(mel, [PROMPT] * 2, beam_size=5, enc=enc)
    probe = oracle.generate(mel, [PROMPT] * 2, beam_size=5, enc=enc, logit_noise=(LOGIT_TOL, 77))
    m = models.Whisper(None, device="cuda", _handles=[h])
    # one utterance per call: 5 rows, the persistent SIMT pass
    out = [m.generate(models.StorageView.from_array(mel[i : i + 1]), [PROMPT], beam_size=5, return_scores=True)[0] for i in range(2)]
    robust = [i for i in range(2) if base[i].sequences_ids == probe[i].sequences_ids]
    assert robust, "neither full-size oracle transcript is a robust decision"
    for i in robust:
        assert out[i].sequences_ids[0] == base[i].sequences_ids[0], i
        assert 5 <= len(out[i].sequences_ids[0]) < 40
        assert abs(out[i].scores[0] - base[i].scores[0]) < 5e-2
    # the same two utterances as rows of one batched pass (10 rows: wgmma GEMM chain + wgmma cross-attention)
    outb = m.generate(models.StorageView.from_array(mel), [PROMPT] * 2, beam_size=5)
    for i in robust:
        assert outb[i].sequences_ids[0] == base[i].sequences_ids[0], i
    h.close()
