"""GPU: Whisper.encode and encoder outputs passed to generate, detect_language and align, on the seeded synthetic models
of gpu_common.  Everything is compared bit for bit with the same call on the features.

* encode (host and device form) equals debug_encode at d = 384 and 1280 and on a 128-mel model, at 1 and 3 windows.
* generate on an encoder output returns the features call's ids and scores: greedy and beam 5, on the warp-MMA, SIMT and
  batched passes, over several groups, in timestamp mode with the history processors and per-window max_length.  This
  holds because the cross-K/V GEMM computes each row from its own input row only.
* detect_language and align likewise; host fp16, fp32 and device outputs through detect -> generate -> align ->
  generate; with option profile only the cross-K/V GEMM runs.
* Source rules (logmel(keep) against load_encoder_output, batch-size mismatch, the encoder cache), a device output
  shared by two handles and freed after both are closed, and two GPUs when present."""
import numpy as np
import pytest

from oracle import logmel as om
from tests import test_gpu_align as TA
from tests.gpu_common import PROMPT, make_blob, mel_inputs
from tests.test_gpu_large_v3 import oracle_mel, v3_dims
from willow_inference_server_b200 import _lib, models, weights as W
from willow_inference_server_b200.models import StorageView

pytestmark = pytest.mark.gpu
TS_PROMPT = PROMPT[:3]


def fresh(dims, **opts):
    h = _lib.Handle.from_host(make_blob(dims), 0)
    for k, v in opts.items():
        h.set_option(k, v)
    return h


def small_dims(d=128, H=2):
    return W.WhisperDims(d_model=d, n_heads=H, n_enc_layers=2, n_dec_layers=2)


def same_results(a, b):
    assert [r.sequences_ids for r in a] == [r.sequences_ids for r in b]
    assert [r.scores for r in a] == [r.scores for r in b]  # float compare: bit-identical scores


# ------------------------------------------------------------------------------------------------ 1. encode
@pytest.mark.parametrize("dims,mel_fn", [
    (small_dims(384, 6), mel_inputs),
    (small_dims(1280, 20), mel_inputs),
    (v3_dims(2, 2), lambda n: oracle_mel([om.synth_utterance(m, 100 + i) for i, m in enumerate([61440, 160000, 480000][:n])])),
], ids=["d384", "d1280", "mel128"])
@pytest.mark.parametrize("n", [1, 3])
def test_encode_equals_debug_encode(dims, mel_fn, n):
    h = fresh(dims)
    m = models.Whisper(None, device="cuda", _handles=[h])
    x = np.ascontiguousarray(mel_fn(3)[:n])
    want = h.debug_encode(x)
    host = m.encode(StorageView.from_array(x), to_cpu=True)
    assert host.device == "cpu" and host.shape == [n, 1500, dims.d_model] and host.array.dtype == np.float16
    assert np.array_equal(host.array.astype(np.float32), want)
    dev = m.encode(x)
    assert (dev.device, dev.device_index, dev.shape) == ("cuda", 0, [n, 1500, dims.d_model])
    back = dev.to_device("cpu")
    assert back.array.dtype == np.float16 and np.array_equal(back.array.view(np.uint16), host.array.view(np.uint16))


# ------------------------------------------------------------------------------------------------ 2. generate
@pytest.mark.parametrize("case", ["greedy_mma", "beam5_mma", "greedy_simt", "beam5_simt", "batched16", "decoder_batch2",
                                  "groups", "timestamps_proc"])
def test_generate_on_encoder_output(case):
    dims = small_dims()
    opts, n, kw = {}, 1, dict(beam_size=5)
    prompt = PROMPT
    if case.startswith("greedy"):
        kw = dict(beam_size=1)
    if case.endswith("simt"):
        opts["mega_mma"] = 0
    if case == "batched16":
        n = 16
    elif case == "decoder_batch2":
        opts["decoder_batch"] = 2
    elif case == "groups":
        opts["batch_rows"], n, kw = 8, 9, dict(beam_size=2)  # 4 windows per group: 3 groups
    elif case == "timestamps_proc":
        n, prompt = 4, TS_PROMPT
        kw = dict(beam_size=5, repetition_penalty=1.2, no_repeat_ngram_size=3, max_length=[448, 20, 60, 448])
    h = fresh(dims, **opts)
    m = models.Whisper(None, device="cuda", _handles=[h])
    x = np.ascontiguousarray(mel_inputs(16)[:n])
    enc = m.encode(StorageView.from_array(x), to_cpu=True)
    want = m.generate(StorageView.from_array(x), [prompt] * n, return_scores=True, **kw)
    assert any(len(r.sequences_ids[0]) > 2 for r in want)
    same_results(m.generate(enc, [prompt] * n, return_scores=True, **kw), want)
    same_results(m.generate(m.encode(x), [prompt] * n, return_scores=True, **kw), want)


# ------------------------------------------------------------------------------------------------ 3. + 4. every call
def test_detect_generate_align_on_three_sources():
    dims = TA.setup()[0]
    h = _lib.Handle.from_host(TA.setup()[2], 0)
    h.set_option("profile", 1)
    m = models.Whisper(None, device="cuda", _handles=[h])
    n = 2
    x = np.ascontiguousarray(mel_inputs(16)[5:5 + n])
    texts, frames = [TA.windows()[0][5], [400, 500, 600]], [3000, 1777]
    feats = StorageView.from_array(x)

    def sequence(src):
        langs = m.detect_language(src)
        g1 = m.generate(src, [PROMPT] * n, beam_size=5, return_scores=True)
        al = m.align(src, TA.START, texts, frames)
        t_align = h.timing()
        g2 = m.generate(src, [TS_PROMPT] * n, beam_size=2, return_scores=True)
        return (langs, g1, al, g2), t_align, h.timing()

    want, ta_f, tg_f = sequence(feats)
    assert ta_f["conv1_ms"] > 0 and tg_f["conv1_ms"] > 0
    host16 = m.encode(feats, to_cpu=True)
    host32 = StorageView.from_array(host16.array.astype(np.float32))
    for src in (host16, host32, m.encode(feats)):
        got, ta, tg = sequence(src)
        assert got[0] == want[0]                                         # language ids and probabilities
        same_results(got[1], want[1])
        same_results(got[3], want[3])
        for a, b in zip(got[2], want[2]):                                # alignment paths and token probabilities
            assert a.alignments == b.alignments and a.text_token_probs == b.text_token_probs
        # only the cross-K/V GEMM ran (one group).  align runs the batched pass, which also times one of its own kernel
        # families in slot 11, so conv1_ms is checked on the 4-row generate (persistent pass) alone
        assert tg["conv1_ms"] == 0
        for t, tf in ((ta, ta_f), (tg, tg_f)):
            assert t["gemm_launches"] == tf["gemm_launches"] - (1 + 4 * dims.n_enc_layers)


def test_fp32_input_is_rounded_to_nearest_even():
    dims = small_dims()
    h = fresh(dims)
    m = models.Whisper(None, device="cuda", _handles=[h])
    x = np.ascontiguousarray(mel_inputs(4)[:2])
    e32 = m.encode(StorageView.from_array(x), to_cpu=True).array.astype(np.float32)
    rng = np.random.default_rng(3)
    e32 *= (1 + rng.uniform(-4e-4, 4e-4, e32.shape)).astype(np.float32)  # values between fp16 neighbours
    e32.reshape(-1)[:4] = [2.0 ** -25, 1 + 2.0 ** -11, 3 * 2.0 ** -12, -(1 + 3 * 2.0 ** -11)]  # ties -> even
    r16 = e32.astype(np.float16)                                            # numpy rounds to nearest even
    assert not np.array_equal(r16.astype(np.float32), e32)
    ids = np.asarray([PROMPT] * 2, np.int32)
    h.load_encoder_output(r16)
    want = h.generate(None, ids, B=2)
    h.load_encoder_output(e32)
    assert h.generate(None, ids, B=2) == want


# ------------------------------------------------------------------------------------------------ 5. source rules
def test_source_rules_and_encoder_cache():
    dims = small_dims()
    h = fresh(dims)
    ids1 = np.asarray([PROMPT], np.int32)
    pcm = om.synth_utterance(160000, 7)
    mel_a = h.logmel(pcm, [0], [pcm.size], keep=True)
    want_a = h.generate(mel_a, ids1)
    other = np.ascontiguousarray(mel_inputs(4)[2:3])
    enc_b = h.encode(other)
    want_b = h.generate(other, ids1)
    assert want_a != want_b
    # logmel(keep) then load: the loaded output decodes; then logmel(keep) again: the features do
    h.logmel(pcm, [0], [pcm.size], keep=True, to_host=False)
    h.load_encoder_output(enc_b)
    assert h.timing()["h2d_ms"] > 0
    assert h.generate(None, ids1, B=1) == want_b
    h.logmel(pcm, [0], [pcm.size], keep=True, to_host=False)
    assert h.generate(None, ids1, B=1) == want_a
    # a call with another batch size fails with code 1
    h.load_encoder_output(np.repeat(enc_b, 2, 0))
    with pytest.raises(ValueError, match="batch size"):
        h.generate(None, ids1, B=1)
    with pytest.raises(ValueError, match="batch size"):
        h.detect_language(None, B=3)
    assert h.generate(None, np.repeat(ids1, 2, 0), B=2) == h.generate(np.repeat(other, 2, 0), np.repeat(ids1, 2, 0))
    # the encoder cache: features F -> encoder output of other audio -> F again re-encodes
    fresh_f = fresh(dims).generate(mel_a, ids1)
    c = fresh(dims, encoder_cache=1, profile=1)
    assert c.generate(mel_a, ids1) == fresh_f
    c.load_encoder_output(enc_b)
    assert c.generate(None, ids1, B=1) == want_b
    assert c.generate(mel_a, ids1) == fresh_f
    assert c.timing()["conv1_ms"] > 0


# ------------------------------------------------------------------------------------------------ 6. two handles
def test_device_output_shared_by_two_handles():
    dims = small_dims()
    blob = make_blob(dims)
    ha, hb = _lib.Handle.from_host(blob, 0), _lib.Handle.from_host(blob, 0)
    ma = models.Whisper(None, device="cuda", _handles=[ha])
    mb = models.Whisper(None, device="cuda", _handles=[hb])
    x = StorageView.from_array(np.ascontiguousarray(mel_inputs(4)[:3]))
    dev = ma.encode(x)
    want = ma.generate(x, [PROMPT] * 3, beam_size=5, return_scores=True)
    same_results(mb.generate(dev, [PROMPT] * 3, beam_size=5, return_scores=True), want)
    assert mb.detect_language(dev) == ma.detect_language(x)
    host = dev.to_device("cpu")
    ma.unload_model()
    mb.unload_model()
    assert np.array_equal(dev.to_device("cpu").array.view(np.uint16), host.array.view(np.uint16))
    buf, dev._buf = dev._buf, None
    _lib.buffer_free(buf)  # after every handle is closed: raises nothing
    with pytest.raises(ValueError):
        _lib.buffer_free(buf)


# ------------------------------------------------------------------------------------------------ 7. two GPUs
def test_two_gpus():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs in one process")
    dims = small_dims()
    blob = make_blob(dims)
    h0, h1 = _lib.Handle.from_host(blob, 0), _lib.Handle.from_host(blob, 1)
    one = models.Whisper(None, device="cuda", _handles=[h0])
    two = models.Whisper(None, device="cuda", device_index=[0, 1], _handles=[h0, h1])
    x = StorageView.from_array(np.ascontiguousarray(mel_inputs(4)))
    want = one.encode(x, to_cpu=True).array
    assert np.array_equal(two.encode(x, to_cpu=True).array.view(np.uint16), want.view(np.uint16))
    devs = [two.encode(x), two.encode(x)]
    dev1 = [d for d in devs if d.device_index == 1][0]
    assert np.array_equal(dev1.to_device("cpu").array.view(np.uint16), want.view(np.uint16))
    want_g = one.generate(x, [PROMPT] * 4, beam_size=5, return_scores=True)
    solo1 = models.Whisper(None, device="cuda", device_index=[1], _handles=[h1])
    same_results(two.generate(dev1, [PROMPT] * 4, beam_size=5, return_scores=True), want_g)
    same_results(solo1.generate(dev1, [PROMPT] * 4, beam_size=5, return_scores=True), want_g)
    with pytest.raises(ValueError, match="no replica"):
        one.generate(dev1, [PROMPT] * 4)
