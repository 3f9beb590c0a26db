"""GPU: Whisper.align (wisb_align) against tests/align_oracle.py.

* Exact tier: the DTW kernel returns transformers' path bit for bit (random, tie-laden integer and 449 x 1500 matrices);
  the full post-processing (standardise, median filter, head mean) is within MAT_TOL of the oracle's matrix and its path
  is the oracle DTW of the engine's own matrix.
* The test model's alignment heads (named in the blob) have sharp, monotone attention peaks
  (``weights.synth_state_dict(align_script=...)``).  The raw capture (``wisb_debug_align_capture``) matches the oracle's
  probabilities within CAPTURE_TOL in log space wherever they are not negligible, so a per-row rescale (a re-softmax
  after the frame cut) or a wrong head / scale shows.
* End to end on 16 windows with mixed text lengths, num_frames and filter widths: identical alignments on the cases whose
  oracle path survives seeded perturbations of the captured probabilities at PROBE_SIGMA (at least 1 in 5 must), on
  every case the text index assigned to each frame agrees with the oracle's on >= 98 % of the frames,
  token probabilities within 2 x LOGIT_TOL in log space everywhere; every window of the batch equals its solo run bit
  for bit.
* generate -> align with the encoder cache (after a generate that left the cross K/V chunk-swizzled) equals align alone
  and does not rerun the encoder.
* Every invalid argument raises ValueError.
"""
import functools

import numpy as np
import pytest
import torch

from oracle.whisper_ref import WhisperOracle
from tests import align_oracle as AO
from tests.gpu_common import LOGIT_TOL, PROMPT, mel_inputs
from willow_inference_server_b200 import _lib, models, weights as W

pytestmark = pytest.mark.gpu
MAT_TOL = 1e-4        # filtered matrix (z-scores of O(1)): fp32 reductions in another order
# error of a captured log-probability against the fp32 oracle: the scripted heads' scores reach ~250 and pass through
# three fp16 roundings (the encoder output, the cross K, the query), ~2^-12 relative each, so a score can move by ~0.2
CAPTURE_TOL = 0.25
PROBE_SIGMA = 0.05    # robustness probe: independent log-normal noise per captured probability (typical capture error)
HEADS = [[2, 1], [3, 0], [3, 1]]
ALIGN_SCRIPT = (30.0, 250.0, 3000.0)
START = PROMPT[:3]    # <|startoftranscript|> <|en|> <|transcribe|>


@functools.lru_cache(maxsize=1)
def setup():
    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=4, alignment_heads=HEADS)
    tensors = W.synth_engine_tensors(dims, seed=11, align_script=ALIGN_SCRIPT)
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    return dims, WhisperOracle.from_blob(buf), buf


def handle():
    return _lib.Handle.from_host(setup()[2], 0)


# ----------------------------------------------------------------------------------------------------- exact tier
def test_dtw_bit_identical():
    h = handle()
    rng = np.random.default_rng(5)
    mats = [rng.standard_normal((r, f)).astype(np.float32) for r, f in [(2, 1), (2, 9), (5, 1), (7, 30), (40, 300)]]
    mats += [rng.integers(0, 3, (r, f)).astype(np.float32) for r, f in [(5, 9), (8, 8), (12, 40), (30, 100)]]
    mats.append(rng.standard_normal((449, 1500)).astype(np.float32))
    nan_col = rng.standard_normal((6, 20)).astype(np.float32)
    nan_col[:, 0] = np.nan  # a frame whose probabilities are equal in every row: the longest path, R + F entries
    mats.append(nan_col)
    for m in mats:
        _, path = h.debug_align_post(m, dtw_only=True)
        ref = AO.dtw(m)
        assert path.shape == ref.shape and (path == ref).all(), m.shape


@pytest.mark.parametrize("A,R,F,width", [(4, 6, 40, 7), (3, 9, 120, 1), (2, 5, 33, 3), (5, 12, 200, 9), (3, 6, 3, 7),
                                         (2, 2, 17, 7), (2, 4, 1, 3), (6, 30, 1500, 31)])
def test_post_processing(A, R, F, width):
    h = handle()
    rng = np.random.default_rng(A * 1000 + R * 10 + F)
    w = torch.softmax(torch.from_numpy(rng.standard_normal((A, R, F + 5)).astype(np.float32) * 3), -1)[..., :F]
    w = np.ascontiguousarray(w.numpy())
    mat, path = h.debug_align_post(w, width)
    ref = AO.filter_matrix(w, width).numpy()
    assert np.abs(mat - ref).max() <= MAT_TOL
    ref_path = AO.dtw(mat)
    assert path.shape == ref_path.shape and (path == ref_path).all()


# ----------------------------------------------------------------------------------------------------- end to end
def windows(n=16):
    dims = setup()[0]
    rng = np.random.default_rng(42)
    texts, frames = [], []
    for b in range(n):
        k = [0, 1, 5, 17, 40, 3, 9, 24][b % 8] if b != 6 else 0
        texts.append([int(t) for t in rng.integers(300, dims.eot, k)])
        frames.append(int([3000, 2400, 1200, 600, 80, 3000, 2, 1777][b % 8]))
    return texts, frames


@functools.lru_cache(maxsize=1)
def oracle_runs():
    dims, oracle, _ = setup()
    mel = mel_inputs(16)
    enc = oracle.encode(mel)
    texts, frames = windows()
    out = []
    for b in range(16):
        weights, tp = AO.capture_window(oracle, enc[b], START, texts[b], frames[b])
        out.append((weights, tp))
    return mel, texts, frames, out


def row_of_frame(path, F):
    """text index of the first path entry at each frame"""
    out = np.full(F, -1)
    for r, f in path[::-1]:
        out[f] = r
    return out


@pytest.mark.parametrize("width", [7, 1, 9])
def test_end_to_end(width):
    mel, texts, frames, ref = oracle_runs()
    h = handle()
    paths, probs = h.align(mel, START, texts, frames, width)
    robust, n_text, worst_agree = 0, 0, 1.0
    for b in range(16):
        weights, tp = ref[b]
        assert len(probs[b]) == len(texts[b])
        if not texts[b]:
            assert paths[b].shape == (0, 2)
            continue
        n_text += 1
        assert np.abs(np.log(np.asarray(probs[b])) - np.log(tp)).max() <= 2 * LOGIT_TOL
        want = AO.dtw(AO.filter_matrix(weights, width).numpy())
        g = torch.Generator().manual_seed(b)
        stable = all(np.array_equal(AO.dtw(AO.filter_matrix(
            weights * np.exp(PROBE_SIGMA * torch.randn(weights.shape, generator=g).numpy()), width).numpy()), want)
            for _ in range(3))
        if stable:
            robust += 1
            assert np.array_equal(paths[b], want), b
        # every case: the text index the path assigns to each frame agrees with the oracle's on >= 98 % of the frames
        # (exact identity hangs on single-frame boundary decisions between neighbouring peaks)
        p = paths[b]
        agree = np.mean(row_of_frame(p, frames[b] // 2) == row_of_frame(want, frames[b] // 2))
        worst_agree = min(worst_agree, float(agree))
        assert agree >= 0.98, (b, agree)
        # whatever the robustness, the path is a valid monotone DTW path over the window
        assert tuple(p[0]) == (0, 0) and tuple(p[-1]) == (len(texts[b]), frames[b] // 2 - 1)
        assert (np.diff(p, axis=0) >= 0).all() and (np.diff(p, axis=0).sum(1) >= 1).all()
    print(f"width {width}: {robust} of {n_text} cases robust, worst frame agreement {worst_agree:.3f}")
    assert robust * 5 >= n_text


def test_capture_matches_oracle():
    mel, texts, frames, ref = oracle_runs()
    h = handle()
    cap = h.debug_align_capture(mel, START, texts, frames, len(HEADS))
    worst = 0.0
    for b in range(16):
        if not texts[b]:
            continue
        want = ref[b][0]  # [A, n + 1, F]
        got = cap[b, :, : want.shape[1], : want.shape[2]]
        big = want >= 1e-3 * want.max(-1, keepdims=True)
        worst = max(worst, float(np.abs(np.log(got[big]) - np.log(want[big])).max()))
        assert np.abs(got - want).max() <= CAPTURE_TOL * want.max()  # (exp(0.25) - 1 of the row peak, at most)
    print(f"capture: worst log-probability error {worst:.3g}")
    assert worst <= CAPTURE_TOL


def test_batch_invariance():
    mel, texts, frames, _ = oracle_runs()
    h = handle()
    paths, probs = h.align(mel, START, texts, frames, 7)
    for b in range(16):
        p1, q1 = h.align(np.ascontiguousarray(mel[b:b + 1]), START, texts[b:b + 1], frames[b:b + 1], 7)
        assert np.array_equal(p1[0], paths[b]) and q1[0] == probs[b], b


def test_encoder_cache_generate_then_align():
    dims = setup()[0]
    mel, texts, frames, _ = oracle_runs()
    one = np.ascontiguousarray(mel[3:4])
    plain = handle()
    want = plain.align(one, START, texts[3:4], frames[3:4], 7)
    launches_plain = plain.align_timing()["launches"]
    h = handle()
    h.set_option("encoder_cache", 1)
    h.generate(one, np.asarray([PROMPT], np.int32), beam_size=1)  # 1 row: the persistent pass, swizzled cross K/V
    got = h.align(one, START, texts[3:4], frames[3:4], 7)
    launches = h.align_timing()["launches"]
    assert np.array_equal(got[0][0], want[0][0]) and got[1] == want[1]
    # no encoder: conv1, conv2, 7 per layer, ln_post are gone; the cross-K/V GEMM reran once (linear layout)
    assert launches == launches_plain - (3 + 7 * dims.n_enc_layers)
    again = h.align(one, START, texts[3:4], frames[3:4], 7)
    assert np.array_equal(again[0][0], want[0][0])
    assert h.align_timing()["launches"] == launches - 1


def test_validation():
    dims = setup()[0]
    h = handle()
    mel = np.ascontiguousarray(mel_inputs(16)[:1])
    ok = dict(start=START, text=[[400, 401]], nf=[3000], width=7)
    bad = [dict(start=[dims.lang_first, dims.transcribe]), dict(start=START + [dims.no_timestamps]),
           dict(start=START + [dims.no_timestamps + 5]), dict(text=[[400, dims.eot]]), dict(text=[[-1]]),
           dict(text=[[400] * (dims.n_text_ctx - len(START))]), dict(nf=[1]), dict(nf=[3001]), dict(width=8),
           dict(width=33), dict(width=-1), dict(text=[[400], [401]])]
    h.align(mel, ok["start"], ok["text"], ok["nf"], ok["width"])
    for case in bad:
        a = {**ok, **case}
        with pytest.raises(ValueError):
            h.align(mel, a["start"], a["text"], a["nf"], a["width"])
    m = models.Whisper(None, _handles=[h])
    with pytest.raises(ValueError):
        m.align(models.StorageView.from_array(mel), START, [[400], [401]], 3000)
    res = m.align(models.StorageView.from_array(mel), START, [[]], 3000)
    assert res[0].alignments == [] and res[0].text_token_probs == []
    res = m.align(models.StorageView.from_array(mel), START, [[400, 401]], 3000)
    assert isinstance(res[0], models.WhisperAlignmentResult) and len(res[0].text_token_probs) == 2
