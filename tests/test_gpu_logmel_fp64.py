"""The log-mel front end (csrc/logmel.cu) against a float64 restatement of its own, at every framing edge of the kernel's
geometry, on loud tones over quiet noise and around the 1e-10 clamp.  Every input goes through the production launch,
``Handle.frontend(0, n_mels).logmel(pcm, offsets, n_samples)``.

Three tiers, as in test_gpu_kernels.py and test_gpu_encoder.py:
  * exact: what must hold bit for bit -- all-zero input, frames that read only padding, the s16 path against the f32
    path on s / 32768, ragged batches against solo runs, overlapping windows of one buffer against copies;
  * bound: every cell within a first-order running-error bound derived from the kernel's arithmetic (``kernel_bound``);
  * bar: every cell within 1e-4 of float64 (the project's log-mel bar), at 80 and 128 bins.

The float64 reference does not reuse oracle/logmel.py, which windows its frames in float32: trim or zero-pad to 480000
samples, reflect-pad 200 at each end, multiply by the float32 periodic Hann window in float64, ``np.fft.rfft`` in
float64, |X|^2, the float32 Slaney filterbank in float64, log10(max(., 1e-10)), the window's max - 8 floor, (x + 4) / 4.

The kernel's geometry, which the signal catalogue is derived from: CTA x of the 94 per window holds frames 32x..32x+31
and reads padded-window indices [5120x - 200, 5120x + 5160) (negative indices and indices >= 480000 reflect); it skips
the DFT, writing log10(1e-10) directly, when that whole span lies in the zero padding, which only CTAs x <= 92 can do.
Frame f reads [160f - 200, 160f + 200)."""
import functools

import numpy as np
import pytest

from oracle import logmel as om
from tests.test_gpu_kernels import bits, note_ratio, worst_ratio

N_SAMPLES, N_FRAMES, N_FFT, HOP, N_BINS = om.N_SAMPLES, om.N_FRAMES, om.N_FFT, om.HOP_LENGTH, om.N_BINS
FT = 32                                 # frames per CTA
SPAN = (FT - 1) * HOP + N_FFT           # 5360 samples feed one CTA
N_CTAS = -(-N_FRAMES // FT)             # 94
BAR = 1e-4
U = 2.0 ** -24                          # unit roundoff of float32
U64 = 2.0 ** -53
MELS = (80, 128)
HANN = om.hann_periodic()               # float32, symmetric: hann[400 - n] == hann[n]
FILTERS = {m: om.slaney_mel_filterbank(n_mels=m) for m in MELS}


# ------------------------------------------------------------------------------------------------ kernel geometry
def cta_first_index(x):
    return HOP * FT * x - N_FFT // 2


def cta_skips(x, n):
    """the kernel's all_zero predicate: CTA x's whole span lies past the audio and short of the right reflection"""
    s0 = cta_first_index(x)
    return s0 >= min(n, N_SAMPLES) and s0 + SPAN <= N_SAMPLES


def reflect(idx):
    idx = np.abs(idx)
    return np.where(idx >= N_SAMPLES, 2 * (N_SAMPLES - 1) - idx, idx)


FRAME_IDX = reflect(np.arange(N_FFT)[None, :] + HOP * np.arange(N_FRAMES)[:, None] - N_FFT // 2)  # [3000, 400]


def padding_frames(n):
    """[3000] bool: frames all of whose 400 samples (after reflection) lie past the audio"""
    return (FRAME_IDX >= min(n, N_SAMPLES)).all(1)


# ------------------------------------------------------------------------------------------------ signal catalogue
EDGE_CTAS = (1, 2, 47, 92)
LENGTHS = sorted({0, 1, 2, 199, 200, 201, 399, 400, 401,
                  *(cta_first_index(x) + d for x in EDGE_CTAS for d in (0, 1)),
                  cta_first_index(N_CTAS - 1), cta_first_index(N_CTAS - 1) + 1,
                  479958, 479959, 479960, 479998, 479999, 480000, 480001, 480200, 560000})
TONES = (100.0, 440.0, 1000.0, 2500.0, 7900.0)
TONE_NOISE = (3e-3, 1e-3)
CLAMP_SIGMAS = (3e-6, 1e-5)  # white noise whose mel power sits around 1e-10


def _t(n):
    return np.arange(n, dtype=np.float64) / om.SAMPLE_RATE


@functools.lru_cache(maxsize=None)
def catalogue():
    """name -> PCM (float32, or int16 for the s16 path).  Lengths are broadband noise so every sample matters."""
    out = {}
    for n in LENGTHS:
        rng = np.random.default_rng([7, n])
        out[f"noise_len{n}"] = (0.3 * rng.standard_normal(n)).astype(np.float32)
    for f0 in TONES:
        for bg in TONE_NOISE:
            rng = np.random.default_rng([11, int(f0), int(bg * 1e4)])
            x = 0.99 * np.sin(2 * np.pi * f0 * _t(N_SAMPLES)) + bg * rng.standard_normal(N_SAMPLES)
            out[f"tone{f0:g}Hz_noise{bg:g}"] = x.astype(np.float32)
    sq = np.where((np.arange(N_SAMPLES) // 8) % 2 == 0, 32767, -32768).astype(np.int16)  # 1 kHz, full scale
    out["square1kHz_s16"] = sq
    for sigma in CLAMP_SIGMAS:
        out[f"clamp_noise{sigma:g}"] = (sigma * np.random.default_rng([13, int(sigma * 1e7)]).standard_normal(N_SAMPLES)).astype(np.float32)
    # a 3e-6 -> 3e-5 swell: mel power crosses 1e-10 inside the window, and the floor (max - 8) lies below the clamp
    out["clamp_swell"] = (np.geomspace(3e-6, 3e-5, N_SAMPLES) * np.random.default_rng(17).standard_normal(N_SAMPLES)).astype(np.float32)
    for n, seed in ((61440, 1234), (171008, 1235), (467968, 1236)):
        out[f"synth_{n}"] = om.synth_utterance(n, seed)
    return out


def as_float64(pcm):
    return pcm.astype(np.float64) / 32768.0 if pcm.dtype == np.int16 else pcm.astype(np.float64)


# ------------------------------------------------------------------------------------------------ float64 reference
def frames64(x, *, length=N_SAMPLES, pad_mode="reflect", left_zero=False, drop_first=False):
    """[3000, 400] float64 frames of the padded window.  The keywords restate known defects for the comparator
    self-tests: trim to another length, numpy's 'symmetric' reflection, zero padding at the left edge, and the
    first of torch's 3001 frames dropped instead of the last."""
    x = om.pad_or_trim(om.pad_or_trim(np.asarray(x, np.float64), length))
    p = np.pad(x, N_FFT // 2, mode=pad_mode)
    if left_zero:
        p[: N_FFT // 2] = 0.0
    idx = np.arange(N_FFT)[None, :] + HOP * (np.arange(N_FRAMES)[:, None] + (1 if drop_first else 0))
    return p[idx]


def power64(fr, hann=HANN):
    s = np.fft.rfft(fr * hann.astype(np.float64), axis=1)
    return s.real, s.imag


def finish(lg, M=None):
    M = lg.max() if M is None else M
    return (np.maximum(lg, M - 8.0) + 4.0) / 4.0


def log10_mel(re, im, fb):
    mel = (re**2 + im**2) @ fb.astype(np.float64).T  # [3000, n_mels]
    return mel, np.log10(np.maximum(mel, 1e-10))


# ------------------------------------------------------------------------------------------------ error bound
def fold(fr):
    """the kernel's even / odd halves of each frame, exact: ev[n] = x[n] + x[400 - n], od[n] = x[n] - x[400 - n]
    for 0 < n < 200, x[0] and x[200] alone -> [3000, 201] each"""
    a = fr[:, :N_BINS]
    b = np.zeros_like(a)
    b[:, 1:N_FFT // 2] = fr[:, N_FFT - 1:N_FFT // 2:-1]
    return a + b, a - b


@functools.lru_cache(maxsize=1)
def twiddles():
    """float64 |hann * cos| and |hann * sin| [201 n, 201 k], and per mel table the chain weights
    W2[m, q] = w[m, q] * (end_m - q): sum over the mel FMA chain's partial sums = p @ W2.T"""
    n = np.arange(N_BINS)
    r = np.outer(n, n) % N_FFT
    h = HANN[:N_BINS].astype(np.float64)[:, None]
    c, s = np.abs(h * np.cos(2 * np.pi * r / N_FFT)), np.abs(h * np.sin(2 * np.pi * r / N_FFT))
    w2 = {}
    for m, fb in FILTERS.items():
        fb = fb.astype(np.float64)
        end = np.array([np.nonzero(row)[0].max() + 1 for row in fb])
        w2[m] = fb * np.maximum(end[:, None] - n[None, :], 0)
    return c, s, w2


def dft_bound(fr):
    """first-order bound on |kernel - exact| of re and im, [3000, 201] each.  The kernel folds in float32 (one
    rounding of e_n), reads float32 tables fl(hann * cos) (one rounding of c_nk) and accumulates the 201 products
    e_n c_nk of each bin in float64, where a product of two floats is exact: u * 2 sum |e_n c_nk| plus the float64
    chain's 201 roundings."""
    c, s, _ = twiddles()
    ev, od = fold(fr)
    return [(2 * U + N_BINS * U64) * (np.abs(e) @ t) for e, t in ((ev, c), (od, s))]


@functools.lru_cache(maxsize=None)
def cached(name):
    """re, im and their bounds of a catalogue signal (shared by both bin counts)"""
    fr = frames64(as_float64(catalogue()[name]))
    re, im = power64(fr)
    dre, dim = dft_bound(fr)
    return re, im, dre, dim


def kernel_bound(re, im, dre, dim, n_mels):
    """-> (float64 reference [n_mels, 3000], bound [n_mels, 3000]).

    power p = re^2 + im^2 in float64, rounded once to float32:  dp = (2|re| + dre) dre + (2|im| + dim) dim + u p
    mel: float32 FMA chain over the nonzero weights (w >= 0):    dmel = fb @ dp + u * sum of partial sums (p @ W2.T)
    log10f:                                                       dlg = dmel / (ln 10 max(mel - dmel, 1e-10)) + 2 ulp
    window max M = max lg:                                        dM = max(dlg at the argmax, max(lg + dlg) - M)
    floor F = fl(M - 8):                                          dF = dM + u |M - 8|
    max(lg, F), 1-Lipschitz in both:                              dF where lg + dlg <= F - dF (floored either way),
                                                                  else max(dlg, dF)
    (x + 4) / 4:                                                  / 4, plus one rounding"""
    _, _, w2 = twiddles()
    fb = FILTERS[n_mels].astype(np.float64)
    p = re**2 + im**2
    dp = (2 * np.abs(re) + dre) * dre + (2 * np.abs(im) + dim) * dim + (U + 2 * U64) * p
    mel, lg = log10_mel(re, im, FILTERS[n_mels])
    dmel = dp @ fb.T + U * ((p + dp) @ w2[n_mels].T)
    dlg = dmel / (np.log(10.0) * np.maximum(mel - dmel, 1e-10)) + 2 * np.spacing(np.abs(lg).astype(np.float32))
    M = lg.max()
    dM = max(float(dlg.flat[np.argmax(lg)]), float((lg + dlg).max() - M))
    F, dF = M - 8.0, dM + U * abs(M - 8.0)
    out = finish(lg, M)
    bnd = 0.25 * np.where(lg + dlg <= F - dF, dF, np.maximum(dlg, dF)) + U * (np.abs(out) + 1.0)
    return out.T, bnd.T


def within(got, ref, bnd):
    return bool(np.all(np.abs(got.astype(np.float64) - ref) <= bnd))


# ------------------------------------------------------------------------------------------------ CPU: catalogue
def test_catalogue_reaches_every_framing_edge():
    cat = catalogue()
    lengths = {len(v) for v in cat.values()}
    for x in range(N_CTAS - 1):  # the all_zero predicate flips between 5120x - 200 and 5120x - 199
        assert cta_skips(x, cta_first_index(x)) and not cta_skips(x, cta_first_index(x) + 1)
    assert not any(cta_skips(N_CTAS - 1, n) for n in (0, cta_first_index(N_CTAS - 1)))  # the last CTA never skips
    for x in EDGE_CTAS + (N_CTAS - 1,):
        assert {cta_first_index(x), cta_first_index(x) + 1} <= lengths, x
    # frame 0 reflects samples 1..200: the lengths around 200 and 400 cut through its left reflection and its span
    assert {0, 1, 2, 199, 200, 201, 399, 400, 401} <= lengths
    # the last frame reads 479640..479999 and, reflected, 479998 down to 479959: the 40 samples it reads twice
    vals, counts = np.unique(FRAME_IDX[-1], return_counts=True)
    twice = vals[counts == 2]
    assert twice.min() == 479959 and twice.max() == 479998 and twice.size == 40
    assert {479958, 479959, 479960, 479998, 479999, 480000, 480001} <= lengths
    assert max(lengths) > N_SAMPLES + 200  # trimmed by more than the reflection reads
    # CTA x's first frame reads only padding at 5120x - 200 and one sample of audio at 5120x - 199
    for x in EDGE_CTAS + (N_CTAS - 1,):
        n = cta_first_index(x)
        assert padding_frames(n)[FT * x] and not padding_frames(n + 1)[FT * x], x
    assert not padding_frames(479958).any() and padding_frames(0).all()
    for f0 in TONES:
        for bg in TONE_NOISE:
            assert f"tone{f0:g}Hz_noise{bg:g}" in cat
    sq = cat["square1kHz_s16"]
    assert sq.dtype == np.int16 and sq.min() == -32768 and sq.max() == 32767
    # mel power straddles the clamp: some cells below 1e-10, some above, at both bin counts
    for name in ("clamp_noise3e-06", "clamp_noise1e-05", "clamp_swell"):
        re, im, _, _ = cached(name)
        for m in MELS:
            mel = log10_mel(re, im, FILTERS[m])[0]
            assert (mel < 1e-10).any() and (mel > 1e-10).any(), (name, m)
    assert {"synth_61440", "synth_171008", "synth_467968"} <= set(cat)


# ------------------------------------------------------------------------------------------------ CPU: comparator
def defect_features(kind):
    """-> (n_mels, correct reference, bound, reference with one known defect) on a catalogue signal"""
    cat = catalogue()
    name = {"s16_32767": "square1kHz_s16", "batch_floor": "clamp_swell", "trim_479999": "noise_len480001",
            "table80_at_128": "synth_171008"}.get(kind, "tone440Hz_noise0.001")
    n_mels = 128 if kind == "table80_at_128" else 80
    pcm = cat[name]
    x = as_float64(pcm)
    ref, bnd = kernel_bound(*cached(name), n_mels)
    fb = FILTERS[n_mels]
    if kind == "left_zero":
        re, im = power64(frames64(x, left_zero=True))
    elif kind == "symmetric_reflect":
        re, im = power64(frames64(x, pad_mode="symmetric"))
    elif kind == "symmetric_hann":
        k = np.arange(N_FFT)
        re, im = power64(frames64(x), (0.5 - 0.5 * np.cos(2 * np.pi * k / (N_FFT - 1))).astype(np.float32))
    elif kind == "drop_first":
        re, im = power64(frames64(x, drop_first=True))
    elif kind == "trim_479999":
        re, im = power64(frames64(x, length=N_SAMPLES - 1))
    elif kind == "s16_32767":
        re, im = power64(frames64(pcm.astype(np.float64) / 32767.0))
    else:
        re, im = power64(frames64(x))
    if kind == "table80_at_128":
        lg = log10_mel(re, im, FILTERS[128])[1]
        lg[:, :80] = log10_mel(re, im, FILTERS[80])[1]
        return n_mels, ref, bnd, finish(lg).T
    lg = log10_mel(re, im, fb)[1]
    if kind == "batch_floor":  # the quiet window floored at a loud window's max
        re2, im2, _, _ = cached("tone440Hz_noise0.001")
        return n_mels, ref, bnd, finish(lg, log10_mel(re2, im2, fb)[1].max()).T
    return n_mels, ref, bnd, finish(lg).T


DEFECTS = ["left_zero", "symmetric_reflect", "symmetric_hann", "drop_first", "trim_479999", "batch_floor", "s16_32767",
           "table80_at_128"]


@pytest.mark.parametrize("kind", DEFECTS)
def test_comparator_rejects_defect(kind):
    n_mels, ref, bnd, bad = defect_features(kind)
    assert ref.shape == bad.shape == bnd.shape == (n_mels, N_FRAMES)
    assert not within(bad.astype(np.float32), ref, bnd), kind
    assert np.abs(bad - ref).max() > 10 * bnd.max() or worst_ratio(bad, ref, bnd) > 10, kind


def test_comparator_accepts_reference_rounded_to_float32():
    n_mels, ref, bnd, _ = defect_features("symmetric_hann")
    assert within(ref.astype(np.float32), ref, bnd)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def fe():
    from willow_inference_server_b200 import _lib

    return {m: _lib.Handle.frontend(0, m) for m in MELS}


def run(h, pcms):
    """one ragged batch out of one buffer -> [B, n_mels, 3000]"""
    n = np.array([len(p) for p in pcms], np.int32)
    off = np.concatenate([[0], np.cumsum(n[:-1], dtype=np.int64)]).astype(np.int64)
    return h.logmel(np.concatenate(pcms), off, n)


@pytest.fixture(scope="module")
def features(fe):
    """catalogue name -> {n_mels: features}, computed in two ragged batches (f32, s16) per bin count"""
    cat = catalogue()
    out = {name: {} for name in cat}
    for m in MELS:
        for dt in (np.float32, np.int16):
            names = [k for k, v in cat.items() if v.dtype == dt]
            got = run(fe[m], [cat[k] for k in names])
            for k, g in zip(names, got):
                out[k][m] = g
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("n_mels", MELS)
def test_all_zero_input_is_minus_1p5(fe, n_mels):
    got = run(fe[n_mels], [np.zeros(N_SAMPLES, np.float32), np.zeros(0, np.float32), np.zeros(12345, np.float32)])
    assert np.all(bits(got) == bits(np.float32(-1.5)))
    got = run(fe[n_mels], [np.zeros(N_SAMPLES + 7, np.int16)])
    assert np.all(bits(got) == bits(np.float32(-1.5)))


@pytest.mark.gpu
@pytest.mark.parametrize("n_mels", MELS)
def test_padding_frames_exact(features, n_mels):
    """a frame that reads only padding has mel power 0, so log10(1e-10) = -10 floored at the window's own max M - 8:
    fp32((max(-10, M - 8) + 4) * 0.25), M recovered from the output's maximum.  Skipped CTAs and computed frames alike."""
    checked = 0
    for n in LENGTHS:
        got = features[f"noise_len{n}"][n_mels]
        pad = padding_frames(n)
        if not pad.any():
            continue
        top = got.max()
        M = np.float32(top * np.float32(4.0) - np.float32(4.0))
        want = np.float32((np.maximum(np.float32(-10.0), np.float32(M - np.float32(8.0))) + np.float32(4.0)) * np.float32(0.25))
        assert np.all(bits(got[:, pad]) == bits(want)), n
        assert got.min() == want, n
        checked += int(pad.sum())
    assert checked > 0


@pytest.mark.gpu
@pytest.mark.parametrize("n_mels", MELS)
def test_s16_equals_f32_on_s_over_32768(fe, n_mels):
    rng = np.random.default_rng(21)
    s = [rng.integers(-32768, 32768, n).astype(np.int16) for n in (N_SAMPLES, 479999, cta_first_index(47) + 1, 401, 1)]
    s[0][:4] = (-32768, 32767, -32768, 32767)
    s[0][-3:] = (32767, -32768, 32767)
    s.append(catalogue()["square1kHz_s16"])
    got16 = run(fe[n_mels], s)
    got32 = run(fe[n_mels], [(v.astype(np.float32) / np.float32(32768.0)) for v in s])
    assert np.array_equal(bits(got16), bits(got32))


@pytest.mark.gpu
@pytest.mark.parametrize("n_mels", MELS)
def test_ragged_batch_equals_solo_runs(fe, n_mels):
    """loud, silent and near-clamp utterances in one batch: a window's floor comes from its own maximum only"""
    cat = catalogue()
    rng = np.random.default_rng(23)
    pcms = [cat["tone1000Hz_noise0.001"], np.zeros(30000, np.float32), (1e-5 * rng.standard_normal(200000)).astype(np.float32),
            cat["synth_61440"], cat["noise_len10041"], cat["noise_len560000"], np.zeros(0, np.float32),
            cat["clamp_noise3e-06"], cat["noise_len1"]]
    got = run(fe[n_mels], pcms)
    for i, p in enumerate(pcms):
        assert np.array_equal(bits(got[i]), bits(run(fe[n_mels], [p])[0])), i


@pytest.mark.gpu
@pytest.mark.parametrize("n_mels", MELS)
def test_overlapping_windows_equal_copies(fe, n_mels):
    rng = np.random.default_rng(29)
    n = 75 * om.SAMPLE_RATE
    buf = (0.3 * np.sin(np.arange(n) * 0.05) + 0.05 * rng.standard_normal(n)).astype(np.float32)
    off = np.array([1, 3, 160001, 240007, 479999, 480001, 719999], np.int64)
    ns = np.array([N_SAMPLES, 479999, cta_first_index(92) + 1, 10041, N_SAMPLES + 1, 5, n - 719999], np.int32)
    got = fe[n_mels].logmel(buf, off, ns)
    want = run(fe[n_mels], [buf[o:o + k].copy() for o, k in zip(off, ns)])
    assert np.array_equal(bits(got), bits(want))


@pytest.mark.gpu
@pytest.mark.parametrize("n_mels", MELS)
def test_within_float64_bound_and_bar(features, n_mels):
    worst_bar, worst_name = 0.0, None
    failures = []
    for name in catalogue():
        got = features[name][n_mels]
        ref, bnd = kernel_bound(*cached(name), n_mels)
        note_ratio(f"log-mel {n_mels} bins vs float64 bound", worst_ratio(got, ref, bnd))
        err = float(np.abs(got.astype(np.float64) - ref).max())
        if err > worst_bar:
            worst_bar, worst_name = err, name
        if not within(got, ref, bnd):
            failures.append(("bound", name, worst_ratio(got, ref, bnd)))
        if err > BAR:
            failures.append(("bar", name, err))
    print(f"log-mel {n_mels} bins: worst |kernel - float64| {worst_bar:.3g} ({worst_name})")
    assert not failures, failures
