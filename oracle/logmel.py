"""Oracle: log-mel front end (numpy restatement of ``wis/audio.py``).

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.

Follows, step for step:
  * constants                 wis/audio.py:17-25
  * ``pad_or_trim``           wis/audio.py:28-51 (numpy branch :43-49)
  * ``mel_filters``           wis/audio.py:54-69 -- the asset
    ``wis/assets/mel_filters.npz`` is ``librosa.filters.mel(sr=16000, n_fft=400,
    n_mels=80)`` (docstring :59-63); ``slaney_mel_filterbank`` below recomputes
    that published algorithm and reproduces the asset BIT-EXACTLY
    (sha256 of the raw f32 = 85818f15...b405498, checked in tests).
  * ``log_mel_spectrogram``   wis/audio.py:72-103
      - periodic Hann(400)                       :93
      - torch.stft(n_fft=400, hop=160, center=True -> reflect pad 200,
        onesided) -> [201, 3001]                 :94
      - drop last frame, |.|^2                   :95
      - filters @ magnitudes                     :97-98
      - clamp(1e-10).log10()                     :100
      - max(x, global_max - 8)                   :101
      - (x + 4) / 4                              :102

PINNED: ``tests/test_oracle_logmel.py`` checks this restatement against golden
outputs of the reference function itself (``tests/golden/logmel_*.npz``).
"""
from __future__ import annotations

import hashlib

import numpy as np

SAMPLE_RATE = 16000
N_FFT = 400
N_MELS = 80
HOP_LENGTH = 160
CHUNK_LENGTH = 30
N_SAMPLES = CHUNK_LENGTH * SAMPLE_RATE  # 480000
N_FRAMES = N_SAMPLES // HOP_LENGTH  # 3000
N_BINS = N_FFT // 2 + 1  # 201

MEL_FILTERS_SHA256 = "85818f156f7e189453901a515e4726d270d307f976e161cf9403e8caab405498"


def _hz_to_mel(f):
    f = np.asanyarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(
        f >= min_log_hz,
        min_log_mel + np.log(np.maximum(f, 1e-30) / min_log_hz) / logstep,
        f / f_sp,
    )


def _mel_to_hz(m):
    m = np.asanyarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(
        m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m
    )


def slaney_mel_filterbank(sr: int = SAMPLE_RATE, n_fft: int = N_FFT, n_mels: int = N_MELS) -> np.ndarray:
    """Slaney-normalised triangular mel filterbank, float32 [n_mels, n_fft//2+1].

    Published algorithm of ``librosa.filters.mel(htk=False, norm='slaney')``,
    which is how the reference asset was produced (wis/audio.py:59-63).
    """
    fft_freqs = np.fft.rfftfreq(n_fft, 1.0 / sr)
    mel_pts = _mel_to_hz(np.linspace(_hz_to_mel(0.0), _hz_to_mel(sr / 2.0), n_mels + 2))
    fdiff = np.diff(mel_pts)
    ramps = np.subtract.outer(mel_pts, fft_freqs)
    w = np.zeros((n_mels, len(fft_freqs)), dtype=np.float32)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        w[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_pts[2 : n_mels + 2] - mel_pts[:n_mels])
    w *= enorm[:, None]
    return w + np.float32(0.0)  # canonicalise -0.0 (the asset holds +0.0)


def mel_filters_sha256(w: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(w, dtype=np.float32).tobytes()).hexdigest()


def pad_or_trim(array: np.ndarray, length: int = N_SAMPLES) -> np.ndarray:
    """wis/audio.py:43-49 -- keep the first ``length`` samples, else right-pad zeros."""
    array = np.asarray(array)
    n = array.shape[-1]
    if n > length:
        array = array[..., :length]
    elif n < length:
        pad = [(0, 0)] * array.ndim
        pad[-1] = (0, length - n)
        array = np.pad(array, pad)
    return array


def hann_periodic(n: int = N_FFT) -> np.ndarray:
    # torch.hann_window(N) is the periodic window: 0.5 - 0.5 cos(2 pi k / N)
    k = np.arange(n, dtype=np.float64)
    return (0.5 - 0.5 * np.cos(2.0 * np.pi * k / n)).astype(np.float32)


def log_mel_spectrogram(audio: np.ndarray, filters: np.ndarray | None = None) -> np.ndarray:
    """float32 [n] (any n >= 201) -> float32 [80, n // 160].

    The reference is always called on a padded 480000-sample window
    (main.py:607-614) and then returns [80, 3000].
    """
    audio = np.asarray(audio, dtype=np.float32)
    assert audio.ndim == 1
    if filters is None:
        filters = slaney_mel_filterbank()
    half = N_FFT // 2
    padded = np.pad(audio, (half, half), mode="reflect")  # center=True, reflect
    n_frames_all = 1 + (padded.shape[0] - N_FFT) // HOP_LENGTH
    idx = np.arange(N_FFT)[None, :] + HOP_LENGTH * np.arange(n_frames_all)[:, None]
    frames = padded[idx] * hann_periodic()[None, :]  # f32 [frames, 400]
    spec = np.fft.rfft(frames.astype(np.float64), axis=1)  # [frames, 201]
    power = (spec.real**2 + spec.imag**2)[:-1].T.astype(np.float32)  # drop last frame -> [201, frames-1]
    mel = filters.astype(np.float32) @ power  # [80, frames-1]
    log_spec = np.log10(np.maximum(mel, np.float32(1e-10))).astype(np.float32)
    log_spec = np.maximum(log_spec, log_spec.max() - np.float32(8.0))
    return ((log_spec + np.float32(4.0)) / np.float32(4.0)).astype(np.float32)


def log_mel_batch(pcm_list, filters: np.ndarray | None = None) -> np.ndarray:
    """What main.py:603-617 builds: each utterance padded/trimmed to 30 s -> [B, 80, 3000]."""
    if filters is None:
        filters = slaney_mel_filterbank()
    return np.stack([log_mel_spectrogram(pad_or_trim(np.asarray(p, np.float32)), filters) for p in pcm_list])


# ---------------------------------------------------------------------------
# Synthetic input recipe fixed by SURVEY.md section 8(d)
# ---------------------------------------------------------------------------
def synth_utterance(n_samples: int, seed: int = 1234) -> np.ndarray:
    """0.3*sin(2 pi (200+300 t) t) + 0.05*N(0,1), 16 kHz mono float32."""
    rng = np.random.default_rng(seed)
    t = np.arange(n_samples, dtype=np.float64) / SAMPLE_RATE
    x = 0.3 * np.sin(2.0 * np.pi * (200.0 + 300.0 * t) * t) + 0.05 * rng.standard_normal(n_samples)
    return x.astype(np.float32)
