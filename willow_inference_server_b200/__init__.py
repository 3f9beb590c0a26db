"""willow_inference_server_b200 -- H100-native Whisper hot path for toverainc/willow-inference-server.

Use it where WIS imports ctranslate2 / wis.audio (INTEGRATION.md):

    import willow_inference_server_b200 as ctranslate2
    from willow_inference_server_b200.audio import log_mel_spectrogram, pad_or_trim, chunk_iter, find_longest_common_sequence

Everything numeric runs in libwisb200.so (hand-written sm_90a CUDA, include/wisb200.h); this package is the thin
host-side mirror of the reference's Python surface.  Importing it does not need a GPU; calling it does.
"""
from . import audio, models, weights  # noqa: F401
from .models import StorageView, Whisper, WhisperGenerationResult, get_supported_compute_types, set_random_seed  # noqa: F401

__all__ = ["audio", "models", "weights", "StorageView", "Whisper", "WhisperGenerationResult",
           "get_supported_compute_types", "set_random_seed"]
__version__ = "0.1.0"
