"""sopro_b200 — H100-native engine for the Sopro TTS hot path behind the reference's API.

    from sopro_b200 import SoproTTS          # drop-in for `from sopro import SoproTTS`

Importing the package does not need a GPU; constructing a model does (no CPU fallback)."""
from .config import SoproTTSConfig  # noqa: F401

__version__ = "0.1.0"
__all__ = ["SoproTTS", "SoproTTSConfig", "encode_flac", "FlacStreamEncoder", "encode_stream_flac", "WordTiming",
           "detect_watermark", "denoise", "level_live", "LiveLeveller", "level_stream", "level_stream_batch", "Cue", "CueFit", "parse_cues"]


def __getattr__(name):  # lazy: keep `import sopro_b200` cheap and GPU-free
    if name in ("encode_flac", "FlacStreamEncoder", "encode_stream_flac"):
        from . import flac

        return getattr(flac, name)
    if name in ("level_live", "LiveLeveller", "level_stream", "level_stream_batch"):
        from . import loudness

        return getattr(loudness, name)
    if name in ("Cue", "CueFit"):
        from . import cues

        return getattr(cues, name)
    if name == "parse_cues":
        from .cues import parse

        return parse
    if name == "detect_watermark":
        from .watermark import detect_watermark

        return detect_watermark
    if name == "denoise":
        from .denoising import denoise

        return denoise
    if name == "SoproTTS":
        from .model import SoproTTS

        return SoproTTS
    if name == "WordTiming":
        from .timestamps import WordTiming

        return WordTiming
    if name == "PreparedReference":
        from .prefill import PreparedReference

        return PreparedReference
    raise AttributeError(name)
