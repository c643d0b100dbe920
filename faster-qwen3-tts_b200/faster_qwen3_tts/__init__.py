"""H100-native drop-in for andimarafioti/faster-qwen3-tts (hot path only; see DESIGN.md)."""
__version__ = "0.3.2+b200.1"

__all__ = ["FasterQwen3TTS", "__version__"]


def __getattr__(name):
    if name == "FasterQwen3TTS":
        from .model import FasterQwen3TTS
        return FasterQwen3TTS
    raise AttributeError(name)
