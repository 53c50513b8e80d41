"""qwen3-tts_b200 — H100-native (sm_90a) hot paths of Qwen3-TTS behind the reference's Python API.

Importable as `qwen3_tts_b200` (see the shim module at the repo root; the directory name carries a hyphen).
"""
from .config import AudioFormat, CodecConfig, SamplingParams, StackConfig, TTSConfig  # noqa: F401

__all__ = ["TTSConfig", "StackConfig", "SamplingParams", "CodecConfig", "AudioFormat",
           "Qwen3TTSModel", "Qwen3TTSTokenizer", "VoiceClonePromptItem", "Voice"]

_PUBLIC = {"Qwen3TTSModel", "Qwen3TTSTokenizer", "VoiceClonePromptItem", "Voice"}


def __getattr__(name):
    """`from qwen3_tts_b200 import Qwen3TTSModel, Qwen3TTSTokenizer, VoiceClonePromptItem` — the reference's public
    names (qwen_tts/__init__.py:21-22), resolved lazily so that importing the package stays light."""
    if name in _PUBLIC:
        from . import model
        return getattr(model, name)
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
