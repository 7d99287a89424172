"""auralis_b200 — H100-native XTTSv2 hot path behind the Auralis engine/plugin API.

Public surface mirrors the reference (`/root/reference/src/auralis/__init__.py`):
``TTS``, ``TTSRequest``, ``TTSOutput``.  Imports are lazy so that ``import auralis_b200``
works on a CPU box (the CUDA library is only loaded when an engine is created).
"""
__version__ = "0.1.0"


def __getattr__(name):
    if name == "TTS":
        from .tts import TTS
        return TTS
    if name == "TTSRequest":
        from .requests import TTSRequest
        return TTSRequest
    if name == "TTSOutput":
        from .output import TTSOutput
        return TTSOutput
    raise AttributeError(name)
