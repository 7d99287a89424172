"""TTSRequest — same fields and defaults as the reference
(`/root/reference/src/auralis/common/definitions/requests.py:135-204`).

Differences, all outside the hot path: language auto-detection uses ``langid`` when it is installed and
otherwise falls back to "en" with a warning (the reference hard-requires langid).

``enhance_speech`` (off by default) cleans the speaker references before conditioning, as the reference's
``EnhancedAudioProcessor`` does (enhancer.py:34-153: VAD trim, spectral gating, clarity shaping, loudness normalisation,
each behind its ``audio_config`` flag), but on the GPU (``xtts_enhance``) and only when ``speaker_files`` is a list,
like the reference.  Where the reference would fail (audio too short for a VAD frame or a 400 ms loudness block, a
non-finite result) the original file is used, with a warning.  Unlike the reference, ``speaker_files`` is not rewritten to
enhanced temporary files: the request keeps its paths, and the engine enhances while it conditions (the speaker cache
key includes ``audio_config``).  The audio is loaded at ``audio_config.sample_rate`` with torchaudio's sinc resampler,
not librosa's soxr.

Additions (not in the reference): ``seed`` (reproducible sampling) and ``speed``, the speaking rate in [0.25, 4.0] (> 1 is
faster; the reference offers speed only in its OpenAI server, as a CPU phase vocoder on the finished waveform).  Here it
time-scales the GPT latents on the GPU before the vocoder, as Coqui's ``Xtts.inference(speed=...)`` does, so the pitch
stays; the tokens are the same at every speed.
"""
from __future__ import annotations

import uuid
import warnings
from dataclasses import dataclass, field
from functools import lru_cache
from typing import AsyncGenerator, Callable, List, Optional, Union

from .config import SPEED_MAX, SPEED_MIN

SUPPORTED_LANGUAGES = ("en", "es", "fr", "de", "it", "pt", "pl", "tr", "ru", "nl", "cs", "ar", "zh-cn", "hu", "ko",
                       "ja", "hi", "auto", "")


@lru_cache(maxsize=1024)
def get_language(text: str) -> str:
    """requests.py:97-113."""
    try:
        import langid
    except ImportError:
        warnings.warn("langid is not installed: language='auto' falls back to 'en'")
        return "en"
    detected = langid.classify(text)[0].strip()
    return "zh-cn" if detected == "zh" else detected


def validate_language(language: str) -> str:
    if language not in SUPPORTED_LANGUAGES:
        raise ValueError(f"Language {language} not supported. Must be one of {SUPPORTED_LANGUAGES}")
    return language


@dataclass
class AudioPreprocessingConfig:
    """The reference's speaker-file enhancement settings (enhancer.py:12-31), same fields and defaults; applied by
    ``xtts_enhance`` when a request sets ``enhance_speech``."""
    sample_rate: int = 22050
    normalize: bool = True
    trim_silence: bool = True
    remove_noise: bool = True
    enhance_speech: bool = True
    # VAD
    vad_threshold: float = 0.02
    vad_frame_length: int = 1024 * 4
    # noise reduction
    noise_reduce_margin: float = 1.0
    noise_reduce_frames: int = 25
    # clarity
    enhance_amount: float = 1.0
    # loudness target
    target_lufs: float = -18.0


@dataclass
class TTSRequest:
    text: Union[AsyncGenerator[str, None], str, List[str]]
    speaker_files: Union[Union[str, List[str]], Union[bytes, List[bytes]]]
    context_partial_function: Optional[Callable] = None
    start_time: Optional[float] = None
    enhance_speech: bool = False
    audio_config: AudioPreprocessingConfig = field(default_factory=AudioPreprocessingConfig)
    language: str = "auto"
    request_id: str = field(default_factory=lambda: uuid.uuid4().hex)
    load_sample_rate: int = 22050
    sound_norm_refs: bool = False
    # voice conditioning (requests.py:179-181)
    max_ref_length: int = 60
    gpt_cond_len: int = 30
    gpt_cond_chunk_len: int = 4
    # generation (requests.py:183-190)
    stream: bool = False
    temperature: float = 0.75
    top_p: float = 0.85
    top_k: int = 50
    repetition_penalty: float = 5.0
    length_penalty: float = 1.0     # carried, not consumed by the engine (SURVEY App. A.3)
    do_sample: bool = True          # carried, not consumed by the engine
    # additions (not in the reference): reproducible sampling, speaking rate
    seed: Optional[int] = None
    speed: float = 1.0

    def __post_init__(self):
        if not (SPEED_MIN <= self.speed <= SPEED_MAX):                 # NaN fails the comparison too
            raise ValueError(f"speed {self.speed} out of range [{SPEED_MIN}, {SPEED_MAX}]")
        if self.language == "auto" and len(self.text) > 0:
            self.language = get_language(self.text if isinstance(self.text, str) else " ".join(self.text))
        validate_language(self.language)

    def enhance_config(self) -> Optional[AudioPreprocessingConfig]:
        """`audio_config` when the speaker files are to be enhanced (requests.py:199-203: a list and enhance_speech)."""
        return self.audio_config if self.enhance_speech and isinstance(self.speaker_files, list) else None

    def infer_language(self):
        if self.language == "auto":
            self.language = get_language(self.text)

    def copy(self) -> "TTSRequest":
        """requests.py:250-277."""
        fields = {k: getattr(self, k) for k in (
            "text", "speaker_files", "enhance_speech", "audio_config", "language", "request_id", "load_sample_rate",
            "sound_norm_refs", "max_ref_length", "gpt_cond_len", "gpt_cond_chunk_len", "stream", "temperature", "top_p",
            "top_k", "repetition_penalty", "length_penalty", "do_sample", "seed", "speed")}
        return TTSRequest(**fields)
