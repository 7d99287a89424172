"""INTEGRATION.md path B as code: the native engine registered as a plugin of the REFERENCE's own façade.

A maintainer who keeps `auralis.TTS`, its `TwoPhaseScheduler` and its HTTP server installs this package next to the
reference and adds one line where the reference registers its models (`src/auralis/models/__init__.py`):

    import auralis_b200.reference_plugin as p; p.register()          # registers model_type "xtts_b200"

`config.json["model_type"] = "xtts_b200"` then makes `auralis.TTS().from_pretrained(...)` build this engine
(`src/auralis/core/tts.py:84-87`, `models/registry.py:1-4`).  The class below derives from the reference's OWN
`BaseAsyncTTSEngine` (`models/base.py:57-224`: an ABC that is also a `torch.nn.Module`, abstract `get_generation_context`,
`process_tokens_to_speech`, `get_memory_usage_curve`) and yields the reference's OWN `TTSOutput`; every tensor op happens in
`libxtts_b200.so` behind `auralis_b200.engine.XTTSv2Engine`.  tests/test_reference_plugin.py drives it through the
reference's unmodified `TTS` (one-shot, streaming, failing chunk)."""
from __future__ import annotations

from typing import Optional


def make_reference_engine(ref_base=None, ref_output=None):
    """-> a subclass of the reference's `auralis.models.base.BaseAsyncTTSEngine` wrapping `XTTSv2Engine`."""
    import torch
    if ref_base is None:
        from auralis.models import base as ref_base                    # noqa: PLC0415 — the reference package
    if ref_output is None:
        from auralis.common.definitions.output import TTSOutput as ref_output      # noqa: PLC0415
    from .engine import XTTSv2Engine

    class XTTSv2B200Engine(ref_base.BaseAsyncTTSEngine):
        model_type = "xtts_b200"

        def __init__(self, inner: XTTSv2Engine):
            super().__init__()
            self.inner = inner
            # no nn.Parameters: the weights live in HBM inside the library — `device` / `dtype` are answered explicitly
            self.max_concurrency = getattr(inner, "max_concurrency", None)
            self.get_memory_usage_curve()

        @classmethod
        def from_pretrained(cls, pretrained_model_name_or_path: str, gpt_model: Optional[str] = None, **kwargs):
            """stands in for XTTSv2Engine.from_pretrained (XTTSv2.py:235-310); same arguments"""
            return cls(XTTSv2Engine.from_pretrained(pretrained_model_name_or_path, gpt_model, **kwargs))

        @property
        def conditioning_config(self):
            return ref_base.ConditioningConfig(speaker_embeddings=True, gpt_like_decoder_conditioning=True)

        @property
        def device(self):
            return self.inner.device

        @property
        def dtype(self):
            return self.inner.dtype

        def get_memory_usage_curve(self):
            self.max_gb_for_vllm_model = self.inner.get_memory_usage_curve()    # the attribute XTTSv2.py:169 sets
            return self.max_gb_for_vllm_model

        async def get_audio_conditioning(self, audio_reference, *args, **kwargs):
            return await self.inner.get_audio_conditioning(audio_reference, *args, **kwargs)

        async def get_generation_context(self, request, gpt_cond_latent=None, speaker_embeddings=None):
            return await self.inner.get_generation_context(request, gpt_cond_latent, speaker_embeddings)

        async def process_tokens_to_speech(self, generator, speaker_embeddings=None, multimodal_data=None, request=None):
            async for out in self.inner.process_tokens_to_speech(generator, speaker_embeddings, multimodal_data, request):
                yield ref_output(array=out.array, start_time=out.start_time, token_length=out.token_length)

        async def shutdown(self):
            await self.inner.shutdown()

    return XTTSv2B200Engine


def register(name: str = "xtts_b200"):
    """Adds the engine to the reference's registry (`auralis.models.registry.register_model`)."""
    from auralis.models.registry import register_model                  # noqa: PLC0415 — the reference package
    cls = make_reference_engine()
    register_model(name, cls)
    return cls
