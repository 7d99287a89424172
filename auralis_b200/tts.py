"""TTS — the public façade, same surface as the reference's
(`/root/reference/src/auralis/core/tts.py:27-361`): ``TTS().from_pretrained(...)``,
``generate_speech`` (sync, optional streaming), ``generate_speech_async``,
``prepare_for_streaming_generation``, ``split_requests``, ``shutdown``.
"""
from __future__ import annotations

import asyncio
import json
import logging
import os
import time
import uuid
from functools import partial
from typing import AsyncGenerator, Dict, Generator, List, Optional, Union

from .base import MODEL_REGISTRY, BaseAsyncTTSEngine
from .output import TTSOutput
from .requests import TTSRequest
from .scheduler import TwoPhaseScheduler

logger = logging.getLogger("auralis_b200")


class TTS:
    def __init__(self, scheduler_max_concurrency: int = 10, vllm_logging_level=logging.DEBUG):
        # `vllm_logging_level` is accepted for signature compatibility (tts.py:27); there is no vLLM here.
        self.scheduler: Optional[TwoPhaseScheduler] = TwoPhaseScheduler(scheduler_max_concurrency)
        self.tts_engine: Optional[BaseAsyncTTSEngine] = None
        self.concurrency = scheduler_max_concurrency
        self.loop = None

    def _ensure_event_loop(self):
        if not self.loop:
            try:
                self.loop = asyncio.get_running_loop()
            except RuntimeError:
                self.loop = asyncio.new_event_loop()
                asyncio.set_event_loop(self.loop)

    def from_pretrained(self, model_name_or_path: str, **kwargs):
        """tts.py:53-89: config.json["model_type"] selects the engine; kwargs (gpt_model=...) are forwarded."""
        from . import engine as _engine  # noqa: F401  (registers "xtts")
        self._ensure_event_loop()
        from .weights import resolve_model_file
        try:
            with open(resolve_model_file(model_name_or_path, "config.json"), "r") as f:      # local dir, else Hub repo (tts.py:72-84)
                config = json.load(f)
        except (FileNotFoundError, NotADirectoryError) as e:
            raise ValueError(f"Could not load model from {model_name_or_path} neither locally or online: {e}")
        kwargs.setdefault("max_concurrency", max(self.concurrency, 1))
        self.tts_engine = MODEL_REGISTRY[config["model_type"]].from_pretrained(model_name_or_path, **kwargs)
        return self

    def from_engine(self, engine: BaseAsyncTTSEngine):
        """Attach an already constructed engine (used by tests/bench to skip the disk round trip)."""
        self._ensure_event_loop()
        self.tts_engine = engine
        return self

    async def prepare_for_streaming_generation(self, request: TTSRequest):
        """tts.py:91-105."""
        cc = self.tts_engine.conditioning_config
        if cc.speaker_embeddings or cc.gpt_like_decoder_conditioning:
            enh = request.enhance_config()
            gpt_cond_latent, speaker_embeddings = await self.tts_engine.get_audio_conditioning(
                request.speaker_files, **({"enhance": enh} if enh is not None else {}))
            return partial(self.tts_engine.get_generation_context, gpt_cond_latent=gpt_cond_latent,
                           speaker_embeddings=speaker_embeddings)

    async def _prepare_generation_context(self, input_request: TTSRequest):
        """tts.py:107-158 (phase 1)."""
        input_request.start_time = time.time()
        if input_request.context_partial_function:
            gens, request_ids, speaker_embeddings, cond = await input_request.context_partial_function(input_request)
        else:
            gens, request_ids, speaker_embeddings, cond = await self.tts_engine.get_generation_context(input_request)
        parallel_inputs = [
            {"generator": gen,
             "speaker_embedding": speaker_embeddings[i] if isinstance(speaker_embeddings, list) else speaker_embeddings,
             "multimodal_data": cond[i] if isinstance(cond, list) else cond,
             "request": input_request}
            for i, gen in enumerate(gens)]
        return {"parallel_inputs": parallel_inputs, "request": input_request}

    async def _second_phase_fn(self, gen_input: Dict):
        """tts.py:160-194 (phase 2), wrapped by the reference in `track_generation` (performance.py:105-151)."""
        from .metrics import track
        async for chunk in self.tts_engine.process_tokens_to_speech(
                generator=gen_input["generator"], speaker_embeddings=gen_input["speaker_embedding"],
                multimodal_data=gen_input["multimodal_data"], request=gen_input["request"]):
            track(chunk, self.tts_engine)
            yield chunk

    async def generate_speech_async(self, request: TTSRequest) -> Union[AsyncGenerator[TTSOutput, None], TTSOutput]:
        """tts.py:196-233."""
        self._ensure_event_loop()

        async def process_chunks():
            acc = TTSOutput.Accumulator()               # = combine_outputs(chunks), copied chunk by chunk as they arrive
            try:
                async for chunk in self.scheduler.run(inputs=request, request_id=request.request_id,
                                                      first_phase_fn=self._prepare_generation_context,
                                                      second_phase_fn=self._second_phase_fn):
                    if request.stream:
                        yield chunk
                    else:
                        acc.add(chunk)
            except Exception as e:
                logger.error(f"Error during speech generation: {e}")
                raise
            if not request.stream:
                yield acc.result()

        if request.stream:
            return process_chunks()
        async for result in process_chunks():
            return result

    @staticmethod
    def split_requests(request: TTSRequest, max_length: int = 100000) -> List[TTSRequest]:
        """tts.py:236-254."""
        if len(request.text) <= max_length:
            return [request]
        out = []
        for i in range(0, len(request.text), max_length):
            c = request.copy()
            c.text = request.text[i:i + max_length]
            c.request_id = uuid.uuid4().hex
            out.append(c)
        return out

    async def _process_multiple_requests(self, requests: List[TTSRequest]) -> TTSOutput:
        """tts.py:257-308: sub-requests run concurrently, audio is concatenated in order."""
        async def one(sub):
            acc = TTSOutput.Accumulator()
            async for chunk in self.scheduler.run(inputs=sub, request_id=sub.request_id,
                                                  first_phase_fn=self._prepare_generation_context,
                                                  second_phase_fn=self._second_phase_fn):
                acc.add(chunk)
            return acc.result()
        parts = await asyncio.gather(*[asyncio.ensure_future(one(r)) for r in requests])
        return parts[0] if len(parts) == 1 else TTSOutput.combine_outputs(list(parts))

    def generate_speech(self, request: TTSRequest) -> Union[Generator[TTSOutput, None, None], TTSOutput]:
        """tts.py:310-355."""
        self._ensure_event_loop()
        requests = self.split_requests(request)
        if request.stream:
            def streaming_wrapper():
                for sub in requests:
                    agen = self.scheduler.run(inputs=sub, request_id=sub.request_id,
                                              first_phase_fn=self._prepare_generation_context,
                                              second_phase_fn=self._second_phase_fn)
                    try:
                        while True:
                            yield self.loop.run_until_complete(agen.__anext__())
                    except StopAsyncIteration:
                        pass
            return streaming_wrapper()
        return self.loop.run_until_complete(self._process_multiple_requests(requests))

    def generate_speech_batch(self, requests: List[TTSRequest]) -> List[TTSOutput]:
        """Several independent requests in one call (what `asyncio.gather(generate_speech_async...)` does in the
        reference's async test, tests/integration/test_generate_audio_async.py:10-55)."""
        self._ensure_event_loop()

        async def run_all():
            return await asyncio.gather(*[self.generate_speech_async(r) for r in requests])
        return self.loop.run_until_complete(run_all())

    async def shutdown(self):
        if self.scheduler:
            await self.scheduler.shutdown()
        if self.tts_engine and hasattr(self.tts_engine, "shutdown"):
            await self.tts_engine.shutdown()
