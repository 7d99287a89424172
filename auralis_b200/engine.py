"""XTTSv2Engine — the reference's engine plugin (`/root/reference/src/auralis/models/xttsv2/XTTSv2.py`)
re-hosted on the native CUDA library.  Same public methods, argument meaning and error behaviour:

* ``from_pretrained(path, gpt_model=..., max_concurrency=...)``            XTTSv2.py:235-310
* ``await get_audio_conditioning(speaker_files, ...) -> (cond, g)``         XTTSv2.py:579-615
* ``await get_generation_context(request, gpt_cond_latent, speaker_embeddings)
      -> (generators, request_ids, speaker_embeddings, gpt_embed_inputs)``   XTTSv2.py:690-760
* ``process_tokens_to_speech(generator, speaker_embeddings, multimodal_data, request)``  XTTSv2.py:762-814
* ``await shutdown()``                                                       XTTSv2.py:818

What is different underneath (SURVEY.md App. B "diverge" items): no vLLM, no second GPT pass (latents are
captured during decode), no semaphore/sleep around the vocoder, per-sequence position counters.  All
tensor work happens in ``libxtts_b200.so``; this file only tokenises, submits and awaits completions.
"""
from __future__ import annotations

import asyncio
import hashlib
import threading
import time
from dataclasses import asdict
from pathlib import Path
from typing import AsyncGenerator, Dict, List, Optional, Tuple, Union

import numpy as np

from . import native
from .base import BaseAsyncTTSEngine, ConditioningConfig, register_model
from .config import XTTSDims
from . import output as _output
from .output import TTSOutput
from .requests import TTSRequest
from .speakers import SpeakerSlots, SpeakerSlotsFull
from .text import XTTSTokenizer
from .weights import load_model_dir


def tune_host_allocator() -> bool:
    """Keeps large host buffers on the malloc heap instead of fresh `mmap` regions.  Every finished chunk arrives as a new
    2.7 MB float32 array (and is copied once more into its request's buffer); glibc serves allocations that large with `mmap`
    and returns them with `munmap`, so each one is page-faulted in again — 0.3-1 s per 4 600 audio-seconds of output on the
    hosts measured, serialised across threads by the process's mm lock.  `mallopt(M_MMAP_THRESHOLD, 1 GiB)` +
    `mallopt(M_TRIM_THRESHOLD, max)` makes the heap keep and reuse those pages.  Process-wide, so it is the APPLICATION's call
    (bench.py makes it; `XTTSv2Engine(tune_malloc=True)` does too).  Returns False where glibc's mallopt is unavailable."""
    import ctypes
    try:
        libc = ctypes.CDLL("libc.so.6")
        ok = libc.mallopt(-3, 1 << 30) == 1            # M_MMAP_THRESHOLD
        return (libc.mallopt(-1, 2 ** 31 - 1) == 1) and ok      # M_TRIM_THRESHOLD
    except Exception:      # noqa: BLE001 — not glibc
        return False


class ChunkOutput:
    """What the reference reads off vLLM's RequestOutput (XTTSv2.py:785-799): finished flag + token ids.
    `partial`: a first-audio piece (engine option `early_emit_tokens`) — the audio of the chunk's leading tokens, delivered
    while the rest of the chunk is still decoding; the final piece then carries only the remaining samples."""

    def __init__(self, request_id: str, token_ids, wav, result, partial: bool = False):
        self.request_id = request_id
        self.finished = True
        self.partial = partial
        self.token_ids = list(token_ids)
        self.wav = wav
        self.result = result


def load_audio(source: Union[str, Path, bytes], sampling_rate: int) -> np.ndarray:
    """Mono float32 in [-1,1] at `sampling_rate` (common/utilities.py:72-97: mean over channels, torchaudio's sinc
    resampler — on the GPU while an `XTTSv2Engine` is alive, see `_resample` — and clip).  RIFF/WAV — integer PCM and
    IEEE float — is decoded here (torchaudio.load needs a codec backend this image does not ship).  FLAC (optionally
    behind an ID3v2 tag) is decoded losslessly on the GPU while an `XTTSv2Engine` is alive and scaled v / 2^(bits - 1)
    into the same [frames, channels] float32 array an integer WAV gives, so a FLAC reference conditions exactly like the
    same PCM in a WAV; a corrupt stream raises ValueError.  Any other container, and FLAC with no engine alive, goes
    through torchaudio.load when it can."""
    from .output import _parse_flac, _parse_riff_wav
    if isinstance(source, (bytes, bytearray)):
        blob = bytes(source)
    else:
        with open(str(source), "rb") as f:
            blob = f.read()
    parsed = _parse_riff_wav(blob)
    if parsed is None:
        parsed = _parse_flac(blob)
    if parsed is None:
        import io
        import torchaudio
        wav, sr = torchaudio.load(io.BytesIO(blob) if isinstance(source, (bytes, bytearray)) else str(source))
        a = wav.mean(dim=0).numpy()
    else:
        frames, sr = parsed
        a = frames.mean(axis=1)
    if sr != sampling_rate:
        a = _resample(np.ascontiguousarray(a, np.float32), int(sr), int(sampling_rate))     # torchaudio's sinc resampler, as the reference
    return np.clip(a, -1.0, 1.0).astype(np.float32)


class XTTSv2Engine(BaseAsyncTTSEngine):
    model_type = "xtts"

    def __init__(self, dims: XTTSDims, gpt_state, core_state, *, device: int = 0, devices: Optional[List[int]] = None,
                 precision: str = "fp16", max_concurrency: int = 64, max_speakers: int = 32,
                 tokenizer_file: Optional[str] = None, early_emit_tokens: int = 0, voc_segment: Optional[int] = None,
                 tune_malloc: bool = False, **_):
        """`devices=[0, 1, ...]`: data parallelism inside the product (north_star: "requests shard data-parallel across the
        8-GPU box") — one native engine (full weight replica, own scheduler thread, own streams) per listed GPU in THIS
        process; every text chunk goes to the engine with the least work in flight, results are re-assembled in request
        order by the façade as before.  `max_concurrency` is per GPU.  Default: the single GPU `device`."""
        prec = {"fp32": native.PRECISION_FP32, "bf16": native.PRECISION_BF16, "fp16": native.PRECISION_FP16}[precision]
        if tune_malloc:
            tune_host_allocator()
        self.dims = dims
        self.precision = precision
        self.devices = [int(d) for d in devices] if devices else [int(device)]
        if len(set(self.devices)) != len(self.devices):
            raise ValueError("devices must be distinct CUDA ordinals")
        self.device_index = self.devices[0]
        self.max_concurrency = max_concurrency
        self.natives = [native.NativeEngine(dims, device=d, precision=prec, max_batch=max_concurrency, max_speakers=max_speakers)
                        for d in self.devices]
        self.native = self.natives[0]
        if len(self.natives) == 1:
            self.native.load_state(gpt_state, core_state)
        else:                                               # replicas load side by side (the C calls release the GIL)
            errs: list = []

            def _load(ne):
                try:
                    ne.load_state(gpt_state, core_state)
                except BaseException as e:      # noqa: BLE001 — re-raised below
                    errs.append(e)
            ts = [threading.Thread(target=_load, args=(ne,)) for ne in self.natives]
            [t.start() for t in ts]
            [t.join() for t in ts]
            if errs:
                raise errs[0]
        if voc_segment is not None:
            for ne in self.natives:
                ne.set_option("voc_segment", int(voc_segment))
        self.tokenizer = XTTSTokenizer(dims.gpt.n_text_tokens, dims.gpt.max_text_tokens, tokenizer_file)
        self.mel_bos_token_id = dims.gpt.start_audio_token
        self.mel_eos_token_id = dims.gpt.stop_audio_token
        self.max_speakers = max_speakers
        # > 0: streaming requests get the audio of their first chunk's leading tokens as soon as those are decoded
        # (time-to-first-audio, SURVEY §8f-3); 0 = one TTSOutput per chunk, exactly like the reference
        self.early_emit_tokens = int(early_emit_tokens)
        self._spks = [SpeakerSlots(max_speakers) for _ in self.natives]     # per GPU: key -> native slot, pins
        self._spk = self._spks[0]
        self._spk_arrays: Dict[str, Tuple["_SpeakerArray", "_SpeakerArray"]] = {}    # reference key -> host (cond, g) pair
        self._next_id = 1
        self._id_lock = threading.Lock()
        self._waiters: Dict[int, tuple] = {}            # sid -> (loop, box, slot, device index, work units)
        self._wlock = threading.Lock()
        self._load = [0] * len(self.natives)            # text ids of the chunks in flight per GPU (under _wlock)
        self._stop = False
        self._parked = 0
        self._paused = False       # set while a caller drives the native completion queue itself (bench device arm)
        self._pollers = [threading.Thread(target=self._poll_loop, args=(i,), name=f"xtts-poll-{i}", daemon=True)
                         for i in range(len(self.natives))]
        [t.start() for t in self._pollers]
        _output.register_gpu_provider(self)             # change_speed, FLAC in / out and resampling run here while it lives

    # ---- plugin API -------------------------------------------------------------------------
    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: str, gpt_model: Optional[str] = None, **kwargs):
        import os
        from .weights import resolve_model_file
        dims, gpt_state, core_state = load_model_dir(pretrained_model_name_or_path, gpt_model)
        if gpt_model and gpt_model.endswith(".safetensors"):
            gsrc = os.path.dirname(gpt_model)
        else:
            gsrc = gpt_model if gpt_model else os.path.join(pretrained_model_name_or_path, "gpt")
        tok = resolve_model_file(gsrc, "tokenizer.json", required=False)      # local directory or Hub repo (XTTSv2.py:84)
        return cls(dims, gpt_state, core_state, tokenizer_file=tok if tok and os.path.exists(tok) else None, **kwargs)

    @property
    def conditioning_config(self) -> ConditioningConfig:
        return ConditioningConfig(speaker_embeddings=True, gpt_like_decoder_conditioning=True)

    @property
    def device(self):
        import torch
        return torch.device("cuda", int(getattr(self, "device_index", 0)))

    @property
    def dtype(self):
        import torch
        return {"bf16": torch.bfloat16, "fp16": torch.float16}.get(self.precision, torch.float32)

    def get_memory_usage_curve(self):
        """XTTSv2.py:152-171 fits a polynomial to measured vLLM footprints; here the footprint is known exactly from the
        geometry: weights + per-slot state (paged KV for a full-length sequence, latent ring, token rows) x max_concurrency
        + the vocoder workspace.  Sets (and returns) `max_gb_for_vllm_model`, the attribute the reference's engine exposes."""
        g, v = self.dims.gpt, self.dims.voc
        kv_elem = 2 if self.precision in ("bf16", "fp16") else 4
        w_elem = 2 if self.precision in ("bf16", "fp16") else 4
        gpt_w = g.layers * (4 * g.hidden * g.hidden + 2 * g.hidden * g.ff) * w_elem
        pages = -(-(g.max_prompt_rows + g.max_audio_tokens) // 32)
        per_slot = pages * 32 * 2 * g.layers * g.hidden * kv_elem + g.max_audio_tokens * g.hidden * 4 + 3 * g.max_audio_tokens * 4
        tz = v.z_frames(g.max_audio_tokens)
        widest = max((v.init_ch >> (i + 1)) * int(np.prod(v.up_rates[: i + 1])) for i in range(len(v.up_rates)))
        voc_ws = 8 * tz * (5 * widest * 4 + (5 * widest * 2 if self.precision in ("bf16", "fp16") else 0) + v.hop * 4)
        total = gpt_w + per_slot * (self.max_concurrency + 1) + voc_ws
        self.max_gb_for_vllm_model = total / 2 ** 30
        return self.max_gb_for_vllm_model

    async def _acquire_speaker(self, key: str, timeout_s: float = 120.0):
        """SpeakerSlots.acquire, waiting (not failing) while every slot is pinned by chunks in flight."""
        t0 = time.monotonic()
        while True:
            try:
                return self._spk.acquire(key)
            except SpeakerSlotsFull:
                if time.monotonic() - t0 > timeout_s:
                    raise
                await asyncio.sleep(0.005)

    async def get_audio_conditioning(self, audio_reference, max_ref_length=30, gpt_cond_len=6, gpt_cond_chunk_len=6,
                                     librosa_trim_db=None, sound_norm_refs=False, load_sr=22050, enhance=None):
        """XTTSv2.py:409-468,579-615: -> (gpt_cond_latents [1,32,H], speaker_embedding [1,d,1]) computed on the GPU
        by ``xtts_condition`` and cached per reference (the per-speaker cache of SURVEY §3.4).

        `enhance` (an AudioPreprocessingConfig): each file is first enhanced on the GPU (``xtts_enhance``, the reference's
        TTSRequest.preprocess_audio, requests.py:214-247): loaded at ``enhance.sample_rate``, enhanced, quantised to 16
        bits as the reference's temporary WAV is, then resampled to `load_sr`.  A file the enhancer rejects
        (XTTS_ERR_INVALID: too short, non-finite result) is used as it is, with a RuntimeWarning."""
        if not isinstance(audio_reference, (bytes, str, Path, list)):
            raise AssertionError(f"audio_reference must be a string, byte or a list but it is {type(audio_reference)}")
        paths = audio_reference if isinstance(audio_reference, list) else [audio_reference]
        hk = hashlib.sha256()
        for p in paths:
            if isinstance(p, (bytes, bytearray)):
                hk.update(p)
            else:                           # a file: its identity is path + size + mtime (a replaced file is a new speaker)
                import os
                try:
                    stt = os.stat(str(p))
                    hk.update(f"{p}|{stt.st_size}|{stt.st_mtime_ns}".encode())
                except OSError:
                    hk.update(str(p).encode())
        hk.update(f"{max_ref_length}|{gpt_cond_len}|{gpt_cond_chunk_len}|{sound_norm_refs}|{load_sr}".encode())
        if enhance is not None:
            hk.update(f"|enhance|{sorted(asdict(enhance).items())}".encode())
        key = hk.hexdigest()
        cached = self._spk_arrays.get(key)
        if cached is not None:
            # no native call on a hit: xtts_get_speaker would wait for the scheduler thread's current iteration and stall
            # every other coroutine of this loop behind it.  Whether the slot still holds this speaker is checked (and the
            # pair uploaded again if not) when a chunk pins it.
            return cached
        while True:
            slot, pending, owner = await self._acquire_speaker(key)
            if owner:
                def work():
                    audios22 = []
                    for p in paths:
                        a = self._enhanced(p, enhance, load_sr) if enhance is not None else load_audio(p, load_sr)
                        a = a[: load_sr * max_ref_length]
                        if sound_norm_refs:
                            a = (a / np.abs(a).max()) * 0.75
                        audios22.append(a)
                    if len(audios22) == 1:
                        self.native.condition(slot, audios22[0], _resample(audios22[0], load_sr, 16000), gpt_cond_len,
                                              gpt_cond_chunk_len)
                        return
                    # several references: d-vector per file, averaged; GPT latents on the concatenation
                    # (XTTSv2.py:446-466)
                    gs = []
                    for a in audios22:
                        self.native.condition(slot, a, _resample(a, load_sr, 16000), gpt_cond_len, gpt_cond_chunk_len)
                        gs.append(self.native.get_speaker(slot)[1])
                    full = np.concatenate(audios22)
                    self.native.condition(slot, full, _resample(audios22[0], load_sr, 16000), gpt_cond_len, gpt_cond_chunk_len)
                    c, _ = self.native.get_speaker(slot)
                    self.native.set_speaker(slot, c, np.mean(np.stack(gs), axis=0))
                fut = asyncio.ensure_future(asyncio.to_thread(work))
                try:
                    await asyncio.shield(fut)
                except asyncio.CancelledError:
                    # the worker thread is still writing into `slot`: the entry stays "being computed" (never evicted, never
                    # a hit) until the thread has really finished, and only then is it dropped
                    fut.add_done_callback(lambda f, k=key: (f.exception(), self._spk.failed(k, RuntimeError("conditioning cancelled"))))
                    raise
                except BaseException as e:
                    self._spk.failed(key, e if isinstance(e, Exception) else RuntimeError("conditioning failed"))
                    raise
                self._spk.ready(key)
            elif pending is not None:                      # another request is computing this speaker right now
                await asyncio.wrap_future(pending)
            cond, g = self.native.get_speaker(slot)
            if self._spk.holds(key, slot):              # not recycled between the wake-up and the read-back
                break
        pair = (_SpeakerArray(cond[None], slot, key), _SpeakerArray(g.reshape(1, -1, 1), slot, key))
        if len(self._spk_arrays) >= 4 * self.max_speakers:           # host copies are 130 KB each: a small bounded cache
            self._spk_arrays.pop(next(iter(self._spk_arrays)))
        self._spk_arrays[key] = pair
        return pair

    def _enhanced(self, source, cfg, load_sr: int) -> np.ndarray:
        """`source` at `load_sr` after the GPU enhancer; the original audio when the enhancer rejects it."""
        import warnings
        try:
            a = self.native.enhance(load_audio(source, cfg.sample_rate), cfg)
        except native.NativeError as e:
            if e.code != native.ERR_INVALID:
                raise
            warnings.warn(f"enhance_speech: {e}; using the original speaker file", RuntimeWarning, stacklevel=2)
            return load_audio(source, load_sr)
        return np.clip(_resample(a, cfg.sample_rate, load_sr), -1.0, 1.0).astype(np.float32)     # as load_audio leaves it

    def register_speaker(self, cond_latents: np.ndarray, d_vector: np.ndarray, dev: int = 0) -> Tuple["_SpeakerArray", "_SpeakerArray"]:
        """Pre-computed conditioning (the pair `prepare_for_streaming_generation` hands back, tts.py:91-105) uploaded to
        GPU `dev` (index into `devices`).  Raises SpeakerSlotsFull when every slot is pinned by chunks in flight."""
        natives = getattr(self, "natives", None) or [self.native]
        spks = getattr(self, "_spks", None) or [self._spk]
        c = np.ascontiguousarray(cond_latents, np.float32).reshape(self.dims.gpt.n_cond_latents, self.dims.gpt.hidden)
        g = np.ascontiguousarray(d_vector, np.float32).reshape(-1)
        key = hashlib.sha256(c.tobytes() + g.tobytes()).hexdigest()
        slot, pending, owner = spks[dev].acquire(key)
        if owner:
            try:
                natives[dev].set_speaker(slot, c, g)
            except BaseException as e:
                spks[dev].failed(key, e if isinstance(e, Exception) else RuntimeError("set_speaker interrupted"))
                raise
            spks[dev].ready(key)
        elif pending is not None:
            pending.result(timeout=120)
        return _SpeakerArray(c[None], slot, key, dev), _SpeakerArray(g.reshape(1, -1, 1), slot, key, dev)

    async def _pin_speaker(self, cond, g, timeout_s: float = 120.0, dev: int = 0) -> int:
        """Slot of GPU `dev` holding this conditioning pair, pinned for one chunk.  A pair whose slot was recycled since it
        was handed out (LRU eviction), or that was computed on another GPU, is uploaded (again) from the host arrays
        instead of selecting another speaker's voice."""
        spks = getattr(self, "_spks", None) or [self._spk]
        t0 = time.monotonic()
        while True:
            key, slot = getattr(cond, "key", None), getattr(cond, "slot", None)
            if key is not None and slot is not None and (getattr(cond, "dev", 0) or 0) == dev and spks[dev].pin(key, slot):
                return slot
            try:
                cond, g = self.register_speaker(np.asarray(cond), np.asarray(g), dev)
            except SpeakerSlotsFull:
                if time.monotonic() - t0 > timeout_s:
                    raise
                await asyncio.sleep(0.005)

    def prepare_text_tokens(self, text: str, language: str) -> List[List[int]]:
        """XTTSv2.py:506-543: per chunk [bos] + ids + [eos]."""
        chunks = self.tokenizer.batch_encode_with_split(text, language)
        return [[self.tokenizer.bos_token_id] + ids + [self.tokenizer.eos_token_id] for ids in chunks]

    async def get_generation_context(self, request: TTSRequest, gpt_cond_latent=None, speaker_embeddings=None):
        if gpt_cond_latent is None or speaker_embeddings is None:
            enh = request.enhance_config() if hasattr(request, "enhance_config") else None
            gpt_cond_latent, speaker_embeddings = await self.get_audio_conditioning(
                request.speaker_files, request.max_ref_length, request.gpt_cond_len, request.gpt_cond_chunk_len,
                **({"enhance": enh} if enh is not None else {}))
        token_lists = self.prepare_text_tokens(request.text, request.language)
        generators, request_ids = [], []
        base_seed = request.seed if getattr(request, "seed", None) is not None else int.from_bytes(hashlib.sha256(request.request_id.encode()).digest()[:6], "little")
        num_beams = getattr(request, "num_beams", 1)
        if num_beams > 1 and num_beams > self.max_concurrency:
            raise ValueError(f"num_beams {num_beams} exceeds the engine's {self.max_concurrency} batch slots")
        for seq_index, ids in enumerate(token_lists):
            # a beam chunk (num_beams > 1) is delivered whole: its best hypothesis is known only when its group ends
            stream_first = request.stream and seq_index == 0 and num_beams == 1
            sp = native.Sampling(temperature=request.temperature, top_p=request.top_p, top_k=request.top_k,
                                 repetition_penalty=request.repetition_penalty,
                                 max_tokens=self.dims.gpt.max_audio_tokens, stop_token=self.mel_eos_token_id,
                                 seed=base_seed, seq_seed=seq_index, vocode=True, priority=seq_index,
                                 early_tokens=self.early_emit_tokens if stream_first else 0,
                                 speed=getattr(request, "speed", 1.0),     # (the reference's own TTSRequest has none)
                                 num_beams=num_beams, length_penalty=getattr(request, "length_penalty", 1.0),
                                 do_sample=getattr(request, "do_sample", True))
            rid = f"{request.request_id}_{seq_index}"
            generators.append(self._chunk_generator(rid, ids, gpt_cond_latent, speaker_embeddings, sp))
            request_ids.append(rid)
        return generators, request_ids, speaker_embeddings, [gpt_cond_latent] * len(generators)

    async def _chunk_generator(self, rid: str, ids: List[int], cond, g, sp: native.Sampling):
        """Lazy like vLLM's generator (App. B.15): the chunk is submitted at the first __anext__.  The speaker slot is
        pinned from submission until the native completion arrives (released by the poller thread), so it cannot be
        recycled under a queued or running chunk even if the awaiting coroutine is cancelled."""
        loop = asyncio.get_running_loop()
        box: asyncio.Queue = asyncio.Queue()            # completions of this chunk: partial pieces, then the final one
        natives = getattr(self, "natives", None) or [self.native]
        spks = getattr(self, "_spks", None) or [self._spk]
        work = len(ids) * max(1, getattr(sp, "num_beams", 1))     # a beam group decodes num_beams rows per step
        with self._wlock:                               # data parallelism: the GPU with the least work in flight takes it
            load = getattr(self, "_load", None)
            if load is None:
                load = self._load = [0] * len(natives)
            dev = min(range(len(natives)), key=lambda d: (load[d], d))
            load[dev] += work
        try:
            slot = await self._pin_speaker(cond, g, dev=dev)
        except BaseException:
            with self._wlock:
                self._load[dev] -= work
            raise
        with self._id_lock:
            sid = self._next_id
            self._next_id += 1
        with self._wlock:
            self._waiters[sid] = (loop, box, slot, dev, work)
        try:
            natives[dev].submit(sid, ids, slot, sp)
        except BaseException:
            with self._wlock:
                self._waiters.pop(sid, None)
                self._load[dev] -= work
            spks[dev].unpin(slot)
            raise
        n_before = 0
        done = False
        try:
            while True:
                payload, err = await box.get()
                if err is not None:
                    done = True
                    raise err
                result, toks, wav = payload
                if result.status > 0:                   # partial piece: the tokens whose audio it carries
                    n_before += len(toks)
                    yield ChunkOutput(rid, toks, wav, result, partial=True)
                    continue
                # the final result lists every token; report only the ones whose audio this piece carries
                done = True
                yield ChunkOutput(rid, toks[n_before:], wav, result)
                return
        finally:
            if not done:
                # the consumer went away (cancelled coroutine, closed stream, failed sibling chunk): abort the native chunk so
                # it gives its batch slot and KV pages back — the reference aborts the vLLM request the same way.  The
                # poller still receives the (cancelled) final result and unpins the speaker slot.
                try:
                    natives[dev].cancel(sid)
                except Exception:      # noqa: BLE001 — engine already shut down
                    pass

    async def process_tokens_to_speech(self, generator, speaker_embeddings=None, multimodal_data=None,
                                       request: TTSRequest = None) -> AsyncGenerator[TTSOutput, None]:
        assert speaker_embeddings is not None, "Speaker embeddings must be provided for speech generation with XTTSv2."
        assert multimodal_data is not None, "Multimodal data must be provided for speech generation with XTTSv2."
        async for output in generator:
            if output.finished:
                yield TTSOutput(array=output.wav, start_time=request.start_time if request else None,
                                token_length=len(output.token_ids))

    def park_poller(self, parked: bool = True):
        """Park / resume the completion pollers (a caller that drives `native.run_batch` itself must own the queue)."""
        self._paused = parked
        n = len(getattr(self, "_pollers", [None]))
        while parked and self._parked < n:    # acknowledged between two poll() calls (<= 50 ms)
            time.sleep(0.002)

    def run_batch_direct(self, jobs, **kw):
        """Drive the (first) native engine synchronously (no asyncio): the poller threads are parked for the duration."""
        was = self._paused
        self.park_poller(True)
        try:
            return self.native.run_batch(jobs, **kw)
        finally:
            if not was:
                self.park_poller(False)

    def stats(self) -> dict:
        """Native counters summed over the GPUs (the numbers the reference's TTSMetricsTracker derives,
        common/metrics/performance.py:105-151): tokens, samples, decode steps, kernel launches, device time."""
        tot: Dict[str, float] = {}
        for ne in (getattr(self, "natives", None) or [self.native]):
            st = ne.stats()
            for k, _ in st._fields_:
                tot[k] = tot.get(k, 0) + getattr(st, k)
        return tot

    def change_speed(self, array, speed_factor: float) -> np.ndarray:
        """`TTSOutput.change_speed` on the first GPU (``xtts_change_speed``): the reference's librosa phase-vocoder time
        stretch (> 1 faster) and peak normalisation.  A factor or an input the reference would reject (not finite or
        <= 0, a non-finite sample, a factor that leaves one STFT frame) raises ValueError."""
        try:
            return self.native.change_speed(np.asarray(array, np.float32), float(speed_factor))
        except native.NativeError as e:
            if e.code == native.ERR_INVALID:
                raise ValueError(str(e)) from e
            raise

    def resample(self, array, orig_sr: int, new_sr: int) -> np.ndarray:
        """`TTSOutput.resample` and speaker-reference resampling on the first GPU (``xtts_resample``):
        torchaudio.functional.resample(array, orig_sr, new_sr) with its defaults, float32 [..., N] -> float32
        [..., ceil(new' N / orig')] (the rates over their gcd), each row on its own.  A rate outside 1 .. 1048575 or a
        non-finite sample raises ValueError."""
        a = np.ascontiguousarray(array, np.float32)
        if a.ndim == 0 or 0 in a.shape[:-1]:
            raise ValueError("resample needs at least one row of samples")
        try:
            rows = [self.native.resample(r, orig_sr, new_sr) for r in a.reshape(-1, a.shape[-1])]
        except native.NativeError as e:
            if e.code == native.ERR_INVALID:
                raise ValueError(str(e)) from e
            raise
        return np.stack(rows).reshape(a.shape[:-1] + rows[0].shape)

    def encode_flac(self, pcm_i16, sample_rate: int, md5: Optional[bytes] = None) -> bytes:
        """`TTSOutput.to_bytes("flac")` on the first GPU (``xtts_encode_flac``): a lossless FLAC stream of mono int16
        samples, with `md5` (16 bytes, or None for zeros) in its STREAMINFO.  A sample rate outside 1 .. 1048575 raises
        ValueError."""
        try:
            return self.native.encode_flac(pcm_i16, int(sample_rate), md5)
        except native.NativeError as e:
            if e.code == native.ERR_INVALID:
                raise ValueError(str(e)) from e
            raise

    def decode_flac(self, data) -> Tuple[np.ndarray, int, int]:
        """FLAC input (`TTSOutput.from_file`, `load_audio`) on the first GPU (``xtts_decode_flac``): a whole FLAC stream
        -> (int32 [channels, samples], sample rate, bits per sample), lossless, its MD5 checked when STREAMINFO has one.
        A stream that breaks the format or fails a check raises ValueError."""
        try:
            return self.native.decode_flac(data)
        except native.NativeError as e:
            if e.code == native.ERR_INVALID:
                raise ValueError(str(e)) from e
            raise

    async def shutdown(self):
        _output.unregister_gpu_provider(self)
        self._stop = True
        for t in getattr(self, "_pollers", []):
            t.join(timeout=5)
        for ne in (getattr(self, "natives", None) or [self.native]):
            ne.close()

    # ---- completion dispatch ----------------------------------------------------------------
    def _poll_loop(self, dev: int = 0):
        natives = getattr(self, "natives", None) or [self.native]
        spks = getattr(self, "_spks", None) or [self._spk]
        ne = natives[dev]
        parked = False
        while not self._stop:
            if self._paused:
                if not parked:
                    parked = True
                    self._parked += 1
                time.sleep(0.002)
                continue
            if parked:
                parked = False
                self._parked -= 1
            try:
                r = ne.poll(50)
            except Exception:
                if self._stop:
                    return
                time.sleep(0.05)
                continue
            if r is None:
                continue
            final = r.status <= 0
            with self._wlock:
                w = self._waiters.pop(r.seq_id, None) if final else self._waiters.get(r.seq_id)
                if final and w is not None and len(w) > 4 and getattr(self, "_load", None) is not None:
                    self._load[w[3]] -= w[4]
            try:
                if r.status < 0:
                    msg = ne.lib.xtts_last_error().decode()
                    try:
                        ne.lib.xtts_fetch(ne.h, r.seq_id, None, None, None)   # release its native buffers
                    except Exception:      # noqa: BLE001
                        pass
                    raise native.NativeError(f"chunk {r.seq_id} " + ("was cancelled" if r.status == native.ERR_CANCELLED
                                                                    else f"failed ({r.status}): {msg}"))
                toks, wav, _ = ne.fetch(r, want_wav=True)
                payload, err = (r, toks, wav), None
            except Exception as e:      # noqa: BLE001 — forwarded to the awaiting coroutine
                payload, err = None, e
            if w is None:
                continue
            loop, box, slot = w[0], w[1], w[2]
            if final:
                spks[dev].unpin(slot)               # the native engine is done with this chunk's speaker slot
            loop.call_soon_threadsafe(box.put_nowait, (payload, err))


class _SpeakerArray(np.ndarray):
    """numpy array that remembers which native speaker slot it was uploaded to and under which cache key (the pair is
    re-validated before every use: a recycled slot is detected and the array uploaded again)."""

    def __new__(cls, arr, slot, key=None, dev=0):
        obj = np.asarray(arr).view(cls)
        obj.slot = slot
        obj.key = key
        obj.dev = dev               # index into the engine's `devices` the slot number refers to
        return obj

    def __array_finalize__(self, obj):
        self.slot = getattr(obj, "slot", None)
        self.key = getattr(obj, "key", None)
        self.dev = getattr(obj, "dev", 0)


def _resample(a: np.ndarray, sr: int, new_sr: int) -> np.ndarray:
    """torchaudio.functional.resample (the reference's resampler, XTTSv2.py:323,360): on the GPU of a live engine
    (`output.gpu_resample`), else torchaudio on the host when importable, scipy polyphase otherwise.  Every resample of a
    speaker reference goes through here."""
    if sr == new_sr:
        return a
    y = _output.gpu_resample(a, sr, new_sr)
    if y is not None:
        return y
    try:
        import torch
        import torchaudio
        return torchaudio.functional.resample(torch.from_numpy(np.ascontiguousarray(a)), sr, new_sr).numpy()
    except Exception:
        from math import gcd
        from scipy.signal import resample_poly
        g = gcd(sr, new_sr)
        return resample_poly(a, new_sr // g, sr // g).astype(np.float32)


register_model("xtts", XTTSv2Engine)
