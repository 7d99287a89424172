"""TTSOutput — the boundary type of the hot path (array/sample_rate/token_length/start_time).

Mirrors `/root/reference/src/auralis/common/definitions/output.py:17-38,95-111` for the fields and
``combine_outputs``.  ``change_speed`` (the reference's librosa phase vocoder + peak normalisation) and 16-bit FLAC
(``to_bytes("flac")``, a lossless LPC + partitioned-Rice encoder) run on the GPU of a live `XTTSv2Engine`
(``register_gpu_provider``), and on librosa / torchaudio when no engine is alive.  The other audio utilities (mp3/opus/aac
encoders, playback) are CPU post-processing outside the hot path (SURVEY.md §2.1 #3): wav/pcm paths are provided with the
standard library, the rest raise with a clear message when their optional dependency is absent.
"""
from __future__ import annotations

import hashlib
import io
import threading
import wave
import weakref
from dataclasses import dataclass
from pathlib import Path
from typing import List, Optional, Union

import numpy as np


def _riff_wav(x: np.ndarray, sample_rate: int, bits: int) -> bytes:
    """Mono RIFF/WAVE: 32 bits -> IEEE float (format tag 3), 16 / 8 -> integer PCM (tag 1)."""
    import struct
    x = np.clip(x, -1.0, 1.0)
    if bits == 32:
        tag, payload = 3, x.astype("<f4").tobytes()
    elif bits == 16:
        tag, payload = 1, (x * 32767).astype("<i2").tobytes()
    elif bits == 8:
        tag, payload = 1, ((x * 127) + 128).astype(np.uint8).tobytes()
    else:
        raise ValueError(f"unsupported bit depth {bits}")
    block = bits // 8
    fmt = struct.pack("<HHIIHH", tag, 1, sample_rate, sample_rate * block, block, bits)
    body = b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt
    if tag == 3:
        body += b"fact" + struct.pack("<II", 4, x.shape[0])
    body += b"data" + struct.pack("<I", len(payload)) + payload
    return b"RIFF" + struct.pack("<I", len(body)) + body


def _parse_riff_wav(blob: bytes):
    """-> (float32 [frames, channels], sample_rate) for integer-PCM (8/16/24/32 bit) and IEEE-float (32/64 bit) WAV, else None."""
    import struct
    if len(blob) < 12 or blob[:4] != b"RIFF" or blob[8:12] != b"WAVE":
        return None
    pos, fmt, data = 12, None, None
    while pos + 8 <= len(blob):
        cid, size = blob[pos:pos + 4], struct.unpack("<I", blob[pos + 4:pos + 8])[0]
        chunk = blob[pos + 8:pos + 8 + size]
        if cid == b"fmt ":
            fmt = struct.unpack("<HHIIHH", chunk[:16])
            if fmt[0] == 0xFFFE and len(chunk) >= 26:             # WAVE_FORMAT_EXTENSIBLE: the real tag is in the sub-format GUID
                fmt = (struct.unpack("<H", chunk[24:26])[0],) + fmt[1:]
        elif cid == b"data":
            data = chunk
        pos += 8 + size + (size & 1)
    if fmt is None or data is None:
        return None
    tag, nch, sr, _, _, bits = fmt
    if tag == 1 and bits == 16:
        a = np.frombuffer(data, dtype="<i2").astype(np.float32) / 32768.0
    elif tag == 1 and bits == 8:
        a = (np.frombuffer(data, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
    elif tag == 1 and bits == 32:
        a = np.frombuffer(data, dtype="<i4").astype(np.float32) / 2147483648.0
    elif tag == 1 and bits == 24:
        b = np.frombuffer(data[: len(data) // 3 * 3], dtype=np.uint8).reshape(-1, 3).astype(np.int32)
        v = b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)
        a = (np.where(v >= 1 << 23, v - (1 << 24), v)).astype(np.float32) / 8388608.0
    elif tag == 3 and bits == 32:
        a = np.frombuffer(data, dtype="<f4").astype(np.float32)
    elif tag == 3 and bits == 64:
        a = np.frombuffer(data, dtype="<f8").astype(np.float32)
    else:
        return None
    n = a.shape[0] // nch * nch
    return a[:n].reshape(-1, nch), int(sr)


_providers: List["weakref.ref"] = []
_providers_lock = threading.Lock()


def register_gpu_provider(engine) -> None:
    """Route `TTSOutput.change_speed` to `engine.change_speed(array, speed_factor) -> np.ndarray`, and 16-bit
    `TTSOutput.to_bytes("flac")` to `engine.encode_flac(pcm_i16, sample_rate, md5) -> bytes` when the engine has that
    method, while the engine is alive (`XTTSv2Engine` registers itself when it is built).  Held through a weak reference, so the registry never keeps
    an engine alive; the most recently registered live engine serves."""
    with _providers_lock:
        _providers[:] = [r for r in _providers if r() is not None and r() is not engine]
        _providers.append(weakref.ref(engine))


def unregister_gpu_provider(engine) -> None:
    """Take `engine` out of the registry (its shutdown)."""
    with _providers_lock:
        _providers[:] = [r for r in _providers if r() is not None and r() is not engine]


def gpu_provider():
    """The engine `TTSOutput.change_speed` and `TTSOutput.to_bytes("flac")` run on, or None."""
    with _providers_lock:
        for r in reversed(_providers):
            e = r()
            if e is not None:
                return e
    return None


@dataclass
class TTSOutput:
    array: Union[np.ndarray, bytes]
    sample_rate: int = 24000
    bit_depth: int = 32
    bit_rate: int = 192
    compression: int = 10
    channel: int = 1
    start_time: Optional[float] = None
    end_time: Optional[float] = None
    token_length: Optional[int] = None

    def __post_init__(self):
        if isinstance(self.array, bytes):          # output.py:30-38
            self.array = np.frombuffer(self.array, dtype=np.int16)
            self.array = self.array.astype(np.float32) / 32768.0
            fade_length = 100
            fade_in = np.linspace(0, 1, fade_length)
            self.array[:fade_length] *= fade_in

    @staticmethod
    def combine_outputs(outputs: List["TTSOutput"]) -> "TTSOutput":
        """output.py:95-111."""
        combined_audio = np.concatenate([out.array for out in outputs])
        return TTSOutput(array=combined_audio, sample_rate=outputs[0].sample_rate)

    class Accumulator:
        """`combine_outputs` done incrementally: each chunk is copied into one growing buffer when it ARRIVES, so that
        the last chunk of a request costs one chunk-sized copy instead of a concatenation of the whole request (the
        reference concatenates at the end, `core/tts.py:228-230,305-308`; with 13 MB per 1 000 characters that pass sat
        on the tail of every batch).  `result()` equals `TTSOutput.combine_outputs(chunks)`."""

        def __init__(self, reserve_chunks: int = 8):
            self.buf: Optional[np.ndarray] = None
            self.n = 0
            self.sample_rate: Optional[int] = None
            self.count = 0
            self._reserve = max(1, reserve_chunks)

        def add(self, out: "TTSOutput") -> None:
            a = np.asarray(out.array)
            if self.buf is None:
                self.sample_rate = out.sample_rate
                self.buf = np.empty(max(1, a.shape[0]) * self._reserve, dtype=a.dtype)      # untouched pages cost nothing
            need = self.n + a.shape[0]
            if a.dtype != self.buf.dtype or need > self.buf.shape[0]:
                dt = np.result_type(self.buf.dtype, a.dtype)
                grown = np.empty(max(need, 2 * self.buf.shape[0]), dtype=dt)
                grown[: self.n] = self.buf[: self.n]
                self.buf = grown
            self.buf[self.n: need] = a
            self.n = need
            self.count += 1

        def result(self) -> "TTSOutput":
            if self.buf is None:
                raise ValueError("need at least one array to concatenate")          # what np.concatenate([]) raises
            return TTSOutput(array=self.buf[: self.n], sample_rate=self.sample_rate)

    def to_tensor(self):
        import torch
        if isinstance(self.array, np.ndarray):
            return torch.from_numpy(self.array)
        return self.array

    def to_bytes(self, format: str = "wav", sample_width: int = 2) -> bytes:
        """output.py:119-187; wav and pcm are native here, mp3/opus/aac need torchaudio+ffmpeg.

        ``flac`` at ``sample_width=2`` (the only width at which the reference writes 16-bit FLAC; it asks for PCM_F at
        any other) runs on the GPU while an `XTTSv2Engine` is alive: the samples are quantised exactly as ``pcm`` /
        ``wav`` quantise them, so the stream decodes to the very samples ``to_bytes("pcm", 2)`` returns, and their MD5
        goes into STREAMINFO.  There is one configuration (fixed 4096-sample blocks, FIXED and LPC predictors up to
        order 12, partitioned Rice residuals): ``compression`` selects nothing on that path.  With no engine alive, with
        one that cannot encode FLAC, or at another width, flac goes through torchaudio like the other codecs."""
        wav = np.clip(np.asarray(self.array, dtype=np.float32), -1.0, 1.0)
        if format == "pcm":
            if sample_width == 2:
                return (wav * 32767).astype(np.int16).tobytes()
            if sample_width == 4:       # float32 arithmetic, as the reference's torch expression (output.py:177-178)
                return (wav * np.float32(2147483647)).astype(np.int32).tobytes()
            return (wav * 127).astype(np.int8).tobytes()
        if format == "wav":
            # output.py:141-149: encoding PCM_S at sample_width 2, PCM_F (IEEE float) otherwise, bits = 8 * sample_width
            if sample_width == 2:
                buf = io.BytesIO()
                with wave.open(buf, "wb") as w:
                    w.setnchannels(1)
                    w.setsampwidth(2)
                    w.setframerate(self.sample_rate)
                    w.writeframes((wav * 32767).astype(np.int16).tobytes())
                return buf.getvalue()
            return _riff_wav(wav, self.sample_rate, 8 * sample_width)
        if format == "flac" and sample_width == 2:
            gpu = gpu_provider()
            if gpu is not None and hasattr(gpu, "encode_flac"):
                pcm = (wav * 32767).astype(np.int16)
                return gpu.encode_flac(pcm, self.sample_rate, hashlib.md5(pcm.astype("<i2").tobytes()).digest())
        if format in ("flac", "mp3", "opus", "aac"):
            try:
                import torch
                import torchaudio
                buffer = io.BytesIO()
                torchaudio.save(buffer, torch.from_numpy(wav)[None], self.sample_rate,
                                format={"aac": "adts"}.get(format, format))
                return buffer.getvalue()
            except Exception as e:   # codec backends are optional
                raise RuntimeError(f"format {format!r} needs a torchaudio codec backend: {e}") from e
        raise ValueError(f"Unsupported format: {format}. Supported formats are: mp3, opus, aac, flac, wav, pcm")

    def save(self, filename: Union[str, Path], sample_rate: Optional[int] = None, format: Optional[str] = None) -> None:
        """output.py:189-222: resample if asked, then write with `bits_per_sample = bit_depth` — 32 (the default) is an
        IEEE-float WAV, which is what torchaudio writes for the reference; other containers go through `to_bytes`."""
        out = self if not sample_rate or sample_rate == self.sample_rate else self.resample(sample_rate)
        fmt = format or (Path(filename).suffix.lstrip(".") or "wav")
        if fmt == "wav":
            data = _riff_wav(np.asarray(out.array, np.float32), out.sample_rate, self.bit_depth)
        else:
            data = out.to_bytes(fmt)
        with open(filename, "wb") as f:
            f.write(data)

    def resample(self, new_sample_rate: int) -> "TTSOutput":
        """output.py:224-246: torchaudio's windowed-sinc resampler, like the reference; scipy's polyphase filter only when
        torchaudio cannot be imported."""
        try:
            import torch
            import torchaudio
            y = torchaudio.functional.resample(torch.from_numpy(np.ascontiguousarray(self.array, np.float32))[None],
                                               orig_freq=self.sample_rate, new_freq=new_sample_rate).squeeze().numpy()
        except ImportError:
            if new_sample_rate == self.sample_rate:
                return self
            from math import gcd
            from scipy.signal import resample_poly
            g = gcd(int(new_sample_rate), int(self.sample_rate))
            y = resample_poly(np.asarray(self.array, np.float32), new_sample_rate // g, self.sample_rate // g).astype(np.float32)
        return TTSOutput(array=y, sample_rate=new_sample_rate)

    def change_speed(self, speed_factor: float) -> "TTSOutput":
        """output.py:40-92: time-stretch the audio by `speed_factor` (> 1 faster, < 1 slower) with librosa's phase
        vocoder (STFT n_fft 2048, hop 512), then peak-normalise it to max |x| = 1.  `<= 0` raises ValueError, `== 1`
        returns this object.  While an `XTTSv2Engine` is alive the stretch runs on its first GPU (`xtts_change_speed`,
        the same arithmetic as librosa 0.10 under numpy's promotion rules) and a factor the reference would reject
        raises ValueError; without one it needs librosa installed and raises RuntimeError otherwise.  Returns a new
        TTSOutput with only `array` and `sample_rate` set, like the reference."""
        if speed_factor <= 0:
            raise ValueError("Speed factor must be positive")
        if speed_factor == 1.0:
            return self
        gpu = gpu_provider()
        if gpu is not None:
            return TTSOutput(array=gpu.change_speed(self.array, speed_factor), sample_rate=self.sample_rate)
        try:
            import librosa
        except ImportError as e:
            raise RuntimeError("change_speed needs librosa (CPU post-processing, outside the hot path)") from e
        wav = np.asarray(self.array, np.float32)
        D = librosa.stft(wav, n_fft=2048, hop_length=512)
        y = librosa.istft(librosa.phase_vocoder(D, rate=speed_factor, hop_length=512), hop_length=512)
        return TTSOutput(array=librosa.util.normalize(y, norm=np.inf), sample_rate=self.sample_rate)

    def get_info(self):
        """output.py:248-256: (number of samples, sample rate, duration in seconds)."""
        n = len(self.array)
        return n, self.sample_rate, n / self.sample_rate

    @classmethod
    def from_tensor(cls, tensor, sample_rate: int = 24000) -> "TTSOutput":
        """output.py:258-272."""
        return cls(array=tensor.squeeze().cpu().numpy(), sample_rate=sample_rate)

    @classmethod
    def from_file(cls, filename: Union[str, Path]) -> "TTSOutput":
        """output.py:274-285.  RIFF/WAV through the standard library (the reference's torchaudio.load needs a codec
        backend that this image does not ship); other containers go through torchaudio when it can load them."""
        with open(str(filename), "rb") as f:
            blob = f.read()
        parsed = _parse_riff_wav(blob)
        if parsed is None:                                   # not RIFF/WAVE (or an exotic encoding): torchaudio's loaders
            import torchaudio
            wav, sr = torchaudio.load(str(filename))
            return cls.from_tensor(wav, sr)
        a, sr = parsed
        return cls(array=(a[:, 0] if a.shape[1] == 1 else a.T).copy(), sample_rate=sr)

    def play(self) -> None:
        """output.py:287-303 (needs the optional `sounddevice` package, like the reference)."""
        try:
            import sounddevice as sd
        except ImportError as e:
            raise RuntimeError("play() needs the optional sounddevice package") from e
        sd.play(np.clip(np.asarray(self.array, np.float32), -1.0, 1.0), self.sample_rate, blocksize=2048)
        sd.wait()

    def display(self):
        """output.py:305-319: IPython audio widget, None outside a notebook."""
        try:
            from IPython.display import Audio, display
            widget = Audio(self.to_bytes(format="wav"), rate=self.sample_rate, autoplay=False)
            display(widget)
            return widget
        except Exception as e:      # noqa: BLE001 — same behaviour as the reference: report and fall back
            print(f"Could not display audio widget: {e}")
            print("Try using .play() method instead")
            return None

    def preview(self) -> None:
        """output.py:321-330."""
        try:
            if self.display() is None:
                self.play()
        except Exception as e:      # noqa: BLE001
            print(f"Error playing audio: {e}")

    @property
    def duration_s(self) -> float:
        return len(self.array) / float(self.sample_rate)
