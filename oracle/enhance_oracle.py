"""CPU oracle of the speaker-reference enhancer (`TTSRequest.enhance_speech`): VAD trim, spectral gating, clarity
shaping and BS.1770 loudness normalisation, restated in numpy / scipy / torchaudio.

The two third-party libraries the reference's enhancer calls are restated here as small module-like namespaces,
``librosa`` (``stft``, ``istft``, ``magphase``, ``util.frame``) and ``pyloudnorm`` (``Meter``), with the semantics of
librosa 0.10 and pyloudnorm 0.1: constant-padded centred STFTs with a periodic Hann window, overlap-add divided by the
squared-window sum where it exceeds float32 ``tiny``, and K-weighted 400 ms / 75 % gated loudness.  The same namespaces
are injected into the reference's own module by ``oracle/ref_enhance.py``, so the glue below is pinned against it; the
restatements themselves are checked against published values in ``tests/test_enhance_host.py``.

`process(audio, cfg)` is the stage; `roundtrip16` is the 16-bit write/read that follows it.  Nothing here reads the
reference tree, so GPU tests may use it.
"""
from __future__ import annotations

import types
from dataclasses import dataclass
from typing import Optional

import numpy as np


class ParameterError(ValueError):
    """librosa.util.exceptions.ParameterError."""


# ---------------------------------------------------------------------------------------------------- librosa
def _hann(n: int) -> np.ndarray:
    """scipy.signal.get_window('hann', n, fftbins=True): periodic, float64."""
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(n) / n)


def _frame(x: np.ndarray, frame_length: int, hop_length: int) -> np.ndarray:
    """librosa.util.frame along the last axis -> [frame_length, n_frames]."""
    x = np.asarray(x)
    if hop_length < 1:
        raise ParameterError(f"Invalid hop_length: {hop_length}")
    if x.shape[-1] < frame_length:
        raise ParameterError(f"Input is too short (n={x.shape[-1]}) for frame_length={frame_length}")
    w = np.lib.stride_tricks.sliding_window_view(x, frame_length)[::hop_length]
    return w.T


def _stft(y: np.ndarray, n_fft: int = 2048, hop_length: Optional[int] = None, center: bool = True,
          pad_mode: str = "constant") -> np.ndarray:
    """librosa.stft with its defaults: periodic Hann, hop n_fft/4, centred, zero padding; complex64 for float32 input."""
    y = np.asarray(y)
    if not np.issubdtype(y.dtype, np.floating):
        raise ParameterError("Audio data must be floating-point")
    if not np.isfinite(y).all():
        raise ParameterError("Audio buffer is not finite everywhere")
    hop = n_fft // 4 if hop_length is None else hop_length
    if center:
        y = np.pad(y, (n_fft // 2, n_fft // 2), mode=pad_mode)
    frames = _frame(y, n_fft, hop)
    cdt = np.complex64 if y.dtype == np.float32 else np.complex128
    return np.fft.rfft(_hann(n_fft)[:, None] * frames, axis=0).astype(cdt)


def _istft(D: np.ndarray, hop_length: Optional[int] = None, center: bool = True) -> np.ndarray:
    """librosa.istft with its defaults (length=None): irfft x window, overlap-add in the output dtype, divide by the
    squared-window sum where it exceeds float32 tiny, drop n_fft/2 samples at each end."""
    n_fft = 2 * (D.shape[0] - 1)
    hop = n_fft // 4 if hop_length is None else hop_length
    T = D.shape[1]
    rdt = np.float32 if D.dtype == np.complex64 else np.float64
    win = _hann(n_fft)
    frames = win[:, None] * np.fft.irfft(D, n=n_fft, axis=0)
    n = n_fft + hop * (T - 1)
    y = np.zeros(n, rdt)
    wss = np.zeros(n, rdt)
    w2 = (win ** 2).astype(rdt)
    for t in range(T):
        y[t * hop: t * hop + n_fft] += frames[:, t].astype(rdt)
        wss[t * hop: t * hop + n_fft] += w2
    start = n_fft // 2 if center else 0
    y, wss = y[start: n - start], wss[start: n - start]
    nz = wss > np.finfo(np.float32).tiny
    y[nz] /= wss[nz]
    return y


def _magphase(D: np.ndarray):
    """librosa.magphase(power=1): phase is 1 where the magnitude is 0."""
    mag = np.abs(D)
    zeros = mag == 0
    nzmag = mag + zeros
    phase = np.empty_like(D)
    phase.real = D.real / nzmag + zeros
    phase.imag = D.imag / nzmag
    return mag, phase


librosa = types.SimpleNamespace(stft=_stft, istft=_istft, magphase=_magphase,
                                util=types.SimpleNamespace(frame=lambda x, frame_length, hop_length, axis=-1:
                                                           _frame(x, frame_length, hop_length)),
                                ParameterError=ParameterError)


# ---------------------------------------------------------------------------------------------------- pyloudnorm
def kweighting(rate: float):
    """pyloudnorm's K-weighting: RBJ high shelf (G 4 dB, Q 1/sqrt 2, 1500 Hz) then RBJ high pass (Q 0.5, 38 Hz),
    coefficients normalised by a0, recomputed for `rate`.  -> [(b, a), (b, a)]."""
    def shelf(G, Q, fc):
        A = 10 ** (G / 40.0)
        w0 = 2.0 * np.pi * (fc / rate)
        alpha = np.sin(w0) / (2.0 * Q)
        c, sA = np.cos(w0), np.sqrt(A)
        b = [A * ((A + 1) + (A - 1) * c + 2 * sA * alpha), -2 * A * ((A - 1) + (A + 1) * c),
             A * ((A + 1) + (A - 1) * c - 2 * sA * alpha)]
        a = [(A + 1) - (A - 1) * c + 2 * sA * alpha, 2 * ((A - 1) - (A + 1) * c), (A + 1) - (A - 1) * c - 2 * sA * alpha]
        return np.array(b) / a[0], np.array(a) / a[0]

    def highpass(Q, fc):
        w0 = 2.0 * np.pi * (fc / rate)
        alpha = np.sin(w0) / (2.0 * Q)
        c = np.cos(w0)
        b = [(1 + c) / 2, -(1 + c), (1 + c) / 2]
        a = [1 + alpha, -2 * c, 1 - alpha]
        return np.array(b) / a[0], np.array(a) / a[0]

    return [shelf(4.0, 1 / np.sqrt(2), 1500.0), highpass(0.5, 38.0)]


def block_bounds(n: int, rate: float, block_size: float = 0.400, overlap: float = 0.75):
    """pyloudnorm's gating blocks: count from np.round, sample bounds by int() truncation."""
    step = 1.0 - overlap
    T = n / rate
    nb = int(np.round(((T - block_size) / (block_size * step)))) + 1
    return [(int(block_size * (j * step) * rate), int(block_size * (j * step + 1) * rate)) for j in range(nb)]


class Meter:
    """pyloudnorm.Meter(rate) for mono input: integrated loudness, ITU-R BS.1770-4."""

    def __init__(self, rate, filter_class="K-weighting", block_size=0.400):
        self.rate = rate
        self.block_size = block_size
        self.last_blocks = None           # per-block loudness of the last call (gating margins in tests)

    def integrated_loudness(self, data):
        from scipy.signal import lfilter
        data = np.asarray(data)
        if not np.issubdtype(data.dtype, np.floating):
            raise ValueError("Data must be floating point.")
        if data.shape[0] < self.block_size * self.rate:
            raise ValueError("Audio must have length greater than the block size.")
        x = data.copy()
        for b, a in kweighting(self.rate):
            x[:] = lfilter(b, a, x)               # written back in the input's dtype, as pyloudnorm does
        scale = 1.0 / (self.block_size * self.rate)
        z = np.array([scale * np.sum(np.square(x[lo:hi])) for lo, hi in block_bounds(x.shape[0], self.rate,
                                                                                        self.block_size)])
        with np.errstate(divide="ignore", invalid="ignore"):
            lj = -0.691 + 10.0 * np.log10(z)
            self.last_blocks = lj
            g_abs = lj >= -70.0
            rel = -0.691 + 10.0 * np.log10(np.mean(z[g_abs]) if g_abs.any() else np.nan) - 10.0
            g = (lj > rel) & g_abs
            zg = np.nan_to_num(np.mean(z[g]) if g.any() else np.nan)
            self.last_gates = (-70.0, rel)
            return -0.691 + 10.0 * np.log10(zg)


pyloudnorm = types.SimpleNamespace(Meter=Meter)


# ---------------------------------------------------------------------------------------------------- the stage
@dataclass
class EnhanceConfig:
    """Field names and defaults of the reference's AudioPreprocessingConfig."""
    sample_rate: int = 22050
    normalize: bool = True
    trim_silence: bool = True
    remove_noise: bool = True
    enhance_speech: bool = True
    vad_threshold: float = 0.02
    vad_frame_length: int = 4096
    noise_reduce_margin: float = 1.0
    noise_reduce_frames: int = 25
    enhance_amount: float = 1.0
    target_lufs: float = -18.0


def _interp_to(v: np.ndarray, n: int) -> np.ndarray:
    return np.interp(np.linspace(0, 1, n), np.linspace(0, 1, len(v)), v)


def vad_signal(audio: np.ndarray, cfg) -> np.ndarray:
    """(energy + mel log-sum) / 2 per frame, both max-normalised and brought to the longer of the two lengths."""
    import torch
    import torchaudio
    fl = cfg.vad_frame_length
    e = np.sum(librosa.util.frame(audio, frame_length=fl, hop_length=fl // 2) ** 2, axis=0)
    e = e / np.max(e)
    mel = torchaudio.transforms.MelSpectrogram(sample_rate=cfg.sample_rate, n_fft=2048, hop_length=512, n_mels=80)(
        torch.FloatTensor(audio).unsqueeze(0))
    s = torch.sum(torch.log(torch.clamp(mel, min=1e-5)), dim=1).numpy().squeeze()
    s = s / np.max(s)                 # the sum is normally negative; divided by its max as the reference does
    if len(e) > len(s):
        s = _interp_to(s, len(e))
    else:
        e = _interp_to(e, len(s))
    return (e + s) / 2


def trim_silence(audio, cfg):
    keep = np.absolute(vad_signal(audio, cfg)) > cfg.vad_threshold
    return audio * _interp_to(keep.astype(float), len(audio))


def noise_floor(mag: np.ndarray, k: int) -> np.ndarray:
    return np.mean(np.sort(mag, axis=1)[:, :k], axis=1)


def remove_noise(audio, cfg):
    D = librosa.stft(audio)
    mag, _ = librosa.magphase(D)
    noise = noise_floor(mag, cfg.noise_reduce_frames)[:, None]
    gate = np.clip(mag - noise * cfg.noise_reduce_margin, 0, None)
    gate = gate / (gate + noise)              # 0/0 = NaN where a bin's floor is 0 and the frame is silent: kept
    return librosa.istft(gate * D)


def clarity_gain(cfg) -> np.ndarray:
    """1 + amount * exp(-|f - 2000| / 1000) per STFT bin, with f from np.fft.fftfreq(1025, 1/sr) as the reference has
    it: spacing sr/1025 and negative frequencies above bin 512, not the bins' real frequencies.  Kept as is."""
    f = np.fft.fftfreq(1025, 1 / cfg.sample_rate)
    return 1 + np.exp(-np.abs(f - 2000) / 1000) * cfg.enhance_amount


def enhance_clarity(audio, cfg):
    D = librosa.stft(np.nan_to_num(audio, nan=0.0, posinf=0.0, neginf=0.0))
    mag, phase = librosa.magphase(D)
    return librosa.istft(mag * clarity_gain(cfg)[:, None] * phase)


def normalize_loudness(audio, cfg, meter: Optional[Meter] = None):
    meter = meter or pyloudnorm.Meter(cfg.sample_rate)
    lufs = meter.integrated_loudness(audio)
    return np.tanh(audio * 10 ** ((cfg.target_lufs - lufs) / 20))


def process(audio: np.ndarray, cfg, taps: Optional[dict] = None) -> np.ndarray:
    """The four stages in order, each behind its flag.  `taps`, when given, receives the intermediates tests check
    margins on: the VAD signal, the per-stage outputs and the loudness blocks and gates."""
    taps = {} if taps is None else taps
    if cfg.trim_silence:
        taps["vad"] = vad_signal(audio, cfg)
        audio = trim_silence(audio, cfg)
        taps["after_vad"] = audio
    if cfg.remove_noise:
        audio = remove_noise(audio, cfg)
        taps["after_gate"] = audio
    if cfg.enhance_speech:
        audio = enhance_clarity(audio, cfg)
        taps["after_clarity"] = audio
    if cfg.normalize:
        m = Meter(cfg.sample_rate)
        taps["lufs"] = m.integrated_loudness(audio)
        audio = np.tanh(audio * 10 ** ((cfg.target_lufs - taps["lufs"]) / 20))
        taps["blocks"], taps["gates"] = m.last_blocks, m.last_gates
    return audio


def synthetic_input(seconds: float, sr: int, seed: int, silence=None, noise: float = 0.01) -> np.ndarray:
    """Seeded speech-like test signal: a gliding harmonic voice under a syllable-rate envelope, plus white noise;
    `silence=(t0, t1)` zeroes that span exactly (the gating stage's NaN path)."""
    rng = np.random.default_rng(seed)
    n = int(round(seconds * sr))
    t = np.arange(n) / sr
    f0 = rng.uniform(110, 220) * (1 + 0.05 * np.sin(2 * np.pi * rng.uniform(0.3, 0.8) * t))
    ph = 2 * np.pi * np.cumsum(f0) / sr
    v = sum(rng.uniform(0.2, 1.0) / h * np.sin(h * ph + rng.uniform(0, 2 * np.pi)) for h in range(1, 12))
    env = np.clip(np.sin(2 * np.pi * rng.uniform(2.5, 4.5) * t + rng.uniform(0, 2 * np.pi)), 0, None) ** 0.5
    x = rng.uniform(0.15, 0.4) * env * v / 2 + noise * rng.standard_normal(n)
    if silence is not None:
        x[int(silence[0] * sr): int(silence[1] * sr)] = 0.0
    return x.astype(np.float32)


def roundtrip16(x: np.ndarray) -> np.ndarray:
    """A 16-bit PCM write and read back: rint(x * 32767) clipped to int16, then / 32768."""
    return (np.clip(np.rint(np.asarray(x, np.float64) * 32767.0), -32768, 32767) / 32768.0).astype(np.float32)


def enhance(audio: np.ndarray, cfg) -> np.ndarray:
    """What `xtts_enhance` returns: process() then the 16-bit round trip.  Raises where the reference's enhancer
    raises (too short for a VAD frame or a loudness block) and on a non-finite result."""
    taps = {}
    out = process(np.asarray(audio, np.float32), cfg, taps)
    if not np.isfinite(out).all() or not np.isfinite(taps.get("lufs", 0.0)):
        raise ValueError("enhanced audio is not finite")
    return roundtrip16(out)
