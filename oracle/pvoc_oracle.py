"""CPU oracle of `TTSOutput.change_speed`: librosa.stft (n_fft 2048, hop 512) -> librosa.phase_vocoder ->
librosa.istft -> librosa.util.normalize(norm=inf), with the two librosa functions the enhancer oracle does not already
restate added here, with the semantics of librosa 0.10 under NumPy's NEP 50 promotion rules:

* ``phase_vocoder``: output frame t reads input frames int(t * rate) and int(t * rate) + 1 of the spectrum padded with
  two zero columns.  ``alpha``, the interpolated magnitude, the wrapped phase advance and the sum added to ``phase_acc``
  are float64; ``phase_acc`` itself stays float32 (each ``+=`` rounds f64(phase_acc) + (phi_advance + dphase) to float32);
  the output frame is (cos, sin)(phase_acc) in float32 times the float64 magnitude, stored as complex64.
* ``normalize_inf``: raises on a non-finite input, divides by max|y| (a float64 true division stored back as float32),
  and leaves the signal as it is where that maximum is below float32 ``tiny``.

``stft`` / ``istft`` are the restatements in ``oracle/enhance_oracle.py``.  ``oracle/ref_change_speed.py`` injects the
``librosa`` namespace below into the reference's own ``TTSOutput.change_speed``, which pins the glue; librosa itself is
not installed, so the restatement is checked against the properties librosa documents (tests/test_change_speed_host.py).
Nothing here reads the reference tree, so GPU tests may use it.
"""
from __future__ import annotations

import types
from typing import Callable, Optional

import numpy as np

from .enhance_oracle import ParameterError, _hann, _istft, _stft

N_FFT, HOP = 2048, 512


def fft_frequencies(sr: float, n_fft: int) -> np.ndarray:
    """librosa.fft_frequencies: np.fft.rfftfreq(n_fft, 1 / sr)."""
    return np.fft.rfftfreq(n=n_fft, d=1.0 / sr)


def angle_f64(z: np.ndarray) -> np.ndarray:
    """An equally accurate stand-in for np.angle of complex64: arctan2 in float64, rounded to float32."""
    return np.arctan2(z.imag.astype(np.float64), z.real.astype(np.float64)).astype(np.float32)


def phasor(angles: np.ndarray, mag=None) -> np.ndarray:
    """librosa.util.phasor: cos + i sin in the angles' precision, then ``z *= mag``."""
    z = np.empty(angles.shape, np.complex64 if angles.dtype == np.float32 else np.complex128)
    z.real = np.cos(angles)
    z.imag = np.sin(angles)
    if mag is not None:
        z *= mag
    return z


def phase_vocoder(D: np.ndarray, *, rate: float, hop_length: Optional[int] = None, n_fft: Optional[int] = None,
                  angle: Callable = np.angle, dtypes: Optional[dict] = None) -> np.ndarray:
    """librosa.phase_vocoder.  `angle` replaces np.angle (the tolerance derivation of the GPU tests); `dtypes`, when
    given, receives the dtypes of the first step's intermediates."""
    if n_fft is None:
        n_fft = 2 * (D.shape[-2] - 1)
    if hop_length is None:
        hop_length = int(n_fft // 4)
    time_steps = np.arange(0, D.shape[-1], rate, dtype=np.float64)
    shape = list(D.shape)
    shape[-1] = len(time_steps)
    d_stretch = np.zeros_like(D, shape=shape)
    phi_advance = hop_length * fft_frequencies(sr=2 * np.pi, n_fft=n_fft)
    phase_acc = angle(D[..., 0])
    pad = [(0, 0)] * D.ndim
    pad[-1] = (0, 2)
    D = np.pad(D, pad, mode="constant")
    for t, step in enumerate(time_steps):
        columns = D[..., int(step): int(step + 2)]
        alpha = np.mod(step, 1.0)
        mag = (1.0 - alpha) * np.abs(columns[..., 0]) + alpha * np.abs(columns[..., 1])
        d_stretch[..., t] = phasor(phase_acc, mag=mag)
        dphase = angle(columns[..., 1]) - angle(columns[..., 0]) - phi_advance
        dphase = dphase - 2.0 * np.pi * np.round(dphase / (2.0 * np.pi))
        inc = phi_advance + dphase
        if dtypes is not None and t == 0:
            dtypes.update(alpha=np.asarray(alpha).dtype, mag=mag.dtype, dphase=dphase.dtype, inc=inc.dtype,
                          phase_acc=phase_acc.dtype, out=d_stretch.dtype)
        phase_acc += inc
    return d_stretch


def normalize_inf(S: np.ndarray, axis: int = 0) -> np.ndarray:
    """librosa.util.normalize(S, norm=np.inf) with its defaults (threshold = tiny(S), fill None)."""
    S = np.asarray(S)
    threshold = np.finfo(S.real.dtype if np.iscomplexobj(S) else S.dtype).tiny
    if not np.all(np.isfinite(S)):
        raise ParameterError("Input must be finite")
    mag = np.abs(S).astype(float)
    length = np.max(mag, axis=axis, keepdims=True)          # ValueError on an empty signal, as numpy raises
    small_idx = length < threshold
    Snorm = np.empty_like(S)
    length[small_idx] = 1.0
    Snorm[:] = S / length
    return Snorm


def _normalize(S, *, norm=np.inf, axis=0, threshold=None, fill=None):
    if norm != np.inf or threshold is not None or fill is not None:
        raise NotImplementedError("only librosa.util.normalize(S, norm=np.inf) is restated")
    return normalize_inf(S, axis=axis)


librosa = types.SimpleNamespace(stft=_stft, istft=_istft, phase_vocoder=phase_vocoder,
                                util=types.SimpleNamespace(normalize=_normalize, phasor=phasor),
                                fft_frequencies=fft_frequencies, ParameterError=ParameterError)


def n_frames(n: int) -> int:
    """STFT frames of n samples (centred, hop 512)."""
    return 1 + n // HOP


def out_frames(n: int, rate: float) -> int:
    """Frames of the stretched spectrum: len(np.arange(0, T, rate)) = ceil(T / rate) in double."""
    return int(np.ceil(n_frames(n) / float(rate)))


def out_len(n: int, rate: float) -> int:
    """Samples `change_speed` returns for n input samples: 512 * (ceil(T / rate) - 1)."""
    return HOP * (out_frames(n, rate) - 1)


def change_speed(wav: np.ndarray, rate: float, angle: Callable = np.angle) -> np.ndarray:
    """What TTSOutput.change_speed returns for rate != 1 (the array; the sample rate is unchanged)."""
    wav = np.asarray(wav, np.float32)
    D = _stft(wav, n_fft=N_FFT, hop_length=HOP)
    y = _istft(phase_vocoder(D, rate=rate, hop_length=HOP, angle=angle), hop_length=HOP)
    return normalize_inf(y)


# ---------------------------------------------------------------------------------------------------- fp32 DFT variant
_bases = None


def _dft_bases():
    global _bases
    if _bases is None:
        k, i = np.arange(N_FFT // 2 + 1), np.arange(N_FFT)
        w = _hann(N_FFT)
        a = 2.0 * np.pi * np.outer(k, i) / N_FFT                                    # [bin][tap]
        ck = np.where((k == 0) | (k == N_FFT // 2), 1.0, 2.0)
        fwd = np.concatenate([np.cos(a), -np.sin(a)]).astype(np.float32)          # [2 * bins][tap]
        inv = np.concatenate([w[:, None] * ck * np.cos(a.T) / N_FFT,
                              np.where(ck == 1.0, 0.0, -w[:, None] * ck * np.sin(a.T) / N_FFT)], axis=1)
        _bases = (w.astype(np.float32), fwd, inv.astype(np.float32).T.copy(), (w ** 2).astype(np.float32))
    return _bases


def change_speed_fp32_dft(wav: np.ndarray, rate: float):
    """change_speed with both transforms evaluated as fp32 DFT-by-matrix products (windowed frames x an fp32 cos / -sin
    basis; fp32 spectra x an fp32 windowed inverse basis, then the same float32 overlap-add), the way a GPU evaluates
    them, instead of numpy's fp64 FFTs.  Just as valid an evaluation of the same expression: its distance from
    `change_speed` shows how far two correct fp32 evaluations drift apart through the phase accumulator.
    -> (output, peak of the signal before normalisation)."""
    w, fwd, inv, w2 = _dft_bases()
    x = np.pad(np.asarray(wav, np.float32), (N_FFT // 2, N_FFT // 2))
    frames = np.lib.stride_tricks.sliding_window_view(x, N_FFT)[::HOP] * w[None, :]
    nb = N_FFT // 2 + 1
    R = frames @ fwd.T                                                              # [T][re bins | im bins]
    D = (R[:, :nb] + 1j * R[:, nb:]).T.astype(np.complex64)
    S = phase_vocoder(D, rate=rate, hop_length=HOP)
    Y = np.concatenate([S.real.T, S.imag.T], axis=1).astype(np.float32) @ inv        # [T'][tap], windowed
    T = Y.shape[0]
    n = N_FFT + HOP * (T - 1)
    y = np.zeros(n, np.float32)
    wss = np.zeros(n, np.float32)
    for t in range(T):
        y[t * HOP: t * HOP + N_FFT] += Y[t]
        wss[t * HOP: t * HOP + N_FFT] += w2
    y, wss = y[N_FFT // 2: n - N_FFT // 2], wss[N_FFT // 2: n - N_FFT // 2]
    nz = wss > np.finfo(np.float32).tiny
    y[nz] /= wss[nz]
    return normalize_inf(y), float(np.abs(y).max()) if y.size else 0.0
