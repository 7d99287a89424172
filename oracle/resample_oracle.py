"""numpy restatement of `torchaudio.functional.resample(x, orig, new)` for float32 `x` with the defaults every caller
uses (``sinc_interp_hann``, ``lowpass_filter_width = 6``, ``rolloff = 0.99``): the arithmetic ``xtts_resample``
implements on the GPU.

torchaudio builds its `new' x (2 width + orig')` coefficient table in the waveform's dtype (float32), then runs a strided
conv1d over every tap.  `coefficients` rebuilds that table with the same float32 operation order; only the cosine and
sine differ: they are evaluated in float64 and rounded to float32 (torchaudio's SIMD sinf / cosf are within 1 ulp of
that, the GPU's within 2).  Outputs are then summed in float64:

* `resample_dense`: all 2 width + L taps, as torchaudio's conv1d does;
* `resample_banded`: only the taps whose scaled argument lies strictly inside the window (-6, 6), the taps the GPU
  kernel evaluates.  The taps outside have the clamped argument +-6 and coefficients below 5e-24;
* `abs_sum`: the per-output bound quantity sum_k |c_k x_k| over all taps, and `skipped_sum` the same over the taps
  outside the window.
"""
from __future__ import annotations

import math
from typing import Tuple

import numpy as np

WIDTH = 6
ROLLOFF = 0.99
MAX_RATE = (1 << 20) - 1
F32 = np.float32


def params(orig: int, new: int) -> Tuple[int, int, float, int]:
    """-> (L, M, base, width): the rates over their gcd, torchaudio's `base_freq` (float64) and filter width."""
    g = math.gcd(int(orig), int(new))
    L, M = int(orig) // g, int(new) // g
    base = min(L, M) * ROLLOFF
    return L, M, base, math.ceil(WIDTH * L / base)


def out_len(n: int, orig: int, new: int) -> int:
    """ceil(M n / L) in integers (torchaudio takes the ceil of the float64 quotient; the two agree for every rate pair
    in range, because a non-integer quotient is at least 1 / L from an integer)."""
    if orig == new:
        return n
    L, M, _, _ = params(orig, new)
    return -(-M * n // L)


def scaled_args(orig: int, new: int, phases=None) -> np.ndarray:
    """t[p][k] before the clamp: f32(f32(f32(-p) / M) + f32(k - width) / L) * f32(base), [phases][2 width + L]
    (default: all M phases)."""
    L, M, base, width = params(orig, new)
    p = np.arange(M) if phases is None else np.asarray(phases)
    idx = (np.arange(-width, width + L, dtype=F32) / F32(L))[None, :]
    t = (-p.astype(F32) / F32(M))[:, None] + idx
    return t * F32(base)


def coefficients(orig: int, new: int, phases=None) -> np.ndarray:
    """torchaudio's float32 kernel [phases][2 width + L], cos / sin correctly rounded to float32."""
    L, M, base, width = params(orig, new)
    t = np.clip(scaled_args(orig, new, phases), F32(-WIDTH), F32(WIDTH))
    arg = t * F32(math.pi) / F32(WIDTH) / F32(2)
    cw = np.cos(arg.astype(np.float64)).astype(F32)
    window = cw * cw
    t = t * F32(math.pi)
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.where(t == 0, F32(1), np.sin(t.astype(np.float64)).astype(F32) / t)
    return (s * (window * F32(base / L))).astype(F32)


def in_window(orig: int, new: int, phases=None) -> np.ndarray:
    """[phases][2 width + L] bool: the taps whose scaled argument is strictly inside (-6, 6) (a contiguous run per
    phase)."""
    t = scaled_args(orig, new, phases)
    return (t > -WIDTH) & (t < WIDTH)


def _rows(orig: int, new: int, phases, kind: str) -> np.ndarray:
    """float64 coefficient rows of `phases` for one of the sums below."""
    c = coefficients(orig, new, phases).astype(np.float64)
    if kind in ("banded", "skipped"):
        w = in_window(orig, new, phases)
        c = np.where(w, c, 0) if kind == "banded" else np.where(w, 0, c)
    return np.abs(c) if kind in ("abs", "skipped") else c


def _sum(x, orig: int, new: int, kind: str, j0: int, j1) -> np.ndarray:
    """sum_k c[p][k] * x[q L + k - width] for outputs j = q M + p in [j0, j1), float64, zero outside [0, n) (|c| |x| for
    "abs" / "skipped"); blocked, and with only the block's phases built, so the gathered taps stay small."""
    L, M, _, width = params(orig, new)
    n = x.shape[0]
    j1 = out_len(n, orig, new) if j1 is None else j1
    taps = 2 * width + L
    xd = x.astype(np.float64)
    if kind in ("abs", "skipped"):
        xd = np.abs(xd)
    out = np.empty((max(j1 - j0, 0),), np.float64)
    step = max(1, (1 << 22) // taps)
    k = np.arange(taps, dtype=np.int64)[None, :]
    for a in range(j0, j1, step):
        j = np.arange(a, min(a + step, j1), dtype=np.int64)
        q, p = j // M, j % M
        phases, inv = np.unique(p, return_inverse=True)
        pos = (q * L - width)[:, None] + k
        xs = np.where((pos >= 0) & (pos < n), xd[np.clip(pos, 0, max(n - 1, 0))] if n else 0.0, 0.0)
        out[a - j0: a - j0 + j.shape[0]] = np.einsum("jk,jk->j", xs, _rows(orig, new, phases, kind)[inv])
    return out


def _check(x) -> np.ndarray:
    x = np.asarray(x)
    if x.ndim != 1:
        raise ValueError("mono input only")
    return x.astype(F32)


def resample_dense(x, orig: int, new: int, j0: int = 0, j1=None) -> np.ndarray:
    """Outputs [j0, j1) (default: all): the float64 sum over all 2 width + L taps of the float32 coefficients."""
    x = _check(x)
    if orig == new:
        return x.astype(np.float64)[j0:j1]
    return _sum(x, orig, new, "dense", j0, j1)


def resample_banded(x, orig: int, new: int, j0: int = 0, j1=None) -> np.ndarray:
    """Outputs [j0, j1): the float64 sum over the in-window taps only."""
    x = _check(x)
    if orig == new:
        return x.astype(np.float64)[j0:j1]
    return _sum(x, orig, new, "banded", j0, j1)


def abs_sum(x, orig: int, new: int, j0: int = 0, j1=None) -> np.ndarray:
    """Outputs [j0, j1): sum_k |c_k x_k| over all taps."""
    return _sum(_check(x), orig, new, "abs", j0, j1)


def skipped_sum(x, orig: int, new: int, j0: int = 0, j1=None) -> np.ndarray:
    """Outputs [j0, j1): sum_k |c_k x_k| over the taps outside the window."""
    return _sum(_check(x), orig, new, "skipped", j0, j1)


def band_taps(orig: int, new: int) -> int:
    """T = 2 width + 2: the most in-window taps any phase has (checked by `in_window`)."""
    return 2 * params(orig, new)[3] + 2


# ---- seeded test signals (tests/golden/make_resample_golden.py and the tests rebuild the same inputs)
GOLDEN_PAIRS = [(44100, 22050), (22050, 16000), (48000, 22050), (44100, 16000), (24000, 44100), (24000, 48000),
                (24000, 16000), (24000, 22050), (8000, 22050), (2, 3), (3, 2), (1009, 1013)]
KINDS = ("noise", "sine", "impulse", "dc")
SPEAKER_PAIRS = [(44100, 22050), (22050, 16000)]          # a 44.1 kHz reference to load_sr, load_sr to 16 kHz


def signal(kind: str, n: int, orig: int, new: int, seed: int) -> np.ndarray:
    """float32 [n]: "noise" (normal, sd 0.3), "sine" (two sines at 0.97 and 0.9 of the lower Nyquist, random
    phases), "impulse" (three impulses: the first, a middle and the last sample), "dc" (0.25)."""
    rng = np.random.RandomState(seed)
    if kind == "noise":
        return (rng.randn(n) * 0.3).astype(F32)
    if kind == "sine":
        ny = min(orig, new) / 2.0
        t = np.arange(n, dtype=np.float64) / orig
        ph = rng.rand(2) * 2 * np.pi
        return (0.5 * np.sin(2 * np.pi * 0.97 * ny * t + ph[0]) + 0.3 * np.sin(2 * np.pi * 0.9 * ny * t + ph[1])).astype(F32)
    if kind == "impulse":
        x = np.zeros(n, F32)
        for i, v in ((0, 1.0), (n // 3, -0.7), (n - 1, 0.5)):
            if 0 <= i < n:
                x[i] = v
        return x
    if kind == "dc":
        return np.full(n, 0.25, F32)
    raise ValueError(kind)


def golden_cases():
    """[(orig, new, n, kind, seed)]: every pair and signal at lengths 0, 1, 2, width, L, 2 width + L +- 1, then noise
    (2 s for the speaker pairs, else 0.25 s) and 0.25 s of sines (at least 4000 samples each)."""
    cases = []
    for pi, (o, nw) in enumerate(GOLDEN_PAIRS):
        L, _, _, w = params(o, nw)
        lengths = sorted({0, 1, 2, w, L, 2 * w + L - 1, 2 * w + L + 1})
        for ki, kind in enumerate(KINDS):
            for n in lengths:
                cases.append((o, nw, n, kind, 1000 * pi + 10 * ki + lengths.index(n)))
        cases.append((o, nw, 2 * o if (o, nw) in SPEAKER_PAIRS else max(o // 4, 4000), "noise", 1000 * pi + 500))
        cases.append((o, nw, max(o // 4, 4000), "sine", 1000 * pi + 501))
    return cases
