"""Reference for the speaking rate (TTSRequest.speed / xtts_submit_speed), restated for the tests.

Coqui XTTS's own speed control (``Xtts.inference(..., speed=1.0)``) time-scales the GPT latents right before the HiFi-GAN
decoder:

    length_scale = 1.0 / max(speed, 0.05)
    if length_scale != 1.0:
        gpt_latents = F.interpolate(gpt_latents.transpose(1, 2), scale_factor=length_scale, mode="linear").transpose(1, 2)
    wav = self.hifigan_decoder(gpt_latents, g=speaker_embedding)

Restated here from Coqui's public code, which is not vendored: **unpinned to Coqui** (the arithmetic itself is torch's own
``F.interpolate``).  The speed reaches every layer as float32, so the scale is computed from that value
(``auralis_b200.config.speed_scale``).  Everything after the stage is the pinned oracle (``oracle/xtts_oracle.py``), applied
unchanged to the scaled latents.  A chunk scaled to zero frames (e.g. 3 latents at speed 4) has an empty waveform.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from auralis_b200.config import speed_scale
from oracle import xtts_oracle as O


def scale_latents(latents: torch.Tensor, speed: float) -> torch.Tensor:
    """[T, C] -> [floor(T * ls), C]; speed 1 returns the latents untouched (Coqui skips the stage)."""
    if float(np.float32(speed)) == 1.0:
        return latents
    ls = speed_scale(speed)
    if math.floor(latents.shape[0] * ls) == 0:
        return latents[:0]
    return F.interpolate(latents.t()[None], scale_factor=ls, mode="linear", align_corners=False)[0].t()


def interp_latents(latents: torch.Tensor, vd, speed: float = 1.0) -> torch.Tensor:
    """z [C, z_frames(T, speed)]: the speed stage, then the vocoder's two interpolations."""
    y = scale_latents(latents, speed)
    if y.shape[0] == 0:
        return torch.zeros(latents.shape[1], 0)
    return O.interp_latents(y, vd)


def vocoder(latents: torch.Tensor, g: torch.Tensor, core, dims, speed: float = 1.0) -> torch.Tensor:
    """wav [n_samples(T, speed)]"""
    y = scale_latents(latents, speed)
    if y.shape[0] == 0:
        return torch.zeros(0)
    return O.vocoder(y.contiguous(), g, core, dims)


def _lin_src(dst: np.ndarray, r: np.float32, n: int):
    """torch's linear source index (align_corners=False) in float32, as the kernel's lin_src.  r * (j + .5) - .5 is one
    fused multiply-add on both sides (nvcc contracts it; ATen's CPU build does too): exact product, one rounding — float64
    holds the product of two float32 values exactly."""
    x = (dst.astype(np.float32) + np.float32(0.5)).astype(np.float64)
    src = (np.float64(np.float32(r)) * x - 0.5).astype(np.float32)
    src = np.maximum(src, np.float32(0.0))
    i0 = np.minimum(src.astype(np.int64), n - 1)
    i1 = i0 + (i0 < n - 1)
    l1 = (src - i0.astype(np.float32)).astype(np.float32)
    return i0, i1, (np.float32(1.0) - l1).astype(np.float32), l1


def _lerp(l0, x0, l1, x1):
    """l0 * x0 + l1 * x1 rounded as ATen's CPU kernel does: fma(l0, x0, l1 * x1)."""
    return (l0[:, None].astype(np.float64) * x0 + (l1[:, None] * x1).astype(np.float32)).astype(np.float32)


def fused_z(latents: np.ndarray, vd, speed: float, z0: int, nz: int) -> np.ndarray:
    """The formula interp_kernel evaluates (csrc/vocoder.cu): z-frames [z0, z0 + nz) of the chunk at their GLOBAL index,
    each from up to 8 latent rows through three chained linear interpolations (two at speed 1).  -> [C, nz] float32"""
    lat = np.asarray(latents, np.float32)
    T = lat.shape[0]
    s1 = vd.code_stride / vd.output_hop_length
    resample = vd.output_sample_rate != vd.input_sample_rate
    s2 = vd.output_sample_rate / vd.input_sample_rate if resample else 1.0
    r1, r2 = np.float32(1.0 / s1), np.float32(1.0 / s2)

    ls = speed_scale(speed)
    Ty = int(math.floor(T * ls))
    if Ty == T:                     # speed 1, or a chunk too short to change length: F.interpolate copies, no stage
        def y0(b):
            return lat[b]
    else:
        r0 = np.float32(1.0 / ls)
        def y0(b):
            c0, c1, p0, p1 = _lin_src(b, r0, T)
            return _lerp(p0, lat[c0], p1, lat[c1])
    T1 = int(math.floor(Ty * s1)) if resample else Ty

    def y1(a):
        b0, b1, n0, n1 = _lin_src(a, r1, Ty)
        return _lerp(n0, y0(b0), n1, y0(b1))

    a0, a1, m0, m1 = _lin_src(np.arange(z0, z0 + nz), r2, T1)
    return _lerp(m0, y1(a0), m1, y1(a1)).T
