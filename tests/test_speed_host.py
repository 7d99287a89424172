"""CPU: the speaking rate (TTSRequest.speed) — request validation, the chunk lengths every layer derives from the speed, and
the fused three-level interpolation formula the vocoder's interp_kernel implements, against the reference's chained
F.interpolate (tests/speed_reference.py)."""
import math

import numpy as np
import pytest
import torch

from auralis_b200.config import XTTSDims, speed_scale
from auralis_b200.requests import TTSRequest

import speed_reference as SR

SPEEDS = [0.25, 0.5, 0.7, 0.77, 1.0, 1.1, 1.3, 2.0, 3.3, 4.0]


def _req(**kw):
    return TTSRequest(text="hello there", speaker_files=["a.wav"], language="en", **kw)


def test_request_speed_default_and_copy():
    r = _req()
    assert r.speed == 1.0 and r.copy().speed == 1.0
    r = _req(speed=1.7)
    c = r.copy()
    assert c.speed == 1.7 and c is not r


@pytest.mark.parametrize("speed", [0.25, 4.0, 0.6, 2.5])
def test_request_speed_in_range_is_accepted(speed):
    assert _req(speed=speed).speed == speed


@pytest.mark.parametrize("speed", [0.0, -1.0, 0.2, 4.5, float("nan"), float("inf"), float("-inf")])
def test_request_speed_out_of_range_raises(speed):
    with pytest.raises(ValueError):
        _req(speed=speed)


@pytest.mark.parametrize("geom", ["small", "full"])
@pytest.mark.parametrize("speed", SPEEDS)
def test_z_frames_equal_the_reference_length(geom, speed):
    """z_frames(T, speed) is the length the reference's chained interpolations produce, for every chunk length; T0 == 0
    (a chunk scaled to no frame at all) gives 0."""
    vd = getattr(XTTSDims, geom)().voc
    zeros = torch.zeros(700, 2)
    n_empty = 0
    for T in range(1, 701):
        n = vd.z_frames(T, speed)
        assert n == SR.interp_latents(zeros[:T], vd, speed).shape[-1], (T, speed)
        assert vd.n_samples(T, speed) == n * vd.hop
        n_empty += n == 0
        if speed == 1.0:
            assert n == vd.z_frames(T)
    assert n_empty == math.ceil(float(np.float32(speed))) - 1            # T0 == 0 exactly when T < speed


def test_zero_frame_chunks():
    vd = XTTSDims.full().voc
    assert [vd.z_frames(T, 4.0) for T in (1, 2, 3, 4)] == [0, 0, 0, vd.z_frames(1)]
    assert SR.vocoder(torch.zeros(3, 8), None, None, None, 4.0).numel() == 0


@pytest.mark.parametrize("geom", ["small", "full"])
@pytest.mark.parametrize("speed", SPEEDS)
def test_fused_formula_equals_chained_interpolate(geom, speed):
    """The kernel's global-index formula (whole chunks and windows starting at z0 > 0) equals the reference's chained
    F.interpolate within 1e-6."""
    vd = getattr(XTTSDims, geom)().voc
    rng = np.random.RandomState(int(speed * 100))
    for T in (1, 2, 3, 7, 40, 123, 605):
        lat = rng.randn(T, 8).astype(np.float32)
        ref = SR.interp_latents(torch.from_numpy(lat), vd, speed).numpy()
        Tz = ref.shape[1]
        assert Tz == vd.z_frames(T, speed)
        T0 = math.floor(T * speed_scale(speed))
        if Tz == 0 or (T0 >= 2 and Tz == math.floor(T0 * vd.code_stride / vd.output_hop_length)):
            # (T0 == 2: the 24 kHz resampling keeps the length, 8 -> 8, and F.interpolate copies instead of resampling;
            # the vocoder resamples those 8 frames, at every speed — outside this formula's scope)
            continue
        for z0, z1 in [(0, Tz), (Tz // 3, Tz), (Tz // 2, Tz - Tz // 4), (Tz - 1, Tz)]:
            if z1 <= z0:
                continue
            got = SR.fused_z(lat, vd, speed, z0, z1 - z0)
            np.testing.assert_allclose(got, ref[:, z0:z1], rtol=0, atol=1e-6, err_msg=f"T={T} speed={speed} [{z0},{z1})")


def test_native_submit_passes_the_speed():
    """NativeEngine.submit goes through xtts_submit_speed with Sampling.speed as float32 (the struct itself cannot grow)."""
    from auralis_b200 import native

    calls = []

    class _Lib:
        def xtts_submit_speed(self, h, sid, ids, n, spk, sp, speed):
            calls.append((sid, n, spk, speed))
            return 0

    eng = object.__new__(native.NativeEngine)
    eng.lib, eng.h = _Lib(), None
    eng.submit(7, [0, 5, 1], 1, native.Sampling(speed=0.7))
    eng.submit(8, [0, 1], 0, native.Sampling())
    assert calls == [(7, 3, 1, 0.7), (8, 2, 0, 1.0)]
