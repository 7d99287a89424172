"""GPU: `xtts_resample` (speaker references, conditioning, `TTSOutput.resample`) against torchaudio's own outputs
(tests/golden/resample_reference.npz) and the float64 oracle (oracle/resample_oracle.py), its exact cases, invariance to
the pass size, long inputs, its errors, and the end-to-end paths through a live engine.

Error bound.  u = 2^-24, g(a) = a u / (1 - a u), S = sum_k |c_k x_k| over all 2 width + L taps (the oracle's `abs_sum`),
Z = the same over the taps outside the window (`skipped_sum`, all with |c| < 5e-24).
* Coefficients: the GPU and torchaudio evaluate the same float32 operations on the same arguments except cosf / sinf:
  CUDA's are within 2 ulp, torchaudio's SIMD ones within 1 ulp, the oracle's correctly rounded.  Two differing sines
  (3 ulp), a squared cosine (2 x 3 ulp) and the four roundings after them that no longer see equal operands (4 x 1 ulp):
  13 ulp <= 26 u relative per coefficient.
* Sums: the GPU's T-tap FMA chain (T = 2 width + 2) is within T u S of the exact sum of its products; torchaudio's
  conv1d sums K = 2 width + L products, within (K - 1) u S in any order; the oracle sums in float64.
* The GPU skips the window's outside taps: at most Z.
So |gpu - torchaudio| <= g(T + K + 26) S + Z and |gpu - oracle| <= g(T + 26) S + Z.  The worst measured fraction of
each bound is printed.
"""
import ctypes as C
import os
import wave

import numpy as np
import pytest

from oracle import resample_oracle as R

pytestmark = [pytest.mark.gpu]
U = 2.0 ** -24
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "resample_reference.npz")
DEFAULT_BLOCK = 1 << 22


def gamma(a):
    return a * U / (1 - a * U)


@pytest.fixture(scope="module")
def eng():
    from auralis_b200 import native
    from auralis_b200.config import XTTSDims
    e = native.NativeEngine(XTTSDims.small(), device=0, max_batch=1, max_speakers=1)      # needs no weights
    yield e
    e.close()


def _bounds(x, o, nw, j0=0, j1=None):
    L, M, base, w = R.params(o, nw)
    T = min(2 * w + 2, 2 * w + L)
    S, Z = R.abs_sum(x, o, nw, j0, j1), R.skipped_sum(x, o, nw, j0, j1)
    return gamma(T + 2 * w + L + 26) * S + Z, gamma(T + 26) * S + Z


def _ratio(err, bound):
    return float(np.max(err / np.maximum(bound, 1e-300), initial=0.0))


def _rounding_ratio(err, x, o, nw, a):
    """The worst (err - Z) / (g(a) S): the share of the rounding part of the bound that is used (outputs whose only
    non-zero taps are skipped ones reach the Z term exactly and say nothing about rounding)."""
    S, Z = R.abs_sum(x, o, nw), R.skipped_sum(x, o, nw)
    return float(np.max(np.maximum(err - Z, 0) / np.maximum(gamma(a) * S, 1e-300), initial=0.0))


def test_golden_parity(eng):
    z = np.load(GOLDEN)
    worst_ta = worst_or = 0.0
    for i, (o, nw, n, k, seed) in enumerate(z["meta"]):
        o, nw, n = int(o), int(nw), int(n)
        x = R.signal(R.KINDS[int(k)], n, o, nw, int(seed))
        y = eng.resample(x, o, nw)
        want = z[f"y{i}"]
        assert y.dtype == np.float32 and y.shape == want.shape == (R.out_len(n, o, nw),), (o, nw, n)
        if n == 0:
            continue
        b_ta, b_or = _bounds(x, o, nw)
        e_ta = np.abs(y.astype(np.float64) - want)
        e_or = np.abs(y.astype(np.float64) - R.resample_dense(x, o, nw))
        assert np.all(e_ta <= b_ta), (o, nw, n, _ratio(e_ta, b_ta))
        assert np.all(e_or <= b_or), (o, nw, n, _ratio(e_or, b_or))
        L, M, base, w = R.params(o, nw)
        T = min(2 * w + 2, 2 * w + L)
        worst_ta = max(worst_ta, _rounding_ratio(e_ta, x, o, nw, T + 2 * w + L + 26))
        worst_or = max(worst_or, _rounding_ratio(e_or, x, o, nw, T + 26))
    print(f"worst share of the rounding bound: vs torchaudio {worst_ta:.3g}, vs the oracle {worst_or:.3g}")


@pytest.mark.parametrize("o,nw,n", [(48000, 8000, 3000), (22050, 44101, 3000), (1, 7, 3000), (7, 1, 3000),
                                    (1048575, 1048573, 2_000_000), (1, 1048575, 5), (1048575, 2, 2_000_000)])
def test_other_rate_pairs_match_the_oracle(eng, o, nw, n):
    """Heavy downsampling, coprime rates (a 44 101-phase table where torchaudio's would be 3.6 GiB), the extremes of the
    rate range (a million phases, or a band of 6.4 M taps read from global memory): the first outputs and a spread of
    others."""
    x = R.signal("noise", n, o, nw, 77)
    y = eng.resample(x, o, nw)
    assert y.shape == (R.out_len(n, o, nw),)
    js = sorted({*range(min(y.shape[0], 64)), *np.linspace(0, y.shape[0] - 1, 12).astype(int).tolist()})
    worst = 0.0
    for j in js:
        _, b = _bounds(x, o, nw, j, j + 1)
        e = np.abs(float(y[j]) - R.resample_dense(x, o, nw, j, j + 1))
        assert np.all(e <= b), (j, _ratio(e, b))
        worst = max(worst, _ratio(e, b))
    print(f"{o} -> {nw}: worst |gpu - oracle| / bound = {worst:.3g}")


def test_exact_cases(eng):
    rng = np.random.RandomState(3)
    x = (rng.randn(5000) * 10).astype(np.float32)
    x[:4] = [0.0, -0.0, 1e-40, -3.4e38]
    y = eng.resample(x, 22050, 22050)
    assert y.tobytes() == x.tobytes()
    for o, nw in R.GOLDEN_PAIRS:
        zr = eng.resample(np.zeros(1234, np.float32), o, nw)
        assert zr.shape == (R.out_len(1234, o, nw),) and not np.any(zr)
        assert eng.resample(np.zeros(0, np.float32), o, nw).shape == (0,)
    a, b = eng.resample(x, 44100, 16000), eng.resample(x, 44100, 16000)
    eng.resample(x, 24000, 44100)                           # another table in between
    c = eng.resample(x, 44100, 16000)
    assert a.tobytes() == b.tobytes() == c.tobytes()


def _blocks(eng, x, o, nw, values):
    outs = []
    try:
        for v in values:
            eng.set_option("resample_block_samples", v)
            outs.append(eng.resample(x, o, nw))
    finally:
        eng.set_option("resample_block_samples", DEFAULT_BLOCK)
    return outs


@pytest.mark.parametrize("o,nw", [(24000, 44100), (22050, 16000), (48000, 8000)])
def test_block_size_invariance(eng, o, nw):
    """Pass sizes 1 and 7 on the first 2 s (one pass per output or seven is 10^6-10^7 passes over 10 minutes), 4096, the
    default and one whole pass on 10 minutes: bit-identical."""
    x = R.signal("noise", 600 * o, o, nw, 11)
    n_out = R.out_len(x.shape[0], o, nw)
    short = x[: 2 * o]
    ref = _blocks(eng, short, o, nw, [DEFAULT_BLOCK])[0]
    for y in _blocks(eng, short, o, nw, [1, 7]):
        assert y.tobytes() == ref.tobytes()
    outs = _blocks(eng, x, o, nw, [4096, DEFAULT_BLOCK, min(n_out, 1 << 26)])
    assert outs[0].shape == (n_out,)
    assert outs[0].tobytes() == outs[1].tobytes() == outs[2].tobytes()
    assert outs[0][: 2 * nw - 100].tobytes() == ref[: 2 * nw - 100].tobytes()   # away from the excerpt's cut


def test_one_hour_book(eng):
    """One hour of 24 kHz speech-band noise to 44.1 kHz, checked against the oracle in chunks across the hour."""
    o, nw = 24000, 44100
    x = R.signal("noise", 3600 * o, o, nw, 12)
    y = eng.resample(x, o, nw)
    n_out = R.out_len(x.shape[0], o, nw)
    assert y.shape == (n_out,) and np.all(np.isfinite(y))
    L, M, _, w = R.params(o, nw)
    worst = 0.0
    for j0 in [0, 1, n_out // 3, n_out // 2 + 7, n_out - 50_000, n_out - 20_000]:
        j1 = min(n_out, j0 + 20_000)
        # the oracle on an excerpt that starts at a multiple of L (so its outputs line up) and holds every sample read
        s = max(0, (j0 // M - w // L - 2) * L)
        e = min(x.shape[0], ((j1 - 1) // M + 1) * L + w + 1)
        xs, k0 = x[s:e], s // L * M
        _, b = _bounds(xs, o, nw, j0 - k0, j1 - k0)
        err = np.abs(y[j0:j1].astype(np.float64) - R.resample_dense(xs, o, nw, j0 - k0, j1 - k0))
        assert np.all(err <= b), (j0, _ratio(err, b))
        worst = max(worst, _ratio(err, b))
    print(f"1 h: worst |gpu - oracle| / bound = {worst:.3g}")


def test_errors(eng):
    from auralis_b200 import native
    x = R.signal("noise", 1000, 44100, 16000, 13)
    before = eng.stats().cond_ms
    for o, nw in [(0, 16000), (44100, 0), (-5, 16000), (1 << 20, 16000), (44100, 1 << 20)]:
        with pytest.raises(native.NativeError) as ei:
            eng.resample(x, o, nw)
        assert ei.value.code == native.ERR_INVALID
    for bad in (np.nan, np.inf, -np.inf):
        for pos in (0, 500, 999):
            xb = x.copy()
            xb[pos] = bad
            with pytest.raises(native.NativeError) as ei:
                eng.resample(xb, 44100, 16000)
            assert ei.value.code == native.ERR_INVALID and "finite" in str(ei.value)
    lib, f32p = eng.lib, C.POINTER(C.c_float)
    n_out = C.c_int64(-1)
    out = np.empty(400, np.float32)
    xp = x.ctypes.data_as(f32p)
    assert lib.xtts_resample(eng.h, xp, 1000, 44100, 16000, out.ctypes.data_as(f32p), 362, C.byref(n_out)) == native.ERR_INVALID
    assert n_out.value == 363                                # ceil(160 * 1000 / 441), set although cap is short
    assert lib.xtts_resample(eng.h, xp, -1, 44100, 16000, out.ctypes.data_as(f32p), 400, C.byref(n_out)) == native.ERR_INVALID
    assert lib.xtts_resample(eng.h, None, 10, 44100, 16000, out.ctypes.data_as(f32p), 400, C.byref(n_out)) == native.ERR_INVALID
    assert lib.xtts_resample(eng.h, xp, 1000, 44100, 16000, None, 400, C.byref(n_out)) == native.ERR_INVALID
    assert lib.xtts_resample(eng.h, xp, 1000, 44100, 16000, out.ctypes.data_as(f32p), 400, None) == native.ERR_INVALID
    assert lib.xtts_resample(eng.h, xp, 1000, 44100, 16000, out.ctypes.data_as(f32p), 363, C.byref(n_out)) == 0
    assert n_out.value == 363
    for v in (0, (1 << 26) + 1):
        with pytest.raises(native.NativeError):
            eng.set_option("resample_block_samples", v)
    y = eng.resample(x, 44100, 16000)                       # still serving
    _, b = _bounds(x, 44100, 16000)
    assert np.all(np.abs(y - R.resample_dense(x, 44100, 16000)) <= b)
    assert eng.stats().cond_ms > before


# ---------------------------------------------------------------------------------------------------- end to end
@pytest.fixture(scope="module")
def tts(tmp_path_factory, dims_small, state_small):
    from auralis_b200 import TTS
    from auralis_b200.weights import save_model_dir
    d = tmp_path_factory.mktemp("model")
    save_model_dir(str(d), dims_small, state_small[0], state_small[1])
    t = TTS(scheduler_max_concurrency=8).from_pretrained(str(d), precision="fp32", max_concurrency=4)
    yield t
    if t.tts_engine is not None and getattr(t.tts_engine, "_stop", False) is False:
        t.loop.run_until_complete(t.shutdown())


def _write_wav(path, x, sr):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(sr)
        w.writeframes((np.clip(x, -1, 1) * 32767).astype("<i2").tobytes())
    return str(path)


def test_speaker_references_condition_through_the_gpu_resampler(tts, tmp_path):
    from auralis_b200 import output
    from auralis_b200.engine import _resample, load_audio
    eng = tts.tts_engine
    assert output.gpu_provider() is eng
    for sr in (44100, 48000):
        t = np.arange(int(2.5 * sr)) / sr
        x = (0.3 * np.sin(2 * np.pi * 150 * t) * (1 + 0.5 * np.sin(2 * np.pi * 3 * t))
             + 0.02 * np.random.RandomState(sr).randn(t.size)).astype(np.float32)
        f = _write_wav(tmp_path / f"r{sr}.wav", x, sr)
        cond, g = tts.loop.run_until_complete(eng.get_audio_conditioning(f, 60, 30, 4))
        slot = eng.max_speakers - 1
        a22 = load_audio(f, 22050)
        eng.native.condition(slot, a22, _resample(a22, 22050, 16000), 30, 4)
        rc, rg = eng.native.get_speaker(slot)
        assert np.asarray(cond)[0].tobytes() == rc.tobytes()
        assert np.asarray(g).reshape(-1).tobytes() == rg.tobytes()
        ta = pytest.importorskip("torchaudio")
        import torch
        pcm = (np.clip(x, -1, 1) * 32767).astype("<i2").astype(np.float32) / 32768.0
        h22 = np.clip(ta.functional.resample(torch.from_numpy(pcm), sr, 22050).numpy(), -1, 1).astype(np.float32)
        np.testing.assert_allclose(a22, h22, rtol=0, atol=1e-5)
        h16 = ta.functional.resample(torch.from_numpy(h22), 22050, 16000).numpy()
        eng.native.condition(slot, h22, h16, 30, 4)
        hc, hg = eng.native.get_speaker(slot)
        assert np.abs(rc - hc).max() < 2e-3 * max(1.0, np.abs(hc).max()), np.abs(rc - hc).max()
        assert np.abs(rg - hg).max() < 2e-4, np.abs(rg - hg).max()


def test_generated_speech_resamples_on_the_gpu(tts, tmp_path):
    from auralis_b200 import TTSRequest
    from auralis_b200.output import _parse_riff_wav
    eng = tts.tts_engine
    f = _write_wav(tmp_path / "s.wav", (0.3 * np.sin(2 * np.pi * 140 * np.arange(50000) / 22050)).astype(np.float32), 22050)
    out = tts.generate_speech(TTSRequest(text="A short sentence to speak.", speaker_files=f, language="en", temperature=0.0))
    assert out.sample_rate == 24000 and out.array.size > 0
    r = out.resample(44100)
    want = eng.resample(out.array, 24000, 44100)
    assert r.sample_rate == 44100 and r.array.tobytes() == want.tobytes()
    out.save(tmp_path / "x.wav", sample_rate=16000)
    a, sr = _parse_riff_wav((tmp_path / "x.wav").read_bytes())
    assert sr == 16000
    assert a[:, 0].tobytes() == np.clip(eng.resample(out.array, 24000, 16000), -1, 1).tobytes()
    stereo = np.stack([out.array, -out.array])
    from auralis_b200.output import TTSOutput
    s = TTSOutput(array=stereo, sample_rate=24000).resample(48000)
    assert s.array.shape == (2, 2 * out.array.size) and np.array_equal(s.array[1], -s.array[0])


def test_after_shutdown_the_host_path_is_back(tts):
    from auralis_b200 import output
    from auralis_b200.output import TTSOutput
    x = R.signal("noise", 3000, 24000, 44100, 14)
    gpu = TTSOutput(array=x, sample_rate=24000).resample(44100).array
    tts.loop.run_until_complete(tts.shutdown())
    assert output.gpu_provider() is None or not hasattr(output.gpu_provider(), "resample") \
        or output.gpu_provider() is not tts.tts_engine
    if output.gpu_provider() is not None:
        pytest.skip("another live engine is registered")
    host = TTSOutput(array=x, sample_rate=24000).resample(44100).array
    assert host.shape == gpu.shape
    try:
        import torch
        import torchaudio
        want = torchaudio.functional.resample(torch.from_numpy(x)[None], 24000, 44100).squeeze().numpy()
        assert host.tobytes() == want.tobytes()
    except ImportError:
        pass
