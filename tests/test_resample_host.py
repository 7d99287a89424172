"""Host side of the GPU resampler: the numpy restatement of torchaudio's resampler (oracle/resample_oracle.py) against
live torchaudio and the golden file, the banded form against the dense one, and the dispatch of `TTSOutput.resample`,
`save(sample_rate=)`, `load_audio` and `engine._resample` between a live engine's `resample` and the host path.

Error bound against torchaudio: the oracle uses torchaudio's float32 coefficients (its cos / sin correctly rounded,
torchaudio's within 1 ulp; with the roundings after them a coefficient differs by at most ~13 ulp = 26 u, u = 2^-24)
and sums in float64; torchaudio's conv1d sums K = 2 width + L products in float32 in some order, at most (K - 1) u of
sum_k |c_k x_k|.  So |torchaudio - oracle| <= g(K + 26) * sum_k |c_k x_k|, g(a) = a u / (1 - a u).
"""
import io
import os
import wave

import numpy as np
import pytest

from oracle import resample_oracle as R

U = 2.0 ** -24
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "resample_reference.npz")


def gamma(a):
    return a * U / (1 - a * U)


def _golden():
    z = np.load(GOLDEN)
    return [(int(o), int(nw), int(n), R.KINDS[int(k)], int(s), z[f"y{i}"]) for i, (o, nw, n, k, s) in enumerate(z["meta"])]


def _check_oracle(x, o, nw, want):
    L, M, base, w = R.params(o, nw)
    assert want.shape == (R.out_len(x.shape[0], o, nw),)
    if x.shape[0] == 0:
        return 0.0
    d = R.resample_dense(x, o, nw)
    bound = gamma(2 * w + L + 26) * R.abs_sum(x, o, nw)
    err = np.abs(want.astype(np.float64) - d)
    assert np.all(err <= bound + 1e-45), (o, nw, x.shape[0], float(np.max(err - bound)))
    return float(np.max(np.where(bound > 0, err / np.maximum(bound, 1e-300), 0)))


def test_golden_cases_cover_the_issue():
    cases = R.golden_cases()
    assert {(o, nw) for o, nw, *_ in cases} == set(R.GOLDEN_PAIRS)
    assert len(_golden()) == len(cases)
    for (o, nw, n, k, s), (go, gn, gl, gk, gs, y) in zip(cases, _golden()):
        assert (o, nw, n, k, s) == (go, gn, gl, gk, gs)
        assert y.dtype == np.float32 and y.shape == (R.out_len(n, o, nw),)


def test_oracle_matches_golden():
    worst = 0.0
    for o, nw, n, kind, seed, y in _golden():
        worst = max(worst, _check_oracle(R.signal(kind, n, o, nw, seed), o, nw, y))
    print(f"golden: worst |torchaudio - oracle| / bound = {worst:.3g}")


def test_oracle_matches_live_torchaudio():
    torch = pytest.importorskip("torch")
    ta = pytest.importorskip("torchaudio")
    rng = np.random.RandomState(123)
    pairs = R.GOLDEN_PAIRS + [(48000, 8000), (16000, 44100), (7, 5)]
    for o, nw in pairs:
        for n in (1, 3, int(rng.randint(5, 30000))):
            x = (rng.randn(n) * rng.choice([1e-3, 0.3, 40.0])).astype(np.float32)
            y = ta.functional.resample(torch.from_numpy(x), o, nw).numpy()
            _check_oracle(x, o, nw, y)


def test_golden_is_live_torchaudio():
    torch = pytest.importorskip("torch")
    ta = pytest.importorskip("torchaudio")
    for o, nw, n, kind, seed, y in _golden()[::7]:
        if n:
            got = ta.functional.resample(torch.from_numpy(R.signal(kind, n, o, nw, seed)), o, nw).numpy()
            np.testing.assert_array_equal(got, y)


@pytest.mark.parametrize("o,nw", R.GOLDEN_PAIRS + [(48000, 8000), (1, 7), (7, 1)])
def test_banded_agrees_with_dense(o, nw):
    """The skipped taps are the ones with the clamped argument +-6, all below 5e-24; every phase's in-window run is
    contiguous and at most 2 width + 2 taps long."""
    win = R.in_window(o, nw)
    c = R.coefficients(o, nw)
    assert np.abs(c[~win]).max(initial=0) < 5e-24
    for p in range(win.shape[0]):
        k = np.nonzero(win[p])[0]
        assert k.size <= R.band_taps(o, nw) and k[-1] - k[0] + 1 == k.size
    x = R.signal("noise", 5000, o, nw, 9)
    d, b = R.resample_dense(x, o, nw), R.resample_banded(x, o, nw)
    assert np.all(np.abs(d - b) <= R.skipped_sum(x, o, nw) + gamma(1) * 1e-9 * R.abs_sum(x, o, nw))


def test_out_len_is_torchaudio_ceil():
    rng = np.random.RandomState(4)
    for _ in range(2000):
        o, nw = (int(v) for v in rng.randint(1, 1 << 20, size=2))
        n = int(rng.randint(0, 1 << 31))
        g = np.gcd(o, nw)
        assert R.out_len(n, o, nw) == (n if o == nw else int(np.ceil((nw // g) * n / (o // g))))


# ---------------------------------------------------------------------------------------------------- dispatch
class _Fake:
    """A provider with resample (the oracle, rounded to float32) that records what reaches it."""

    def __init__(self, fail=False):
        self.calls = []
        self.fail = fail

    def resample(self, array, orig_sr, new_sr):
        a = np.asarray(array)
        assert a.dtype == np.float32 and type(orig_sr) is int and type(new_sr) is int
        self.calls.append((a.shape, orig_sr, new_sr))
        if self.fail:
            raise ValueError("rejected")
        rows = [R.resample_dense(r, orig_sr, new_sr).astype(np.float32) for r in a.reshape(-1, a.shape[-1])]
        return np.stack(rows).reshape(a.shape[:-1] + rows[0].shape)


class _NoResample:
    pass


@pytest.fixture
def registry(monkeypatch):
    from auralis_b200 import output
    monkeypatch.setattr(output, "_providers", [])
    return output


def _register(output, eng):
    output.register_gpu_provider(eng)
    return eng


def _wav16(x, sr):
    buf = io.BytesIO()
    with wave.open(buf, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(sr)
        w.writeframes((np.clip(x, -1, 1) * 32767).astype("<i2").tobytes())
    return buf.getvalue()


def test_tts_output_resample_reaches_the_provider(registry):
    from auralis_b200.output import TTSOutput
    fake = _register(registry, _Fake())
    x = R.signal("noise", 2400, 24000, 44100, 1)
    out = TTSOutput(array=x, sample_rate=24000).resample(44100)
    assert fake.calls == [((2400,), 24000, 44100)]
    assert out.sample_rate == 44100 and out.array.dtype == np.float32
    np.testing.assert_array_equal(out.array, R.resample_dense(x, 24000, 44100).astype(np.float32))
    out = TTSOutput(array=x, sample_rate=24000).resample(16000.0)            # an integral float rate
    assert fake.calls[-1] == ((2400,), 24000, 16000) and out.array.shape == (1600,)


def test_save_with_sample_rate_reaches_the_provider(registry, tmp_path):
    from auralis_b200.output import TTSOutput, _parse_riff_wav
    fake = _register(registry, _Fake())
    x = R.signal("sine", 2400, 24000, 16000, 2)
    TTSOutput(array=x, sample_rate=24000).save(tmp_path / "a.wav", sample_rate=16000)
    assert fake.calls == [((2400,), 24000, 16000)]
    a, sr = _parse_riff_wav((tmp_path / "a.wav").read_bytes())
    assert sr == 16000
    np.testing.assert_array_equal(a[:, 0], np.clip(R.resample_dense(x, 24000, 16000).astype(np.float32), -1, 1))


def test_load_audio_and_engine_resample_reach_the_provider(registry, tmp_path):
    from auralis_b200 import engine
    fake = _register(registry, _Fake())
    x = R.signal("noise", 4410, 44100, 22050, 3) * 0.5
    f = tmp_path / "r.wav"
    f.write_bytes(_wav16(x, 44100))
    got = engine.load_audio(str(f), 22050)
    assert fake.calls == [((4410,), 44100, 22050)]
    pcm = (np.clip(x, -1, 1) * 32767).astype("<i2").astype(np.float32) / 32768.0
    np.testing.assert_array_equal(got, np.clip(R.resample_dense(pcm, 44100, 22050).astype(np.float32), -1, 1))
    y = engine._resample(got, 22050, 16000)
    assert fake.calls[-1] == ((2205,), 22050, 16000)
    np.testing.assert_array_equal(y, R.resample_dense(got, 22050, 16000).astype(np.float32))
    assert engine._resample(got, 22050, 22050) is got and len(fake.calls) == 2        # equal rates: no call


def _host_paths(x, o, nw):
    """Today's host results: TTSOutput.resample's and engine._resample's torchaudio / scipy code."""
    try:
        import torch
        import torchaudio
        t = torchaudio.functional.resample(torch.from_numpy(np.ascontiguousarray(x, np.float32))[None], o, nw).squeeze().numpy()
        e = torchaudio.functional.resample(torch.from_numpy(np.ascontiguousarray(x)), o, nw).numpy()
    except ImportError:
        from math import gcd
        from scipy.signal import resample_poly
        g = gcd(nw, o)
        t = e = resample_poly(np.asarray(x, np.float32), nw // g, o // g).astype(np.float32)
    return t, e


@pytest.mark.parametrize("provider", ["raises", "no_resample", "none"])
def test_host_path_is_unchanged_without_a_usable_provider(registry, provider):
    from auralis_b200 import engine
    from auralis_b200.output import TTSOutput
    fake = {"raises": _Fake(fail=True), "no_resample": _NoResample(), "none": None}[provider]
    if fake is not None:
        _register(registry, fake)
    x = R.signal("noise", 3000, 22050, 16000, 5)
    want_t, want_e = _host_paths(x, 22050, 16000)
    out = TTSOutput(array=x, sample_rate=22050).resample(16000)
    assert out.array.tobytes() == want_t.tobytes() and out.array.shape == want_t.shape
    y = engine._resample(x, 22050, 16000)
    assert y.tobytes() == want_e.tobytes() and y.shape == want_e.shape
    if provider == "raises":
        assert len(fake.calls) == 2


def test_non_integer_rates_and_float64_stay_on_the_host(registry):
    from auralis_b200 import engine
    from auralis_b200.output import gpu_resample
    fake = _register(registry, _Fake())
    x = R.signal("noise", 300, 22050, 16000, 6)
    assert gpu_resample(x, 22050, 16000.5) is None
    assert gpu_resample(x, 22050, 0) is None and gpu_resample(x, -3, 16000) is None
    assert gpu_resample(x, True, 16000) is None
    assert gpu_resample(x.astype(np.float64), 22050, 16000) is None
    assert fake.calls == []
    engine._resample(x.astype(np.float64), 22050, 16000)
    assert fake.calls == []


@pytest.mark.parametrize("shape", [(2400,), (2, 2400), (1, 2400), (3,), (2, 3), (1, 1)])
def test_squeezed_shapes_match_torchaudio(registry, shape):
    """torchaudio's path squeezes every size-1 dimension of [1, *shape[:-1], N']; the GPU path returns the same shape."""
    from auralis_b200.output import TTSOutput
    x = np.random.RandomState(7).randn(*shape).astype(np.float32) * 0.1
    n_out = R.out_len(shape[-1], 24000, 16000)
    want = tuple(d for d in shape[:-1] + (n_out,) if d != 1)
    _register(registry, _Fake())
    got = TTSOutput(array=x, sample_rate=24000).resample(16000)
    assert got.array.shape == want and got.array.dtype == np.float32 and got.sample_rate == 16000
    try:
        import torchaudio  # noqa: F401
    except ImportError:
        return
    registry._providers[:] = []
    host = TTSOutput(array=x, sample_rate=24000).resample(16000)
    assert host.array.shape == want
