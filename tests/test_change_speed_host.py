"""CPU: `TTSOutput.change_speed`.  The repo oracle (oracle/pvoc_oracle.py) against the reference's own `change_speed` with
the restated librosa injected, the committed golden, the restatement against properties librosa documents, the dtypes
NumPy's NEP 50 promotion gives its intermediates, and the dispatch of `TTSOutput.change_speed` with a fake GPU provider."""
import gc
import os
import sys

import numpy as np
import pytest

from oracle import enhance_oracle as E
from oracle import pvoc_oracle as P
from oracle import ref_import

GOLD = os.path.join(os.path.dirname(__file__), "golden")
sys.path.insert(0, GOLD)
import make_change_speed_golden as G          # noqa: E402

live = pytest.mark.skipif(not ref_import.available(), reason="reference tree not mounted")


# ---------------------------------------------------------------------------------------------------- oracle vs reference
@live
@pytest.mark.parametrize("seed,sr,sec,silence,rate", [
    (201, 24000, 0.9, None, 0.5), (202, 24000, 1.3, (0.4, 0.7), 0.8), (203, 22050, 1.1, None, 1.1),
    (204, 22050, 0.7, (0.0, 0.2), 1.5), (205, 24000, 1.0, None, 2.0), (206, 16000, 0.5, None, 3.7),
    (207, 24000, 0.3, None, 0.3),
])
def test_oracle_matches_reference_fresh(seed, sr, sec, silence, rate):
    from oracle import ref_change_speed
    x = E.synthetic_input(sec, sr, seed, silence)
    ref = ref_change_speed.change_speed(x, rate, sample_rate=sr)
    ours = P.change_speed(x, rate)
    assert ref.array.dtype == ours.dtype == np.float32
    assert ref.array.tobytes() == ours.tobytes()
    assert ref.sample_rate == sr and ref.start_time is None and ref.token_length is None


@live
def test_reference_contract():
    """The reference's own shortcut and error, with the restated librosa injected."""
    from oracle import ref_change_speed
    x = E.synthetic_input(0.2, 24000, 9)
    assert ref_change_speed.change_speed(x, 1.0).array is x
    for bad in (0.0, -1.0):
        with pytest.raises(ValueError, match="Speed factor must be positive"):
            ref_change_speed.change_speed(x, bad)
    with pytest.raises(ValueError):                 # one output frame: np.max of an empty array
        ref_change_speed.change_speed(x[:100], 2.0)
    bad = x.copy(); bad[5] = np.nan
    with pytest.raises(ValueError):                 # librosa.stft: audio buffer is not finite
        ref_change_speed.change_speed(bad, 1.5)


@live
def test_golden_regenerates_identically():
    for name, o in G.reference_outputs().items():
        assert np.asarray(o.array).tobytes() == G.golden(name).tobytes(), name


@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_matches_golden(name):
    rate = G.CASES[name][4]
    assert P.change_speed(G.case_input(name), rate).tobytes() == G.golden(name).tobytes()


def test_golden_file_is_small_and_complete():
    z = np.load(os.path.join(GOLD, "change_speed_reference.npz"))
    assert set(G.CASES) <= set(z.files)
    assert all(z[n].dtype == np.float32 for n in G.CASES)
    assert os.path.getsize(os.path.join(GOLD, "change_speed_reference.npz")) < 256 * 1024


# ---------------------------------------------------------------------------------------------------- restatement
def test_nep50_dtypes():
    x = E.synthetic_input(0.3, 24000, 3)
    D = P._stft(x, n_fft=2048, hop_length=512)
    assert D.dtype == np.complex64
    d = {}
    P.phase_vocoder(D, rate=0.8, hop_length=512, dtypes=d)
    assert d == dict(alpha=np.float64, mag=np.float64, dphase=np.float64, inc=np.float64, phase_acc=np.float32,
                     out=np.complex64)
    assert P.normalize_inf(np.array([0.5, -2.0], np.float32)).dtype == np.float32


def test_rate_one_keeps_magnitudes_and_phases():
    """At rate 1 every output frame is input frame t: its magnitude factor is |D[t]| exactly (alpha = 0), so |S| is |D|
    up to the float32 rounding of the phasor's cos / sin and products; phases to the float32 rounding of phase_acc (the
    accumulated advance telescopes to angle(D[t]) modulo 2 pi)."""
    x = E.synthetic_input(1.0, 24000, 4)
    D = P._stft(x, n_fft=2048, hop_length=512)
    S = P.phase_vocoder(D, rate=1.0, hop_length=512)
    assert S.shape == D.shape and S.dtype == np.complex64
    mag = np.abs(D).astype(np.float64)
    np.testing.assert_allclose(np.abs(S), mag, rtol=4 * np.finfo(np.float32).eps, atol=0)
    # phase: the error is the float32 rounding of an accumulator of size |phi_advance| * t, a few ulps of it
    T = D.shape[1]
    acc_scale = (512 * np.pi * np.arange(1025) / 1024)[:, None] * np.arange(1, T + 1)[None, :] + np.pi
    err = np.abs(np.angle(S * np.conj(D)))
    strong = mag > 1e-3 * mag.max()
    assert np.all(err[strong] <= 8 * np.finfo(np.float32).eps * acc_scale[strong] + 1e-4)


@pytest.mark.parametrize("rate", [0.5, 2.0])
def test_stationary_sinusoid_keeps_its_bin(rate):
    sr, k = 24000, 85                                    # a bin-centre frequency: k * sr / 2048
    t = np.arange(3 * sr) / sr
    x = (0.5 * np.sin(2 * np.pi * k * sr / 2048 * t)).astype(np.float32)
    y = P.change_speed(x, rate)
    Y = np.abs(P._stft(y, n_fft=2048, hop_length=512))
    mid = Y[:, 4:-4]
    assert np.all(np.argmax(mid, axis=0) == k)


@pytest.mark.parametrize("n", [0, 1, 511, 512, 513, 1023, 1024, 1025, 512 * 7 - 1, 512 * 7, 512 * 7 + 1])
@pytest.mark.parametrize("rate", [0.5, 0.8, 1.1, 1.5, 2.0, 3.0])
def test_output_length(n, rate):
    x = np.random.default_rng(n).standard_normal(n).astype(np.float32) * 0.1
    T = 1 + n // 512
    frames = int(np.ceil(T / rate))
    assert P.out_frames(n, rate) == frames == len(np.arange(0, T, rate, dtype=np.float64))
    if frames == 1:
        with pytest.raises(ValueError):
            P.change_speed(x, rate)
        return
    y = P.change_speed(x, rate)
    assert y.shape == (512 * (frames - 1),) == (P.out_len(n, rate),)


def test_normalize_inf():
    y = np.array([0.25, -0.5, 0.125], np.float32)
    assert P.normalize_inf(y).tolist() == [0.5, -1.0, 0.25]
    z = np.zeros(4, np.float32)
    assert P.normalize_inf(z).tobytes() == z.tobytes()
    tiny = np.array([1e-39, -5e-39], np.float32)       # below float32 tiny: left as is
    assert P.normalize_inf(tiny).tobytes() == tiny.tobytes()
    with pytest.raises(P.ParameterError):
        P.normalize_inf(np.array([1.0, np.inf], np.float32))
    with pytest.raises(ValueError):
        P.normalize_inf(np.zeros(0, np.float32))


def test_fft_frequencies():
    f = P.fft_frequencies(sr=2 * np.pi, n_fft=2048)
    assert f.dtype == np.float64 and f.shape == (1025,)
    np.testing.assert_allclose(512 * f, np.pi * np.arange(1025) / 2, rtol=1e-15)


# ---------------------------------------------------------------------------------------------------- TTSOutput dispatch
class _FakeEngine:
    def __init__(self):
        self.calls = []

    def change_speed(self, array, speed_factor):
        self.calls.append((np.asarray(array).copy(), speed_factor))
        if not np.isfinite(speed_factor):
            raise ValueError("change_speed: the speed factor must be finite and positive")
        return np.full(7, 0.5, np.float32)


@pytest.fixture
def fake_provider():
    from auralis_b200 import output
    eng = _FakeEngine()
    output.register_gpu_provider(eng)
    yield eng
    output.unregister_gpu_provider(eng)


def test_dispatch_to_provider(fake_provider):
    from auralis_b200 import TTSOutput
    x = E.synthetic_input(0.2, 22050, 5)
    o = TTSOutput(array=x, sample_rate=22050, start_time=1.0, token_length=12)
    r = o.change_speed(1.5)
    assert isinstance(r, TTSOutput) and r.sample_rate == 22050 and r.start_time is None and r.token_length is None
    assert r.array.tolist() == [0.5] * 7
    assert len(fake_provider.calls) == 1 and fake_provider.calls[0][1] == 1.5
    assert np.array_equal(fake_provider.calls[0][0], x)
    with pytest.raises(ValueError):
        o.change_speed(float("nan"))


def test_shortcuts_before_any_native_call(fake_provider):
    from auralis_b200 import TTSOutput
    o = TTSOutput(array=np.ones(100, np.float32))
    assert o.change_speed(1.0) is o
    for bad in (0, 0.0, -1.0, -np.inf):
        with pytest.raises(ValueError, match="Speed factor must be positive"):
            o.change_speed(bad)
    assert fake_provider.calls == []


@pytest.fixture
def empty_registry(monkeypatch):
    from auralis_b200 import output
    monkeypatch.setattr(output, "_providers", [])


def test_no_provider_keeps_the_librosa_path(empty_registry):
    from auralis_b200 import TTSOutput, output
    assert output.gpu_provider() is None
    o = TTSOutput(array=np.ones(4096, np.float32))
    try:
        import librosa  # noqa: F401
    except ImportError:
        with pytest.raises(RuntimeError, match="librosa"):
            o.change_speed(1.5)


def test_registry_holds_engines_weakly(empty_registry):
    from auralis_b200 import output
    a, b = _FakeEngine(), _FakeEngine()
    output.register_gpu_provider(a)
    output.register_gpu_provider(b)
    assert output.gpu_provider() is b                      # the most recent live engine serves
    del b
    gc.collect()
    assert output.gpu_provider() is a
    output.unregister_gpu_provider(a)
    assert output.gpu_provider() is None
    output.register_gpu_provider(a)
    del a
    gc.collect()
    assert output.gpu_provider() is None


def test_engine_maps_invalid_to_value_error():
    """XTTSv2Engine.change_speed turns the native ERR_INVALID into ValueError and passes other errors on."""
    from auralis_b200 import native
    from auralis_b200.engine import XTTSv2Engine

    class _Native:
        def __init__(self, code):
            self.code = code

        def change_speed(self, wav, rate):
            if self.code:
                raise native.NativeError("change_speed failed", self.code)
            return np.asarray(wav, np.float32)[::2]

    eng = XTTSv2Engine.__new__(XTTSv2Engine)
    eng.native = _Native(0)
    assert eng.change_speed([1.0, 2.0, 3.0], 2.0).tolist() == [1.0, 3.0]
    eng.native = _Native(native.ERR_INVALID)
    with pytest.raises(ValueError):
        eng.change_speed(np.ones(8), 0.0)
    eng.native = _Native(-2)
    with pytest.raises(native.NativeError):
        eng.change_speed(np.ones(8), 1.5)
