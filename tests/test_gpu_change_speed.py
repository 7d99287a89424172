"""GPU: `xtts_change_speed` (TTSOutput.change_speed) against the goldens the reference's own `change_speed` produced and
against the repo oracle (oracle/pvoc_oracle.py): exact lengths, peaks, zeros, block invariance, determinism, the
reference's error cases, and the end-to-end path through TTS.generate_speech.

Tolerance.  This is not a plain STFT error bound.  The phase vocoder's accumulator is float32 and is rounded once per
output frame, to a value near pi * 512 * t / 2 * (k / 512) — for a high bin late in a long signal that is millions of
radians, where one float32 ulp is ~0.1 rad or more.  Any difference in the inputs of one step (the fp32 DFT-by-GEMM
spectrum instead of numpy's fp64 FFT, one ulp of an angle) can flip one of those roundings, and the flip stays in the
accumulator for the rest of the signal.  Two equally correct evaluations therefore drift apart with the length of the
signal.  The test measures that drift on the same input with two re-evaluations of the oracle:
  * `angle` as float64 arctan2 rounded to float32 instead of numpy's float32 arctan2 (one-ulp angle differences);
  * both transforms as fp32 DFT-by-matrix products (`change_speed_fp32_dft`), the arithmetic class the GPU uses.
The GPU's max-abs and relative-L2 distances from the oracle must be at most twice the larger of the two variants'
distances, plus STFT_ERR (the enhancer tests' fp32 STFT round-trip error, 2e-5 of full scale) scaled by 1 / peak, since
the output is peak-normalised.
Magnitudes depend much less on those roundings, but not on nothing: the output's STFT re-analyses overlapping frames whose
relative phases have drifted, so a long signal's magnitudes move too (measured on an H100: the GPU's log-spectral distance
from the oracle tracks the fp32-DFT variant's).  The log-spectral distance (mean / 99th percentile of |20 log10| over
every bin within 60 dB of the oracle's peak) must be at most twice the fp32-DFT variant's plus LSD_FLOOR_DB, and, for
inputs up to 60 s, within the fixed LSD_MEAN_DB / LSD_P99_DB."""
import gc
import math
import os
import sys

import numpy as np
import pytest

from oracle import enhance_oracle as E
from oracle import pvoc_oracle as P

pytestmark = [pytest.mark.gpu]
GOLD = os.path.join(os.path.dirname(__file__), "golden")
sys.path.insert(0, GOLD)
import make_change_speed_golden as G          # noqa: E402

STFT_ERR = 2e-5
LSD_MEAN_DB = 0.05          # inputs up to 60 s
LSD_P99_DB = 1.0
LSD_FLOOR_DB = (0.01, 0.1)  # (mean, p99) added to twice the fp32-DFT variant's distance
RATES = [0.5, 0.8, 1.1, 1.5, 2.0]


@pytest.fixture(scope="module")
def eng():
    from auralis_b200 import native
    from auralis_b200.config import XTTSDims
    e = native.NativeEngine(XTTSDims.small(), device=0, max_batch=1, max_speakers=1)      # needs no weights
    yield e
    e.close()


def _lsd(a, b):
    """(mean, 99th percentile) of |20 log10(|STFT a| / |STFT b|)| over the bins of b within 60 dB of its peak."""
    A = np.abs(P._stft(a, n_fft=2048, hop_length=512)).astype(np.float64)
    B = np.abs(P._stft(b, n_fft=2048, hop_length=512)).astype(np.float64)
    m = B > 1e-3 * B.max()
    d = np.abs(20 * np.log10(np.maximum(A[m], 1e-30) / B[m]))
    return float(d.mean()), float(np.percentile(d, 99))


def _dist(a, b):
    return float(np.abs(a - b).max()), float(np.linalg.norm(a - b) / np.linalg.norm(b))


def _check_parity(out, x, rate, want=None):
    """out: the GPU's result on x; want: the oracle's (computed when not given)."""
    want = P.change_speed(x, rate) if want is None else want
    assert out.shape == want.shape
    var_a = _dist(P.change_speed(x, rate, angle=P.angle_f64), want)
    f32, peak = P.change_speed_fp32_dft(x, rate)
    var_f = _dist(f32, want)
    floor = STFT_ERR / peak
    tol_max = 2 * max(var_a[0], var_f[0]) + floor
    tol_rel = 2 * max(var_a[1], var_f[1]) + floor
    got = _dist(out, want)
    lsd, lsd_f = _lsd(out, want), _lsd(f32, want)
    print(f"n={x.size} rate={rate}: max {got[0]:.3g} (tol {tol_max:.3g}), rel {got[1]:.3g} (tol {tol_rel:.3g}); "
          f"variants angle {var_a[0]:.3g}/{var_a[1]:.3g} fp32-dft {var_f[0]:.3g}/{var_f[1]:.3g}; "
          f"lsd {lsd[0]:.3g}/{lsd[1]:.3g} dB, fp32-dft variant {lsd_f[0]:.3g}/{lsd_f[1]:.3g} dB")
    assert got[0] <= tol_max
    assert got[1] <= tol_rel
    assert lsd[0] <= 2 * lsd_f[0] + LSD_FLOOR_DB[0] and lsd[1] <= 2 * lsd_f[1] + LSD_FLOOR_DB[1]
    if x.size <= 60 * 24000:
        assert lsd[0] <= LSD_MEAN_DB and lsd[1] <= LSD_P99_DB


# ---------------------------------------------------------------------------------------------------- exact properties
@pytest.mark.parametrize("n", [511, 512, 513, 1023, 1024, 1025, 24000, 24000 * 3 + 77])
@pytest.mark.parametrize("rate", RATES + [0.3, 3.0])
def test_length_and_peak(eng, n, rate):
    x = E.synthetic_input(n / 24000, 24000, n)[:n]
    x = np.pad(x, (0, n - x.size))
    if P.out_frames(n, rate) == 1:
        return                                               # covered by test_invalid
    out = eng.change_speed(x, rate)
    assert out.dtype == np.float32 and out.shape == (P.out_len(n, rate),)
    assert np.abs(out).max() == np.float32(1.0)


def test_zero_input_stays_zero(eng):
    out = eng.change_speed(np.zeros(24000, np.float32), 1.5)
    assert out.shape == (P.out_len(24000, 1.5),) and not out.any()


def test_deterministic(eng):
    x = E.synthetic_input(20.0, 24000, 8, silence=(5.0, 6.0))
    assert eng.change_speed(x, 0.8).tobytes() == eng.change_speed(x, 0.8).tobytes()


@pytest.mark.parametrize("rate", [0.5, 1.5])
def test_bit_identical_for_every_block_size(eng, rate):
    x = E.synthetic_input(600.0, 24000, 12)
    frames = P.out_frames(x.size, rate)
    ref = eng.change_speed(x, rate)                          # default block
    try:
        for b in (1, 7, 1000, frames):                       # frames: the whole signal in one block
            eng.set_option("pvoc_block_frames", b)
            assert eng.change_speed(x, rate).tobytes() == ref.tobytes(), b
    finally:
        eng.set_option("pvoc_block_frames", 4096)


def test_invalid(eng):
    from auralis_b200 import native
    x = E.synthetic_input(1.0, 24000, 2)
    T = 1 + x.size // 512
    bad_x = x.copy(); bad_x[1000] = np.nan
    cases = [(x, 0.0), (x, -1.0), (x, math.nan), (x, math.inf), (x, float(T)), (x, T + 0.5), (bad_x, 1.5)]
    for a, rate in cases:
        with pytest.raises(native.NativeError) as ei:
            eng.change_speed(a, rate)
        assert ei.value.code == native.ERR_INVALID, rate
    with pytest.raises(native.NativeError):
        eng.set_option("pvoc_block_frames", 0)


def test_time_counts_as_conditioning(eng):
    before = eng.stats().cond_ms
    eng.change_speed(E.synthetic_input(5.0, 24000, 3), 1.5)
    assert eng.stats().cond_ms > before


# ---------------------------------------------------------------------------------------------------- parity
@pytest.mark.parametrize("name", list(G.CASES))
def test_matches_reference_goldens(eng, name):
    x, rate = G.case_input(name), G.CASES[name][4]
    _check_parity(eng.change_speed(x, rate), x, rate, want=G.golden(name))


@pytest.mark.parametrize("seconds", [1.0, 60.0, 600.0])
@pytest.mark.parametrize("rate", RATES)
def test_matches_oracle(eng, seconds, rate):
    x = E.synthetic_input(seconds, 24000, 42)
    _check_parity(eng.change_speed(x, rate), x, rate)


# ---------------------------------------------------------------------------------------------------- end to end
def test_tts_output_change_speed_end_to_end(tmp_path, dims_small, state_small):
    from auralis_b200 import TTS, TTSOutput, TTSRequest, output
    from auralis_b200.engine import XTTSv2Engine
    from auralis_b200.weights import save_model_dir
    d = tmp_path / "model"
    d.mkdir()
    save_model_dir(str(d), dims_small, state_small[0], state_small[1])
    engine = XTTSv2Engine.from_pretrained(str(d), precision="fp32", max_concurrency=4)
    tts = TTS(scheduler_max_concurrency=4).from_engine(engine)
    spk = str(tmp_path / "spk.wav")
    TTSOutput(array=E.synthetic_input(3.0, 22050, 5), sample_rate=22050).save(spk)
    try:
        out = tts.generate_speech(TTSRequest(text="A short sentence to stretch.", speaker_files=[spk], language="en",
                                             temperature=0.0))
        assert out.array.size > 0
        fast = out.change_speed(1.5)
        assert isinstance(fast, TTSOutput) and fast.sample_rate == out.sample_rate
        assert fast.array.tobytes() == engine.change_speed(out.array, 1.5).tobytes()
        assert fast.array.shape == (P.out_len(out.array.size, 1.5),)
        assert out.change_speed(1.0) is out
        for bad in (math.nan, math.inf, float(1 + out.array.size // 512)):
            with pytest.raises(ValueError):
                out.change_speed(bad)
    finally:
        tts.loop.run_until_complete(tts.shutdown())
    # after shutdown the registry no longer serves the engine: with no other engine alive, the librosa path again
    assert output.gpu_provider() is not engine
    try:
        import librosa  # noqa: F401
    except ImportError:
        if output.gpu_provider() is None:
            with pytest.raises(RuntimeError, match="librosa"):
                out.change_speed(1.5)
    del tts, engine
    gc.collect()
