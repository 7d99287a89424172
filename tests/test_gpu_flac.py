"""GPU: `xtts_encode_flac` (TTSOutput.to_bytes("flac")).  Every stream is decoded by the independent oracle decoder
(oracle/flac_oracle.py), which checks every CRC and the MD5, and must give back exactly the input samples.  Compression
is checked frame by frame against the exact FIXED-only yardstick, and the stream against determinism and the batch size.
"""
import gc
import hashlib
import shutil
import subprocess

import numpy as np
import pytest

from oracle import enhance_oracle as E
from oracle import flac_oracle as F

pytestmark = [pytest.mark.gpu]


@pytest.fixture(scope="module")
def eng():
    from auralis_b200 import native
    from auralis_b200.config import XTTSDims
    e = native.NativeEngine(XTTSDims.small(), device=0, max_batch=1, max_speakers=1)      # needs no weights
    yield e
    e.close()


def _pcm(x):
    return (np.clip(np.asarray(x, np.float32), -1.0, 1.0) * 32767).astype(np.int16)


def _md5(s):
    return hashlib.md5(s.astype("<i2").tobytes()).digest()


def _encode_check(eng, s, sr=24000):
    """Encode, decode with the oracle, check samples, STREAMINFO and the size bound -> (stream, decoded)."""
    data = eng.encode_flac(s, sr, _md5(s))
    assert len(data) <= 42 + -(-s.size // 4096) * 8211
    d = F.decode(data, expect=s)
    assert np.array_equal(d["samples"], s) and d["md5_checked"]
    si = d["streaminfo"]
    assert (si["total_samples"], si["sample_rate"], si["bits_per_sample"], si["channels"]) == (s.size, sr, 16, 1)
    assert si["min_block"] == si["max_block"] == 4096
    sizes = [f["bytes"] for f in d["frames"]]
    assert (si["min_frame"], si["max_frame"]) == ((min(sizes), max(sizes)) if sizes else (0, 0))
    assert len(d["frames"]) == -(-s.size // 4096)
    return data, d


def _inputs():
    rng = np.random.default_rng(7)
    sq = np.where((np.arange(30000) // 50) % 2 == 0, 32767, -32767).astype(np.int16)
    return {
        "silence": np.zeros(30000, np.int16),
        "dc": np.full(30000, 1234, np.int16),
        "square": sq,
        "clipped_noise": _pcm(np.clip(rng.normal(0, 1.0, 30000), -1, 1)),
        "white_noise": rng.integers(-32768, 32768, 30000).astype(np.int16),
        "speech": _pcm(E.synthetic_input(5.0, 24000, 11, silence=(1.0, 1.5))),
    }


# ---------------------------------------------------------------------------------------------------- lossless
@pytest.mark.parametrize("sr", [24000, 22050, 44100, 16000, 12345])
def test_speech_like_at_rates(eng, sr):
    _encode_check(eng, _pcm(E.synthetic_input(3.0, sr, 3)), sr)


@pytest.mark.parametrize("name", list(_inputs()))
def test_signals(eng, name):
    _encode_check(eng, _inputs()[name])


@pytest.mark.parametrize("n", [0, 1, 15, 4095, 4096, 4097, 3 * 4096 + 5])
def test_lengths(eng, n):
    s = _pcm(E.synthetic_input(max(n, 1) / 24000 + 0.01, 24000, n))[:n]
    data, d = _encode_check(eng, s)
    if n == 0:
        assert len(data) == 42 and d["frames"] == []
    if n == 1:
        assert d["frames"][0]["type"] == "CONSTANT"


def test_ten_minutes(eng):
    s = _pcm(E.synthetic_input(600.0, 24000, 5))
    data, d = _encode_check(eng, s)
    print(f"10 min: {len(data)} bytes, {len(data) / (2 * s.size):.3f} of 16-bit PCM, "
          f"{sum(f['type'] == 'LPC' for f in d['frames'])} / {len(d['frames'])} LPC frames")


def test_md5_none_writes_zeros(eng):
    s = _inputs()["speech"]
    d = F.decode(eng.encode_flac(s, 24000, None), expect=s)
    assert d["streaminfo"]["md5"] == bytes(16) and not d["md5_checked"]


# ---------------------------------------------------------------------------------------------------- compression
def _frames_within_fixed_only(s, d):
    fixed_total = 0
    for f in d["frames"]:
        block = s[4096 * f["number"]: 4096 * f["number"] + f["blocksize"]]
        fo = F.fixed_only_bits(block)
        fixed_total += f["header_bytes"] + -(-fo // 8) + 2
        assert f["bytes"] <= f["header_bytes"] + -(-fo // 8) + 2, f["number"]
    return fixed_total


@pytest.mark.parametrize("name", list(_inputs()))
def test_no_frame_above_fixed_only(eng, name):
    s = _inputs()[name]
    _, d = _encode_check(eng, s)
    _frames_within_fixed_only(s, d)
    if name == "silence":
        assert all(f["type"] == "CONSTANT" for f in d["frames"])
    if name == "white_noise":
        assert all(f["bytes"] <= f["header_bytes"] + 1 + 2 * f["blocksize"] + 2 for f in d["frames"])


def test_speech_like_beats_fixed_only(eng):
    s = _pcm(E.synthetic_input(20.0, 24000, 21, silence=(5.0, 6.0)))
    data, d = _encode_check(eng, s)
    fixed_total = 42 + _frames_within_fixed_only(s, d)
    n_lpc = sum(f["type"] == "LPC" for f in d["frames"])
    print(f"speech-like 20 s: {len(data)} bytes vs fixed-only {fixed_total}; LPC in {n_lpc} / {len(d['frames'])} "
          f"frames; {len(data) / (2 * s.size):.3f} of 16-bit PCM")
    assert len(data) < fixed_total
    assert n_lpc >= 1


# ---------------------------------------------------------------------------------------------------- robustness
def test_deterministic_and_batch_invariant(eng):
    s = _pcm(E.synthetic_input(60.0, 24000, 8, silence=(10.0, 12.0)))
    ref = eng.encode_flac(s, 24000, _md5(s))
    assert eng.encode_flac(s, 24000, _md5(s)) == ref
    try:
        for b in (1, 3, 4096, 8192):
            eng.set_option("flac_batch_frames", b)
            assert eng.encode_flac(s, 24000, _md5(s)) == ref, b
    finally:
        eng.set_option("flac_batch_frames", 8192)


def test_invalid(eng):
    from auralis_b200 import native
    s = np.zeros(100, np.int16)
    for sr in (0, -1, 1 << 20):
        with pytest.raises(native.NativeError) as ei:
            eng.encode_flac(s, sr)
        assert ei.value.code == native.ERR_INVALID
    for b in (0, (1 << 20) + 1):
        with pytest.raises(native.NativeError):
            eng.set_option("flac_batch_frames", b)
    _encode_check(eng, np.arange(-5000, 5000, dtype=np.int16), 1048575)


def test_time_counts_as_conditioning(eng):
    before = eng.stats().cond_ms
    eng.encode_flac(_inputs()["speech"], 24000)
    assert eng.stats().cond_ms > before


def test_external_decoder_agrees(eng, tmp_path):
    s = _inputs()["speech"]
    (tmp_path / "a.flac").write_bytes(eng.encode_flac(s, 24000, _md5(s)))
    if shutil.which("flac"):
        subprocess.run(["flac", "-d", "-s", "-f", "--force-raw-format", "--endian=little", "--sign=signed", "-o",
                        str(tmp_path / "a.raw"), str(tmp_path / "a.flac")], check=True)
    elif shutil.which("ffmpeg"):
        subprocess.run(["ffmpeg", "-loglevel", "error", "-y", "-i", str(tmp_path / "a.flac"), "-f", "s16le",
                        str(tmp_path / "a.raw")], check=True)
    else:
        pytest.skip("neither a flac nor an ffmpeg binary is installed")
    assert np.array_equal(np.fromfile(tmp_path / "a.raw", "<i2"), s)


# ---------------------------------------------------------------------------------------------------- end to end
def test_tts_output_flac_end_to_end(tmp_path, dims_small, state_small):
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
        out = tts.generate_speech(TTSRequest(text="A short sentence to compress.", speaker_files=[spk], language="en",
                                             temperature=0.0))
        assert out.array.size > 0
        data = out.to_bytes("flac")
        pcm = np.frombuffer(out.to_bytes("pcm", 2), np.int16)
        dec = F.decode(data, expect=pcm)
        assert np.array_equal(dec["samples"], pcm) and dec["md5_checked"]
        assert dec["streaminfo"]["sample_rate"] == out.sample_rate
        out.save(tmp_path / "a.flac")
        assert (tmp_path / "a.flac").read_bytes() == data
        print(f"generated speech: {len(data)} bytes, {len(data) / (2 * pcm.size):.3f} of 16-bit PCM")
    finally:
        tts.loop.run_until_complete(tts.shutdown())
    assert output.gpu_provider() is not engine
    if output.gpu_provider() is None:                   # the torchaudio path again
        try:
            import torchcodec  # noqa: F401
        except ImportError:
            with pytest.raises(RuntimeError, match="codec backend"):
                out.to_bytes("flac")
    del tts, engine
    gc.collect()
