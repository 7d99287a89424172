"""GPU: `xtts_decode_flac` (FLAC speaker references and `TTSOutput.from_file`).  Every stream must decode to exactly
the samples it was made from, and to what the sequential oracle (oracle/flac_stream.py) returns: the GPU encoder's
streams, the writer's whole feature matrix, streams with false syncs in their payloads, for every batch size.
Malformed input must be rejected with ERR_INVALID and leave the engine working.  End to end, a FLAC file must read and
condition bit for bit like the same PCM in a WAV.
"""
import ctypes as C
import gc
import hashlib
import shutil
import struct
import subprocess

import numpy as np
import pytest

from oracle import enhance_oracle as E
from oracle import flac_stream as S

pytestmark = [pytest.mark.gpu]


@pytest.fixture(scope="module")
def eng():
    from auralis_b200 import native
    from auralis_b200.config import XTTSDims
    e = native.NativeEngine(XTTSDims.small(), device=0, max_batch=1, max_speakers=1)      # needs no weights
    yield e
    e.close()


@pytest.fixture(scope="module")
def matrix():
    return S.feature_matrix()


def _pcm(x):
    return (np.clip(np.asarray(x, np.float32), -1.0, 1.0) * 32767).astype(np.int16)


def _md5(s):
    return hashlib.md5(s.astype("<i2").tobytes()).digest()


def _check(eng, data, want, sr=None, bps=None):
    got, gsr, gbps = eng.decode_flac(data)
    want = np.asarray(want, np.int64).reshape(got.shape[0], -1)
    assert got.dtype == np.int32 and np.array_equal(got, want)
    if sr is not None:
        assert (gsr, gbps) == (sr, bps)
    return got


# ---------------------------------------------------------------------------------------------------- lossless
def _encoder_inputs():
    rng = np.random.default_rng(7)
    sq = np.where((np.arange(30000) // 50) % 2 == 0, 32767, -32767).astype(np.int16)
    d = {"silence": np.zeros(30000, np.int16), "dc": np.full(30000, 1234, np.int16), "square": sq,
         "clipped_noise": _pcm(np.clip(rng.normal(0, 1.0, 30000), -1, 1)),
         "white_noise": rng.integers(-32768, 32768, 30000).astype(np.int16),
         "speech": _pcm(E.synthetic_input(5.0, 24000, 11, silence=(1.0, 1.5)))}
    for n in (0, 1, 15, 4095, 4096, 4097):
        d[f"len{n}"] = _pcm(E.synthetic_input(max(n, 1) / 24000 + 0.01, 24000, n))[:n]
    return d


@pytest.mark.parametrize("name", list(_encoder_inputs()))
def test_encoder_round_trip(eng, name):
    s = _encoder_inputs()[name]
    _check(eng, eng.encode_flac(s, 24000, _md5(s)), s[None], 24000, 16)


def test_encoder_round_trip_ten_minutes(eng):
    s = _pcm(E.synthetic_input(600.0, 24000, 5))
    _check(eng, eng.encode_flac(s, 24000, _md5(s)), s[None], 24000, 16)


MATRIX_NAMES = ["mono16_fixed_orders", "mono16_lpc", "mono16_constant_verbatim", "stereo16_assignments", "ch8_24bit",
                "stereo24_rice2_escape", "escape_zero_width", "stereo32_side", "mono4bit", "mono8bit", "mono12bit",
                "mono20bit", "wasted_bits", "variable_blocking", "header_codes", "metadata_id3", "total_zero_id3v1",
                "total_zero_md5_zero", "partition_order_15", "blocks_65535", "false_sync", "false_sync_crc"]


def test_matrix_names_cover_the_matrix(matrix):
    assert sorted(matrix) == sorted(MATRIX_NAMES)


@pytest.mark.parametrize("name", MATRIX_NAMES)
def test_feature_matrix_matches_pcm_and_oracle(eng, matrix, name):
    from auralis_b200 import native
    s = matrix[name]
    ref = S.decode(s.data, expect=s.pcm)
    got = _check(eng, s.data, s.pcm, s.sample_rate, s.bps)
    assert np.array_equal(got, ref["samples"])
    info = native.XttsFlacInfo()
    out = np.empty(got.size, np.int32)
    buf = np.frombuffer(s.data, np.uint8)
    rc = eng.lib.xtts_decode_flac(eng.h, buf.ctypes.data_as(C.POINTER(C.c_uint8)), buf.size,
                                  out.ctypes.data_as(C.POINTER(C.c_int32)), out.size, C.byref(info))
    assert rc == 0
    si = ref["streaminfo"]
    assert (info.sample_rate, info.channels, info.bits_per_sample, info.min_block, info.max_block,
            info.total_samples, bytes(info.md5)) == (si["sample_rate"], si["channels"], si["bits_per_sample"],
                                                     si["min_block"], si["max_block"], si["total_samples"], si["md5"])


def test_false_syncs_decode_exactly(eng):
    for variant in (1, 2):
        s = S.fake_sync_stream(variant)
        _check(eng, s.data, s.pcm)


# ---------------------------------------------------------------------------------------------------- batches
def test_batch_invariance(eng, matrix):
    long = _pcm(E.synthetic_input(60.0, 24000, 8, silence=(10.0, 12.0)))
    streams = [eng.encode_flac(long, 24000, _md5(long))] + [matrix[k].data for k in (
        "variable_blocking", "false_sync", "false_sync_crc", "blocks_65535", "ch8_24bit", "total_zero_id3v1")]
    ref = [eng.decode_flac(d)[0] for d in streams]
    try:
        for b in (1, 3, 4096, 8192):
            eng.set_option("flac_batch_frames", b)
            for d, r in zip(streams, ref):
                assert np.array_equal(eng.decode_flac(d)[0], r), b
    finally:
        eng.set_option("flac_batch_frames", 8192)


# ---------------------------------------------------------------------------------------------------- malformed
def _rejected(eng, data):
    from auralis_b200 import native
    with pytest.raises(native.NativeError) as ei:
        eng.decode_flac(data)
    assert ei.value.code == native.ERR_INVALID


def test_malformed_input_is_rejected(eng, matrix):
    s = matrix["stereo16_assignments"]
    a, b = s.frame_offsets[0], len(s.data)
    for cut in (0, 3, 20, a - 1, a, a + 3, a + 10, (a + b) // 2, b - 2, b - 1):
        _rejected(eng, s.data[:cut])
    rng = np.random.default_rng(3)
    for p in sorted(set(rng.integers(a, b, 40).tolist() + [a, a + 1, a + 5, b - 1])):
        bad = bytearray(s.data)
        bad[p] ^= int(rng.integers(1, 256))
        _rejected(eng, bytes(bad))
    h = s.frame_offsets[0]
    for off, fn in ((h + 3, lambda v: v | 1), (h + 3, lambda v: (v & 0xF1) | 6), (h + 2, lambda v: v | 15),
                    (h + 1, lambda v: v | 2), (4, lambda v: 0x7F)):
        bad = bytearray(s.data)
        bad[off] = fn(bad[off])
        _rejected(eng, bytes(bad))
    bad = bytearray(s.data)
    bad[8 + 18] ^= 0x55                                    # STREAMINFO's MD5
    _rejected(eng, bytes(bad))
    _rejected(eng, b"")
    _rejected(eng, b"RIFF0000WAVE")
    # the engine still works
    x = _encoder_inputs()["speech"]
    _check(eng, eng.encode_flac(x, 24000, _md5(x)), x[None])
    _check(eng, s.data, s.pcm)


def test_lpc_precision_and_shift_are_rejected(eng):
    x = S.signal(1, 256, 16, 3)
    s = S.write_stream(x, 16, 24000, [S.Frame(256, subs=[S.Sub("LPC", order=4, precision=15, shift=0)])], md5=False)
    hlen = S.parse_header(s.data, s.frame_offsets[0], len(s.data), S.parse_metadata(s.data)[0])["length"]
    bits = np.unpackbits(np.frombuffer(s.data, np.uint8)).copy()
    p = 8 * (s.frame_offsets[0] + hlen) + 8 + 4 * 16
    for at, v in ((p, [1, 1, 1, 1]), (p + 4, [1, 0, 0, 0, 0])):
        b = bits.copy()
        b[at:at + len(v)] = v
        body = np.packbits(b).tobytes()
        fix = bytearray(body)                              # a correct CRC-16, so only the field is wrong
        fix[-2:] = S.crc16(bytes(fix[s.frame_offsets[0]:-2])).to_bytes(2, "big")
        _rejected(eng, bytes(fix))
    _check(eng, s.data, x)


def test_value_error_through_the_engine(tmp_path, tts):
    from auralis_b200 import TTSOutput
    (tmp_path / "bad.flac").write_bytes(b"fLaC" + bytes(40))
    with pytest.raises(ValueError):
        TTSOutput.from_file(tmp_path / "bad.flac")


def test_time_counts_as_conditioning(eng, matrix):
    before = eng.stats().cond_ms
    eng.decode_flac(matrix["ch8_24bit"].data)
    assert eng.stats().cond_ms > before


def test_external_decoder_agrees(eng, tmp_path):
    x = _encoder_inputs()["speech"]
    (tmp_path / "a.raw").write_bytes(x.astype("<i2").tobytes())
    if shutil.which("flac"):
        subprocess.run(["flac", "-s", "-f", "--force-raw-format", "--endian=little", "--sign=signed", "--channels=1",
                        "--bps=16", "--sample-rate=24000", "-o", str(tmp_path / "a.flac"), str(tmp_path / "a.raw")],
                       check=True)
    elif shutil.which("ffmpeg"):
        subprocess.run(["ffmpeg", "-loglevel", "error", "-y", "-f", "s16le", "-ar", "24000", "-ac", "1", "-i",
                        str(tmp_path / "a.raw"), str(tmp_path / "a.flac")], check=True)
    else:
        pytest.skip("neither a flac nor an ffmpeg binary is installed")
    _check(eng, (tmp_path / "a.flac").read_bytes(), x[None])


# ---------------------------------------------------------------------------------------------------- end to end
@pytest.fixture(scope="module")
def tts(tmp_path_factory, dims_small, state_small):
    from auralis_b200 import TTS
    from auralis_b200.weights import save_model_dir
    d = tmp_path_factory.mktemp("model")
    save_model_dir(str(d), dims_small, state_small[0], state_small[1])
    t = TTS(scheduler_max_concurrency=8).from_pretrained(str(d), precision="fp32", max_concurrency=4)
    yield t
    t.loop.run_until_complete(t.shutdown())
    del t
    gc.collect()


def _wav24(pcm, sr):
    C = pcm.shape[0]
    payload = np.ascontiguousarray(pcm.T).astype("<i4").view(np.uint8).reshape(-1, 4)[:, :3].tobytes()
    fmt = struct.pack("<HHIIHH", 1, C, sr, sr * C * 3, C * 3, 24)
    body = b"WAVE" + b"fmt " + struct.pack("<I", 16) + fmt + b"data" + struct.pack("<I", len(payload)) + payload
    return b"RIFF" + struct.pack("<I", len(body)) + body


def test_save_flac_reads_back_like_wav(tts, tmp_path):
    from auralis_b200 import TTSOutput
    o = TTSOutput(array=E.synthetic_input(4.0, 24000, 31), sample_rate=24000)
    o.save(tmp_path / "a.flac")
    o.bit_depth = 16
    o.save(tmp_path / "a.wav")
    a, w = TTSOutput.from_file(tmp_path / "a.flac"), TTSOutput.from_file(tmp_path / "a.wav")
    assert a.sample_rate == w.sample_rate == 24000
    assert a.array.tobytes() == w.array.tobytes()


def test_flac_speaker_conditions_like_wav(tts, tmp_path):
    from auralis_b200.requests import AudioPreprocessingConfig
    eng = tts.tts_engine
    x = S.signal(2, 48000 * 3, 24, 41, level=0.3)
    s = S.write_stream(x, 24, 48000, [S.Frame(4608, S.MID_SIDE, [S.Sub("LPC", order=12, shift=13)] * 2)
                                      for _ in range(31)] + [S.Frame(48000 * 3 - 31 * 4608, S.LEFT_SIDE)])
    (tmp_path / "r.flac").write_bytes(s.data)
    (tmp_path / "r.wav").write_bytes(_wav24(x, 48000))
    run = tts.loop.run_until_complete
    for enhance in (None, AudioPreprocessingConfig()):
        want = run(eng.get_audio_conditioning(str(tmp_path / "r.wav"), 60, 30, 4, enhance=enhance))
        for src in (str(tmp_path / "r.flac"), s.data):
            got = run(eng.get_audio_conditioning(src, 60, 30, 4, enhance=enhance))
            assert np.asarray(got[0]).tobytes() == np.asarray(want[0]).tobytes()
            assert np.asarray(got[1]).tobytes() == np.asarray(want[1]).tobytes()


def test_generate_speech_with_a_flac_speaker(tts, tmp_path):
    from auralis_b200 import TTSOutput, TTSRequest
    spk = tmp_path / "spk.flac"
    TTSOutput(array=E.synthetic_input(3.0, 22050, 5), sample_rate=22050).save(spk)
    assert spk.read_bytes()[:4] == b"fLaC"
    out = tts.generate_speech(TTSRequest(text="A short sentence from a FLAC voice.", speaker_files=[str(spk)],
                                         language="en", temperature=0.0))
    assert out.array.size > 0 and np.isfinite(out.array).all()
