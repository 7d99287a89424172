"""CPU: the FLAC decoding oracle (oracle/flac_stream.py) and the FLAC input dispatch of `TTSOutput.from_file` and
`engine.load_audio`.  The writer's streams cover every feature `xtts_decode_flac` accepts and must decode back to
their PCM exactly; streams `flac_oracle.decode` can read must decode to the same samples there; truncations and
single-byte flips must be rejected; and FLAC input must reach a live engine's `decode_flac` (and WAV never must)."""
import io
import struct

import numpy as np
import pytest

from oracle import flac_oracle as F
from oracle import flac_stream as S

MATRIX = S.feature_matrix()


@pytest.mark.parametrize("name", list(MATRIX))
def test_writer_streams_decode_exactly(name):
    s = MATRIX[name]
    d = S.decode(s.data, expect=s.pcm)
    assert np.array_equal(d["samples"], s.pcm)
    si = d["streaminfo"]
    assert (si["channels"], si["bits_per_sample"], si["sample_rate"]) == (s.pcm.shape[0], s.bps, s.sample_rate)
    assert si["total_samples"] == s.pcm.shape[1]
    assert [f["offset"] for f in d["frames"]] == s.frame_offsets


def test_fake_syncs_are_in_the_payload():
    for variant in (1, 2):
        s = S.fake_sync_stream(variant)
        d = S.decode(s.data)
        assert np.array_equal(d["samples"], s.pcm)
        for i, off in enumerate(s.frame_offsets[1:], 1):    # each frame's header also sits inside the frame before it
            h = s.data[off:off + 6]
            inner = s.data.find(h, s.frame_offsets[i - 1] + 6, off)
            assert s.frame_offsets[i - 1] < inner < off
            if variant == 2:                                # and the CRC-16 of the prefix before it checks
                assert F.crc16(s.data[s.frame_offsets[i - 1]:inner - 2]) == int.from_bytes(s.data[inner - 2:inner], "big")


@pytest.mark.parametrize("n", [1, 15, 4095, 4096, 4097, 3 * 4096 + 5])
def test_agrees_with_the_mono_16_bit_oracle(n):
    x = S.signal(1, n, 16, n)
    sizes = [4096] * (n // 4096) + ([n % 4096] if n % 4096 else [])
    kinds = [S.Sub("FIXED", order=2), S.Sub("LPC", order=12, shift=11), S.Sub("VERBATIM"), S.Sub("FIXED", order=0, porder=2)]
    fr = [S.Frame(b, subs=[kinds[i % 4] if b > 12 else S.Sub("VERBATIM")]) for i, b in enumerate(sizes)]
    s = S.write_stream(x, 16, 24000, fr, max_block=4096)
    new, old = S.decode(s.data), F.decode(s.data)
    assert np.array_equal(new["samples"][0], old["samples"]) and np.array_equal(old["samples"], x[0])
    for k in ("min_block", "max_block", "sample_rate", "channels", "bits_per_sample", "total_samples", "md5"):
        assert new["streaminfo"][k] == old["streaminfo"][k], k


@pytest.mark.parametrize("name", ["stereo16_assignments", "variable_blocking", "header_codes", "stereo24_rice2_escape"])
def test_truncations_are_rejected(name):
    s = MATRIX[name]
    a, b = s.frame_offsets[0], len(s.data)
    for cut in sorted(set(np.linspace(0, b - 1, 60).astype(int).tolist() + [a, a + 1, b - 2, b - 1])):
        with pytest.raises(F.FlacError):
            S.decode(s.data[:cut])


@pytest.mark.parametrize("name", ["mono16_lpc", "stereo16_assignments", "variable_blocking", "header_codes",
                                  "wasted_bits", "total_zero_md5_zero"])
def test_single_byte_flips_are_rejected(name):
    s = MATRIX[name]
    a, b = s.frame_offsets[0], len(s.data)
    rng = np.random.default_rng(len(name))
    for p in sorted(set(rng.integers(a, b, 150).tolist() + [a, a + 1, a + 4, b - 2, b - 1])):
        bad = bytearray(s.data)
        bad[p] ^= int(rng.integers(1, 256))
        with pytest.raises(F.FlacError):
            S.decode(bytes(bad), check_md5=False)


def test_metadata_errors():
    s = MATRIX["metadata_id3"].data
    si = S.parse_metadata(s)[0]
    assert si["total_samples"] == 2 * 4096 + 3
    plain = MATRIX["mono16_lpc"].data
    for bad in (b"fLaX" + plain[4:], plain[:4] + bytes([0x7F]) + plain[5:],       # no marker; type 127 first
                plain[:4] + bytes([0x01]) + plain[5:],                              # first block not STREAMINFO
                plain[:20]):                                                        # truncated metadata
        with pytest.raises(F.FlacError):
            S.decode(bad)
    md5_bad = bytearray(plain)
    md5_bad[8 + 18] ^= 1
    with pytest.raises(F.FlacError, match="MD5"):
        S.decode(bytes(md5_bad))


def test_reserved_codes_are_rejected():
    s = MATRIX["mono16_lpc"]
    hdr_at = s.frame_offsets[0]
    for patch in ((hdr_at + 3, lambda b: b | 1),                 # reserved bit after the sample size
                  (hdr_at + 3, lambda b: (b & 0xF1) | (3 << 1)),  # sample-size code 3
                  (hdr_at + 2, lambda b: (b & 0xF0) | 15),        # sample-rate code 15
                  (hdr_at + 1, lambda b: b | 2)):                 # reserved bit in the sync word
        bad = bytearray(s.data)
        bad[patch[0]] = patch[1](bad[patch[0]])
        with pytest.raises(F.FlacError):
            S.decode(bytes(bad))


def test_writer_refuses_lpc_precision_and_shift_out_of_range():
    x = S.signal(1, 256, 16, 3)
    s = S.write_stream(x, 16, 24000, [S.Frame(256, subs=[S.Sub("LPC", order=4, precision=15, shift=0)])])
    assert np.array_equal(S.decode(s.data)["samples"], x)
    # precision code 1111 and a negative shift, written by hand into the subframe after the header and warm-up
    hlen = S.parse_header(s.data, s.frame_offsets[0], len(s.data), S.parse_metadata(s.data)[0])["length"]
    bits = np.unpackbits(np.frombuffer(s.data, np.uint8)).copy()
    p = 8 * (s.frame_offsets[0] + hlen) + 8 + 4 * 16
    for field in ((p, [1, 1, 1, 1]), (p + 4, [1, 0, 0, 0, 0])):
        b = bits.copy()
        b[field[0]:field[0] + len(field[1])] = field[1]
        with pytest.raises(F.FlacError, match="precision|shift"):
            S.decode(np.packbits(b).tobytes())


# ---------------------------------------------------------------------------------------------------- dispatch
class _FakeFlac:
    """A provider with decode_flac (the oracle) that records what reaches it."""

    def __init__(self):
        self.calls = []

    def decode_flac(self, blob):
        self.calls.append(len(blob))
        d = S.decode(blob)
        return d["samples"].astype(np.int32), d["streaminfo"]["sample_rate"], d["streaminfo"]["bits_per_sample"]


@pytest.fixture
def fake(monkeypatch):
    from auralis_b200 import output
    monkeypatch.setattr(output, "_providers", [])
    eng = _FakeFlac()
    output.register_gpu_provider(eng)
    yield eng


def _wav(pcm, sr, bits):
    """Integer-PCM WAV of pcm [C, N] at 16 or 24 bits."""
    C, N = pcm.shape
    inter = np.ascontiguousarray(pcm.T).astype("<i4")
    payload = inter.astype("<i2").tobytes() if bits == 16 else inter.view(np.uint8).reshape(-1, 4)[:, :3].tobytes()
    fmt = struct.pack("<HHIIHH", 1, C, sr, sr * C * bits // 8, C * bits // 8, bits)
    body = b"WAVE" + b"fmt " + struct.pack("<I", 16) + fmt + b"data" + struct.pack("<I", len(payload)) + payload
    return b"RIFF" + struct.pack("<I", len(body)) + body


@pytest.mark.parametrize("C,bits", [(1, 16), (2, 24), (3, 12)])
def test_from_file_flac_goes_to_the_provider(fake, tmp_path, C, bits):
    from auralis_b200 import TTSOutput
    x = S.signal(C, 5000, bits, C)
    s = S.write_stream(x, bits, 48000, [S.Frame(4096, subs=[S.Sub("FIXED")] * C), S.Frame(904, subs=[S.Sub("FIXED")] * C)])
    (tmp_path / "a.flac").write_bytes(s.data)
    o = TTSOutput.from_file(tmp_path / "a.flac")
    want = x.astype(np.float32) / np.float32(2 ** (bits - 1))
    assert o.sample_rate == 48000 and o.array.dtype == np.float32
    assert np.array_equal(o.array, want[0] if C == 1 else want)
    assert fake.calls == [len(s.data)]
    if bits in (16, 24):                                   # the same PCM in a WAV reads back bit for bit the same
        (tmp_path / "a.wav").write_bytes(_wav(x, 48000, bits))
        assert np.array_equal(TTSOutput.from_file(tmp_path / "a.wav").array, o.array)
        assert fake.calls == [len(s.data)]                # WAV never reaches the provider


def test_id3v2_tagged_flac_is_detected(fake, tmp_path):
    from auralis_b200 import TTSOutput
    s = MATRIX["metadata_id3"]
    (tmp_path / "a.flac").write_bytes(s.data)
    assert np.array_equal(TTSOutput.from_file(tmp_path / "a.flac").array, s.pcm[0].astype(np.float32) / 32768)


def test_load_audio_flac_equals_wav(fake, tmp_path, monkeypatch):
    from auralis_b200 import engine
    x = S.signal(2, 9000, 24, 5)
    s = S.write_stream(x, 24, 48000, [S.Frame(4096, S.MID_SIDE), S.Frame(4096, S.LEFT_SIDE), S.Frame(808)])
    w = _wav(x, 48000, 24)
    (tmp_path / "a.flac").write_bytes(s.data)
    (tmp_path / "a.wav").write_bytes(w)
    monkeypatch.setattr(engine, "_resample", lambda a, sr, new: a[::2].copy())     # any deterministic stand-in
    want = engine.load_audio(w, 24000)
    for src in (s.data, str(tmp_path / "a.flac")):
        got = engine.load_audio(src, 24000)
        assert got.dtype == np.float32 and np.array_equal(got, want)
    assert len(fake.calls) == 2
    engine.load_audio(str(tmp_path / "a.wav"), 24000)
    assert len(fake.calls) == 2


def test_no_provider_keeps_the_torchaudio_path(monkeypatch, tmp_path):
    from auralis_b200 import TTSOutput, engine, output
    monkeypatch.setattr(output, "_providers", [])
    s = MATRIX["mono16_lpc"]
    (tmp_path / "a.flac").write_bytes(s.data)
    called = []

    class _TA:
        @staticmethod
        def load(src):
            called.append(src)
            import torch
            return torch.zeros(1, 4), 16000

    monkeypatch.setitem(__import__("sys").modules, "torchaudio", _TA)
    o = TTSOutput.from_file(tmp_path / "a.flac")
    assert o.sample_rate == 16000 and called == [str(tmp_path / "a.flac")]
    output.register_gpu_provider(_NoDecode())             # a provider without decode_flac: still torchaudio
    engine.load_audio(s.data, 16000)
    assert len(called) == 2 and isinstance(called[1], io.BytesIO)


class _NoDecode:
    def change_speed(self, a, f):
        return a


def test_engine_maps_invalid_to_value_error():
    from auralis_b200 import native
    from auralis_b200.engine import XTTSv2Engine

    class _Native:
        def __init__(self, code):
            self.code = code

        def decode_flac(self, data):
            if self.code:
                raise native.NativeError("decode_flac failed", self.code)
            return np.zeros((1, 0), np.int32), 24000, 16

    eng = XTTSv2Engine.__new__(XTTSv2Engine)
    eng.native = _Native(0)
    assert eng.decode_flac(b"x")[1] == 24000
    eng.native = _Native(native.ERR_INVALID)
    with pytest.raises(ValueError):
        eng.decode_flac(b"x")
    eng.native = _Native(-2)
    with pytest.raises(native.NativeError):
        eng.decode_flac(b"x")


def test_md5_helper_matches_the_oracle():
    from auralis_b200 import native
    for C, b in ((1, 8), (2, 16), (3, 24), (2, 32), (1, 4), (1, 20)):
        x = S.signal(C, 777, b, C + b)
        assert native.flac_md5(x.astype(np.int32), b) == S.md5_of(x, b)
