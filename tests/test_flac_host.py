"""CPU: the FLAC test oracle (oracle/flac_oracle.py) on streams assembled bit by bit here from the format (RFC 9639), and
the dispatch of `TTSOutput.to_bytes("flac")` / `save("*.flac")` with a fake GPU provider."""
import hashlib

import numpy as np
import pytest

from oracle import flac_oracle as F


# ---------------------------------------------------------------------------------------------------- a bit writer
class _W:
    def __init__(self):
        self.bits = []

    def put(self, v: int, n: int):
        v &= (1 << n) - 1
        self.bits += [(v >> (n - 1 - i)) & 1 for i in range(n)]

    def rice(self, r: int, k: int):
        u = 2 * r if r >= 0 else -2 * r - 1
        self.bits += [0] * (u >> k) + [1]
        if k:
            self.put(u, k)

    def pad(self):
        self.bits += [0] * (-len(self.bits) % 8)

    def bytes(self) -> bytes:
        assert len(self.bits) % 8 == 0
        return np.packbits(np.array(self.bits, np.uint8)).tobytes()


def _utf8(v: int) -> bytes:
    if v < 0x80:
        return bytes([v])
    n = 2
    while v >> (5 * n + 1):
        n += 1
    out = [((0xFF00 >> n) & 0xFF) | (v >> (6 * (n - 1)))]
    out += [0x80 | ((v >> (6 * c)) & 0x3F) for c in range(n - 2, -1, -1)]
    return bytes(out)


def _frame(number: int, nb: int, body) -> bytes:
    """One frame at 24 kHz: header (block size 4096 or a 16-bit size - 1), `body(w)` writes the subframe."""
    code = 12 if nb == 4096 else 7
    h = bytes([0xFF, 0xF8, code << 4 | 7, 0x08]) + _utf8(number)
    if code == 7:
        h += (nb - 1).to_bytes(2, "big")
    h += bytes([F.crc8(h)])
    w = _W()
    w.bits = [int(b) for b in np.unpackbits(np.frombuffer(h, np.uint8))]
    body(w)
    w.pad()
    b = w.bytes()
    return b + F.crc16(b).to_bytes(2, "big")


def _residual(w: _W, r, k: int):
    w.put(0, 2)          # method 00
    w.put(0, 4)          # partition order 0
    w.put(k, 4)
    for v in r:
        w.rice(int(v), k)


def _stream(frames, n: int, md5: bytes) -> bytes:
    sizes = [len(f) for f in frames]
    si = (4096).to_bytes(2, "big") * 2 + min(sizes).to_bytes(3, "big") + max(sizes).to_bytes(3, "big")
    si += (24000 << 44 | 15 << 36 | n).to_bytes(8, "big") + md5
    return b"fLaC" + bytes([0x80, 0, 0, 34]) + si + b"".join(frames)


def _assembled():
    """Four frames: CONSTANT, VERBATIM, FIXED order 2, LPC order 2 (short last frame of 1000 samples)."""
    rng = np.random.default_rng(3)
    c = np.full(4096, -1234, np.int64)
    v = rng.integers(-32768, 32768, 4096)
    t = np.arange(4096)
    fx = np.round(8000 * np.sin(t / 40.0)).astype(np.int64) + rng.integers(-3, 4, 4096)
    q, shift = [1900, -900], 10                   # LPC: (1900 s1 - 900 s2) >> 10
    lp = np.zeros(1000, np.int64)
    lp[:2] = [100, 180]
    er = rng.integers(-20, 21, 1000)
    for i in range(2, 1000):
        lp[i] = er[i] + ((q[0] * lp[i - 1] + q[1] * lp[i - 2]) >> shift)
    assert np.abs(lp).max() < 32768
    frames = [
        _frame(0, 4096, lambda w: (w.put(0, 8), w.put(-1234, 16))),
        _frame(1, 4096, lambda w: (w.put(1 << 1, 8), [w.put(int(x), 16) for x in v])),
        _frame(2, 4096, lambda w: (w.put((8 | 2) << 1, 8), w.put(int(fx[0]), 16), w.put(int(fx[1]), 16),
                                   _residual(w, fx[2:] - 2 * fx[1:-1] + fx[:-2], 3))),
        _frame(3, 1000, lambda w: (w.put((32 | 1) << 1, 8), w.put(100, 16), w.put(180, 16), w.put(11, 4),
                                   w.put(shift, 5), w.put(q[0], 12), w.put(q[1], 12),
                                   _residual(w, er[2:], 5))),
    ]
    x = np.concatenate([c, v, fx, lp]).astype(np.int16)
    return _stream(frames, x.size, hashlib.md5(x.astype("<i2").tobytes()).digest()), x


# ---------------------------------------------------------------------------------------------------- the oracle
def test_crc_check_values():
    assert F.crc8(b"123456789") == 0xF4
    assert F.crc16(b"123456789") == 0xFEE8


@pytest.mark.parametrize("v", [0, 0x7F, 0x80, 0x7FF, 0x800, 0xFFFF, 0x10000, 2 ** 31 - 1])
def test_frame_number_round_trip(v):
    b = _utf8(v)
    assert F.utf8_decode(b + b"\x00", 0) == (v, len(b))


def test_zigzag_and_rice_round_trip():
    r = np.array([0, -1, 1, -2, 2, 12345, -12345, 2 ** 31 - 1, -(2 ** 31 - 1)], np.int64)
    u = F.zigzag(r)
    assert u[:5].tolist() == [0, 1, 2, 3, 4]
    assert np.array_equal(F.unzigzag(u), r)
    for k in (0, 1, 5, 14):
        small = r[np.abs(r) < 1 << 16]
        w = _W()
        for v in small:
            w.rice(int(v), k)
        w.pad()
        bits = F._Bits(w.bytes())
        assert np.array_equal(F.unzigzag(bits.rice(small.size, k)), small)


def test_assembled_stream_decodes():
    data, x = _assembled()
    for expect in (None, x):
        d = F.decode(data, expect=expect)
        assert d["samples"].dtype == np.int16 and np.array_equal(d["samples"], x)
        assert d["md5_checked"]
        assert [f["type"] for f in d["frames"]] == ["CONSTANT", "VERBATIM", "FIXED", "LPC"]
        assert [f["order"] for f in d["frames"]] == [0, 0, 2, 2]
        assert [f["blocksize"] for f in d["frames"]] == [4096, 4096, 4096, 1000]
        assert d["frames"][0]["bits"] == 24 and d["frames"][1]["bits"] == 8 + 16 * 4096
        si = d["streaminfo"]
        assert (si["sample_rate"], si["channels"], si["bits_per_sample"], si["total_samples"]) == (24000, 1, 16, x.size)


def test_fixed_only_bits():
    assert F.fixed_only_bits(np.full(4096, 7)) == 24
    ramp = np.arange(4096) - 2048
    # order 2 leaves all zeros: 8 + 32 warm-up + 6 + 4 + 4094 one-bit codes, at partition order 0
    assert F.fixed_only_bits(ramp) == 8 + 32 + 6 + 4 + 4094
    v = np.random.default_rng(0).integers(-32768, 32768, 4096)
    assert F.fixed_only_bits(v) <= 8 + 16 * 4096


@pytest.mark.parametrize("where", ["frame", "crc16", "crc8", "md5"])
def test_corruption_is_rejected(where):
    data, x = _assembled()
    b = bytearray(data)
    f = F.decode(data)["frames"]
    if where == "frame":
        b[f[2]["offset"] + f[2]["header_bytes"] + 40] ^= 0x10
    elif where == "crc16":
        b[f[1]["offset"] + f[1]["bytes"] - 1] ^= 0x01
    elif where == "crc8":
        b[f[3]["offset"] + f[3]["header_bytes"] - 1] ^= 0x80
    else:
        b[8 + 18 + 5] ^= 0x04
    with pytest.raises(F.FlacError):
        F.decode(bytes(b), expect=x)


# ---------------------------------------------------------------------------------------------------- TTSOutput dispatch
class _FakeFlac:
    def __init__(self):
        self.calls = []

    def change_speed(self, array, speed_factor):
        raise AssertionError("not called here")

    def encode_flac(self, pcm_i16, sample_rate, md5):
        self.calls.append((np.array(pcm_i16, copy=True), sample_rate, md5))
        if sample_rate > 1048575:
            raise ValueError("encode_flac: sample rate outside 1 .. 1048575 Hz")
        return b"fLaC-fake"


class _NoFlac:
    def change_speed(self, array, speed_factor):
        raise AssertionError("not called here")


@pytest.fixture
def fake(monkeypatch):
    from auralis_b200 import output
    monkeypatch.setattr(output, "_providers", [])
    eng = _FakeFlac()
    output.register_gpu_provider(eng)
    yield eng
    output.unregister_gpu_provider(eng)


def _x():
    from oracle import enhance_oracle as E
    x = E.synthetic_input(0.3, 24000, 9)
    x[:10] = [1.5, -1.5, 1.0, -1.0, 0.99999, -0.99999, 0.0, 2e-5, -2e-5, 0.5]
    return x


def test_flac_dispatch_passes_the_pcm_samples(fake):
    from auralis_b200 import TTSOutput
    o = TTSOutput(array=_x(), sample_rate=22050)
    assert o.to_bytes("flac") == b"fLaC-fake"
    pcm, sr, md5 = fake.calls[0]
    want = o.to_bytes("pcm", 2)
    assert pcm.dtype == np.int16 and pcm.tobytes() == want
    assert sr == 22050 and md5 == hashlib.md5(want).digest()


def _old_path(o, width):
    """What the torchaudio path does with these arguments: its bytes, or the error it raises."""
    try:
        return o.to_bytes("flac", sample_width=width)
    except Exception as e:              # noqa: BLE001
        return type(e), str(e)


@pytest.mark.parametrize("width", [1, 4])
def test_other_widths_keep_the_old_path(fake, monkeypatch, width):
    from auralis_b200 import TTSOutput, output
    o = TTSOutput(array=_x())
    got = _old_path(o, width)
    monkeypatch.setattr(output, "_providers", [])
    assert got == _old_path(o, width)
    assert fake.calls == []


def test_no_provider_keeps_the_old_path(monkeypatch):
    from auralis_b200 import TTSOutput, output
    monkeypatch.setattr(output, "_providers", [])
    o = TTSOutput(array=_x())
    got = _old_path(o, 2)
    assert got != b"fLaC-fake"
    try:
        import torchaudio  # noqa: F401
        import torchcodec  # noqa: F401
    except ImportError:
        assert got[0] is RuntimeError and "codec backend" in got[1]


def test_provider_without_encode_flac_keeps_the_old_path(monkeypatch):
    from auralis_b200 import TTSOutput, output
    monkeypatch.setattr(output, "_providers", [])
    o = TTSOutput(array=_x())
    want = _old_path(o, 2)
    eng = _NoFlac()
    output.register_gpu_provider(eng)
    assert output.gpu_provider() is eng
    assert _old_path(o, 2) == want


def test_invalid_becomes_value_error(fake):
    from auralis_b200 import TTSOutput
    with pytest.raises(ValueError):
        TTSOutput(array=_x(), sample_rate=2_000_000).to_bytes("flac")


def test_save_writes_the_flac_bytes(fake, tmp_path):
    from auralis_b200 import TTSOutput
    o = TTSOutput(array=_x(), sample_rate=24000)
    o.save(tmp_path / "x.flac")
    assert (tmp_path / "x.flac").read_bytes() == o.to_bytes("flac") == b"fLaC-fake"


def test_engine_maps_invalid_to_value_error():
    """XTTSv2Engine.encode_flac turns the native ERR_INVALID into ValueError and passes other errors on."""
    from auralis_b200 import native
    from auralis_b200.engine import XTTSv2Engine

    class _Native:
        def __init__(self, code):
            self.code = code

        def encode_flac(self, pcm, sr, md5):
            if self.code:
                raise native.NativeError("encode_flac failed", self.code)
            return b"ok"

    eng = XTTSv2Engine.__new__(XTTSv2Engine)
    eng.native = _Native(0)
    assert eng.encode_flac(np.zeros(4, np.int16), 24000) == b"ok"
    eng.native = _Native(native.ERR_INVALID)
    with pytest.raises(ValueError):
        eng.encode_flac(np.zeros(4, np.int16), 0)
    eng.native = _Native(-2)
    with pytest.raises(native.NativeError):
        eng.encode_flac(np.zeros(4, np.int16), 24000)
