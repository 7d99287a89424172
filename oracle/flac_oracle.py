"""Test oracle for the GPU FLAC encoder (auralis_b200/csrc/flac.cu): an independent decoder and an exact yardstick.

Written from the FLAC format (RFC 9639), not from the encoder.  `decode` checks the sync code, every reserved bit, each
frame's CRC-8 and CRC-16, the frame numbers of a fixed-blocksize stream, the block sizes against STREAMINFO, the zero
padding, the total sample count and the MD5, and returns the samples with the STREAMINFO fields and, per frame, the
subframe type, order and size in bits.  `fixed_only_bits` is the exact smallest coded size of a block over CONSTANT,
VERBATIM and FIXED orders 0..4 with the best partitioned Rice coding (integer arithmetic only).

Test infrastructure only: the product package never imports it.
"""
from __future__ import annotations

import hashlib
from typing import Dict, List, Optional

import numpy as np


class FlacError(ValueError):
    """The stream breaks the format or fails one of its checks."""


# ---------------------------------------------------------------------------------------------------- checksums
def _crc_table(poly: int, width: int) -> List[int]:
    top, mask = 1 << (width - 1), (1 << width) - 1
    tab = []
    for i in range(256):
        c = i << (width - 8)
        for _ in range(8):
            c = ((c << 1) ^ poly) if c & top else c << 1
        tab.append(c & mask)
    return tab


_CRC8 = _crc_table(0x07, 8)
_CRC16 = _crc_table(0x8005, 16)


def crc8(data: bytes) -> int:
    """CRC-8, polynomial x^8 + x^2 + x + 1 (0x07), initial value 0: the frame-header checksum."""
    c = 0
    for b in data:
        c = _CRC8[c ^ b]
    return c


def crc16(data: bytes) -> int:
    """CRC-16, polynomial x^16 + x^15 + x^2 + 1 (0x8005), initial value 0: the whole-frame checksum."""
    c = 0
    for b in data:
        c = ((c << 8) & 0xFFFF) ^ _CRC16[(c >> 8) ^ b]
    return c


# ---------------------------------------------------------------------------------------------------- small codes
def utf8_decode(data: bytes, pos: int):
    """The frame number coded UTF-8-style at data[pos:] -> (value, bytes used)."""
    b0 = data[pos]
    if b0 < 0x80:
        return b0, 1
    n = 0
    while n < 8 and b0 & (0x80 >> n):
        n += 1
    if n < 2 or n > 7:
        raise FlacError(f"bad frame-number lead byte {b0:#04x}")
    v = b0 & (0x7F >> n)
    for i in range(1, n):
        c = data[pos + i]
        if c & 0xC0 != 0x80:
            raise FlacError(f"bad frame-number continuation byte {c:#04x}")
        v = (v << 6) | (c & 0x3F)
    return v, n


def zigzag(r):
    """Signed residual -> the folded value Rice codes: r >= 0 -> 2r, r < 0 -> -2r - 1."""
    r = np.asarray(r, np.int64)
    return np.where(r >= 0, 2 * r, -2 * r - 1)


def unzigzag(u):
    u = np.asarray(u, np.int64)
    return (u >> 1) ^ -(u & 1)


BLOCK_SIZES = {1: 192, 2: 576, 3: 1152, 4: 2304, 5: 4608, **{c: 256 << (c - 8) for c in range(8, 16)}}
SAMPLE_RATES = {1: 88200, 2: 176400, 3: 192000, 4: 8000, 5: 16000, 6: 22050, 7: 24000, 8: 32000, 9: 44100, 10: 48000,
                11: 96000}
FIXED_COEFS = {0: [], 1: [1], 2: [2, -1], 3: [3, -3, 1], 4: [4, -6, 4, -1]}


# ---------------------------------------------------------------------------------------------------- bit reader
class _Bits:
    """MSB-first reader over a byte string, one byte per bit in `s` so that `find` runs in C."""

    def __init__(self, buf: bytes):
        self.a = np.unpackbits(np.frombuffer(buf, np.uint8))
        self.s = self.a.tobytes()
        self.p = 0

    def need(self, n: int):
        if self.p + n > self.a.size:
            raise FlacError("frame runs past the end of the stream")

    def read(self, n: int) -> int:
        self.need(n)
        v = 0
        for b in self.s[self.p:self.p + n]:
            v = (v << 1) | b
        self.p += n
        return v

    def signed(self, n: int) -> int:
        v = self.read(n)
        return v - (1 << n) if v >> (n - 1) else v

    def signed_array(self, count: int, n: int) -> np.ndarray:
        self.need(count * n)
        w = self.a[self.p:self.p + count * n].reshape(count, n).astype(np.int64)
        v = w @ (1 << np.arange(n - 1, -1, -1, dtype=np.int64))
        self.p += count * n
        return np.where(v >> (n - 1), v - (1 << n), v)

    def rice(self, count: int, k: int) -> np.ndarray:
        """`count` Rice codes with parameter k -> folded values."""
        ones = np.empty(count, np.int64)
        p, s = self.p, self.s
        for i in range(count):
            o = s.find(b"\x01", p)
            if o < 0:
                raise FlacError("Rice code runs past the end of the stream")
            ones[i] = o
            p = o + 1 + k
        starts = np.empty(count, np.int64)
        if count:
            starts[0] = self.p
            starts[1:] = ones[:-1] + 1 + k
        self.p = p
        self.need(0)
        q = ones - starts
        if k == 0:
            return q
        low = np.zeros(count, np.int64)
        for j in range(k):
            low = (low << 1) | self.a[ones + 1 + j]
        return (q << k) | low


# ---------------------------------------------------------------------------------------------------- decoder
def _residual(bits: _Bits, nb: int, order: int) -> np.ndarray:
    method = bits.read(2)
    if method > 1:
        raise FlacError(f"reserved residual coding method {method}")
    pbits = 4 if method == 0 else 5
    porder = bits.read(4)
    parts = 1 << porder
    if nb % parts or (nb >> porder) < order:
        raise FlacError(f"partition order {porder} does not fit a block of {nb} with order {order}")
    out = []
    for j in range(parts):
        cnt = (nb >> porder) - (order if j == 0 else 0)
        k = bits.read(pbits)
        if k == (1 << pbits) - 1:                       # escape: cnt raw signed values of n bits
            n = bits.read(5)
            out.append(bits.signed_array(cnt, n) if n else np.zeros(cnt, np.int64))
        else:
            out.append(unzigzag(bits.rice(cnt, k)))
    return np.concatenate(out) if out else np.zeros(0, np.int64)


def _predict(warm: np.ndarray, coefs: List[int], shift: int, r: np.ndarray, expect: Optional[np.ndarray]):
    """Samples of a predicted subframe.  With `expect` (the samples the caller expects), the decoded block equals it
    exactly when the warm-up matches and every residual equals expect[n] - prediction(expect[n-1], ...), which is
    checked vectorised; otherwise (or when it does not hold) the recursion runs sample by sample."""
    order, nb = len(coefs), len(warm) + len(r)
    if expect is not None and len(expect) == nb and np.array_equal(warm, expect[:order]):
        e = expect.astype(np.int64)
        acc = np.zeros(nb - order, np.int64)
        for j, c in enumerate(coefs):
            acc += c * e[order - 1 - j: nb - 1 - j]
        if np.array_equal(e[order:] - (acc >> shift), r):
            return e
    s = [int(v) for v in warm] + [0] * len(r)
    rl = r.tolist()
    for n in range(order, nb):
        acc = 0
        for j, c in enumerate(coefs):
            acc += c * s[n - 1 - j]
        s[n] = rl[n - order] + (acc >> shift)
    return np.asarray(s, np.int64)


def _subframe(bits: _Bits, nb: int, expect: Optional[np.ndarray]):
    if bits.read(1):
        raise FlacError("subframe padding bit set")
    t = bits.read(6)
    if bits.read(1):
        raise FlacError("wasted-bits flag set (not produced for 16-bit mono here)")
    start = bits.p - 8
    info: Dict = {"order": 0}
    if t == 0:
        info["type"] = "CONSTANT"
        samples = np.full(nb, bits.signed(16), np.int64)
    elif t == 1:
        info["type"] = "VERBATIM"
        samples = bits.signed_array(nb, 16)
    elif 8 <= t <= 12:
        order = t - 8
        if order > nb:
            raise FlacError("FIXED order larger than the block")
        info.update(type="FIXED", order=order)
        warm = bits.signed_array(order, 16) if order else np.zeros(0, np.int64)
        samples = _predict(warm, FIXED_COEFS[order], 0, _residual(bits, nb, order), expect)
    elif t >= 32:
        order = t - 31
        if order > nb:
            raise FlacError("LPC order larger than the block")
        warm = bits.signed_array(order, 16)
        prec = bits.read(4) + 1
        if prec == 16:
            raise FlacError("invalid LPC precision 1111")
        shift = bits.signed(5)
        if shift < 0:
            raise FlacError("negative LPC shift")
        coefs = [bits.signed(prec) for _ in range(order)]
        info.update(type="LPC", order=order, precision=prec, shift=shift, coefs=coefs)
        samples = _predict(warm, coefs, shift, _residual(bits, nb, order), expect)
    else:
        raise FlacError(f"reserved subframe type {t:#04x}")
    info["bits"] = bits.p - start
    return samples, info


def _streaminfo(b: bytes) -> Dict:
    v = int.from_bytes(b[10:18], "big")
    return {"min_block": int.from_bytes(b[0:2], "big"), "max_block": int.from_bytes(b[2:4], "big"),
            "min_frame": int.from_bytes(b[4:7], "big"), "max_frame": int.from_bytes(b[7:10], "big"),
            "sample_rate": v >> 44, "channels": ((v >> 41) & 7) + 1, "bits_per_sample": ((v >> 36) & 31) + 1,
            "total_samples": v & ((1 << 36) - 1), "md5": bytes(b[18:34])}


def decode(data: bytes, expect=None) -> Dict:
    """Decode a mono 16-bit fixed-blocksize FLAC stream and check it -> {"samples": int16 [n], "streaminfo": {...},
    "frames": [{"number", "offset", "bytes", "blocksize", "type", "order", "bits", ...}], "md5_checked": bool}.
    `expect` (int16 samples) only speeds up decoding of predicted subframes (see `_predict`); the result is the same.
    Raises FlacError on any violation."""
    data = bytes(data)
    if data[:4] != b"fLaC":
        raise FlacError("no fLaC marker")
    pos, si, last = 4, None, False
    while not last:
        if pos + 4 > len(data):
            raise FlacError("truncated metadata")
        last, btype, blen = bool(data[pos] & 0x80), data[pos] & 0x7F, int.from_bytes(data[pos + 1:pos + 4], "big")
        body = data[pos + 4:pos + 4 + blen]
        if si is None:
            if btype != 0 or blen != 34:
                raise FlacError("the first metadata block is not a 34-byte STREAMINFO")
            si = _streaminfo(body)
        pos += 4 + blen
    if si["channels"] != 1 or si["bits_per_sample"] != 16:
        raise FlacError("not mono 16-bit")
    if not 16 <= si["min_block"] <= si["max_block"]:
        raise FlacError("bad STREAMINFO block sizes")
    total = si["total_samples"]
    ex = None if expect is None else np.asarray(expect, np.int16)
    out, frames, done = [], [], 0
    while done < total:
        f0 = pos
        hdr = data[pos:pos + 16]
        if len(hdr) < 6 or hdr[0] != 0xFF or hdr[1] & 0xFE != 0xF8:
            raise FlacError(f"no frame sync at byte {pos}")
        if hdr[1] & 1:
            raise FlacError("variable-blocksize frame in a fixed-blocksize stream")
        bcode, rcode = hdr[2] >> 4, hdr[2] & 15
        chan, scode, res = hdr[3] >> 4, (hdr[3] >> 1) & 7, hdr[3] & 1
        if chan != 0 or scode not in (0, 4) or res:
            raise FlacError(f"frame header byte 3 {hdr[3]:#04x}: not mono 16-bit, or reserved bit set")
        if bcode == 0 or rcode == 15:
            raise FlacError("reserved block-size or sample-rate code")
        number, n = utf8_decode(data, pos + 4)
        p = pos + 4 + n
        if bcode == 6:
            nb, p = data[p] + 1, p + 1
        elif bcode == 7:
            nb, p = int.from_bytes(data[p:p + 2], "big") + 1, p + 2
        else:
            nb = BLOCK_SIZES[bcode]
        if rcode == 12:
            rate, p = data[p] * 1000, p + 1
        elif rcode == 13:
            rate, p = int.from_bytes(data[p:p + 2], "big"), p + 2
        elif rcode == 14:
            rate, p = int.from_bytes(data[p:p + 2], "big") * 10, p + 2
        else:
            rate = SAMPLE_RATES.get(rcode, si["sample_rate"])
        if rate != si["sample_rate"]:
            raise FlacError(f"frame sample rate {rate} != STREAMINFO's {si['sample_rate']}")
        if crc8(data[pos:p]) != data[p]:
            raise FlacError(f"CRC-8 mismatch in frame {len(frames)}")
        p += 1
        if number != len(frames):
            raise FlacError(f"frame number {number}, expected {len(frames)}")
        if nb > si["max_block"] or (done + nb < total and (nb != si["max_block"] or nb < si["min_block"])):
            raise FlacError(f"block size {nb} in frame {number}")
        if done + nb > total:
            raise FlacError("frames hold more samples than STREAMINFO says")
        hlen = p - pos
        bits = _Bits(data[p:p + 5 * nb + 256])               # more than any subframe of nb samples takes
        samples, info = _subframe(bits, nb, None if ex is None else ex[done:done + nb])
        pad = (-bits.p) % 8
        if pad and bits.read(pad):
            raise FlacError("non-zero frame padding")
        end = p + bits.p // 8
        if end + 2 > len(data):
            raise FlacError("truncated frame")
        if crc16(data[pos:end]) != int.from_bytes(data[end:end + 2], "big"):
            raise FlacError(f"CRC-16 mismatch in frame {number}")
        if samples.min(initial=0) < -32768 or samples.max(initial=0) > 32767:
            raise FlacError("decoded sample outside 16 bits")
        pos = end + 2
        info.update(number=number, offset=f0, bytes=pos - f0, header_bytes=hlen, blocksize=nb)
        frames.append(info)
        out.append(samples.astype(np.int16))
        done += nb
    if pos != len(data):
        raise FlacError(f"{len(data) - pos} bytes after the last frame")
    samples = np.concatenate(out) if out else np.zeros(0, np.int16)
    md5_checked = si["md5"] != bytes(16)
    if md5_checked and hashlib.md5(samples.astype("<i2").tobytes()).digest() != si["md5"]:
        raise FlacError("MD5 mismatch")
    return {"samples": samples, "streaminfo": si, "frames": frames, "md5_checked": md5_checked}


# ---------------------------------------------------------------------------------------------------- yardstick
def rice_bits(u: np.ndarray, nb: int, order: int, max_porder: int = 6) -> int:
    """Exact smallest partitioned-Rice size in bits (method 00, parameters 0..14, partition orders 0..max_porder with
    nb divisible by 2^p and (nb >> p) > order) of the folded residuals u of samples order .. nb-1, method and
    partition-order fields included."""
    u = np.asarray(u, np.int64)
    best = None
    for p in range(max_porder + 1):
        if nb % (1 << p) or (nb >> p) <= order:
            break
        L = nb >> p
        full = np.concatenate([np.zeros(order, np.int64), u]).reshape(1 << p, L)
        cnt = np.full(1 << p, L, np.int64)
        cnt[0] -= order
        cost = np.stack([(full >> k).sum(axis=1) + cnt * (k + 1) for k in range(15)])     # [k][partition]
        total = 6 + int((4 + cost.min(axis=0)).sum())
        best = total if best is None else min(best, total)
    return best


def fixed_only_bits(block) -> int:
    """Exact smallest subframe size in bits of `block` (int16) over CONSTANT (all samples equal), VERBATIM and FIXED
    orders 0..4 (those below the block length) with the best partitioned Rice coding."""
    s = np.asarray(block, np.int64)
    nb = s.size
    best = 8 + 16 * nb
    if np.all(s == s[0]):
        best = min(best, 8 + 16)
    for order in range(5):
        if order >= nb:
            break
        r = s[order:].copy()
        for j, c in enumerate(FIXED_COEFS[order]):
            r -= c * s[order - 1 - j: nb - 1 - j]
        best = min(best, 8 + 16 * order + rice_bits(zigzag(r), nb, order))
    return best
