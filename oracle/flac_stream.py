"""Test oracle for the GPU FLAC decoder (auralis_b200/csrc/flac.cu, `xtts_decode_flac`): a general FLAC stream writer
with explicit per-frame choices, and a general sequential decoder, both written from the format (RFC 9639).

`write_stream` takes PCM [C, N] and a bit depth and writes exactly what it is told: block sizes and blocking strategy,
channel assignment, subframe type / order / wasted bits per channel, LPC precision, shift and coefficients, RICE or
RICE2 residuals with a partition order and per-partition parameters or escapes, the header's block-size and
sample-rate codes, metadata blocks, an ID3v2 prefix, an ID3v1 trailer, a zero STREAMINFO total or MD5, and fake frame
headers inside VERBATIM payloads (false syncs).

`decode` walks the stream strictly in order, parsing each frame to its end and taking the next frame to start there.
It makes the same checks as `xtts_decode_flac` and raises `FlacError` where that call returns XTTS_ERR_INVALID.

Test infrastructure only: the product package never imports it.
"""
from __future__ import annotations

import hashlib
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np

from .flac_oracle import BLOCK_SIZES, FIXED_COEFS, SAMPLE_RATES, FlacError, crc8, crc16

SAMPLE_SIZES = {1: 8, 2: 12, 4: 16, 5: 20, 6: 24, 7: 32}
INDEPENDENT, LEFT_SIDE, SIDE_RIGHT, MID_SIDE = "independent", "left_side", "side_right", "mid_side"
_CA_CODE = {LEFT_SIDE: 8, SIDE_RIGHT: 9, MID_SIDE: 10}


# ---------------------------------------------------------------------------------------------------- helpers
def md5_of(samples: np.ndarray, bps: int) -> bytes:
    """STREAMINFO's MD5: samples [C, N] interleaved, little-endian, ceil(bps / 8) bytes each."""
    s = np.ascontiguousarray(np.asarray(samples, np.int64).T).astype("<i4")
    nb = (bps + 7) // 8
    raw = s.view(np.uint8).reshape(-1, 4)[:, :nb]
    return hashlib.md5(raw.tobytes()).digest()


def _fold(r: np.ndarray) -> np.ndarray:
    r = np.asarray(r, np.int64)
    return np.where(r >= 0, 2 * r, -2 * r - 1)


def _utf8(v: int) -> bytes:
    if v < 0x80:
        return bytes([v])
    n = 2
    while v >> (5 * n + 1):
        n += 1
    out = [((0xFF00 >> n) & 0xFF) | (v >> (6 * (n - 1)))]
    out += [0x80 | ((v >> (6 * c)) & 0x3F) for c in range(n - 2, -1, -1)]
    return bytes(out)


class _BitWriter:
    def __init__(self):
        self.bits: List[np.ndarray] = []
        self.n = 0

    def put(self, v: int, n: int):
        if n:
            v &= (1 << n) - 1
            self.bits.append(np.array([(v >> (n - 1 - i)) & 1 for i in range(n)], np.uint8))
            self.n += n

    def put_array(self, vals: np.ndarray, n: int):
        """Each value in n bits, two's complement."""
        if n and len(vals):
            v = np.asarray(vals, np.int64) & ((1 << n) - 1)
            self.bits.append(((v[:, None] >> np.arange(n - 1, -1, -1)) & 1).astype(np.uint8).reshape(-1))
            self.n += n * len(vals)

    def put_rice(self, u: np.ndarray, k: int):
        """Rice codes of the folded values u: q zeros, a one, then the k low bits."""
        if not len(u):
            return
        q = (u >> k).astype(np.int64)
        lens = q + 1 + k
        out = np.zeros(int(lens.sum()), np.uint8)
        starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
        out[starts + q] = 1
        for j in range(k):
            out[starts + q + 1 + j] = (u >> (k - 1 - j)) & 1
        self.bits.append(out)
        self.n += out.size

    def pad(self):
        self.put(0, (-self.n) % 8)

    def tobytes(self) -> bytes:
        return np.packbits(np.concatenate(self.bits) if self.bits else np.zeros(0, np.uint8)).tobytes()


# ---------------------------------------------------------------------------------------------------- writer
@dataclass
class Sub:
    """One subframe.  kind: CONSTANT, VERBATIM, FIXED (order 0..4) or LPC (order 1..32).  coefs None: least squares,
    quantised at `precision` bits with `shift`.  rice2: 5-bit parameters.  params: one Rice parameter per partition,
    or None for the cheapest; escape: {partition: raw bit width} (0 = every residual of the partition is zero)."""
    kind: str = "FIXED"
    order: int = 2
    wasted: int = 0
    precision: int = 12
    shift: int = 10
    coefs: Optional[Sequence[int]] = None
    rice2: bool = False
    porder: int = 0
    params: Optional[Sequence[int]] = None
    escape: Dict[int, int] = field(default_factory=dict)


@dataclass
class Frame:
    """One frame: its block size, channel assignment, one Sub per channel (None: FIXED 2 everywhere).
    bs_code: None = the table code when there is one, else 6 / 7; or 6 / 7 forced.  rate_code: None = the table code
    or 0 ("from STREAMINFO"); 0, 12, 13 or 14 forced.  size_code: None = the table code; 0 = from STREAMINFO.
    fake_sync: 1 = the next frame's header is written into this frame's VERBATIM payload of channel 0 at sample
    `fake_at`; 2 = also the two bytes before it make the CRC-16 of the frame prefix they close."""
    blocksize: int
    assignment: str = INDEPENDENT
    subs: Optional[List[Sub]] = None
    bs_code: Optional[int] = None
    rate_code: Optional[int] = None
    size_code: Optional[int] = None
    fake_sync: int = 0
    fake_at: int = 8


@dataclass
class Stream:
    data: bytes
    pcm: np.ndarray            # [C, N] int64: what the stream holds (fake syncs rewrite some samples)
    sample_rate: int
    bps: int
    frame_offsets: List[int]


def _header(fr: Frame, number: int, variable: bool, C: int, bps: int, sr: int) -> bytes:
    nb = fr.blocksize
    bc = fr.bs_code
    if bc is None:
        bc = next((c for c, v in BLOCK_SIZES.items() if v == nb), 6 if nb <= 256 else 7)
    rc = fr.rate_code
    if rc is None:
        rc = next((c for c, v in SAMPLE_RATES.items() if v == sr), 0)
    sc = fr.size_code
    if sc is None:
        sc = next((c for c, v in SAMPLE_SIZES.items() if v == bps), 0)
    ca = C - 1 if fr.assignment == INDEPENDENT else _CA_CODE[fr.assignment]
    h = bytearray([0xFF, 0xF8 | int(variable), bc << 4 | rc, ca << 4 | sc << 1])
    h += _utf8(number)
    if bc == 6:
        h.append(nb - 1)
    elif bc == 7:
        h += (nb - 1).to_bytes(2, "big")
    if rc == 12:
        h.append(sr // 1000)
    elif rc == 13:
        h += sr.to_bytes(2, "big")
    elif rc == 14:
        h += (sr // 10).to_bytes(2, "big")
    h.append(crc8(bytes(h)))
    return bytes(h)


def _lpc_coefs(x: np.ndarray, order: int, precision: int, shift: int) -> List[int]:
    n = x.size
    if n <= order:
        return [0] * order
    A = np.stack([x[order - 1 - j: n - 1 - j] for j in range(order)], axis=1).astype(np.float64)
    c, *_ = np.linalg.lstsq(A, x[order:].astype(np.float64), rcond=None)
    lim = 1 << (precision - 1)
    return [int(v) for v in np.clip(np.round(c * (1 << shift)), -lim, lim - 1)]


def _residual(bw: _BitWriter, r: np.ndarray, nb: int, order: int, s: Sub):
    pbits, esc = (5, 31) if s.rice2 else (4, 15)
    parts = 1 << s.porder
    if nb % parts or (nb >> s.porder) < order:
        raise ValueError("partition order does not fit the block")
    bw.put(1 if s.rice2 else 0, 2)
    bw.put(s.porder, 4)
    L = nb >> s.porder
    u_all = _fold(r)
    if u_all.size and u_all.max() >= 1 << 32:
        raise ValueError("a residual does not fit 32 bits")
    pos = 0
    for j in range(parts):
        cnt = L - (order if j == 0 else 0)
        rj, u = r[pos:pos + cnt], u_all[pos:pos + cnt]
        pos += cnt
        if j in s.escape:
            n = s.escape[j]
            if (n == 0 and np.any(rj)) or (n and rj.size and (rj.min() < -(1 << (n - 1)) or rj.max() >= 1 << (n - 1))):
                raise ValueError(f"partition {j} does not fit {n} raw bits")
            bw.put(esc, pbits)
            bw.put(n, 5)
            bw.put_array(rj, n)
            continue
        if s.params is not None:
            k = s.params[j]
            if not 0 <= k < esc:
                raise ValueError(f"Rice parameter {k} does not fit {pbits} bits")
        else:
            ks = range(esc)
            k = min(ks, key=lambda k: int((u >> k).sum()) + cnt * (k + 1))
        bw.put(k, pbits)
        bw.put_rice(u, k)


def _subframe(bw: _BitWriter, x: np.ndarray, sbits: int, s: Sub):
    """x: the subframe's samples (int64), in sbits bits."""
    nb = x.size
    w = s.wasted
    if w:
        if np.any(x & ((1 << w) - 1)):
            raise ValueError("samples do not have that many wasted bits")
        x = x >> w
    b = sbits - w
    if s.kind == "CONSTANT":
        t = 0
    elif s.kind == "VERBATIM":
        t = 1
    elif s.kind == "FIXED":
        t = 8 + s.order
    else:
        t = 31 + s.order
    bw.put(0, 1)
    bw.put(t, 6)
    bw.put(1 if w else 0, 1)
    if w:
        bw.put(1, w)                      # w - 1 zeros and a one
    if s.kind == "CONSTANT":
        if np.any(x != x[0]):
            raise ValueError("CONSTANT subframe of a non-constant block")
        bw.put(int(x[0]), b)
        return
    if s.kind == "VERBATIM":
        bw.put_array(x, b)
        return
    o = s.order
    bw.put_array(x[:o], b)
    if s.kind == "FIXED":
        coefs, shift = FIXED_COEFS[o], 0
    else:
        coefs = list(s.coefs) if s.coefs is not None else _lpc_coefs(x, o, s.precision, s.shift)
        shift = s.shift
        bw.put(s.precision - 1, 4)
        bw.put(shift, 5)
        bw.put_array(np.asarray(coefs), s.precision)
    acc = np.zeros(max(nb - o, 0), np.int64)
    for j, c in enumerate(coefs):
        acc += int(c) * x[o - 1 - j: nb - 1 - j]
    _residual(bw, x[o:] - (acc >> shift), nb, o, s)


def _channels(fr: Frame, blk: np.ndarray, bps: int):
    """-> [(samples, sbits)] of the coded channels."""
    a = fr.assignment
    if a == INDEPENDENT:
        return [(blk[c], bps) for c in range(blk.shape[0])]
    L, R = blk[0], blk[1]
    if a == LEFT_SIDE:
        return [(L, bps), (L - R, bps + 1)]
    if a == SIDE_RIGHT:
        return [(L - R, bps + 1), (R, bps)]
    return [((L + R) >> 1, bps), (L - R, bps + 1)]


def write_stream(pcm, bps: int, sample_rate: int, frames: List[Frame], variable: bool = False,
                 metadata: Sequence = (), id3v2: int = 0, id3v1: bool = False, total_zero: bool = False,
                 md5: bool = True, min_block: Optional[int] = None, max_block: Optional[int] = None) -> Stream:
    """A FLAC stream of pcm [C, N] (signed integers in bps bits).  frames must cover the N samples.  metadata:
    (type, payload bytes) blocks after STREAMINFO.  id3v2: the size of an ID3v2 tag in front (0 = none); id3v1: a
    128-byte "TAG" trailer."""
    pcm = np.array(pcm, np.int64, copy=True)
    if pcm.ndim == 1:
        pcm = pcm[None]
    C, N = pcm.shape
    if sum(f.blocksize for f in frames) != N:
        raise ValueError("frames do not cover the samples")
    out, offsets, done = bytearray(), [], 0
    for i, fr in enumerate(frames):
        nb = fr.blocksize
        number = done if variable else i
        hdr = _header(fr, number, variable, C, bps, sample_rate)
        subs = fr.subs or [Sub() for _ in range(C)]
        if fr.fake_sync:
            nxt = frames[i + 1] if i + 1 < len(frames) else fr
            fake = _header(nxt, done + nb if variable else i + 1, variable, C, bps, sample_rate)
            if fr.assignment != INDEPENDENT or subs[0].kind != "VERBATIM" or bps != 16 or subs[0].wasted:
                raise ValueError("fake syncs go into a 16-bit VERBATIM channel 0")
            if len(fake) % 2:
                fake += b"\x00"         # pad to whole samples (the byte after the header is payload)
            at = fr.fake_at
            vals = np.frombuffer(fake, ">i2").astype(np.int64)
            pcm[0, done + at + 1: done + at + 1 + vals.size] = vals
            if fr.fake_sync == 2:       # sample `at` = CRC-16 of everything in the frame before it
                prefix = hdr + bytes([0x02]) + pcm[0, done:done + at].astype(">i2").tobytes()
                c = crc16(prefix)
                pcm[0, done + at] = c - 65536 if c >= 32768 else c
        blk = pcm[:, done:done + nb]
        bw = _BitWriter()
        for (x, sbits), s in zip(_channels(fr, blk, bps), subs):
            _subframe(bw, x, sbits, s)
        bw.pad()
        body = hdr + bw.tobytes()
        offsets.append(len(out))
        out += body + crc16(body).to_bytes(2, "big")
        done += nb
    sizes = [f.blocksize for f in frames]
    mx = max_block if max_block is not None else max(sizes + [16])
    mn = min_block if min_block is not None else max(16, min(sizes[:-1] or [mx]))
    fsz = np.diff(offsets + [len(out)]) if offsets else np.zeros(1, np.int64)
    si = bytearray(mn.to_bytes(2, "big") + mx.to_bytes(2, "big") + int(fsz.min()).to_bytes(3, "big")
                   + int(fsz.max()).to_bytes(3, "big"))
    packed = sample_rate << 44 | (C - 1) << 41 | (bps - 1) << 36 | (0 if total_zero else N)
    si += packed.to_bytes(8, "big") + (md5_of(pcm, bps) if md5 else bytes(16))
    blocks = [(0, bytes(si))] + [(t, bytes(p)) for t, p in metadata]
    head = bytearray(b"fLaC")
    for j, (t, p) in enumerate(blocks):
        head += bytes([(0x80 if j == len(blocks) - 1 else 0) | t]) + len(p).to_bytes(3, "big") + p
    pre = b""
    if id3v2:
        sz = id3v2
        pre = b"ID3\x03\x00\x00" + bytes([(sz >> 21) & 0x7F, (sz >> 14) & 0x7F, (sz >> 7) & 0x7F, sz & 0x7F]) + bytes(sz)
    tail = (b"TAG" + bytes(range(125))) if id3v1 else b""
    base = len(pre) + len(head)
    return Stream(pre + bytes(head) + bytes(out) + tail, pcm, sample_rate, bps, [base + o for o in offsets])


# metadata payloads for write_stream
def padding(n: int = 64):
    return (1, bytes(n))


def vorbis_comment():
    vendor = b"flac_stream writer"
    c = b"TITLE=test"
    return (4, len(vendor).to_bytes(4, "little") + vendor + (1).to_bytes(4, "little") + len(c).to_bytes(4, "little") + c)


def seektable():
    return (3, (0).to_bytes(8, "big") + (0).to_bytes(8, "big") + (4096).to_bytes(2, "big"))


def picture():
    mime, desc, img = b"image/png", b"cover", bytes(100)
    p = (3).to_bytes(4, "big") + len(mime).to_bytes(4, "big") + mime + len(desc).to_bytes(4, "big") + desc
    return (6, p + (1).to_bytes(4, "big") * 2 + (24).to_bytes(4, "big") + (0).to_bytes(4, "big")
            + len(img).to_bytes(4, "big") + img)


def unknown_block():
    return (9, b"\x01\x02\x03")


# ---------------------------------------------------------------------------------------------------- decoder
class _Reader:
    """MSB-first bit reader over data[start:limit]; every read past `limit` raises.  Bits are unpacked in a window that
    doubles on demand, so a frame costs what it spans, not what follows it."""

    def __init__(self, data: bytes, start: int, limit: int):
        self.data, self.start, self.limit = data, start, limit
        self.p = 0
        self._unpack(min(limit - start, 1 << 15))

    def _unpack(self, nbytes: int):
        self.a = np.unpackbits(np.frombuffer(self.data, np.uint8, count=nbytes, offset=self.start))
        self.s = self.a.tobytes()

    def _grow(self) -> bool:
        have = self.a.size // 8
        if have >= self.limit - self.start:
            return False
        self._unpack(min(self.limit - self.start, 2 * have + 16))
        return True

    def need(self, n: int):
        while self.p + n > self.a.size:
            if not self._grow():
                raise FlacError("frame runs past the end of the data")

    def read(self, n: int) -> int:
        self.need(n)
        v = 0
        for b in self.s[self.p:self.p + n]:
            v = (v << 1) | b
        self.p += n
        return v

    def signed(self, n: int) -> int:
        v = self.read(n)
        return v - (1 << n) if n and v >> (n - 1) else v

    def signed_array(self, count: int, n: int) -> np.ndarray:
        if n == 0:
            return np.zeros(count, np.int64)
        self.need(count * n)
        w = self.a[self.p:self.p + count * n].reshape(count, n).astype(np.int64)
        v = np.zeros(count, np.int64)
        for j in range(n):
            v = (v << 1) | w[:, j]
        self.p += count * n
        return np.where(v >> (n - 1), v - (1 << n), v)

    def rice(self, count: int, k: int) -> np.ndarray:
        ones = np.empty(count, np.int64)
        p, i = self.p, 0
        while i < count:
            o = self.s.find(b"\x01", p)
            if o < 0 or o + 1 + k > self.a.size:
                if not self._grow():
                    raise FlacError("Rice code runs past the end of the data")
                continue
            ones[i] = o
            p = o + 1 + k
            i += 1
        starts = np.empty(count, np.int64)
        if count:
            starts[0] = self.p
            starts[1:] = ones[:-1] + 1 + k
        self.p = p
        q = ones - starts
        if count and int(q.max()) >= 1 << (32 - k):
            raise FlacError("a residual does not fit 32 bits")
        low = np.zeros(count, np.int64)
        for j in range(k):
            low = (low << 1) | self.a[ones + 1 + j]
        return (q << k) | low


def _unfold(u):
    return (u >> 1) ^ -(u & 1)


def _read_residual(rd: _Reader, nb: int, order: int) -> np.ndarray:
    method = rd.read(2)
    if method > 1:
        raise FlacError(f"reserved residual coding method {method}")
    pbits, esc = (4, 15) if method == 0 else (5, 31)
    porder = rd.read(4)
    if nb % (1 << porder) or (nb >> porder) < order:
        raise FlacError(f"partition order {porder} does not fit a block of {nb} with order {order}")
    out = []
    for j in range(1 << porder):
        cnt = (nb >> porder) - (order if j == 0 else 0)
        k = rd.read(pbits)
        if k == esc:
            out.append(rd.signed_array(cnt, rd.read(5)))
        else:
            out.append(_unfold(rd.rice(cnt, k)))
    return np.concatenate(out)


def _restore(warm, coefs, shift, r, lo, hi, expect):
    """s[n] = r[n] + (sum_j c_j s[n-1-j]) >> shift, every sample inside [lo, hi].  With `expect` (the samples the caller
    expects) the recursion is checked vectorised instead: the result is the same, only faster."""
    order, nb = len(coefs), len(warm) + len(r)
    if expect is not None and len(expect) == nb and np.array_equal(warm, expect[:order]):
        e = np.asarray(expect, np.int64)
        acc = np.zeros(nb - order, np.int64)
        for j, c in enumerate(coefs):
            acc += c * e[order - 1 - j: nb - 1 - j]
        if np.array_equal(e[order:] - (acc >> shift), r) and (nb == 0 or (e.min() >= lo and e.max() <= hi)):
            return e
    s = [int(v) for v in warm] + [0] * len(r)
    rl = r.tolist()
    for n in range(order, nb):
        acc = 0
        for j, c in enumerate(coefs):
            acc += c * s[n - 1 - j]
        v = rl[n - order] + (acc >> shift)
        if v < lo or v > hi:
            raise FlacError("a predicted sample does not fit the subframe's bits")
        s[n] = v
    return np.asarray(s, np.int64)


def _read_subframe(rd: _Reader, nb: int, sbits: int, expect):
    if rd.read(1):
        raise FlacError("subframe padding bit set")
    t = rd.read(6)
    w = 0
    if rd.read(1):
        w = 1
        while rd.read(1) == 0:
            w += 1
            if w >= sbits:
                break
        if w >= sbits:
            raise FlacError("wasted bits leave no sample bits")
    b = sbits - w
    lo, hi = -(1 << (b - 1)), (1 << (b - 1)) - 1
    ex = None if expect is None or w else expect
    if t == 0:
        x = np.full(nb, rd.signed(b), np.int64)
    elif t == 1:
        x = rd.signed_array(nb, b)
    elif 8 <= t <= 12:
        o = t - 8
        if o > nb:
            raise FlacError("FIXED order larger than the block")
        warm = rd.signed_array(o, b)
        x = _restore(warm, FIXED_COEFS[o], 0, _read_residual(rd, nb, o), lo, hi, ex)
    elif t >= 32:
        o = t - 31
        if o > nb:
            raise FlacError("LPC order larger than the block")
        warm = rd.signed_array(o, b)
        prec = rd.read(4) + 1
        if prec == 16:
            raise FlacError("invalid LPC precision 1111")
        shift = rd.signed(5)
        if shift < 0:
            raise FlacError("negative LPC shift")
        coefs = [rd.signed(prec) for _ in range(o)]
        x = _restore(warm, coefs, shift, _read_residual(rd, nb, o), lo, hi, ex)
    else:
        raise FlacError(f"reserved subframe type {t:#04x}")
    return x << w, {"type": t, "wasted": w}


def _utf8_read(data: bytes, p: int, end: int, maxlen: int):
    if p >= end:
        raise FlacError("truncated frame header")
    b0 = data[p]
    if b0 < 0x80:
        return b0, 1
    n = 0
    while n < 8 and b0 & (0x80 >> n):
        n += 1
    if n < 2 or n > maxlen:
        raise FlacError(f"bad frame-number lead byte {b0:#04x}")
    if p + n > end:
        raise FlacError("truncated frame header")
    v = b0 & (0x7F >> n)
    for i in range(1, n):
        c = data[p + i]
        if c & 0xC0 != 0x80:
            raise FlacError("bad frame-number continuation byte")
        v = (v << 6) | (c & 0x3F)
    return v, n


def parse_header(data: bytes, p: int, end: int, si: Dict):
    """The frame header at data[p:] -> {var, number, blocksize, assignment, length}; FlacError if it is not a valid,
    CRC-8-correct header that agrees with STREAMINFO (sample rate, channels, bit depth, block size <= max)."""
    if p + 4 > end or data[p] != 0xFF or data[p + 1] & 0xFE != 0xF8:
        raise FlacError(f"no frame sync at byte {p}")
    var = data[p + 1] & 1
    bc, rc = data[p + 2] >> 4, data[p + 2] & 15
    ca, sc, res = data[p + 3] >> 4, (data[p + 3] >> 1) & 7, data[p + 3] & 1
    if bc == 0 or rc == 15 or ca > 10 or sc == 3 or res:
        raise FlacError("reserved value in the frame header")
    if (2 if ca >= 8 else ca + 1) != si["channels"]:
        raise FlacError("frame channel count differs from STREAMINFO")
    if sc and SAMPLE_SIZES[sc] != si["bits_per_sample"]:
        raise FlacError("frame bit depth differs from STREAMINFO")
    number, n = _utf8_read(data, p + 4, end, 7 if var else 6)
    q = p + 4 + n
    extra = (1 if bc == 6 else 2 if bc == 7 else 0) + (1 if rc == 12 else 2 if rc in (13, 14) else 0)
    if q + extra + 1 > end:
        raise FlacError("truncated frame header")
    if bc == 6:
        nb, q = data[q] + 1, q + 1
    elif bc == 7:
        nb, q = int.from_bytes(data[q:q + 2], "big") + 1, q + 2
    else:
        nb = BLOCK_SIZES[bc]
    if rc == 12:
        rate, q = data[q] * 1000, q + 1
    elif rc == 13:
        rate, q = int.from_bytes(data[q:q + 2], "big"), q + 2
    elif rc == 14:
        rate, q = int.from_bytes(data[q:q + 2], "big") * 10, q + 2
    else:
        rate = SAMPLE_RATES.get(rc, si["sample_rate"])
    if rate != si["sample_rate"]:
        raise FlacError("frame sample rate differs from STREAMINFO")
    if crc8(data[p:q]) != data[q]:
        raise FlacError(f"CRC-8 mismatch at byte {p}")
    if nb > si["max_block"]:
        raise FlacError(f"block size {nb} above STREAMINFO's maximum")
    return {"var": var, "number": number, "blocksize": nb, "assignment": ca, "length": q + 1 - p}


def parse_metadata(data: bytes):
    """-> (STREAMINFO dict, offset of the first frame).  Skips an ID3v2 tag and every metadata block."""
    n, pos = len(data), 0
    if data[:3] == b"ID3":
        if n < 10 or any(b & 0x80 for b in data[6:10]):
            raise FlacError("bad ID3v2 header")
        sz = (data[6] << 21) | (data[7] << 14) | (data[8] << 7) | data[9]
        pos = 10 + sz + (10 if data[5] & 0x10 else 0)
    if data[pos:pos + 4] != b"fLaC":
        raise FlacError("no fLaC marker")
    pos += 4
    si, last = None, False
    while not last:
        if pos + 4 > n:
            raise FlacError("truncated metadata")
        last, t, ln = bool(data[pos] & 0x80), data[pos] & 0x7F, int.from_bytes(data[pos + 1:pos + 4], "big")
        if t == 127:
            raise FlacError("metadata block type 127")
        if pos + 4 + ln > n:
            raise FlacError("truncated metadata")
        if si is None:
            if t != 0 or ln != 34:
                raise FlacError("the first metadata block is not a 34-byte STREAMINFO")
            b = data[pos + 4:pos + 38]
            v = int.from_bytes(b[10:18], "big")
            si = {"min_block": int.from_bytes(b[0:2], "big"), "max_block": int.from_bytes(b[2:4], "big"),
                  "sample_rate": v >> 44, "channels": ((v >> 41) & 7) + 1, "bits_per_sample": ((v >> 36) & 31) + 1,
                  "total_samples": v & ((1 << 36) - 1), "md5": bytes(b[18:34])}
        pos += 4 + ln
    if si["sample_rate"] == 0 or si["bits_per_sample"] < 4 or not 16 <= si["min_block"] <= si["max_block"]:
        raise FlacError("bad STREAMINFO")
    return si, pos


def decode(data: bytes, expect=None, check_md5: bool = True) -> Dict:
    """Decode strictly in order -> {"samples": int64 [C, N], "streaminfo", "frames": [{offset, bytes, number,
    blocksize, assignment}]}.  `expect` ([C, N], optional) only speeds up predicted subframes.  Raises FlacError."""
    data = bytes(data)
    si, pos = parse_metadata(data)
    C, bps, total = si["channels"], si["bits_per_sample"], si["total_samples"]
    end = len(data)
    if total == 0 and end - pos >= 128 and data[end - 128:end - 125] == b"TAG":
        end -= 128
    ex = None if expect is None else np.asarray(expect, np.int64).reshape(C, -1)
    outs, frames, done, strategy, block, must_end = [], [], 0, None, None, False
    while (done < total) if total else (pos < end):
        if must_end:
            raise FlacError("a block size changed before the last frame of a fixed-blocksize stream")
        h = parse_header(data, pos, end, si)
        if strategy is None:
            strategy = h["var"]
        if h["var"] != strategy:
            raise FlacError("blocking strategy changed")
        nb = h["blocksize"]
        if h["number"] != (done if strategy else len(frames)):
            raise FlacError(f"frame number {h['number']} out of sequence")
        if total and done + nb > total:
            raise FlacError("frames hold more samples than STREAMINFO says")
        if not strategy:
            if block is None:
                block = nb
            elif nb != block:
                must_end = True
        rd = _Reader(data, pos + h["length"], end)
        ca = h["assignment"]
        chans = []
        for c in range(C):
            side = (ca == 8 and c == 1) or (ca == 9 and c == 0) or (ca == 10 and c == 1)
            e = None
            if ex is not None and ca < 8 and ex.shape[1] >= done + nb:
                e = ex[c, done:done + nb]
            x, _ = _read_subframe(rd, nb, bps + side, e)
            chans.append(x)
        pad = (-rd.p) % 8
        if rd.read(pad):
            raise FlacError("non-zero frame padding")
        fend = pos + h["length"] + rd.p // 8
        if fend + 2 > end:
            raise FlacError("truncated frame")
        if crc16(data[pos:fend]) != int.from_bytes(data[fend:fend + 2], "big"):
            raise FlacError(f"CRC-16 mismatch in the frame at byte {pos}")
        if ca == 8:
            chans = [chans[0], chans[0] - chans[1]]
        elif ca == 9:
            chans = [chans[0] + chans[1], chans[1]]
        elif ca == 10:
            m = (chans[0] << 1) | (chans[1] & 1)
            chans = [(m + chans[1]) >> 1, (m - chans[1]) >> 1]
        blk = np.stack(chans)
        lim = 1 << (bps - 1)
        if blk.size and (blk.min() < -lim or blk.max() >= lim):
            raise FlacError("decoded sample outside the stream's bit depth")
        frames.append({"offset": pos, "bytes": fend + 2 - pos, "number": h["number"], "blocksize": nb,
                       "assignment": ca})
        outs.append(blk)
        done += nb
        pos = fend + 2
    samples = np.concatenate(outs, axis=1) if outs else np.zeros((C, 0), np.int64)
    if check_md5 and si["md5"] != bytes(16) and md5_of(samples, bps) != si["md5"]:
        raise FlacError("MD5 mismatch")
    return {"samples": samples, "streaminfo": {**si, "total_samples": done}, "frames": frames}


# ---------------------------------------------------------------------------------------------------- test matrix
def signal(C: int, n: int, bps: int, seed: int, level: float = 0.5) -> np.ndarray:
    """Speech-like integer test PCM [C, n] in bps bits: a few drifting partials plus a little noise, per channel."""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    out = []
    for c in range(C):
        x = sum(np.sin(2 * np.pi * f * t / 24000 + rng.uniform(0, 6)) * a
                for f, a in ((rng.uniform(90, 200), 0.5), (rng.uniform(300, 900), 0.3), (rng.uniform(1000, 3000), 0.1)))
        x = x * (0.6 + 0.4 * np.sin(2 * np.pi * t / max(n, 1))) + rng.normal(0, 0.01, n)
        out.append(np.clip(np.round(x * level * (2 ** (bps - 1) - 1)), -(2 ** (bps - 1)), 2 ** (bps - 1) - 1))
    return np.asarray(out, np.int64)


def feature_matrix() -> Dict[str, Stream]:
    """Writer streams covering every feature the decoder accepts, by name."""
    m: Dict[str, Stream] = {}
    x = signal(1, 3 * 4096 + 100, 16, 1)
    m["mono16_fixed_orders"] = write_stream(x, 16, 24000, [
        Frame(4096, subs=[Sub("FIXED", order=0, porder=3)]), Frame(4096, subs=[Sub("FIXED", order=1, porder=6)]),
        Frame(4096, subs=[Sub("FIXED", order=3)]), Frame(100, subs=[Sub("FIXED", order=4, porder=2)])])
    x = signal(1, 3 * 4096, 16, 2)
    m["mono16_lpc"] = write_stream(x, 16, 22050, [
        Frame(4096, subs=[Sub("LPC", order=1, precision=12, shift=10)]),
        Frame(4096, subs=[Sub("LPC", order=12, precision=15, shift=13, porder=4)]),
        Frame(4096, subs=[Sub("LPC", order=32, precision=15, shift=14, rice2=True)])])
    x = signal(1, 2 * 4096 + 7, 16, 3)
    m["mono16_constant_verbatim"] = write_stream(np.concatenate([np.full((1, 4096), -1234), x[:, 4096:]], axis=1),
                                                 16, 44100, [Frame(4096, subs=[Sub("CONSTANT")]),
                                                             Frame(4096, subs=[Sub("VERBATIM")]),
                                                             Frame(7, subs=[Sub("VERBATIM")])])
    x = signal(2, 4 * 4096, 16, 4)
    x[1] = (x[0] * 3 + x[1]) // 4
    m["stereo16_assignments"] = write_stream(x, 16, 48000, [
        Frame(4096, a, [Sub("FIXED", order=2, porder=2), Sub("LPC", order=8, shift=11)])
        for a in (INDEPENDENT, LEFT_SIDE, SIDE_RIGHT, MID_SIDE)])
    x = signal(8, 2 * 4096 + 555, 24, 5)
    kinds = [Sub("FIXED", order=c % 5) for c in range(5)] + [Sub("LPC", order=20, precision=14, shift=13),
                                                              Sub("VERBATIM"), Sub("FIXED", order=2, rice2=True)]
    m["ch8_24bit"] = write_stream(x, 24, 96000, [Frame(4096, subs=kinds), Frame(4096, subs=kinds[::-1]),
                                                 Frame(555, subs=kinds)])
    x = signal(2, 4096 * 2, 24, 6)
    m["stereo24_rice2_escape"] = write_stream(x, 24, 48000, [
        Frame(4096, MID_SIDE, [Sub("LPC", order=16, precision=15, shift=14, rice2=True, porder=4, escape={1: 24, 5: 23}),
                               Sub("FIXED", order=2, rice2=True, porder=2, escape={0: 25})]),
        Frame(4096, LEFT_SIDE, [Sub("FIXED", order=1, params=[14]), Sub("FIXED", order=2, rice2=True, params=[29])])])
    z = np.zeros((1, 512), np.int64)
    m["escape_zero_width"] = write_stream(z, 16, 24000, [Frame(512, subs=[Sub("FIXED", order=0, porder=1,
                                                                               escape={0: 0, 1: 0})])])
    big = np.array([[2 ** 31 - 1, -2 ** 31, 5, -7] * 256, [-2 ** 31, 2 ** 31 - 1, -5, 7] * 256], np.int64)
    sm = signal(2, 1024, 32, 7, level=0.25)
    m["stereo32_side"] = write_stream(np.concatenate([big, sm, sm], axis=1), 32, 192000, [
        Frame(1024, LEFT_SIDE, [Sub("VERBATIM"), Sub("VERBATIM")]),
        Frame(1024, MID_SIDE, [Sub("FIXED", order=2, rice2=True), Sub("LPC", order=4, precision=15, shift=14, rice2=True)]),
        Frame(1024, SIDE_RIGHT, [Sub("VERBATIM"), Sub("FIXED", order=1, rice2=True)])])
    for b in (4, 8, 12, 20):
        x = signal(1, 4096 + 50, b, 8 + b)
        m[f"mono{b}bit"] = write_stream(x, b, 16000, [Frame(4096, subs=[Sub("FIXED", order=2)]),
                                                      Frame(50, subs=[Sub("VERBATIM")])])
    x = signal(2, 2 * 4096, 16, 9) * 8
    x[1] = x[0] + 16 * (x[1] // 16 - x[0] // 16)      # a side channel with wasted bits too
    m["wasted_bits"] = write_stream(np.clip(x, -32768, 32767) & ~7, 16, 24000, [
        Frame(4096, LEFT_SIDE, [Sub("FIXED", order=2, wasted=3), Sub("FIXED", order=1, wasted=3)]),
        Frame(4096, INDEPENDENT, [Sub("LPC", order=6, wasted=2, shift=11), Sub("VERBATIM", wasted=3)])])
    sizes = [100, 4096, 17, 1000, 2048, 333]
    x = signal(2, sum(sizes), 16, 10)
    m["variable_blocking"] = write_stream(x, 16, 24000, [
        Frame(s, MID_SIDE if i % 2 else INDEPENDENT, [Sub("FIXED", order=min(2, s - 1))] * 2)
        for i, s in enumerate(sizes)], variable=True)
    x = signal(1, 6 * 256, 16, 11)
    m["header_codes"] = write_stream(x, 16, 32000, [
        Frame(256, bs_code=6, rate_code=12), Frame(256, bs_code=7, rate_code=13), Frame(256, rate_code=14),
        Frame(256, rate_code=0, size_code=0), Frame(256, bs_code=7, rate_code=12), Frame(256, bs_code=6, rate_code=0)])
    x = signal(1, 2 * 4096 + 3, 16, 12)
    fr = [Frame(4096), Frame(4096, subs=[Sub("LPC", order=10, shift=11)]), Frame(3, subs=[Sub("VERBATIM")])]
    meta = [padding(100), vorbis_comment(), seektable(), picture(), unknown_block()]
    m["metadata_id3"] = write_stream(x, 16, 44100, fr, metadata=meta, id3v2=200, id3v1=True)
    m["total_zero_id3v1"] = write_stream(x, 16, 44100, fr, metadata=meta, id3v1=True, total_zero=True)
    m["total_zero_md5_zero"] = write_stream(x, 16, 44100, fr, total_zero=True, md5=False)
    x = signal(1, 32768, 16, 13)
    m["partition_order_15"] = write_stream(x, 16, 24000, [Frame(32768, subs=[Sub("FIXED", order=1, porder=15)])],
                                           max_block=32768)
    x = signal(2, 2 * 65535 + 10, 16, 14)
    m["blocks_65535"] = write_stream(x, 16, 24000, [
        Frame(65535, MID_SIDE, [Sub("FIXED", order=2), Sub("LPC", order=32, precision=15, shift=14)]),
        Frame(65535, INDEPENDENT, [Sub("LPC", order=8, shift=11), Sub("FIXED", order=3)]),
        Frame(10, subs=[Sub("VERBATIM"), Sub("VERBATIM")])], max_block=65535)
    m["false_sync"] = fake_sync_stream(1)
    m["false_sync_crc"] = fake_sync_stream(2)
    return m


def fake_sync_stream(variant: int) -> Stream:
    """Frames of 1024 samples whose VERBATIM payloads hold the next frame's header (variant 2: behind two bytes that
    make the CRC-16 of the frame prefix before them)."""
    x = signal(1, 6 * 1024, 16, 20 + variant)
    fr = [Frame(1024, subs=[Sub("VERBATIM")], fake_sync=variant, fake_at=8 + 100 * i) for i in range(5)]
    return write_stream(x, 16, 24000, fr + [Frame(1024)])
