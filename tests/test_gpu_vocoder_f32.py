"""The vocoder's CUDA-core kernels (csrc/vocoder.cu) launched one at a time through xtts_debug_vocoder, with the arguments
the engine passes, against references of the same operation:

* interp_kernel (every vocoder call, every precision): a float32 emulation of its arithmetic with every fma computed
  exactly, bit for bit; torch CPU's chained F.interpolate (the oracle's z, with or without the speed stage), bit for bit;
  and the fp16 atom image it writes for the tensor-core path.
* conv1d_kernel / conv_transpose1d_kernel (the fp32 parity-mode convolutions): exact-grid data, where every fp32
  accumulation order is exact, bit for bit; Gaussian data at the production scales within a worst-case fp32 bound of a
  float64 reference on the same fp32 activations.
* conv_post_kernel (every vocoder call): float64 tanh of the float64 sum, within the sum's fp32 bound plus two ulps of
  tanhf, item by item of a ragged batch.

Outputs start as sentinels (or as the accumulate base): every element a kernel must not write has to come back unchanged,
bit for bit, and the harness's guard words catch a write past either end of the output."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from auralis_b200.config import VocoderDims, speed_scale
from auralis_b200.native import NativeError, atoms_lpad

import speed_reference as SR

_F32, _F64 = np.float32, np.float64
PADL = 64                                       # head pad rows of an atom image (kAtomPadL)
STORE, ACCUM = 0, 1
VD = VocoderDims()                              # the interpolation ratios are those of both geometries
RB_KD = [(3, 1), (3, 3), (3, 5), (7, 1), (7, 3), (7, 5), (11, 1), (11, 3), (11, 5)]   # resblock (K, dil) pairs
SPEEDS = [1.0, 0.25, 0.5, 0.8, 0.97, 1.3, 2.0, 4.0]
GAUSS_SHARE = {}                                # largest share of the Gaussian error bound used, per op


# ------------------------------------------------------------------------------------------------ exact float32 arithmetic
def _round_f32_exact(q: Fraction) -> np.float32:
    """q rounded to float32, to nearest with ties to even"""
    c = _F32(float(q))
    cands = [np.nextafter(c, _F32(-np.inf)), c, np.nextafter(c, _F32(np.inf))]
    return min(cands, key=lambda v: (abs(Fraction(float(v)) - q), int(np.array(v).view(np.uint32)) & 1))


def fma32(a, b, c):
    """float32 fma(a, b, c), one rounding of the exact a * b + c.  The product of two float32 values is exact in float64;
    the float64 sum rounded to float32 is correct unless the float64 addition rounded (its error term, TwoSum, is not 0)
    and landed on a float32 midpoint, where the second rounding may break the tie the wrong way: those elements are
    recomputed exactly."""
    a, b, c = np.broadcast_arrays(np.asarray(a, _F32), np.asarray(b, _F32), np.asarray(c, _F32))
    p, c64 = a.astype(_F64) * b.astype(_F64), c.astype(_F64)
    s = p + c64
    bb = s - p
    inexact = ((p - (s - bb)) + (c64 - bb)) != 0
    r = s.astype(_F32)
    with np.errstate(invalid="ignore"):
        nb = np.nextafter(r, np.where(s > r, _F32(np.inf), _F32(-np.inf)).astype(_F32))
        mid = inexact & (s != r.astype(_F64)) & ((r.astype(_F64) + nb.astype(_F64)) * 0.5 == s)
    r = np.array(r)
    for idx in zip(*np.nonzero(mid)):
        r[idx] = _round_f32_exact(Fraction(float(a[idx])) * Fraction(float(b[idx])) + Fraction(float(c[idx])))
    return r


def lin_src(dst, r, n):
    """interp_kernel's lin_src: torch's source index fma(r, dst + .5, -.5) clamped below at 0, the two taps (the upper one
    clamped to n - 1) and their weights, all float32"""
    src = fma32(_F32(r), np.asarray(dst).astype(_F32) + _F32(0.5), _F32(-0.5))
    src = np.maximum(src, _F32(0.0))
    i0 = np.minimum(src.astype(np.int64), n - 1)
    i1 = i0 + (i0 < n - 1)
    l1 = (src - i0.astype(_F32)).astype(_F32)
    return i0, i1, (_F32(1.0) - l1).astype(_F32), l1


def lerp(l0, x0, l1, x1):
    """l0 * x0 + l1 * x1 as ATen's CPU kernel rounds it: fma(l0, x0, l1 * x1), per row of x"""
    return fma32(l0[:, None], x0, (l1[:, None] * x1).astype(_F32))


def emulate_z(lat, it, r1, r2):
    """interp_kernel's z for one item: z-frames [z0, z0 + nz) -> [C, nz] float32.  it = (T, T0, T1, z0, nz, r0)."""
    T, T0, T1, z0, nz, r0 = it
    y0 = np.asarray(lat, _F32)[:T]
    if r0 > 0:                                  # the speed stage: T0 time-scaled frames
        c0, c1, p0, p1 = lin_src(np.arange(T0), r0, T)
        y0 = lerp(p0, y0[c0], p1, y0[c1])
    b0, b1, n0, n1 = lin_src(np.arange(T1), r1, y0.shape[0])
    y1 = lerp(n0, y0[b0], n1, y0[b1])
    a0, a1, m0, m1 = lin_src(np.arange(z0, z0 + nz), r2, T1)
    return lerp(m0, y1[a0], m1, y1[a1]).T


def interp_item(T, speed, vd=VD):
    """Engine::interp_item: (T, T0, T1, r0) of a chunk of T latents at `speed`, and its z-frame count"""
    T0, r0, Ty = 0, 0.0, T
    if speed != 1.0 and math.floor(T * speed_scale(speed)) != T:
        ls = speed_scale(speed)
        T0 = Ty = math.floor(T * ls)
        r0 = float(_F32(1.0 / ls))
    resample = vd.output_sample_rate != vd.input_sample_rate
    T1 = math.floor(Ty * (vd.code_stride / vd.output_hop_length)) if resample else Ty
    return T, T0, T1, r0, vd.z_frames(T, speed)


def ratios(vd=VD):
    """the kernel's source steps r1 = (float)(1 / scale1), r2 = (float)(1 / scale2)"""
    s1 = vd.code_stride / vd.output_hop_length
    s2 = vd.output_sample_rate / vd.input_sample_rate if vd.output_sample_rate != vd.input_sample_rate else 1.0
    return _F32(1.0 / s1), _F32(1.0 / s2)


def torch_z(lat, speed, vd=VD):
    """the oracle's z: torch CPU F.interpolate, chained as oracle/xtts_oracle.py and tests/speed_reference.py chain it"""
    return SR.interp_latents(torch.from_numpy(np.asarray(lat, _F32)), vd, speed).numpy()


def length_kept(T, speed, vd=VD):
    """the 24 kHz resample keeps the length (T1 <= 11): torch copies there, the kernel interpolates (DESIGN.md §5)"""
    _, _, T1, _, _ = interp_item(T, speed, vd)
    return math.floor(T1 * (vd.output_sample_rate / vd.input_sample_rate)) == T1


def bits(a):
    return np.asarray(a, _F32).view(np.uint32)


# ------------------------------------------------------------------------------------------------ float64 references
def lrelu32(x, in_scale, slope):
    """the kernels' fused input activation in float32: v = in_scale * x, v > 0 ? v : v * slope"""
    v = (_F32(in_scale) * np.asarray(x, _F32)).astype(_F32)
    return np.where(v > 0, v, (v * _F32(slope)).astype(_F32)).astype(_F32)


def ref_conv(a, w, up=0, dil=1):
    """float64 Conv1d ("same" padding, dilation dil; w [Cout][Cin][K]) or ConvTranspose1d(kernel 2u, stride u, padding
    u/2; w [Cin][Cout][2u]) of a [B][Cin][L]"""
    A, W = torch.from_numpy(np.asarray(a, _F64)), torch.from_numpy(np.asarray(w, _F64))
    if up:
        return F.conv_transpose1d(A, W, stride=up, padding=up // 2).numpy()
    return F.conv1d(A, W, padding=(W.shape[2] - 1) // 2 * dil, dilation=dil).numpy()


# ------------------------------------------------------------------------------------------------ launches
def run_interp(eng, C, items, lats, Lz, atoms=False, fill16=-1234.0):
    """items: (T, T0, T1, z0, nz, r0) per item.  -> (z [B][C][Lz], atom image [B][C/8][lpad][8] or None), both starting
    as sentinels (NaN, fill16)"""
    B = len(items)
    lpad = atoms_lpad(Lz)
    dims = [C, B, Lz, int(atoms), lpad, VD.code_stride, VD.output_hop_length, VD.input_sample_rate, VD.output_sample_rate]
    for T, T0, T1, z0, nz, _ in items:
        dims += [T, T0, T1, z0, nz]
    n32, n16 = B * C * Lz, (B * C * lpad if atoms else 0)
    out = np.concatenate([np.full(n32, np.nan, _F32), np.full(n16, fill16, _F32)])
    got = eng.debug_vocoder("INTERP", dims, lats, out=out, scal=[it[5] for it in items])
    z = got[:n32].reshape(B, C, Lz)
    return z, (got[n32:].reshape(B, C // 8, lpad, 8) if atoms else None)


def check_interp(eng, C, cases, Lz=None, atoms=False, torch_parity=False, seed=0):
    """cases: (T, speed, z0, nz or None = the whole chunk).  One launch; every item's columns < nz equal the emulation bit
    for bit (and the torch chain's, torch_parity), columns >= nz keep their NaN, the atom image holds fp16_rn(z) at rows
    64 + j < 64 + nz and its sentinel everywhere else."""
    rng = np.random.RandomState(seed)
    r1, r2 = ratios()
    items, lats = [], []
    for T, speed, z0, nz in cases:
        _, T0, T1, r0, nzf = interp_item(T, speed)
        items.append((T, T0, T1, z0, nzf - z0 if nz is None else nz, r0))
        lats.append(rng.randn(T, C).astype(_F32))
    Lz = Lz or max(it[4] for it in items)
    z, img = run_interp(eng, C, items, lats, Lz, atoms)
    for i, (it, lat, (T, speed, _, _)) in enumerate(zip(items, lats, cases)):
        nz = it[4]
        ctx = f"item {i}: T={T} speed={speed} z0={it[3]} nz={nz} C={C}"
        want = emulate_z(lat, it, r1, r2)
        np.testing.assert_array_equal(bits(z[i, :, :nz]), bits(want), err_msg=ctx)
        assert np.isnan(z[i, :, nz:]).all() and (bits(z[i, :, nz:]) == bits(_F32(np.nan))).all(), ctx
        if torch_parity:
            tz = torch_z(lat, speed)[:, it[3]:it[3] + nz]
            assert tz.shape == want.shape, ctx
            np.testing.assert_array_equal(bits(z[i, :, :nz]), bits(tz), err_msg=ctx)
        if atoms:
            exp = np.full(img.shape[1:], -1234.0, _F32)
            exp[:, PADL:PADL + nz, :] = want.astype(np.float16).astype(_F32).reshape(C // 8, 8, nz).transpose(0, 2, 1)
            np.testing.assert_array_equal(img[i], exp, err_msg=ctx)
    return z


def run_conv(eng, seed, Cin, Cout, L, K=3, dil=1, up=0, B=1, exact=True, mode=STORE, bias=True, cbias=True, resid=True,
             in_scale=None, slope=None):
    """One CONV1D (up 0) or CONV_T launch against the float64 reference: exact grid bit for bit, Gaussian within the fp32
    accumulation bound."""
    rng = np.random.RandomState(seed)
    Kw = 2 * up if up else K
    Lout = L * up if up else L
    wshape = (Cin, Cout, Kw) if up else (Cout, Cin, Kw)
    cb_stride = Cout + 5                        # speaker-bias rows are strided wider than Cout in the engine
    if exact:
        in_scale = 0.5 if in_scale is None else in_scale
        slope = 0.125 if slope is None else slope
        x = rng.randint(-16, 17, (B, Cin, L)) / 16.0
        w = rng.randint(-16, 17, wshape) / 16.0
        small = lambda shape: rng.randint(-64, 65, shape) / 256.0
        big = lambda shape: rng.randint(-256, 257, shape) / 256.0
    else:
        in_scale = 1.0 / 3.0 if in_scale is None else in_scale
        slope = 0.1 if slope is None else slope
        x = rng.randn(B, Cin, L)
        w = 0.02 * rng.randn(*wshape)
        small = lambda shape: 0.1 * rng.randn(*shape)
        big = lambda shape: rng.randn(*shape)
    x, w = x.astype(_F32), w.astype(_F32)
    b = small((Cout,)).astype(_F32) if bias else None
    cb = small((B, cb_stride)).astype(_F32) if cbias else None
    r = big((B, Cout, Lout)).astype(_F32) if (resid and not up) else None
    base = big((B, Cout, Lout)).astype(_F32) if mode == ACCUM else np.full((B, Cout, Lout), np.nan, _F32)
    ins = [x, w] + [a for a in (b, cb, r) if a is not None]
    if up:
        dims = [Cin, Cout, up, Kw, L, B, int(b is not None), int(cb is not None), cb_stride]
        got = eng.debug_vocoder("CONV_T", dims, ins, out=base, scal=[in_scale, slope])
    else:
        dims = [Cin, Cout, K, dil, L, B, mode, int(b is not None), int(cb is not None), cb_stride, int(r is not None)]
        got = eng.debug_vocoder("CONV1D", dims, ins, out=base, scal=[in_scale, slope])
    got = got.reshape(B, Cout, Lout)

    a = lrelu32(x, in_scale, slope)
    v = ref_conv(a, w, up, dil)
    absv = ref_conv(np.abs(a), np.abs(w), up, dil)
    n_terms = Cin * (2 if up else K)
    for add in (b[None, :, None] if b is not None else None, cb[:, :Cout, None] if cb is not None else None, r,
                base if mode == ACCUM else None):
        if add is not None:
            v, absv, n_terms = v + add, absv + np.abs(add), n_terms + 1
    ctx = f"Cin={Cin} Cout={Cout} K={Kw} dil={dil} up={up} L={L} B={B} mode={mode} exact={exact}"
    assert np.isfinite(got).all(), ctx
    if exact:
        assert absv.max() < 2.0 ** 12, ctx          # multiples of 2^-12 below 2^12: every partial sum exact in fp32
        np.testing.assert_array_equal(got, v.astype(_F32), err_msg=ctx)
        assert np.array_equal(v.astype(_F32).astype(_F64), v), "reference not exact in fp32"
        return got
    bound = n_terms * 2.0 ** -23 * absv
    share = float((np.abs(got.astype(_F64) - v) / (bound + 1e-300)).max())
    key = "conv_t" if up else "conv1d"
    GAUSS_SHARE[key] = max(GAUSS_SHARE.get(key, 0.0), share)
    print("gaussian bound share", ctx, GAUSS_SHARE)
    assert share <= 1.0, (ctx, share)
    return got


def run_post(eng, seed, Cin, L, lens=None, B=None, wav_stride=None, in_scale=1.0 / 3.0, slope=0.01, K=7):
    """One CONV_POST launch: x past each item's length is NaN (a read of it reaches a stored sample), wav starts as NaN
    sentinels; samples t < L_i within the bound of float64 tanh of the float64 sum, every other sample untouched."""
    rng = np.random.RandomState(seed)
    lens_given = lens is not None
    lens = list(lens) if lens_given else [L] * B
    B = len(lens)
    ws = wav_stride or L
    x = (3.0 * rng.randn(B, Cin, L)).astype(_F32)
    for i, n in enumerate(lens):
        x[i, :, n:] = np.nan
    w = (0.3 * rng.randn(Cin, K)).astype(_F32)
    dims = [Cin, K, L, B, ws, int(lens_given)] + (lens if lens_given else [])
    got = eng.debug_vocoder("CONV_POST", dims, [x, w], out=np.full(B * ws, np.nan, _F32), scal=[in_scale, slope])
    got = got.reshape(B, ws)
    for i, n in enumerate(lens):
        ctx = f"Cin={Cin} L={L} item {i} len={n} wav_stride={ws}"
        assert (bits(got[i, n:]) == bits(_F32(np.nan))).all(), ctx
        if n == 0:
            continue
        a = lrelu32(np.nan_to_num(x[i:i + 1, :, :n]), in_scale, slope)
        S = ref_conv(a, w[None], 0, 1)[0, 0]
        E = (Cin * K) * 2.0 ** -23 * ref_conv(np.abs(a), np.abs(w[None]), 0, 1)[0, 0]
        t = np.tanh(S)
        ulp = np.spacing(np.abs(t).astype(_F32)).astype(_F64)
        assert np.isfinite(got[i, :n]).all(), ctx
        err = np.abs(got[i, :n].astype(_F64) - t)
        share = float((err / (E + 2 * ulp)).max(initial=0.0))
        GAUSS_SHARE["conv_post"] = max(GAUSS_SHARE.get("conv_post", 0.0), share)
        assert share <= 1.0, (ctx, share)
    return got


# ------------------------------------------------------------------------------------------------ CPU: the references
def test_fma32_is_exact():
    """fma32 against exact rational arithmetic, including exact float32 ties and sums whose float64 rounding lands on a
    float32 midpoint: (1 + 2^-12)^2 = 1 + 2^-11 + 2^-24 is the midpoint between 1 + 2^-11 and its successor, and
    +-2^-80 decides the rounding but is lost in float64"""
    rng = np.random.RandomState(0)
    a, b, c = (rng.randn(3, 4000) * np.array([[1.0], [1.0], [1e-3]])).astype(_F32)
    one, h = _F32(1.0), _F32(1.0 + 2.0 ** -12)
    a = np.concatenate([a, [one + _F32(2.0 ** -23), h, h, h, _F32(1.5)]]).astype(_F32)
    b = np.concatenate([b, [one + _F32(2.0 ** -23), h, h, h, one + _F32(2.0 ** -23)]]).astype(_F32)
    c = np.concatenate([c, [-one, _F32(2.0 ** -80), _F32(-2.0 ** -80), _F32(0.0), _F32(2.0 ** -30)]]).astype(_F32)
    got = fma32(a, b, c)
    assert got[-4] == _F32(1.0 + 2.0 ** -11 + 2.0 ** -23) and got[-3] == _F32(1.0 + 2.0 ** -11)
    for i in range(a.size):
        assert got[i] == _round_f32_exact(Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))), i


def test_round_f32_ties_to_even():
    lo = Fraction(1) + Fraction(1, 2 ** 24)                   # halfway between 1 and 1 + 2^-23: even is 1
    hi = Fraction(1) + Fraction(3, 2 ** 24)                   # halfway between 1 + 2^-23 and 1 + 2^-22: even is the latter
    assert _round_f32_exact(lo) == _F32(1.0)
    assert _round_f32_exact(hi) == _F32(1.0 + 2.0 ** -22)


@pytest.mark.parametrize("speed", SPEEDS)
def test_emulation_equals_torch_interpolate(speed):
    """the float32 emulation of interp_kernel equals torch CPU's chained F.interpolate bit for bit wherever the 24 kHz
    resample changes the length; where it keeps it, torch copies and the two differ only there"""
    rng = np.random.RandomState(int(speed * 100))
    r1, r2 = ratios()
    for T in [1, 2, 3, 5, 23, 96, 605]:
        lat = rng.randn(T, 128).astype(_F32)
        _, T0, T1, r0, nzf = interp_item(T, speed)
        if nzf == 0:
            continue
        want = torch_z(lat, speed)
        got = emulate_z(lat, (T, T0, T1, 0, nzf, r0), r1, r2)
        assert got.shape == want.shape
        if length_kept(T, speed):
            continue
        np.testing.assert_array_equal(bits(got), bits(want), err_msg=f"T={T} speed={speed}")


def test_emulation_window_is_the_slice():
    """a window's z-frames are evaluated at their global index, so a window is the slice of the whole chunk"""
    rng = np.random.RandomState(3)
    r1, r2 = ratios()
    lat = rng.randn(40, 16).astype(_F32)
    for speed in (1.0, 0.5, 2.0):
        T, T0, T1, r0, nzf = interp_item(40, speed)
        whole = emulate_z(lat, (T, T0, T1, 0, nzf, r0), r1, r2)
        np.testing.assert_array_equal(emulate_z(lat, (T, T0, T1, 17, 33, r0), r1, r2), whole[:, 17:50])


@pytest.mark.parametrize("K,dil", [(3, 1), (7, 3), (11, 5)])
def test_reference_conv_matches_loop(K, dil):
    rng = np.random.RandomState(K)
    B, Cin, Cout, L = 2, 3, 4, 13
    x, w = rng.randn(B, Cin, L), rng.randn(Cout, Cin, K)
    want = np.zeros((B, Cout, L))
    c = (K - 1) // 2
    for b in range(B):
        for t in range(L):
            for j in range(K):
                s = t + (j - c) * dil
                if 0 <= s < L:
                    want[b, :, t] += w[:, :, j] @ x[b, :, s]
    np.testing.assert_allclose(ref_conv(x, w, 0, dil), want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("u", [2, 4, 8])
def test_reference_conv_transpose_matches_loop(u):
    """ConvTranspose1d(kernel 2u, stride u, padding u/2): x[s] * w[k] lands on t = s*u + k - u/2, t < L*u"""
    rng = np.random.RandomState(u)
    B, Cin, Cout, L = 2, 3, 4, 5
    x, w = rng.randn(B, Cin, L), rng.randn(Cin, Cout, 2 * u)
    want = np.zeros((B, Cout, L * u))
    for b in range(B):
        for s in range(L):
            for k in range(2 * u):
                t = s * u + k - u // 2
                if 0 <= t < L * u:
                    want[b, :, t] += x[b, :, s] @ w[:, :, k]
    np.testing.assert_allclose(ref_conv(x, w, u, 1), want, rtol=1e-12, atol=1e-12)


def test_exact_grid_is_exact():
    """grid activations (k/16 times 1/2, times 1/8 when negative) times grid weights k/16 are multiples of 2^-12, and so
    are the biases; conv_pre's 1024 x 7 products of at most 1/2 and four addends of at most 1 stay below 2^12"""
    k = np.arange(-16, 17) / 16.0
    a = lrelu32(k, 0.5, 0.125).astype(_F64)
    prod = np.outer(a, k)
    assert np.array_equal(np.round(prod * 2 ** 12), prod * 2 ** 12)
    assert 1024 * 7 * 0.5 + 4 < 2 ** 12


# ------------------------------------------------------------------------------------------------ GPU: INTERP
@pytest.mark.gpu
@pytest.mark.parametrize("C", [128, 1024])
def test_interp_equals_emulation_and_torch(engine_small, C):
    """whole chunks at speed 1 and at speeds on both sides of it, one launch per speed: bit for bit the emulation, and the
    chained torch F.interpolate (the oracle's z) wherever the 24 kHz resample changes the length"""
    Ts = [1, 2, 3, 5, 23, 96, 605] if C == 128 else [3, 23, 605]
    for k, speed in enumerate(SPEEDS):
        cases = [(T, speed, 0, None) for T in Ts if interp_item(T, speed)[4] > 0]
        parity = [c for c in cases if not length_kept(c[0], speed)]
        kept = [c for c in cases if length_kept(c[0], speed)]
        check_interp(engine_small, C, parity, torch_parity=True, seed=k)
        if kept:
            check_interp(engine_small, C, kept, seed=k)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [128, 1024])
def test_interp_window_is_the_slice(engine_small, C):
    """a window (z0 > 0, nz short of the whole) equals the matching slice of the whole chunk's z"""
    rng = np.random.RandomState(C)
    r1, r2 = ratios()
    for speed in (1.0, 0.5, 3.0):
        T, T0, T1, r0, nzf = interp_item(150, speed)
        lat = rng.randn(T, C).astype(_F32)
        whole, _ = run_interp(engine_small, C, [(T, T0, T1, 0, nzf, r0)], [lat], nzf)
        for z0, nz in [(1, 31), (37, 100), (nzf - 45, 45), (200, 65)]:
            z0 = min(z0, nzf - nz)
            win, _ = run_interp(engine_small, C, [(T, T0, T1, z0, nz, r0)], [lat], nz)
            np.testing.assert_array_equal(bits(win[0]), bits(whole[0, :, z0:z0 + nz]), err_msg=f"speed={speed} z0={z0}")
        np.testing.assert_array_equal(bits(whole[0]), bits(emulate_z(lat, (T, T0, T1, 0, nzf, r0), r1, r2)))


@pytest.mark.gpu
@pytest.mark.parametrize("C", [128, 1024])
def test_interp_ragged_batch_and_atoms(engine_small, C):
    """32 items of mixed T, speed and window, nz not a multiple of 32, nz = Lz and nz = 0 among them, z32 and the fp16
    atom image (rows 64 + j) in one launch, as the tensor-core vocoder issues it"""
    rng = np.random.RandomState(7)
    Lz = 437
    cases = []
    for i in range(32):
        T = int(rng.randint(1, 140))
        speed = SPEEDS[i % len(SPEEDS)]
        nzf = interp_item(T, speed)[4]
        if nzf == 0:
            T, speed, nzf = 30, 1.0, interp_item(30, 1.0)[4]
        z0 = int(rng.randint(0, max(1, nzf - 20)))
        nz = int(min(Lz, nzf - z0, rng.randint(1, Lz + 1)))
        cases.append((T, speed, z0, nz))
    cases[3] = (120, 0.5, 10, Lz)               # nz = Lz
    cases[9] = (100, 1.0, 0, Lz)
    cases[17] = (50, 1.0, 5, 0)                 # an empty window
    cases[20] = (60, 2.0, 3, 33)
    check_interp(engine_small, C, cases, Lz=Lz, atoms=True)


# ------------------------------------------------------------------------------------------------ GPU: CONV1D
CONV_SHAPES = [(128, 64, 7, 1), (1024, 512, 7, 1), (256, 256, 11, 5)] + [(C, C, K, d) for C in (64, 32) for K, d in RB_KD] + \
              [(32, 16, 3, 1), (16, 8, 11, 5)]


@pytest.mark.gpu
@pytest.mark.parametrize("Cin,Cout,K,dil", CONV_SHAPES)
def test_conv1d_production_shapes(engine_small, Cin, Cout, K, dil):
    """conv_pre and every resblock (K, dil) at the fp32 path's channel counts (Cout > 32: 64-channel blocks; <= 32:
    32-channel blocks): two items with their own speaker bias, bias + residual, exact grid and Gaussian"""
    L = 300 if Cin >= 512 else 700
    run_conv(engine_small, Cin + K + dil, Cin, Cout, L, K, dil, B=2)
    run_conv(engine_small, Cin + K + dil + 1, Cin, Cout, L, K, dil, B=2, exact=False)


@pytest.mark.gpu
@pytest.mark.parametrize("K,dil", [(3, 1), (7, 5), (11, 5)])
def test_conv1d_lengths_and_ragged_channels(engine_small, K, dil):
    """L below the halo, at the 128-step tile edge and across several tiles; Cout not a multiple of 8 on both block
    shapes and Cin not a multiple of the 8 staged input channels"""
    for L in [1, 2, (K - 1) // 2 * dil - 1, 127, 128, 129, 300, 513]:
        if L >= 1:
            run_conv(engine_small, L, 32, 32, L, K, dil)
    for Cin, Cout in [(32, 37), (64, 70), (13, 64), (13, 5), (100, 29)]:
        run_conv(engine_small, Cin * Cout, Cin, Cout, 129, K, dil, B=3)
        run_conv(engine_small, Cin * Cout + 1, Cin, Cout, 129, K, dil, B=3, exact=False)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [STORE, ACCUM], ids=["store", "accum"])
def test_conv1d_epilogue(engine_small, mode):
    """STORE and ACCUM with bias, speaker bias (stride > Cout, one row per item) and residual each present and absent"""
    seed = 0
    for bias in (False, True):
        for cbias in (False, True):
            for resid in (False, True):
                seed += 1
                run_conv(engine_small, seed, 64, 64, 200, 7, 3, B=3, mode=mode, bias=bias, cbias=cbias, resid=resid)
    run_conv(engine_small, 99, 32, 32, 200, 11, 5, B=3, mode=mode, exact=False)


# ------------------------------------------------------------------------------------------------ GPU: CONV_T
CONVT = [(512, 256, 8), (256, 128, 8), (128, 64, 2), (64, 32, 2),          # the full geometry's upsamplers
         (64, 32, 8), (32, 16, 8), (16, 8, 2), (8, 4, 2),                   # the small geometry's
         (32, 20, 4)]                                                       # Cout not a multiple of 16


@pytest.mark.gpu
@pytest.mark.parametrize("Cin,Cout,u", CONVT)
def test_conv_transpose(engine_small, Cin, Cout, u):
    """every upsampler; Lin at the 128-step output tile's edges (128 / u - 1, 128 / u, 128 / u + 1) and several tiles;
    in_scale 1 (the first stage) and 1/3 (the later ones)"""
    edge = 128 // u
    for Lin in [1, edge - 1, edge, edge + 1, 3 * edge + 5]:
        if Lin >= 1:
            run_conv(engine_small, Lin, Cin, Cout, Lin, up=u, B=2, in_scale=1.0)
    run_conv(engine_small, 97, Cin, Cout, 3 * edge + 5, up=u, B=2, exact=False, in_scale=1.0)
    run_conv(engine_small, 98, Cin, Cout, edge + 1, up=u, B=2, exact=False)
    run_conv(engine_small, 99, Cin, Cout, edge + 1, up=u, B=2, bias=False, cbias=False)


# ------------------------------------------------------------------------------------------------ GPU: CONV_POST
@pytest.mark.gpu
@pytest.mark.parametrize("Cin", [4, 32])
def test_conv_post(engine_small, Cin):
    """the small and full geometry's last stage: equal lengths at and around the 256-sample block edge, and ragged
    batches with lengths 0 and L, row stride L and a wider wav_stride"""
    for L in [1, 3, 255, 256, 257, 1000]:
        run_post(engine_small, L, Cin, L, B=2)
    rng = np.random.RandomState(Cin)
    L = 2048
    lens = [L, 0, 1, 255, 256, 257, L - 1] + list(rng.randint(0, L + 1, 24)) + [0]
    run_post(engine_small, 1, Cin, L, lens=lens)
    run_post(engine_small, 2, Cin, L, lens=lens, wav_stride=L + 77)
    run_post(engine_small, 3, Cin, 300, lens=[300, 0, 120], wav_stride=512, in_scale=1.0)


# ------------------------------------------------------------------------------------------------ GPU: rejections
@pytest.mark.gpu
def test_rejections_leave_the_engine_usable(engine_small):
    """arguments the kernels cannot take are refused on the host, before anything launches"""
    e = engine_small
    x = np.zeros((1, 8, 40), _F32)
    conv = lambda Cin=8, Cout=8, K=3, dil=1, L=40, B=1: [Cin, Cout, K, dil, L, B, STORE, 0, 0, 0, 0]
    w3 = np.zeros((8, 8, 3), _F32)
    it = [8, 1, 40, 0, 0, 1024, 256, 22050, 24000]
    bad = [
        (7, conv(), [x, w3], 320, [1.0, 0.1]),                                             # unknown op
        ("CONV1D", conv(B=33), [np.zeros((33, 8, 40)), w3], 33 * 320, [1.0, 0.1]),         # 33 items
        ("CONV1D", conv(B=0), [x, w3], 320, [1.0, 0.1]),                                   # 0 items
        ("INTERP", it[:2] + [10] + it[3:] + [4, 0, 16, 0, 11], [np.zeros((4, 8))], 80, [0.0]),  # nz > Lz
        ("CONV1D", conv(K=5), [x, np.zeros((8, 8, 5))], 320, [1.0, 0.1]),                  # K 5
        ("CONV_T", [8, 8, 4, 6, 40, 1, 0, 0, 0], [x, np.zeros((8, 8, 6))], 1280, [1.0, 0.1]),   # K != 2u
        ("CONV_T", [8, 8, 3, 6, 40, 1, 0, 0, 0], [x, np.zeros((8, 8, 6))], 960, [1.0, 0.1]),    # u odd
        ("CONV_T", [8, 8, 6, 12, 40, 1, 0, 0, 0], [x, np.zeros((8, 8, 12))], 1920, [1.0, 0.1]), # u not dividing 128
        ("CONV_POST", [8, 7, 40, 2, 40, 1, 40, 41], [np.zeros((2, 8, 40)), np.zeros((8, 7))], 80, [1.0, 0.01]),
        ("CONV1D", conv(), [x, w3[:, :, :2]], 320, [1.0, 0.1]),                            # weight length
        ("CONV1D", conv(), [x, w3], 321, [1.0, 0.1]),                                      # out length
        ("CONV1D", conv(), [x], 320, [1.0, 0.1]),                                          # missing input
        ("CONV_POST", [8, 7, 40, 1, 39, 0], [x, np.zeros((8, 7))], 39, [1.0, 0.01]),       # wav_stride < L
        ("INTERP", [12, 1, 40, 1, 64 + 40] + it[5:] + [4, 0, 16, 0, 40], [np.zeros((4, 12))], 40 * 12 + 12 * 104, [0.0]),
    ]
    e.debug_vocoder("CONV_POST", [8, 7, 40, 1, 40, 0], [x, np.zeros((8, 7))], out_len=40, scal=[1.0, 0.01])   # valid
    for i, (op, dims, ins, n_out, scal) in enumerate(bad):
        with pytest.raises(NativeError):
            e.debug_vocoder(op, dims, ins, out_len=n_out, scal=scal)
            pytest.fail(f"case {i} ({op}) was accepted")
    run_conv(e, 5, 16, 24, 50, 3, 1)
