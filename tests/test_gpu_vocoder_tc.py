"""The fast-mode vocoder convolution (conv1d_tc_kernel: every Conv1d of the vocoder, and every ConvTranspose1d as u
two-tap phases) launched on its own through xtts_debug_conv_tc and compared with a float64 torch reference of the same
operation on the fp16-rounded operands.

Exact-grid data: x and w are k/16 with |k| <= 32 (exact in fp16); bias, speaker bias, residual and accumulate base are
multiples of 2^-8.  Every product is then a multiple of 2^-8 and every partial sum stays below 2^15, so every fp32
accumulation order is exact: out32 and the fp16 output atom image must equal the reference bit for bit.  One wrong tap,
channel, row or bias changes a value and fails.  Gaussian data at the vocoder's magnitudes checks the same launches
against a worst-case fp32 error bound.

The input atom image is NaN outside each item's signal until the production pad routine clears the rows it claims the
kernel reads, and the outputs start as NaN sentinels (or as the accumulate base): a read outside the cleared rows reaches
a stored output as NaN, and a write outside [0, Lout_i) changes a sentinel."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from auralis_b200.native import NativeEngine, NativeError, atoms_lpad

PADL = 64                                       # head pad rows of an atom image (kAtomPadL)
STORE, ACCUM = NativeEngine.CONV_STORE, NativeEngine.CONV_ACCUM
SLOPE = 0.1                                     # leaky-ReLU slope of the vocoder
RB_KD = [(3, 1), (3, 3), (7, 5), (11, 5), (11, 1)]     # resblock (kernel, dilation) pairs of the full geometry
CONVT = [(512, 256, 8), (256, 128, 8), (128, 64, 2), (64, 32, 2), (64, 32, 4)]   # (Cin, Cout, u) of the upsamplers
_F64, _F32 = np.float64, np.float32
GAUSS_SHARE = {}                                # largest share of the Gaussian error bound used, per output


def tile_rows(Cout_gemm):
    """time rows per tile of conv1d_tc_plan: 128 * MB, MB = 1 / 2 / 4 for N = 256 / 128 / <= 64"""
    N = min(Cout_gemm, 256)
    return 128 * (1 if N >= 256 else 2 if N >= 128 else 4)


# ------------------------------------------------------------------------------------------------ references
def f16(a):
    """fp32 values rounded to fp16 (round to nearest even), as float64"""
    return np.asarray(a, _F32).astype(np.float16).astype(_F64)


def ref_conv(x, w, up, dil, lens):
    """float64 Conv1d ("same" padding, dilation dil) or ConvTranspose1d(kernel 2u, stride u, padding u/2) of item i's
    x[:, :L_i] with zeros beyond -> [B, Cout, Lout], rows >= Lout_i zero."""
    xz = np.array(x, _F64)
    for b, n in enumerate(lens):
        xz[b, :, n:] = 0.0
    X, W = torch.from_numpy(xz), torch.from_numpy(np.asarray(w, _F64))
    if up:
        y = F.conv_transpose1d(X, W, stride=up, padding=up // 2).numpy()
    else:
        K = W.shape[2]
        y = F.conv1d(X, W, padding=(K - 1) // 2 * dil, dilation=dil).numpy()
    for b, n in enumerate(lens):
        y[b, :, n * (up or 1):] = 0.0
    return y


def emulate16(v32, scale16):
    """out16 = fp16_rn(lrelu(v * scale16, slope)) in fp32 arithmetic, as the kernel's epilogue computes it"""
    v = np.asarray(v32, _F32) * _F32(scale16)
    v = np.where(v > 0, v, v * _F32(SLOPE))
    return v.astype(np.float16).astype(_F32)


def to_atoms(v, lpad, fill=np.nan):
    """[B, C, n] -> atom image [B, C/8, lpad, 8], signal at rows PADL .. PADL + n, `fill` elsewhere"""
    B, C, n = v.shape
    img = np.full((B, C // 8, lpad, 8), fill, _F32)
    img[:, :, PADL:PADL + n, :] = np.asarray(v, _F32).reshape(B, C // 8, 8, n).transpose(0, 1, 3, 2)
    return img


def from_atoms(img, n):
    """atom image [B, C/8, lpad, 8] -> [B, C, n] (rows PADL .. PADL + n)"""
    B, P = img.shape[:2]
    return np.ascontiguousarray(img[:, :, PADL:PADL + n, :].transpose(0, 1, 3, 2)).reshape(B, P * 8, n)


def exact_sum_bound(n_products, n_addends):
    """largest |partial sum| of exact-grid data: n products of |x|, |w| <= 2, plus addends of magnitude <= 1/4"""
    return n_products * 2.0 * 2.0 + n_addends * 0.25


# ------------------------------------------------------------------------------------------------ one checked launch
def run_case(eng, seed, Cin, Cout, L, K=3, dil=1, up=0, lens=None, B=None, exact=True, mode=STORE, resid=True,
             bias=True, cbias=True, want32=True, want16=True, scale16=1.0, max_ctas=0, ragged=None):
    """Launch once and check every output row against the reference: stored rows equal (exact grid) or within the fp32
    bound (Gaussian), no stored value NaN, every other row keeps its sentinel.  -> (out32, out16) as returned."""
    rng = np.random.RandomState(seed)
    if lens is None:
        lens = [L] * (B or 1)
    B = len(lens)
    ragged = any(n != L for n in lens) if ragged is None else ragged
    Kw = 2 * up if up else K
    n_prod = Cin * (2 if up else K)              # products per output: a transposed-conv phase has two taps
    Lout = L * up if up else L
    lpad_out = atoms_lpad(Lout)
    wshape = (Cin, Cout, Kw) if up else (Cout, Cin, Kw)
    cb_stride = Cout + 5                         # speaker-bias rows are strided wider than Cout in the engine
    f32 = lambda a: np.asarray(a, _F32).astype(_F64)            # the fp32 values the kernel is handed
    if exact:
        x = rng.randint(-32, 33, (B, Cin, L)) / 16.0
        w = rng.randint(-32, 33, wshape) / 16.0
        small = big = lambda shape: rng.randint(-64, 65, shape) / 256.0
    else:
        x = rng.randn(B, Cin, L)
        w = 0.02 * rng.randn(*wshape)
        small = lambda shape: f32(0.1 * rng.randn(*shape))
        big = lambda shape: f32(rng.randn(*shape))
    base = big((B, Cout, Lout))
    b = small((Cout,)) if bias else None
    cb = small((B, cb_stride)) if cbias else None
    r = big((B, Cout, Lout)) if resid else None
    if exact:
        n_add = 1 + (b is not None) + (cb is not None) + (r is not None) + (mode == ACCUM)
        assert exact_sum_bound(n_prod, n_add) < 2.0 ** 15, (Cin, Kw)
        for a in (x, w):
            assert np.array_equal(f16(a), a)
    in32 = (base.astype(_F32) if mode == ACCUM else np.full((B, Cout, Lout), np.nan, _F32)) if want32 else None
    in16 = np.full((B, Cout // 8, lpad_out, 8), np.nan, _F32) if want16 else None
    got32, got16 = eng.debug_conv_tc(x, w, up=up, dil=dil, item_len=lens if ragged else None, bias=b, cbias=cb,
                                      resid=r, mode=mode, slope_out=SLOPE, scale16=scale16, max_ctas=max_ctas,
                                      out32=in32, out16=in16)

    xr, wr = f16(x), f16(w)
    v = ref_conv(xr, wr, up, dil, lens)
    absv = ref_conv(np.abs(xr), np.abs(wr), up, dil, lens)
    for add in (b[None, :, None] if b is not None else None, cb[:, :Cout, None] if cb is not None else None, r,
                base if mode == ACCUM else None):
        if add is not None:
            v = v + add
            absv = absv + np.abs(add)
    stored = np.zeros((B, Cout, Lout), bool)
    for i, n in enumerate(lens):
        stored[i, :, :n * (up or 1)] = True
    stored16 = np.zeros((B, Cout // 8, lpad_out, 8), bool)
    if want16:
        stored16[:] = np.isfinite(to_atoms(np.where(stored, 0.0, np.nan), lpad_out))
    ctx = f"Cin={Cin} Cout={Cout} K={Kw} dil={dil} up={up} L={L} lens={lens} mode={mode} scale16={scale16}"

    if exact:
        v32 = v.astype(_F32)
        assert np.array_equal(v32.astype(_F64)[stored], v[stored]), "reference not exact in fp32"
        if want32:
            exp32 = np.where(stored, v32, in32)
            assert np.isfinite(got32[stored]).all(), ctx
            np.testing.assert_array_equal(got32, exp32, err_msg=ctx)
        if want16:
            exp16 = np.where(stored16, to_atoms(emulate16(v32, scale16), lpad_out), in16)
            assert np.isfinite(got16[stored16]).all(), ctx
            np.testing.assert_array_equal(got16, exp16, err_msg=ctx)
        return got32, got16

    n_terms = n_prod + 4
    bound32 = n_terms * 2.0 ** -23 * absv
    if want32:
        assert np.isfinite(got32[stored]).all(), ctx
        np.testing.assert_array_equal(got32[~stored], in32[~stored], err_msg=ctx)
        err = np.abs(got32.astype(_F64) - v)[stored]
        share = float((err / (bound32[stored] + 1e-300)).max(initial=0.0))
        GAUSS_SHARE["out32"] = max(GAUSS_SHARE.get("out32", 0.0), share)
        assert share <= 1.0, (ctx, share)
    if want16:
        assert np.isfinite(got16[stored16]).all(), ctx
        np.testing.assert_array_equal(got16[~stored16], in16[~stored16], err_msg=ctx)
        s = float(_F32(scale16))
        a = v * s
        ref16 = np.where(a > 0, a, a * float(_F32(SLOPE)))
        bound16 = s * bound32 + np.abs(ref16) * (2.0 ** -11 + 2.0 ** -22) + 2.0 ** -25
        g16 = from_atoms(got16, Lout).astype(_F64)
        err = np.abs(g16 - ref16)[stored]
        share = float((err / bound16[stored]).max(initial=0.0))
        GAUSS_SHARE["out16"] = max(GAUSS_SHARE.get("out16", 0.0), share)
        assert share <= 1.0, (ctx, share)
    print("gaussian bound share", ctx, GAUSS_SHARE)
    return got32, got16


# ------------------------------------------------------------------------------------------------ CPU: the references
@pytest.mark.parametrize("K,dil", [(1, 1), (3, 1), (3, 3), (5, 2)])
def test_reference_conv_matches_loop(K, dil):
    rng = np.random.RandomState(K * 10 + dil)
    B, Cin, Cout, L = 2, 3, 4, 9
    x, w = rng.randn(B, Cin, L), rng.randn(Cout, Cin, K)
    lens = [L, 6]
    want = np.zeros((B, Cout, L))
    c = (K - 1) // 2
    for b in range(B):
        for t in range(lens[b]):
            for j in range(K):
                s = t + (j - c) * dil
                if 0 <= s < lens[b]:
                    want[b, :, t] += w[:, :, j] @ x[b, :, s]
    np.testing.assert_allclose(ref_conv(x, w, 0, dil, lens), want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("u", [2, 4, 8])
def test_reference_conv_transpose_matches_loop(u):
    """ConvTranspose1d(kernel 2u, stride u, padding u/2): x[s] * w[k] lands on t = s*u + k - u/2; output length L*u"""
    rng = np.random.RandomState(u)
    B, Cin, Cout, L = 2, 3, 4, 5
    x, w = rng.randn(B, Cin, L), rng.randn(Cin, Cout, 2 * u)
    lens = [L, 3]
    want = np.zeros((B, Cout, L * u))
    for b in range(B):
        for s in range(lens[b]):
            for k in range(2 * u):
                t = s * u + k - u // 2
                if 0 <= t < lens[b] * u:
                    want[b, :, t] += x[b, :, s] @ w[:, :, k]
    np.testing.assert_allclose(ref_conv(x, w, u, 1, lens), want, rtol=1e-12, atol=1e-12)


def test_atom_image_round_trips():
    """channel c of step t sits at [c / 8][PADL + t][c % 8]; every other row is the fill"""
    rng = np.random.RandomState(0)
    v = rng.randn(2, 24, 37).astype(_F32)
    lpad = atoms_lpad(37)
    assert lpad == 64 + 512 + 64 and atoms_lpad(511) == 64 + 512 + 64 and atoms_lpad(512) == 64 + 1024 + 64
    img = to_atoms(v, lpad)
    assert img[1, 2, PADL + 5, 3] == v[1, 2 * 8 + 3, 5]
    np.testing.assert_array_equal(from_atoms(img, 37), v)
    assert np.isnan(img[:, :, :PADL]).all() and np.isnan(img[:, :, PADL + 37:]).all()


def test_exact_grid_bound_holds():
    """the largest exact-grid case (conv_pre: 1024 channels x 7 taps, four addends) stays below 2^15, where every
    multiple of 2^-8 is an fp32 number; grid values are exact in fp16 and their products multiples of 2^-8"""
    assert exact_sum_bound(1024 * 7, 4) < 2.0 ** 15
    assert exact_sum_bound(512 * 2, 2) < 2.0 ** 15            # the widest transposed conv: 512 channels x 2 taps
    k = np.arange(-32, 33)
    assert np.array_equal(f16(k / 16.0), k / 16.0)
    prod = np.outer(k, k) / 256.0
    assert np.array_equal(np.round(prod * 256), prod * 256)
    big = np.float64(2.0 ** 15 - 2.0 ** -8)                    # 23 significant bits: exact in fp32
    assert np.float64(np.float32(big)) == big


# ------------------------------------------------------------------------------------------------ GPU: Conv1d
CONV_SHAPES = [(1024, 512, 7, 1)] + [(C, C, K, d) for C in (256, 128, 64, 32) for K, d in RB_KD] + [(16, 32, 3, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("Cin,Cout,K,dil", CONV_SHAPES)
def test_conv_production_shapes(engine_small, Cin, Cout, K, dil):
    """conv_pre, every resblock (C, K, dil) of the full geometry (N = 256 / 128 / 64 / 32, CK = 64 / 32) and Cin = 16
    (CK = 16, one k-step): two items with their own speaker bias, bias + residual, out32 and out16."""
    L = 300 if Cin == 1024 else 700
    run_case(engine_small, Cin + K * 7 + dil, Cin, Cout, L, K, dil, B=2)
    run_case(engine_small, Cin + K * 7 + dil + 1, Cin, Cout, L, K, dil, B=2, exact=False)


@pytest.mark.gpu
@pytest.mark.parametrize("C,K,dil", [(64, 11, 5), (128, 7, 5), (256, 3, 3), (32, 11, 1)])
def test_conv_lengths(engine_small, C, K, dil):
    """lengths at and around every 64-row block and tile edge (tiles of 512, 256 and 128 rows)"""
    for L in [1, 2, 63, 64, 127, 128, 129, 255, 256, 257, 511, 512, 513]:
        run_case(engine_small, L, C, C, L, K, dil)


@pytest.mark.gpu
def test_conv_production_lengths(engine_small):
    """conv_pre over the z-frames of a 605-token chunk, and a C = 256 resblock conv over its first upsampled length"""
    run_case(engine_small, 1, 1024, 512, 2634, 7, 1)
    run_case(engine_small, 2, 1024, 512, 2634, 7, 1, exact=False)
    run_case(engine_small, 3, 256, 256, 2634 * 8, 11, 5)


# ------------------------------------------------------------------------------------------------ GPU: ConvTranspose1d
@pytest.mark.gpu
@pytest.mark.parametrize("Cin,Cout,u", CONVT)
def test_conv_transpose(engine_small, Cin, Cout, u):
    """every upsampler shape; L_in + 1 rows (the signal and the zero row x[L]) just below, at and just above a tile"""
    tile = tile_rows(u * Cout)
    for L in [1, tile - 2, tile - 1, tile, tile + 1]:
        run_case(engine_small, L, Cin, Cout, L, up=u, B=2, resid=False)
    run_case(engine_small, 99, Cin, Cout, tile + 1, up=u, B=2, resid=False, exact=False)


# ------------------------------------------------------------------------------------------------ GPU: ragged batches
def _lens32(L, tile, rng):
    """32 unsorted lengths: 0 first, in the middle and last; 1, tile - 1, tile, tile + 1 and L among the rest"""
    lens = [1, tile - 1, tile, tile + 1, L, L] + list(rng.randint(1, L + 1, 23))
    rng.shuffle(lens)
    return [0] + lens[:15] + [0] + lens[15:] + [0]


@pytest.mark.gpu
@pytest.mark.parametrize("up", [0, 2, 8])
def test_ragged_batches(engine_small, up):
    """batches of 1, 3 and 32 items with unsorted lengths (0 included), a speaker bias per item: stored rows equal the
    per-item reference, rows past Lout_i and pad rows keep their sentinels, nothing reads outside the cleared pads"""
    rng = np.random.RandomState(up)
    if up == 0:      # (Cin, Cout, K, dil, L)
        cases = [(64, 64, 11, 5, 1100), (256, 256, 7, 5, 400), (128, 128, 3, 3, 600)]
    elif up == 2:
        cases = [(64, 32, 0, 1, 1100), (128, 64, 0, 1, 600)]
    else:
        cases = [(256, 128, 0, 1, 300), (512, 256, 0, 1, 140)]
    for i, (Cin, Cout, K, dil, L) in enumerate(cases):
        tile = tile_rows(up * Cout if up else Cout)
        kw = dict(K=K, dil=dil, up=up, resid=up == 0)
        for j, lens in enumerate([[L - 37], [tile + 1, 0, 1], [0, L, tile - 1], [tile, L - 1, 0], _lens32(L, tile, rng),
                                  [0, 0, 0, 0]]):                   # the last: nothing is written
            run_case(engine_small, 10 * i + j, Cin, Cout, L, lens=lens, **kw)
        run_case(engine_small, 10 * i + 9, Cin, Cout, L, lens=_lens32(L, tile, rng), exact=False, **kw)


# ------------------------------------------------------------------------------------------------ GPU: epilogue modes
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [STORE, ACCUM], ids=["store", "accum"])
def test_epilogue_modes(engine_small, mode):
    """STORE and ACCUM, with and without the residual, out32 / out16 / both, scale16 1 and 1/3 (the last resblock's
    ACCUM + out16 = lrelu(sum / 3)); a ragged batch of three on N = 128 tiles"""
    outs = [(True, True), (True, False)] if mode == ACCUM else [(True, True), (True, False), (False, True)]
    seed = 0
    for resid in (False, True):
        for want32, want16 in outs:
            for scale16 in (1.0, 1.0 / 3.0):
                seed += 1
                run_case(engine_small, seed, 128, 128, 300, 7, 5, lens=[300, 0, 257], mode=mode, resid=resid,
                         want32=want32, want16=want16, scale16=scale16)
    run_case(engine_small, 50, 128, 128, 300, 7, 5, lens=[300, 0, 257], mode=mode, scale16=1.0 / 3.0, exact=False)
    run_case(engine_small, 51, 256, 256, 300, 11, 1, B=2, mode=mode, bias=False, cbias=False, scale16=1.0 / 3.0)


# ------------------------------------------------------------------------------------------------ GPU: grid cap
@pytest.mark.gpu
@pytest.mark.parametrize("up", [0, 2])
def test_grid_cap_and_determinism(engine_small, up):
    """max_ctas 0 (one CTA per SM), 1 (a single CTA wraps both rings over every tile), 3 and 7: bit-identical outputs,
    also across repeated runs, within the bound of the reference"""
    if up == 0:
        args = dict(Cin=256, Cout=256, L=1500, K=11, dil=5, lens=[1500, 700, 1290])
    else:
        args = dict(Cin=128, Cout=64, L=700, up=2, resid=False, lens=[700, 255, 513])
    first = None
    for max_ctas in (0, 1, 3, 7, 0, 1):
        got = run_case(engine_small, 5, exact=False, max_ctas=max_ctas, **args)
        if first is None:
            first = got
        np.testing.assert_array_equal(got[0], first[0])
        np.testing.assert_array_equal(got[1], first[1])
    run_case(engine_small, 6, exact=True, max_ctas=1, **args)


# ------------------------------------------------------------------------------------------------ GPU: rejections
@pytest.mark.gpu
def test_rejections_leave_the_engine_usable(engine_small):
    """geometries the kernel cannot run are refused on the host with an error, before anything launches"""
    rng = np.random.RandomState(0)
    x64, x24 = rng.randn(1, 64, 40), rng.randn(1, 24, 40)
    w64 = 0.02 * rng.randn(64, 64, 3)
    bad = [
        dict(x=x64, w=0.02 * rng.randn(64, 32, 6), up=3),                         # up not in {0, 2, 4, 8}
        dict(x=x64, w=0.02 * rng.randn(64, 64, 4)),                               # even Conv1d K
        dict(x=x24, w=0.02 * rng.randn(64, 24, 3)),                               # Cin = 24: no plan
        dict(x=x64, w=0.02 * rng.randn(16, 64, 3)),                               # Cout = 16: no plan
        dict(x=x64, w=0.02 * rng.randn(64, 64, 11), dil=13),                      # halo 5 * 13 > 64
        dict(x=rng.randn(33, 64, 8), w=w64),                                      # 33 items
        dict(x=rng.randn(2, 64, 40), w=w64, item_len=[40, 41]),                   # L_i > L
        dict(x=rng.randn(2, 64, 40), w=w64, item_len=[-1, 40]),                   # L_i < 0
        dict(x=x64, w=0.02 * rng.randn(64, 16, 4), up=2),                         # ConvTranspose1d Cout = 16
        dict(x=x64, w=0.02 * rng.randn(64, 4, 16), up=8,                          # Cout = 4 (neither % 32 nor, for out16, % 8)
             out16=np.zeros((1, 1, atoms_lpad(320), 4), _F32)),
        dict(x=x64, w=w64, mode=ACCUM),                                           # accumulate without out32
    ]
    for i, kw in enumerate(bad):
        with pytest.raises(NativeError):
            engine_small.debug_conv_tc(**kw)
            pytest.fail(f"case {i} was accepted")
    run_case(engine_small, 3, 64, 64, 40, 3, 1)
