"""The staged epilogue of the fast-mode vocoder convolution (engine option tc_epilogue = 1: residual / accumulate base
prefetched into shared-memory slabs, outputs drained by bulk copies) against the direct epilogue (tc_epilogue = 0), bit
for bit: out32 and the whole out16 atom image, sentinels and pad rows included, on the same inputs.

The staged path runs for Conv1d launches whose fp32 rows are 16-byte aligned (output length a multiple of 4, as every
resblock stage of the vocoder is) and whose slab ring fits beside the A/B rings; other launches keep the direct epilogue,
so the lengths below are mostly multiples of 4, with a few that are not to check the fall-back."""
import numpy as np
import pytest

from auralis_b200.native import NativeEngine, atoms_lpad

STORE, ACCUM = NativeEngine.CONV_STORE, NativeEngine.CONV_ACCUM
RB_KD = [(3, 1), (3, 3), (7, 5), (11, 5), (11, 1)]


def _both(eng, seed, Cin, Cout, L, K=3, dil=1, lens=None, mode=STORE, resid=True, want32=True, want16=True,
          scale16=1.0, max_ctas=0):
    """one launch with each epilogue on identical inputs (Gaussian data, NaN sentinels) -> asserts bit identity"""
    rng = np.random.RandomState(seed)
    B = len(lens) if lens is not None else 1
    x = rng.randn(B, Cin, L).astype(np.float32)
    w = (0.05 * rng.randn(Cout, Cin, K)).astype(np.float32)
    b = (0.1 * rng.randn(Cout)).astype(np.float32)
    cb = (0.1 * rng.randn(B, Cout + 3)).astype(np.float32)
    r = rng.randn(B, Cout, L).astype(np.float32) if resid else None
    in32 = None
    if want32:
        in32 = rng.randn(B, Cout, L).astype(np.float32) if mode == ACCUM else np.full((B, Cout, L), np.nan, np.float32)
    in16 = np.full((B, Cout // 8, atoms_lpad(L), 8), np.nan, np.float32) if want16 else None
    outs = []
    try:
        for e in (0, 1):
            eng.set_option("tc_epilogue", e)
            outs.append(eng.debug_conv_tc(x, w, dil=dil, item_len=lens, bias=b, cbias=cb, resid=r, mode=mode,
                                          scale16=scale16, max_ctas=max_ctas, out32=in32, out16=in16))
    finally:
        eng.set_option("tc_epilogue", 1)
    ctx = f"Cin={Cin} Cout={Cout} K={K} dil={dil} L={L} lens={lens} mode={mode} resid={resid} scale16={scale16}"
    for a, s in zip(outs[0], outs[1]):
        if a is not None:
            assert np.array_equal(a.view(np.uint32), s.view(np.uint32)), ctx
    if want32:                                           # something was actually computed
        assert np.isfinite(outs[1][0][0, :, :(lens[0] if lens else L)]).all(), ctx


@pytest.mark.gpu
@pytest.mark.parametrize("C", [256, 128, 64, 32])
@pytest.mark.parametrize("K,dil", RB_KD)
def test_production_shapes(engine_small, C, K, dil):
    """every resblock conv of the full geometry: c2 (residual, out32 + out16), c1 (out16 only), last c2 (STORE and
    ACCUM, with and without the emitted atoms)"""
    L = 1000
    _both(engine_small, C + K + dil, C, C, L, K, dil, lens=[L, L - 200])
    _both(engine_small, C + K + dil + 1, C, C, L, K, dil, resid=False, want32=False)
    for mode in (STORE, ACCUM):
        for want16 in (False, True):
            _both(engine_small, 2 * C + K + dil, C, C, L, K, dil, lens=[L, 404], mode=mode, want16=want16,
                  scale16=1.0 / 3.0)
    _both(engine_small, 7, 1024, 512, 2636, 7, 1, resid=False, want32=False)      # conv_pre


@pytest.mark.gpu
@pytest.mark.parametrize("C,K,dil", [(256, 11, 5), (128, 11, 5), (64, 3, 1), (32, 11, 5)])
def test_lengths(engine_small, C, K, dil):
    """1 .. 513 around the 64-row blocks, tiles and slab edges; Lout_i - t0 = 1, 2, 3 (mod 4) through ragged items"""
    for L in [4, 8, 60, 64, 124, 128, 132, 252, 256, 260, 508, 512, 516, 1, 3, 129, 255, 513]:
        _both(engine_small, L, C, C, L, K, dil)
    for L in [260, 516]:
        for t in (1, 2, 3, 5, 6, 7, 129, 130, 131, 257, 258, 259):
            _both(engine_small, L + t, C, C, L, K, dil, lens=[min(t, L), L - (L - t) % 4 if t < L else L])


@pytest.mark.gpu
def test_epilogue_variants(engine_small):
    """STORE / ACCUM x residual x out32 / out16 / both x scale16 1 and 1/3"""
    seed = 0
    for mode in (STORE, ACCUM):
        for resid in (False, True):
            for want32, want16 in [(True, True), (True, False), (False, True)]:
                if mode == ACCUM and not want32:          # accumulating needs out32 (rejected on the host)
                    continue
                for scale16 in (1.0, 1.0 / 3.0):
                    seed += 1
                    _both(engine_small, seed, 128, 128, 600, 7, 3, lens=[600, 257, 0], mode=mode, resid=resid,
                          want32=want32, want16=want16, scale16=scale16)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [256, 64])
def test_ragged_batches_and_grid_caps(engine_small, C):
    """batches of 1, 3 and 32 items with zero-length items first, in the middle and last, on grid caps 0, 1, 3, 7"""
    rng = np.random.RandomState(C)
    L = 1100
    lens32 = [0] + list(rng.randint(1, L + 1, 15)) + [0] + list(rng.randint(1, L + 1, 14)) + [0]
    for lens in ([L - 36], [0, 517, 1], [300, 0, L], lens32):
        for cap in (0, 1, 3, 7):
            _both(engine_small, len(lens) + cap, C, C, L, 11, 5, lens=[int(n) for n in lens], mode=ACCUM,
                  max_ctas=cap)
