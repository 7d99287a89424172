"""The fused tensor-core resblock (resblock_tc: one launch per ResBlock1 of the 64- and 32-channel vocoder stages, the
residual stream kept in shared memory) against the six conv1d_tc launches it replaces, bit for bit: the MRF sum and the
whole emitted atom image, sentinels and pad rows included, on identical inputs through xtts_debug_resblock_tc.  Then one
whole fast-mode vocoder pass at full geometry with the fused resblocks against the six-launch path (option tc_resblock).

The fused kernel tiles time by tile_rows = span - 2 * halo rows (span 384 rows at C = 64, 768 at C = 32; halo 12, 36, 60
rows for K = 3, 7, 11 at dilations 1, 3, 5), so the lengths below sit around those tile edges as well as around the 64-row
MMA blocks."""
import numpy as np
import pytest

from auralis_b200.config import XTTSDims
from auralis_b200.native import NativeEngine, atoms_lpad

STORE, ACCUM = NativeEngine.CONV_STORE, NativeEngine.CONV_ACCUM
SPAN = {64: 384, 32: 768}


def _tile(C, K):
    return SPAN[C] - 2 * 12 * (K - 1) // 2


def _pair(eng, seed, C, K, lens, L=None, mode=STORE, emit=False, max_ctas=0, ragged=True):
    """one resblock through both paths on identical inputs (Gaussian data, NaN sentinels) -> asserts bit identity"""
    rng = np.random.RandomState(seed)
    B = len(lens)
    L = L or max(4, (max(lens) + 3) // 4 * 4)
    x = rng.randn(B, C, L).astype(np.float32)
    ws = [(0.05 * rng.randn(C, C, K)).astype(np.float32) for _ in range(6)]
    bs = [(0.1 * rng.randn(C)).astype(np.float32) for _ in range(6)]
    zs = rng.randn(B, C, L).astype(np.float32) if mode == ACCUM else np.full((B, C, L), np.nan, np.float32)
    pa = np.full((B, C // 8, atoms_lpad(L), 8), np.nan, np.float32) if emit else None
    kw = dict(item_len=lens if ragged else None, zs=zs, mode=mode, pa=pa, scale16=1.0 / 3.0, max_ctas=max_ctas)
    six = eng.debug_resblock_tc(x, ws, bs, fused=False, **kw)
    fused = eng.debug_resblock_tc(x, ws, bs, fused=True, **kw)
    ctx = f"C={C} K={K} L={L} lens={lens} mode={mode} emit={emit} max_ctas={max_ctas}"
    for a, f in zip(six, fused):
        if a is not None:
            assert np.array_equal(a.view(np.uint32), f.view(np.uint32)), ctx
    for b, n in enumerate(lens):                        # every kept row was computed
        assert np.isfinite(fused[0][b, :, :n]).all(), ctx
        if emit:
            assert np.isfinite(fused[1][b, :, 64:64 + n]).all(), ctx


@pytest.mark.gpu
@pytest.mark.parametrize("C", [64, 32])
@pytest.mark.parametrize("K", [3, 7, 11])
@pytest.mark.parametrize("mode,emit", [(STORE, False), (STORE, True), (ACCUM, False), (ACCUM, True)])
def test_lengths_around_tile_edges(engine_small, C, K, mode, emit):
    """one ragged batch whose items cover short signals, the 64-row blocks, one / two tile edges and a few thousand rows"""
    tr = _tile(C, K)
    lens = [1, 3, 11, 12, 13, 59, 60, 61, 119, 120, 121, tr - 1, tr, tr + 1, 2 * tr - 1, 2 * tr, 2 * tr + 1, 3001]
    _pair(engine_small, C * 100 + K * 10 + mode * 2 + emit, C, K, lens, mode=mode, emit=emit)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [64, 32])
@pytest.mark.parametrize("L", [4, 12, 60, 120, 2 * 264, 2 * 648, 4000])
def test_whole_batch_lengths(engine_small, C, L):
    """items of the full buffer length (no item lengths given), STORE and ACCUM with the emitted atoms"""
    for K in (3, 11):
        _pair(engine_small, C + L + K, C, K, [L, L], ragged=False)
        _pair(engine_small, C + L + K + 1, C, K, [L], mode=ACCUM, emit=True, ragged=False)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [64, 32])
@pytest.mark.parametrize("lens", [[0], [517], [0, 300, 77], [300, 0, 77], [300, 77, 0],
                                  [0] + [13 * i + 1 for i in range(30)] + [0],
                                  [(37 * i) % 900 if i % 7 else 0 for i in range(32)]])
def test_ragged_batches(engine_small, C, lens):
    """batches of 1, 3 and 32 items, zero-length items first, in the middle and last"""
    _pair(engine_small, len(lens) + C, C, 7, lens, mode=ACCUM, emit=True)
    _pair(engine_small, len(lens) + C + 1, C, 11, lens, mode=STORE, emit=False)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [64, 32])
@pytest.mark.parametrize("max_ctas", [0, 1, 3, 7])
def test_grid_caps(engine_small, C, max_ctas):
    """a persistent CTA walks several tiles of several items: the same bits at every grid size"""
    _pair(engine_small, max_ctas + C, C, 11, [1500, 0, 700, 2100, 64], mode=ACCUM, emit=True, max_ctas=max_ctas)


@pytest.mark.gpu
def test_rejects_unsupported_geometry(engine_small):
    x = np.zeros((1, 128, 16), np.float32)
    ws = [np.zeros((128, 128, 3), np.float32)] * 6
    bs = [np.zeros(128, np.float32)] * 6
    with pytest.raises(RuntimeError):
        engine_small.debug_resblock_tc(x, ws, bs)                       # C = 128: the six launches only
    x = np.zeros((1, 64, 18), np.float32)
    ws = [np.zeros((64, 64, 3), np.float32)] * 6
    bs = [np.zeros(64, np.float32)] * 6
    with pytest.raises(RuntimeError):
        engine_small.debug_resblock_tc(x, ws, bs)                       # L % 4 != 0


@pytest.mark.gpu
@pytest.mark.parametrize("C,K,dil", [(64, 3, (1, 1, 1)), (32, 5, (1, 2, 3)), (64, 7, (2, 2, 3))])
def test_halo_not_multiple_of_4_stays_on_six_launches(engine_small, C, K, dil):
    """the fused kernel bulk-copies the fp32 span in 16-byte units, so it only takes chains whose halo
    (K-1)/2 * (d0 + d1 + d2 + 3) is a multiple of 4: other dilation sets are refused before any launch, and the six
    launches still run them"""
    rng = np.random.RandomState(K)
    L = 200
    x = rng.randn(2, C, L).astype(np.float32)
    ws = [(0.05 * rng.randn(C, C, K)).astype(np.float32) for _ in range(6)]
    bs = [(0.1 * rng.randn(C)).astype(np.float32) for _ in range(6)]
    with pytest.raises(RuntimeError, match="multiple of 4"):
        engine_small.debug_resblock_tc(x, ws, bs, dil=dil, item_len=[L, 77])
    zs, _ = engine_small.debug_resblock_tc(x, ws, bs, dil=dil, item_len=[L, 77], fused=False)
    assert np.isfinite(zs[0]).all() and np.isfinite(zs[1, :, :77]).all()


def _profiled_vocode(eng, lat):
    eng.set_option("profile", 1)
    try:
        wav = eng.vocode(lat, 0)
        prof = eng.kernel_profile()
    finally:
        eng.set_option("profile", 0)
    return wav, prof


@pytest.mark.gpu
@pytest.mark.parametrize("T", [7, 96])
def test_whole_vocoder_pass(engine_full_bf16, dims_full, T):
    """a fast-mode vocoder pass at full geometry: fused resblocks for the 64- and 32-channel stages, bit-identical to the
    six-launch path; the 256- and 128-channel stages keep the tensor-core conv"""
    eng = engine_full_bf16
    lat = np.random.RandomState(T).randn(T, dims_full.voc.in_dim).astype(np.float32)
    try:
        eng.set_option("tc_resblock", 0)
        six, p6 = _profiled_vocode(eng, lat)
    finally:
        eng.set_option("tc_resblock", 1)
    fused, pf = _profiled_vocode(eng, lat)
    assert np.isfinite(fused).all()
    assert np.array_equal(six.view(np.uint32), fused.view(np.uint32))
    assert "resblock_tc_f16_wgmma" not in p6
    assert pf["resblock_tc_f16_wgmma"]["launches"] == 2 * 3          # two stages x three resblocks
    assert pf["conv1d_tc_f16_wgmma"]["launches"] == p6["conv1d_tc_f16_wgmma"]["launches"] - 2 * 3 * 6


@pytest.mark.gpu
def test_engine_with_other_dilations_uses_six_launches(state_full, speakers_full):
    """a full-geometry engine whose resblock dilations give halos that are not multiples of 4 vocodes every resblock
    through the six tensor-core conv launches, as before the fused kernel existed"""
    import dataclasses
    from auralis_b200 import native
    dims = XTTSDims.full()
    dims = dataclasses.replace(dims, voc=dataclasses.replace(dims.voc, rb_dilations=(1, 2, 3)))
    eng = native.NativeEngine(dims, device=0, precision=1, max_batch=2, max_speakers=2)
    try:
        eng.load_state(*state_full)
        c, g = speakers_full[0]
        eng.set_speaker(0, c.numpy(), g.numpy())
        lat = np.random.RandomState(5).randn(9, dims.voc.in_dim).astype(np.float32)
        wav, prof = _profiled_vocode(eng, lat)
    finally:
        eng.close()
    assert np.isfinite(wav).all() and wav.shape[0] == dims.voc.n_samples(9)
    assert "resblock_tc_f16_wgmma" not in prof
    assert prof["conv1d_tc_f16_wgmma"]["launches"] > 4 * 3 * 6
