"""The fp8 KV format (auralis_b200/csrc/kv_fp8.cuh) restated on the host: the per-(token, head) power-of-two quantiser and the
page layout.  The GPU tests (tests/test_gpu_kv_fp8.py) compare the kernels' bytes with this quantiser bit for bit; the
checks here tie it to torch's float8_e4m3fn cast and to the exponent rule."""
import numpy as np
import pytest
import torch

PT, D = 32, 64                         # tokens per KV page, head dim
BLOCK = PT * D + PT                    # bytes of one (page, head) block: e4m3 data, then one exponent byte per token
E4M3_MAX = 448.0


def exponent(amax):
    """the smallest integer e with amax * 2^-e <= 448, clamped to int8; -128 for an all-zero row"""
    a = np.asarray(amax, np.float32).astype(np.float64)
    m, E = np.frexp(a)                                  # a = m * 2^E, m in [0.5, 1); 448 = 0.875 * 2^9
    e = np.where(m <= 0.875, E - 9, E - 8)
    e = np.where(a > 0, e, -128)
    return np.clip(e, -128, 127).astype(np.int8)


def to_e4m3(x):
    """fp32 -> e4m3 bytes, round to nearest even (torch's float8_e4m3fn cast)"""
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def from_e4m3(q):
    return torch.from_numpy(np.ascontiguousarray(q, np.uint8)).view(torch.float8_e4m3fn).to(torch.float64).numpy()


def quantize(x):
    """rows x [..., 64] fp32 -> (e4m3 bytes [..., 64], exponents int8 [...]); byte = e4m3(x * 2^-e), the scaling exact"""
    x = np.asarray(x, np.float32)
    e = exponent(np.abs(x).max(axis=-1))
    scaled = (x.astype(np.float64) * np.exp2(-e.astype(np.float64))[..., None]).astype(np.float32)
    return to_e4m3(scaled), e


def dequantize(q, e):
    """the values the cache holds, float64: e4m3 * 2^e"""
    return from_e4m3(q) * np.exp2(np.asarray(e, np.int8).astype(np.float64))[..., None]


def pack(q, e, kv):
    """bytes [pages, heads, 32 tok, 64] + exponents [pages, heads, 32] -> device blocks [pages, heads, 2080]:
    K data [64/16][32 tok][16], V data [32 tok][64], then the 32 exponents"""
    p, h = q.shape[:2]
    data = q.reshape(p, h, PT, D // 16, 16).transpose(0, 1, 3, 2, 4) if kv == "k" else q
    return np.concatenate([np.ascontiguousarray(data).reshape(p, h, PT * D), e.view(np.uint8)], axis=2)


def unpack(blocks, kv):
    p, h = blocks.shape[:2]
    data, e = blocks[..., :PT * D], blocks[..., PT * D:].view(np.int8)
    if kv == "k":
        data = data.reshape(p, h, D // 16, PT, 16).transpose(0, 1, 3, 2, 4)
    return np.ascontiguousarray(data).reshape(p, h, PT, D), np.ascontiguousarray(e)


# ------------------------------------------------------------------------------------------------ checks
def test_quantiser_matches_torch_cast_and_never_saturates():
    rng = np.random.RandomState(0)
    x = rng.randn(600, D).astype(np.float32)
    x *= np.exp2(rng.randint(-140, 120, size=(600, 1))).astype(np.float32)        # row scales across fp32's range
    x[::7, ::3] = 0.0
    q, e = quantize(x)
    for r in range(x.shape[0]):
        want = torch.from_numpy((x[r].astype(np.float64) * 2.0 ** -int(e[r])).astype(np.float32)).to(torch.float8_e4m3fn)
        np.testing.assert_array_equal(q[r], want.view(torch.uint8).numpy())
    assert not np.isin(q & 0x7F, [0x7F]).any()                      # no NaN code: nothing saturated past 448
    amax = np.abs(x).max(axis=1).astype(np.float64)
    assert (amax * np.exp2(-e.astype(np.float64)) <= E4M3_MAX).all()
    tight = e > -128
    assert (amax[tight] * np.exp2(-(e[tight].astype(np.float64) - 1)) > E4M3_MAX).all()    # e is the smallest such
    # one rounding of e4m3 (3 mantissa bits: half an ulp = 2^-4 relative), or half its subnormal step 2^-10 at the row's scale
    deq = dequantize(q, e)
    tol = 2.0 ** -4 * np.abs(x) + 2.0 ** -10 * np.exp2(e.astype(np.float64))[:, None]
    assert (np.abs(deq - x) <= tol).all()


def test_exponent_rule_edges():
    k = np.arange(-60, 60)
    at = (E4M3_MAX * np.exp2(k)).astype(np.float32)                 # exactly 448 * 2^k: scales to 448 itself
    np.testing.assert_array_equal(exponent(at), k)
    up = np.nextafter(at, np.float32(np.inf))
    np.testing.assert_array_equal(exponent(up), k + 1)
    down = np.nextafter(at, np.float32(0))
    np.testing.assert_array_equal(exponent(down), k)
    assert exponent(np.float32(0.0)) == -128                        # all-zero row: the minimum
    assert exponent(np.float32(1e-45)) == -128                      # clamped below
    assert exponent(np.float32(3e38)) == 120                        # 3e38 = 0.88 * 2^128
    assert exponent(np.float32(1.0)) == -8                          # 1 * 2^8 = 256 <= 448 < 512
    q, e = quantize(np.zeros((1, D), np.float32))
    assert e[0] == -128 and (q == 0).all()


def test_rounding_ties_to_even_and_subnormals():
    # at 1: e4m3 step 2^-3.  1 + 2^-4 ties to 1 (even), 1 + 3 * 2^-4 ties to 1.25, 1 + 2^-4 + 2^-12 goes up
    v = np.array([1 + 2.0 ** -4, 1 + 3 * 2.0 ** -4, 1 + 2.0 ** -4 + 2.0 ** -12], np.float32)
    np.testing.assert_array_equal(from_e4m3(to_e4m3(v)), [1.0, 1.25, 1.125])
    # subnormal step 2^-9: 2^-10 ties to 0, 3 * 2^-10 ties to 2^-8, 2^-9 + 2^-11 rounds down
    v = np.array([2.0 ** -10, 3 * 2.0 ** -10, 2.0 ** -9 + 2.0 ** -11, 2.0 ** -9], np.float32)
    np.testing.assert_array_equal(from_e4m3(to_e4m3(v)), [0.0, 2.0 ** -8, 2.0 ** -9, 2.0 ** -9])
    # through the quantiser: a row whose largest element is 448 keeps e = 0 and its small entries go subnormal
    row = np.zeros((1, D), np.float32)
    row[0, :5] = [448.0, 2.0 ** -10, 3 * 2.0 ** -10, -3 * 2.0 ** -10, 2.0 ** -12]
    q, e = quantize(row)
    assert e[0] == 0
    np.testing.assert_array_equal(dequantize(q, e)[0, :5], [448.0, 0.0, 2.0 ** -8, -(2.0 ** -8), 0.0])


@pytest.mark.parametrize("kv", ["k", "v"])
def test_page_layout_round_trip(kv):
    rng = np.random.RandomState(1 if kv == "k" else 2)
    x = rng.randn(5, 3, PT, D).astype(np.float32) * 10
    q, e = quantize(x)
    blocks = pack(q, e, kv)
    assert blocks.shape == (5, 3, BLOCK) and blocks.dtype == np.uint8
    q2, e2 = unpack(blocks, kv)
    np.testing.assert_array_equal(q2, q)
    np.testing.assert_array_equal(e2, e)
    for _ in range(200):
        p, h, t, d = rng.randint(5), rng.randint(3), rng.randint(PT), rng.randint(D)
        off = ((d // 16) * PT + t) * 16 + d % 16 if kv == "k" else t * D + d
        assert blocks[p, h, off] == q[p, h, t, d]
        assert blocks[p, h, PT * D + t].view(np.int8) == e[p, h, t]
