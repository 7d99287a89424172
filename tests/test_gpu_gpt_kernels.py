"""The GPT forward's remaining kernels launched on their own and compared with a float64 reference of the same operation:
the one-tile tensor-core GEMM in the configurations the decode step and fast-mode prefill use (16-bit output with GELU, a
residual that aliases the output, PDL launches, every decode tile width, the deep ring and the L2 prefetch), the decode
LayerNorm -> GEMM pair with and without dependency counters, the LayerNorm and GPT head norm kernels in all three output
types, the prefill's paged-cache write and both row builds.  The reference sees the operands rounded exactly as the kernel
rounds them, so each bound is the output rounding plus an fp32 arithmetic term derived next to it.  Scheduling options must
not change a single bit; the end-to-end test checks that for the decode step's non-default execution paths."""
import numpy as np
import pytest
import torch

from auralis_b200.native import NativeEngine, Sampling
from conftest import text_ids
from oracle import xtts_oracle as O
from test_gpu_decode_kernels import HALF_ULP, PT, D, U, bits, pack_k, pack_v, ref_layernorm, rnd

_F64 = np.float64
KIND_NAMES = {0: "fp32", 1: "bf16", 2: "fp16"}
SQRT_2_PI = np.sqrt(2.0 / np.pi)


# ------------------------------------------------------------------------------------------------ float64 references
def gelu_new(x):
    """tanh GELU in float64 (the kernels' gelu_new, the oracle's gelu_new)."""
    return 0.5 * x * (1.0 + np.tanh(SQRT_2_PI * (x + 0.044715 * x ** 3)))


def gelu_slope(x):
    """d gelu_new / dx in float64."""
    t = np.tanh(SQRT_2_PI * (x + 0.044715 * x ** 3))
    return 0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * SQRT_2_PI * (1.0 + 3 * 0.044715 * x * x)


GELU_CURVATURE = 0.8          # max |gelu_new''| over the reals (0.798 at x = 0)


def gemm_products(A16, W16):
    """(A16 . W16^T, |A16| . |W16|^T) in float64: the exact product and the scale of its accumulation error."""
    return A16 @ W16.T, np.abs(A16) @ np.abs(W16).T


def ref_gemm16(A16, W16, bias, resid, gelu, out_kind, prod=None):
    """Reference and element-wise bound of the tensor-core GEMM epilogue, operands already rounded to the 16-bit type
    (float64 arrays of their exact values).  The kernel computes, per element, in fp32:
        acc = sum_k a_k w_k          error <= 1e-5 * sum_k |a_k w_k|  (tensor-core accumulation; S below)
        x   = acc + bias             one rounding: u |x|
        g   = gelu_new(x)            fp32 evaluation: the argument's three roundings move tanh by at most
                                     5u |t| sech^2(t) <= 2.3u, tanhf is within 2 ulp, 1 + tanh and the two products add 3u of
                                     0.5 |x| (1 + |tanh|): in all <= u (8 |x| + 4 |g|); the input error E passes through at
                                     the local slope, |gelu'(z)| + 0.8 E (|gelu''| <= 0.8)
        y   = g + resid              one rounding: u |y|
        out = rn16(y)                half an ulp of the output type, relative (fp16: plus half its smallest subnormal)
    prod: gemm_products(A16, W16) when already computed.  -> (ref [M, N] float64, tol [M, N])."""
    z, S = prod if prod is not None else gemm_products(A16, W16)
    E = 1e-5 * S
    if bias is not None:
        z = z + bias
    E = E + U * (np.abs(z) + E)
    if gelu:
        g = gelu_new(z)
        E = (np.abs(gelu_slope(z)) + GELU_CURVATURE * E) * E + U * (8 * np.abs(z) + 4 * np.abs(g) + 12 * E)
        z = g
    if resid is not None:
        z = z + resid
        E = E + U * (np.abs(z) + E)
    h = HALF_ULP[out_kind]
    tol = (1 + h) * E + h * np.abs(z) + (2.0 ** -25 if out_kind == 2 else 0.0) + 1e-30
    return z, tol


def ln_slack(x, w, b, mu, rstd):
    """fp32 error of one LayerNorm evaluation (two-pass statistics, (x - mean) * rstd * w + b), as in
    test_splitk_reduce_layernorm_matches_fp64: the mean's error scaled by rstd, the normalised value's roundings."""
    xh = np.abs((x - mu) * rstd)
    return U * ((16 * np.abs(mu) * rstd + 32 * (xh + 1.0)) * np.abs(w) + 32 * np.abs(b))


def ref_ln_chain(x, params, eps):
    """float64 LayerNorms applied one after the other: params = [(w, b), ...].  Each stage's bound carries the previous
    stage's worst error e through the LayerNorm's sensitivity, |dy| <= |w| rstd (|e| + mean|e| + |xh| mean(|xh| |e|))
    <= |w| rstd max|e| (2 + |xh|) (mean |xh| <= 1), plus its own fp32 slack.  -> [(ref, slack) per stage]."""
    out = []
    cur = np.asarray(x, _F64)
    carried = np.zeros(cur.shape[0])
    for w, b in params:
        y, mu, rstd = ref_layernorm(cur, w, b, eps)
        xh = np.abs((cur - mu) * rstd)
        s = np.abs(w) * rstd * carried[:, None] * (2.0 + xh) + ln_slack(cur, w, b, mu, rstd)
        out.append((y, s))
        cur, carried = y, s.max(axis=1)
    return out


def ln_rows(M, H, rng, mean_offset=1e3):
    """Rows cycle through: a 1e3 mean offset (two-pass variance), variance below eps (spread 1e-3: eps dominates rstd), a
    constant row (zero variance: the output is the bias), and plain rows."""
    X = rng.randn(M, H)
    for i in range(M):
        k = i % 4
        if k == 0:
            X[i] += mean_offset
        elif k == 1:
            X[i] = 0.3 + 1e-3 * rng.randn(H)
        elif k == 2:
            X[i] = -2.75
    return X.astype(np.float32)


# ------------------------------------------------------------------------------------------------ CPU checks
def test_reference_gelu_matches_torch():
    x = np.concatenate([np.linspace(-12, 12, 20001), np.random.RandomState(0).randn(1000) * 4])
    got = gelu_new(x)
    exp = torch.nn.functional.gelu(torch.from_numpy(x), approximate="tanh").numpy()
    np.testing.assert_allclose(got, exp, rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(got, O.gelu_new(torch.from_numpy(x)).numpy(), rtol=1e-13, atol=1e-15)
    h = 1e-6
    np.testing.assert_allclose(gelu_slope(x), (gelu_new(x + h) - gelu_new(x - h)) / (2 * h), rtol=1e-6, atol=1e-8)
    assert np.abs(gelu_slope(x)).max() < 1.13
    second = (gelu_slope(x + h) - gelu_slope(x - h)) / (2 * h)
    assert np.abs(second).max() <= GELU_CURVATURE


def test_reference_gemm_bound_covers_fp32_evaluation():
    """The bound of ref_gemm16 covers an explicit fp32 evaluation of the same epilogue (torch, float32 throughout)."""
    rng = np.random.RandomState(1)
    for kind in (1, 2):
        A = rnd(rng.randn(33, 256).astype(np.float32) * 3, kind)[1]
        W = rnd((rng.randn(96, 256) * 0.05).astype(np.float32), kind)[1]
        b = rng.randn(96).astype(np.float32)
        r = rng.randn(33, 96).astype(np.float32)
        for gelu, resid in ((False, None), (True, None), (True, r), (False, r)):
            x = torch.from_numpy(A.astype(np.float32)) @ torch.from_numpy(W.astype(np.float32)).T + torch.from_numpy(b)
            if gelu:
                x = 0.5 * x * (1.0 + torch.tanh(np.float32(SQRT_2_PI) * (x + np.float32(0.044715) * x * x * x)))
            if resid is not None:
                x = x + torch.from_numpy(resid)
            got = rnd(x.numpy(), kind)[1]
            ref, tol = ref_gemm16(A, W, b, resid, gelu, kind)
            assert (np.abs(got - ref) <= tol).all(), (kind, gelu, resid is not None)


def test_reference_ln_chain_matches_torch():
    rng = np.random.RandomState(2)
    H = 192
    x = ln_rows(9, H, rng).astype(_F64)
    params = [(1.0 + 0.1 * rng.randn(H), 0.1 * rng.randn(H)) for _ in range(3)]
    chain = ref_ln_chain(x, params, 1e-5)
    t = torch.from_numpy(x)
    for (w, b), (y, s) in zip(params, chain):
        ln = torch.nn.LayerNorm(H, eps=1e-5, dtype=torch.float64)
        with torch.no_grad():
            ln.weight.copy_(torch.from_numpy(w)); ln.bias.copy_(torch.from_numpy(b))
            t = ln(t)
        np.testing.assert_allclose(y, t.numpy(), rtol=1e-10, atol=1e-10)
        assert (s > 0).all()
    # the carried bound covers a float32 evaluation of the chain in the kernels' formula (two-pass statistics, then
    # (x - mean) * rstd * w + b), each stage fed the previous stage's float32 output
    f = np.float32
    cur = x.astype(f)
    for (w, b), (y, s) in zip(params, chain):
        mean = cur.sum(axis=1, dtype=f, keepdims=True) / f(H)
        d = cur - mean
        rstd = f(1.0) / np.sqrt((d * d).sum(axis=1, dtype=f, keepdims=True) / f(H) + f(1e-5))
        cur = d * rstd * w.astype(f) + b.astype(f)
        assert (np.abs(cur - y) <= s).all()


def _tables(H, rng, n_text=11, n_tpos=9, n_audio=13, n_wpe=10, n_spk=3, n_cond=32):
    f = lambda *s: rng.randn(*s).astype(np.float32)
    return dict(text_emb=f(n_text, H), text_pos=f(n_tpos, H), wte=f(n_audio, H), wpe=f(n_wpe, H), spk_cond=f(n_spk, n_cond, H))


def ref_build_rows(rows, t):
    """float32 numpy: kind 0 spk_cond[c][a]; 1 text_emb[a] + text_pos[b]; 2 wte[a] + wpe[b]."""
    out = []
    for kind, a, b, c in rows:
        if kind == 0:
            out.append(t["spk_cond"][c][a])
        elif kind == 1:
            out.append(t["text_emb"][a] + t["text_pos"][b])
        else:
            out.append(t["wte"][a] + t["wpe"][b])
    return np.stack(out).astype(np.float32)


def prompt_row_descs(n_cond, n_text_ids, start_audio_token, speaker):
    """The engine's RowDesc list of one prompt (build_prefill): cond rows, text rows, the start-audio row."""
    return ([(0, i, 0, speaker) for i in range(n_cond)] + [(1, tid, i, 0) for i, tid in enumerate(n_text_ids)]
            + [(2, start_audio_token, 0, 0)])


def test_reference_build_rows_matches_oracle_prompt(dims_small, state_small, speakers_small):
    gs, cs = state_small
    orc = O.GPTOracle(gs, cs, dims_small)
    g = dims_small.gpt
    t = dict(text_emb=cs["text_embedding.weight"].numpy(), text_pos=cs["text_pos_embedding.emb.weight"].numpy(),
             wte=gs["gpt.wte.weight"].numpy(), wpe=gs["gpt.wpe.emb.weight"].numpy(),
             spk_cond=np.stack([c.numpy() for c, _ in speakers_small]))
    for spk, n in ((0, 5), (2, 17)):
        ids = text_ids(dims_small, n, 30 + n)
        got = ref_build_rows(prompt_row_descs(g.n_cond_latents, ids, g.start_audio_token, spk), t)
        exp = orc.prompt_rows(speakers_small[spk][0], ids).numpy()
        np.testing.assert_array_equal(got, exp)


# ------------------------------------------------------------------------------------------------ GEMM
def _gemm_shapes(dims_small, dims_full):
    """(N, K) of the qkv, fc, fc2 and head GEMMs of both geometries (the head padded to a multiple of 32 as the engine
    pads it), then N tails that are not a multiple of 128 and the shortest K."""
    out = []
    for d in (dims_small, dims_full):
        g = d.gpt
        out += [(3 * g.hidden, g.hidden), (g.ff, g.hidden), (g.hidden, g.ff), (-(-g.n_audio_tokens // 32) * 32, g.hidden)]
    return out + [(1056, 1024), (288, 192), (96, 256), (384, 64)]


def _gemm_data(M, N, K, kind, seed):
    rng = np.random.RandomState(seed)
    A = (rng.randn(M, K) * 1.5).astype(np.float32)
    W = (rng.randn(N, K) * (1.0 / np.sqrt(K))).astype(np.float32)
    b = rng.randn(N).astype(np.float32)
    r = rng.randn(M, N).astype(np.float32)
    return A, W, b, r, rnd(A, kind)[1], rnd(W, kind)[1]


def _check(got, ref, tol, label):
    assert np.isfinite(got).all(), label
    err = np.abs(got - ref)
    bad = np.argwhere(err > tol)
    assert bad.size == 0, (label, bad[:5].tolist(), float((err / tol).max()))
    return float((err / tol).max())


# the epilogue variants the engine uses: (gelu, out16, resid, inplace, pdl)
#   qkv / head: bias only; fc: GELU + 16-bit out; o-proj / down-proj without split-K: residual in place; plus a PDL launch
GEMM_VARIANTS = [(False, False, False, False, False), (True, True, False, False, False), (False, False, True, True, False),
                 (True, False, True, False, True), (True, True, False, False, True), (False, False, True, True, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 7, 8, 9, 64, 65, 127, 128, 129, 168, 255])
@pytest.mark.parametrize("mode", [1, 2], ids=["bf16", "fp16"])
def test_gemm_narrow_epilogues_match_fp64(engine_small, dims_small, dims_full, mode, M):
    """The one-tile tensor-core GEMM (M < 256 never reaches the wide kernel) against the fp64 product of the rounded
    operands under ref_gemm16's element-wise bound, for every decode / prefill epilogue: bias only, GELU with 16-bit output
    (the fc GEMM of every decode step), the residual aliasing the output, and PDL launches of them.  M = 168 is the bench
    regime's row count."""
    worst = {}
    for si, (N, K) in enumerate(_gemm_shapes(dims_small, dims_full)):
        A, W, b, r, A16, W16 = _gemm_data(M, N, K, mode, seed=M * 131 + si)
        prod = gemm_products(A16, W16)
        refs = {}
        for gelu, out16, resid, inplace, pdl in GEMM_VARIANTS:
            out, _ = engine_small.debug_gemm(mode, A, W, b, r if resid else None, gelu, out16=out16, inplace=inplace, pdl=pdl)
            key = (gelu, resid, 1 if out16 else 0)
            if key not in refs:
                refs[key] = ref_gemm16(A16, W16, b, r if resid else None, gelu, mode if out16 else 0, prod)
            name = ("gelu+" if gelu else "") + ("out16" if out16 else "f32") + ("+resid-inplace" if inplace else "+resid" if resid else "") + ("+pdl" if pdl else "")
            share = _check(out, *refs[key], (KIND_NAMES[mode], M, N, K, name))
            worst[name] = max(worst.get(name, 0.0), share)
    print(f"narrow GEMM {KIND_NAMES[mode]} M={M}, largest share of the error bound used: "
          + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2], ids=["bf16", "fp16"])
def test_gemm_wide_vs_narrow(engine_small, mode):
    """Prefill shapes (M >= 256) on the persistent wide-tile kernel and, with "gemm_wide" 0, on the one-tile kernel: GELU
    with 16-bit output and the in-place residual, each within the fp64 bound.  Nothing promises the two kernels the same
    bits, so whether they match is printed, not asserted."""
    eng = engine_small
    worst, same = 0.0, []
    for M in (256, 257, 513, 1000):
        for (N, K) in ((4096, 1024), (1024, 4096), (1056, 1024), (288, 192)):
            A, W, b, r, A16, W16 = _gemm_data(M, N, K, mode, seed=M + N + K)
            prod = gemm_products(A16, W16)
            for gelu, out16, inplace in ((True, True, False), (False, False, True)):
                ref, tol = ref_gemm16(A16, W16, b, r if inplace else None, gelu, mode if out16 else 0, prod)
                got = {}
                try:
                    for wide in (4, 0):
                        eng.set_option("gemm_wide", wide)
                        got[wide], _ = eng.debug_gemm(mode, A, W, b, r if inplace else None, gelu, out16=out16, inplace=inplace)
                        worst = max(worst, _check(got[wide], ref, tol, (KIND_NAMES[mode], M, N, K, gelu, out16, inplace, wide)))
                finally:
                    eng.set_option("gemm_wide", 4)
                same.append(bool(np.array_equal(bits(got[4]), bits(got[0]))))
    print(f"wide vs narrow GEMM {KIND_NAMES[mode]}: largest share of the error bound used {worst:.3g}; "
          f"bit-identical in {sum(same)} / {len(same)} cases")


# Deep-ring shapes: K / 64 k-blocks exceed the default ring (BN 32: 5 stages, BN 64: 4), M <= 256, no split-K
DEEP_RING_SHAPES = [(1, 1024, 4096), (7, 4096, 1024), (168, 3072, 1024), (255, 1056, 1024), (256, 1024, 1024), (33, 384, 512)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2], ids=["bf16", "fp16"])
def test_gemm_scheduling_options_are_bit_identical(engine_small, mode):
    """Within the one-tile kernel, the tile width ("gemm_bn" 0 / 32 / 64 / 128), the deep ring ("gemm_deep_ring"), the L2
    prefetch of later weight tiles ("gemm_l2_prefetch") and a PDL launch change scheduling only: every output element sees
    the same MMAs in the same k order, so all 32 combinations give the same bits, in the fp32 and the 16-bit epilogue."""
    eng = engine_small
    try:
        eng.set_option("gemm_wide", 0)                  # M = 256 stays on the one-tile kernel for the plain launch too
        for (M, N, K) in DEEP_RING_SHAPES:
            A, W, b, r, A16, W16 = _gemm_data(M, N, K, mode, seed=M * 7 + N + K)
            prod = gemm_products(A16, W16)
            for gelu, out16, inplace in ((True, True, False), (False, False, True)):
                ref, tol = ref_gemm16(A16, W16, b, r if inplace else None, gelu, mode if out16 else 0, prod)
                base = None
                for bn in (0, 32, 64, 128):
                    for deep in (0, 1):
                        for l2 in (0, 1):
                            for pdl in (False, True):
                                eng.set_option("gemm_bn", bn); eng.set_option("gemm_deep_ring", deep)
                                eng.set_option("gemm_l2_prefetch", l2)
                                out, _ = eng.debug_gemm(mode, A, W, b, r if inplace else None, gelu, out16=out16,
                                                        inplace=inplace, pdl=pdl)
                                label = (KIND_NAMES[mode], M, N, K, gelu, out16, bn, deep, l2, pdl)
                                if base is None:
                                    _check(out, ref, tol, label)
                                    base = out
                                np.testing.assert_array_equal(bits(out), bits(base), err_msg=str(label))
    finally:
        for k, v in (("gemm_wide", 4), ("gemm_bn", 0), ("gemm_deep_ring", 0), ("gemm_l2_prefetch", 0)):
            eng.set_option(k, v)


def test_gemm_flag_word_keeps_gelu_bit():
    """The flag word of xtts_debug_gemm keeps bit 1 = GELU, so 0 / 1 still mean what the old gelu argument meant."""
    from auralis_b200 import native
    assert native.GEMM_GELU == 1
    assert len({native.GEMM_GELU, native.GEMM_OUT16, native.GEMM_INPLACE, native.GEMM_PDL}) == 4


@pytest.mark.gpu
def test_gemm_rejects_bad_flag_combinations(engine_small):
    from auralis_b200.native import NativeError
    A = np.ones((4, 64), np.float32)
    W = np.ones((32, 64), np.float32)
    r = np.ones((4, 32), np.float32)
    for kw in (dict(mode=0, out16=True), dict(mode=0, pdl=True), dict(mode=1, inplace=True), dict(mode=1, out16=True, resid=r,
                                                                                                   inplace=True)):
        mode = kw.pop("mode")
        with pytest.raises(NativeError):
            engine_small.debug_gemm(mode, A, W, None, kw.pop("resid", None), **kw)
    with pytest.raises(NativeError):
        engine_small.debug_gemm(1, A[:, :40], W[:, :40])            # K % 64
    with pytest.raises(NativeError):
        engine_small.debug_ln_gemm(1, 2, A, A[0], A[0], W, resid=r)   # a counter cannot order a residual read


# ------------------------------------------------------------------------------------------------ LayerNorm -> GEMM pair
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2], ids=["bf16", "fp16"])
def test_decode_ln_gemm_launch_modes(engine_small, dims_small, dims_full, mode):
    """The decode step's LayerNorm -> GEMM pair (the first LN and the qkv GEMM of decode_layers_rows; GELU + 16-bit output as
    the fc GEMM) in its three launch modes — plain, PDL, PDL plus dependency counters — gives the same bits in all three;
    the LN output is within one 16-bit rounding of the fp64 LayerNorm, the GEMM output within ref_gemm16's bound of the
    product of the kernel's own LN output; each counter ends at exactly the CTA count of its kernel (M for the LN)."""
    eng = engine_small
    eps = dims_small.gpt.ln_eps
    worst_y = worst_o = 0.0
    for (N, K) in ((3 * dims_full.gpt.hidden, dims_full.gpt.hidden), (dims_full.gpt.ff, dims_full.gpt.hidden),
                   (3 * dims_small.gpt.hidden, dims_small.gpt.hidden)):
        for M in (1, 9, 64, 168, 255):
            rng = np.random.RandomState(M * 17 + N)
            X = ln_rows(M, K, rng)
            ln_w = (1.0 + 0.1 * rng.randn(K)).astype(np.float32)
            ln_b = (0.1 * rng.randn(K)).astype(np.float32)
            W = (rng.randn(N, K) / np.sqrt(K)).astype(np.float32)
            bias = rng.randn(N).astype(np.float32)
            W16 = rnd(W, mode)[1]
            for gelu, out16 in ((False, False), (True, True)):
                res = {}
                for launch in (0, 1, 2):
                    Y, out, n_ctas, cnt = eng.debug_ln_gemm(mode, launch, X, ln_w, ln_b, W, bias, gelu=gelu, out16=out16)
                    label = (KIND_NAMES[mode], M, N, K, gelu, launch)
                    res[launch] = (Y, out)
                    assert n_ctas > 0, label
                    if launch == 2:
                        assert cnt.tolist() == [M, n_ctas], (label, cnt.tolist(), n_ctas)
                    else:
                        assert cnt.tolist() == [0, 0], label
                Y, out = res[0]
                for launch in (1, 2):
                    np.testing.assert_array_equal(bits(res[launch][0]), bits(Y), err_msg=str((label, "Y")))
                    np.testing.assert_array_equal(bits(res[launch][1]), bits(out), err_msg=str((label, "out")))
                (y_ref, s), = ref_ln_chain(X, [(ln_w, ln_b)], eps)
                worst_y = max(worst_y, _check(Y, y_ref, HALF_ULP[mode] * np.abs(y_ref) + (1 + HALF_ULP[mode]) * s + 1e-30,
                                              (label, "Y")))
                ref, tol = ref_gemm16(Y.astype(_F64), W16, bias, None, gelu, mode if out16 else 0)
                worst_o = max(worst_o, _check(out, ref, tol, (label, "out")))
    print(f"decode LN -> GEMM {KIND_NAMES[mode]}, largest share of the error bound used: Y {worst_y:.3g}, out {worst_o:.3g}")


# ------------------------------------------------------------------------------------------------ LayerNorm / head norms
def _ln_params(H, rng, n):
    return [((1.0 + 0.1 * rng.randn(H)).astype(np.float32), (0.1 * rng.randn(H)).astype(np.float32)) for _ in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 192, 1024])
@pytest.mark.parametrize("kind", [0, 1, 2], ids=["fp32", "bf16", "fp16"])
def test_layernorm_matches_fp64(engine_small, dims_small, kind, H):
    """layernorm_kernel<fp32 | bf16 | fp16>: within one output rounding plus the fp32 slack of the fp64 LayerNorm, on rows with
    a 1e3 mean offset, variance below eps, a constant value (the output is exactly-rounded bias) and plain rows."""
    eps = dims_small.gpt.ln_eps
    rng = np.random.RandomState(H + 10 * kind)
    X = ln_rows(37, H, rng)
    (w, b), = _ln_params(H, rng, 1)
    Y, lat = engine_small.debug_norms(kind, X, w, b)
    assert lat is None
    (y_ref, s), = ref_ln_chain(X, [(w, b)], eps)
    h = HALF_ULP[kind]
    share = _check(Y, y_ref, h * np.abs(y_ref) + (1 + h) * s + 1e-30, (KIND_NAMES[kind], H))
    const = np.arange(37) % 4 == 2
    np.testing.assert_array_equal(Y[const], np.broadcast_to(rnd(b, kind)[1], Y[const].shape))
    print(f"layernorm {KIND_NAMES[kind]} H={H}, largest share of the error bound used {share:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 192, 1024])
@pytest.mark.parametrize("kind", [0, 1, 2], ids=["fp32", "bf16", "fp16"])
def test_head_norms_match_fp64_and_write_only_their_latent_rows(engine_small, dims_small, kind, H):
    """head_norms_kernel: Y = LN_fn(LN_lnf(X[row])) in the output type, latents = LN_fn(Y in fp32) in fp32, each within the
    chained fp64 bound.  Rows are picked through row_index (out of order, repeated) or taken in order; the latent position
    is lat_pos[i] or n_gen[slot].  Every latent row that is not some (slot, pos) with 0 <= pos < lat_rows keeps its NaN
    sentinel bit for bit — positions -1, lat_rows and beyond are dropped."""
    eps = dims_small.gpt.ln_eps
    rng = np.random.RandomState(H * 3 + kind)
    x_rows, n_slots, lat_rows = 23, 7, 5
    X = ln_rows(x_rows, H, rng)
    (w1, b1), (w2, b2) = _ln_params(H, rng, 2)
    sentinel = np.full((n_slots, lat_rows, H), np.nan, np.float32)
    sentinel.view(np.uint32)[:] = 0x7FC0DEAD
    h = HALF_ULP[kind]
    worst = 0.0
    cases = [
        # (row_index, slots, lat_pos, n_gen)
        (rng.permutation(x_rows)[:6], [3, 0, 6, 2, 5, 1], [0, lat_rows - 1, -1, lat_rows, 2, 1], None),
        (None, [4, 2, 0, 6, 1, 3, 5], None, [0, 1, lat_rows - 1, lat_rows, -1, 3, 7]),
        (np.array([5, 5, 0, 22]), [1, 2, 3, 4], [4, 4, 0, 3], None),
    ]
    for ci, (ri, slots, lat_pos, n_gen) in enumerate(cases):
        M = len(slots)
        Y, lat = engine_small.debug_norms(kind, X, w1, b1, w2, b2, M=M, row_index=ri, latents=sentinel, slots=slots,
                                          lat_pos=lat_pos, n_gen=n_gen)
        rows = np.asarray(ri) if ri is not None else np.arange(M)
        (_, _), (y_ref, s2), (l_ref, s3) = ref_ln_chain(X[rows], [(w1, b1), (w2, b2), (w2, b2)], eps)
        label = (KIND_NAMES[kind], H, ci)
        worst = max(worst, _check(Y, y_ref, h * np.abs(y_ref) + (1 + h) * s2 + 1e-30, (label, "Y")))
        # the latent LayerNorm runs on the fp32 y, not the rounded Y: its input error is s2 alone
        expect = sentinel.copy()
        written = np.zeros((n_slots, lat_rows), bool)
        for i, slot in enumerate(slots):
            p = lat_pos[i] if lat_pos is not None else n_gen[slot]
            if 0 <= p < lat_rows:
                written[slot, p] = True
                worst = max(worst, _check(lat[slot, p], l_ref[i], s3[i] + 1e-30, (label, "latent", i)))
        np.testing.assert_array_equal(bits(lat[~written]), bits(expect[~written]), err_msg=str(label))
        assert written.sum() >= 3, label
    print(f"head norms {KIND_NAMES[kind]} H={H}, largest share of the error bound used {worst:.3g}")


# ------------------------------------------------------------------------------------------------ KV write
@pytest.mark.gpu
@pytest.mark.parametrize("heads", [2, 16])
@pytest.mark.parametrize("kind", [0, 1, 2], ids=["fp32", "bf16", "fp16"])
def test_kv_write_places_every_element_exactly(engine_small, kind, heads):
    """kv_write_kernel (prefill): rows of several slots with non-contiguous, shuffled block tables at positions 0, 31, 32, 33,
    the last of a page and deeper, by row_pos and by ctx_len.  Every written element equals rnd(value, kind) exactly at its
    (page, head, token, dim) in the device layout; every other pool element keeps its NaN sentinel bit for bit."""
    rng = np.random.RandomState(heads + kind)
    H = heads * D
    n_slots, max_pages, n_pages = 5, 6, 40
    bt = rng.permutation(n_pages)[: n_slots * max_pages].reshape(n_slots, max_pages).astype(np.int32)
    positions = [0, 31, 32, 33, 63, 95, 64, 127, 150, 1]
    for use_ctx in (False, True):
        if use_ctx:
            slots = np.array([4, 0, 2, 3], np.int32)
            ctx_len = np.array([33, 7, 31, 64, 159], np.int32)
            pos = ctx_len[slots]
        else:
            slots = np.array([i % n_slots for i in range(len(positions))], np.int32)
            pos = np.array(positions, np.int32)
            ctx_len = None
        M = slots.size
        qkv = rng.randn(M, 3 * H).astype(np.float32)
        ktok = np.full((n_pages, heads, PT, D), np.nan, np.float32)
        kraw = rnd(ktok, kind)[0]
        kpool, vpool = pack_k(kraw, kind), pack_v(kraw)
        k_after, v_after = kraw.copy(), kraw.copy()
        knew = rnd(qkv[:, H:2 * H].reshape(M, heads, D), kind)[0]
        vnew = rnd(qkv[:, 2 * H:].reshape(M, heads, D), kind)[0]
        for r in range(M):
            pg = bt[slots[r], pos[r] // PT]
            k_after[pg, :, pos[r] % PT] = knew[r]
            v_after[pg, :, pos[r] % PT] = vnew[r]
        kp, vp = engine_small.debug_kv_write(kind, heads, qkv, slots, bt, kpool, vpool,
                                             row_pos=None if use_ctx else pos, ctx_len=ctx_len)
        label = (KIND_NAMES[kind], heads, use_ctx)
        np.testing.assert_array_equal(bits(kp), bits(pack_k(k_after, kind)), err_msg=str(label))
        np.testing.assert_array_equal(bits(vp), bits(pack_v(v_after)), err_msg=str(label))


# ------------------------------------------------------------------------------------------------ row builds
@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 1024])
def test_build_rows_match_float32_add(engine_small, H):
    """build_rows_kernel, all three RowDesc kinds in one launch, with indices at both ends of every table: each row equals
    the float32 numpy add of its two table rows (or the speaker row) exactly."""
    rng = np.random.RandomState(H)
    t = _tables(H, rng)
    rows = ([(0, a, 0, c) for c in (2, 0) for a in (0, 31, 7)] + [(1, a, b, 0) for a, b in ((0, 0), (10, 8), (5, 3), (10, 0))]
            + [(2, a, b, 0) for a, b in ((12, 0), (0, 9), (6, 4), (12, 9))] + [(0, 1, 5, 1)])
    rows = [rows[i] for i in rng.permutation(len(rows))]
    X = engine_small.debug_build_rows(rows, **t)
    np.testing.assert_array_equal(X, ref_build_rows(rows, t))


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 1024])
def test_build_decode_rows_and_counter_reset(engine_small, H):
    """build_decode_rows_kernel: X[i] = wte[last_tok[s]] + wpe[n_gen[s]] (s = active[i], shuffled, sparse slots) exactly as
    a float32 add; the first n_flags counter words become 0 and the guard words after them are untouched."""
    rng = np.random.RandomState(H + 1)
    t = _tables(H, rng)
    n_slots = 9
    last_tok = rng.randint(0, t["wte"].shape[0], n_slots).astype(np.int32)
    n_gen = rng.randint(0, t["wpe"].shape[0], n_slots).astype(np.int32)
    last_tok[0], n_gen[0] = t["wte"].shape[0] - 1, t["wpe"].shape[0] - 1
    for active, n_flags, guard in (([3, 0, 8, 5, 1], 4 * 2 * 7, 16), ([0], 0, 8), (list(rng.permutation(n_slots)), 4 * 30 * 7, 33)):
        counters = rng.randint(1, 2 ** 32 - 1, n_flags + guard, dtype=np.uint64).astype(np.uint32)
        X, after = engine_small.debug_build_decode_rows(active, last_tok, n_gen, t["wte"], t["wpe"], counters, n_flags)
        s = np.asarray(active)
        np.testing.assert_array_equal(X, t["wte"][last_tok[s]] + t["wpe"][n_gen[s]])
        np.testing.assert_array_equal(after[:n_flags], 0)
        np.testing.assert_array_equal(after[n_flags:], counters[n_flags:])


# ------------------------------------------------------------------------------------------------ end to end
OPTION_DEFAULTS = dict(dep_flags=0, pdl=1, branch_stagger_us=0, voc_batch=32)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["fp16", "bf16"])
def test_decode_execution_options_are_bit_identical(request, dims_full, which):
    """The decode step's non-default execution paths — dependency counters instead of griddepcontrol.wait ("dep_flags" 1),
    no programmatic dependent launch ("pdl" 0), a delayed second row branch ("branch_stagger_us" 50) — and one vocoder
    window per launch ("voc_batch" 1) change scheduling only.  With both row branches running (microbatch_min_rows 2) and
    the step replayed from CUDA graphs after its eager steps, tokens, latents and waveforms must equal the defaults' bit for
    bit."""
    eng = request.getfixturevalue(f"engine_full_{which}")
    g = dims_full.gpt
    jobs = [(i, text_ids(dims_full, 7 + 5 * i, 300 + i), i % 3,
             Sampling(temperature=0.75, top_p=0.85, top_k=50, repetition_penalty=5.0, max_tokens=18, seed=21, seq_seed=i,
                      stop_token=g.stop_audio_token)) for i in range(4)]
    try:
        eng.set_option("microbatch_min_rows", 2)
        ref = eng.run_batch(jobs, timeout_s=180, want_latents=True)
        for key, val in (("dep_flags", 1), ("pdl", 0), ("branch_stagger_us", 50), ("voc_batch", 1)):
            try:
                eng.set_option(key, val)
                got = eng.run_batch(jobs, timeout_s=180, want_latents=True)
            finally:
                eng.set_option(key, OPTION_DEFAULTS[key])
            for sid in ref:
                _, toks, wav, lat = got[sid]
                assert list(toks) == list(ref[sid][1]), (which, key, sid)
                np.testing.assert_array_equal(bits(lat), bits(ref[sid][3]), err_msg=str((which, key, sid)))
                np.testing.assert_array_equal(bits(wav), bits(ref[sid][2]), err_msg=str((which, key, sid)))
    finally:
        eng.set_option("microbatch_min_rows", 48)
        for k, v in OPTION_DEFAULTS.items():
            eng.set_option(k, v)
