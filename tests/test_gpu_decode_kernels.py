"""Decode-path kernels launched on their own and compared with a float64 numpy reference of the same operation:
the paged decode attention (register and bulk-copy forms, every warp count, ring depth, grid cap and L2 option), the
prefill / encoder attention (ragged launches, causal with nk >= nq, the three stride layouts the engine uses) and the
split-K GEMM with the fused residual + LayerNorm reduction.  The reference sees the operands rounded exactly as the kernel
rounds them (K/V to the cache type, GEMM operands to bf16 / fp16), so the bounds are one rounding of the output type plus
an fp32 arithmetic term.  The CPU tests check the KV layout packing and the references themselves."""
import numpy as np
import pytest
import torch

from auralis_b200.native import NativeEngine

PT, D = 32, 64                                  # tokens per KV page, head dim
U = 2.0 ** -24                                  # fp32 unit roundoff
HALF_ULP = {0: 0.0, 1: 2.0 ** -8, 2: 2.0 ** -11}   # one round-to-nearest into fp32 / bf16 / fp16 (half an ulp), relative
KV_NAMES = {0: "fp32", 1: "bf16", 2: "fp16"}
_F64 = np.float64


# ------------------------------------------------------------------------------------------------ rounding and layout
def rnd(x, kind):
    """fp32 values -> (raw elements of type `kind` as stored on the device, their exact float64 values).  Round to nearest
    even, as __float2bfloat16_rn / __float2half_rn; bf16 travels as its uint16 bit pattern."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    if kind == 0:
        return x.copy(), x.astype(_F64)
    if kind == 1:
        t = torch.from_numpy(x).to(torch.bfloat16)
        return t.view(torch.int16).numpy().view(np.uint16).copy(), t.to(torch.float64).numpy()
    h = x.astype(np.float16)
    return h, h.astype(_F64)


def raw_to_f64(raw, kind):
    if kind == 1:
        return torch.from_numpy(raw.view(np.int16).copy()).view(torch.bfloat16).to(torch.float64).numpy()
    return raw.astype(_F64)


def atom(kind):
    return 16 // (4 if kind == 0 else 2)        # elements per 16-byte K atom


def pack_k(tok, kind):
    """[pages, heads, 32 tok, 64] -> device K layout [pages, heads, 64/X * 32 * X]: [D/X][32 tok][X] per (page, head)."""
    X = atom(kind)
    p, h = tok.shape[:2]
    return np.ascontiguousarray(tok.reshape(p, h, PT, D // X, X).transpose(0, 1, 3, 2, 4)).reshape(p, h, PT * D)


def unpack_k(raw, kind):
    X = atom(kind)
    p, h = raw.shape[:2]
    return np.ascontiguousarray(raw.reshape(p, h, D // X, PT, X).transpose(0, 1, 3, 2, 4)).reshape(p, h, PT, D)


def pack_v(tok):
    """[pages, heads, 32 tok, 64] -> device V layout [pages, heads, 32 * 64] (token-major rows)."""
    return np.ascontiguousarray(tok).reshape(tok.shape[0], tok.shape[1], PT * D)


def bits(a):
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint16)


# ------------------------------------------------------------------------------------------------ float64 references
def ref_attention(q, k, v, scale, mask=None):
    """q [nq, 64] (fp32, pre-scaled in fp32 like the kernels), k / v [nk, 64] float64, mask [nq, nk] bool (True = visible).
    -> (out [nq, 64] float64, S [nq]: largest sum_d |q_d k_d| of a visible key, the conditioning of the scores)."""
    qs = (np.asarray(q, np.float32) * np.float32(scale)).astype(_F64)
    s = qs @ k.T
    a = np.abs(qs) @ np.abs(k).T
    if mask is not None:
        s = np.where(mask, s, -np.inf)
        a = np.where(mask, a, 0.0)
    p = np.exp(s - s.max(axis=1, keepdims=True))
    return (p @ v) / p.sum(axis=1, keepdims=True), a.max(axis=1)


def fp32_slack(vscale, S, n):
    """fp32 error of an online-softmax attention output: the score error (~ u * sum |q k|) goes through exp unchanged as a
    relative error of p, plus the accumulation over n keys — times the largest |v| attended."""
    return vscale * U * 8.0 * (S + np.sqrt(n) + 2.0)


def ref_layernorm(x, w, b, eps):
    x = x.astype(_F64)
    mu = x.mean(axis=1, keepdims=True)
    var = ((x - mu) ** 2).mean(axis=1, keepdims=True)
    rstd = 1.0 / np.sqrt(var + eps)
    return (x - mu) * rstd * w + b, mu, rstd


def causal_mask(nq, nk):
    """key j visible to query i iff j <= i + (nk - nq): the last query sees every key."""
    return np.arange(nk)[None, :] <= np.arange(nq)[:, None] + (nk - nq)


# ------------------------------------------------------------------------------------------------ CPU checks
@pytest.mark.parametrize("kind", [0, 1, 2], ids=["fp32", "bf16", "fp16"])
def test_kv_layout_packing_round_trips(kind):
    """The numpy packing is the layout of kernels.h: element (token t, dim d) of a (page, head) block sits at
    K: ((d / X) * 32 + t) * X + d % X,  V: t * 64 + d."""
    rng = np.random.RandomState(kind)
    tok = rng.randn(5, 3, PT, D).astype(np.float32)
    raw, _ = rnd(tok, kind)
    pk = pack_k(raw, kind)
    np.testing.assert_array_equal(bits(unpack_k(pk, kind)), bits(raw))
    X = atom(kind)
    for _ in range(200):
        p, h, t, d = rng.randint(5), rng.randint(3), rng.randint(PT), rng.randint(D)
        assert bits(pk[p, h, ((d // X) * PT + t) * X + d % X]) == bits(raw[p, h, t, d])
        assert bits(pack_v(raw)[p, h, t * D + d]) == bits(raw[p, h, t, d])


def test_rounding_is_round_to_nearest_even():
    """bf16 / fp16 rounding of the reference: exact ties go to the even neighbour, everything else to the nearest."""
    one_plus = np.array([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1.0 + 2.0 ** -8 + 2.0 ** -20], np.float32)
    np.testing.assert_array_equal(rnd(one_plus, 1)[1], [1.0, 1.0 + 2.0 ** -6, 1.0 + 2.0 ** -7])
    one_plus = np.array([1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11], np.float32)
    np.testing.assert_array_equal(rnd(one_plus, 2)[1], [1.0, 1.0 + 2.0 ** -9])
    x = np.random.RandomState(0).randn(1000).astype(np.float32)
    for kind in (1, 2):
        raw, f = rnd(x, kind)
        np.testing.assert_array_equal(raw_to_f64(raw, kind), f)
        assert np.abs(f - x).max() <= HALF_ULP[kind] * np.abs(x).max()
        assert (np.abs(f - x) <= HALF_ULP[kind] * np.abs(x)).all()


@pytest.mark.parametrize("nq,nk,causal", [(1, 1, True), (17, 17, True), (5, 40, True), (16, 16, False), (32, 47, False)])
def test_reference_attention_matches_sdpa(nq, nk, causal):
    rng = np.random.RandomState(nq * 100 + nk)
    q, k, v = rng.randn(nq, D).astype(np.float32), rng.randn(nk, D), rng.randn(nk, D)
    mask = causal_mask(nq, nk) if causal else None
    got, _ = ref_attention(q, k, v, 0.125, mask)
    tq, tk, tv = (torch.from_numpy(np.asarray(a, _F64))[None, None] for a in (q, k, v))
    # torch's own causal flag aligns the mask top-left; bottom-right (what the kernels do) is an explicit lower band
    tm = torch.ones(nq, nk, dtype=torch.bool).tril(diagonal=nk - nq) if causal else None
    exp = torch.nn.functional.scaled_dot_product_attention(tq, tk, tv, attn_mask=tm, scale=0.125)[0, 0].numpy()
    np.testing.assert_allclose(got, exp, rtol=1e-12, atol=1e-12)
    if causal and nq == nk:
        exp2 = torch.nn.functional.scaled_dot_product_attention(tq, tk, tv, is_causal=True, scale=0.125)[0, 0].numpy()
        np.testing.assert_allclose(got, exp2, rtol=1e-12, atol=1e-12)


def test_reference_layernorm_matches_torch():
    rng = np.random.RandomState(3)
    x = rng.randn(7, 96) * np.array([1.0, 1.0, 1e-3, 5.0, 1.0, 1.0, 1.0])[:, None] + np.array([0, 1e3, 0, -7, 0, 0, 2])[:, None]
    w, b = rng.randn(96), rng.randn(96)
    got, _, _ = ref_layernorm(x, w, b, 1e-5)
    exp = torch.nn.functional.layer_norm(torch.from_numpy(x), (96,), torch.from_numpy(w), torch.from_numpy(b), eps=1e-5).numpy()
    np.testing.assert_allclose(got, exp, rtol=1e-10, atol=1e-10)


# ------------------------------------------------------------------------------------------------ decode attention
ATTN_DEFAULTS = dict(attn_warps=4, attn_bulk=0, attn_stages=8, attn_ctas_per_sm=0, attn_l2_ahead=1, attn_l2_pages=0)
ATTN_VARIANTS = (
    [dict(attn_warps=w) for w in (1, 2, 4, 8, 16)]                                         # register kernel
    + [dict(attn_bulk=1, attn_warps=w, attn_stages=s) for w in (4, 8, 16) for s in (4, 8, 24)]   # bulk-copy kernel
    + [dict(attn_ctas_per_sm=g) for g in (-1, -3, -1000)]                                   # grid caps (0 is above)
    + [dict(attn_bulk=1, attn_ctas_per_sm=g) for g in (0, -1, -3, -1000)]
    + [dict(attn_warps=16, attn_ctas_per_sm=-3), dict(attn_bulk=1, attn_warps=16, attn_stages=24, attn_ctas_per_sm=-1)]
    + [dict(attn_bulk=1, attn_l2_ahead=0), dict(attn_l2_pages=3), dict(attn_warps=1, attn_l2_pages=3)]
)

# rows of one launch: (cached tokens, style); styles: rand; big (scores ~ +-80: exp overflows without the max shift);
# first / last / self (one key dominates: in the first page, the last cached token, the step's own token); equal (all
# keys identical).  Contexts cross every page boundary and the 32-page round of the bulk producer (33 pages at 1041).
DECODE_CASES = [
    ([(0, "rand"), (1041, "rand"), (31, "rand"), (1, "rand"), (1024, "rand"), (63, "rand"), (33, "rand"), (500, "rand"),
      (65, "rand")], 12),
    ([(32, "equal"), (1025, "big"), (64, "first"), (97, "last"), (1023, "self"), (1041, "first"), (0, "self"), (33, "big"),
      (31, "last")], 13),
    ([(1041, "last")], 3),
    ([(97, "equal")], 2),
]
MAX_PAGES = 33                                  # 32 + 404 + 1 + 605 tokens of the full geometry


def _decode_case(kind, heads, rows, n_slots, seed):
    rng = np.random.RandomState(seed)
    M, H = len(rows), heads * D
    slots = rng.permutation(n_slots)[:M]        # permuted, skipping slots
    ctx_len = rng.randint(0, 50, n_slots).astype(np.int32)          # (unused slots: never read)
    need = [c // PT + 1 for c, _ in rows]                            # pages incl. the one the new token goes to
    n_pages = sum(need) + 24
    perm = rng.permutation(n_pages)
    unowned = perm[sum(need):]
    bt = np.full((n_slots, MAX_PAGES), unowned[0], np.int32)         # entries past a slot's pages: a poisoned page
    ktok = np.full((n_pages, heads, PT, D), np.nan, np.float32)     # every unowned page and page tail is NaN
    vtok = np.full_like(ktok, np.nan)
    qkv = np.zeros((M, 3 * H), np.float32)
    off = 0
    for i, (past, style) in enumerate(rows):
        s = slots[i]
        ctx_len[s] = past
        bt[s, :need[i]] = perm[off:off + need[i]]
        off += need[i]
        q = rng.randn(heads, D)
        k = rng.randn(heads, past + 1, D)        # [.., past] = the step's own token
        v = rng.randn(heads, past + 1, D)
        if style == "big":
            q, k = 10.0 * q, 8.0 * k
        elif style == "equal":
            k[:] = rng.randn(heads, 1, D)
        elif style in ("first", "last", "self"):
            k *= 0.3
            j = {"first": 0, "last": max(past - 1, 0), "self": past}[style]
            k[:, j] = q * (30.0 / (0.125 * (q * q).sum(axis=1, keepdims=True)))     # score ~ +30 over the rest
        t = np.arange(past)
        ktok[bt[s, t // PT], :, t % PT] = k[:, :past].transpose(1, 0, 2)
        vtok[bt[s, t // PT], :, t % PT] = v[:, :past].transpose(1, 0, 2)
        qkv[i, :H], qkv[i, H:2 * H], qkv[i, 2 * H:] = q.reshape(-1), k[:, past].reshape(-1), v[:, past].reshape(-1)
    kraw, kf = rnd(ktok, kind)
    vraw, vf = rnd(vtok, kind)
    # expected output and pools
    knew_raw, knew = rnd(qkv[:, H:2 * H].reshape(M, heads, D), kind)
    vnew_raw, vnew = rnd(qkv[:, 2 * H:].reshape(M, heads, D), kind)
    ref = np.zeros((M, heads, D))
    slack = np.zeros((M, heads, 1))
    k_after, v_after = kraw.copy(), vraw.copy()
    for i, (past, _) in enumerate(rows):
        s, t = slots[i], np.arange(past)
        pg = bt[s, past // PT]
        k_after[pg, :, past % PT], v_after[pg, :, past % PT] = knew_raw[i], vnew_raw[i]
        for h in range(heads):
            K = np.concatenate([kf[bt[s, t // PT], h, t % PT], knew[i, h][None]])
            V = np.concatenate([vf[bt[s, t // PT], h, t % PT], vnew[i, h][None]])
            o, S = ref_attention(qkv[i, h * D:(h + 1) * D][None], K, V, 0.125)
            ref[i, h] = o[0]
            slack[i, h] = fp32_slack(np.abs(V).max(), S[0], past + 1)
    return dict(M=M, heads=heads, qkv=qkv, active=slots.astype(np.int32), ctx_len=ctx_len, bt=bt,
                kpool=pack_k(kraw, kind), vpool=pack_v(vraw), k_after=pack_k(k_after, kind), v_after=pack_v(v_after),
                ref=ref, slack=slack)


def _set_options(eng, opts):
    for k, v in {**ATTN_DEFAULTS, **opts}.items():
        eng.set_option(k, v)


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [2, 16])
@pytest.mark.parametrize("kind", [0, 1, 2], ids=["fp32", "bf16", "fp16"])
def test_decode_attention_matches_fp64(engine_small, kind, heads):
    """Output within one rounding of the cache type (plus fp32 slack) of the float64 attention over the rounded cache and the
    step's own token; NaN in every unowned page and page tail never reaches the output; both pools bit-identical to their
    input except the M x heads appended positions, which hold the rounded k / v of the QKV row; every variant with the same
    warp count (register or bulk kernel, any ring depth, grid cap or L2 option) gives the same bits."""
    eng = engine_small
    variants = ATTN_VARIANTS if kind else [v for v in ATTN_VARIANTS if not v.get("attn_bulk") and v.get("attn_warps", 4) == 4]
    dt = NativeEngine.KV_DTYPES[kind]
    worst = {}
    try:
        for ci, (rows, n_slots) in enumerate(DECODE_CASES):
            c = _decode_case(kind, heads, rows, n_slots, seed=100 * ci + heads + kind)
            assert c["kpool"].dtype == dt
            by_warps = {}
            for opts in variants:
                _set_options(eng, opts)
                out, kp, vp = eng.debug_attn_decode(kind, heads, c["qkv"], c["active"], c["ctx_len"], c["bt"], c["kpool"], c["vpool"])
                out = out.reshape(c["M"], heads, D)
                label = (KV_NAMES[kind], heads, ci, opts)
                assert np.isfinite(out).all(), label
                tol = HALF_ULP[kind] * np.abs(c["ref"]) + c["slack"]
                err = np.abs(out - c["ref"])
                bad = np.argwhere(err > tol)
                assert bad.size == 0, (label, bad[:5].tolist(), float((err / tol).max()))
                np.testing.assert_array_equal(bits(kp), bits(c["k_after"]), err_msg=str(label))
                np.testing.assert_array_equal(bits(vp), bits(c["v_after"]), err_msg=str(label))
                nw = opts.get("attn_warps", 4) if kind else 4
                if nw in by_warps:
                    np.testing.assert_array_equal(out, by_warps[nw], err_msg=str(label))
                by_warps.setdefault(nw, out)
                key = ("bulk" if opts.get("attn_bulk") else "reg") + f"{nw}w"
                worst[key] = max(worst.get(key, 0.0), float((err / tol).max()))
    finally:
        _set_options(eng, {})
    print(f"decode attention {KV_NAMES[kind]} heads={heads}, largest share of the error bound used: "
          + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))


# ------------------------------------------------------------------------------------------------ prefill attention
def _prefill_check(out, ref, slack, kind, rows_written, label):
    assert np.isfinite(out[rows_written]).all(), label
    unwritten = np.setdiff1d(np.arange(out.shape[0]), rows_written)
    assert np.isnan(out[unwritten]).all(), label                # nothing written outside the sequences
    got = out[rows_written]
    err = np.abs(got - ref)
    tol = HALF_ULP[kind] * np.abs(ref) + slack
    bad = np.argwhere(err > tol)
    assert bad.size == 0, (label, bad[:5].tolist(), float((err / tol).max()))
    return float((err / tol).max())


def _ref_rows(qrows, krows, vrows, heads, scale, mask):
    """per-head reference of one sequence: q rows [nq, heads, 64], k / v rows [nk, heads, 64] -> out [nq, heads*64] and
    its fp32 slack [nq, heads*64]"""
    nq, nk = qrows.shape[0], krows.shape[0]
    out, sl = np.zeros((nq, heads, D)), np.zeros((nq, heads, 1))
    for h in range(heads):
        o, S = ref_attention(qrows[:, h], krows[:, h].astype(_F64), vrows[:, h].astype(_F64), scale, mask)
        out[:, h] = o
        vis = mask if mask is not None else np.ones((nq, nk), bool)
        vmax = np.array([np.abs(vrows[vis[i], h]).max() for i in range(nq)])
        sl[:, h, 0] = fp32_slack(vmax, S, nk)
    return out.reshape(nq, -1), np.broadcast_to(sl, (nq, heads, D)).reshape(nq, -1)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [0, 1, 2], ids=["fp32", "bf16", "fp16"])
def test_prefill_attention_gpt_layout(engine_small, kind):
    """GPT prefill layout (one QKV row [q | k | v], head stride 64), causal: a ragged launch of sequences with nq in
    {1, 15, 16, 17, 33, 250} (most CTAs of the short ones exit at once), with nk == nq and with nk > nq (keys before the
    first query; key j visible to query i iff j <= i + nk - nq), 16 heads."""
    heads, H = 16, 16 * D
    rng = np.random.RandomState(7 + kind)
    worst = 0.0
    for extra in (0, 40):                                            # nk - nq
        seqs, start = [], 3                                          # rows 0..2 belong to no sequence
        for nq in (250, 1, 15, 16, 17, 33):
            nk = nq + extra
            seqs.append((start + extra, nq, start, nk))              # queries are the last nq of the nk rows
            start += nk + 2
        rows = start + 1
        qkv = rng.randn(rows, 3 * H).astype(np.float32)
        out = engine_small.debug_attn_prefill(kind, heads, seqs, True, 0.125, qkv, 3 * H, D, qkv, 3 * H, D, H, 2 * H, rows)
        written = np.concatenate([np.arange(s[0], s[0] + s[1]) for s in seqs])
        ref, slack = np.zeros((rows, H)), np.zeros((rows, H))
        r = qkv.reshape(rows, 3, heads, D)
        for (qs, nq, ks, nk) in seqs:
            ref[qs:qs + nq], slack[qs:qs + nq] = _ref_rows(r[qs:qs + nq, 0], r[ks:ks + nk, 1], r[ks:ks + nk, 2], heads, 0.125,
                                                          causal_mask(nq, nk))
        worst = max(worst, _prefill_check(out, ref[written], slack[written], kind, written, (KV_NAMES[kind], extra)))
    print(f"prefill attention (GPT layout) {KV_NAMES[kind]}: largest share of the error bound used {worst:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [0, 1, 2], ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("T", [15, 33, 250])
def test_prefill_attention_conditioning_layouts(engine_small, kind, T):
    """The two non-causal uses in cond.cu: the conditioning encoder (q / k / v interleaved per head, head stride 3 * 64,
    nq = nk = T) and the perceiver (separate q [32, inner] and kv [32 + T, 2 * inner] buffers, nq = 32, nk = 32 + T)."""
    rng = np.random.RandomState(T + 10 * kind)
    worst = 0.0
    # conditioning encoder, 16 heads
    heads, H = 16, 16 * D
    qkv = rng.randn(T, 3 * H).astype(np.float32)
    out = engine_small.debug_attn_prefill(kind, heads, [(0, T, 0, T)], False, 0.125, qkv, 3 * H, 3 * D, qkv, 3 * H, 3 * D, D, 2 * D, T + 2)
    r = qkv.reshape(T, heads, 3, D)
    ref, slack = _ref_rows(r[:, :, 0], r[:, :, 1], r[:, :, 2], heads, 0.125, None)
    worst = max(worst, _prefill_check(out, ref, slack, kind, np.arange(T), ("encoder", KV_NAMES[kind], T)))
    # perceiver, 8 heads of 64 (inner = 512)
    heads, inner, NC = 8, 8 * D, 32
    q = rng.randn(NC, inner).astype(np.float32)
    kv = rng.randn(NC + T, 2 * inner).astype(np.float32)
    out = engine_small.debug_attn_prefill(kind, heads, [(0, NC, 0, NC + T)], False, 0.125, q, inner, D, kv, 2 * inner, D, 0, inner, NC + 1)
    ref, slack = _ref_rows(q.reshape(NC, heads, D), kv[:, :inner].reshape(NC + T, heads, D), kv[:, inner:].reshape(NC + T, heads, D),
                           heads, 0.125, None)
    worst = max(worst, _prefill_check(out, ref, slack, kind, np.arange(NC), ("perceiver", KV_NAMES[kind], T)))
    print(f"prefill attention (conditioning layouts) {KV_NAMES[kind]} T={T}: largest share of the error bound used {worst:.3g}")


# ------------------------------------------------------------------------------------------------ split-K + reduce / LN
def _splitk_data(M, H, K, seed):
    """Rows cycle through three kinds: a residual with a ~1e3 mean offset (two-pass variance), a row whose new X has a
    spread of ~1e-3 (variance below eps: the eps term matters), and a plain one."""
    rng = np.random.RandomState(seed)
    A = rng.randn(M, K).astype(np.float32)
    W = (rng.randn(H, K) * 0.05).astype(np.float32)
    bias = rng.randn(H).astype(np.float32)
    X = rng.randn(M, H).astype(np.float32)
    for i in range(M):
        if i % 3 == 0:
            X[i] += np.float32(1e3)
        elif i % 3 == 1:
            A[i] = 0.0
            X[i] = -bias + np.float32(1e-3) * rng.randn(H).astype(np.float32)
    ln_w = (1.0 + 0.1 * rng.randn(H)).astype(np.float32)
    ln_b = (0.1 * rng.randn(H)).astype(np.float32)
    return A, W, bias, X, ln_w, ln_b


SPLITK_M = (1, 2, 8, 9, 17, 33, 65)


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 1024])
@pytest.mark.parametrize("mode", [1, 2], ids=["bf16", "fp16"])
def test_splitk_reduce_layernorm_matches_fp64(engine_small, dims_small, mode, H):
    """X' = X + bias + A16 . W16^T within fp32 accumulation error; Y = LN(X') within one output rounding of the float64
    LayerNorm of the kernel's X'; the last-layer form (no LN) updates X alone; repeated runs give the same bits.  Shapes: the
    engine's K = H / 4 splits and K = 4H / 8 splits, plus 1 and 2 splits; every M tile and A-box branch; gemm_bn forced."""
    eng = engine_small
    eps = dims_small.gpt.ln_eps
    rnd16 = (lambda a: rnd(a, mode)[1])
    worst_x = worst_y = 0.0
    shapes = [(K, s) for K, s in ((H, 4), (4 * H, 8), (H, 1), (H, 2)) if (K // 64) % s == 0]
    try:
        for K, splits in shapes:
            for M in SPLITK_M:
                A, W, bias, X, ln_w, ln_b = _splitk_data(M, H, K, seed=M * 31 + K + splits)
                prod = rnd16(A) @ rnd16(W).T
                x_ref = X.astype(_F64) + bias + prod
                # fp32 additions of the residual, bias and partials (16 u each), the tensor-core accumulation over K (1e-5 of
                # sum |a w|)
                x_tol = 16 * U * (np.abs(X) + np.abs(bias) + np.abs(prod)) + 1e-5 * (np.abs(rnd16(A)) @ np.abs(rnd16(W)).T) + 1e-30
                for bn in (0, 32, 64, 128):
                    eng.set_option("gemm_bn", bn)
                    label = (mode, M, H, K, splits, bn)
                    x1, y1 = eng.debug_splitk_ln(mode, A, W, bias, X, splits, ln_w, ln_b)
                    assert np.isfinite(x1).all() and np.isfinite(y1).all(), label
                    ex = np.abs(x1 - x_ref)
                    assert (ex <= x_tol).all(), (label, "X", np.argwhere(ex > x_tol)[:5].tolist())
                    y_ref, mu, rstd = ref_layernorm(x1, ln_w, ln_b, eps)
                    xh = np.abs((x1 - mu) * rstd)
                    # fp32 statistics: the mean's error (~ u |mean| per reduction level) scaled by rstd, the normalised value's
                    y_slack = U * ((16 * np.abs(mu) * rstd + 32 * (xh + 1.0)) * np.abs(ln_w) + 32 * np.abs(ln_b))
                    ey = np.abs(y1 - y_ref)
                    y_tol = HALF_ULP[mode] * np.abs(y_ref) + y_slack
                    assert (ey <= y_tol).all(), (label, "Y", np.argwhere(ey > y_tol)[:5].tolist(), float((ey / y_tol).max()))
                    worst_x = max(worst_x, float((ex / x_tol).max()))
                    worst_y = max(worst_y, float((ey / y_tol).max()))
                    if bn == 0:
                        x2, y2 = eng.debug_splitk_ln(mode, A, W, bias, X, splits, ln_w, ln_b)
                        np.testing.assert_array_equal(x2, x1, err_msg=str(label))
                        np.testing.assert_array_equal(y2, y1, err_msg=str(label))
                        x3, y3 = eng.debug_splitk_ln(mode, A, W, bias, X, splits)           # last layer: X only
                        assert y3 is None
                        np.testing.assert_array_equal(x3, x1, err_msg=str(label))
    finally:
        eng.set_option("gemm_bn", 0)
    print(f"split-K + reduce/LN {'bf16' if mode == 1 else 'fp16'} H={H}, largest share of the error bound used: "
          f"X {worst_x:.3g}, Y {worst_y:.3g}")
