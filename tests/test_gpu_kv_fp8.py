"""GPU: the fp8 KV cache (engine option "kv_fp8", kv_cache_dtype="fp8").  The kernels in isolation against the host
quantiser of tests/test_kv_fp8_host.py — the prefill write and the decode attention's append bit for bit, the attention
output against float64 attention over the dequantised cache, the beam fork's partial-page copy with its exponents — and
the engine: teacher-forced and greedy runs against the fp32 oracle, determinism at the bench batch, the option's round trip,
its refusals, beam search and the halved KV pool."""
import numpy as np
import pytest
import torch

from auralis_b200.native import ERR_INVALID, NativeError, Sampling
from oracle import xtts_oracle as O
from conftest import text_ids, _make_engine
from test_gpu_decode_kernels import ATTN_VARIANTS, DECODE_CASES, HALF_ULP, MAX_PAGES, _set_options, fp32_slack, ref_attention
from test_gpu_beam_kernels import HEADS, LAYERS, MP, CAP, _logits, _seen, _sp, _state
from test_gpu_gpt import _margin_report
from test_kv_fp8_host import BLOCK, D, PT, dequantize, pack, quantize, unpack

pytestmark = pytest.mark.gpu

OUT_KIND = {3: 2, 4: 1}                 # kv_type -> the 16-bit output type (HALF_ULP key): 3 fp16 out, 4 bf16 out
NO_STOP = 4095
ERR_STATE = -3                          # XTTS_ERR_STATE


def _poisoned_pool(rng, n_pages, heads):
    """random bytes, e4m3 NaN (0x7F) in every data byte: whatever a test does not write must never reach an output"""
    pool = rng.randint(-128, 128, size=(n_pages, heads, BLOCK)).astype(np.int8).view(np.uint8)
    pool[..., :PT * D] = 0x7F
    return pool


# ------------------------------------------------------------------------------------------------ kernels in isolation
@pytest.mark.parametrize("kv_type", [3, 4])
def test_kv_write_matches_host_quantiser(engine_small_fp16, kv_type):
    """k / v of each row quantised per head with their own exponents, written at (page, head, token) of the row's slot and
    position, bit-identical to the host quantiser; every other byte, exponents included, untouched.  Rows address several
    slots, positions in first / middle / last page slots and permuted page ids, through row_pos and through ctx_len."""
    eng = engine_small_fp16
    rng = np.random.RandomState(kv_type)
    heads, n_slots, mp, n_pages = 16, 5, 6, 40
    H = heads * D
    bt = rng.permutation(n_pages)[: n_slots * mp].reshape(n_slots, mp).astype(np.int32)
    for use_pos in (True, False):
        M = 23 if use_pos else n_slots
        row_slot = (rng.permutation(np.arange(M) % n_slots) if use_pos else rng.permutation(n_slots)).astype(np.int32)
        seen = {}                                       # distinct (slot, position) pairs
        pos = np.zeros(M, np.int32)
        for i, s in enumerate(row_slot):
            seen[s] = seen.get(s, -1) + 1
            pos[i] = [0, 1, 31, 32, 63, 95, 100, 150, 191][(seen[s] + 2 * int(s)) % 9]
        ctx = np.zeros(n_slots, np.int32)
        if not use_pos:
            ctx[row_slot] = pos
        qkv = rng.randn(M, 3 * H).astype(np.float32) * np.exp2(rng.randint(-20, 20, size=(M, 1))).astype(np.float32)
        qkv[0, H:H + D] = 0.0                                                   # an all-zero K row: exponent -128
        kpool, vpool = _poisoned_pool(rng, n_pages, heads), _poisoned_pool(rng, n_pages, heads)
        k_exp, v_exp = kpool.copy(), vpool.copy()
        for r in range(M):
            page, t = bt[row_slot[r], pos[r] // PT], pos[r] % PT
            for blocks, src in ((k_exp, qkv[r, H:2 * H]), (v_exp, qkv[r, 2 * H:])):
                kv = "k" if blocks is k_exp else "v"
                qd, ed = unpack(blocks[page:page + 1], kv)
                q, e = quantize(src.reshape(heads, D))
                qd[0, :, t], ed[0, :, t] = q, e
                blocks[page:page + 1] = pack(qd, ed, kv)
        kp, vp = eng.debug_kv_write(kv_type, heads, qkv, row_slot, bt, kpool, vpool,
                                    row_pos=pos if use_pos else None, ctx_len=None if use_pos else ctx)
        np.testing.assert_array_equal(kp, k_exp, err_msg=f"K use_pos={use_pos}")
        np.testing.assert_array_equal(vp, v_exp, err_msg=f"V use_pos={use_pos}")
        assert unpack(kp, "k")[1][bt[row_slot[0], pos[0] // PT], 0, pos[0] % PT] == -128


def _decode_case8(heads, rows, n_slots, seed):
    """test_gpu_decode_kernels._decode_case for the fp8 cache: the cached tokens quantised by the host quantiser, page tails
    and unowned pages poisoned; the reference attends over the dequantised cache and the step's own token dequantised."""
    rng = np.random.RandomState(seed)
    M, H = len(rows), heads * D
    slots = rng.permutation(n_slots)[:M]
    ctx_len = rng.randint(0, 50, n_slots).astype(np.int32)
    need = [c // PT + 1 for c, _ in rows]
    n_pages = sum(need) + 24
    perm = rng.permutation(n_pages)
    bt = np.full((n_slots, MAX_PAGES), perm[sum(need):][0], np.int32)
    kq = np.full((n_pages, heads, PT, D), 0x7F, np.uint8)
    vq = kq.copy()
    ke = rng.randint(-128, 128, size=(n_pages, heads, PT)).astype(np.int8)
    ve = rng.randint(-128, 128, size=(n_pages, heads, PT)).astype(np.int8)
    qkv = np.zeros((M, 3 * H), np.float32)
    off = 0
    toks = []
    for i, (past, style) in enumerate(rows):
        s = slots[i]
        ctx_len[s] = past
        bt[s, :need[i]] = perm[off:off + need[i]]
        off += need[i]
        q = rng.randn(heads, D)
        k = rng.randn(heads, past + 1, D) * np.exp2(rng.randint(-3, 4, size=(1, past + 1, 1)))    # per-token scales
        v = rng.randn(heads, past + 1, D) * np.exp2(rng.randint(-3, 4, size=(1, past + 1, 1)))
        if style == "big":
            q, k = 10.0 * q, 8.0 * k
        elif style == "equal":
            k[:] = rng.randn(heads, 1, D)
        elif style in ("first", "last", "self"):
            k *= 0.3
            j = {"first": 0, "last": max(past - 1, 0), "self": past}[style]
            k[:, j] = q * (30.0 / (0.125 * (q * q).sum(axis=1, keepdims=True)))
        k, v = k.astype(np.float32), v.astype(np.float32)
        t = np.arange(past)
        kqi, kei = quantize(k[:, :past].transpose(1, 0, 2))
        vqi, vei = quantize(v[:, :past].transpose(1, 0, 2))
        kq[bt[s, t // PT], :, t % PT], ke[bt[s, t // PT], :, t % PT] = kqi, kei
        vq[bt[s, t // PT], :, t % PT], ve[bt[s, t // PT], :, t % PT] = vqi, vei
        qkv[i, :H], qkv[i, H:2 * H], qkv[i, 2 * H:] = q.reshape(-1), k[:, past].reshape(-1), v[:, past].reshape(-1)
        toks.append(t)
    kpool, vpool = pack(kq, ke, "k"), pack(vq, ve, "v")
    k_after, v_after = kpool.copy(), vpool.copy()
    ref, slack = np.zeros((M, heads, D)), np.zeros((M, heads, 1))
    kdeq, vdeq = dequantize(kq, ke), dequantize(vq, ve)
    for i, (past, _) in enumerate(rows):
        s, t = slots[i], toks[i]
        knq, kne = quantize(qkv[i, H:2 * H].reshape(heads, D))
        vnq, vne = quantize(qkv[i, 2 * H:].reshape(heads, D))
        pg = bt[s, past // PT]
        for blocks, nq, ne, kv in ((k_after, knq, kne, "k"), (v_after, vnq, vne, "v")):
            qd, ed = unpack(blocks[pg:pg + 1], kv)
            qd[0, :, past % PT], ed[0, :, past % PT] = nq, ne
            blocks[pg:pg + 1] = pack(qd, ed, kv)
        knew, vnew = dequantize(knq, kne), dequantize(vnq, vne)
        for h in range(heads):
            K = np.concatenate([kdeq[bt[s, t // PT], h, t % PT], knew[h][None]])
            V = np.concatenate([vdeq[bt[s, t // PT], h, t % PT], vnew[h][None]])
            o, S = ref_attention(qkv[i, h * D:(h + 1) * D][None], K, V, 0.125)
            ref[i, h] = o[0]
            slack[i, h] = fp32_slack(np.abs(V).max(), S[0], past + 1)
    return dict(M=M, qkv=qkv, active=slots.astype(np.int32), ctx_len=ctx_len, bt=bt, kpool=kpool, vpool=vpool,
                k_after=k_after, v_after=v_after, ref=ref, slack=slack)


@pytest.mark.parametrize("heads", [1, 16])
@pytest.mark.parametrize("kv_type", [3, 4], ids=["fp16out", "bf16out"])
def test_decode_attention_fp8_matches_fp64(engine_small_fp16, kv_type, heads):
    """fp8 decode attention within one rounding of the output type plus the fp32 slack (the 16-bit kinds' bound) of the
    float64 attention over the dequantised cache and the dequantised own token; poisoned page tails never reach the output;
    the pools come back with exactly the appended bytes and exponents, which equal what the prefill write stores for the
    same rows; every grid cap gives the same bits.  Contexts of 0 .. 1041 tokens: several pages, partial last pages."""
    eng = engine_small_fp16
    worst = 0.0
    try:
        for ci, (rows, n_slots) in enumerate(DECODE_CASES):
            c = _decode_case8(heads, rows, n_slots, seed=200 * ci + heads + kv_type)
            first = None
            for opts in ATTN_VARIANTS:
                _set_options(eng, opts)
                out, kp, vp = eng.debug_attn_decode(kv_type, heads, c["qkv"], c["active"], c["ctx_len"], c["bt"],
                                                    c["kpool"], c["vpool"])
                out = out.reshape(c["M"], heads, D)
                label = (kv_type, heads, ci, opts)
                assert np.isfinite(out).all(), label
                tol = HALF_ULP[OUT_KIND[kv_type]] * np.abs(c["ref"]) + c["slack"]
                err = np.abs(out - c["ref"])
                bad = np.argwhere(err > tol)
                assert bad.size == 0, (label, bad[:5].tolist(), float((err / tol).max()))
                np.testing.assert_array_equal(kp, c["k_after"], err_msg=str(label))
                np.testing.assert_array_equal(vp, c["v_after"], err_msg=str(label))
                if first is None:
                    first = out
                    kw, vw = eng.debug_kv_write(kv_type, heads, c["qkv"], c["active"], c["bt"], c["kpool"], c["vpool"],
                                                ctx_len=c["ctx_len"])
                    np.testing.assert_array_equal(kw, kp, err_msg=str(label))
                    np.testing.assert_array_equal(vw, vp, err_msg=str(label))
                np.testing.assert_array_equal(out, first, err_msg=str(label))
                worst = max(worst, float((err / tol).max()))
    finally:
        _set_options(eng, {})
    print(f"fp8 decode attention kv_type={kv_type} heads={heads}: largest share of the error bound used {worst:.3g}")


def test_beam_fork_copies_fp8_bytes_and_exponents(engine_small_fp16):
    """a decode step of a 4-beam group whose beam 0 gives two children: the forked partial page receives the parent's
    e4m3 bytes and exponents of the copied tokens; the rest of that page and every other page stay as they were"""
    eng = engine_small_fp16
    rng = np.random.RandomState(31)
    nb, L = 4, 70
    sp = _sp(nb, 1.0)
    lg = _logits(rng, nb)
    lg[0, 7] = lg[0, 11] = 30.0
    bt = np.full((nb, MP), -1, np.int32)
    for j in range(nb):
        bt[j, 0], bt[j, 1], bt[j, 2] = 0, 1 + j // 2, 1 + (nb + 1) // 2 + j
    n_used, n_free = 1 + (nb + 1) // 2 + nb, nb
    n_pages = n_used + n_free
    pool = np.full(nb * MP, -1, np.int32)
    pool[:n_free] = rng.permutation(np.arange(n_used, n_pages)).astype(np.int32)
    page = HEADS * BLOCK
    kp = rng.randint(0, 256, size=LAYERS * n_pages * page).astype(np.uint8)
    vp = rng.randint(0, 256, size=LAYERS * n_pages * page).astype(np.uint8)
    st = _state(nb, False, n_free, -(-L // 32))
    k0, v0 = kp.copy(), vp.copy()
    seen = _seen(nb, [[3, 9], [4], [], [500]])
    hist = np.full((CAP, 8, 2), -7, np.int32)
    eng.debug_beam_step(3, HEADS, LAYERS, sp, False, 1, lg, np.full(nb, 5, np.int32), np.full(nb, L - 1, np.int32), seen,
                        bt, pool, hist, st, kp, vp)
    copies = [(st.copy_src[c], st.copy_dst[c], st.copy_ntok[c]) for c in range(st.n_copy)]
    assert copies and all(n == L % 32 for _, _, n in copies)
    dsts = {d for _, d, _ in copies}
    for name, before, after in (("k", k0, kp), ("v", v0, vp)):
        b = before.reshape(LAYERS, n_pages, HEADS, BLOCK)
        a = after.reshape(LAYERS, n_pages, HEADS, BLOCK)
        keep = [p for p in range(n_pages) if p not in dsts]
        np.testing.assert_array_equal(a[:, keep], b[:, keep])
        for src, dst, n in copies:
            got_q, got_e = unpack(a[:, dst], name)
            src_q, src_e = unpack(b[:, src], name)
            old_q, old_e = unpack(b[:, dst], name)
            np.testing.assert_array_equal(got_q[:, :, :n], src_q[:, :, :n])
            np.testing.assert_array_equal(got_e[:, :, :n], src_e[:, :, :n])
            np.testing.assert_array_equal(got_q[:, :, n:], old_q[:, :, n:])
            np.testing.assert_array_equal(got_e[:, :, n:], old_e[:, :, n:])


# ------------------------------------------------------------------------------------------------ engine
def _fp8_engine(dims, state, speakers, precision, max_batch):
    eng = _make_engine(dims, state, speakers, precision, max_batch=max_batch)
    eng.set_option("kv_fp8", 1)
    return eng


@pytest.fixture(scope="module")
def fp8_small(dims_small, state_small, speakers_small):
    engs = {p: _fp8_engine(dims_small, state_small, speakers_small, p, 8) for p in (1, 2)}
    yield engs
    for e in engs.values():
        e.close()


@pytest.fixture(scope="module")
def fp8_full(dims_full, state_full, speakers_full):
    engs = {p: _fp8_engine(dims_full, state_full, speakers_full, p, 4) for p in (1, 2)}
    yield engs
    for e in engs.values():
        e.close()


# Teacher-forced logits against the fp32 oracle: the bf16 test's bar (5 % of max |logit|, disagreements near-ties under 0.15)
LOGIT_BAR, TIE_BAR = 0.05, 0.15


@pytest.mark.parametrize("geom", ["small", "full"])
@pytest.mark.parametrize("prec", [1, 2], ids=["bf16", "fp16"])
def test_fp8_teacher_forced_and_greedy_vs_oracle(fp8_small, fp8_full, dims_small, dims_full, state_small, state_full,
                                                 speakers_small, speakers_full, geom, prec):
    dims, state, spk = (dims_small, state_small, speakers_small) if geom == "small" else (dims_full, state_full, speakers_full)
    eng = (fp8_small if geom == "small" else fp8_full)[prec]
    g = dims.gpt
    n = 40 if geom == "small" else 20
    orc = O.GPTOracle(state[0], state[1], dims)
    ids = text_ids(dims, 17, 4 + prec)
    osp = O.SamplingParams(temperature=0.0, repetition_penalty=5.0, max_tokens=n, stop_token=g.stop_audio_token)
    toks, _, lg = orc.generate(spk[0][0], ids, osp, return_logits=True)
    sp = Sampling(temperature=0.0, repetition_penalty=5.0, max_tokens=n, stop_token=g.stop_audio_token)
    logits, _, sampled = eng.gpt_teacher_forced(ids, 0, toks, sp)
    err = float(np.abs(logits - lg.numpy()).max())
    scale = max(1.0, float(lg.abs().max()))
    print(f"fp8 KV {geom} prec={prec}: teacher-forced logits max err {err:.4g} = {err / scale:.4f} of max |logit|")
    assert err < LOGIT_BAR * scale
    for k, a, b, margin in _margin_report(lg.numpy(), sampled, toks):
        assert margin < TIE_BAR, (k, a, b, margin)
    # greedy end to end (graph replay after two eager steps): the first divergence, if any, is a near-tie of the oracle
    r, got, wav, _ = eng.run_batch([(1, ids, 0, sp)], timeout_s=120)[1]
    assert r.n_tokens == len(got) and np.isfinite(wav).all()
    bad = _margin_report(lg.numpy(), got, toks)
    assert not bad or bad[0][3] < TIE_BAR, bad[:3]


@pytest.fixture(scope="module")
def fp8_wide(dims_full, state_full, speakers_full):
    eng = _fp8_engine(dims_full, state_full, speakers_full, 2, 192)
    yield eng
    eng.close()


def test_fp8_bench_batch_deterministic(fp8_wide, dims_full):
    """168 chunks (two decode branches, graph replay, rows in both GEMM tiles): two runs give the same tokens and samples"""
    jobs = [(i, text_ids(dims_full, 10 + (7 * i) % 70, 1000 + i), i % 3,
             Sampling(temperature=0.0, repetition_penalty=5.0, max_tokens=12, stop_token=NO_STOP)) for i in range(168)]
    a = fp8_wide.run_batch(jobs, timeout_s=300)
    b = fp8_wide.run_batch([(i + 1000, *j[1:]) for i, j in enumerate(jobs)], timeout_s=300)
    for i in range(168):
        np.testing.assert_array_equal(a[i][1], b[i + 1000][1], err_msg=str(i))
        np.testing.assert_array_equal(a[i][2], b[i + 1000][2], err_msg=str(i))


def _jobs(dims):
    return [(i, text_ids(dims, 12 + 5 * i, 70 + i), i % 3,
             Sampling(temperature=0.75, top_p=0.85, top_k=50, repetition_penalty=5.0, max_tokens=24, seed=11, seq_seed=i,
                      stop_token=NO_STOP)) for i in range(3)]


def test_fp8_round_trip_back_to_16bit_is_bit_identical(engine_small_fp16, dims_small, state_small, speakers_small):
    """an engine switched to fp8 and back gives the bits of an engine that never switched"""
    ref = engine_small_fp16.run_batch(_jobs(dims_small), timeout_s=120)
    eng = _make_engine(dims_small, state_small, speakers_small, 2)
    try:
        eng.set_option("kv_fp8", 1)
        fp8 = eng.run_batch(_jobs(dims_small), timeout_s=120)
        eng.set_option("kv_fp8", 0)
        back = eng.run_batch(_jobs(dims_small), timeout_s=120)
    finally:
        eng.close()
    for i in range(3):
        np.testing.assert_array_equal(back[i][1], ref[i][1])
        np.testing.assert_array_equal(back[i][2], ref[i][2])
    print("fp8 vs fp16 sampled tokens equal:", sum(int(np.array_equal(fp8[i][1], ref[i][1])) for i in range(3)), "/ 3")


def test_fp8_option_refusals(engine_small, dims_small, state_small, speakers_small):
    """fp32 parity mode: ERR_INVALID; a queued chunk: ERR_STATE and the format stays; other values: ERR_INVALID"""
    with pytest.raises(NativeError) as ex:
        engine_small.set_option("kv_fp8", 1)
    assert ex.value.code == ERR_INVALID
    eng = _make_engine(dims_small, state_small, speakers_small, 1)
    try:
        with pytest.raises(NativeError) as ex:
            eng.set_option("kv_fp8", 2)
        assert ex.value.code == ERR_INVALID
        g = dims_small.gpt
        sp = Sampling(temperature=0.0, repetition_penalty=5.0, max_tokens=8, stop_token=g.stop_audio_token)
        eng.set_option("hold_admission", 1)
        eng.submit(1, text_ids(dims_small, 9, 1), 0, sp)
        with pytest.raises(NativeError) as ex:
            eng.set_option("kv_fp8", 1)
        assert ex.value.code == ERR_STATE
        eng.set_option("hold_admission", 0)
        r = None
        while r is None:
            r = eng.poll(10000)
        eng.fetch(r)
        eng.set_option("kv_fp8", 1)                    # idle again: accepted
    finally:
        eng.close()


def test_fp8_beam_search_repeats(fp8_small, dims_small):
    """num_beams = 2 under the fp8 cache: finishes, and a second run repeats it bit for bit"""
    eng = fp8_small[2]
    g = dims_small.gpt
    sp = Sampling(temperature=1.0, repetition_penalty=5.0, max_tokens=30, stop_token=g.stop_audio_token, num_beams=2,
                  length_penalty=1.0, do_sample=False)
    ids = text_ids(dims_small, 15, 8)
    a = eng.run_batch([(1, ids, 0, sp)], timeout_s=120)[1]
    b = eng.run_batch([(2, ids, 0, sp)], timeout_s=120)[2]
    assert a[0].n_tokens >= 1 and np.isfinite(a[2]).all()
    np.testing.assert_array_equal(a[1], b[1])
    np.testing.assert_array_equal(a[2], b[2])


def test_fp8_kv_pools_take_half_the_memory(dims_full, state_full, speakers_full):
    """switching frees the 16-bit pools and allocates fp8 ones of 2080 / 4096 of their size (device free memory)"""
    g = dims_full.gpt
    eng = _make_engine(dims_full, state_full, speakers_full, 2, max_batch=16)
    try:
        torch.cuda.synchronize()
        free16, _ = torch.cuda.mem_get_info(0)
        eng.set_option("kv_fp8", 1)
        free8, _ = torch.cuda.mem_get_info(0)
    finally:
        eng.close()
    max_pages = -(-(g.n_cond_latents + g.max_text_tokens + 3 + g.max_audio_tokens) // PT)
    pool16 = 2 * g.layers * 17 * max_pages * g.heads * PT * D * 2
    saved = free8 - free16
    print(f"16-bit KV pools {pool16 / 2**20:.1f} MiB, freed by the switch {saved / 2**20:.1f} MiB")
    # 60 pool buffers, each rounded up to the allocator's 2 MiB granularity
    expect = pool16 * (1 - BLOCK / (2 * PT * D))
    assert abs(saved - expect) <= 2 * g.layers * 2 ** 21 + 0.005 * pool16
