"""GPU: the beam kernels in isolation (xtts_debug_beam_step) against a numpy restatement: the selection exactly (ranked on
the scores the kernel returns), the scores themselves, the state fork, the page remap invariants and the partial-page
copies in fp32, bf16 and fp16 KV."""
import numpy as np
import pytest

from auralis_b200.native import Sampling, XttsBeamState

pytestmark = pytest.mark.gpu

V, HEADS, LAYERS, MP, CAP = 1026, 2, 3, 4, 64
STOP, START = 1025, 1024
F32 = np.float32


def _sp(nb, lp=1.0, max_tokens=40, penalty=5.0, stop=STOP):
    return Sampling(temperature=0.75, top_p=0.85, top_k=50, repetition_penalty=penalty, max_tokens=max_tokens,
                    stop_token=stop, seed=3, seq_seed=1, num_beams=nb, length_penalty=lp, do_sample=False)


def _seen(nb, extra):
    w = (V + 31) // 32
    s = np.zeros((nb, w), np.uint32)
    for b in range(nb):
        for t in [1, START] + list(extra[b]):
            s[b, t >> 5] |= np.uint32(1 << (t & 31))
    return s


def _ids(seen_row):
    return [v for v in range(V) if (int(seen_row[v >> 5]) >> (v & 31)) & 1]


def _state(nb, first, n_free, held):
    st = XttsBeamState()
    for j in range(8):
        st.fin_score[j] = -1e9
    st.heur_unsat = 1
    st.n_free = n_free
    for j in range(nb):
        st.n_pages[j] = held if (j == 0 or not first) else 0
    if not first:
        for j in range(nb):
            st.run_score[j] = -float(j) - 1.0
    return st


def _group(nb, first, kv_type, rng, L=70):
    """beam tables: page 0 shared by every beam, the second page shared by pairs, the third (partial) private"""
    held = -(-L // 32)
    esz = 4 if kv_type == 0 else 2
    page = HEADS * 32 * 64 * esz
    bt = np.full((nb, MP), -1, np.int32)
    if first:
        bt[0, :held] = np.arange(held)
        n_used, n_free = held, 2 * nb
    else:
        for j in range(nb):
            bt[j, 0] = 0
            bt[j, 1] = 1 + j // 2
            bt[j, 2] = 1 + (nb + 1) // 2 + j
        n_used, n_free = 1 + (nb + 1) // 2 + nb, nb
    n_pages = n_used + n_free
    pool = np.full(nb * MP, -1, np.int32)
    pool[:n_free] = rng.permutation(np.arange(n_used, n_pages)).astype(np.int32)
    kp = rng.randint(0, 256, size=LAYERS * n_pages * page).astype(np.uint8)
    vp = rng.randint(0, 256, size=LAYERS * n_pages * page).astype(np.uint8)
    st = _state(nb, first, n_free, held)
    return bt, pool, kp, vp, st, page


def _logprob(logits, seen, penalty):
    z = logits.astype(np.float64)
    lp = z - z.max(-1, keepdims=True)
    lp = lp - np.log(np.exp(lp).sum(-1, keepdims=True))
    for b in range(lp.shape[0]):
        for v in _ids(seen[b]):
            lp[b, v] = lp[b, v] * penalty if lp[b, v] < 0 else lp[b, v] / penalty
    return lp


def _select(sc, st0, t, stop, max_tok, lp):
    """transformers' selection / finished merge / heuristic on the kernel's scores, fp32, ties to the lower index"""
    nb = sc.shape[0]
    K = 2 * nb
    flat = sc.reshape(-1)
    order = np.lexsort((np.arange(flat.size), -flat.astype(np.float64)))[:K]
    cs = [F32(flat[f]) for f in order]
    cb = [int(f) // V for f in order]
    ct = [int(f) % V for f in order]
    fl = [ct[i] == stop or t + 1 >= max_tok for i in range(K)]
    rs = [F32(cs[i] + F32(-1e9)) if fl[i] else cs[i] for i in range(K)]
    pick = sorted(range(K), key=lambda i: (-rs[i], i))[:nb]
    den = F32(float(t + 1) ** lp)
    merged = [(F32(st0.fin_score[i]), st0.fin_valid[i], st0.fin_step[i], st0.fin_beam[i], st0.fin_tok[i]) for i in range(nb)]
    for i in range(K):
        did = i < nb and fl[i]
        s = F32(cs[i] / den)
        if not st0.heur_unsat:
            s = F32(s + F32(-1e9))
        if not did:
            s = F32(s + F32(-1e9))
        merged.append((s, int(did), t, cb[i], ct[i]))
    fin = [merged[i] for i in sorted(range(len(merged)), key=lambda i: (-merged[i][0], i))[:nb]]
    run = [rs[i] for i in pick]
    best = F32(run[0] / den)
    worst = min(f[0] for f in fin)
    unsat = bool(st0.heur_unsat) and any(best > (worst if f[1] else F32(-1e9)) for f in fin)
    done = not (unsat and not all(fl))
    return [cb[i] for i in pick], [ct[i] for i in pick], run, fin, unsat, done


def _copy_state(st):
    c = XttsBeamState()
    C_bytes = bytes(memoryview(st))
    import ctypes
    ctypes.memmove(ctypes.addressof(c), C_bytes, len(C_bytes))
    return c


def _step(eng, nb, first, kv_type, logits, sp, n_gen, L, rng, st_edit=None, extra_seen=None):
    bt, pool, kp, vp, st, page = _group(nb, first, kv_type, rng, L)
    if st_edit:
        st_edit(st)
    advance = 0 if first else 1
    ng = np.full(nb, n_gen, np.int32)
    ctx = np.full(nb, L - advance, np.int32)
    seen = _seen(nb, extra_seen or [[] for _ in range(nb)])
    hist = np.full((CAP, 8, 2), -7, np.int32)
    before = dict(bt=bt.copy(), pool=pool.copy(), kp=kp.copy(), vp=vp.copy(), st=_copy_state(st), seen=seen.copy())
    last, sc = eng.debug_beam_step(kv_type, HEADS, LAYERS, sp, first, advance, logits, ng, ctx, seen, bt, pool, hist, st, kp, vp)
    return before, dict(bt=bt, pool=pool, kp=kp, vp=vp, st=st, seen=seen, ng=ng, ctx=ctx, hist=hist, last=last, sc=sc, page=page)


def _check(before, after, nb, first, sp, n_gen, L, logits, kv_type):
    st0, st = before["st"], after["st"]
    # scores: log_softmax, penalty, + running score
    lg = np.repeat(logits[:1], nb, 0) if first else logits
    run0 = np.array([0.0] + [-1e9] * (nb - 1)) if first else np.array([st0.run_score[j] for j in range(nb)])
    want = _logprob(lg, before["seen"], sp.repetition_penalty) + run0[:, None]
    np.testing.assert_allclose(after["sc"], want, rtol=1e-6, atol=3e-5)
    # selection, exactly
    par, tok, run, fin, unsat, done = _select(after["sc"], st0, n_gen, sp.stop_token, sp.max_tokens, sp.length_penalty)
    assert [st.sel_parent[j] for j in range(nb)] == par and [st.sel_tok[j] for j in range(nb)] == tok
    assert [F32(st.run_score[j]) for j in range(nb)] == run
    assert [(F32(st.fin_score[j]), st.fin_valid[j], st.fin_step[j], st.fin_beam[j], st.fin_tok[j]) for j in range(nb)] == \
        [(f[0], int(f[1]), f[2], f[3], f[4]) for f in fin]
    assert bool(st.heur_unsat) == unsat and bool(st.done) == done
    assert [tuple(after["hist"][n_gen, j]) for j in range(nb)] == list(zip(par, tok))
    if done:
        return par, tok, st
    # state fork
    for j in range(nb):
        exp = before["seen"][par[j]].copy()
        exp[tok[j] >> 5] |= np.uint32(1 << (tok[j] & 31))
        assert np.array_equal(after["seen"][j], exp)
    assert list(after["last"]) == tok and set(after["ng"]) == {n_gen + 1} and set(after["ctx"]) == {L}
    # page remap
    f, part = L // 32, L % 32
    held = -(-L // 32)
    old_tab = [list(before["bt"][j, :(held if (j == 0 or not first) else 0)]) for j in range(nb)]
    new_tab = [list(after["bt"][j, :f + 1]) for j in range(nb)]
    assert [st.n_pages[j] for j in range(nb)] == [f + 1] * nb
    first_child = [par.index(par[j]) == j for j in range(nb)]
    for j in range(nb):
        assert new_tab[j][:f] == old_tab[par[j]][:f]                  # a child's prefix is its parent's
        if part and first_child[j]:
            assert new_tab[j][f] == old_tab[par[j]][f]
    private = [new_tab[j][f] for j in range(nb) if not (part and first_child[j])]
    referenced = {p for t in new_tab for p in t}
    assert len(set(private)) == len(private)                             # private pages are disjoint
    for j in range(nb):
        if not (part and first_child[j]):
            others = {p for i, t in enumerate(new_tab) for k, p in enumerate(t) if (i, k) != (j, f)}
            assert new_tab[j][f] not in others
    old_all = {p for t in old_tab for p in t} | set(before["pool"][:st0.n_free].tolist())
    new_pool = after["pool"][:st.n_free].tolist()
    assert len(set(new_pool)) == len(new_pool) and not (set(new_pool) & referenced)
    assert referenced | set(new_pool) == old_all                         # pool pages are conserved
    # partial-page copies, byte for byte, and nothing else written
    copies = [(st.copy_src[c], st.copy_dst[c], st.copy_ntok[c]) for c in range(st.n_copy)]
    assert sorted(copies) == sorted((old_tab[par[j]][f], new_tab[j][f], part) for j in range(nb)
                                    if part and not first_child[j])
    assert not ({c[1] for c in copies} & {c[0] for c in copies})
    page = after["page"]
    esz = 4 if kv_type == 0 else 2
    for key, shape, tax in (("kp", (HEADS, 64 * esz // 16, 32, 16), 2), ("vp", (HEADS, 32, 64 * esz), 1)):
        b = before[key].reshape(LAYERS, -1, page)
        a = after[key].reshape(LAYERS, -1, page)
        dsts = {d for _, d, _ in copies}
        keep = [p for p in range(b.shape[1]) if p not in dsts]
        assert np.array_equal(a[:, keep], b[:, keep])
        for src, dst, n in copies:
            for layer in range(LAYERS):
                got = a[layer, dst].reshape(shape)
                s_ = b[layer, src].reshape(shape)
                old = b[layer, dst].reshape(shape)
                sl = [slice(None)] * len(shape)
                sl[tax] = slice(0, n)
                assert np.array_equal(got[tuple(sl)], s_[tuple(sl)])
                sl[tax] = slice(n, 32)
                assert np.array_equal(got[tuple(sl)], old[tuple(sl)])
    return par, tok, st


def _logits(rng, nb):
    return (rng.randn(nb, V) * 3).astype(np.float32)


def test_first_step(engine_small):
    rng = np.random.RandomState(1)
    sp = _sp(4)
    lg = _logits(rng, 1)
    before, after = _step(engine_small, 4, True, 0, lg, sp, 0, 70, rng)
    par, _, _ = _check(before, after, 4, True, sp, 0, 70, lg, 0)
    assert par == [0, 0, 0, 0]


@pytest.mark.parametrize("kv_type", [0, 1, 2])
@pytest.mark.parametrize("L", [70, 96])
def test_decode_step_fork_and_copies(engine_small, kv_type, L):
    """a decode step with diverged tables, in every KV type; L = 96 starts a page (no copies, fresh pages)"""
    rng = np.random.RandomState(10 + kv_type + L)
    nb = 4
    sp = _sp(nb, 1.0)
    lg = _logits(rng, nb)
    lg[0, 7] = lg[0, 11] = 30.0                                         # beam 0 gives two children
    before, after = _step(engine_small, nb, False, kv_type, lg, sp, 5, L, rng,
                          extra_seen=[[3, 9], [4], [], [500]])
    par, _, _ = _check(before, after, nb, False, sp, 5, L, lg, kv_type)
    assert par.count(0) >= 2


def test_tie_rule(engine_small):
    rng = np.random.RandomState(3)
    nb = 3
    sp = _sp(nb, 1.0, penalty=1.0)
    lg = _logits(rng, nb)
    lg[1] = lg[0]
    lg[:2, 5] = lg[:2, 9] = 40.0

    def edit(st):
        st.run_score[0] = st.run_score[1] = -2.0
    before, after = _step(engine_small, nb, False, 0, lg, sp, 2, 70, rng, st_edit=edit)
    par, tok, _ = _check(before, after, nb, False, sp, 2, 70, lg, 0)
    assert list(zip(par, tok)) == [(0, 5), (0, 9), (1, 5)]


def test_all_top_candidates_stop(engine_small):
    """every beam's best token is the stop token: the top nb candidates finish, the running set comes from the rest"""
    rng = np.random.RandomState(4)
    nb = 4
    sp = _sp(nb, 2.0, penalty=1.0)
    lg = _logits(rng, nb)
    lg[:, STOP] = 50.0
    before, after = _step(engine_small, nb, False, 1, lg, sp, 6, 70, rng)
    _, tok, st = _check(before, after, nb, False, sp, 6, 70, lg, 1)
    assert STOP not in tok and all(st.fin_valid[j] for j in range(nb)) and all(st.fin_tok[j] == STOP for j in range(nb))


def test_max_length_step_finishes_group(engine_small):
    rng = np.random.RandomState(5)
    nb = 2
    sp = _sp(nb, 1.0, max_tokens=9)
    lg = _logits(rng, nb)
    before, after = _step(engine_small, nb, False, 0, lg, sp, 8, 70, rng)
    _, _, st = _check(before, after, nb, False, sp, 8, 70, lg, 0)
    assert st.done == 1 and st.fin_valid[0] == 1 and st.fin_step[0] == 8


def test_finished_hypotheses_replaced_and_heuristic(engine_small):
    """a full finished set: better new hypotheses replace the worst; then a set no running beam can beat ends the group"""
    rng = np.random.RandomState(6)
    nb = 3
    sp = _sp(nb, 1.0, penalty=1.0)
    lg = _logits(rng, nb)
    lg[:, STOP] = 45.0

    def edit(st):
        for j, s in enumerate([-0.5, -3.0, -80.0]):
            st.fin_score[j], st.fin_valid[j], st.fin_step[j], st.fin_beam[j], st.fin_tok[j] = s, 1, 1, j, STOP
    before, after = _step(engine_small, nb, False, 0, lg, sp, 4, 70, rng, st_edit=edit)
    _, _, st = _check(before, after, nb, False, sp, 4, 70, lg, 0)
    assert F32(-80.0) not in [F32(st.fin_score[j]) for j in range(nb)]

    def edit2(st):
        for j in range(nb):
            st.fin_score[j], st.fin_valid[j], st.fin_step[j], st.fin_beam[j], st.fin_tok[j] = -1e-3, 1, 1, j, STOP
    lg2 = _logits(rng, nb)
    before, after = _step(engine_small, nb, False, 0, lg2, sp, 4, 70, rng, st_edit=edit2)
    _, _, st = _check(before, after, nb, False, sp, 4, 70, lg2, 0)
    assert st.heur_unsat == 0 and st.done == 1
