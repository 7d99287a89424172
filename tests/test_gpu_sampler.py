"""The fused sampler (sample_kernel) launched on its own through xtts_debug_sample_slots and compared token for token with
an exact numpy restatement of its contract, with the per-slot state it writes read back.

Reference (`reference`):
- penalty z / pen (z > 0) or z * pen on seen ids, then z / T: single fp32 operations, reproduced exactly in float32
  (the library is built without fast-math);
- greedy when fp32(T) < fp32(1e-5): lowest index of the maximum;
- top-k keeps z >= the k-th largest (float compare, ties kept) when 0 < top_k < V;
- top-p on the ascending (value, index) order: float64 cumulative softmax c_i, drop c_i <= fp32(1 - fp32(top_p)), the
  last (largest) element always kept;
- draw: token = argmax p / e over the kept set (lowest index on ties), p the float64 softmax of the kept set, e = -log(u)
  with u = ((r >> 9) + 0.5) * 2^-23 and r word v & 3 of Philox4x32-10(counter (v / 4, n, seq_seed, 0), key seed).

Decisiveness.  The kernel computes the same quantities in fp32; a row counts as decisive when every top-p comparison and
the winning ratio clear this bound on the kernel's error (u = 2^-24):
- a term exp(d), d = x - max, carries d's rounding (|d| u) plus expf's 2 ulp (4u); d = 0 gives exactly 1;
- every fp32 sum of non-negative terms is within H u of the exact sum, H = 128 being the longest chain of additions any
  term passes through (the fast path's serial scan of its 128 candidates; the full path's per-thread, scan and
  shuffle-tree sums are shorter); terms that underflow add at most 2^-125 each (the total is >= 1: the max term is 1);
- c = fl(S_k * fl(1 / S)) adds 2u, so |c' - c| <= c (r_k + r + 2 H u + 3u) with r_k, r the relative error of the terms;
- a ratio p / e carries its term's error, one rounding for p = e / S, logf's 1 ulp (2u) and one rounding for the
  division; S's own error scales every p alike and cannot reorder them.
Rows whose kept set is n equal values, n a power of two, are exact in fp32 (sums of ones, a power-of-two reciprocal):
their top-p compares hold with no margin, which is how the top-p `<=` boundary itself is tested.

Boundary cases choose their seeds so that the token changes when the boundary element's fate flips (`discriminating`
rows); without that a boundary test would pass whatever the kernel did at the boundary."""
import numpy as np
import pytest
import torch

from auralis_b200.native import NativeError, Sampling
from oracle import xtts_oracle as O

U = 2.0 ** -24
H = 128
EXP_ERR = 4 * U                          # expf: 2 ulp
LOG_ERR = 2 * U                          # logf: 1 ulp
TINY = 2.0 ** -125
_M32 = np.uint64(0xFFFFFFFF)
REPORT = {}                              # case -> (rows, decisive share, discriminating rows)


# ------------------------------------------------------------------------------------------------ Philox / noise
def philox(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10, vectorised over broadcast uint32 inputs -> [..., 4] uint32"""
    c0, c1, c2, c3, k0, k1 = np.broadcast_arrays(*[np.asarray(a, np.uint64) & _M32 for a in (c0, c1, c2, c3, k0, k1)])
    M0, M1, W0, W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
    for _ in range(10):
        p0, p1 = c0 * M0, c2 * M1           # < 2^64: exact
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _M32
        k0, k1 = (k0 + W0) & _M32, (k1 + W1) & _M32
    return np.stack([c0, c1, c2, c3], -1).astype(np.uint32)


def noise_bits(seed, seq_seed, n, V):
    """r [R, V] uint32: word v & 3 of block v / 4 for each row's (seed, seq_seed, n)"""
    flat = lambda a: np.asarray(a, dtype=object).ravel()          # Python ints: seeds >= 2^63 stay exact
    seed = np.array([int(s) for s in flat(seed)], dtype=np.uint64)
    ss = np.array([int(s) & 0xFFFFFFFF for s in flat(seq_seed)], dtype=np.uint64)
    n = np.array([int(x) & 0xFFFFFFFF for x in flat(n)], dtype=np.uint64)
    blk = np.arange((V + 3) // 4, dtype=np.uint64)[None]
    r = philox(blk, n[:, None], ss[:, None], 0, (seed & _M32)[:, None], (seed >> np.uint64(32))[:, None])
    return r.reshape(len(seed), -1)[:, :V]


def exp_noise(r):
    return -np.log(((r >> np.uint32(9)).astype(np.float64) + 0.5) * 2.0 ** -23)


# ------------------------------------------------------------------------------------------------ reference
class Ref:
    pass


def reference(z, seen, T, top_k, top_p, pen, seed, seq_seed, n, flip=None):
    """Rows of z [R, V] fp32 with per-row parameters -> Ref(token, decisive, kept [R, V], path, order, ...).
    flip [R, V] (optional) toggles entries of the kept set before the draw (the discriminating-row test)."""
    z = np.asarray(z, np.float32)
    R, V = z.shape
    rows = np.arange(R)
    T32, tp32, pen32 = (np.asarray(a, np.float32).reshape(R) for a in (T, top_p, pen))
    tk = np.asarray(top_k, np.int64).reshape(R)
    seen = np.asarray(seen, bool).reshape(R, V)
    with np.errstate(all="ignore"):
        pz = pen32[:, None]
        zp = np.where(seen & (pz != 1), np.where(z > 0, z / pz, z * pz), z).astype(np.float32)
        greedy = T32 < np.float32(1e-5)
        zt = np.where(greedy[:, None], zp, zp / np.where(greedy, np.float32(1), T32)[:, None]).astype(np.float32)
    order = np.argsort(zt, axis=1, kind="stable")
    srt = np.take_along_axis(zt, order, 1)
    apply_k = (tk > 0) & (tk < V)
    kth = np.where(apply_k, srt[rows, np.clip(V - tk, 0, V - 1)], -np.inf).astype(np.float32)
    keep = srt >= kth[:, None]
    survivors = keep.sum(1)
    srt_k = np.where(keep, srt, -np.inf)
    mx = srt[:, -1].astype(np.float64)
    fin, fin_all = np.isfinite(srt_k), np.isfinite(srt)
    with np.errstate(all="ignore"):
        d = np.where(fin_all, srt.astype(np.float64) - mx[:, None], 0.0)
    e_all = np.where(fin_all, np.exp(d), 0.0)                # every finite term (a flipped-in entry draws with it)
    eps_all = np.where(fin_all & (d != 0), 1.01 * np.abs(d) * U + 1.01 * EXP_ERR, 0.0)
    e, eps = np.where(fin, e_all, 0.0), np.where(fin, eps_all, 0.0)
    S, Se = np.cumsum(e, 1), np.cumsum(e * eps, 1)
    tot = S[:, -1:]
    c = S / tot
    thr = (np.float32(1) - tp32).astype(np.float64)[:, None]
    apply_p = (tp32 < 1)[:, None]
    drop = apply_p & (c <= thr)
    drop[:, -1] = False
    kept_s = fin & ~drop
    nfin = fin.sum(1)
    exact = ((fin & (d != 0)).sum(1) == 0) & ((nfin & (nfin - 1)) == 0)
    with np.errstate(all="ignore"):
        rk = np.where(S > 0, Se / np.where(S > 0, S, 1), 0.0)
    bound = c * (rk + Se[:, -1:] / tot + 2 * H * U + 3 * U) + np.cumsum(fin, 1) * TINY
    close = apply_p & fin & (np.abs(c - thr) <= bound) & ~exact[:, None]
    close[:, -1] = False
    kept = np.zeros((R, V), bool)
    kept[rows[:, None], order] = kept_s
    if flip is not None:
        kept ^= flip
    e_o, eps_o = np.zeros((R, V)), np.zeros((R, V))
    e_o[rows[:, None], order], eps_o[rows[:, None], order] = e_all, eps_all
    totk = np.maximum((e_o * kept).sum(1, keepdims=True), 1e-300)
    ee = exp_noise(noise_bits(seed, seq_seed, n, V))
    live = kept & (e_o > 0)
    ratio = np.where(live, e_o / totk / ee, -1.0)
    win = np.argmax(ratio, 1)
    rho = eps_o + 2 * U + LOG_ERR + 2 * U
    hi = np.where(live, ratio * (1 + rho) + TINY, -1.0)
    hi[rows, win] = -np.inf
    lo_w = ratio[rows, win] * (1 - rho[rows, win]) - TINY
    r = Ref()
    r.greedy = greedy
    r.token = np.where(greedy, np.argmax(zp, 1), win)
    r.decisive = greedy | ((lo_w > hi.max(1)) & ~close.any(1))
    r.kept, r.order, r.zt, r.kth, r.survivors = kept, order, zt, kth, survivors
    r.path = np.where(greedy, "greedy", np.where((tk > 0) & (tk <= 64) & (tk < V) & (survivors <= 128), "fast", "full"))
    r.first_kept = np.where(kept_s.any(1), np.argmax(kept_s, 1), V - 1)      # sorted position of the smallest kept
    return r


def token_if_flipped(z, prm, flip):
    return reference(z, flip=flip, **prm).token


# ------------------------------------------------------------------------------------------------ cases
T_SET = [0.0, 9.99e-6, 1e-5, 1e-3, 0.75, 1.0, 10.0]
TOPP_SET = [1.0, 0.999999, 0.85, 0.5, 0.01, 0.0]
PEN_SET = [1.0, 5.0, 1.3, 0.5]
SCALES = [0.1, 0.3, 1.0, 3.0, 10.0, 30.0]


def topk_set(V):
    return [0, -1, 1, 2, 50, 63, 64, 65, 127, 128, V - 1, V, V + 5]


def seen_pattern(i, V, rng):
    s = np.zeros(V, bool)
    k = i % 5
    if k == 1:
        s[:] = True
    elif k == 2:
        s[::2] = True
    elif k == 3:
        s[rng.rand(V) < 0.1] = True
    elif k == 4:
        s[max(0, V - 1 - (V - 1) % 32):] = True        # the partially used last bitmap word
    return s


def logit_row(i, V, rng):
    z = rng.randn(V) * SCALES[i % 6]
    k = (i // 6) % 5
    if k == 1:                                          # +-80 offsets: exp underflows for most terms
        z += np.where(rng.rand(V) < 0.02, 80.0, -80.0 * (rng.rand(V) < 0.5))
    elif k == 2:                                        # -inf entries, often fewer finite logits than top_k
        z[rng.rand(V) < 0.9] = -np.inf
        z[rng.randint(V)] = rng.randn()
    elif k == 3:                                        # exactly one finite logit
        z[:] = -np.inf
        z[rng.randint(V)] = rng.randn()
    return z.astype(np.float32)


def sweep_case(V, R, seed):
    """R rows at vocabulary V cycling through every temperature, top_k, top_p, penalty, seen and logit pattern."""
    rng = np.random.RandomState(seed)
    K = topk_set(V)
    z = np.stack([logit_row(i, V, rng) for i in range(R)])
    prm = dict(T=[T_SET[i % 7] for i in range(R)], top_k=[K[i % 13] for i in range(R)],
               top_p=[TOPP_SET[i % 6] for i in range(R)], pen=[PEN_SET[i % 4] for i in range(R)],
               seen=np.stack([seen_pattern(i, V, rng) for i in range(R)]),
               seed=rng.randint(0, 2 ** 62, R, dtype=np.int64), seq_seed=rng.randint(-2 ** 31, 2 ** 31 - 1, R),
               n=rng.randint(0, 605, R))
    return z, prm


def rows_params(R, T=1.0, top_k=0, top_p=1.0, pen=1.0, seen=None, V=None, seed=0, seq_seed=0, n=0):
    full = lambda a: np.broadcast_to(np.asarray(a), (R,)).copy()
    return dict(T=full(T), top_k=full(top_k), top_p=full(top_p), pen=full(pen),
                seen=np.zeros((R, V), bool) if seen is None else seen, seed=full(seed), seq_seed=full(seq_seed),
                n=full(n))


def select(z, prm, disc, R, need):
    """R rows of a candidate pool, discriminating rows first (at least `need` of them)."""
    idx = np.concatenate([np.nonzero(disc)[0], np.nonzero(~disc)[0]])[:R]
    assert disc.sum() >= need, (int(disc.sum()), need)
    pick = lambda a: a[idx] if isinstance(a, np.ndarray) and a.ndim >= 1 else a
    return z[idx], {k: pick(np.asarray(v)) for k, v in prm.items()}, disc[idx]


def signed_zero_case(pool=400):
    V = 130
    z = np.full((pool, V), -1.0, np.float32)
    z[:, 0], z[:, 1], z[:, 2] = 1.0, 0.0, -0.0
    prm = rows_params(pool, top_k=2, V=V, seed=np.arange(pool), seq_seed=3, n=5)
    disc = reference(z, **prm).token == 2               # the fast path before the fix could never draw -0.0's id
    return V, z, prm, disc


def tie_case(survivors, pool=600, V=1026):
    """top_k 50 with the 50th value tied so that exactly `survivors` entries are >= it (128: fast path, 129: full)."""
    rng = np.random.RandomState(survivors)
    z = (rng.randn(pool, V) * 0.3 - 3.0).astype(np.float32)
    for r in range(pool):
        ids = rng.permutation(V)[:survivors]
        z[r, ids[:40]] = (1.0 + 0.2 * rng.rand(40)).astype(np.float32)
        z[r, ids[40:]] = 0.75
    prm = rows_params(pool, top_k=50, V=V, seed=rng.randint(0, 2 ** 40, pool), seq_seed=rng.randint(0, 1000, pool))
    ref = reference(z, **prm)
    assert (ref.survivors == survivors).all()
    disc = z[np.arange(pool), ref.token] == np.float32(0.75)   # the token is one of the tied k-th values
    return V, z, prm, disc


def topk_boundary_case(k, V=1026, pool=None):
    """near-flat distinct logits, top_k k, top_p 1: discriminating rows draw the (k+1)-th largest once it is kept."""
    pool = pool or 24 * (k + 1)
    rng = np.random.RandomState(k)
    z = (rng.randn(pool, V) * 0.01).astype(np.float32)
    prm = rows_params(pool, top_k=k, V=V, seed=rng.randint(0, 2 ** 40, pool), seq_seed=7, n=rng.randint(0, 600, pool))
    ref = reference(z, **prm)
    srt = np.sort(z, 1)
    flip = z == srt[:, V - k - 1][:, None]
    disc = token_if_flipped(z, prm, flip) != ref.token
    return V, z, prm, disc


def topp_boundary_case(path, top_p, pool=300):
    """kept set of 8 equal values (exact in fp32) with top_p 0.5 or 0: the cumulative sum hits 1 - top_p exactly."""
    V = 130
    rng = np.random.RandomState(int(top_p * 10) + (path == "fast"))
    z = np.full((pool, V), -np.inf if path == "full" else -5.0, np.float32)
    for r in range(pool):
        z[r, 1 + rng.permutation(V - 1)[:8]] = 2.0          # id 0 never kept: a dropped max would show as token 0
    prm = rows_params(pool, top_k=8 if path == "fast" else 0, top_p=top_p, V=V, seed=rng.randint(0, 2 ** 40, pool),
                      seq_seed=rng.randint(0, 99, pool), n=3)
    ref = reference(z, **prm)
    assert (ref.path == path).all()
    pos = np.arange(pool)
    if top_p == 0.0:                                        # only the last (highest-index max) survives
        return V, z, prm, np.ones(pool, bool)
    # the element whose cumulative sum equals the threshold: kept under `<`, dropped under `<=`
    flip = np.zeros((pool, V), bool)
    flip[pos, ref.order[pos, ref.first_kept - 1]] = True
    disc = token_if_flipped(z, prm, flip) != ref.token
    return V, z, prm, disc


def topp_random_case(path, pool=3000, V=1026):
    rng = np.random.RandomState(17 + (path == "fast"))
    z = (rng.randn(pool, V) * (1.5 if path == "fast" else 4.0)).astype(np.float32)
    prm = rows_params(pool, T=0.75, top_k=50 if path == "fast" else 0, top_p=0.85, V=V,
                      seed=rng.randint(0, 2 ** 40, pool), seq_seed=rng.randint(0, 99, pool), n=rng.randint(0, 600, pool))
    ref = reference(z, **prm)
    pos = np.arange(pool)
    flip = np.zeros((pool, V), bool)
    flip[pos, ref.order[pos, ref.first_kept]] = True        # drop the smallest kept element
    disc = (token_if_flipped(z, prm, flip) != ref.token) & ref.decisive
    return V, z, prm, disc


# ------------------------------------------------------------------------------------------------ one checked launch
def sps_for(prm, rows_of_slot, n_slots, rng, max_tokens=None, stop=None):
    out = []
    for s in range(n_slots):
        r = rows_of_slot[s]
        if r < 0:                                          # inactive slot: arbitrary parameters
            out.append(Sampling(temperature=float(rng.rand()), top_p=0.5, top_k=int(rng.randint(0, 80)),
                                repetition_penalty=2.0, max_tokens=3, stop_token=1, seed=int(rng.randint(1 << 30)),
                                seq_seed=5))
            continue
        out.append(Sampling(temperature=float(prm["T"][r]), top_p=float(prm["top_p"][r]), top_k=int(prm["top_k"][r]),
                            repetition_penalty=float(prm["pen"][r]),
                            max_tokens=int(max_tokens[r]) if max_tokens is not None else 100000,
                            stop_token=int(stop[r]) if stop is not None else -1, seed=int(prm["seed"][r]),
                            seq_seed=int(prm["seq_seed"][r])))
    return out


def expect_state(st0, active, drawn, sps, cap, advance_ctx, forced):
    st = {k: v.copy() for k, v in st0.items()}
    for r, s in enumerate(active):
        n = int(st0["n_gen"][s])
        tok = int(drawn[r])
        if forced is not None and forced[s, n] >= 0:
            tok = int(forced[s, n])
        if n < cap:
            st["tokens"][s, n], st["sampled"][s, n] = tok, drawn[r]
        st["last_tok"][s] = tok
        st["seen"][s, tok] = 1
        st["n_gen"][s] = n + 1
        st["ctx_len"][s] += advance_ctx
        if tok == sps[s].stop_token or n + 1 >= sps[s].max_tokens:
            st["finished"][s] = 1
    return st


def run_checked(eng, name, V, z, prm, seed=0, extra_slots=3, ld_pad=5, cap=None, forced=None, advance_ctx=0,
                max_tokens=None, stop=None, finished=None, disc=None, need_disc=0, min_decisive=0.9, st0=None,
                active=None):
    """One launch over the rows of z (row r -> a shuffled sparse slot); every decisive token must equal the reference,
    every state array must equal the state the reference implies.  -> (state after, Ref, active)"""
    rng = np.random.RandomState(seed)
    R = z.shape[0]
    n_slots = R + extra_slots if st0 is None else len(st0["n_gen"])
    if active is None:
        active = rng.permutation(n_slots)[:R].astype(np.int32)
    rows_of_slot = np.full(n_slots, -1)
    rows_of_slot[active] = np.arange(R)
    cap = cap or int(np.max(prm["n"])) + 2
    lg = np.full((R, V + ld_pad), np.nan, np.float32)
    lg[:, :V] = z
    sps = sps_for(prm, rows_of_slot, n_slots, rng, max_tokens, stop)
    if st0 is None:
        st0 = dict(n_gen=rng.randint(0, cap, n_slots).astype(np.int32), ctx_len=rng.randint(0, 900, n_slots).astype(np.int32),
                   finished=(rng.rand(n_slots) < 0.3).astype(np.int32) if finished is None else finished,
                   last_tok=rng.randint(0, V, n_slots).astype(np.int32),
                   seen=(rng.rand(n_slots, V) < 0.2).astype(np.uint8),
                   tokens=rng.randint(-5, V, (n_slots, cap)).astype(np.int32),
                   sampled=rng.randint(-5, V, (n_slots, cap)).astype(np.int32))
        st0["n_gen"][active] = prm["n"]
        st0["seen"][active] = prm["seen"]
    st = eng.debug_sample_slots(V, lg, active, sps, cap=cap, advance_ctx=advance_ctx, forced=forced,
                                **{k: st0[k] for k in eng.SAMPLE_STATE})
    prm_rows = dict(prm, n=st0["n_gen"][active], seen=st0["seen"][active].astype(bool))
    ref = reference(z, **prm_rows)
    n = st0["n_gen"][active]
    got = np.where(n < cap, st["sampled"][active, np.minimum(n, cap - 1)], st["last_tok"][active])
    assert ((got >= 0) & (got < V)).all(), name
    bad = np.nonzero(ref.decisive & (got != ref.token))[0]
    assert bad.size == 0, (name, [(int(r), ref.path[r], int(got[r]), int(ref.token[r])) for r in bad[:8]])
    share = float(ref.decisive.mean())
    assert share >= min_decisive, (name, share)
    nd = int((disc & ref.decisive).sum()) if disc is not None else 0
    assert nd >= need_disc, (name, nd, need_disc)
    drawn = np.where(ref.decisive, ref.token, got)
    exp = expect_state(st0, active, drawn, sps, cap, advance_ctx, forced)
    for k in eng.SAMPLE_STATE:
        np.testing.assert_array_equal(st[k], exp[k], err_msg=f"{name}: {k}")
    REPORT[name] = (R, share, nd)
    print(f"sampler case {name}: rows {R}, decisive {share:.3f}, discriminating {nd}, "
          f"paths {dict(zip(*np.unique(ref.path, return_counts=True)))}")
    return st, ref, active


# ------------------------------------------------------------------------------------------------ CPU: the reference
KAT = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
       ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
       ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
        (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_philox_known_answers(ctr, key, want):
    """Random123's published philox4x32-10 known-answer vectors, for the vectorised Philox and the oracle's."""
    np.testing.assert_array_equal(philox(*ctr, *key), np.array(want, np.uint32))
    np.testing.assert_array_equal(O.philox4x32(ctr, key), np.array(want, np.uint32))


def test_noise_matches_oracle():
    for seed, ss, n, V in [(0, 0, 0, 5), (2 ** 32 - 1, 7, 1, 130), (2 ** 32, -1, 604, 1026), (2 ** 63 + 5, 2 ** 31 - 1, 9, 7)]:
        r = noise_bits([seed], [ss], [n], V)[0]
        want = [O.philox4x32((v // 4, n, ss & 0xFFFFFFFF, 0), (seed & 0xFFFFFFFF, seed >> 32))[v % 4] for v in range(V)]
        np.testing.assert_array_equal(r, np.array(want, np.uint32))
        # the oracle takes the log in fp32, this reference in float64
        np.testing.assert_allclose(exp_noise(r[None])[0], O.exp_noise(seed, ss & 0xFFFFFFFF, n, V), rtol=2.0 ** -22, atol=0)


def _direct(z, seen, T, top_k, top_p, pen, seed, seq_seed, n):
    """one row, plain loops in Python floats (fp32 where the kernel rounds)"""
    V = len(z)
    f = np.float32
    zz = []
    for v in range(V):
        x = f(z[v])
        if seen[v] and f(pen) != 1:
            x = f(x / f(pen)) if x > 0 else f(x * f(pen))
        zz.append(x)
    if f(T) < f(1e-5):
        return max(range(V), key=lambda v: (zz[v], -v))
    zz = [f(x / f(T)) for x in zz]
    srt = sorted(range(V), key=lambda v: (zz[v], v))
    keep = set(range(V))
    if 0 < top_k < V:
        kth = zz[srt[V - top_k]]
        keep = {v for v in range(V) if zz[v] >= kth}
    if f(top_p) < 1:
        mx = float(zz[srt[-1]])
        ids = [v for v in srt if v in keep]
        tot = sum(np.exp(float(zz[v]) - mx) for v in ids)
        run, thr = 0.0, float(f(1) - f(top_p))
        for v in ids[:-1]:
            run += np.exp(float(zz[v]) - mx)
            if run / tot <= thr:
                keep.discard(v)
    mx = max(float(zz[v]) for v in keep)
    tot = sum(np.exp(float(zz[v]) - mx) for v in keep)
    best, besti = -1.0, V
    key = (seed & 0xFFFFFFFF, seed >> 32)
    for v in sorted(keep):
        r = int(O.philox4x32((v // 4, n, seq_seed & 0xFFFFFFFF, 0), key)[v % 4])
        ratio = np.exp(float(zz[v]) - mx) / tot / -np.log(((r >> 9) + 0.5) * 2.0 ** -23)
        if ratio > best:
            best, besti = ratio, v
    return besti


def test_reference_matches_direct_loop():
    for V, seed in [(1, 0), (4, 1), (5, 2), (13, 3), (40, 4)]:
        z, prm = sweep_case(V, 91, seed)
        ref = reference(z, **prm)
        for r in range(91):
            if ref.decisive[r] and np.isfinite(z[r]).any():
                one = {k: (v[r] if k != "seen" else v[r]) for k, v in prm.items()}
                want = _direct(z[r], one["seen"], one["T"], int(one["top_k"]), one["top_p"], one["pen"], int(one["seed"]),
                               int(one["seq_seed"]), int(one["n"]))
                assert ref.token[r] == want, (V, r, ref.token[r], want)


def test_reference_matches_oracle():
    """decisive rows agree with O.sample_token, and the reference's kept set with O.topk_topp_mask"""
    for V, seed in [(130, 5), (1026, 6), (257, 7)]:
        z, prm = sweep_case(V, 91, seed)
        ref = reference(z, **prm)
        checked = 0
        for r in np.nonzero(ref.decisive)[0]:
            seen = set(np.nonzero(prm["seen"][r])[0].tolist())
            sp = O.SamplingParams(temperature=float(np.float32(prm["T"][r])), top_p=float(np.float32(prm["top_p"][r])),
                                  top_k=int(prm["top_k"][r]), repetition_penalty=float(np.float32(prm["pen"][r])),
                                  seed=int(prm["seed"][r]))
            want = O.sample_token(torch.from_numpy(z[r].copy()), seen, sp, int(prm["seq_seed"][r]) & 0xFFFFFFFF,
                                  int(prm["n"][r]))
            assert ref.token[r] == want, (V, r, ref.path[r], ref.token[r], want)
            if not ref.greedy[r]:
                m = O.topk_topp_mask(torch.from_numpy(ref.zt[r].copy()), int(prm["top_k"][r]), float(np.float32(prm["top_p"][r])))
                oracle_kept = torch.isfinite(m).numpy() & np.isfinite(ref.zt[r])
                np.testing.assert_array_equal(oracle_kept, ref.kept[r] & np.isfinite(ref.zt[r]))
            checked += 1
        assert checked >= 0.9 * 91, (V, checked)


def test_decisiveness_bound_holds_for_fp32_arithmetic():
    """The top-p bound covers an fp32 evaluation of the cumulative softmax in both of the kernel's orders (serial, and
    8-wide per-thread partials combined by a scan)."""
    rng = np.random.RandomState(0)
    worst = 0.0
    for trial in range(40):
        V = [130, 1026, 2048][trial % 3]
        x = np.sort((rng.randn(V) * [0.1, 1, 5, 30][trial % 4]).astype(np.float32))
        mx = x[-1]
        e32 = np.exp((x - mx).astype(np.float32)).astype(np.float32)
        e64 = np.exp(x.astype(np.float64) - float(mx))
        serial = np.cumsum(e32, dtype=np.float32)
        part = np.concatenate([np.zeros(1, np.float32), np.cumsum(e32.reshape(-1, 2)[:, 0] + e32.reshape(-1, 2)[:, 1],
                                                                   dtype=np.float32)]) if V % 2 == 0 else serial
        for s32 in (serial,) if V % 2 else (serial, np.repeat(part[1:], 2)):
            c32 = (s32 * (np.float32(1) / s32[-1])).astype(np.float64)
            S = np.cumsum(e64)
            c = S / S[-1]
            d = x.astype(np.float64) - float(mx)
            eps = np.where(d != 0, 1.01 * np.abs(d) * U + 1.01 * EXP_ERR, 0)
            bound = c * (np.cumsum(e64 * eps) / S + (e64 * eps).sum() / S[-1] + 2 * H * U + 3 * U) + np.arange(1, V + 1) * TINY
            sel = slice(None) if s32 is serial else slice(1, None, 2)
            assert (np.abs(c32 - c)[sel] <= bound[sel]).all()
            worst = max(worst, float((np.abs(c32 - c)[sel] / bound[sel]).max()))
    assert worst > 1e-3            # the bound is not vacuous


def test_signed_zero_case_discriminates():
    """CPU side of the +-0 regression: the reference keeps both zeros (as the oracle does) and draws -0.0's id often."""
    V, z, prm, disc = signed_zero_case()
    assert disc.sum() >= 30
    m = O.topk_topp_mask(torch.from_numpy(z[0].copy()), 2, 1.0)
    assert torch.isfinite(m)[:3].all() and not torch.isfinite(m)[3:].any()


# ------------------------------------------------------------------------------------------------ GPU
gpu = pytest.mark.gpu


@gpu
@pytest.mark.parametrize("V", [1, 4, 5, 64, 65, 129, 130, 257, 1026, 2047, 2048])
def test_sampler_sweep(engine_small, V):
    """Every temperature x top_k pair twice, cycling top_p, penalty, seen bits and logit patterns, per-slot parameters,
    shuffled sparse slots, NaN in the padding columns."""
    z, prm = sweep_case(V, 182, 100 + V)
    run_checked(engine_small, f"sweep V={V}", V, z, prm, seed=V)


@gpu
def test_sampler_signed_zero(engine_small):
    """top_k 2 over {1.0, +0.0, -0.0, -1 ...}: both zeros tie at the k-th value and both must be kept on the fast path."""
    V, z, prm, disc = signed_zero_case()
    z, prm, disc = select(z, prm, disc, 64, 16)
    _, ref, _ = run_checked(engine_small, "signed zero", V, z, prm, disc=disc, need_disc=16)
    assert (ref.path == "fast").all()


@gpu
@pytest.mark.parametrize("survivors,path", [(128, "fast"), (129, "full")])
def test_sampler_ties_at_kth(engine_small, survivors, path):
    V, z, prm, disc = tie_case(survivors)
    z, prm, disc = select(z, prm, disc, 64, 24)
    _, ref, _ = run_checked(engine_small, f"ties {survivors}", V, z, prm, disc=disc, need_disc=24)
    assert (ref.path == path).all()


@gpu
@pytest.mark.parametrize("k", [1, 2, 50, 63, 64, 65, 127, 128])
def test_sampler_topk_boundary(engine_small, k):
    V, z, prm, disc = topk_boundary_case(k)
    z, prm, disc = select(z, prm, disc, 32, 8)
    _, ref, _ = run_checked(engine_small, f"top_k boundary {k}", V, z, prm, disc=disc, need_disc=8)
    assert (ref.path == ("fast" if k <= 64 else "full")).all()


@gpu
@pytest.mark.parametrize("path", ["fast", "full"])
@pytest.mark.parametrize("top_p", [0.5, 0.0])
def test_sampler_topp_exact_boundary(engine_small, path, top_p):
    """8 equal kept values: with top_p 0.5 the 4th cumulative sum is exactly 0.5 = 1 - top_p and must be dropped; with
    top_p 0 only the highest-index maximum survives, never id 0."""
    V, z, prm, disc = topp_boundary_case(path, top_p)
    z, prm, disc = select(z, prm, disc, 48, 12)
    run_checked(engine_small, f"top_p exact {path} {top_p}", V, z, prm, disc=disc, need_disc=12, min_decisive=1.0)


@gpu
@pytest.mark.parametrize("path", ["fast", "full"])
def test_sampler_topp_random_boundary(engine_small, path):
    V, z, prm, disc = topp_random_case(path)
    z, prm, disc = select(z, prm, disc, 64, 12)
    run_checked(engine_small, f"top_p boundary {path}", V, z, prm, disc=disc, need_disc=12)


@gpu
@pytest.mark.parametrize("V,top_k", [(1026, 0), (2048, 0), (64, 63), (5, 0)])
def test_sampler_philox_bits(engine_small, V, top_k):
    """Equal logits, top_p 1, T 1: the token is argmax u, which pins the kernel's Philox words for the high key word,
    negative and maximal seq_seed, and the counter at 0, 1, 604, cap - 1 and cap."""
    cap = 605
    seeds, sss, ns = [0, 2 ** 32 - 1, 2 ** 32, 2 ** 63 + 5], [0, 7, -1, 2 ** 31 - 1], [0, 1, 604, cap - 1, cap]
    grid = [(a, b, c) for a in seeds for b in sss for c in ns]
    R = len(grid)
    z = np.zeros((R, V), np.float32)
    prm = rows_params(R, top_k=top_k, V=V, seed=np.array([g[0] for g in grid], dtype=np.uint64),
                      seq_seed=[g[1] for g in grid], n=[g[2] for g in grid])
    _, ref, _ = run_checked(engine_small, f"philox V={V} top_k={top_k}", V, z, prm, cap=cap, min_decisive=1.0)
    u = noise_bits(prm["seed"], prm["seq_seed"], prm["n"], V) >> np.uint32(9)
    np.testing.assert_array_equal(ref.token, np.argmax(u, 1))


@gpu
@pytest.mark.parametrize("M", [1, 3, 64, 257])
def test_sampler_batches(engine_small, M):
    """M rows in one launch mixing greedy, fast-path and full-path rows with per-slot parameters, sparse shuffled slots."""
    V = 1026
    z, prm = sweep_case(V, M, 7 * M + 1)
    _, ref, _ = run_checked(engine_small, f"batch M={M}", V, z, prm, seed=M, extra_slots=M + 2)
    if M >= 64:
        assert set(ref.path) == {"greedy", "fast", "full"}


@gpu
@pytest.mark.parametrize("advance_ctx", [0, 1])
def test_sampler_state(engine_small, advance_ctx):
    """forced ids (some rows), the stop token forced and drawn, max_tokens at n + 1 and n + 2, finished already set,
    n >= cap (no tokens / sampled write): every slot's state as the reference implies, inactive slots untouched."""
    V, R, cap = 130, 48, 16
    rng = np.random.RandomState(advance_ctx)
    z, prm = sweep_case(V, R, 40 + advance_ctx)
    prm["n"] = rng.randint(0, cap, R)
    prm["n"][:6] = [cap, cap + 3, cap, cap + 1, cap + 7, cap]             # past the token buffer
    ref = reference(z, **prm)
    stop = rng.randint(0, V, R)
    stop[6:14] = ref.token[6:14]                                          # the drawn id is the stop token
    max_tokens = prm["n"] + rng.randint(1, 4, R)                          # n + 1 >= max_tokens on about a third
    n_slots = R + 6
    active = rng.permutation(n_slots)[:R].astype(np.int32)
    forced = rng.randint(-3, V, (n_slots, cap)).astype(np.int32)
    forced[active[:6]] = -1                                              # the rows past cap are not forced
    for r in range(6, 14):                                                # the stop token drawn, not forced
        forced[active[r], prm["n"][r]] = -1
    for r in range(14, 20):                                               # the stop token forced
        forced[active[r], prm["n"][r]] = stop[r]
    finished = (rng.rand(n_slots) < 0.25).astype(np.int32)
    st0 = dict(n_gen=rng.randint(0, cap, n_slots).astype(np.int32), ctx_len=rng.randint(0, 900, n_slots).astype(np.int32),
               finished=finished, last_tok=rng.randint(0, V, n_slots).astype(np.int32),
               seen=(rng.rand(n_slots, V) < 0.2).astype(np.uint8), tokens=rng.randint(-5, V, (n_slots, cap)).astype(np.int32),
               sampled=rng.randint(-5, V, (n_slots, cap)).astype(np.int32))
    st0["n_gen"][active] = prm["n"]
    st0["seen"][active] = prm["seen"]
    with pytest.raises(NativeError):                                      # forced with n >= cap is rejected
        run_checked(engine_small, "state", V, z, prm, cap=cap, forced=forced, st0=st0, active=active,
                    max_tokens=max_tokens, stop=stop, advance_ctx=advance_ctx)
    # the rows past cap without forced, the rest with it
    run_checked(engine_small, f"state past cap adv={advance_ctx}", V, z[:6], {k: v[:6] for k, v in prm.items()},
                cap=cap, st0=st0, active=active[:6], max_tokens=max_tokens[:6], stop=stop[:6], advance_ctx=advance_ctx,
                extra_slots=n_slots - 6)
    sub = {k: v[6:] for k, v in prm.items()}
    st, ref2, _ = run_checked(engine_small, f"state forced adv={advance_ctx}", V, z[6:], sub, cap=cap, forced=forced,
                              st0=st0, active=active[6:], max_tokens=max_tokens[6:], stop=stop[6:],
                              advance_ctx=advance_ctx, extra_slots=n_slots - (R - 6))
    assert st["finished"][active[14:20]].all()
    assert st["finished"][active[6:14]][ref2.decisive[:8]].all()


@gpu
def test_sampler_multi_step(engine_small):
    """8 steps feeding the returned state back in: the kernel's own seen bits drive the next penalty and its n_gen the
    next Philox counter."""
    V, R = 1026, 24
    rng = np.random.RandomState(3)
    z0, prm = sweep_case(V, R, 77)
    prm["T"] = np.array([[0.0, 0.75, 1.0][i % 3] for i in range(R)])
    prm["pen"] = np.full(R, 5.0)
    prm["n"] = np.arange(R) % 5
    st, _, active = run_checked(engine_small, "multi-step 0", V, z0, prm, seed=1, cap=40)
    for step in range(1, 8):
        z = (rng.randn(R, V) * 2).astype(np.float32)
        p = dict(prm, n=st["n_gen"][active], seen=st["seen"][active])
        st, _, _ = run_checked(engine_small, f"multi-step {step}", V, z, p, cap=40, st0=st, active=active)


@gpu
def test_sampler_repeatable(engine_small):
    V = 2048
    z, prm = sweep_case(V, 64, 5)
    rng = np.random.RandomState(0)
    active = rng.permutation(70)[:64]
    lg = np.full((64, V + 3), np.nan, np.float32)
    lg[:, :V] = z
    sps = [Sampling(temperature=float(prm["T"][i % 64]), top_p=float(prm["top_p"][i % 64]), top_k=int(prm["top_k"][i % 64]),
                    repetition_penalty=float(prm["pen"][i % 64]), seed=i, seq_seed=i) for i in range(70)]
    outs = [engine_small.debug_sample_slots(V, lg, active, sps, n_gen=np.arange(70), seen=np.zeros((70, V), np.uint8),
                                            cap=80) for _ in range(3)]
    for o in outs[1:]:
        for k in engine_small.SAMPLE_STATE:
            np.testing.assert_array_equal(o[k], outs[0][k])


@gpu
def test_sampler_rejections(engine_small):
    V = 130
    lg = np.zeros((2, V), np.float32)
    sps = [Sampling() for _ in range(3)]
    ok = dict(V=V, logits=lg, active=[0, 2], sps=sps, cap=4)
    engine_small.debug_sample_slots(**ok)
    bad = [dict(V=0), dict(V=2049), dict(active=[0, 0]), dict(active=[0, 3]), dict(active=[-1, 1]),
           dict(active=[0, 1, 2, 1], logits=np.zeros((4, V), np.float32)), dict(active=[], logits=np.zeros((0, V), np.float32)),
           dict(logits=np.zeros((2, V - 1), np.float32)), dict(cap=0), dict(n_gen=[-1, 0, 0]),
           dict(forced=np.zeros((3, 4), np.int32), n_gen=[0, 0, 4]), dict(forced=np.full((3, 4), V, np.int32))]
    for b in bad:
        kw = dict(ok, **b)
        if kw["V"] > lg.shape[1] and "logits" not in b:
            kw["logits"] = np.zeros((len(kw["active"]), max(kw["V"], 1)), np.float32)
        with pytest.raises((NativeError, ValueError)):
            engine_small.debug_sample_slots(**kw)
    # NULL required pointers, straight through the C ABI
    import ctypes as C
    lib, h = engine_small.lib, engine_small.h
    cs = (type(sps[0].c()) * 3)(*[s.c() for s in sps])
    act = np.array([0, 2], np.int32)
    i3 = [np.zeros(3, np.int32) for _ in range(4)]
    seen = np.zeros((3, V), np.uint8)
    tok = [np.zeros((3, 4), np.int32) for _ in range(2)]
    ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))
    args = [h, V, 2, ip(act), 3, lg.ctypes.data_as(C.POINTER(C.c_float)), V, cs, 4, 0, None, *[ip(a) for a in i3],
            seen.ctypes.data_as(C.POINTER(C.c_uint8)), ip(tok[0]), ip(tok[1])]
    assert lib.xtts_debug_sample_slots(*args) == 0
    for pos in [3, 5, 7, 11, 12, 13, 14, 15, 16, 17]:
        a = list(args)
        a[pos] = None
        assert lib.xtts_debug_sample_slots(*a) != 0, pos
