"""The speaker-conditioning kernels (csrc/cond.cu) launched one at a time through xtts_debug_cond, with the launch
configuration xtts_condition uses, and compared with plain float64 references of the same operations.

Tolerances: frame_window and transpose move or multiply exactly once, so they are bit-exact.  preemphasis, se_apply and
relu_bn_rows round once (a contracted fma), so they are within 1 ulp of the float64 result rounded to fp32.  Ops with
logf / erff / expf get a few ulp plus the propagated input error.  Reductions get the bound stated beside each one; the
CPU tests check that an fp32 simulation of the kernel's summation order stays inside it.  Outputs go through guard words
on the device, so a kernel that writes outside its output fails the call."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import xtts_oracle as O

U = 2.0 ** -24                     # unit roundoff of fp32
_F64 = np.float64
_F32 = np.float32


def f32(a):
    return np.asarray(a, dtype=_F32)


def ulp(x):
    return np.spacing(np.abs(np.asarray(x, _F64)).astype(_F32)).astype(_F64)


# ------------------------------------------------------------------------------------------------ float64 references
def ref_frame_window(x, win, hop, off, pad, mode, frames):
    x = np.asarray(x, _F64)
    if mode == 0:
        xp = np.pad(x, pad, mode="reflect")
    else:
        xp = np.pad(np.where(np.isfinite(x), x, 0.0), pad)
    wlen = len(win)
    idx = np.arange(frames)[:, None] * hop + off + np.arange(wlen)[None]
    return np.asarray(win, _F64)[None] * xp[idx]


def ref_power(D, nb):
    D = np.asarray(D, _F64)
    return D[:, :nb] ** 2 + D[:, nb:] ** 2


def ref_mel_log(M, stats, mode):
    M = np.asarray(M, _F64).reshape(-1)
    if mode == 0:
        C = len(stats)
        return np.log(np.maximum(M, float(_F32(1e-5)))) / np.asarray(stats, _F64)[np.arange(M.size) % C]
    return np.log(M + float(_F32(1e-6)))


def ref_preemphasis(x, coef):
    x = np.asarray(x, _F64)
    prev = np.concatenate([[x[1]], x[:-1]])
    return x - float(_F32(coef)) * prev


def ref_instnorm_t(X, eps):                      # [T][C] -> [C][T]
    X = np.asarray(X, _F64)
    m = X.mean(0)
    v = ((X - m) ** 2).mean(0)
    return ((X - m) / np.sqrt(v + eps)).T


def ref_groupnorm(X, w, b, groups, eps):         # rows [T][C]
    X = np.asarray(X, _F64)
    T, C = X.shape
    g = X.reshape(T, groups, C // groups)
    m = g.mean(axis=(0, 2), keepdims=True)
    v = ((g - m) ** 2).mean(axis=(0, 2), keepdims=True)
    return ((g - m) / np.sqrt(v + eps)).reshape(T, C) * np.asarray(w, _F64) + np.asarray(b, _F64)


def ref_geglu(Hc):
    Hc = np.asarray(Hc, _F64)
    Fh = Hc.shape[1] // 2
    x, gate = Hc[:, :Fh], Hc[:, Fh:]
    return 0.5 * gate * (1.0 + np.vectorize(math.erf)(gate / math.sqrt(2.0))) * x


def ref_rmsnorm_accum(X, gamma, acc, scale):
    X = np.asarray(X, _F64)
    n = np.maximum(np.sqrt((X ** 2).sum(1, keepdims=True)), 1e-12)
    return np.asarray(acc, _F64) + X / n * math.sqrt(X.shape[1]) * np.asarray(gamma, _F64) * float(_F32(scale))


def conv_out(n, k, stride):
    return (n + 2 * (k // 2) - k) // stride + 1


def ref_conv2d(x, w, bias, bn, stride, relu_before_bn):
    """x [Cin][H][W], w [Cout][Cin][k][k], padding k/2; y = bn(relu?(conv + bias))."""
    x, w = np.asarray(x, _F64), np.asarray(w, _F64)
    Cin, H, W = x.shape
    Cout, _, k, _ = w.shape
    p = k // 2
    Ho, Wo = conv_out(H, k, stride), conv_out(W, k, stride)
    xp = np.pad(x, ((0, 0), (p, p), (p, p)))
    y = np.zeros((Cout, Ho, Wo))
    for ky in range(k):
        for kx in range(k):
            patch = xp[:, ky: ky + stride * (Ho - 1) + 1: stride, kx: kx + stride * (Wo - 1) + 1: stride]
            y += np.einsum("oc,chw->ohw", w[:, :, ky, kx], patch)
    if bias is not None:
        y += np.asarray(bias, _F64)[:, None, None]
    if relu_before_bn:
        y = np.maximum(y, 0.0)
    if bn is not None:
        y = y * np.asarray(bn[0], _F64)[:, None, None] + np.asarray(bn[1], _F64)[:, None, None]
    return y


def ref_se_gate(m, w1, b1, w2, b2):
    h = np.maximum(np.asarray(w1, _F64) @ np.asarray(m, _F64) + b1, 0.0)
    return 1.0 / (1.0 + np.exp(-(np.asarray(w2, _F64) @ h + b2)))


def ref_se_apply(x, gate, resid):
    return np.maximum(np.asarray(x, _F64) * np.asarray(gate, _F64)[:, None] + resid, 0.0)


def ref_relu_bn_rows(X, sc, sh):
    return np.maximum(np.asarray(X, _F64), 0.0) * np.asarray(sc, _F64) + np.asarray(sh, _F64)


def ref_asp(A, X):
    """logits A [T][C], features X [C][T] -> (mu [C], sg [C]) (hifigan_decoder.py:632-640)."""
    A, X = np.asarray(A, _F64), np.asarray(X, _F64)
    w = np.exp(A - A.max(0))
    w = (w / w.sum(0)).T
    mu = (w * X).sum(1)
    return mu, np.sqrt(np.maximum((w * X * X).sum(1) - mu ** 2, 1e-5))


def ref_l2norm(x):
    x = np.asarray(x, _F64)
    return x / max(np.sqrt((x ** 2).sum()), 1e-12)


def ref_gemv(W, g, b):
    y = np.asarray(W, _F64) @ np.asarray(g, _F64)
    return y + np.asarray(b, _F64) if b is not None else y


def ref_mel22(wav, mel_stats, n_mels):
    """Hann 1024 inside a 2048-point frame (taps 512..1535), hop 256, reflect pad 1024, slaney mel, log / stats."""
    from auralis_b200.weights import mel_filterbank
    n = len(wav)
    T = 1 + n // 256
    win = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(1024) / 1024)
    Fr = ref_frame_window(wav, win, 256, 512, 1024, 0, T)
    full = np.zeros((T, 2048))
    full[:, 512:1536] = Fr
    P = np.abs(np.fft.rfft(full, axis=1)) ** 2
    fb = mel_filterbank(1025, 0.0, 8000.0, n_mels, 22050, "slaney").double().numpy()
    return np.log(np.maximum(P @ fb, 1e-5)) / np.asarray(mel_stats, _F64)


def ref_mel16(wav, core):
    """pre-emphasis 0.97, Hamming 400 inside a 512-point frame (taps 56..455), hop 160, reflect pad 256, mel,
    log(+1e-6), InstanceNorm over time -> [64][T]."""
    s = "hifigan_decoder.speaker_encoder."
    x = ref_preemphasis(wav, 0.97)
    T = 1 + len(x) // 160
    Fr = ref_frame_window(x, core[s + "torch_spec.1.spectrogram.window"].double().numpy(), 160, 56, 256, 0, T)
    full = np.zeros((T, 512))
    full[:, 56:456] = Fr
    P = np.abs(np.fft.rfft(full, axis=1)) ** 2
    mel = np.log(P @ core[s + "torch_spec.1.mel_scale.fb"].double().numpy() + 1e-6)
    return ref_instnorm_t(mel, 1e-5)


# ------------------------------------------------------------------------------------------------ error bounds
# block_sum (common.cuh): element e is summed sequentially on thread e % threads, then a 5-level butterfly inside each
# warp and a 5-level butterfly over the warp sums.  Each partial sum passes through at most
#   depth(n, threads) = ceil(n / threads) + 10
# additions, so |fl(sum) - sum| <= depth * u * sum |terms|.
def depth(n, threads):
    return -(-n // threads) + 10


def norm_bound(X, axis_n, threads, eps):
    """Bound on (x - mean) * rstd for a two-pass mean / biased-variance normalisation over n = axis_n values:
    e_mean = (depth + 2) u mean|x|;  e_var = (depth + 4) u var + 2 e_mean mean|x - mean| + e_mean^2;
    rstd relative error r = (e_var / (var + eps) + u) / 2 + 3u;
    |err| <= (e_mean + |x - mean| (r + 3u)) * rstd.  X: float64 [..., n] with the reduction over the last axis."""
    k = depth(axis_n, threads)
    m = X.mean(-1, keepdims=True)
    d = np.abs(X - m)
    v = (d ** 2).mean(-1, keepdims=True)
    e_mean = (k + 2) * U * np.abs(X).mean(-1, keepdims=True)
    e_var = (k + 4) * U * v + 2 * e_mean * d.mean(-1, keepdims=True) + e_mean ** 2
    rstd = 1.0 / np.sqrt(v + eps)
    r = 0.5 * (e_var / (v + eps) + U) + 3 * U
    return (e_mean + d * (r + 3 * U)) * rstd


def sumsq_scale_bound(X, threads):
    """Relative error of x / sqrt(sum x^2) (l2norm, rmsnorm): (depth / 2 + 4) u."""
    return (depth(X.shape[-1], threads) / 2 + 4) * U


def asp_bound(A, X, threads=128):
    """ASP: e_t = expf(a_t - max) carries relative error eps_e = (3 + max|a - max|) u (the rounded difference moves the
    exponent); the three sums add depth u.  With s = depth + 2 and q = s u + eps_e:
      |d mu| <= q (sum w|x| + |mu|);  |d m2| <= q (sum w x^2 + m2);  |d var| <= |d m2| + 2|mu||d mu| + 4u m2;
      |d sg| <= |d var| / (sg + sqrt(1e-5)) + 2u sg."""
    A, X = np.asarray(A, _F64), np.asarray(X, _F64)
    T = A.shape[0]
    w = np.exp(A - A.max(0))
    w = (w / w.sum(0)).T
    q = (depth(T, threads) + 2) * U + (3 + (A.max(0) - A.min(0))) * U
    mu = (w * X).sum(1)
    m2 = (w * X * X).sum(1)
    dmu = q * ((w * np.abs(X)).sum(1) + np.abs(mu))
    dvar = q * (m2 + m2) + 2 * np.abs(mu) * dmu + 4 * U * m2
    sg = np.sqrt(np.maximum(m2 - mu ** 2, 1e-5))
    return dmu + 2 * U * np.abs(mu), dvar / (sg + math.sqrt(1e-5)) + 2 * U * sg


def gemv_bound(W, g, b):
    """launch_gemv: lane l sums columns l, l + 32, ... then a 5-level butterfly, plus the bias:
    (ceil(cols / 32) + 6) u sum|W g| + u |y|."""
    W, g = np.asarray(W, _F64), np.asarray(g, _F64)
    k = -(-W.shape[1] // 32) + 6
    y = ref_gemv(W, g, b)
    return k * U * (np.abs(W) @ np.abs(g)) + U * np.abs(y)


def conv2d_bound(x, w, bias, bn, stride, relu):
    """Sequential fma over Cin * k * k taps: n u sum|w x|; then + bias (u), relu, * scale + shift (2u):
    |err| <= |scale| (n u sum|w x| + u |conv + bias|) + 2u (|y| + |shift|)."""
    Cin, k = w.shape[1], w.shape[2]
    n = Cin * k * k
    s = ref_conv2d(np.abs(x), np.abs(w), None, None, stride, 0)
    pre = np.abs(ref_conv2d(x, w, bias, None, stride, 0))
    y = np.abs(ref_conv2d(x, w, bias, bn, stride, relu))
    sc = np.abs(np.asarray(bn[0], _F64))[:, None, None] if bn is not None else 1.0
    sh = np.abs(np.asarray(bn[1], _F64))[:, None, None] if bn is not None else 0.0
    return sc * (n * U * s + U * pre) + 2 * U * (y + sh)


# ------------------------------------------------------------------------------------------------ fp32 simulations
def sim_block_sum(terms, threads, square=False):
    """block_sum of fp32 terms in the kernel's order (fmaf(x, x, s) when square)."""
    t = f32(terms).reshape(-1)
    n = t.size
    rows = -(-n // threads)
    p = np.zeros(rows * threads, _F32)
    p[:n] = t
    p = p.reshape(rows, threads)
    acc = np.zeros(threads, _F32)
    for r in range(rows):
        acc = f32(acc.astype(_F64) + p[r].astype(_F64) ** 2) if square else f32(acc + p[r])

    def warp(v):
        v = f32(v)
        for o in (16, 8, 4, 2, 1):
            v = f32(v + v[np.arange(32) ^ o])
        return v[0]
    red = np.zeros(32, _F32)
    nw = threads // 32
    red[:nw] = [warp(acc[i * 32:(i + 1) * 32]) for i in range(nw)]
    return warp(red)


def sim_norm(x, eps, threads=256, one_pass=False):
    """instnorm_transpose / groupnorm's normalisation of one channel (group) x [n] in fp32."""
    x = f32(x)
    n = x.size
    mean = f32(sim_block_sum(x, threads) / _F32(n))
    if one_pass:
        var = f32(f32(sim_block_sum(x, threads, True) / _F32(n)) - mean * mean)
    else:
        var = f32(sim_block_sum(f32(x - mean), threads, True) / _F32(n))
    rstd = f32(_F32(1) / np.sqrt(f32(var + _F32(eps))))
    return f32(f32(x - mean) * rstd)


def stress_rows(rng, n):
    """Series for the normalisations: plain, a 1e3 DC offset, a 1e3 offset with spread 1e-2, and constant."""
    return [rng.randn(n), 1e3 + rng.randn(n), 1e3 + 1e-2 * rng.randn(n), np.full(n, 0.75)]


# ------------------------------------------------------------------------------------------------ CPU checks
def test_reference_frame_window_and_dft_match_torch_stft():
    rng = np.random.RandomState(0)
    for n_fft, wlen, hop, win, n in ((2048, 1024, 256, torch.hann_window(1024, dtype=torch.float64), 9000),
                                     (512, 400, 160, torch.hamming_window(400, dtype=torch.float64), 4321)):
        x = rng.randn(n)
        off, pad, T = (n_fft - wlen) // 2, n_fft // 2, 1 + n // hop
        Fr = ref_frame_window(x, win.numpy(), hop, off, pad, 0, T)
        full = np.zeros((T, n_fft))
        full[:, off:off + wlen] = Fr
        got = np.fft.rfft(full, axis=1)
        exp = torch.stft(torch.from_numpy(x), n_fft, hop, wlen, window=win, center=True, pad_mode="reflect",
                         return_complex=True).numpy().T
        np.testing.assert_allclose(got, exp, rtol=0, atol=1e-9 * np.abs(exp).max())
        np.testing.assert_allclose(ref_power(np.concatenate([got.real, got.imag], 1), n_fft // 2 + 1), np.abs(exp) ** 2,
                                   rtol=1e-12, atol=1e-9)
    # zero padding with NaN / inf read as 0 (librosa.stft(center=True) after np.nan_to_num, as the enhancer uses it)
    x = rng.randn(600)
    x[[0, 5, 599]] = [np.nan, np.inf, -np.inf]
    Fr = ref_frame_window(x, np.ones(64), 16, 0, 32, 1, 1 + 600 // 16)
    xz = np.pad(np.nan_to_num(x, nan=0.0, posinf=0.0, neginf=0.0), 32)
    assert np.array_equal(Fr[3], xz[48:112])


def test_reference_norms_and_activations_match_torch():
    rng = np.random.RandomState(1)
    X = rng.randn(37, 24) + 5.0
    t = torch.from_numpy(X)
    np.testing.assert_allclose(ref_instnorm_t(X, 1e-5), F.instance_norm(t.T[None], eps=1e-5)[0].numpy(), atol=1e-12)
    w, b = rng.randn(24), rng.randn(24)
    for groups in (1, 6, 24):
        exp = F.group_norm(t.T[None], groups, torch.from_numpy(w), torch.from_numpy(b), 1e-5)[0].T.numpy()
        np.testing.assert_allclose(ref_groupnorm(X, w, b, groups, 1e-5), exp, atol=1e-12)
    gamma, acc = rng.randn(24), rng.randn(37, 24)
    exp = acc + F.normalize(t, dim=-1).numpy() * math.sqrt(24) * gamma * float(_F32(1 / 3))
    np.testing.assert_allclose(ref_rmsnorm_accum(X, gamma, acc, 1 / 3), exp, atol=1e-12)
    np.testing.assert_allclose(ref_l2norm(X[0]), F.normalize(t[0], dim=0).numpy(), atol=1e-15)
    assert np.array_equal(ref_l2norm(np.zeros(5)), np.zeros(5))
    Hc = rng.randn(5, 16) * 3
    h = torch.from_numpy(Hc)
    np.testing.assert_allclose(ref_geglu(Hc), (F.gelu(h[:, 8:]) * h[:, :8]).numpy(), atol=1e-12)


@pytest.mark.parametrize("k,stride,bias,bn,relu", [(3, 1, True, True, True), (3, 2, False, True, False), (1, 2, False, True, False),
                                                   (3, 1, False, False, False)])
def test_reference_conv2d_matches_torch(k, stride, bias, bn, relu):
    rng = np.random.RandomState(2)
    x, w = rng.randn(3, 7, 10), rng.randn(5, 3, k, k)
    b = rng.randn(5) if bias else None
    sc, sh = rng.rand(5) + 0.5, rng.randn(5)
    got = ref_conv2d(x, w, b, (sc, sh) if bn else None, stride, relu)
    y = F.conv2d(torch.from_numpy(x)[None], torch.from_numpy(w), torch.from_numpy(b) if bias else None, stride=stride,
                 padding=k // 2)[0]
    if relu:
        y = F.relu(y)
    if bn:
        y = y * torch.from_numpy(sc)[:, None, None] + torch.from_numpy(sh)[:, None, None]
    np.testing.assert_allclose(got, y.numpy(), atol=1e-12)


def test_reference_se_asp_gemv_match_torch():
    rng = np.random.RandomState(3)
    C, R, T = 12, 3, 40
    m, w1, b1, w2, b2 = rng.randn(C), rng.randn(R, C), rng.randn(R), rng.randn(C, R), rng.randn(C)
    exp = torch.sigmoid(torch.from_numpy(w2) @ F.relu(torch.from_numpy(w1) @ torch.from_numpy(m) + torch.from_numpy(b1))
                        + torch.from_numpy(b2))
    np.testing.assert_allclose(ref_se_gate(m, w1, b1, w2, b2), exp.numpy(), atol=1e-14)
    A, X = rng.randn(T, C) * 3, rng.randn(C, T)
    x, a = torch.from_numpy(X)[None], torch.from_numpy(A.T)[None]
    wt = torch.softmax(a, dim=2)
    mu = torch.sum(x * wt, dim=2)
    sg = torch.sqrt((torch.sum(x ** 2 * wt, dim=2) - mu ** 2).clamp(min=1e-5))
    got = ref_asp(A, X)
    np.testing.assert_allclose(got[0], mu[0].numpy(), atol=1e-13)
    np.testing.assert_allclose(got[1], sg[0].numpy(), atol=1e-13)
    W, g, b = rng.randn(9, 33), rng.randn(33), rng.randn(9)
    np.testing.assert_allclose(ref_gemv(W, g, b), F.linear(torch.from_numpy(g), torch.from_numpy(W), torch.from_numpy(b)).numpy(),
                               atol=1e-13)


@pytest.mark.parametrize("name", ["small", "full"])
def test_reference_frontends_match_oracle(name, request):
    dims = request.getfixturevalue(f"dims_{name}")
    core = request.getfixturevalue(f"state_{name}")[1]
    w22 = O.synthetic_reference_wav(0.5, 22050, 130.0, 4).double()
    exp = O.mel_cloning(w22, core["mel_stats"].double(), dims.cond.n_mels).numpy().T
    np.testing.assert_allclose(ref_mel22(w22.numpy(), core["mel_stats"].numpy(), dims.cond.n_mels), exp, atol=1e-9)
    w16 = O.synthetic_reference_wav(0.7, 16000, 130.0, 4).double()
    exp = O.speaker_frontend(w16, core)[0].numpy()
    np.testing.assert_allclose(ref_mel16(w16.numpy(), core), exp, atol=1e-8)


@pytest.mark.parametrize("n", [1, 100, 300, 1000, 4001])
def test_norm_bound_covers_fp32_two_pass(n):
    """The two-pass normalisation bound covers the kernel's fp32 order, and a one-pass variance (E[x^2] - E[x]^2)
    breaks it once a DC offset is present."""
    rng = np.random.RandomState(n)
    broke = False
    for x in stress_rows(rng, n):
        xs = f32(x)
        ref = ref_instnorm_t(xs.astype(_F64)[:, None], 1e-5)[0]
        bound = norm_bound(xs.astype(_F64)[None], n, 256, 1e-5)[0]
        assert (np.abs(sim_norm(xs, 1e-5) - ref) <= bound).all()
        with np.errstate(invalid="ignore"):         # a one-pass variance can go negative: NaN counts as outside
            broke |= bool((~(np.abs(sim_norm(xs, 1e-5, one_pass=True) - ref) <= bound)).any())
    assert broke or n == 1


def test_sum_bounds_cover_fp32_simulation():
    rng = np.random.RandomState(5)
    for n, threads in ((1, 256), (37, 256), (300, 256), (5000, 256), (2048, 128), (77, 128)):
        x = f32(rng.randn(n) * 10 + 3)
        s = sim_block_sum(x, threads)
        assert abs(float(s) - x.astype(_F64).sum()) <= depth(n, threads) * U * np.abs(x.astype(_F64)).sum()
        ss = sim_block_sum(x, threads, square=True)
        nrm = np.sqrt((x.astype(_F64) ** 2).sum())
        y = f32(x / np.maximum(np.sqrt(ss), _F32(1e-12)))
        assert (np.abs(y - x / nrm) <= sumsq_scale_bound(x[None], threads) * np.abs(x / nrm) + U * np.abs(x / nrm)).all()
    # ASP in fp32, kernel order, logits around +-80 with a spread of 8
    for T in (1, 50, 300):
        A = f32(np.where(np.arange(6) % 2, 80.0, -80.0)[None] + 8 * rng.randn(T, 6))
        X = f32(rng.randn(6, T))
        X[5] = 0.5
        mu_r, sg_r = ref_asp(A, X)
        bmu, bsg = asp_bound(A, X)
        for c in range(6):
            mx = A[:, c].max()
            e = f32(np.exp(f32(A[:, c] - mx).astype(_F64)))
            se = sim_block_sum(e, 128)
            s1 = sim_block_sum(f32(e * X[c]), 128)
            s2 = sim_block_sum(f32(e * f32(X[c] * X[c])), 128)
            mu = f32(s1 / se)
            sg = np.sqrt(np.maximum(f32(f32(s2 / se) - mu * mu), _F32(1e-5)))
            assert abs(mu - mu_r[c]) <= bmu[c] and abs(sg - sg_r[c]) <= bsg[c], (T, c)
    # gemv, warp order
    W, g = f32(rng.randn(13, 70)), f32(rng.randn(70))
    lanes = np.zeros((13, 32), _F32)
    for c0 in range(0, 70, 32):
        blk = f32(W[:, c0:c0 + 32].astype(_F64) * g[c0:c0 + 32])
        lanes[:, :blk.shape[1]] = f32(lanes[:, :blk.shape[1]] + blk)
    for o in (16, 8, 4, 2, 1):
        lanes = f32(lanes + lanes[:, np.arange(32) ^ o])
    assert (np.abs(lanes[:, 0] - ref_gemv(W, g, None)) <= gemv_bound(W, g, None)).all()


# ------------------------------------------------------------------------------------------------ GPU
def run(eng, op, dims, inputs=(), out=None, out_len=None, scal=()):
    return eng.debug_cond(op, dims, inputs, out=out, out_len=out_len, scal=scal)


def check(got, ref, tol, what=""):
    got = np.asarray(got, _F64).reshape(np.shape(ref))
    err = np.abs(got - ref)
    bad = ~(err <= tol)
    assert not bad.any(), f"{what}: {bad.sum()} of {bad.size} outside the bound, worst {np.max(err - tol):.3e} at {np.argmax(err - tol)}"


gpu = pytest.mark.gpu


@gpu
@pytest.mark.parametrize("n,wlen,hop,off,pad,mode,threads", [
    (1025, 1024, 256, 512, 1024, 0, 256),     # 22.05 kHz front-end, n just above pad: reflect at both ends
    (2000, 1024, 256, 512, 1024, 0, 256),
    (257, 400, 160, 56, 256, 0, 128),         # 16 kHz front-end: 400 taps on 128 threads, n just above pad
    (4321, 400, 160, 56, 256, 0, 128),
    (3000, 2048, 512, 0, 1024, 1, 256),       # the enhancer's zero-padded librosa frame, NaN / inf samples
])
def test_frame_window_bit_exact(engine_small, n, wlen, hop, off, pad, mode, threads):
    rng = np.random.RandomState(n)
    x = f32(rng.randn(n))
    if mode == 1:
        x[[0, 7, 1500, n - 1]] = [np.nan, np.inf, -np.inf, np.nan]
    win = f32(rng.rand(wlen) + 0.1)
    T = 1 + n // hop
    got = run(engine_small, "FRAME_WINDOW", [n, wlen, hop, off, pad, mode, T, threads], [x, win], out_len=T * wlen)
    exp = f32(ref_frame_window(x, win, hop, off, pad, mode, T)).reshape(-1)
    assert np.array_equal(got.view(np.uint32), exp.view(np.uint32))


@gpu
def test_power_and_transpose(engine_small):
    rng = np.random.RandomState(7)
    T, nb = 13, 257
    D = f32(rng.randn(T, 2 * nb) * np.exp(rng.randn(T, 2 * nb)))
    got = run(engine_small, "POWER", [T, nb], [D], out_len=T * nb)
    ref = ref_power(D, nb)
    # contracted to fma(re, re, im * im) (or the mirror): one product and the sum round, |err| <= 2u P
    check(got, ref, 2 * U * ref, "power")
    for R, Cc in ((2048, 3), (5, 131), (1, 1)):
        x = f32(rng.randn(R, Cc))
        got = run(engine_small, "TRANSPOSE", [R, Cc], [x], out_len=R * Cc)
        assert np.array_equal(got.reshape(Cc, R), x.T)


@gpu
def test_mel_log(engine_small):
    rng = np.random.RandomState(8)
    C, T = 80, 7
    M = f32(np.exp(rng.randn(T, C) * 4))
    M[0, :10] = 0.0
    M[1, :10] = 3e-6                  # below the 1e-5 clamp
    M[2, :10] = f32(1e-5)
    stats = f32(0.5 + rng.rand(C) * 2)
    got = run(engine_small, "MEL_LOG", [T * C, C, 0], [stats], out=M)
    ref = ref_mel_log(M, stats, 0).reshape(T, C)
    check(got, ref, 4 * U * np.abs(ref) + 2 * U / stats, "mel_log mode 0")
    M1 = f32(np.exp(rng.randn(1001) * 4))
    M1[:5] = 0.0
    got = run(engine_small, "MEL_LOG", [1001, 64, 1], [], out=M1)
    ref = ref_mel_log(M1, None, 1)
    check(got, ref, 4 * U * np.abs(ref) + 2 * U, "mel_log mode 1")


@gpu
@pytest.mark.parametrize("n", [2, 3, 400, 70001])
def test_preemphasis(engine_small, n):
    x = f32(np.random.RandomState(n).randn(n))
    got = run(engine_small, "PREEMPHASIS", [n], [x], out_len=n, scal=[0.97])
    ref = ref_preemphasis(x, 0.97)
    check(got, f32(ref), ulp(ref), "preemphasis")


@gpu
@pytest.mark.parametrize("T", [1, 100, 256, 257, 1051])
def test_instnorm_transpose(engine_small, T):
    rng = np.random.RandomState(T)
    C = 64
    X = rng.randn(T, C)
    X[:, 1::4] += 1e3                 # a large DC offset: a one-pass variance fails here
    X[:, 2::4] = 1e3 + 1e-2 * rng.randn(T, C // 4)
    X[:, 3] = 0.25                    # constant: variance 0, eps alone
    X = f32(X)
    got = run(engine_small, "INSTNORM_T", [T, C], [X], out_len=T * C, scal=[1e-5])
    check(got, ref_instnorm_t(X, 1e-5), norm_bound(X.T.astype(_F64), T, 256, 1e-5), "instnorm")


@gpu
@pytest.mark.parametrize("T,C,groups", [(1, 128, 32), (61, 128, 32), (300, 128, 128), (97, 1024, 32), (3, 64, 16)])
def test_groupnorm(engine_small, T, C, groups):
    rng = np.random.RandomState(T + C)
    X = rng.randn(T, C) * 2
    X[:, : C // 2] += 3e2
    X = f32(X)
    w, b = f32(1 + 0.3 * rng.randn(C)), f32(rng.randn(C))
    got = run(engine_small, "GROUPNORM", [T, C, groups], [X, w, b], out_len=T * C, scal=[1e-5])
    ref = ref_groupnorm(X, w, b, groups, 1e-5)
    cpg = C // groups
    g = X.astype(_F64).reshape(T, groups, cpg).transpose(1, 0, 2).reshape(groups, T * cpg)
    nb = norm_bound(g, T * cpg, 256, 1e-5).reshape(groups, T, cpg).transpose(1, 0, 2).reshape(T, C)
    check(got, ref, nb * np.abs(w) + 3 * U * (np.abs(ref) + np.abs(b)), "groupnorm")


@gpu
def test_geglu(engine_small):
    rng = np.random.RandomState(9)
    rows, Fh = 32, 2048
    Hc = f32(rng.randn(rows, 2 * Fh) * 4)
    got = run(engine_small, "GEGLU", [rows, Fh], [Hc], out_len=rows * Fh)
    ref = ref_geglu(Hc)
    # 1 + erff(gate * 0.7071f) carries 5u absolute (erff 2 ulp, the rounded argument moves it by <= 0.5u, the sum u);
    # the products add 3u relative
    check(got, ref, 0.5 * np.abs(Hc[:, Fh:].astype(_F64) * Hc[:, :Fh]) * 5 * U + 6 * U * np.abs(ref), "geglu")


@gpu
@pytest.mark.parametrize("C", [128, 1024])
def test_rmsnorm_accum(engine_small, C):
    rng = np.random.RandomState(C)
    rows = 32
    X = f32(rng.randn(rows, C) * 3)
    X[5] = 0.0                         # zero row: the norm clamps at 1e-12 and acc is unchanged
    gamma, acc = f32(rng.randn(C)), f32(rng.randn(rows, C))
    got = run(engine_small, "RMSNORM_ACCUM", [rows, C], [X, gamma], out=acc, scal=[1 / 3])
    ref = ref_rmsnorm_accum(X, gamma, acc, 1 / 3)
    term = np.abs(ref - acc)
    check(got, ref, term * (sumsq_scale_bound(X, 256) + 6 * U) + U * np.abs(ref), "rmsnorm_accum")
    assert np.array_equal(got.reshape(rows, C)[5], acc[5])


CONV_CASES = [
    # Cin, Cout, H, W, k, stride, bias, bn, relu
    (1, 8, 64, 61, 3, 1, True, True, True),        # the stem at the golden length
    (8, 16, 64, 301, 3, 2, False, True, True),     # odd W, Wout 151 > 128: two x-blocks
    (8, 16, 64, 301, 1, 2, False, True, False),    # downsample at odd T
    (8, 6, 7, 260, 3, 1, True, False, False),      # Cout 6: the co0 + c < Cout tail, odd H, Wout 260
    (16, 4, 32, 102, 3, 2, False, True, False),
    (256, 256, 8, 33, 3, 1, False, True, False),   # Cin 256: 36 KB of shared memory, the production maximum
    (128, 256, 16, 132, 1, 2, False, True, False),
    (64, 64, 9, 129, 3, 2, True, True, True),      # odd H with stride 2
]


@gpu
@pytest.mark.parametrize("Cin,Cout,H,W,k,stride,bias,bn,relu", CONV_CASES)
def test_conv2d(engine_full, Cin, Cout, H, W, k, stride, bias, bn, relu):
    rng = np.random.RandomState(Cin * 7 + Cout + W)
    x = f32(rng.randn(Cin, H, W))
    w = f32(rng.randn(Cout, Cin, k, k) / math.sqrt(Cin * k * k))   # no symmetry: a transposed tap is visible
    b = f32(rng.randn(Cout)) if bias else None
    sc, sh = f32(rng.rand(Cout) + 0.5), f32(rng.randn(Cout))
    ins = [x, w] + ([b] if bias else []) + ([sc, sh] if bn else [])
    Ho, Wo = conv_out(H, k, stride), conv_out(W, k, stride)
    got = run(engine_full, "CONV2D", [Cin, Cout, H, W, k, stride, int(relu), int(bias), int(bn)], ins, out_len=Cout * Ho * Wo)
    bnp = (sc, sh) if bn else None
    check(got, ref_conv2d(x, w, b, bnp, stride, relu), conv2d_bound(x, w, b, bnp, stride, relu), "conv2d")


@gpu
def test_channel_mean_se_gate_se_apply(engine_small):
    rng = np.random.RandomState(10)
    for C, HW in ((8, 64 * 61), (256, 8 * 13), (3, 1)):
        x = f32(rng.randn(C, HW) + 2)
        got = run(engine_small, "CHANNEL_MEAN", [C, HW], [x], out_len=C)
        ref = x.astype(_F64).mean(1)
        check(got, ref, (depth(HW, 256) + 2) * U * np.abs(x.astype(_F64)).mean(1), "channel_mean")
    for C, R in ((8, 1), (512, 32)):             # R = 1: the small geometry's squeeze
        m, w1, b1 = f32(rng.randn(C)), f32(rng.randn(R, C) / math.sqrt(C)), f32(rng.randn(R))
        w2, b2 = f32(rng.randn(C, R) / math.sqrt(R)), f32(rng.randn(C))
        got = run(engine_small, "SE_GATE", [C, R], [m, w1, b1, w2, b2], out_len=C)
        ref = ref_se_gate(m, w1, b1, w2, b2)
        # hidden: C fma terms; pre-activation: R terms plus the hidden error; sigmoid slope <= 1/4, expf 2 ulp
        h = np.maximum(w1.astype(_F64) @ m + b1, 0)
        eh = (C + 1) * U * (np.abs(w1.astype(_F64)) @ np.abs(m) + np.abs(b1))
        es = (R + 1) * U * (np.abs(w2.astype(_F64)) @ h + np.abs(b2)) + np.abs(w2.astype(_F64)) @ eh
        check(got, ref, 0.25 * es + ref * (1 - ref) * 3 * U + 4 * U * ref, "se_gate")
        HW = 77
        x, resid = f32(rng.randn(C, HW)), f32(rng.randn(C, HW))
        gate = f32(rng.rand(C))
        got = run(engine_small, "SE_APPLY", [C, HW], [x, gate, resid], out_len=C * HW)
        ref = ref_se_apply(x, gate, resid)
        check(got, f32(ref), ulp(ref), "se_apply")


@gpu
def test_relu_bn_rows(engine_small):
    rng = np.random.RandomState(11)
    rows, C = 101, 128
    X = f32(rng.randn(rows, C))
    sc, sh = f32(rng.randn(C)), f32(rng.randn(C))
    got = run(engine_small, "RELU_BN_ROWS", [rows, C], [sc, sh], out=X)
    ref = ref_relu_bn_rows(X, sc, sh)
    check(got, f32(ref), ulp(ref), "relu_bn_rows")


@gpu
@pytest.mark.parametrize("T,C", [(1, 64), (100, 512), (128, 64), (263, 2048)])
def test_asp(engine_full, T, C):
    rng = np.random.RandomState(T + C)
    A = f32(np.where(np.arange(C) % 4 == 1, 80.0, np.where(np.arange(C) % 4 == 2, -80.0, 0.0))[None]
            + np.where(np.arange(C) % 4 == 3, 0.05, 8.0)[None] * rng.randn(T, C))
    X = f32(rng.randn(C, T))
    X[::5] = 0.3                                  # constant features: the variance clamps at 1e-5
    got = run(engine_full, "ASP", [T, C], [A, X], out_len=2 * C).reshape(2, C)
    mu, sg = ref_asp(A, X)
    bmu, bsg = asp_bound(A, X)
    check(got[0], mu, bmu, "asp mean")
    check(got[1], sg, bsg, "asp std")


@gpu
@pytest.mark.parametrize("n", [32, 512, 2047])
def test_l2norm(engine_small, n):
    x = f32(np.random.RandomState(n).randn(n) * 5)
    got = run(engine_small, "L2NORM", [n], [], out=x)
    ref = ref_l2norm(x)
    check(got, ref, (sumsq_scale_bound(x[None], 256) + U) * np.abs(ref), "l2norm")
    z = np.zeros(n, _F32)
    assert np.array_equal(run(engine_small, "L2NORM", [n], [], out=z), z)


@gpu
@pytest.mark.parametrize("rows,cols,bias", [(13, 7, True), (512, 1024, True), (31, 45, False), (1, 31, True), (1027, 512, True)])
def test_gemv(engine_small, rows, cols, bias):
    rng = np.random.RandomState(rows + cols)
    W, g = f32(rng.randn(rows, cols)), f32(rng.randn(cols))
    b = f32(rng.randn(rows) * 4) if bias else None
    got = run(engine_small, "GEMV", [rows, cols, int(bias)], [W, g] + ([b] if bias else []), out_len=rows)
    check(got, ref_gemv(W, g, b), gemv_bound(W, g, b), "gemv")


# The front-ends compose fp32 DFT-by-GEMM (1024 or 400 taps) and mel GEMMs with the engine's own tables, so they carry
# accumulated GEMM rounding (under 1e-4 on an H100 for these inputs); 1e-3 absolute on a log / normalised scale is far
# below what a wrong window, reflection or filterbank does (O(0.1) and more).  A DFT basis shifted by whole taps is a
# circular shift of the frame and leaves the power spectrum unchanged, so these ops cannot see one.
MEL_TOL = 1e-3


@gpu
@pytest.mark.parametrize("name", ["small", "full"])
@pytest.mark.parametrize("seconds", [0.33, 1.0, 4.0])
def test_mel22_matches_reference(name, seconds, request):
    eng = request.getfixturevalue(f"engine_{name}")
    dims = request.getfixturevalue(f"dims_{name}")
    core = request.getfixturevalue(f"state_{name}")[1]
    for n in (int(22050 * seconds), int(22050 * seconds) // 256 * 256):      # off and on the hop grid
        wav = O.synthetic_reference_wav(n / 22050 + 1e-6, 22050, 150.0, n % 97).numpy()[:n]
        T = 1 + n // 256
        got = run(eng, "MEL22", [n], [wav], out_len=T * dims.cond.n_mels).reshape(T, dims.cond.n_mels)
        ref = ref_mel22(wav, core["mel_stats"].numpy(), dims.cond.n_mels)
        print("mel22", name, n, "max err", np.abs(got - ref).max())
        check(got, ref, MEL_TOL, f"mel22 n={n}")


@gpu
@pytest.mark.parametrize("name", ["small", "full"])
@pytest.mark.parametrize("n", [400, 16000, 16160, 16001, 168000])
def test_mel16_matches_reference(name, n, request):
    eng = request.getfixturevalue(f"engine_{name}")
    dims = request.getfixturevalue(f"dims_{name}")
    core = request.getfixturevalue(f"state_{name}")[1]
    wav = O.synthetic_reference_wav(n / 16000 + 1e-6, 16000, 150.0, n % 89).numpy()[:n]
    T = 1 + n // 160
    got = run(eng, "MEL16", [n], [wav], out_len=dims.cond.spk_mels * T).reshape(dims.cond.spk_mels, T)
    ref = ref_mel16(wav, core)
    print("mel16", name, n, "max err", np.abs(got - ref).max())
    check(got, ref, MEL_TOL, f"mel16 n={n}")


@gpu
def test_rejections(engine_small):
    from auralis_b200.native import NativeError
    x = np.zeros(100, _F32)
    cases = [
        ("FRAME_WINDOW", [100, 4, 2, 0, 2, 0, 51, 256], [x, np.ones(5)], 51 * 4),     # window length != wlen
        ("FRAME_WINDOW", [100, 4, 2, 0, 2, 0, 51, 64], [x, np.ones(4)], 51 * 4),      # block size not 128 / 256
        ("POWER", [10, 4], [x], 40),                                                   # D is 100, not 10 * 2 * 4
        ("PREEMPHASIS", [100], [x], 99),                                               # out_len
        ("GROUPNORM", [10, 10, 3], [x, x[:10], x[:10]], 100),                          # C % groups
        ("CONV2D", [512, 4, 4, 4, 3, 1, 0, 0, 0], [np.zeros(512 * 16), np.zeros(4 * 512 * 9)], 64),   # 72 KB slice
        ("CONV2D", [1, 4, 4, 4, 2, 1, 0, 0, 0], [np.zeros(16), np.zeros(16)], 64),    # even k
        ("CONV2D", [1, 4, 4, 4, 3, 1, 0, 1, 0], [np.zeros(16), np.zeros(36)], 64),    # has_bias but no bias
        ("GEMV", [10, 10, 0], [x], 10),                                                # missing g
        ("MEL16", [300], [x[:1].repeat(300)], 64 * 2),                                 # shorter than 400
        (19, [1], [], 1),                                                              # unknown op
        (-1, [1], [], 1),
    ]
    for op, dims, ins, n in cases:
        with pytest.raises(NativeError):
            run(engine_small, op, dims, ins, out_len=n)
    got = run(engine_small, "TRANSPOSE", [10, 10], [x], out_len=100)          # the engine still works
    assert np.array_equal(got, x)
