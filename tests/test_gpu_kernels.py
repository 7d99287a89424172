"""GPU: single-kernel parity through the C ABI — GEMMs (fp32 CUDA-core and bf16 wgmma) and the fused sampler."""
import numpy as np
import pytest
import torch

from auralis_b200.native import Sampling
from oracle import xtts_oracle as O
from test_gpu_decode_kernels import rnd
from test_gpu_gpt_kernels import gemm_products, ref_gemm16
from test_gpu_sampler import reference

pytestmark = pytest.mark.gpu


def _ref_gemm(A, W, bias, resid, gelu):
    y = A.astype(np.float64) @ W.astype(np.float64).T
    if bias is not None:
        y = y + bias
    if gelu:
        y = 0.5 * y * (1.0 + np.tanh(np.sqrt(2.0 / np.pi) * (y + 0.044715 * y ** 3)))
    if resid is not None:
        y = y + resid
    return y


@pytest.mark.parametrize("M,N,K", [(1, 384, 128), (7, 128, 512), (150, 3072, 1024), (300, 1024, 4096), (33, 1026, 1024),
                                   (5, 96, 80), (9, 64, 2730)])
def test_gemm_f32(engine_small, M, N, K):
    rng = np.random.RandomState(M * 7 + N)
    A = rng.randn(M, K).astype(np.float32)
    W = (rng.randn(N, K) * 0.05).astype(np.float32)
    b = rng.randn(N).astype(np.float32)
    r = rng.randn(M, N).astype(np.float32)
    for gelu, resid in ((False, None), (True, None), (False, r)):
        out, _ = engine_small.debug_gemm(0, A, W, b, resid, gelu)
        ref = _ref_gemm(A, W, b, resid, gelu)
        err = np.abs(out - ref).max()
        assert err < 2e-4 * max(1.0, np.abs(ref).max()), (M, N, K, gelu, resid is not None, err)


def _bf16(x):
    return torch.from_numpy(x).to(torch.bfloat16).to(torch.float32).numpy()


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (1, 384, 128), (7, 128, 512), (150, 3072, 1024), (300, 1024, 4096),
                                   (33, 1056, 1024), (257, 4096, 1024), (256, 256, 64), (1000, 3072, 1024), (513, 288, 192),
                                   (2304, 1056, 1024)])
@pytest.mark.parametrize("mode", [1, 2], ids=["bf16", "fp16"])
def test_gemm_bf16_tcgen05(engine_small, mode, M, N, K):
    """Tensor-core path (bf16 and IEEE fp16 operands) vs an fp64 product of the rounded operands, element by element under
    the bound of test_gpu_gpt_kernels.ref_gemm16 (isolates layout/descriptor bugs from rounding).  M >= 256 and N >= 256
    shapes run on the persistent wide-tile kernel: full and ragged 128 x 256 tiles, more tiles than CTAs (the stage ring
    wraps across tiles), N tails that are not a multiple of 256."""
    rng = np.random.RandomState(M * 13 + N)
    A = rng.randn(M, K).astype(np.float32)
    W = (rng.randn(N, K) * 0.05).astype(np.float32)
    b = rng.randn(N).astype(np.float32)
    r = rng.randn(M, N).astype(np.float32)
    A16, W16 = rnd(A, mode)[1], rnd(W, mode)[1]
    prod = gemm_products(A16, W16)
    worst = 0.0
    for gelu, resid in ((False, None), (True, None), (False, r)):
        out, _ = engine_small.debug_gemm(mode, A, W, b, resid, gelu)
        ref, tol = ref_gemm16(A16, W16, b, resid, gelu, 0, prod)
        assert np.isfinite(out).all()
        err = np.abs(out - ref)
        bad = np.argwhere(err > tol)
        assert bad.size == 0, (mode, M, N, K, gelu, resid is not None, bad[:5].tolist(), float((err / tol).max()))
        worst = max(worst, float((err / tol).max()))
    print(f"tensor-core GEMM mode={mode} M={M} N={N} K={K}: largest share of the error bound used {worst:.3g}")


def _f16(x):
    return x.astype(np.float16).astype(np.float32)


@pytest.mark.parametrize("mode", [1, 2], ids=["bf16", "fp16"])
@pytest.mark.parametrize("depth", [2, 3, 4])
def test_gemm_wide_ring_depths(engine_small, depth, mode):
    """Engine option "gemm_wide" = ring depth (2, 3 or 4 stages) of the persistent wide-tile kernel, with bf16 and IEEE fp16
    operands (the two wgmma instruction types).  Every depth, on ragged tiles with more tiles than CTAs, must give the default
    depth's result bit for bit (same MMA order per output element)."""
    rnd = _bf16 if mode == 1 else _f16
    for (M, N, K) in ((1000, 3072, 1024), (513, 288, 192), (2304, 1056, 1024)):
        rng = np.random.RandomState(M + N)
        A = rng.randn(M, K).astype(np.float32)
        W = (rng.randn(N, K) * 0.05).astype(np.float32)
        b = rng.randn(N).astype(np.float32)
        r = rng.randn(M, N).astype(np.float32)
        try:
            engine_small.set_option("gemm_wide", depth)
            got, _ = engine_small.debug_gemm(mode, A, W, b, r, True)
        finally:
            engine_small.set_option("gemm_wide", 4)
        ref = _ref_gemm(rnd(A), rnd(W), b, r, True)
        assert np.isfinite(got).all()
        assert np.abs(got - ref).max() < 2e-3 * max(1.0, np.abs(ref).max()), (depth, mode, M, N, K)
        base, _ = engine_small.debug_gemm(mode, A, W, b, r, True)
        np.testing.assert_array_equal(got, base)


def test_gemm_tcgen05_speed_report(engine_small):
    """Not a pass/fail perf gate: prints achieved TFLOP/s of both GEMM paths at a prefill-like and a decode-like shape."""
    for (M, N, K) in ((4096, 4096, 1024), (160, 3072, 1024)):
        rng = np.random.RandomState(1)
        A = rng.randn(M, K).astype(np.float32)
        W = (rng.randn(N, K) * 0.05).astype(np.float32)
        for mode in (0, 1):
            _, ms = engine_small.debug_gemm(mode, A, W, None, None, False, iters=20)
            print(f"gemm mode={mode} M={M} N={N} K={K}: {ms * 1e3:.1f} us  {2.0 * M * N * K / ms / 1e9:.2f} TFLOP/s")
        if M >= 256:
            engine_small.set_option("gemm_wide", 0)
            _, ms = engine_small.debug_gemm(1, A, W, None, None, False, iters=20)
            engine_small.set_option("gemm_wide", 4)
            print(f"gemm one-tile-per-CTA kernel M={M} N={N} K={K}: {ms * 1e3:.1f} us  {2.0 * M * N * K / ms / 1e9:.2f} TFLOP/s")


def _oracle_tokens(logits, seen, sp, step):
    osp = O.SamplingParams(temperature=sp.temperature, top_p=sp.top_p, top_k=sp.top_k,
                           repetition_penalty=sp.repetition_penalty, seed=sp.seed)
    out = []
    for b in range(logits.shape[0]):
        s = set(np.nonzero(seen[b])[0].tolist())
        out.append(O.sample_token(torch.from_numpy(logits[b].copy()), s, osp, sp.seq_seed + b, step))
    return np.array(out)


def _exact_tokens(logits, seen, sp, step):
    B = logits.shape[0]
    return reference(logits, seen, [sp.temperature] * B, [sp.top_k] * B, [sp.top_p] * B, [sp.repetition_penalty] * B,
                     [sp.seed] * B, sp.seq_seed + np.arange(B), [step] * B)


def test_sampler_greedy_with_penalty(engine_small, dims_small):
    V = dims_small.gpt.n_audio_tokens
    rng = np.random.RandomState(3)
    logits = rng.randn(8, V).astype(np.float32)
    seen = (rng.rand(8, V) < 0.3).astype(np.uint8)
    sp = Sampling(temperature=0.0, repetition_penalty=5.0, stop_token=dims_small.gpt.stop_audio_token)
    got = engine_small.debug_sample(logits, seen, sp, step=4)
    np.testing.assert_array_equal(got, _oracle_tokens(logits, seen, sp, 4))


@pytest.mark.parametrize("top_k,quantised", [(50, False), (0, False), (100, False), (50, True)])
def test_sampler_topk_topp_seeded(engine_small, dims_small, top_k, quantised):
    """Same Philox stream, same kept set -> the same token as the exact reference on every decisive row (one whose
    top-p compares and winning ratio clear the kernel's fp32 error bound, tests/test_gpu_sampler.py).
    top_k=50 takes the radix-select fast path; 0 / 100 and the heavily tied (quantised) logits take the full sort."""
    V = dims_small.gpt.n_audio_tokens
    rng = np.random.RandomState(5)
    decisive = total = 0
    for step in range(6):
        logits = (rng.randn(8, V) * 2.0).astype(np.float32)
        if quantised:
            logits = np.round(logits)                # many exact ties at the k-th value
        seen = (rng.rand(8, V) < 0.1).astype(np.uint8)
        sp = Sampling(temperature=0.75, top_p=0.85, top_k=top_k, repetition_penalty=5.0, seed=1234 + step, seq_seed=7,
                      stop_token=dims_small.gpt.stop_audio_token)
        got = engine_small.debug_sample(logits, seen, sp, step=step)
        ref = _exact_tokens(logits, seen, sp, step)
        d = ref.decisive
        np.testing.assert_array_equal(got[d], ref.token[d])
        np.testing.assert_array_equal(ref.token[d], _oracle_tokens(logits, seen, sp, step)[d])
        decisive += int(d.sum()); total += got.size
    assert decisive >= 0.9 * total, (decisive, total)


def test_sampler_distribution(engine_small, dims_small):
    V = dims_small.gpt.n_audio_tokens
    p = np.full(V, 1e-9); p[:4] = [0.5, 0.25, 0.15, 0.1]
    logits = np.tile(np.log(p / p.sum()).astype(np.float32), (8, 1))
    counts = np.zeros(V)
    for i in range(100):
        sp = Sampling(temperature=1.0, top_p=1.0, top_k=0, repetition_penalty=1.0, seed=i, seq_seed=0,
                      stop_token=dims_small.gpt.stop_audio_token)
        for t in engine_small.debug_sample(logits, None, sp, step=i):
            counts[t] += 1
    f = counts[:4] / counts.sum()
    assert np.abs(f - [0.5, 0.25, 0.15, 0.1]).max() < 0.06, f
