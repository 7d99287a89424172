"""Per-stage time of the fast-mode vocoder's resblocks: one ResBlock1 (lrelu -> c1(k, d) -> lrelu -> c2(k, 1) -> +x for
d = 1, 3, 5, then the MRF store / accumulate) of each kernel size k = 3, 7, 11 per stage, run as the six conv1d_tc
launches the vocoder issues for it and, where the engine has it (C <= 64), as one fused resblock_tc launch.  Both go
through NativeEngine.debug_resblock_tc on identical inputs under torch.profiler; only the kernel durations of the trace
are counted (conv1d_tc_kernel for the six launches, resblock_tc_kernel for the fused one).  On a build without the fused
kernel the six launches are timed through debug_conv_tc instead.

Workloads: a batch of windows of 96 tokens (450 z-frames each, 8 by default) and one whole 605-token chunk (2634
z-frames).  The stage-s signal is Lz * (8, 64, 128, 256)[s] rows of C = (256, 128, 64, 32)[s] channels.  Also timed:
conv_pre and the four transposed convs, so the resblocks' share of the whole conv family is printed.  Per stage: us of
the three resblocks (best of the repeats), TFLOP/s and GB/s from the algorithmic counts, and the share of the binding
data-sheet floor (989 TFLOP/s fp16 dense, 3.35 TB/s HBM3; H100 SXM at 700 W).  The card name and power limit are printed
with the numbers.

python tools/resblock_probe.py [windows]"""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile

if not torch.cuda.is_available():
    sys.exit("resblock_probe: no CUDA device")
from auralis_b200 import native
from auralis_b200.config import XTTSDims
from auralis_b200.weights import synth_state

PEAK_FLOPS, PEAK_BW = 989e12, 3.35e12
STORE, ACCUM = native.NativeEngine.CONV_STORE, native.NativeEngine.CONV_ACCUM
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card, flush=True)

NW = int(sys.argv[1]) if len(sys.argv) > 1 else 8
REPS = 3
dims = XTTSDims.full()
eng = native.NativeEngine(dims, precision=2, max_batch=8, max_speakers=2)
eng.load_state(*synth_state(dims, 1234))
fused_api = hasattr(eng, "debug_resblock_tc")
rng = np.random.RandomState(0)


def kernel_us(fn, name):
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in p.events() if name in e.name]
    return sum(getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0) for e in ev), len(ev)


def rb_counts(C, K, Lsum):
    """algorithmic FLOPs and HBM bytes of one resblock: six convs; in: atoms + fp32 x, out: fp32 sum (ACCUM: read too)"""
    fl = 6 * 2.0 * C * C * K * Lsum
    six = Lsum * C * (2 + 2 + (2 + 4 + 4 + 2) + (2 + 2) + (2 + 4 + 4 + 2) + (2 + 2) + (2 + 4 + 8)) + 6 * 2.0 * C * C * K
    fused = Lsum * C * (2 + 4 + 8) + 6 * 2.0 * C * C * K
    return fl, six, fused


def fmt(us, fl, by):
    floor = max(fl / PEAK_FLOPS, by / PEAK_BW) * 1e6
    b = "m" if fl / PEAK_FLOPS > by / PEAK_BW else "h"
    return f"{us:10.1f} {fl / us / 1e6:8.1f} {by / us / 1e3:7.0f} {floor:8.1f}{b} {floor / us:6.2f}"


for label, Lz, B in (("%d windows x 450 z-frames" % NW, 450, NW), ("605-token chunk", 2634, 1)):
    print(f"\n== {label}", flush=True)
    print(f"{'stage / path':28s} {'us':>10s} {'TFLOP/s':>8s} {'GB/s':>7s} {'floor us':>9s} {'share':>6s}")
    total_six, total_fused, total_other, st34_six, st34_fused = 0.0, 0.0, 0.0, 0.0, 0.0
    # conv_pre and the transposed convs (the rest of the conv family)
    x = rng.randn(B, 1024, Lz).astype(np.float32)
    w = (0.03 * rng.randn(512, 1024, 7)).astype(np.float32)
    o16 = np.zeros((B, 64, native.atoms_lpad(Lz), 8), np.float32)
    t = min(kernel_us(lambda: eng.debug_conv_tc(x, w, out16=o16), "conv1d_tc_kernel")[0] for _ in range(REPS))
    total_other += t
    print(f"{'conv_pre':28s} {t:10.1f}", flush=True)
    L, C = Lz, 512
    for s, u in enumerate((8, 8, 2, 2)):
        x = rng.randn(B, C, L).astype(np.float32)
        w = (0.03 * rng.randn(C, C // 2, 2 * u)).astype(np.float32)
        o32 = np.zeros((B, C // 2, L * u), np.float32)
        o16 = np.zeros((B, C // 16, native.atoms_lpad(L * u), 8), np.float32)
        t = min(kernel_us(lambda: eng.debug_conv_tc(x, w, up=u, out32=o32, out16=o16), "conv1d_tc_kernel")[0]
                for _ in range(REPS))
        total_other += t
        print(f"{'up%d' % s:28s} {t:10.1f}", flush=True)
        L, C = L * u, C // 2
        Lsum = float(B * L)
        six_us, fused_us, fl_s, by6_s, byf_s = 0.0, 0.0, 0.0, 0.0, 0.0
        has_fused = fused_api and C <= 64
        for K in (3, 7, 11):
            x = rng.randn(B, C, L).astype(np.float32)
            ws = [(0.03 * rng.randn(C, C, K)).astype(np.float32) for _ in range(6)]
            bs = [(0.1 * rng.randn(C)).astype(np.float32) for _ in range(6)]
            zs = rng.randn(B, C, L).astype(np.float32)
            if fused_api:
                res = {0: [], 1: []}
                for rep in range(REPS):
                    for f in ((0, 1) if has_fused else (0,)):
                        name = "resblock_tc_kernel" if f else "conv1d_tc_kernel"
                        call = lambda: eng.debug_resblock_tc(x, ws, bs, zs=zs, mode=ACCUM, fused=bool(f))
                        res[f].append(kernel_us(call, name)[0])
                six_us += min(res[0])
                if has_fused:
                    fused_us += min(res[1])
            else:
                # parent build: the six launches one by one (c1 atoms only; c2 residual, fp32 + atoms; last c2 ACCUM)
                xa = np.zeros((B, C // 8, native.atoms_lpad(L), 8), np.float32)
                r32 = np.zeros((B, C, L), np.float32)
                best = None
                for rep in range(REPS):
                    tt = 0.0
                    for d, last in ((1, False), (3, False), (5, True)):
                        tt += kernel_us(lambda: eng.debug_conv_tc(x, ws[0], dil=d, out16=xa), "conv1d_tc_kernel")[0]
                        if last:
                            tt += kernel_us(lambda: eng.debug_conv_tc(x, ws[1], resid=x, mode=ACCUM, out32=zs),
                                            "conv1d_tc_kernel")[0]
                        else:
                            tt += kernel_us(lambda: eng.debug_conv_tc(x, ws[1], resid=x, out32=r32, out16=xa),
                                            "conv1d_tc_kernel")[0]
                    best = tt if best is None else min(best, tt)
                six_us += best
            fl, b6, bf = rb_counts(C, K, Lsum)
            fl_s += fl; by6_s += b6; byf_s += bf
        total_six += six_us
        total_fused += fused_us if has_fused else six_us
        if C <= 64:
            st34_six += six_us
            st34_fused += fused_us if has_fused else six_us
        print(f"{'s%d C=%d resblocks, six' % (s + 1, C):28s} {fmt(six_us, fl_s, by6_s)}", flush=True)
        if has_fused:
            print(f"{'s%d C=%d resblocks, fused' % (s + 1, C):28s} {fmt(fused_us, fl_s, byf_s)}", flush=True)
    fam_six = total_six + total_other
    print(f"conv family (3 resblocks per stage, one of each k), six-launch path: {fam_six:.1f} us; "
          f"stages 3 + 4: {st34_six:.1f} us = {100 * st34_six / fam_six:.1f} %")
    if fused_api:
        fam_f = total_fused + total_other
        print(f"with the fused stages 3 + 4: {fam_f:.1f} us (stages 3 + 4: {st34_fused:.1f} us), "
              f"{fam_six / fam_f:.2f}x the six-launch family")
print("\ncard:", card)
eng.close()
