"""Per-shape time of the fast-mode vocoder convolution (conv1d_tc_kernel) with the direct (tc_epilogue = 0) and the
staged (tc_epilogue = 1) epilogue, alternating A/B/A/B.  Every production shape of the full geometry is launched through
NativeEngine.debug_conv_tc under torch.profiler; only the conv1d_tc_kernel durations of the trace are counted.

Workloads: a batch of windows of 96 tokens (~450 z-frames each, margins included; 8 by default, as filling the host
arrays of 32 takes minutes) and one whole 605-token chunk (2634 z-frames).  The windows are of equal length here, so the
launch is a plain batch.  Per shape: us per launch (best of the repeats), TFLOP/s and GB/s from the algorithmic counts
launch_conv1d_tc / launch_convT_tc use, and the share of the binding data-sheet floor (989 TFLOP/s fp16 dense,
3.35 TB/s HBM3; H100 SXM at 700 W).  The card name and power limit are printed with the numbers.

python tools/conv_tc_probe.py [windows]"""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile

if not torch.cuda.is_available():
    sys.exit("conv_tc_probe: no CUDA device")
from auralis_b200 import native
from auralis_b200.config import XTTSDims
from auralis_b200.weights import synth_state

PEAK_FLOPS, PEAK_BW = 989e12, 3.35e12
STORE, ACCUM = native.NativeEngine.CONV_STORE, native.NativeEngine.CONV_ACCUM
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card, flush=True)

NW = int(sys.argv[1]) if len(sys.argv) > 1 else 8
dims = XTTSDims.full()
eng = native.NativeEngine(dims, precision=2, max_batch=8, max_speakers=2)
eng.load_state(*synth_state(dims, 1234))
rng = np.random.RandomState(0)


def shapes(Lz):
    """(name, kwargs of debug_conv_tc minus x, Cin, Cout, K, L_in) of the production launches at Lz z-frames"""
    out = [("conv_pre", dict(resid=False, want32=False), 1024, 512, 7, 1, Lz)]
    L, C = Lz, 512
    for s, u in enumerate((8, 8, 2, 2)):
        out.append((f"up{s}", dict(up=u), C, C // 2, 2 * u, 1, L))
        L, C = L * u, C // 2
        for K, d in ((3, 1), (7, 3), (11, 5)):
            out.append((f"s{s + 1} c1 K{K} d{d}", dict(resid=False, want32=False), C, C, K, d, L))
        out.append((f"s{s + 1} c2 K11", dict(), C, C, 11, 1, L))
        out.append((f"s{s + 1} last-c2 STORE", dict(mode=STORE), C, C, 11, 1, L))
        out.append((f"s{s + 1} last-c2 ACCUM", dict(mode=ACCUM, want16=True, scale16=1 / 3), C, C, 11, 1, L))
    return out


def counts(Cin, Cout, K, up, Lsum, resid, want32, want16, mode):
    if up:
        return 4.0 * Cin * Cout * Lsum * up, Lsum * 2.0 * Cin + Lsum * up * Cout * 6.0 + 4.0 * Cin * Cout * up
    by = Lsum * (2.0 * Cin + (4.0 * Cout if resid else 0) + ((8.0 if mode == ACCUM else 4.0) * Cout if want32 else 0) +
                 (2.0 * Cout if want16 else 0)) + 2.0 * Cin * Cout * K
    return 2.0 * Cin * Cout * K * Lsum, by


def kernel_us(fn):
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in p.events() if "conv1d_tc_kernel" in e.name]
    t = sum(getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0) for e in ev)
    return t, len(ev)


for label, Lz, lens in (("%d windows x 450 z-frames" % NW, 450, [450] * NW), ("605-token chunk", 2634, [2634])):
    print(f"\n== {label}", flush=True)
    print(f"{'shape':24s} {'direct us':>10s} {'staged us':>10s} {'TFLOP/s':>8s} {'GB/s':>7s} {'floor':>6s} "
          f"{'share d':>7s} {'share s':>7s}")
    for name, kw, Cin, Cout, K, dil, L in shapes(Lz):
        up = kw.get("up", 0)
        resid, want32, want16 = kw.get("resid", True) and not up, kw.get("want32", True), kw.get("want16", True)
        mode, scale16 = kw.get("mode", STORE), kw.get("scale16", 1.0)
        B = len(lens)
        Lout = L * up if up else L
        if B * Cout * Lout * 4 > 6e9:          # keep the host arrays reasonable for stage 4 at 32 windows
            continue
        x = rng.randn(B, Cin, L).astype(np.float32)
        w = (0.03 * rng.randn(Cin, Cout, 2 * up) if up else 0.03 * rng.randn(Cout, Cin, K)).astype(np.float32)
        r = rng.randn(B, Cout, Lout).astype(np.float32) if resid else None
        o32 = rng.randn(B, Cout, Lout).astype(np.float32) if want32 else None
        o16 = np.zeros((B, Cout // 8, native.atoms_lpad(Lout), 8), np.float32) if want16 else None
        call = lambda: eng.debug_conv_tc(x, w, up=up, dil=dil, resid=r, mode=mode, scale16=scale16,
                                         out32=o32, out16=o16)
        call()                                 # warm-up of both paths
        res = {0: [], 1: []}
        for rep in range(4):
            e = rep % 2
            eng.set_option("tc_epilogue", e)
            t, n = kernel_us(call)
            res[e].append(t / max(n, 1))
        eng.set_option("tc_epilogue", 1)
        fl, by = counts(Cin, Cout, K, up, float(B * L), resid, want32, want16, mode)
        floor_us = max(fl / PEAK_FLOPS, by / PEAK_BW) * 1e6
        bound = "hbm" if by / PEAK_BW > fl / PEAK_FLOPS else "mma"
        d, s = min(res[0]), min(res[1])
        print(f"{name:24s} {d:10.1f} {s:10.1f} {fl / s / 1e6:8.1f} {by / s / 1e3:7.0f} {floor_us:5.1f}{bound[0]} "
              f"{floor_us / d:7.2f} {floor_us / s:7.2f}", flush=True)
print("\ncard:", card)
eng.close()
