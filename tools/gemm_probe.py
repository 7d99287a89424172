"""Persistent wide-tile GEMM (gemm_wgmma_wide.cu) across shapes and ring depths.   python tools/gemm_probe.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from auralis_b200 import native
from auralis_b200.config import XTTSDims
eng = native.NativeEngine(XTTSDims.small(), precision=1, max_batch=4, max_speakers=2)
rng = np.random.RandomState(1)
names = {0: "one tile per CTA", 4: "wide, 4-stage ring (default)", 2: "wide, 2-stage ring", 3: "wide, 3-stage ring"}
for (M, N, K) in ((4096, 4096, 1024), (4096, 4096, 4096), (2304, 3072, 1024), (2304, 4096, 1024), (2304, 1024, 4096), (8192, 8192, 1024)):
    A = rng.randn(M, K).astype(np.float32); W = (rng.randn(N, K) * 0.05).astype(np.float32)
    for v in (4, 2, 3, 0):
        eng.set_option("gemm_wide", v)
        _, ms = eng.debug_gemm(1, A, W, None, None, False, iters=20)
        print(f"M={M} N={N} K={K} {names[v]:30s}: {ms * 1e3:7.1f} us  {2.0 * M * N * K / ms / 1e9:7.1f} TFLOP/s", flush=True)
eng.close()
