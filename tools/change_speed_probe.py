"""Times xtts_change_speed (TTSOutput.change_speed on the GPU) on 10 / 60 / 600 s inputs at 24 kHz and rates 0.8 and 1.5:
the median wall time of a call, H2D and D2H included (the call ends with a stream synchronise), next to the CPU oracle
(oracle/pvoc_oracle.py) on the same input.  The per-bin phase accumulation runs on only 1025 threads, so its share of the
call is reported separately, from one torch.profiler run per case (CUDA activities).  Prints the card name and power
limit with the numbers.

    python tools/change_speed_probe.py [--reps 5]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _accumulate_share(eng, x, rate):
    """(accumulate kernel ms, all kernels ms, kernel count) of one call, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.change_speed(x, rate)
        torch.cuda.synchronize()
    acc = tot = 0.0
    n = 0
    for ev in prof.events():
        if getattr(ev, "device_type", None) is None or "CUDA" not in str(ev.device_type):
            continue
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        tot += us
        n += 1
        if "pv_accumulate" in ev.name:
            acc += us
    return acc / 1e3, tot / 1e3, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    from auralis_b200 import native
    from auralis_b200.config import XTTSDims
    from oracle import enhance_oracle as E
    from oracle import pvoc_oracle as P
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"card: {q}")
    eng = native.NativeEngine(XTTSDims.small(), device=0, max_batch=1, max_speakers=1)    # no weights needed
    print(f"{'input':>6} {'rate':>5} {'gpu ms':>9} {'accumulate ms':>14} {'share':>6} {'cpu oracle ms':>14}")
    for sec in (10, 60, 600):
        x = E.synthetic_input(sec, 24000, 42)
        for rate in (0.8, 1.5):
            eng.change_speed(x, rate)                            # warm-up: bases, workspaces
            ts = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                eng.change_speed(x, rate)
                ts.append((time.perf_counter() - t0) * 1e3)
            gpu = float(np.median(ts))
            try:
                acc, kern, n = _accumulate_share(eng, x, rate)
                acc_s = f"{acc:14.2f} {acc / gpu:6.1%}" if n else f"{'not captured':>14} {'':>6}"
            except Exception as e:      # noqa: BLE001 — the profiler is optional for the timing itself
                acc_s = f"{'n/a':>14} {'':>6}"
                print(f"  (profiler: {e})")
            t0 = time.perf_counter()
            P.change_speed(x, rate)
            cpu = (time.perf_counter() - t0) * 1e3
            print(f"{sec:>5}s {rate:>5} {gpu:9.2f} {acc_s} {cpu:14.1f}", flush=True)
    eng.close()


if __name__ == "__main__":
    main()
