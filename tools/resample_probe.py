"""Times xtts_resample (speaker references, conditioning and TTSOutput.resample on the GPU) for a 60 s speaker reference
(44.1 kHz -> 22.05 kHz, 22.05 kHz -> 16 kHz) and a 1 h book at 24 kHz (-> 44.1 / 48 / 16 kHz):
* the median wall time of a call, host -> device and device -> host copies included (the call ends with a stream
  synchronise);
* the kernel time of one call from torch.profiler (CUDA activities, a run of its own), and the bytes the kernels must
  move (input span read once, output written once, as float32) over that time against the H100 SXM's 3.35 TB/s;
* torchaudio's CPU time on the same host (torch's default thread count), or "not measured" without torchaudio.
Prints the card name and power limit with the numbers.

    python tools/resample_probe.py [--reps 5]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35
CASES = [("60 s reference", 60, 44100, 22050), ("60 s reference", 60, 22050, 16000),
         ("1 h book", 3600, 24000, 44100), ("1 h book", 3600, 24000, 48000), ("1 h book", 3600, 24000, 16000)]


def _kernel_ms(eng, x, o, nw):
    """(resample kernel ms, all kernels ms) of one call, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.resample(x, o, nw)
        torch.cuda.synchronize()
    rs = tot = 0.0
    for ev in prof.events():
        if getattr(ev, "device_type", None) is None or "CUDA" not in str(ev.device_type):
            continue
        if "memcpy" in ev.name.lower() or "memset" in ev.name.lower():
            continue
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        tot += us
        if "rs_resample" in ev.name:
            rs += us
    return rs / 1e3, tot / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    from auralis_b200 import native
    from auralis_b200.config import XTTSDims
    from oracle import resample_oracle as R
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"card: {q}")
    try:
        import torch
        import torchaudio
        print(f"torchaudio {torchaudio.__version__}, {torch.get_num_threads()} torch threads")
    except ImportError:
        torchaudio = None
    eng = native.NativeEngine(XTTSDims.small(), device=0, max_batch=1, max_speakers=1)    # no weights needed
    print(f"{'case':>15} {'rates':>13} {'call ms':>9} {'kernel ms':>10} {'kern GB/s':>10} {'of HBM':>7} "
          f"{'all kernels ms':>15} {'torchaudio cpu ms':>18}")
    for name, sec, o, nw in CASES:
        x = R.signal("noise", sec * o, o, nw, 1)
        eng.resample(x, o, nw)                                  # warm-up: band table, workspaces
        ts = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            y = eng.resample(x, o, nw)
            ts.append((time.perf_counter() - t0) * 1e3)
        call = float(np.median(ts))
        try:
            kern, allk = _kernel_ms(eng, x, o, nw)
        except Exception as e:      # noqa: BLE001 — the profiler is optional for the wall-clock numbers
            kern = allk = float("nan")
            print(f"  (profiler: {e})")
        nbytes = 4 * (x.size + y.size)
        gbs = nbytes / (kern * 1e-3) / 1e9 if kern > 0 else float("nan")
        cpu = "not measured"
        if torchaudio is not None:
            xt = torch.from_numpy(x)
            torchaudio.functional.resample(xt, o, nw)
            cs = []
            for _ in range(max(1, args.reps // 2)):
                t0 = time.perf_counter()
                torchaudio.functional.resample(xt, o, nw)
                cs.append((time.perf_counter() - t0) * 1e3)
            cpu = f"{float(np.median(cs)):.1f}"
        print(f"{name:>15} {o:>6}->{nw:<6} {call:9.2f} {kern:10.3f} {gbs:10.1f} {gbs / (HBM_TBS * 1e3):7.1%} "
              f"{allk:15.3f} {cpu:>18}", flush=True)
    eng.close()


if __name__ == "__main__":
    main()
