"""Times xtts_enhance per stage (each stage alone, then all four) on 10 / 30 / 60 s inputs at 22.05 kHz with CUDA events
on the engine stream, next to the CPU oracle (oracle/enhance_oracle.py) on the same input.  Prints the card name and
power limit with the numbers.

    python tools/enhance_probe.py [--reps 5]
"""
import argparse
import os
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    warnings.simplefilter("ignore", RuntimeWarning)
    from auralis_b200 import native
    from auralis_b200.config import XTTSDims
    from oracle import enhance_oracle as E
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"card: {q}")
    eng = native.NativeEngine(XTTSDims.small(), device=0, max_batch=1, max_speakers=1)    # no weights needed
    off = dict(trim_silence=False, remove_noise=False, enhance_speech=False, normalize=False)
    stages = {"vad": {**off, "trim_silence": True}, "gate": {**off, "remove_noise": True},
              "clarity": {**off, "enhance_speech": True}, "loudness": {**off, "normalize": True}, "all": {}}
    E.enhance(E.synthetic_input(1.0, 22050, 1), E.EnhanceConfig())      # oracle warm-up: torch / scipy imports
    print(f"{'input':>6} {'stage':>8} {'gpu ms':>9} {'cpu oracle ms':>14}")
    for sec in (10, 30, 60):
        x = E.synthetic_input(sec, 22050, 42)
        for name, over in stages.items():
            cfg = E.EnhanceConfig(**over)
            eng.enhance(x, cfg)                                  # warm-up: bases, filterbank, workspaces
            ts = []
            for _ in range(args.reps):
                eng.timer_start()
                eng.enhance(x, cfg)
                ts.append(eng.timer_stop_ms())
            t0 = time.perf_counter()
            E.enhance(x, cfg)
            cpu = (time.perf_counter() - t0) * 1e3
            print(f"{sec:>5}s {name:>8} {np.median(ts):9.2f} {cpu:14.1f}")
    eng.close()


if __name__ == "__main__":
    main()
