"""Beam search cost on the GPU: for N chunks at B beams each (B in {1, 2, 4, 8}) against N * B plain chunks, the wall time
per decode step and the audio-seconds per second, and the beam kernels' own device time per step (torch.profiler over
one run, kernels named beam_* / kv_page_copy_*).  The card's name and power limit are read in the same call.

    python tools/beam_probe.py [N] [max_tokens]
"""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from auralis_b200 import native
from auralis_b200.config import XTTSDims
from auralis_b200.weights import synth_state

N = int(sys.argv[1]) if len(sys.argv) > 1 else 4
MT = int(sys.argv[2]) if len(sys.argv) > 2 else 200
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print(f"card: {card}", flush=True)
dims = XTTSDims.full()
gs, cs = synth_state(dims, 1234)
g = torch.Generator().manual_seed(500)
cond = torch.randn(32, 1024, generator=g)
dv = torch.nn.functional.normalize(torch.randn(512, generator=g), dim=0)
eng = native.NativeEngine(dims, precision=2, max_batch=max(8 * N, 8), max_speakers=2)
eng.load_state(gs, cs)
eng.set_speaker(0, cond.numpy(), dv.numpy())
rng = np.random.RandomState(1)
texts = [[0] + rng.randint(2, 6000, size=60).tolist() + [1] for _ in range(8 * N)]


def jobs(n, nb):
    return [(i, texts[i], 0, native.Sampling(max_tokens=MT, stop_token=-1, seed=1, seq_seed=i, num_beams=nb,
                                             do_sample=False)) for i in range(n)]


def run(n, nb):
    st0 = eng.stats().decode_steps
    t0 = time.time()
    res = eng.run_batch(jobs(n, nb), timeout_s=1200)
    dt = time.time() - t0
    steps = eng.stats().decode_steps - st0
    audio = sum(r.n_samples for r, _, _, _ in res.values()) / 24000.0
    return dt, steps, audio


run(2, 2)                                                    # warm-up: graphs, modules
for nb in (1, 2, 4, 8):
    dt, steps, audio = run(N, nb)
    pdt, psteps, paudio = run(N * nb, 1)
    print(f"B={nb}: {N} beam chunks {1e3 * dt / max(steps, 1):7.2f} ms/step, {audio / dt:7.1f} audio-s/s | "
          f"{N * nb} plain chunks {1e3 * pdt / max(psteps, 1):7.2f} ms/step, {paudio / pdt:7.1f} audio-s/s", flush=True)
    if nb > 1:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            _, steps, _ = run(N, nb)
        us = sum(e.device_time_total for e in prof.key_averages()
                 if "beam_" in e.key or "kv_page_copy" in e.key)
        print(f"      beam kernels {us / max(steps, 1):7.1f} us/step (device time)", flush=True)
eng.close()
