"""8 full-length chunks through the engine so that the vocoder runs exactly as in the bench (batch of 8 x 605 latents).
    python tools/profile_vocoder_batch.py [tokens]   (run under a profiler, e.g. torch.profiler or a CUDA-event wrapper)
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from auralis_b200 import native
from auralis_b200.config import XTTSDims
from auralis_b200.weights import synth_state
dims = XTTSDims.full()
gs, cs = synth_state(dims, 1234)
g = torch.Generator().manual_seed(500)
cond = torch.randn(32, 1024, generator=g); dv = torch.nn.functional.normalize(torch.randn(512, generator=g), dim=0)
eng = native.NativeEngine(dims, precision=1, max_batch=8, max_speakers=2)
eng.load_state(gs, cs); eng.set_speaker(0, cond.numpy(), dv.numpy())
rng = np.random.RandomState(1)
nt = int(sys.argv[1]) if len(sys.argv) > 1 else 605
jobs = [(i, [0] + rng.randint(2, 6000, size=78).tolist() + [1], 0,
         native.Sampling(temperature=0.75, top_p=0.85, top_k=50, max_tokens=nt, seed=1, seq_seed=i, vocode=True, stop_token=-1)) for i in range(8)]
res = eng.run_batch(jobs, timeout_s=600, want_wav=False)
print("done", sum(r.n_samples for (r, _, _, _) in res.values()))
