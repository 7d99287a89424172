"""Small driver for ncu: full-size engine, a handful of chunks, every kernel family launched at its real shapes.
    ncu --set full -k regex:<name> -c N -o gpurun_out/prof python tools/profile_kernels.py [n_chunks] [tokens]
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from auralis_b200 import native
from auralis_b200.config import XTTSDims
from auralis_b200.weights import synth_state

nb = int(sys.argv[1]) if len(sys.argv) > 1 else 32
nt = int(sys.argv[2]) if len(sys.argv) > 2 else 24
voc_T = int(sys.argv[3]) if len(sys.argv) > 3 else 605
dims = XTTSDims.full()
gs, cs = synth_state(dims, 1234)
g = torch.Generator().manual_seed(500)
cond = torch.randn(32, 1024, generator=g); dv = torch.nn.functional.normalize(torch.randn(512, generator=g), dim=0)
eng = native.NativeEngine(dims, precision=1, max_batch=max(nb, 8), max_speakers=2)
eng.load_state(gs, cs); eng.set_speaker(0, cond.numpy(), dv.numpy())
eng.set_option("cuda_graphs", 0)
for kv in os.environ.get("XTTS_OPTS", "").split(","):      # e.g. XTTS_OPTS=attn_ctas_per_sm=4,microbatches=1
    if "=" in kv: eng.set_option(kv.split("=")[0], int(kv.split("=")[1]))
          # ncu attributes kernels per launch either way; eager keeps names simple
rng = np.random.RandomState(1)
jobs = [(i, [0] + rng.randint(2, 6000, size=78).tolist() + [1], 0,
         native.Sampling(temperature=0.75, top_p=0.85, top_k=50, max_tokens=nt, seed=1, seq_seed=i, vocode=False, stop_token=4095)) for i in range(nb)]
eng.run_batch(jobs, timeout_s=600, want_wav=False)
lat = rng.randn(voc_T, 1024).astype(np.float32)
eng.vocode(lat, 0)
print("done")
