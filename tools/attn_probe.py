"""Decode-step time at the bench's batch (163 rows, ~430 cached tokens) for 1 and 2 row branches ("microbatches") with the
decode-attention grid uncapped or capped ("attn_ctas_per_sm" = CTAs per SM).  ms per decode step = (run to 400 tokens - run
to 300 tokens) / 100, interleaved repeats, minimum reported.  Options are set and never reset: every config of a list names
every option the list varies.
python tools/attn_probe.py [rows] [precision] [key=value ...]"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from auralis_b200 import native
from auralis_b200.config import XTTSDims
from auralis_b200.weights import synth_state

dims = XTTSDims.full()
gs, cs = synth_state(dims, 1234)
g = torch.Generator().manual_seed(500)
cond = torch.randn(32, 1024, generator=g); dv = torch.nn.functional.normalize(torch.randn(512, generator=g), dim=0)
NB = int(sys.argv[1]) if len(sys.argv) > 1 else 163
PREC = int(sys.argv[2]) if len(sys.argv) > 2 else 2
eng = native.NativeEngine(dims, precision=PREC, max_batch=max(NB, 8), max_speakers=2)
eng.load_state(gs, cs); eng.set_speaker(0, cond.numpy(), dv.numpy())
rng = np.random.RandomState(1)
ids = [[0] + rng.randint(2, 6000, size=78).tolist() + [1] for _ in range(NB)]
def jobs(nt):
    return [(i, ids[i], 0, native.Sampling(temperature=0.75, top_p=0.85, top_k=50, max_tokens=nt, seed=1, seq_seed=i, vocode=False, stop_token=4095)) for i in range(NB)]
eng.run_batch(jobs(8), timeout_s=600, want_wav=False)
def measure(**opts):
    for k, v in opts.items(): eng.set_option(k, v)
    eng.run_batch(jobs(12), timeout_s=600, want_wav=False)          # graph capture for this configuration
    t = []
    for nt in (300, 400):
        t0 = time.time(); eng.run_batch(jobs(nt), timeout_s=600, want_wav=False); t.append(time.time() - t0)
    return 1e3 * (t[1] - t[0]) / 100
import json
cfgs = [dict(attn_ctas_per_sm=c, microbatches=mb) for mb in (1, 2) for c in (0, 2, 4, 8)]
if os.environ.get("STEP_CFGS"):          # any list of option dicts, e.g. STEP_CFGS='[{"gemm_bn":0},{"gemm_bn":64}]'
    cfgs = json.loads(os.environ["STEP_CFGS"])
for extra in sys.argv[3:]:
    eng.set_option(extra.split("=")[0], int(extra.split("=")[1]))
measure(**cfgs[0])
res = {}
for rep in range(3):
    for i in (range(len(cfgs)) if rep % 2 == 0 else reversed(range(len(cfgs)))):
        res.setdefault(i, []).append(measure(**cfgs[i]))
for i, c in enumerate(cfgs):
    v = res[i]
    print(" ".join(f"{k}={val}" for k, val in c.items()) + ": " + " ".join(f"{x:6.3f}" for x in v) + f"   min {min(v):6.3f} ms/decode-step", flush=True)
eng.close()
