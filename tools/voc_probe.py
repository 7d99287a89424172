"""Vocoder timing: 16 full-length chunks finish together (batch submit) -> batched vocoder passes; engine vocoder_ms and
the tensor-core conv family's profile.   python tools/voc_probe.py [tokens]"""
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
eng = native.NativeEngine(dims, precision=1, max_batch=16, max_speakers=2)
eng.load_state(gs, cs); eng.set_speaker(0, cond.numpy(), dv.numpy())
rng = np.random.RandomState(1)
nt = int(sys.argv[1]) if len(sys.argv) > 1 else 605
NB = 16
def jobs():
    return [(i, [0] + rng.randint(2, 6000, size=78).tolist() + [1], 0,
             native.Sampling(temperature=0.75, top_p=0.85, top_k=50, max_tokens=nt, seed=1, seq_seed=i, vocode=True, stop_token=-1)) for i in range(NB)]
eng.set_option("d2h_wav", 0)
eng.run_batch(jobs(), timeout_s=600, want_wav=False)
for rep in range(2):
    eng.set_option("reset_stats", 0)
    res = eng.run_batch(jobs(), timeout_s=600, want_wav=False)
    st = eng.stats()
    audio = sum(r.n_samples for (r, _, _, _) in res.values()) / 24000.0
    print(f"run {rep}: vocoder {st.vocoder_ms:8.2f} ms for {NB} chunks ({st.vocoder_ms / NB:.3f} ms/chunk, {audio / (st.vocoder_ms / 1e3):.0f} audio-s/s vocoder-only); gpt {st.gpt_ms:.0f} ms", flush=True)
eng.set_option("profile", 1)
eng.run_batch(jobs(), timeout_s=600, want_wav=False)
prof = eng.kernel_profile(); eng.set_option("profile", 0)
v = prof.get("conv1d_tc_f16_wgmma")
print(f"  profile: conv1d_tc {v['ms']:.2f} ms, {v['launches']} launches, {v['flops'] / v['ms'] / 1e9:.1f} TFLOP/s, {v['bytes'] / v['ms'] / 1e6:.0f} GB/s")
