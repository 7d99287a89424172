"""Writes resample_reference.npz: torchaudio.functional.resample (CPU, torchaudio 2.x, default arguments) of the seeded
signals `oracle.resample_oracle.golden_cases()` lists, so the GPU tests can compare against torchaudio where it is not
installed.  torchaudio cannot resample an empty waveform (it raises); length-0 cases store the empty result the
contract specifies.  Run from the repository root: `python tests/golden/make_resample_golden.py`."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    import torch
    import torchaudio
    from oracle import resample_oracle as R
    out = {}
    meta = []
    for i, (o, nw, n, kind, seed) in enumerate(R.golden_cases()):
        x = R.signal(kind, n, o, nw, seed)
        if n == 0:
            y = np.zeros(0, np.float32)
        else:
            y = torchaudio.functional.resample(torch.from_numpy(x), o, nw).numpy()
        assert y.dtype == np.float32 and y.shape == (R.out_len(n, o, nw),)
        out[f"y{i}"] = y
        meta.append((o, nw, n, R.KINDS.index(kind), seed))
    out["meta"] = np.asarray(meta, np.int64)
    out["torchaudio"] = np.asarray(torchaudio.__version__)
    path = os.path.join(ROOT, "tests", "golden", "resample_reference.npz")
    np.savez_compressed(path, **out)
    print(f"{len(meta)} cases -> {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
