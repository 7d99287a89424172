"""Writes tests/golden/change_speed_reference.npz: the reference's own `TTSOutput.change_speed`
(oracle/ref_change_speed.py, librosa restated) on seeded speech-like inputs at 24 kHz and 22.05 kHz.  Inputs are not
stored: `case_input` regenerates them.  Outputs are stored as the float32 arrays the reference returns.

    python tests/golden/make_change_speed_golden.py        (needs the reference tree)
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "change_speed_reference.npz")

# name -> (seconds, sample rate, seed, exact-silence span or None, speed factor).  No length is a multiple of 512.
CASES = {
    "24k_r0.5": (0.4, 24000, 61, None, 0.5),
    "24k_r0.8": (0.5, 24000, 62, None, 0.8),
    "24k_r1.1_silence": (0.6, 24000, 63, (0.2, 0.35), 1.1),
    "22k_r1.5": (0.7, 22050, 64, None, 1.5),
    "22k_r2.0_silence": (0.8, 22050, 65, (0.1, 0.3), 2.0),
}


def case_input(name):
    from oracle.enhance_oracle import synthetic_input
    sec, sr, seed, sil, rate = CASES[name]
    return synthetic_input(sec, sr, seed, sil)


def golden(name):
    return np.load(OUT)[name]


def reference_outputs():
    """name -> the reference's TTSOutput for each case (the reference tree must be mounted)."""
    from oracle import ref_change_speed
    out = {}
    for name, (sec, sr, seed, sil, rate) in CASES.items():
        out[name] = ref_change_speed.change_speed(case_input(name), rate, sample_rate=sr)
    return out


def main():
    sys.path.insert(0, ROOT)
    out = {}
    for name, o in reference_outputs().items():
        y = np.asarray(o.array)
        assert y.dtype == np.float32 and np.isfinite(y).all(), name
        out[name] = y
        print(name, y.shape, float(np.abs(y).max()))
    out["cases"] = np.frombuffer(json.dumps(CASES).encode(), np.uint8)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
