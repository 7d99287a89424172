"""Writes tests/golden/enhance_reference.npz: the reference's own enhancer module (oracle/ref_enhance.py, librosa and
pyloudnorm restated) on seeded synthetic speaker references.  Inputs are not stored: `case_input` regenerates them.
Outputs are stored as the 16-bit PCM codes the reference writes to its temporary WAV (rint(y * 32767), int16), which is
all a consumer of the enhanced file sees and keeps the file small; `golden_codes` reads them back.

    python tests/golden/make_enhance_golden.py        (needs the reference tree)
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "enhance_reference.npz")

_OFF = dict(trim_silence=False, remove_noise=False, enhance_speech=False, normalize=False)
# name -> (seconds, sample rate, seed, exact-silence span or None, AudioPreprocessingConfig overrides).  No length is a
# multiple of 512 samples.
CASES = {
    "vad": (1.0, 22050, 11, None, {**_OFF, "trim_silence": True}),
    "gate": (1.0, 22050, 11, None, {**_OFF, "remove_noise": True}),
    "clarity": (0.8, 22050, 11, None, {**_OFF, "enhance_speech": True}),
    "loudness": (1.0, 22050, 11, None, {**_OFF, "normalize": True}),
    "all_silence": (1.8, 22050, 11, (0.5, 1.3), {}),
    "all_16k_m23": (1.2, 16000, 11, None, {"sample_rate": 16000, "target_lufs": -23.0}),
}

def case_config(name):
    from oracle.enhance_oracle import EnhanceConfig
    sec, sr, seed, sil, over = CASES[name]
    return EnhanceConfig(**{"sample_rate": sr, **over})


def case_input(name):
    from oracle.enhance_oracle import synthetic_input
    sec, sr, seed, sil, over = CASES[name]
    return synthetic_input(sec, sr, seed, sil)


def codes16(y):
    """The int16 samples a 16-bit PCM write of `y` stores."""
    return np.clip(np.rint(np.asarray(y, np.float64) * 32767.0), -32768, 32767).astype(np.int16)


def golden_codes(name):
    return np.load(OUT)[name]


def main():
    sys.path.insert(0, ROOT)
    from dataclasses import asdict
    from oracle import ref_enhance
    out = {}
    for name in CASES:
        cfg = case_config(name)
        y = ref_enhance.process(case_input(name), **asdict(cfg))
        assert np.isfinite(y).all(), name
        out[name] = codes16(y)
        print(name, y.shape, y.dtype, float(np.abs(y).max()))
    out["cases"] = np.frombuffer(json.dumps(CASES).encode(), np.uint8)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
