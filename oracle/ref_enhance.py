"""TEST INFRASTRUCTURE — loads the reference's own enhancer module (`common/definitions/enhancer.py`), unmodified, as a
fresh module object, with librosa and pyloudnorm bound to the restatements in ``oracle/enhance_oracle.py`` and the real
torchaudio.  This pins the reference's glue (stage order, thresholds, the fftfreq gain, nan_to_num, tanh) while the two
third-party libraries stay restated.  Only usable where the reference tree is mounted; never on the GPU box.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

from . import enhance_oracle as E
from . import ref_import

_mod = None


def load():
    """-> the reference enhancer module (AudioPreprocessingConfig, EnhancedAudioProcessor)."""
    global _mod
    if _mod is not None:
        return _mod
    if not ref_import.available():
        raise RuntimeError("reference tree not mounted")
    path = os.path.join(ref_import.REF_SRC, "auralis", "common", "definitions", "enhancer.py")
    lib = types.ModuleType("librosa")
    lib.__dict__.update(vars(E.librosa))
    pln = types.ModuleType("pyloudnorm")
    pln.Meter = E.Meter
    saved = {k: sys.modules.get(k) for k in ("librosa", "pyloudnorm")}
    sys.modules["librosa"], sys.modules["pyloudnorm"] = lib, pln
    try:
        spec = importlib.util.spec_from_file_location("_auralis_ref_enhancer", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    _mod = mod
    return mod


def process(audio, **cfg):
    """The reference's EnhancedAudioProcessor(AudioPreprocessingConfig(**cfg)).process(audio)."""
    m = load()
    return m.EnhancedAudioProcessor(m.AudioPreprocessingConfig(**cfg)).process(audio)
