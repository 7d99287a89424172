"""TEST INFRASTRUCTURE — runs the reference's own `TTSOutput.change_speed` (`common/definitions/output.py`), unmodified,
with ``librosa`` bound to the restatement in ``oracle/pvoc_oracle.py`` for the duration of the call.  `change_speed`
imports librosa inside the method, so the module is in ``sys.modules`` only while it runs.  This pins the reference's
glue (n_fft, hop, the normalisation, the ``== 1`` shortcut, the ``<= 0`` error, the returned fields) while librosa stays
restated.  Only usable where the reference tree is mounted; never on the GPU box.
"""
from __future__ import annotations

import sys
import types

from . import pvoc_oracle as P
from . import ref_facade


def _librosa_module() -> types.ModuleType:
    lib = types.ModuleType("librosa")
    lib.__dict__.update(vars(P.librosa))
    util = types.ModuleType("librosa.util")
    util.__dict__.update(vars(P.librosa.util))
    lib.util = util
    return lib


def change_speed(array, speed_factor, sample_rate: int = 24000):
    """-> the reference's TTSOutput(array=array, sample_rate=sample_rate).change_speed(speed_factor) (a reference
    TTSOutput, or the object itself for speed 1)."""
    out_cls = ref_facade.load().TTSOutput
    saved = {k: sys.modules.get(k) for k in ("librosa", "librosa.util")}
    lib = _librosa_module()
    sys.modules["librosa"], sys.modules["librosa.util"] = lib, lib.util
    try:
        return out_cls(array=array, sample_rate=sample_rate).change_speed(speed_factor)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
