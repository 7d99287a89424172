"""CPU: the C-ABI library loads and exports every symbol include/xtts_b200.h declares; creating an engine
without a GPU fails loudly (no CPU fallback)."""
import ctypes
import os
import re

import pytest
import torch

from auralis_b200 import native
from auralis_b200.build import build_native
from auralis_b200.config import XTTSDims

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    build_native()
    return native.load_library()


def test_header_symbols_are_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "xtts_b200.h")).read()
    declared = set(re.findall(r"\b(xtts_[a-z_0-9]+)\s*\(", hdr))
    assert declared == set(native.ABI_SYMBOLS), declared ^ set(native.ABI_SYMBOLS)
    for s in declared:
        assert hasattr(lib, s), s
    assert b"sm_90a" in lib.xtts_version()


def test_struct_layouts_match_header():
    # sizes implied by the header (all 4-byte fields except the 8-byte ones noted there)
    assert ctypes.sizeof(native.XttsSampling) == 48
    assert ctypes.sizeof(native.XttsResult) == 48
    assert ctypes.sizeof(native.XttsStats) == 9 * 8
    assert ctypes.sizeof(native.XttsConfig) == 4 * (4 + 12 + 3 + 8 + 1 + 8 + 1 + 4 + 6 + 8 + 2)


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only check")
def test_no_cpu_fallback(lib):
    with pytest.raises(native.NativeError) as ei:
        native.NativeEngine(XTTSDims.small())
    assert "no CUDA device" in str(ei.value) or "CUDA" in str(ei.value)


def test_product_package_never_imports_oracle():
    pkg = os.path.join(ROOT, "auralis_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, os.path.join(dp, f)
