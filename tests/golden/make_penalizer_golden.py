"""Golden outputs of the reference's own `LogitsRepetitionPenalizer` (models/xttsv2/components/vllm/hijack.py, lifted by
source: the module itself imports vLLM) on the cases of tests/test_oracle_gpt.py::penalizer_trials.

    python tests/golden/make_penalizer_golden.py          (needs the reference source tree, see oracle/ref_import.py)
"""
import ast
import os
import sys
from typing import List

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from auralis_b200.config import XTTSDims  # noqa: E402
from oracle import ref_import  # noqa: E402
from test_oracle_gpt import PENALIZER_GOLDEN, penalizer_trials  # noqa: E402


def main():
    path = os.path.join(ref_import.REF_SRC, "auralis", "models", "xttsv2", "components", "vllm", "hijack.py")
    tree = ast.parse(open(path).read())
    cls = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "LogitsRepetitionPenalizer"]
    ns = {"torch": torch, "List": List}
    exec(compile(ast.Module(body=cls, type_ignores=[]), path, "exec"), ns)
    Pen = ns["LogitsRepetitionPenalizer"]
    rec = {f"trial{i}": Pen(p)(prompt, gen, z.clone()).numpy() for i, (z, prompt, gen, p) in enumerate(penalizer_trials(XTTSDims.small()))}
    np.savez_compressed(PENALIZER_GOLDEN, **rec)
    print(f"{PENALIZER_GOLDEN}: {os.path.getsize(PENALIZER_GOLDEN)} bytes")


if __name__ == "__main__":
    main()
