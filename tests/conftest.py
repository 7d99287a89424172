import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from auralis_b200.config import XTTSDims               # noqa: E402
from auralis_b200.weights import synth_state           # noqa: E402

SEED = 1234


# The CPU oracle is small-tensor torch work: on a many-core GPU host the default (one thread per core) spends
# its time in thread wake-ups, so the checker is pinned to a modest pool.
torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a)")
    config.addinivalue_line("markers", "slow: long-running")


def has_gpu() -> bool:
    return torch.cuda.is_available()


def pytest_collection_modifyitems(config, items):
    """A machine with the library built but no H100: GPU tests are skipped, not errored (the library has no CPU fallback)."""
    ok = has_gpu() and torch.cuda.get_device_capability(0) == (9, 0)
    if ok:
        return
    skip = pytest.mark.skip(reason="needs an sm_90 GPU (libxtts_b200 has no CPU fallback)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def dims_small():
    return XTTSDims.small()


@pytest.fixture(scope="session")
def dims_full():
    return XTTSDims.full()


@pytest.fixture(scope="session")
def state_small(dims_small):
    return synth_state(dims_small, SEED)


@pytest.fixture(scope="session")
def state_full(dims_full):
    return synth_state(dims_full, SEED)


def _speakers(dims, n=3):
    """Deterministic synthetic speaker conditioning (cond latents [32,H], unit d-vector)."""
    out = []
    for i in range(n):
        g = torch.Generator().manual_seed(500 + i)
        cond = torch.randn(dims.gpt.n_cond_latents, dims.gpt.hidden, generator=g)
        dv = torch.nn.functional.normalize(torch.randn(dims.voc.d_vector, generator=g), dim=0)
        out.append((cond, dv))
    return out


@pytest.fixture(scope="session")
def speakers_small(dims_small):
    return _speakers(dims_small)


@pytest.fixture(scope="session")
def speakers_full(dims_full):
    return _speakers(dims_full)


def _make_engine(dims, state, speakers, precision, max_batch=8):
    from auralis_b200 import native
    eng = native.NativeEngine(dims, device=0, precision=precision, max_batch=max_batch, max_speakers=8)
    eng.load_state(*state)
    for i, (c, g) in enumerate(speakers):
        eng.set_speaker(i, c.numpy(), g.numpy())
    return eng


@pytest.fixture(scope="module")
def engine_small(dims_small, state_small, speakers_small):
    eng = _make_engine(dims_small, state_small, speakers_small, 0)
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def engine_small_bf16(dims_small, state_small, speakers_small):
    eng = _make_engine(dims_small, state_small, speakers_small, 1)
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def engine_full(dims_full, state_full, speakers_full):
    eng = _make_engine(dims_full, state_full, speakers_full, 0, max_batch=4)
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def engine_full_bf16(dims_full, state_full, speakers_full):
    eng = _make_engine(dims_full, state_full, speakers_full, 1, max_batch=4)
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def engine_small_fp16(dims_small, state_small, speakers_small):
    eng = _make_engine(dims_small, state_small, speakers_small, 2)
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def engine_full_fp16(dims_full, state_full, speakers_full):
    eng = _make_engine(dims_full, state_full, speakers_full, 2, max_batch=4)
    yield eng
    eng.close()


def text_ids(dims, n, seed):
    """[bos] + n synthetic BPE ids + [eos] (XTTSv2.py:519-522); ids 0/1 stand in for [START]/[STOP]."""
    rng = np.random.RandomState(seed)
    body = rng.randint(2, dims.gpt.n_text_tokens, size=n).tolist()
    return [0] + body + [1]
