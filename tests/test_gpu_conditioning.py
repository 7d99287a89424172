"""GPU: speaker conditioning (mel STFT -> ConditioningEncoder -> Perceiver; ResNet speaker encoder) through
xtts_condition, vs the oracle and vs the golden vectors the reference's own modules produced."""
import os

import numpy as np
import pytest
import torch

from oracle import xtts_oracle as O

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _ref(dims, cs, wav22, wav16, length=30, chunk=4):
    with torch.no_grad():
        cond = O.gpt_cond_latents(torch.from_numpy(wav22), cs, dims, length, chunk).numpy()
        g = O.speaker_embedding(torch.from_numpy(wav16), cs, dims).numpy()
    return cond, g


@pytest.mark.parametrize("name", ["small", "full"])
def test_condition_matches_reference_golden(name, request):
    eng = request.getfixturevalue(f"engine_{name}")
    z = np.load(os.path.join(GOLD, f"conditioning_{name}.npz"))
    eng.condition(6, z["wav22"], z["wav16"], 30, 4)            # 0.6 s -> a single piece
    cond, g = eng.get_speaker(6)
    e1, e2 = np.abs(cond - z["perceiver"]).max(), np.abs(g - z["dvector"]).max()
    print("golden", name, "cond err", e1, "max", np.abs(z["perceiver"]).max(), "dvec err", e2)
    assert e1 < 2e-3 * max(1.0, np.abs(z["perceiver"]).max())
    assert e2 < 2e-4
    assert abs(np.linalg.norm(g) - 1.0) < 1e-4


def _check_against_oracle(eng, dims, state, w22, w16, slot):
    eng.condition(slot, w22, w16, 30, 4)
    cond, g = eng.get_speaker(slot)
    rc, rg = _ref(dims, state[1], w22, w16)
    print("oracle", dims.gpt.hidden, len(w16), "cond err", np.abs(cond - rc).max(), "max", np.abs(rc).max(),
          "dvec err", np.abs(g - rg).max())
    assert np.abs(cond - rc).max() < 2e-3 * max(1.0, np.abs(rc).max()), np.abs(cond - rc).max()
    assert np.abs(g - rg).max() < 2e-4, np.abs(g - rg).max()


def test_condition_multi_piece_small(engine_small, dims_small, state_small):
    """6 s reference cut into 4 s pieces (one 4 s + one 2 s), averaged (XTTSv2.py:361-391)."""
    w22 = O.synthetic_reference_wav(6.0, 22050, 140.0, 3).numpy()
    w16 = O.synthetic_reference_wav(6.0, 16000, 140.0, 3).numpy()
    _check_against_oracle(engine_small, dims_small, state_small, w22, w16, 5)


# 16 kHz lengths: T = 1 + N/160 frames is odd at 1.00 s (101) and 10.5 s (1051), even at 1.01 s (102).  An odd T leaves
# the stride-2 layers an odd width to round up (the downsample branch writes ceil(T/2) columns), and 10.5 s makes layer
# 4 132 columns wide, more than one 128-wide conv2d block.  The 6 s case above has T = 601.
@pytest.mark.parametrize("name,sec16", [("small", 1.0), ("small", 1.01), ("full", 1.0), ("full", 1.01), ("small", 10.5)])
def test_condition_dvector_lengths_match_oracle(name, sec16, request):
    """The d-vector of a 16 kHz reference of sec16 seconds (and the latents of the same 6 s 22.05 kHz reference)."""
    eng = request.getfixturevalue(f"engine_{name}")
    w22 = O.synthetic_reference_wav(6.0, 22050, 140.0, 3).numpy()
    w16 = O.synthetic_reference_wav(sec16, 16000, 140.0, 3).numpy()
    _check_against_oracle(eng, request.getfixturevalue(f"dims_{name}"), request.getfixturevalue(f"state_{name}"), w22, w16, 5)


def test_condition_truncation_and_short_tail(engine_small, dims_small, state_small):
    """gpt_cond_len truncation and the < 0.33 s tail being dropped."""
    w22 = O.synthetic_reference_wav(4.2, 22050, 100.0, 9).numpy()     # 4 s piece + 0.2 s tail (dropped)
    w16 = O.synthetic_reference_wav(4.2, 16000, 100.0, 9).numpy()
    engine_small.condition(4, w22, w16, 3, 2)                         # cut to 3 s, 2 s pieces -> 2 + 1
    cond, _ = engine_small.get_speaker(4)
    rc, _ = _ref(dims_small, state_small[1], w22, w16, 3, 2)
    assert np.abs(cond - rc).max() < 2e-3 * max(1.0, np.abs(rc).max())


def test_conditioned_speaker_drives_synthesis(engine_small, dims_small, state_small):
    """the slot written by xtts_condition is usable by the GPT and the vocoder."""
    from auralis_b200.native import Sampling
    from conftest import text_ids
    w22 = O.synthetic_reference_wav(2.0, 22050, 170.0, 5).numpy()
    w16 = O.synthetic_reference_wav(2.0, 16000, 170.0, 5).numpy()
    engine_small.condition(3, w22, w16, 30, 4)
    cond, g = engine_small.get_speaker(3)
    orc = O.GPTOracle(state_small[0], state_small[1], dims_small)
    ids = text_ids(dims_small, 8, 21)
    sp = Sampling(temperature=0.0, repetition_penalty=5.0, max_tokens=16, stop_token=dims_small.gpt.stop_audio_token)
    r, toks, wav, _ = engine_small.run_batch([(9, ids, 3, sp)], timeout_s=60)[9]
    osp = O.SamplingParams(temperature=0.0, repetition_penalty=5.0, max_tokens=16, stop_token=dims_small.gpt.stop_audio_token)
    etoks, lats = orc.generate(torch.from_numpy(cond), ids, osp)
    assert list(toks) == etoks
    ewav = O.vocoder(lats, torch.from_numpy(g), state_small[1], dims_small).numpy()
    assert np.abs(wav - ewav).max() < 5e-4
