"""GPU: HiFi-GAN vocoder kernels vs the oracle and vs the reference-produced golden waveform."""
import os

import numpy as np
import pytest
import torch

from oracle import xtts_oracle as O

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 2e-4          # fp32 waveform tolerance (tanh output in [-1,1]); fp32 accumulation order differs from ATen


def _check_stages(eng, dims, cs, lat, spk_idx, g):
    wav_ref, stages = O.vocoder(torch.from_numpy(lat), g, cs, dims, return_stages=True)
    nk = len(dims.voc.rb_kernels)
    report = []
    for name, ref in stages.items():
        got_wav, got = eng.vocode(lat, spk_idx, stage=name, stage_shape=tuple(ref.shape))
        scale = nk if name.startswith("mrf") else 1.0        # engine keeps the un-normalised MRF sum
        err = np.abs(got / scale - ref.numpy()).max()
        report.append((name, float(err), float(np.abs(ref.numpy()).max())))
    return wav_ref.numpy(), report


@pytest.mark.parametrize("T", [1, 5, 23])
def test_vocoder_small_vs_oracle(engine_small, dims_small, state_small, speakers_small, T):
    rng = np.random.RandomState(T)
    lat = rng.randn(T, dims_small.voc.in_dim).astype(np.float32)
    wav_ref, report = _check_stages(engine_small, dims_small, state_small[1], lat, 1, speakers_small[1][1])
    wav = engine_small.vocode(lat, 1)
    print(report)
    assert wav.shape == wav_ref.shape
    for name, err, mag in report:
        assert err < 1e-3 * max(1.0, mag), report
    assert np.abs(wav - wav_ref).max() < TOL, np.abs(wav - wav_ref).max()


@pytest.mark.parametrize("name", ["small", "full"])
def test_vocoder_vs_reference_golden(name, request):
    """CUDA path against the waveform the reference's own HifiDecoder produced (tests/golden)."""
    eng = request.getfixturevalue(f"engine_{name}")
    z = np.load(os.path.join(GOLD, f"vocoder_{name}.npz"))
    eng.set_speaker(7, np.zeros((eng.dims.gpt.n_cond_latents, eng.dims.gpt.hidden), np.float32), z["g"])
    wav = eng.vocode(z["latents"], 7)
    err = np.abs(wav - z["wav"]).max()
    print("golden", name, "max-abs err", err, "signal max", np.abs(z["wav"]).max())
    assert err < TOL


def test_vocoder_full_vs_oracle(engine_full, dims_full, state_full, speakers_full):
    rng = np.random.RandomState(11)
    lat = rng.randn(40, dims_full.voc.in_dim).astype(np.float32)
    wav_ref, report = _check_stages(engine_full, dims_full, state_full[1], lat, 0, speakers_full[0][1])
    print(report)
    wav = engine_full.vocode(lat, 0)
    assert np.abs(wav - wav_ref).max() < TOL, (np.abs(wav - wav_ref).max(), report)
    mse = float(np.mean((wav - wav_ref) ** 2))
    assert mse < 1e-9, mse


def test_vocoder_max_length_shape(engine_full, dims_full):
    """the BASELINE unit of work: 605 latents -> 674304 samples; finite, bounded by tanh."""
    rng = np.random.RandomState(2)
    lat = rng.randn(605, dims_full.voc.in_dim).astype(np.float32)
    wav = engine_full.vocode(lat, 0)
    assert wav.shape == (674304,) and np.isfinite(wav).all() and np.abs(wav).max() <= 1.0


# ------------------------------------------------------------------------------------------------
# fast mode: Conv1d on the tensor cores (wgmma, fp16 operands, fp32 accumulate) — the precision the
# reference itself runs the vocoder at on GPU (torch.amp.autocast fp16, hifigan_decoder.py:241-242)
# ------------------------------------------------------------------------------------------------
TOL_FP16 = 2e-2


@pytest.mark.parametrize("T", [1, 5, 23])
def test_vocoder_tc_small_vs_oracle(engine_small_bf16, dims_small, state_small, speakers_small, T):
    rng = np.random.RandomState(T)
    lat = rng.randn(T, dims_small.voc.in_dim).astype(np.float32)
    wav_ref, report = _check_stages(engine_small_bf16, dims_small, state_small[1], lat, 1, speakers_small[1][1])
    wav = engine_small_bf16.vocode(lat, 1)
    print("tc", report, "wav err", np.abs(wav - wav_ref).max())
    for name, err, mag in report:
        assert err < 2e-2 * max(1.0, mag), report
    assert np.abs(wav - wav_ref).max() < TOL_FP16


def test_vocoder_tc_full_vs_oracle_and_fp32_path(engine_full_bf16, dims_full, state_full, speakers_full):
    rng = np.random.RandomState(11)
    lat = rng.randn(40, dims_full.voc.in_dim).astype(np.float32)
    wav_ref, report = _check_stages(engine_full_bf16, dims_full, state_full[1], lat, 0, speakers_full[0][1])
    wav = engine_full_bf16.vocode(lat, 0)
    err = np.abs(wav - wav_ref).max()
    mse = float(np.mean((wav - wav_ref) ** 2))
    print("tc full", report, "wav max err", err, "mse", mse, "signal rms", float(np.sqrt(np.mean(wav_ref ** 2))))
    assert err < TOL_FP16 and mse < 1e-5
    # the same engine with the tensor-core convs switched off must reproduce the fp32 result
    engine_full_bf16.set_option("tc_vocoder", 0)
    wav32 = engine_full_bf16.vocode(lat, 0)
    engine_full_bf16.set_option("tc_vocoder", 1)
    assert np.abs(wav32 - wav_ref).max() < TOL
