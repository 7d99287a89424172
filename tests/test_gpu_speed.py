"""GPU: the speaking rate (xtts_submit_speed / xtts_vocode_speed, TTSRequest.speed).

A speed other than 1 time-scales the chunk's GPT latents by one more linear interpolation in front of the vocoder's two
(Coqui's Xtts.inference, restated in tests/speed_reference.py), fused into the vocoder's interpolation kernel.  The GPT never
sees the speed.  Checked here: parity with the reference on both vocoder paths, speed 1 being the old path bit for bit,
chunks stretched past one vocoder window, windows / segments / streaming pieces reproducing the unsplit chunk, ragged
batches mixing speeds, and the range check."""
import math

import numpy as np
import pytest
import torch

from auralis_b200 import native
from auralis_b200.native import Sampling
from conftest import text_ids
import speed_reference as SR

pytestmark = pytest.mark.gpu
TOL = 2e-4             # fp32 waveform tolerance of the vocoder tests (tests/test_gpu_vocoder.py)
TOL_FP16 = 2e-2        # fast-mode (fp16 tensor-core convs) waveform tolerance, same file
NO_STOP = 4095         # a stop token outside the vocabulary: the chunk runs to max_tokens


def _lat(dims, T, seed):
    return np.random.RandomState(seed).randn(T, dims.voc.in_dim).astype(np.float32)


def _tc_launches(eng, fn):
    eng.set_option("profile", 1)
    try:
        out = fn()
        return out, eng.kernel_profile().get("conv1d_tc_f16_wgmma", {}).get("launches", 0)
    finally:
        eng.set_option("profile", 0)


def _jobs(dims, lens, speeds, early=0, temperature=0.0, base=300, stop=None):
    jobs = []
    for i, (n, s) in enumerate(zip(lens, speeds)):
        sp = Sampling(temperature=temperature, top_p=0.85, top_k=50, repetition_penalty=5.0, max_tokens=n,
                      stop_token=dims.gpt.stop_audio_token if stop is None else stop, seed=7, seq_seed=i,
                      early_tokens=early, speed=s)
        jobs.append((base + i, text_ids(dims, 9 + 3 * (i % 5), i), i % 2, sp))
    return jobs


# ---- 4. parity with the reference ------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,speed", [(5, 0.5), (23, 0.77), (23, 1.3), (9, 2.0), (23, 3.3), (23, 4.0), (40, 0.25)])
def test_vocode_speed_small_vs_reference(engine_small, dims_small, state_small, speakers_small, T, speed):
    """fp32 vocoder at a speed == the reference (Coqui's stage + the pinned oracle).  T = 40 at speed 0.25 is longer than
    one vocoder window of the small geometry: it is vocoded in several, stitched."""
    lat = _lat(dims_small, T, T)
    ref = SR.vocoder(torch.from_numpy(lat), speakers_small[1][1], state_small[1], dims_small, speed).numpy()
    wav = engine_small.vocode_speed(lat, 1, speed)
    assert wav.shape == ref.shape == (dims_small.voc.n_samples(T, speed),)
    assert np.abs(wav - ref).max() < TOL, np.abs(wav - ref).max()


@pytest.mark.parametrize("which", ["engine_full", "engine_full_bf16", "engine_full_fp16"])
def test_vocode_speed_full_vs_reference(request, dims_full, state_full, speakers_full, which):
    """Full geometry, both vocoder paths: fp32 convs within the fp32 tolerance, the fast modes' fp16 tensor-core convs
    within the fast-mode tolerance (and they did run)."""
    eng = request.getfixturevalue(which)
    lat = _lat(dims_full, 40, 11)
    for speed in (0.7, 2.0):
        ref = SR.vocoder(torch.from_numpy(lat), speakers_full[0][1], state_full[1], dims_full, speed).numpy()
        wav, n_tc = _tc_launches(eng, lambda: eng.vocode_speed(lat, 0, speed))
        assert wav.shape == ref.shape
        err, mse = float(np.abs(wav - ref).max()), float(np.mean((wav - ref) ** 2))
        print(which, speed, "max err", err, "mse", mse)
        if which == "engine_full":
            assert n_tc == 0 and err < TOL and mse < 1e-9
        else:
            assert n_tc > 0 and err < TOL_FP16 and mse < 1e-5


def test_zero_frame_chunk(engine_small, dims_small):
    """3 latents at speed 4 scale to no frame: an empty waveform, no launch."""
    assert dims_small.voc.n_samples(3, 4.0) == 0
    assert engine_small.vocode_speed(_lat(dims_small, 3, 1), 0, 4.0).shape == (0,)


# ---- 5. speed 1 is the old path ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["engine_small", "engine_full_bf16"])
def test_speed_one_is_the_old_path(request, which, monkeypatch):
    eng = request.getfixturevalue(which)
    dims = eng.dims
    lat = _lat(dims, 37, 5)
    Tz = dims.voc.z_frames(37)
    np.testing.assert_array_equal(eng.vocode_speed(lat, 0, 1.0), eng.vocode(lat, 0))
    np.testing.assert_array_equal(eng.vocode_speed(lat, 0, 1.0, Tz // 3, Tz // 2), eng.vocode_window(lat, 0, Tz // 3, Tz // 2))
    jobs = _jobs(dims, [12, 30, 21], [1.0, 1.0, 1.0], temperature=0.75)
    new = eng.run_batch(jobs, timeout_s=120)

    def raw_submit(sid, ids, spk, sp):                     # the speed-less entry point
        t = np.ascontiguousarray(ids, dtype=np.int32)
        cs = sp.c()
        rc = eng.lib.xtts_submit(eng.h, sid, t.ctypes.data_as(native.C.POINTER(native.C.c_int32)), t.size, spk,
                                 native.C.byref(cs))
        assert rc == 0, eng.lib.xtts_last_error()
    monkeypatch.setattr(eng, "submit", raw_submit)
    old = eng.run_batch(jobs, timeout_s=120)
    for sid in old:
        np.testing.assert_array_equal(new[sid][1], old[sid][1])
        np.testing.assert_array_equal(new[sid][2], old[sid][2])


# ---- 6. a chunk longer than one vocoder window -------------------------------------------------------------------------
_SPLIT_REF = {}


@pytest.mark.parametrize("which", ["engine_full", "engine_full_bf16"])
def test_window_split_of_a_stretched_chunk(request, dims_full, state_full, speakers_full, which):
    """T = 200 at speed 0.25 is 3482 z-frames, more than the 2634 of one window (605 tokens at speed 1): the whole-chunk
    vocode stitches the scheduler's windows.  It matches the reference, and a decoded chunk of that length (forced by
    max_tokens, no stop token) gets exactly those samples."""
    eng, dims = request.getfixturevalue(which), dims_full
    T, speed = 200, 0.25
    assert dims.voc.z_frames(T, speed) == 3482 and dims.voc.z_frames(dims.gpt.max_audio_tokens) == 2634
    lat = _lat(dims, T, 3)
    if "ref" not in _SPLIT_REF:
        _SPLIT_REF["ref"] = SR.vocoder(torch.from_numpy(lat), speakers_full[0][1], state_full[1], dims, speed).numpy()
    ref = _SPLIT_REF["ref"]
    wav = eng.vocode_speed(lat, 0, speed)
    err = float(np.abs(wav - ref).max())
    print(which, "split whole-chunk max err", err)
    assert wav.shape == ref.shape and err < (TOL if which == "engine_full" else TOL_FP16)
    eng.set_option("voc_segment", 0)
    sp = Sampling(temperature=0.75, max_tokens=T, stop_token=NO_STOP, seed=5, speed=speed)
    r, toks, got, glat = eng.run_batch([(1, text_ids(dims, 12, 4), 0, sp)], timeout_s=300, want_latents=True)[1]
    assert r.n_tokens == T and r.n_samples == dims.voc.n_samples(T, speed) == got.shape[0]
    np.testing.assert_array_equal(got, eng.vocode_speed(glat, 0, speed))


# ---- 7. windows --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which,T", [("engine_small", 40), ("engine_full_bf16", 120), ("engine_full", 60)])
def test_window_interior_equals_whole_chunk_at_speed(request, which, T):
    """xtts_vocode_speed windows: samples more than 16 z-frames from an inner window edge are the whole chunk's, bit for
    bit, at speeds != 1 (the source positions of all three levels depend on the global index only)."""
    eng = request.getfixturevalue(which)
    dims, hop, HZ = eng.dims, eng.dims.voc.hop, 16
    lat = _lat(dims, T, 77)
    for speed in (0.5, 1.7, 3.3):
        full = eng.vocode_speed(lat, 0, speed)
        Tz = dims.voc.z_frames(T, speed)
        assert full.shape[0] == Tz * hop
        for z0, z1 in [(0, Tz // 2), (Tz // 3, Tz - 5), (Tz // 2, Tz), (max(0, Tz - 40), Tz)]:
            if z1 - z0 <= 2 * HZ or z1 - z0 > dims.voc.z_frames(dims.gpt.max_audio_tokens):
                continue
            w = eng.vocode_speed(lat, 0, speed, z0, z1 - z0)
            a = 0 if z0 == 0 else HZ
            b = (z1 - z0) if z1 == Tz else (z1 - z0 - HZ)
            np.testing.assert_array_equal(w[a * hop: b * hop], full[(z0 + a) * hop: (z0 + b) * hop])


# ---- 8. the engine: ragged batches mixing speeds ----------------------------------------------------------------------
@pytest.mark.parametrize("which", ["engine_small", "engine_full_bf16"])
def test_ragged_batch_mixing_speeds(request, which):
    """Tokens equal the speed-1 run (the GPT never sees the speed); each chunk's samples equal the same chunk run alone and
    xtts_vocode_speed of its own latents."""
    eng = request.getfixturevalue(which)
    dims = eng.dims
    lens = [5, 33, 12, 40, 7, 26, 40, 19]
    speeds = [0.5, 1.0, 1.7, 4.0, 0.5, 4.0, 0.77, 1.3]
    res = eng.run_batch(_jobs(dims, lens, speeds), timeout_s=300, want_latents=True)
    base = eng.run_batch(_jobs(dims, lens, [1.0] * len(lens)), timeout_s=300)
    for (sid, ids, spk, sp), n, s in zip(_jobs(dims, lens, speeds), lens, speeds):
        r, toks, wav, lat = res[sid]
        np.testing.assert_array_equal(toks, base[sid][1])
        assert r.n_tokens == n and r.n_samples == dims.voc.n_samples(n, s)
        wav = wav if wav is not None else np.zeros(0, np.float32)
        assert wav.shape[0] == r.n_samples
        alone = eng.run_batch([(sid, ids, spk, sp)], timeout_s=120)[sid]
        np.testing.assert_array_equal(wav, alone[2] if alone[2] is not None else np.zeros(0, np.float32))
        np.testing.assert_array_equal(wav, eng.vocode_speed(lat, spk, s))


def test_zero_frame_chunk_gets_a_final_result(engine_small, dims_small):
    """3 tokens at speed 4: a normal final result listing its tokens, with no samples."""
    res = engine_small.run_batch(_jobs(dims_small, [3, 3], [4.0, 1.0], stop=NO_STOP), timeout_s=60)
    r, toks, wav, _ = res[300]
    assert r.status == 0 and r.n_tokens == 3 and len(toks) == 3 and r.n_samples == 0 and wav is None
    assert res[301][0].n_samples == dims_small.voc.n_samples(3)


# ---- 9. segmented vocoding and streaming -------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["engine_small", "engine_full_bf16"])
def test_segmented_vocoding_equals_whole_at_speed(request, which):
    eng = request.getfixturevalue(which)
    dims = eng.dims
    lens = [40, 31, 40, 9] if dims.gpt.hidden < 512 else [64, 50, 33]
    try:
        for speed in (0.5, 2.0):
            jobs = _jobs(dims, lens, [speed] * len(lens), temperature=0.75)
            eng.set_option("voc_segment", 0)
            ref = eng.run_batch(jobs, timeout_s=300)
            for seg in (8, 13, 16):
                eng.set_option("voc_segment", seg)
                got = eng.run_batch(jobs, timeout_s=300)
                assert not eng.last_partials
                for sid in ref:
                    np.testing.assert_array_equal(got[sid][1], ref[sid][1])
                    np.testing.assert_array_equal(got[sid][2], ref[sid][2])
    finally:
        eng.set_option("voc_segment", 0)


@pytest.mark.parametrize("which", ["engine_small", "engine_small_bf16"])
def test_streaming_pieces_at_speed(request, dims_small, which):
    """early_tokens at speeds 0.5 / 2: partial pieces, then the final result, in order, with contiguous sample ranges;
    together they are the unsplit chunk, and the final result lists every token.  (At 0.5 the rest of the 40-token chunk
    is longer than one window of the small geometry: the final result is stitched from internal windows.)"""
    eng = request.getfixturevalue(which)
    try:
        for speed in (0.5, 2.0):
            eng.set_option("voc_segment", 0)
            ref = eng.run_batch(_jobs(dims_small, [40, 40, 40], [speed] * 3), timeout_s=120)
            for seg in (0, 10):
                eng.set_option("voc_segment", seg)
                got = eng.run_batch(_jobs(dims_small, [40, 40, 40], [speed] * 3, early=10), timeout_s=120)
                parts = dict(eng.last_partials)
                for sid in ref:
                    r, toks, wav, _ = got[sid]
                    ps = parts.get(sid, [])
                    assert ps and all(p[0].status == 1 and p[0].t_done <= r.t_done for p in ps)
                    np.testing.assert_array_equal(toks, ref[sid][1])
                    np.testing.assert_array_equal(np.concatenate([p[1] for p in ps]), ref[sid][1][: sum(len(p[1]) for p in ps)])
                    assert ps[0][0].n_tokens == 10 and ps[0][0].n_samples == dims_small.voc.n_samples(10, speed)
                    n = len(ref[sid][1])                    # 40, or fewer where the stop token came first
                    assert sum(p[0].n_samples for p in ps) + r.n_samples == dims_small.voc.n_samples(n, speed)
                    assert r.n_tokens == n and len(toks) == n
                    np.testing.assert_array_equal(np.concatenate([p[2] for p in ps] + [wav]), ref[sid][2])
    finally:
        eng.set_option("voc_segment", 0)


# ---- 10. validation ----------------------------------------------------------------------------------------------------
def test_out_of_range_speed_fails_only_its_submit(engine_small, dims_small):
    ids = np.ascontiguousarray(text_ids(dims_small, 6, 0), dtype=np.int32)
    cs = Sampling(temperature=0.0, max_tokens=4, stop_token=dims_small.gpt.stop_audio_token).c()
    for bad in (0.0, 0.2, 4.5, -1.0, float("nan"), float("inf")):
        rc = engine_small.lib.xtts_submit_speed(engine_small.h, 60, ids.ctypes.data_as(native.C.POINTER(native.C.c_int32)),
                                                ids.size, 0, native.C.byref(cs), bad)
        assert rc == -1, (bad, rc)                          # XTTS_ERR_INVALID
        with pytest.raises(native.NativeError):
            engine_small.vocode_speed(_lat(dims_small, 5, 0), 0, bad)
    res = engine_small.run_batch(_jobs(dims_small, [6, 6], [0.25, 4.0]), timeout_s=60)
    assert all(res[s][0].n_tokens == 6 for s in res)
    assert res[300][0].n_samples == dims_small.voc.n_samples(6, 0.25)
