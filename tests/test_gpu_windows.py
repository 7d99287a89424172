"""GPU: the vocoder as WINDOWS of a chunk, on its own stream, in ragged batches (round 2).

The scheduler no longer vocodes whole chunks at the end of their decode: finished chunks of any length share a launch
(per-item lengths in the tensor-core conv kernels), and — engine option "voc_segment" / xtts_sampling.early_tokens — a
chunk's audio is produced window by window while it is still decoding.  Everything here is a size-independent property:
windows, ragged batches and streaming pieces must reproduce the unsplit, single-chunk result sample for sample."""
import numpy as np
import pytest
import torch

from auralis_b200 import native
from auralis_b200.native import Sampling
from conftest import text_ids

pytestmark = pytest.mark.gpu


def _jobs(dims, n_seq, max_tokens, early=0, temperature=0.0, base=100):
    jobs = []
    for i in range(n_seq):
        mt = max_tokens[i] if isinstance(max_tokens, (list, tuple)) else max_tokens
        sp = Sampling(temperature=temperature, top_p=0.85, top_k=50, repetition_penalty=5.0, max_tokens=mt,
                      stop_token=dims.gpt.stop_audio_token, seed=7, seq_seed=i,
                      early_tokens=(early[i] if isinstance(early, (list, tuple)) else early))
        jobs.append((base + i, text_ids(dims, 9 + 3 * (i % 5), i), i % 2, sp))
    return jobs


@pytest.mark.parametrize("which,dims_name,T", [("engine_small", "dims_small", 40), ("engine_small_bf16", "dims_small", 40),
                                                ("engine_full_bf16", "dims_full", 605), ("engine_full", "dims_full", 60)])
def test_window_interior_equals_whole_chunk(request, which, dims_name, T):
    """xtts_vocode_window: samples further than the receptive field (16 z-frames) from an inner window edge are the whole
    chunk's, bit for bit (same arithmetic on the same inputs); window edges that coincide with the chunk's edges need no
    margin.  engine_full_bf16 runs the fp16 tensor-core convs; the others run the fp32 convs (the small geometry has no
    tensor-core plan, so engine_small_bf16 falls back to them)."""
    eng, dims = request.getfixturevalue(which), request.getfixturevalue(dims_name)
    hop, HZ = dims.voc.hop, 16
    lat = torch.randn(T, dims.voc.in_dim, generator=torch.Generator().manual_seed(77)).numpy()
    eng.set_option("profile", 1)
    try:
        full = eng.vocode(lat, 0)
        Tz = dims.voc.z_frames(T)
        assert full.shape[0] == Tz * hop
        for z0, z1 in [(0, Tz // 2), (Tz // 3, Tz - 5), (Tz // 2, Tz), (0, Tz), (max(0, Tz - 40), Tz)]:
            if z1 - z0 <= 2 * HZ:
                continue
            w = eng.vocode_window(lat, 0, z0, z1 - z0)
            a = 0 if z0 == 0 else HZ
            b = (z1 - z0) if z1 == Tz else (z1 - z0 - HZ)
            np.testing.assert_array_equal(w[a * hop: b * hop], full[(z0 + a) * hop: (z0 + b) * hop])
        n_tc = eng.kernel_profile().get("conv1d_tc_f16_wgmma", {}).get("launches", 0)
    finally:
        eng.set_option("profile", 0)
    assert (n_tc > 0) == (which == "engine_full_bf16"), n_tc


@pytest.mark.parametrize("which", ["engine_small", "engine_small_bf16", "engine_small_fp16", "engine_full_bf16"])
def test_ragged_batch_equals_single_chunks(request, which):
    """chunks of different lengths finish at different steps and share vocoder launches (per-item lengths): tokens and
    waveform of each equal what the same chunk gives alone; the waveform also equals xtts_vocode of its own latents.
    engine_full_bf16 vocodes these ragged batches with the tensor-core convs."""
    eng = request.getfixturevalue(which)
    dims = eng.dims
    lens = [5, 33, 12, 40, 7, 26, 40, 19]
    jobs = _jobs(dims, len(lens), lens)
    eng.set_option("profile", 1)
    try:
        res = eng.run_batch(jobs, timeout_s=120, want_latents=True)
        n_tc = eng.kernel_profile().get("conv1d_tc_f16_wgmma", {}).get("launches", 0)
    finally:
        eng.set_option("profile", 0)
    assert (n_tc > 0) == (which == "engine_full_bf16"), n_tc
    for (sid, ids, spk, sp), n in zip(jobs, lens):
        r, toks, wav, lat = res[sid]
        assert r.n_tokens == n and r.n_samples == dims.voc.n_samples(n) == wav.shape[0]
        alone = eng.run_batch([(sid, ids, spk, sp)], timeout_s=60)[sid]
        np.testing.assert_array_equal(toks, alone[1])
        np.testing.assert_array_equal(wav, alone[2])
        np.testing.assert_array_equal(wav, eng.vocode(lat, spk))


@pytest.mark.parametrize("which", ["engine_small", "engine_small_bf16", "engine_full_bf16", "engine_full_fp16"])
def test_segmented_vocoding_equals_whole(request, which):
    """option voc_segment: windows cut while the chunk decodes (the vocoder overlapping the decode step on its own stream,
    with and without an SM cap) give the same result as one window at the end."""
    eng = request.getfixturevalue(which)
    dims = eng.dims
    lens = [40, 31, 40, 9] if dims.gpt.hidden < 512 else [64, 50, 33]
    jobs = _jobs(dims, len(lens), lens, temperature=0.75)
    try:
        eng.set_option("voc_segment", 0)
        ref = eng.run_batch(jobs, timeout_s=300)
        for seg, sms in [(8, 0), (13, 24), (16, 0)]:
            eng.set_option("voc_segment", seg)
            eng.set_option("voc_sms", sms)
            got = eng.run_batch(jobs, timeout_s=300)
            assert not eng.last_partials                    # nobody asked for streaming pieces
            for sid in ref:
                np.testing.assert_array_equal(got[sid][1], ref[sid][1])
                np.testing.assert_array_equal(got[sid][2], ref[sid][2])
    finally:
        eng.set_option("voc_segment", 0)
        eng.set_option("voc_sms", 0)


@pytest.mark.parametrize("which", ["engine_small", "engine_small_bf16"])
def test_streaming_pieces_concatenate_to_the_unsplit_chunk(request, dims_small, which):
    """xtts_sampling.early_tokens: partial results (status 1) while the chunk decodes, oldest first, each carrying its own
    tokens and samples; partials + final == the unsplit chunk.  Sequence 1 never asks and gets one result."""
    eng = request.getfixturevalue(which)
    ref = eng.run_batch(_jobs(dims_small, 3, 40), timeout_s=120)
    assert not eng.last_partials
    try:
        for seg, n_parts in [(0, 1), (10, 3)]:               # first cut only / then every 10 tokens (10, 20, 30)
            eng.set_option("voc_segment", seg)
            got = eng.run_batch(_jobs(dims_small, 3, 40, early=[10, 0, 10]), timeout_s=120)
            parts = dict(eng.last_partials)
            assert sorted(parts) == [100, 102]
            for sid in (100, 101, 102):
                r, toks, wav, _ = got[sid]
                np.testing.assert_array_equal(toks, ref[sid][1])
                ps = parts.get(sid, [])
                assert len(ps) == (n_parts if sid != 101 else 0)
                assert all(p[0].status == 1 and p[0].t_done <= r.t_done for p in ps)
                if ps:
                    assert ps[0][0].n_tokens == 10 and ps[0][0].n_samples == dims_small.voc.n_samples(10)
                    np.testing.assert_array_equal(np.concatenate([p[1] for p in ps]), ref[sid][1][: 10 * len(ps)])
                np.testing.assert_array_equal(np.concatenate([p[2] for p in ps] + [wav]), ref[sid][2])
    finally:
        eng.set_option("voc_segment", 0)


def test_short_chunks_are_never_split(engine_small, dims_small):
    """a chunk that ends before the frames behind its first cut exist is delivered whole"""
    got = engine_small.run_batch(_jobs(dims_small, 3, 12, early=10), timeout_s=60)
    assert not engine_small.last_partials and all(got[s][0].n_tokens == 12 for s in got)


def test_cancel_frees_the_slot_and_reports_cancelled(engine_full_bf16, dims_full):
    """xtts_cancel (ADVICE r1): a queued chunk is dropped, a decoding one stops (full geometry: 605 tokens take ~1 s, the
    cancel lands mid-decode); each reports XTTS_ERR_CANCELLED exactly once, the others finish, every slot is usable again."""
    import time
    eng, dims = engine_full_bf16, dims_full
    long_sp = Sampling(temperature=0.75, repetition_penalty=5.0, max_tokens=dims.gpt.max_audio_tokens,
                       stop_token=4095, seed=3)             # an id outside the vocabulary: the chunk runs to max_tokens
    ids = text_ids(dims, 12, 1)
    eng.set_option("hold_admission", 1)
    for sid in (1, 2, 3):
        eng.submit(sid, ids, 0, long_sp)
    eng.cancel(2)                                           # still queued
    eng.cancel(999)                                         # unknown: ignored
    eng.set_option("hold_admission", 0)
    time.sleep(0.25)
    eng.cancel(3)                                           # decoding
    seen, t0 = {}, time.time()
    while len(seen) < 3:
        r = eng.poll(2000)
        assert r is not None
        if r.status == 0:
            eng.fetch(r)
        else:
            eng.lib.xtts_fetch(eng.h, r.seq_id, None, None, None)
        seen[r.seq_id] = (r.status, r.n_tokens, time.time() - t0)
    assert seen[1][:2] == (0, dims.gpt.max_audio_tokens)
    assert seen[2][0] == native.ERR_CANCELLED and seen[3][0] == native.ERR_CANCELLED
    assert seen[3][2] < seen[1][2]                          # the cancelled chunk did not decode to the end
    res = eng.run_batch(_jobs(dims, 4, 16), timeout_s=60)   # every slot is usable again
    assert all(res[s][0].n_tokens == 16 for s in res)


def test_bad_text_id_fails_only_its_submit(engine_small, dims_small):
    """ADVICE r1: an out-of-range text id is rejected by xtts_submit itself (not inside the batched step)."""
    sp = Sampling(temperature=0.0, max_tokens=4, stop_token=dims_small.gpt.stop_audio_token)
    with pytest.raises(native.NativeError):
        engine_small.submit(50, [0, dims_small.gpt.n_text_tokens + 3, 1], 0, sp)
    res = engine_small.run_batch(_jobs(dims_small, 2, 6), timeout_s=60)
    assert all(res[s][0].n_tokens == 6 for s in res)
