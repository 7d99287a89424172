"""GPU: beam-search decoding (xtts_submit_beams) against the oracle's transformers-5.5 beam search on GPTOracle, and its
place in the engine: latents and audio of the returned hypothesis, sharing steps with ordinary chunks, cancel."""
import ctypes as C
import itertools
import time

import numpy as np
import pytest

from auralis_b200.native import ERR_CANCELLED, NativeError, Sampling, XttsBeam
from oracle import beam_oracle as BO
from oracle import xtts_oracle as O
from conftest import _make_engine, text_ids

pytestmark = pytest.mark.gpu


def _sp(g, nb, lp=1.0, do_sample=False, mt=24, **kw):
    base = dict(temperature=0.75, top_p=0.85, top_k=50, repetition_penalty=5.0, max_tokens=mt,
                stop_token=g.stop_audio_token, seed=5, seq_seed=1)
    base.update(kw)
    return Sampling(num_beams=nb, length_penalty=lp, do_sample=do_sample, **base)


def _oracle(dims, state, speakers, spk, ids, sp):
    step = BO.GPTStep(O.GPTOracle(state[0], state[1], dims), speakers[spk][0], ids)
    r = BO.beam_search(step, step.first_logits, O.prompt_seen_set(dims.gpt), sp.num_beams, sp.max_tokens, sp.stop_token,
                       penalty=sp.repetition_penalty, length_penalty=sp.length_penalty, do_sample=sp.do_sample,
                       temperature=sp.temperature, top_k=sp.top_k, top_p=sp.top_p, seed=sp.seed, seq_seed=sp.seq_seed)
    return r, step


def _check_vs_oracle(dims, state, speakers, ids, sp, toks):
    ref, step = _oracle(dims, state, speakers, 0, ids, sp)
    if list(toks) != ref.tokens:
        # only an oracle near-tie may flip the choice: the engine's hypothesis must score like the oracle's best
        got = step.score(speakers[0][0], ids, list(toks), O.prompt_seen_set(dims.gpt), sp.repetition_penalty,
                         sp.length_penalty)
        assert abs(got - ref.score) <= 1e-4 * max(1.0, abs(ref.score)), (list(toks), ref.tokens, got, ref.score)
    return ref


@pytest.mark.parametrize("nb,lp", list(itertools.product([2, 4, 8], [0.0, 1.0, 2.0])))
def test_beam_search_matches_oracle(engine_small, dims_small, state_small, speakers_small, nb, lp):
    g = dims_small.gpt
    ids = text_ids(dims_small, 9, 40 + nb)
    sp = _sp(g, nb, lp)
    r, toks, wav, lat = engine_small.run_batch([(1, ids, 0, sp)], timeout_s=300, want_latents=True)[1]
    _check_vs_oracle(dims_small, state_small, speakers_small, ids, sp, toks)
    assert r.n_tokens == len(toks) and lat.shape == (len(toks), g.hidden)


def test_beam_sampling_matches_oracle(engine_small, dims_small, state_small, speakers_small):
    g = dims_small.gpt
    ids = text_ids(dims_small, 12, 7)
    sp = _sp(g, 4, 1.0, do_sample=True, seed=99, seq_seed=3)
    _, toks, _, _ = engine_small.run_batch([(2, ids, 0, sp)], timeout_s=300)[2]
    _check_vs_oracle(dims_small, state_small, speakers_small, ids, sp, toks)


def test_beam_stop_token_ends_group(engine_small, dims_small, state_small, speakers_small):
    """with a stop id the beams actually pick, the group ends on a finished hypothesis that carries the stop token"""
    g = dims_small.gpt
    ids = text_ids(dims_small, 6, 77)
    ref, _ = _oracle(dims_small, state_small, speakers_small, 0, ids, _sp(g, 4, 1.0, mt=30))
    sp = _sp(g, 4, 1.0, mt=30, stop_token=ref.tokens[5])
    _, toks, _, _ = engine_small.run_batch([(3, ids, 0, sp)], timeout_s=300)[3]
    ref = _check_vs_oracle(dims_small, state_small, speakers_small, ids, sp, toks)
    assert toks[-1] == sp.stop_token and len(toks) < 30


def test_beam_latents_and_audio(engine_small, dims_small, speakers_small):
    """the returned latents are the teacher-forced latents of the returned tokens; the audio is the vocoder's of those
    latents, bit for bit, at speed 1 and at another speed"""
    g = dims_small.gpt
    ids = text_ids(dims_small, 10, 11)
    sp = _sp(g, 4, 1.0)
    _, toks, wav, lat = engine_small.run_batch([(4, ids, 1, sp)], timeout_s=300, want_latents=True)[4]
    _, tf_lat, _ = engine_small.gpt_teacher_forced(ids, 1, list(toks), Sampling(temperature=0.0, max_tokens=len(toks),
                                                                                stop_token=g.stop_audio_token))
    np.testing.assert_allclose(lat, tf_lat, atol=3e-4, rtol=0)
    assert np.array_equal(wav, engine_small.vocode(lat, 1))
    sp2 = _sp(g, 4, 1.0, speed=1.5)
    _, toks2, wav2, lat2 = engine_small.run_batch([(5, ids, 1, sp2)], timeout_s=300, want_latents=True)[5]
    assert list(toks2) == list(toks) and np.array_equal(lat2, lat)
    assert np.array_equal(wav2, engine_small.vocode_speed(lat2, 1, 1.5))


def _submit_beams_raw(eng, sid, ids, spk, sp, beam):
    t = np.ascontiguousarray(ids, np.int32)
    cs = sp.c()
    rc = eng.lib.xtts_submit_beams(eng.h, sid, t.ctypes.data_as(C.POINTER(C.c_int32)), t.size, spk, C.byref(cs),
                                   float(sp.speed), C.byref(beam))
    return rc


def test_submit_beams_one_beam_is_submit_speed(engine_small, dims_small):
    g = dims_small.gpt
    ids = text_ids(dims_small, 8, 3)
    sp = Sampling(temperature=0.75, top_p=0.85, top_k=50, repetition_penalty=5.0, max_tokens=40,
                  stop_token=g.stop_audio_token, seed=21, seq_seed=2, speed=1.25)
    _, toks, wav, lat = engine_small.run_batch([(6, ids, 2, sp)], timeout_s=300, want_latents=True)[6]
    assert _submit_beams_raw(engine_small, 7, ids, 2, sp, XttsBeam(1, 2.0, 0)) == 0
    r = None
    while r is None:
        r = engine_small.poll(1000)
    assert r.seq_id == 7 and r.status == 0
    toks1, wav1, lat1 = engine_small.fetch(r, True, True)
    assert np.array_equal(toks1, toks) and np.array_equal(wav1, wav) and np.array_equal(lat1, lat)


def test_submit_beams_rejects_bad_arguments(engine_small, dims_small):
    g = dims_small.gpt
    ids = text_ids(dims_small, 4, 1)
    sp = _sp(g, 2)
    for bm in (XttsBeam(0, 1.0, 0), XttsBeam(9, 1.0, 0), XttsBeam(2, float("nan"), 0)):
        assert _submit_beams_raw(engine_small, 8, ids, 0, sp, bm) < 0
    with pytest.raises(NativeError):
        engine_small.submit(8, ids, 0, _sp(g, 2, early_tokens=8))
    with pytest.raises(NativeError):
        engine_small.submit(8, ids, 0, _sp(g, 9))


def test_beam_groups_share_steps_with_ordinary_chunks(dims_small, state_small, speakers_small):
    """>= 48 rows (both decode branches), graphs replayed: ordinary chunks are bit-identical with and without beam groups
    beside them, and the groups' results do not depend on cuda_graphs or microbatches"""
    g = dims_small.gpt
    eng = _make_engine(dims_small, state_small, speakers_small, 1, max_batch=64)
    try:
        plain = []
        for i in range(40):
            sp = Sampling(temperature=0.75, top_p=0.85, top_k=50, repetition_penalty=5.0, max_tokens=48,
                          stop_token=g.stop_audio_token, seed=i, seq_seed=i)
            plain.append((100 + i, text_ids(dims_small, 5 + i % 20, 300 + i), i % 3, sp))
        beams = [(200, text_ids(dims_small, 14, 9), 0, _sp(g, 4, 1.0, mt=48)),
                 (201, text_ids(dims_small, 7, 8), 1, _sp(g, 4, 0.0, mt=48, do_sample=True, seed=4))]
        alone = eng.run_batch(plain, timeout_s=600, want_latents=True)
        runs = []
        for graphs, micro in ((1, 2), (0, 2), (1, 1)):
            eng.set_option("cuda_graphs", graphs)
            eng.set_option("microbatches", micro)
            runs.append(eng.run_batch(plain + beams, timeout_s=600, want_latents=True))
        eng.set_option("cuda_graphs", 1)
        eng.set_option("microbatches", 2)
        for sid, (_, t, w, l) in alone.items():
            _, t2, w2, l2 = runs[0][sid]
            assert np.array_equal(t, t2) and np.array_equal(w, w2) and np.array_equal(l, l2), sid
        for sid, _, _, _ in beams:
            _, t0, w0, l0 = runs[0][sid]
            for run in runs[1:]:
                _, t1, w1, l1 = run[sid]
                assert np.array_equal(t0, t1) and np.array_equal(w0, w1) and np.array_equal(l0, l1), sid
    finally:
        eng.close()


def test_cancel_returns_group_slots_and_pages(engine_full, dims_full):
    """a group cancelled mid-decode ends with XTTS_ERR_CANCELLED and gives back all of its slots and pages: afterwards
    max_batch / B groups are admitted in one wave (same first-token time) and complete"""
    g = dims_full.gpt
    ids = text_ids(dims_full, 20, 5)
    eng = engine_full
    steps0 = eng.stats().decode_steps
    eng.submit(300, ids, 0, _sp(g, 4, mt=400, stop_token=-1))
    t_end = time.time() + 60
    while eng.stats().decode_steps < steps0 + 3 and time.time() < t_end:
        time.sleep(0.002)
    eng.cancel(300)
    r = None
    while r is None:
        r = eng.poll(1000)
    assert r.seq_id == 300 and r.status == ERR_CANCELLED
    eng.fetch(r, False, False)
    for nb in (4, 2):
        jobs = [(400 + nb * 10 + k, text_ids(dims_full, 10 + k, k), k % 2, _sp(g, nb, mt=12)) for k in range(4 // nb)]
        res = eng.run_batch(jobs, timeout_s=300)
        assert sorted(res) == sorted(j[0] for j in jobs)
        assert all(r.status == 0 and r.n_tokens > 0 for r, _, _, _ in res.values())
        assert len({r.t_first_token for r, _, _, _ in res.values()}) == 1


def test_beam_search_fp16_full_geometry(engine_full_fp16, dims_full, state_full, speakers_full):
    """fp16 at full geometry, B = 4: the oracle's teacher-forced score of the returned hypothesis is within tolerance of
    the oracle's own best beam-search hypothesis"""
    g = dims_full.gpt
    ids = text_ids(dims_full, 12, 21)
    sp = _sp(g, 4, 1.0, mt=16)
    _, toks, _, _ = engine_full_fp16.run_batch([(500, ids, 0, sp)], timeout_s=300)[500]
    ref, step = _oracle(dims_full, state_full, speakers_full, 0, ids, sp)
    got = step.score(speakers_full[0][0], ids, list(toks), O.prompt_seen_set(g), sp.repetition_penalty, sp.length_penalty)
    assert len(toks) >= 1 and abs(got - ref.score) <= 0.02 * abs(ref.score) + 0.05, (got, ref.score, list(toks), ref.tokens)


def test_generate_speech_with_beams(tmp_path_factory, dims_small, state_small):
    """the public path: generate_speech(num_beams=4, do_sample=False) is reproducible, and stream=True delivers the same
    audio as whole chunks, one per text chunk"""
    from auralis_b200 import TTS, TTSRequest
    from auralis_b200.weights import save_model_dir
    from test_gpu_api import TEXT, _wav_bytes
    d = tmp_path_factory.mktemp("beam_model")
    save_model_dir(str(d), dims_small, state_small[0], state_small[1])
    tts = TTS(scheduler_max_concurrency=16).from_pretrained(str(d), precision="fp32", max_concurrency=8)
    try:
        spk = _wav_bytes(2.5, 150.0, 4)
        req = lambda **kw: TTSRequest(text=TEXT, speaker_files=spk, language="en", num_beams=4, do_sample=False, seed=1, **kw)
        a = tts.generate_speech(req())
        b = tts.generate_speech(req())
        assert a.array.size > 0 and np.array_equal(a.array, b.array)
        n_chunks = len(tts.tts_engine.prepare_text_tokens(TEXT, "en"))
        chunks = list(tts.generate_speech(req(stream=True)))
        assert len(chunks) == n_chunks >= 2
        assert np.array_equal(np.concatenate([c.array for c in chunks]), a.array)
    finally:
        tts.loop.run_until_complete(tts.shutdown())
