"""CPU: the oracle restatement against the REFERENCE's own modules on inputs OTHER than tests/golden/{vocoder,conditioning}_*.npz
— ragged lengths, a one-frame chunk, several speakers, reference audio that is cut into more than one conditioning chunk,
prompt construction and the GPT wrapper's embedding splice.  What the reference computed on these inputs is stored in
tests/golden/oracle_live.npz (made by tests/golden/make_oracle_live_golden.py, which imports the reference modules
unmodified through oracle/ref_import.py or lifts their source where the module itself imports vLLM)."""
import os

import numpy as np
import pytest
import torch

from oracle import xtts_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_live.npz")
VOCODER_LENGTHS = [1, 2, 7, 33]
CONDITIONING_CASES = [(0.4, 95.0), (1.3, 180.0)]
SPEAKER_CASES = [(0.35, 110.0), (0.9, 210.0)]
CHUNKING_CASES = [(2.6, 30, 1), (2.6, 2, 1), (1.2, 30, 4), (2.2, 30, 1)]     # 2.2 s / 1 s: last piece 0.2 s is dropped
PROMPT_CASES = [(1, 0), (3, 1)]
PLACEHOLDER_TEXT_LENS = [3, 17]
WRAPPER_IDS = [0, 17, 5, 44, 9, 1]


def WRAPPER_DECODE(g):
    return [(3, 1), (g.start_audio_token - 1, 7), (60, g.max_audio_tokens)]


def vocoder_inputs(dims, T):
    """(latents [T, in_dim], unit d-vector) of two speakers for a chunk of T frames"""
    g = torch.Generator().manual_seed(1000 + T)
    out = []
    for _ in range(2):
        lat = torch.randn(T, dims.voc.in_dim, generator=g)
        gv = torch.nn.functional.normalize(torch.randn(dims.voc.d_vector, generator=g), dim=0)
        out.append((lat, gv))
    return out


def prompt_chunks(dims, n_chunks, seed):
    rng = np.random.RandomState(seed)
    g = dims.gpt
    return [rng.randint(2, g.n_text_tokens, size=int(rng.randint(1, g.max_text_tokens - 1))).tolist() for _ in range(n_chunks)]


@pytest.fixture(scope="module")
def want():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("T", VOCODER_LENGTHS)
def test_vocoder_live(want, dims_small, state_small, T):
    for spk, (lat, gv) in enumerate(vocoder_inputs(dims_small, T)):
        ref = want[f"voc_T{T}_s{spk}"]
        got = O.vocoder(lat, gv, state_small[1], dims_small)
        assert got.shape == ref.shape == (dims_small.voc.n_samples(T),)
        np.testing.assert_allclose(got.numpy(), ref, atol=2e-6, rtol=0)


@pytest.mark.parametrize("seconds,f0", CONDITIONING_CASES)
def test_conditioning_live(want, dims_small, state_small, seconds, f0):
    cs, dims = state_small[1], dims_small
    case = CONDITIONING_CASES.index((seconds, f0))
    wav22 = O.synthetic_reference_wav(seconds, 22050, f0, 21)
    mel = want[f"cond{case}_mel"]
    np.testing.assert_allclose(O.mel_cloning(wav22, cs["mel_stats"], dims.cond.n_mels).numpy(), mel, atol=2e-5, rtol=0)
    got_h = O.cond_encoder(torch.from_numpy(mel), cs, dims)
    np.testing.assert_allclose(got_h.numpy(), want[f"cond{case}_h"], atol=2e-5, rtol=0)
    np.testing.assert_allclose(O.perceiver(got_h.t(), cs, dims).numpy(), want[f"cond{case}_latents"], atol=5e-5, rtol=0)


def test_speaker_encoder_live(want, dims_small, state_small):
    cs, dims = state_small[1], dims_small
    for i, (seconds, f0) in enumerate(SPEAKER_CASES):
        wav16 = O.synthetic_reference_wav(seconds, 16000, f0, 5)
        np.testing.assert_allclose(O.speaker_embedding(wav16, cs, dims).numpy(), want[f"spk{i}"], atol=2e-6, rtol=0)


def test_gpt_cond_latents_chunking_live(want, dims_small, state_small):
    """XTTSv2Engine.get_gpt_cond_latents (XTTSv2.py:349-407) run AS WRITTEN — truncation to `length` seconds, `chunk_length`
    pieces, pieces under 0.33 s dropped, mean over pieces — on the reference's own encoder modules, against the oracle."""
    cs, dims = state_small[1], dims_small
    for i, (seconds, length, chunk) in enumerate(CHUNKING_CASES):
        wav = O.synthetic_reference_wav(seconds, 22050, 140.0, 31)
        got = O.gpt_cond_latents(wav, cs, dims, length=length, chunk_length=chunk)
        ref = want[f"gcl{i}"]
        assert got.shape == ref.shape == (dims.gpt.n_cond_latents, dims.gpt.hidden)
        np.testing.assert_allclose(got.numpy(), ref, atol=5e-5, rtol=0)


def test_prompt_construction_live(want, dims_small, state_small, speakers_small):
    """Rows a1-a2 of the hot path: XTTSv2Engine.prepare_text_tokens_async + _merge_conditioning (XTTSv2.py:506-543,330-347)
    and LearnedPositionEmbeddings (vllm_mm_gpt.py:165-214), executed as written with the synthetic embedding tables, against
    the oracle's prompt rows ([cond latents ; text_emb + text_pos] — the audio-bos row is added by the GPT wrapper,
    vllm_mm_gpt.py:806-813)."""
    gs, cs = state_small
    g = dims_small.gpt
    orc = O.GPTOracle(gs, cs, dims_small)
    cond = speakers_small[0][0]                                        # [32, H]
    for n_chunks, seed in PROMPT_CASES:
        chunks = prompt_chunks(dims_small, n_chunks, seed)
        assert want[f"prompt{n_chunks}_fake_lens"].tolist() == [len(c) + 2 for c in chunks]   # placeholder ids [1]*(L+2) (App. A.2)
        for j, c in enumerate(chunks):
            ids = [0] + c + [1]
            rows = orc.prompt_rows(cond, ids)
            assert rows.shape[0] == g.n_cond_latents + len(ids) + 1
            np.testing.assert_allclose(rows[:-1].numpy(), want[f"prompt{n_chunks}_{j}"], atol=1e-6, rtol=0)


def test_gpt_wrapper_embedding_and_splice_live(want, dims_small, state_small, speakers_small):
    """Row a5: the embedding / conditioning-splice part of the reference's GPT2Model.forward (vllm_mm_gpt.py:768-833) executed
    as written with zero transformer layers: prefill rows = [prefix ; wte[start] + wpe[0]], decode row k = wte[t_k] + wpe[k],
    and a mixed prefill + decode batch — against the oracle's prompt_rows / audio_row."""
    gs, cs = state_small
    g = dims_small.gpt
    orc = O.GPTOracle(gs, cs, dims_small)
    rows = orc.prompt_rows(speakers_small[1][0], WRAPPER_IDS)
    np.testing.assert_allclose(want["wrapper_prefill"], rows.numpy(), atol=1e-6, rtol=0)
    for i, (tok, k) in enumerate(WRAPPER_DECODE(g)):
        np.testing.assert_allclose(want[f"wrapper_decode{i}"], orc.audio_row(tok, k).numpy(), atol=1e-6, rtol=0)
    # one sequence decoding (row first), another one starting in the same step (spliced after it)
    np.testing.assert_allclose(want["wrapper_mixed"], torch.cat([orc.audio_row(9, 4)[None], rows], dim=0).numpy(), atol=1e-6, rtol=0)


def test_placeholder_prompt_and_penalty_seed_live(want, dims_small):
    """Row a3: input_processor_for_xtts2_gpt (vllm_mm_gpt.py:296-334) executed as written — the prompt vLLM sees is
    [1]*(32+Lt) + [start_audio_token], so the repetition penaliser's prompt set is {1, start} (App. B.7), which is what the
    oracle and the CUDA sampler seed their 'seen' set with."""
    g = dims_small.gpt
    for n_text in PLACEHOLDER_TEXT_LENS:
        ids = want[f"placeholder{n_text}"].tolist()
        assert ids == [1] * (g.n_cond_latents + n_text) + [g.start_audio_token]
        assert set(ids) == O.prompt_seen_set(g)
