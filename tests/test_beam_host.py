"""CPU: the beam-search oracle (oracle/beam_oracle.py) pinned to transformers' own beam search, its warper chain, the
law of its Exp(1)-race draws, and TTSRequest.num_beams."""
import itertools

import numpy as np
import pytest
import torch

from oracle import beam_oracle as BO
from auralis_b200.requests import TTSRequest

transformers = pytest.importorskip("transformers")

V_HF = 48
START, STOP = V_HF - 2, V_HF - 1


def _tiny_model(seed: int):
    torch.manual_seed(seed)
    cfg = transformers.GPT2Config(vocab_size=V_HF, n_positions=128, n_embd=32, n_layer=2, n_head=2,
                                  bos_token_id=START, eos_token_id=STOP)
    m = transformers.GPT2LMHeadModel(cfg).double().eval()
    with torch.no_grad():                        # spread the logits so that beams stop early in some cases
        m.lm_head.weight.mul_(8.0)
    return m


def _prompt(n_text: int):
    return torch.tensor([1] * (32 + n_text) + [START])    # XTTS-shaped: [1] * (32 + Lt) + [start]


CASES = [(b, lp, pen, seed) for b, lp, pen in itertools.product([2, 3, 4, 8], [0.0, 1.0, 2.0], [1.0, 5.0])
         for seed in (0,)]


@pytest.mark.parametrize("num_beams,length_penalty,penalty,seed", CASES)
def test_oracle_equals_transformers_beam_search(num_beams, length_penalty, penalty, seed):
    m = _tiny_model(seed + num_beams)
    prompt = _prompt(3)
    max_new = 12
    out = m.generate(prompt[None], num_beams=num_beams, do_sample=False, max_new_tokens=max_new, eos_token_id=STOP,
                     pad_token_id=STOP, length_penalty=length_penalty, repetition_penalty=penalty, early_stopping=False,
                     num_return_sequences=1, return_dict_in_generate=True, output_scores=True)
    first, step = BO.hf_step(m, prompt)
    r = BO.beam_search(step, first(), set(prompt.tolist()), num_beams, max_new, STOP, penalty=penalty,
                       length_penalty=length_penalty)
    got = out.sequences[0, prompt.shape[0]:].tolist()
    n = len(r.tokens)
    assert got[:n] == r.tokens
    assert all(t == STOP for t in got[n:])            # padding after an early stop
    assert np.float32(out.sequences_scores[0].item()) == np.float32(r.score)


def test_pin_covers_early_stop_and_max_length():
    """the parametrized pin has cases that end on the stop token before max_new_tokens and cases that reach it"""
    ended_early = reached_max = 0
    for b, lp, pen, seed in CASES:
        m = _tiny_model(seed + b)
        prompt = _prompt(3)
        first, step = BO.hf_step(m, prompt)
        r = BO.beam_search(step, first(), set(prompt.tolist()), b, 12, STOP, penalty=pen, length_penalty=lp)
        if r.tokens[-1] == STOP and len(r.tokens) < 12:
            ended_early += 1
        if len(r.tokens) == 12:
            reached_max += 1
    assert ended_early > 0 and reached_max > 0, (ended_early, reached_max)


@pytest.mark.parametrize("temperature,top_k,top_p", [(0.75, 50, 0.85), (1.3, 5, 1.0), (0.5, 0, 0.6), (1.0, 1, 0.3)])
def test_warper_chain_matches_transformers_processors(temperature, top_k, top_p):
    from transformers.generation.logits_process import (LogitsProcessorList, RepetitionPenaltyLogitsProcessor,
                                                        TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper)
    g = torch.Generator().manual_seed(3)
    B, V = 4, 1026
    logits = torch.randn(B, V, generator=g) * 4
    ids = torch.randint(0, V, (B, 40), generator=g)
    procs = LogitsProcessorList([RepetitionPenaltyLogitsProcessor(5.0)])
    if temperature != 1.0:
        procs.append(TemperatureLogitsWarper(temperature))
    if top_k > 0:
        procs.append(TopKLogitsWarper(top_k, min_tokens_to_keep=2))
    if top_p < 1.0:
        procs.append(TopPLogitsWarper(top_p, min_tokens_to_keep=2))
    want = procs(ids, torch.log_softmax(logits, dim=-1))
    got = BO.process(logits, [set(r.tolist()) for r in ids], 5.0, True, temperature, top_k, top_p)
    assert torch.equal(torch.isinf(got), torch.isinf(want))
    fin = ~torch.isinf(want)
    assert torch.equal(got[fin], want[fin])


def test_exp_race_draw_law():
    """K candidates by the Exp(1) race follow sampling without replacement: over 4000 Philox streams, the frequency of
    every ordered 2-subset of a 4-way distribution is within 4.5 standard errors of its probability"""
    p = np.array([0.4, 0.3, 0.2, 0.1])
    acc = torch.log(torch.tensor(p, dtype=torch.float32))[None]
    n = 4000
    counts = {}
    for s in range(n):
        keys = BO.race_keys(acc, seed=12345, seq_seed=s, step=7)
        o = tuple(torch.sort(keys, descending=True, stable=True)[1][:2].tolist())
        counts[o] = counts.get(o, 0) + 1
    for i, j in itertools.permutations(range(4), 2):
        q = p[i] * p[j] / (1 - p[i])
        f = counts.get((i, j), 0) / n
        assert abs(f - q) <= 4.5 * np.sqrt(q * (1 - q) / n), ((i, j), f, q)


def test_request_num_beams():
    r = TTSRequest(text="hello", speaker_files=["a.wav"], language="en")
    assert r.num_beams == 1
    r = TTSRequest(text="hello", speaker_files=["a.wav"], language="en", num_beams=4, do_sample=False, length_penalty=2.0)
    c = r.copy()
    assert (c.num_beams, c.do_sample, c.length_penalty) == (4, False, 2.0)
    for bad in (0, 9, -1, 2.0, "2", True, None):
        with pytest.raises(ValueError):
            TTSRequest(text="hello", speaker_files=["a.wav"], language="en", num_beams=bad)
