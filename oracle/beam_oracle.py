"""Beam search as transformers 5.5 runs it (GenerationMixin._beam_search, generation/utils.py:2876-3372) for one batch
item, num_return_sequences 1 and early_stopping unset, over a step function — the restatement the engine's beam kernels
(auralis_b200/csrc/beam.cu) are compared with.

Differences from transformers, both deliberate: ties are broken by the lower flat index beam * V + token (a stable
sort; torch.topk leaves tie order unspecified), and do_sample draws K candidates by an Exp(1) race on the engine's
Philox stream instead of torch.multinomial (same law, different numbers).

Adapters: `hf_step` drives a transformers causal LM (the pin, tests/test_beam_host.py); `GPTStep` drives the fp32
GPTOracle with one incremental KV cache per beam (the GPU comparisons).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, List, Sequence

import numpy as np
import torch

from . import xtts_oracle as O


@dataclass
class BeamResult:
    tokens: List[int]              # the best finished hypothesis, stop token included
    score: float                   # its length-penalised score (transformers' sequences_scores)


def warp(scores: torch.Tensor, temperature: float, top_k: int, top_p: float, min_keep: int = 2) -> torch.Tensor:
    """TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper on [B, V] fp32 scores (logits_process.py)."""
    if temperature != 1.0 and temperature > 0:
        scores = scores / temperature
    if top_k > 0:
        k = min(max(top_k, min_keep), scores.shape[-1])
        kth = torch.topk(scores, k)[0][..., -1, None]
        scores = scores.masked_fill(scores < kth, -float("inf"))
    if top_p < 1.0:
        srt, idx = torch.sort(scores, descending=False)
        cum = srt.softmax(dim=-1).cumsum(dim=-1)
        rm = cum <= (1 - top_p)
        rm[..., -min_keep:] = False
        scores = scores.masked_fill(rm.scatter(1, idx, rm), -float("inf"))
    return scores


def process(logits: torch.Tensor, seen: Sequence[set], penalty: float, do_sample: bool, temperature: float,
            top_k: int, top_p: float) -> torch.Tensor:
    """log_softmax in fp32, repetition penalty over each beam's ids, then (do_sample) the warpers."""
    lp = torch.log_softmax(logits.float(), dim=-1)
    for b, ids in enumerate(seen):
        idx = torch.as_tensor(sorted(ids), dtype=torch.long)
        s = lp[b, idx]
        lp[b, idx] = torch.where(s < 0, s * penalty, s / penalty)
    if do_sample:
        lp = warp(lp, temperature, top_k, top_p)
    return lp


def race_keys(acc: torch.Tensor, seed: int, seq_seed: int, step: int) -> torch.Tensor:
    """Exp(1) race keys p / e over the flat candidates, e from Philox(counter = (f / 4, step, seq_seed, 0))."""
    flat = acc.reshape(-1).float()
    N = flat.shape[0]
    e = torch.from_numpy(O.exp_noise(seed, seq_seed, step, N))
    mx = flat.max()
    ex = torch.where(torch.isinf(flat), torch.zeros_like(flat), torch.exp(flat - mx))
    p = ex / ex.sum()
    return p / e


def beam_search(step: Callable[[List[int], List[int], int], torch.Tensor], first_logits: torch.Tensor, prompt_ids: set,
                num_beams: int, max_new_tokens: int, stop_token: int, penalty: float = 1.0, length_penalty: float = 1.0,
                do_sample: bool = False, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0, seed: int = 0,
                seq_seed: int = 0) -> BeamResult:
    """step(parents, tokens, t) -> logits [B, V] of step t + 1: beam j continues beam parents[j] with tokens[j]."""
    B = num_beams
    K = 2 * B
    V = first_logits.shape[-1]
    f32 = np.float32
    logits = first_logits.reshape(1, V).expand(B, V).clone()
    run = torch.full((B,), -1e9, dtype=torch.float32)
    run[0] = 0.0
    hyps: List[List[int]] = [[] for _ in range(B)]
    fin = [(f32(-1e9), False, None)] * B               # (score, is_sent_finished, tokens)
    unsat = True
    for t in range(max_new_tokens):
        seen = [set(prompt_ids) | set(h) for h in hyps]
        acc = process(logits, seen, penalty, do_sample, temperature, top_k, top_p) + run[:, None]
        flat = acc.reshape(-1)
        keys = race_keys(acc, seed, seq_seed, t) if do_sample else flat
        order = torch.sort(keys, descending=True, stable=True)[1][:K].tolist()
        cs = [f32(flat[f].item()) for f in order]
        cb = [f // V for f in order]
        ct = [f % V for f in order]
        fl = [ct[i] == stop_token or t + 1 >= max_new_tokens for i in range(K)]
        rs = [f32(cs[i] + f32(-1e9)) if fl[i] else cs[i] for i in range(K)]
        pick = sorted(range(K), key=lambda i: (-rs[i], i))[:B]
        den = f32((t + 1) ** length_penalty)
        cand = []
        for i in range(K):
            did = i < B and fl[i]
            s = f32(cs[i] / den)
            if not unsat:
                s = f32(s + f32(-1e9))
            if not did:
                s = f32(s + f32(-1e9))
            cand.append((s, did, hyps[cb[i]] + [ct[i]]))
        merged = fin + cand
        fin = [merged[i] for i in sorted(range(len(merged)), key=lambda i: (-merged[i][0], i))[:B]]
        hyps = [hyps[cb[i]] + [ct[i]] for i in pick]
        run = torch.tensor([rs[i] for i in pick], dtype=torch.float32)
        best_possible = f32(run[0].item() / den)
        worst = min(f[0] for f in fin)
        unsat = unsat and any(best_possible > (worst if f[1] else f32(-1e9)) for f in fin)
        if not (unsat and not all(fl)):
            break
        logits = step([cb[i] for i in pick], [ct[i] for i in pick], t)
    return BeamResult(tokens=list(fin[0][2]), score=float(fin[0][0]))


def hf_step(model, prompt: torch.Tensor):
    """Step function over a transformers causal LM without a cache: beam j's logits from its whole sequence."""
    state = {"seqs": [list(prompt.tolist())]}

    def first():
        with torch.no_grad():
            return model(input_ids=prompt[None]).logits[0, -1].float()

    def step(parents, tokens, t):
        seqs = [state["seqs"][p if len(state["seqs"]) > 1 else 0] + [tok] for p, tok in zip(parents, tokens)]
        state["seqs"] = seqs
        with torch.no_grad():
            return model(input_ids=torch.tensor(seqs)).logits[:, -1].float()

    return first, step


class GPTStep:
    """GPTOracle as a step function: one incremental KV cache per beam, forked from the parent's each step."""

    def __init__(self, orc: O.GPTOracle, cond_latents: torch.Tensor, text_ids: Sequence[int]):
        self.orc = orc
        with torch.no_grad():
            h, cache = orc.forward_rows(orc.prompt_rows(cond_latents, text_ids))
            self.first_logits, _ = orc.head(h[-1:])
        self.first_logits = self.first_logits[0]
        self.caches = [cache]

    def __call__(self, parents, tokens, t):
        out, caches = [], []
        with torch.no_grad():
            for p, tok in zip(parents, tokens):
                h, c = self.orc.forward_rows(self.orc.audio_row(tok, t + 1)[None], self.caches[p])
                lg, _ = self.orc.head(h)
                out.append(lg[0]); caches.append(c)
        self.caches = caches
        return torch.stack(out)

    def score(self, cond_latents, text_ids, tokens: Sequence[int], prompt_ids: set, penalty: float,
              length_penalty: float) -> float:
        """Teacher-forced beam score of one hypothesis: sum of penalised log-probs over gen_len ** length_penalty."""
        lg, _ = self.orc.teacher_forced(cond_latents, text_ids, tokens)
        seen, total = set(prompt_ids), 0.0
        for k, tok in enumerate(tokens):
            lp = process(lg[k:k + 1], [seen], penalty, False, 1.0, 0, 1.0)[0]
            total += float(lp[tok])
            seen.add(int(tok))
        return total / (len(tokens) ** length_penalty)

