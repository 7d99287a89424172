"""TEST INFRASTRUCTURE — CPU oracle for the XTTSv2 hot path (fp32, torch-CPU ops).

This file is the checker, never the product: only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs import it.  The shipped path (``auralis_b200``) is CUDA-only and never calls it.

Parity pin status
-----------------
* Vocoder, conditioning encoder, perceiver, mel front-end, speaker encoder: the
  restatements below are checked bit-for-bit (or to 1e-5) against the reference's
  OWN modules imported unmodified from /root/reference (``oracle/ref_import.py``)
  by ``tests/test_oracle_vs_reference.py`` (container only) and against the golden
  vectors those modules produced (``tests/golden/*.npz``, generator
  ``tests/golden/make_golden.py``) everywhere else.  -> pinned to reference outputs.
  The reference-audio chunking around them (``XTTSv2Engine.get_gpt_cond_latents``: truncation, pieces, the 0.33 s drop,
  the mean) and the repetition penaliser (``LogitsRepetitionPenalizer``) are the reference's own code inside modules
  that import vLLM 0.6.4: those two are lifted BY SOURCE and executed as written against the restatement
  (``tests/test_oracle_vs_reference.py``, ``tests/test_oracle_gpt.py``).
* GPT block arithmetic + sampler live in third-party vLLM 0.6.4.post1
  (requirements.txt:31), not vendored under /root/reference and not installable here
  (SURVEY.md §8c).  They are restated from the reference's call sites and checked
  against HF ``transformers.GPT2Model`` (same arithmetic: Conv1D, gelu_new, pre-LN)
  in ``tests/test_oracle_gpt.py``; the top-k / top-p mask is additionally compared (ties included) with
  ``apply_top_k_top_p_pytorch`` lifted by source from the vLLM that IS installed (0.22, v1 sampler — same
  published algorithm, different version).  The reference holds no golden vector for this
  path (SURVEY.md §4) -> **parity unpinned** for the GPT/sampler beyond that.

Every function cites the reference lines it restates.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

State = Dict[str, torch.Tensor]

# =============================================================================================
# GPT-2 acoustic model
# =============================================================================================


def gelu_new(x: torch.Tensor) -> torch.Tensor:
    """tanh GELU ("gelu_new", checkpoint_converter.py:197; vLLM get_act_fn)."""
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x * x * x)))


def layer_norm(x, w, b, eps=1e-5):
    return F.layer_norm(x, (x.shape[-1],), w, b, eps)


@dataclass
class SamplingParams:
    """Per-chunk sampling knobs exactly as the engine builds them (XTTSv2.py:726-739)."""
    temperature: float = 0.75
    top_p: float = 0.85
    top_k: int = 50
    repetition_penalty: float = 5.0
    max_tokens: int = 605
    stop_token: int = 1025
    seed: int = 0


class GPTOracle:
    """fp32 restatement of XttsGPT (vllm_mm_gpt.py:341-733) + GPT2Model (:735-849) + the vLLM
    GPT2Block it instantiates (third-party; structure per SURVEY.md §8c)."""

    def __init__(self, gpt_state: State, core_state: State, dims):
        self.g = dims.gpt
        self.w = gpt_state
        self.text_emb = core_state["text_embedding.weight"]
        self.text_pos = core_state["text_pos_embedding.emb.weight"]
        # engine-side final_norm (XTTSv2.py:137,687) == GPT-side final_norm weights
        self.fn_w = core_state["final_norm.weight"]
        self.fn_b = core_state["final_norm.bias"]

    # ---- prompt construction: XTTSv2.py:519-528, :345 ; vllm_mm_gpt.py:806-813,778-783 (SURVEY A.2)
    def prompt_rows(self, cond_latents: torch.Tensor, text_ids: Sequence[int]) -> torch.Tensor:
        """cond_latents [32,H]; text_ids = [bos]+bpe+[eos] already. Returns [P,H], P = 32+Lt+1."""
        ids = torch.as_tensor(list(text_ids), dtype=torch.long)
        temb = self.text_emb[ids] + self.text_pos[torch.arange(len(ids))]
        bos = self.w["gpt.wte.weight"][self.g.start_audio_token] + self.w["gpt.wpe.emb.weight"][0]
        return torch.cat([cond_latents, temb, bos[None]], dim=0)

    def audio_row(self, token: int, k: int) -> torch.Tensor:
        """decode step k input: wte[t_k] + wpe[k] (vllm_mm_gpt.py:480, :815-825)."""
        return self.w["gpt.wte.weight"][token] + self.w["gpt.wpe.emb.weight"][k]

    # ---- one block on rows [n,H] attending to (cached ++ own) keys, causal
    def _block(self, i: int, x: torch.Tensor, kc: Optional[torch.Tensor], vc: Optional[torch.Tensor]):
        g, w = self.g, self.w
        p = f"gpt.h.{i}."
        H, nh, hd = g.hidden, g.heads, g.head_dim
        h = layer_norm(x, w[p + "ln_1.weight"], w[p + "ln_1.bias"], g.ln_eps)
        qkv = h @ w[p + "attn.c_attn.weight"] + w[p + "attn.c_attn.bias"]
        q, k, v = qkv.split(H, dim=-1)
        n = x.shape[0]
        q = q.view(n, nh, hd).transpose(0, 1)
        k = k.view(n, nh, hd).transpose(0, 1)
        v = v.view(n, nh, hd).transpose(0, 1)
        if kc is not None:
            k_all = torch.cat([kc, k], dim=1)
            v_all = torch.cat([vc, v], dim=1)
        else:
            k_all, v_all = k, v
        past = k_all.shape[1] - n
        s = (q @ k_all.transpose(1, 2)) * (hd ** -0.5)
        mask = torch.arange(k_all.shape[1])[None, :] > (torch.arange(n)[:, None] + past)
        s = s.masked_fill(mask[None], float("-inf"))
        a = torch.softmax(s, dim=-1) @ v_all
        a = a.transpose(0, 1).reshape(n, H)
        x = x + a @ w[p + "attn.c_proj.weight"] + w[p + "attn.c_proj.bias"]
        h = layer_norm(x, w[p + "ln_2.weight"], w[p + "ln_2.bias"], g.ln_eps)
        h = gelu_new(h @ w[p + "mlp.c_fc.weight"] + w[p + "mlp.c_fc.bias"])
        x = x + h @ w[p + "mlp.c_proj.weight"] + w[p + "mlp.c_proj.bias"]
        return x, k_all, v_all

    def forward_rows(self, rows: torch.Tensor, cache=None):
        """rows [n,H] appended to cache; returns (ln_f(h) [n,H], new cache). vllm_mm_gpt.py:839-849."""
        x = rows
        new = []
        for i in range(self.g.layers):
            kc, vc = (cache[i] if cache is not None else (None, None))
            x, k, v = self._block(i, x, kc, vc)
            new.append((k, v))
        x = layer_norm(x, self.w["gpt.ln_f.weight"], self.w["gpt.ln_f.bias"], self.g.ln_eps)
        return x, new

    def head(self, h_lnf: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """compute_logits (vllm_mm_gpt.py:664-688): y = final_norm(ln_f(h)); logits = mel_head(y)+b.
        Also returns the vocoder latent final_norm(y) (XTTSv2.py:687, SURVEY A.4 / App. B.2)."""
        y = layer_norm(h_lnf, self.w["final_norm.weight"], self.w["final_norm.bias"], self.g.ln_eps)
        logits = y @ self.w["mel_head.weight"].t() + self.w["mel_head.bias"]
        lat = layer_norm(y, self.fn_w, self.fn_b, self.g.ln_eps)
        return logits, lat

    @torch.no_grad()
    def generate(self, cond_latents: torch.Tensor, text_ids: Sequence[int], sp: SamplingParams,
                 seq_seed: int = 0, return_logits: bool = False):
        """Free-running decode of one chunk.  Returns (token_ids incl. stop token, latents [n,H]).
        Loop semantics: SURVEY A.2 step 5 / A.4 (stop on 1025 or max_tokens; ids include the stop
        token; latent rows are those fed by bos, t_1..t_{n-1})."""
        rows = self.prompt_rows(cond_latents, text_ids)
        h, cache = self.forward_rows(rows)
        seen = prompt_seen_set(self.g)
        toks: List[int] = []
        lats = []
        all_logits = []
        h_last = h[-1:]
        for k in range(1, sp.max_tokens + 1):
            logits, lat = self.head(h_last)
            lats.append(lat[0])
            z = logits[0].clone()
            if return_logits:
                all_logits.append(z.clone())
            tok = sample_token(z, seen, sp, seq_seed, k - 1)
            toks.append(tok)
            seen.add(tok)
            if tok == sp.stop_token or k == sp.max_tokens:
                break
            h_last, cache = self.forward_rows(self.audio_row(tok, k)[None], cache)
        out = (toks, torch.stack(lats))
        if return_logits:
            out = out + (torch.stack(all_logits),)
        return out

    @torch.no_grad()
    def generate_batched(self, cond_latents: Sequence[torch.Tensor], text_ids: Sequence[Sequence[int]], sp: SamplingParams,
                         fast_rng: bool = False, return_logits: bool = False):
        """The same decode for B chunks AT ONCE — what a CPU deployment of the reference would do (vLLM batches the
        decode; a B = 1 loop streams the 1.5 GB of fp32 weights once per token instead of once per B tokens).  Prompts are
        prefilled one by one (`forward_rows`), their K/V copied into a left-aligned padded cache [B, heads, L, 64]; every
        decode step is one pass over all still-running rows.  Arithmetic per row == `generate` (tests/test_oracle_gpt.py).
        fast_rng: Exp(1) noise from torch's generator instead of the Philox stream shared with the CUDA sampler (the
        reference itself is unseeded) — used by bench.py's CPU arm so the timing is not dominated by a Python RNG."""
        g, w = self.g, self.w
        B, H, nh, hd, L = len(text_ids), self.g.hidden, self.g.heads, self.g.head_dim, self.g.layers
        lens, h_last = [], []
        P = [g.n_cond_latents + len(t) + 1 for t in text_ids]
        cap = max(P) + sp.max_tokens
        K = [torch.zeros(B, nh, cap, hd) for _ in range(L)]
        V = [torch.zeros(B, nh, cap, hd) for _ in range(L)]
        for b in range(B):
            h, cache = self.forward_rows(self.prompt_rows(cond_latents[b], text_ids[b]))
            for i in range(L):
                K[i][b, :, :P[b]] = cache[i][0]
                V[i][b, :, :P[b]] = cache[i][1]
            h_last.append(h[-1])
        x_lnf = torch.stack(h_last)                                    # [B,H] ln_f output of the last prompt row
        ctx = torch.tensor(P)                                          # cached positions per row
        seen = [prompt_seen_set(g) for _ in range(B)]
        toks: List[List[int]] = [[] for _ in range(B)]
        lats: List[List[torch.Tensor]] = [[] for _ in range(B)]
        all_logits: List[List[torch.Tensor]] = [[] for _ in range(B)]
        alive = list(range(B))
        gen = torch.Generator().manual_seed(sp.seed) if fast_rng else None
        wte, wpe = w["gpt.wte.weight"], w["gpt.wpe.emb.weight"]
        for k in range(1, sp.max_tokens + 1):
            logits, lat = self.head(x_lnf)
            nxt, keep = [], []
            for j, b in enumerate(alive):
                lats[b].append(lat[j])
                z = logits[j].clone()
                if return_logits:
                    all_logits[b].append(z.clone())
                if fast_rng and sp.temperature >= _SAMPLING_EPS:
                    z = apply_repetition_penalty(z.float(), seen[b], sp.repetition_penalty) / sp.temperature
                    p = torch.softmax(topk_topp_mask(z, sp.top_k, sp.top_p), dim=-1)
                    tok = int(torch.argmax(p / torch.empty_like(p).exponential_(generator=gen)))
                else:
                    tok = sample_token(z, seen[b], sp, b, k - 1)
                toks[b].append(tok)
                seen[b].add(tok)
                if not (tok == sp.stop_token or k == sp.max_tokens):
                    nxt.append(tok); keep.append(j)
            if not keep:
                break
            alive = [alive[j] for j in keep]
            rows = torch.tensor(alive)
            x = wte[torch.tensor(nxt)] + wpe[k]                        # [M,H] decode inputs of the running rows
            pos = ctx[rows]                                            # where this step's K/V go
            M = len(alive)
            ar = torch.arange(M)
            Lmax = int(pos.max()) + 1
            mask = torch.arange(Lmax)[None, :] > pos[:, None]          # [M,Lmax] True = not visible
            for i in range(L):
                pfx = f"gpt.h.{i}."
                hN = layer_norm(x, w[pfx + "ln_1.weight"], w[pfx + "ln_1.bias"], g.ln_eps)
                qkv = hN @ w[pfx + "attn.c_attn.weight"] + w[pfx + "attn.c_attn.bias"]
                q, kk, vv = qkv.split(H, dim=-1)
                K[i][rows, :, pos] = kk.view(M, nh, hd)
                V[i][rows, :, pos] = vv.view(M, nh, hd)
                Kr, Vr = K[i][rows, :, :Lmax], V[i][rows, :, :Lmax]    # [M,nh,Lmax,hd]
                sc = torch.einsum("mhd,mhld->mhl", q.view(M, nh, hd), Kr) * (hd ** -0.5)
                sc = sc.masked_fill(mask[:, None, :], float("-inf"))
                a = torch.einsum("mhl,mhld->mhd", torch.softmax(sc, dim=-1), Vr).reshape(M, H)
                x = x + a @ w[pfx + "attn.c_proj.weight"] + w[pfx + "attn.c_proj.bias"]
                hN = layer_norm(x, w[pfx + "ln_2.weight"], w[pfx + "ln_2.bias"], g.ln_eps)
                hN = gelu_new(hN @ w[pfx + "mlp.c_fc.weight"] + w[pfx + "mlp.c_fc.bias"])
                x = x + hN @ w[pfx + "mlp.c_proj.weight"] + w[pfx + "mlp.c_proj.bias"]
            ctx[rows] = pos + 1
            x_lnf = layer_norm(x, w["gpt.ln_f.weight"], w["gpt.ln_f.bias"], g.ln_eps)
            del ar
        out = (toks, [torch.stack(l) for l in lats])
        if return_logits:
            out = out + ([torch.stack(l) for l in all_logits],)
        return out

    @torch.no_grad()
    def teacher_forced(self, cond_latents, text_ids, tokens: Sequence[int]):
        """The reference's 2nd pass (XTTSv2.py:617-687) without the 4 causally-irrelevant EOS rows:
        one prefill over [prefix ; bos ; t_1..t_{n-1}] -> (raw logits [n,V], latents [n,H])."""
        rows = [self.prompt_rows(cond_latents, text_ids)]
        for k, t in enumerate(tokens[:-1], start=1):
            rows.append(self.audio_row(int(t), k)[None])
        h, _ = self.forward_rows(torch.cat(rows, 0))
        n = len(tokens)
        h_a = h[-n:]
        return self.head(h_a)


def prompt_seen_set(g) -> set:
    """Penalty set seed: prompt ids are [1]*(32+Lt)+[start] (vllm_mm_gpt.py:325) -> {1, 1024}."""
    return {1, g.start_audio_token}


# ---------------------------------------------------------------------------------------------
# sampler: LogitsRepetitionPenalizer (hijack.py:49-88) then vLLM Sampler (SURVEY A.3)
# ---------------------------------------------------------------------------------------------
_SAMPLING_EPS = 1e-5


def apply_repetition_penalty(z: torch.Tensor, seen, penalty: float) -> torch.Tensor:
    """hijack.py:67-86 — applied once per unique id (index-assign semantics)."""
    if penalty == 1.0 or not seen:
        return z
    idx = torch.as_tensor(sorted(seen), dtype=torch.long)
    r = z[idx]
    z[idx] = torch.where(r > 0, r / penalty, r * penalty)
    return z


def topk_topp_mask(z: torch.Tensor, top_k: int, top_p: float) -> torch.Tensor:
    """vLLM _apply_top_k_top_p: ascending sort; top-k keeps >= k-th largest (ties kept);
    top-p drops entries whose ascending cumulative softmax <= 1-p, last always kept.
    Returns masked logits (dropped = -inf) in original order."""
    V = z.shape[0]
    srt, idx = torch.sort(z, descending=False, stable=True)
    if 0 < top_k < V:
        kth = srt[V - top_k]
        srt = srt.masked_fill(srt < kth, float("-inf"))
    if top_p < 1.0:
        probs = torch.softmax(srt, dim=-1)
        cs = torch.cumsum(probs, dim=-1)
        thr = float(np.float32(1.0) - np.float32(top_p))      # fp32 threshold, as the kernel computes it
        m = cs <= thr
        m[-1] = False
        srt = srt.masked_fill(m, float("-inf"))
    out = torch.empty_like(z)
    out[idx] = srt
    return out


def philox4x32(counter: Sequence[int], key: Sequence[int]) -> np.ndarray:
    """Philox-4x32-10 (Salmon et al. 2011), the counter RNG the CUDA sampler uses so that seeded
    sampling is reproducible token-for-token between oracle and kernel.  (The reference is
    unseeded — vLLM's q.exponential_() — so only the distribution is a reference property.)"""
    M0, M1 = 0xD2511F53, 0xCD9E8D57
    W0, W1 = 0x9E3779B9, 0xBB67AE85
    c = [int(x) & 0xFFFFFFFF for x in counter]
    k = [int(x) & 0xFFFFFFFF for x in key]
    for _ in range(10):
        p0 = M0 * c[0]
        p1 = M1 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k[0]) & 0xFFFFFFFF, p1 & 0xFFFFFFFF,
             ((p0 >> 32) ^ c[3] ^ k[1]) & 0xFFFFFFFF, p0 & 0xFFFFFFFF]
        k = [(k[0] + W0) & 0xFFFFFFFF, (k[1] + W1) & 0xFFFFFFFF]
    return np.array(c, dtype=np.uint32)


def exp_noise(seed: int, seq_seed: int, step: int, V: int) -> np.ndarray:
    """Exp(1) variate per vocabulary entry: e = -log(u), u = ((r >> 9) + 0.5) * 2^-23 — a 23-bit
    uniform that is exact in fp32 and never rounds to 0 or 1.
    counter = (v/4, step, seq_seed, 0), key = (seed lo, seed hi)."""
    out = np.empty(((V + 3) // 4) * 4, dtype=np.float32)
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    for blk in range((V + 3) // 4):
        r = philox4x32((blk, step, seq_seed, 0), key)
        u = ((r >> np.uint32(9)).astype(np.float32) + np.float32(0.5)) * np.float32(1.0 / 8388608.0)
        out[blk * 4: blk * 4 + 4] = (-np.log(u)).astype(np.float32)
    return out[:V]


def sample_token(z: torch.Tensor, seen, sp: SamplingParams, seq_seed: int, step: int) -> int:
    """penalty -> (greedy | /T -> top-k -> top-p -> softmax -> argmax(p / Exp(1)))."""
    z = apply_repetition_penalty(z.float(), seen, sp.repetition_penalty)
    if sp.temperature < _SAMPLING_EPS:
        return int(torch.argmax(z))
    z = z / sp.temperature
    z = topk_topp_mask(z, sp.top_k, sp.top_p)
    p = torch.softmax(z, dim=-1)
    e = torch.from_numpy(exp_noise(sp.seed, seq_seed, step, z.shape[0]))
    return int(torch.argmax(p / e))


# =============================================================================================
# HiFi-GAN vocoder  (hifigan_decoder.py:228-260, 776-802; SURVEY A.5)
# =============================================================================================

def fold_weight_norm(g: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """torch weight_norm(dim=0): w = g * v / ||v||, norm over all dims but 0."""
    n = v.reshape(v.shape[0], -1).norm(dim=1).reshape(g.shape)
    return v * (g / n)


def _wn(core: State, prefix: str) -> torch.Tensor:
    if prefix + ".weight" in core:
        return core[prefix + ".weight"]
    return fold_weight_norm(core[prefix + ".parametrizations.weight.original0"],
                            core[prefix + ".parametrizations.weight.original1"])


def interp_latents(latents: torch.Tensor, vd) -> torch.Tensor:
    """[T,C] -> z [C,T'] : two linear interpolations, align_corners=False (hifigan_decoder.py:787-800)."""
    z = F.interpolate(latents.t()[None], scale_factor=vd.code_stride / vd.output_hop_length,
                      mode="linear", align_corners=False)
    if vd.output_sample_rate != vd.input_sample_rate:
        z = F.interpolate(z, scale_factor=vd.output_sample_rate / vd.input_sample_rate,
                          mode="linear", align_corners=False)
    return z[0]


@torch.no_grad()
def vocoder(latents: torch.Tensor, g: torch.Tensor, core: State, dims, return_stages: bool = False):
    """latents [T,in_dim] fp32, g [d_vector] -> wav [256*T'] fp32.  fp32 throughout (the reference's
    autocast is a no-op on CPU, SURVEY §0.5)."""
    vd = dims.voc
    p = "hifigan_decoder.waveform_decoder."
    gg = g.reshape(1, -1, 1)
    z = interp_latents(latents, vd)[None]
    stages = {"z": z[0]}
    x = F.conv1d(z, core[p + "conv_pre.weight"], core[p + "conv_pre.bias"], padding=3)
    x = x + F.conv1d(gg, core[p + "cond_layer.weight"], core[p + "cond_layer.bias"])
    stages["pre"] = x[0]
    nk = len(vd.rb_kernels)
    for i, (u, k) in enumerate(zip(vd.up_rates, vd.up_kernels)):
        x = F.leaky_relu(x, 0.1)
        x = F.conv_transpose1d(x, _wn(core, p + f"ups.{i}"), core[p + f"ups.{i}.bias"],
                               stride=u, padding=(k - u) // 2)
        x = x + F.conv1d(gg, core[p + f"conds.{i}.weight"], core[p + f"conds.{i}.bias"])
        stages[f"up{i}"] = x[0]
        zs = None
        for j, kk in enumerate(vd.rb_kernels):
            r = x
            rb = p + f"resblocks.{i * nk + j}."
            for t, d in enumerate(vd.rb_dilations):
                xt = F.leaky_relu(r, 0.1)
                xt = F.conv1d(xt, _wn(core, rb + f"convs1.{t}"), core[rb + f"convs1.{t}.bias"],
                              dilation=d, padding=(kk * d - d) // 2)
                xt = F.leaky_relu(xt, 0.1)
                xt = F.conv1d(xt, _wn(core, rb + f"convs2.{t}"), core[rb + f"convs2.{t}.bias"],
                              padding=(kk - 1) // 2)
                r = xt + r
            zs = r if zs is None else zs + r
        x = zs / nk
        stages[f"mrf{i}"] = x[0]
    x = F.leaky_relu(x, 0.01)          # default slope (hifigan_decoder.py:257; App. B.3)
    x = F.conv1d(x, core[p + "conv_post.weight"], None, padding=3)
    x = torch.tanh(x)
    wav = x.reshape(-1)
    return (wav, stages) if return_stages else wav


# =============================================================================================
# Conditioning: mel -> ConditioningEncoder -> Perceiver ; speaker d-vector  (SURVEY A.7)
# =============================================================================================

def mel_cloning(wav: torch.Tensor, mel_stats: torch.Tensor, n_mels: int = 80) -> torch.Tensor:
    """wav [N] @22.05k -> [n_mels, frames]: torchaudio MelSpectrogram(n_fft 2048, hop 256, win 1024,
    power 2, slaney norm, htk scale, f 0..8000, center/reflect) -> log(clamp 1e-5)/mel_stats
    (common/utilities.py:53-70 with the args of XTTSv2.py:374-386)."""
    from auralis_b200.weights import mel_filterbank
    n_fft, hop, win = 2048, 256, 1024
    window = torch.hann_window(win, dtype=wav.dtype)
    spec = torch.stft(wav, n_fft, hop, win, window=window, center=True, pad_mode="reflect",
                      normalized=False, onesided=True, return_complex=True)
    power = spec.real ** 2 + spec.imag ** 2                   # [1025, frames]
    fb = mel_filterbank(n_fft // 2 + 1, 0.0, 8000.0, n_mels, 22050, "slaney").to(wav.dtype)  # [1025, n_mels]
    mel = (power.t() @ fb).t()
    mel = torch.log(torch.clamp(mel, min=1e-5))
    return mel / mel_stats.to(wav.dtype)[:, None]


def cond_encoder(mel: torch.Tensor, core: State, dims) -> torch.Tensor:
    """mel [80,T] -> [H,T]  (latent_encoder.py:242-253 ; AttentionBlock :188-206 ; QKVAttention :101-131)."""
    g, c = dims.gpt, dims.cond
    H, nh = g.hidden, g.heads
    p = "conditioning_encoder."
    h = F.conv1d(mel[None], core[p + "init.weight"], core[p + "init.bias"])
    for i in range(c.cond_blocks):
        q = p + f"attn.{i}."
        groups = _gn_groups(H)
        xn = F.group_norm(h, groups, core[q + "norm.weight"], core[q + "norm.bias"], 1e-5)
        qkv = F.conv1d(xn, core[q + "qkv.weight"], core[q + "qkv.bias"])
        T = qkv.shape[-1]
        ch = H // nh
        qq, kk, vv = qkv.reshape(nh, ch * 3, T).split(ch, dim=1)
        scale = 1.0 / math.sqrt(math.sqrt(ch))
        wgt = torch.einsum("bct,bcs->bts", qq * scale, kk * scale)
        wgt = torch.softmax(wgt.float(), dim=-1)
        a = torch.einsum("bts,bcs->bct", wgt, vv).reshape(1, H, T)
        hh = F.conv1d(a, core[q + "proj_out.weight"], core[q + "proj_out.bias"])
        h = xn + hh           # residual adds the NORMALISED x (latent_encoder.py:199,205-206; App. B.6)
    return h[0]


def _gn_groups(channels: int) -> int:
    """latent_encoder.py:53-72."""
    groups = 32
    if channels <= 16:
        groups = 8
    elif channels <= 64:
        groups = 16
    while channels % groups != 0:
        groups = int(groups / 2)
    return groups


def perceiver(ctx: torch.Tensor, core: State, dims) -> torch.Tensor:
    """ctx [T,H] -> latents [32,H] (perceiver_encoder.py:422-442, Attention :459-485, GEGLU :322-336,
    RMSNorm :262-276)."""
    c = dims.cond
    nh, dh = c.perceiver_heads, c.perceiver_dim_head
    p = "conditioning_perceiver."
    lat = core[p + "latents"]
    for l in range(c.perceiver_depth):
        a = p + f"layers.{l}.0."
        f = p + f"layers.{l}.1."
        kv_in = torch.cat([lat, ctx], dim=0)
        q = lat @ core[a + "to_q.weight"].t()
        kv = kv_in @ core[a + "to_kv.weight"].t()
        k, v = kv.chunk(2, dim=-1)
        n, m = q.shape[0], k.shape[0]
        qh = q.view(n, nh, dh).transpose(0, 1)
        kh = k.view(m, nh, dh).transpose(0, 1)
        vh = v.view(m, nh, dh).transpose(0, 1)
        sim = (qh @ kh.transpose(1, 2)) * (dh ** -0.5)
        o = (sim.softmax(dim=-1) @ vh).transpose(0, 1).reshape(n, nh * dh)
        lat = o @ core[a + "to_out.weight"].t() + lat
        hcat = lat @ core[f + "0.weight"].t() + core[f + "0.bias"]
        xv, gate = hcat.chunk(2, dim=-1)
        hmid = F.gelu(gate) * xv
        lat = hmid @ core[f + "2.weight"].t() + core[f + "2.bias"] + lat
    H = lat.shape[-1]
    return F.normalize(lat, dim=-1) * (H ** 0.5) * core[p + "norm.gamma"]


def gpt_cond_latents(wav22k: torch.Tensor, core: State, dims, length: int = 30, chunk_length: int = 4):
    """XTTSv2.py:349-407: cut to `length` s, 4 s pieces, drop < 0.33 s, mean of per-piece latents -> [32,H]."""
    audio = wav22k[: 22050 * length] if length > 0 else wav22k
    embs = []
    for i in range(0, audio.shape[0], 22050 * chunk_length):
        piece = audio[i: i + 22050 * chunk_length]
        if piece.shape[0] < 22050 * 0.33:
            continue
        mel = mel_cloning(piece, core["mel_stats"], dims.cond.n_mels)
        h = cond_encoder(mel, core, dims)
        embs.append(perceiver(h.t(), core, dims))
    return torch.stack(embs).mean(dim=0)


def speaker_frontend(wav16k: torch.Tensor, core: State) -> torch.Tensor:
    """wav [N] @16k -> InstanceNorm'd log-mel [1, 64, frames] in wav's dtype (hifigan_decoder.py:452-482, 602-613)."""
    s = "hifigan_decoder.speaker_encoder."
    dt = wav16k.dtype
    x = wav16k[None]
    x = F.pad(x[:, None], (1, 0), mode="reflect")
    x = F.conv1d(x, core[s + "torch_spec.0.filter"].to(dt))[:, 0]
    spec = torch.stft(x[0], 512, 160, 400, window=core[s + "torch_spec.1.spectrogram.window"].to(dt),
                      center=True, pad_mode="reflect", normalized=False, onesided=True,
                      return_complex=True)
    power = spec.real ** 2 + spec.imag ** 2                     # [257, frames]
    mel = (power.t() @ core[s + "torch_spec.1.mel_scale.fb"].to(dt)).t()[None]   # [1,64,frames]
    mel = torch.log(mel + 1e-6)
    return F.instance_norm(mel)                                  # nn.InstanceNorm1d(64), no affine


def speaker_embedding(wav16k: torch.Tensor, core: State, dims) -> torch.Tensor:
    """wav [N] @16k -> L2-normalised d-vector [proj]  (hifigan_decoder.py:452-482, 602-646)."""
    c = dims.cond
    s = "hifigan_decoder.speaker_encoder."
    x = speaker_frontend(wav16k, core)[:, None]

    def bn(x, pfx):
        return F.batch_norm(x, core[pfx + ".running_mean"], core[pfx + ".running_var"],
                            core[pfx + ".weight"], core[pfx + ".bias"], False, 0.0, 1e-5)

    x = F.conv2d(x, core[s + "conv1.weight"], core[s + "conv1.bias"], padding=1)
    x = bn(F.relu(x), s + "bn1")
    for li, nb in enumerate(c.spk_layers):
        for b in range(nb):
            p = s + f"layer{li + 1}.{b}."
            stride = 2 if (li > 0 and b == 0) else 1
            r = x
            y = F.conv2d(x, core[p + "conv1.weight"], None, stride=stride, padding=1)
            y = bn(F.relu(y), p + "bn1")
            y = F.conv2d(y, core[p + "conv2.weight"], None, padding=1)
            y = bn(y, p + "bn2")
            se = y.mean(dim=(2, 3))
            se = F.relu(se @ core[p + "se.fc.0.weight"].t() + core[p + "se.fc.0.bias"])
            se = torch.sigmoid(se @ core[p + "se.fc.2.weight"].t() + core[p + "se.fc.2.bias"])
            y = y * se[:, :, None, None]
            if p + "downsample.0.weight" in core:
                r = bn(F.conv2d(r, core[p + "downsample.0.weight"], None, stride=stride), p + "downsample.1")
            x = F.relu(y + r)
    x = x.reshape(1, -1, x.shape[-1])
    a = F.conv1d(x, core[s + "attention.0.weight"], core[s + "attention.0.bias"])
    a = F.batch_norm(F.relu(a), core[s + "attention.2.running_mean"], core[s + "attention.2.running_var"],
                     core[s + "attention.2.weight"], core[s + "attention.2.bias"], False, 0.0, 1e-5)
    a = F.conv1d(a, core[s + "attention.3.weight"], core[s + "attention.3.bias"])
    w = torch.softmax(a, dim=2)
    mu = torch.sum(x * w, dim=2)
    sg = torch.sqrt((torch.sum((x ** 2) * w, dim=2) - mu ** 2).clamp(min=1e-5))
    e = torch.cat((mu, sg), 1) @ core[s + "fc.weight"].t() + core[s + "fc.bias"]
    return F.normalize(e, p=2, dim=1)[0]


# =============================================================================================
# end-to-end chunk (what one `process_tokens_to_speech` yields, XTTSv2.py:762-814)
# =============================================================================================

@torch.no_grad()
def synthesize_chunk(gpt: GPTOracle, core: State, dims, cond_latents, g_vec, text_ids, sp: SamplingParams,
                     seq_seed: int = 0):
    toks, lats = gpt.generate(cond_latents, text_ids, sp, seq_seed)
    wav = vocoder(lats, g_vec, core, dims)
    return toks, lats, wav


def synthetic_reference_wav(seconds: float = 6.0, sr: int = 22050, f0: float = 120.0, seed: int = 7) -> torch.Tensor:
    """SURVEY §8d synthetic speaker reference: 0.3 sin(2π (f0 + 40 sin 2π3t) t) + 0.01 N(0,1)."""
    n = int(seconds * sr)
    t = torch.arange(n, dtype=torch.float64) / sr
    g = torch.Generator().manual_seed(seed)
    x = 0.3 * torch.sin(2 * math.pi * (f0 + 40.0 * torch.sin(2 * math.pi * 3.0 * t)) * t)
    x = x.float() + 0.01 * torch.randn(n, generator=g)
    return x.clamp(-1, 1)
