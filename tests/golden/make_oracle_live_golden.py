"""Golden outputs of the REFERENCE's own modules (imported unmodified through oracle/ref_import.py, or lifted by source
where the module itself imports vLLM) for tests/test_oracle_vs_reference.py: ragged vocoder lengths, a one-frame chunk,
several speakers, conditioning audio that is cut into more than one chunk, prompt construction and the GPT wrapper's
embedding splice — on the synthetic small-geometry weights (auralis_b200.weights.synth_state, seed 1234).

    python tests/golden/make_oracle_live_golden.py          (needs the reference source tree, see oracle/ref_import.py)
"""
import __future__
import ast
import asyncio
import importlib.util
import logging
import os
import random
import sys
import types
from typing import List, Optional, Tuple, Union

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from auralis_b200.config import XTTSDims  # noqa: E402
from auralis_b200.weights import synth_state  # noqa: E402
from conftest import SEED, _speakers  # noqa: E402
from oracle import ref_import  # noqa: E402
from oracle import xtts_oracle as O  # noqa: E402
from test_oracle_vs_reference import (CHUNKING_CASES, CONDITIONING_CASES, PLACEHOLDER_TEXT_LENS, PROMPT_CASES,  # noqa: E402
                                      SPEAKER_CASES, VOCODER_LENGTHS, WRAPPER_DECODE, WRAPPER_IDS, prompt_chunks, vocoder_inputs)

OUT = os.path.join(HERE, "oracle_live.npz")


def _golden_tools():
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "make_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _lift_methods(path, cls_name, names):
    """Methods of a reference class lifted by source into plain functions (the module itself imports vLLM 0.6.4)."""
    tree = ast.parse(open(path).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls_name)
    fns = [n for n in cls.body if isinstance(n, (ast.FunctionDef, ast.AsyncFunctionDef)) and n.name in names]
    assert len(fns) == len(names)
    return fns


def _cond_modules(ref, cs, dims):
    ce = ref.ConditioningEncoder(dims.cond.n_mels, dims.gpt.hidden, attn_blocks=dims.cond.cond_blocks, num_attn_heads=dims.gpt.heads)
    ce.load_state_dict({k[len("conditioning_encoder."):]: t for k, t in cs.items() if k.startswith("conditioning_encoder.")})
    pr = ref.PerceiverResampler(dim=dims.gpt.hidden, depth=dims.cond.perceiver_depth, dim_context=dims.gpt.hidden,
                                num_latents=dims.gpt.n_cond_latents, dim_head=dims.cond.perceiver_dim_head,
                                heads=dims.cond.perceiver_heads, ff_mult=dims.cond.perceiver_ff_mult, use_flash_attn=False)
    pr.load_state_dict({k[len("conditioning_perceiver."):]: t for k, t in cs.items() if k.startswith("conditioning_perceiver.")})
    return ce, pr


def vocoder(ref, dims, cs, rec):
    hd = _golden_tools().ref_vocoder(ref, dims, cs)
    for T in VOCODER_LENGTHS:
        for spk, (lat, gv) in enumerate(vocoder_inputs(dims, T)):
            with torch.no_grad():
                rec[f"voc_T{T}_s{spk}"] = ref.HifiDecoder.forward(hd, lat[None], g=gv.reshape(1, -1, 1)).reshape(-1).numpy()


def conditioning(ref, dims, cs, rec):
    ce, pr = _cond_modules(ref, cs, dims)
    for i, (seconds, f0) in enumerate(CONDITIONING_CASES):
        wav22 = O.synthetic_reference_wav(seconds, 22050, f0, 21)
        mel = ref.wav_to_mel_cloning(wav22[None], mel_norms=cs["mel_stats"], n_fft=2048, hop_length=256, win_length=1024, power=2,
                                     normalized=False, sample_rate=22050, f_min=0, f_max=8000, n_mels=80)
        with torch.no_grad():
            h = ce(mel)
            lat = pr(h.permute(0, 2, 1))[0]
        rec[f"cond{i}_mel"], rec[f"cond{i}_h"], rec[f"cond{i}_latents"] = mel[0].numpy(), h[0].numpy(), lat.numpy()


def speaker_encoder(ref, dims, cs, rec):
    se = ref.ResNetSpeakerEncoder(input_dim=dims.cond.spk_mels, proj_dim=dims.cond.spk_proj, layers=list(dims.cond.spk_layers),
                                  num_filters=list(dims.cond.spk_filters), log_input=True, use_torch_spec=True,
                                  audio_config={"fft_size": 512, "win_length": 400, "hop_length": 160, "sample_rate": 16000,
                                                "preemphasis": 0.97, "num_mels": 64})
    pre = "hifigan_decoder.speaker_encoder."
    se.load_state_dict({k[len(pre):]: t for k, t in cs.items() if k.startswith(pre)})
    se.eval()
    for i, (seconds, f0) in enumerate(SPEAKER_CASES):
        wav16 = O.synthetic_reference_wav(seconds, 16000, f0, 5)
        with torch.no_grad():
            rec[f"spk{i}"] = se.forward(wav16[None].clone(), l2_norm=True)[0].numpy()


def gpt_cond_latents_chunking(ref, dims, cs, rec):
    import torchaudio
    path = os.path.join(ref_import.REF_SRC, "auralis", "models", "xttsv2", "XTTSv2.py")
    fns = _lift_methods(path, "XTTSv2Engine", ("get_gpt_cond_latents", "get_style_emb"))
    ns = {"torch": torch, "torchaudio": torchaudio, "wav_to_mel_cloning": ref.wav_to_mel_cloning, "Optional": Optional}
    exec(compile(ast.Module(body=fns, type_ignores=[]), path, "exec"), ns)
    ce, pr = _cond_modules(ref, cs, dims)
    me = types.SimpleNamespace(gpt_config=types.SimpleNamespace(use_perceiver_resampler=True), mel_stats=cs["mel_stats"],
                               device=torch.device("cpu"), conditioning_encoder=ce, conditioning_perceiver=pr)
    me.get_style_emb = lambda mel, rl=False: ns["get_style_emb"](me, mel, rl)
    for i, (seconds, length, chunk) in enumerate(CHUNKING_CASES):
        wav = O.synthetic_reference_wav(seconds, 22050, 140.0, 31)
        with torch.no_grad():
            rec[f"gcl{i}"] = ns["get_gpt_cond_latents"](me, wav[None], 22050, length=length, chunk_length=chunk)[0].numpy()


def prompt_construction(dims, gs, cs, speakers, rec):
    g = dims.gpt
    base = os.path.join(ref_import.REF_SRC, "auralis", "models", "xttsv2")
    fns = _lift_methods(os.path.join(base, "XTTSv2.py"), "XTTSv2Engine", ("prepare_text_tokens_async", "_merge_conditioning"))
    tree = ast.parse(open(os.path.join(base, "components", "vllm_mm_gpt.py")).read())
    lpe = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "LearnedPositionEmbeddings"]
    ns = {"torch": torch, "nn": torch.nn, "random": random, "List": List, "Tuple": Tuple, "Union": Union}
    exec(compile(ast.Module(body=lpe + fns, type_ignores=[]), "lifted", "exec"), ns)
    text_emb = torch.nn.Embedding(g.n_text_tokens, g.hidden)
    text_emb.weight.data.copy_(cs["text_embedding.weight"])
    text_pos = ns["LearnedPositionEmbeddings"](g.max_text_tokens + 2, g.hidden)
    text_pos.emb.weight.data.copy_(cs["text_pos_embedding.emb.weight"])
    cond = speakers[0][0]
    for n_chunks, seed in PROMPT_CASES:
        chunks = prompt_chunks(dims, n_chunks, seed)
        tok = types.SimpleNamespace(bos_token_id=0, eos_token_id=1,
                                    batch_encode_with_split=lambda text, lang, _c=chunks: [list(c) for c in _c])
        me = types.SimpleNamespace(tokenizer=tok, text_embedding=text_emb, text_pos_embedding=text_pos, logger=logging.getLogger("x"),
                                   llm_engine=types.SimpleNamespace(engine=types.SimpleNamespace(model_config=types.SimpleNamespace(dtype=torch.float32))))

        async def go():
            fake, embeds = await ns["prepare_text_tokens_async"](me, "ignored", "en", split_text=True)
            merged = await ns["_merge_conditioning"](me, embeds, cond[None])
            return fake, merged
        with torch.no_grad():
            fake, merged = asyncio.new_event_loop().run_until_complete(go())
        rec[f"prompt{n_chunks}_fake_lens"] = np.array([len(f) for f in fake], np.int64)
        for j, m in enumerate(merged):
            rec[f"prompt{n_chunks}_{j}"] = m.numpy()


def gpt_wrapper(dims, gs, cs, speakers, rec):
    g = dims.gpt
    path = os.path.join(ref_import.REF_SRC, "auralis", "models", "xttsv2", "components", "vllm_mm_gpt.py")
    tree = ast.parse(open(path).read())
    lpe = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "LearnedPositionEmbeddings"]
    fns = _lift_methods(path, "GPT2Model", ("forward", "_insert_conditioning_into_hidden_states"))
    for f in fns:
        f.decorator_list = []
    ns = {"torch": torch, "nn": torch.nn, "random": random,
          "get_pp_group": lambda: types.SimpleNamespace(is_first_rank=True, is_last_rank=True)}
    exec(compile(ast.Module(body=lpe + fns, type_ignores=[]), "lifted", "exec", flags=__future__.annotations.compiler_flag), ns)
    wte = torch.nn.Embedding(g.n_audio_tokens, g.hidden)
    wte.weight.data.copy_(gs["gpt.wte.weight"])
    wpe = ns["LearnedPositionEmbeddings"](g.max_audio_tokens + 3, g.hidden)
    wpe.emb.weight.data.copy_(gs["gpt.wpe.emb.weight"])
    me = types.SimpleNamespace(wte=wte, wpe=wpe, audio_start_generation_token=g.start_audio_token, embed_dim=g.hidden,
                               start_layer=0, end_layer=0, h=[], ln_f=lambda x: x,
                               _insert_conditioning_into_hidden_states=ns["_insert_conditioning_into_hidden_states"])
    prefix = O.GPTOracle(gs, cs, dims).prompt_rows(speakers[1][0], WRAPPER_IDS)[:-1]     # what _merge_conditioning hands to vLLM
    empty = torch.empty(0, dtype=torch.long)
    with torch.no_grad():
        rec["wrapper_prefill"] = ns["forward"](me, empty, empty, [], None, None, input_embeds=[prefix[None]], starting_sequence_start_ids=[0],
                                               is_logit_only=torch.tensor([False])).numpy()
        for i, (tok, k) in enumerate(WRAPPER_DECODE(g)):
            rec[f"wrapper_decode{i}"] = ns["forward"](me, torch.tensor([tok]), torch.tensor([k]), [], None, None)[0].numpy()
        rec["wrapper_mixed"] = ns["forward"](me, torch.tensor([9]), torch.tensor([4]), [], None, None, input_embeds=[prefix[None]],
                                             starting_sequence_start_ids=[1], is_logit_only=torch.tensor([False])).numpy()


def placeholder_prompt(dims, rec):
    path = os.path.join(ref_import.REF_SRC, "auralis", "models", "xttsv2", "components", "vllm_mm_gpt.py")
    tree = ast.parse(open(path).read())
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "input_processor_for_xtts2_gpt"]
    ns = {"token_inputs": lambda **kw: kw, "PlaceholderRange": lambda **kw: kw}
    exec(compile(ast.Module(body=fn, type_ignores=[]), "lifted", "exec", flags=__future__.annotations.compiler_flag), ns)
    g = dims.gpt
    ctx = types.SimpleNamespace(model_config=types.SimpleNamespace(hf_config=types.SimpleNamespace(start_audio_token=g.start_audio_token)))
    for n_text in PLACEHOLDER_TEXT_LENS:
        embeds = torch.zeros(g.n_cond_latents + n_text, g.hidden)
        out = ns["input_processor_for_xtts2_gpt"](ctx, {"multi_modal_data": {"audio": {"embeds": embeds}}, "prompt_token_ids": [1] * n_text})
        rec[f"placeholder{n_text}"] = np.array(out["prompt_token_ids"], np.int64)


def main():
    torch.set_num_threads(8)
    ref = ref_import.load()
    dims = XTTSDims.small()
    gs, cs = synth_state(dims, SEED)
    speakers = _speakers(dims)
    rec = {}
    vocoder(ref, dims, cs, rec)
    conditioning(ref, dims, cs, rec)
    speaker_encoder(ref, dims, cs, rec)
    gpt_cond_latents_chunking(ref, dims, cs, rec)
    prompt_construction(dims, gs, cs, speakers, rec)
    gpt_wrapper(dims, gs, cs, speakers, rec)
    placeholder_prompt(dims, rec)
    np.savez_compressed(OUT, **rec)
    print(f"{OUT}: {len(rec)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
