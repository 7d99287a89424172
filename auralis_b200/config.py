"""Model dimensions of the XTTSv2 hot path, restated as plain dataclasses.

Follows the reference's HF config classes for the values only
(`/root/reference/src/auralis/models/xttsv2/config/xttsv2_gpt_config.py:133-229`,
`.../config/xttsv2_config.py:237-301`, vocoder defaults
`.../components/tts/layers/xtts/hifigan_decoder.py:698-723`).
No transformers dependency: the native library only needs the integers.
"""
from __future__ import annotations

from dataclasses import dataclass, field, asdict
from typing import Tuple


@dataclass
class GPTDims:
    hidden: int = 1024            # xttsv2_gpt_config.py:136
    layers: int = 30              # :137
    heads: int = 16               # :138  (head_dim is fixed to 64 in the kernels)
    ff: int = 4096                # :139 n_inner
    n_text_tokens: int = 6681     # :143
    n_audio_tokens: int = 1026    # :148
    start_audio_token: int = 1024 # :149
    stop_audio_token: int = 1025  # :150
    max_audio_tokens: int = 605   # :153
    max_text_tokens: int = 402    # :154
    n_cond_latents: int = 32      # perceiver output length (vllm_mm_gpt.py:231)
    ln_eps: float = 1e-5          # :171
    activation: str = "gelu_new"  # checkpoint_converter.py:197

    @property
    def head_dim(self) -> int:
        return self.hidden // self.heads

    @property
    def n_wpe(self) -> int:        # vllm_mm_gpt.py:753  max_audio_tokens + 3
        return self.max_audio_tokens + 3

    @property
    def n_text_pos(self) -> int:   # XTTSv2.py:105-110 max_text_tokens + 2
        return self.max_text_tokens + 2

    @property
    def max_prompt_rows(self) -> int:  # 32 cond + (402+2) text + bos
        return self.n_cond_latents + self.n_text_pos + 1

    @property
    def max_ctx(self) -> int:      # prompt rows + generated tokens
        return self.max_prompt_rows + self.max_audio_tokens


@dataclass
class VocoderDims:
    in_dim: int = 1024                          # decoder_input_dim
    init_ch: int = 512                          # upsample_initial_channel_decoder
    up_rates: Tuple[int, ...] = (8, 8, 2, 2)
    up_kernels: Tuple[int, ...] = (16, 16, 4, 4)
    rb_kernels: Tuple[int, ...] = (3, 7, 11)
    rb_dilations: Tuple[int, ...] = (1, 3, 5)
    d_vector: int = 512
    input_sample_rate: int = 22050
    output_sample_rate: int = 24000
    output_hop_length: int = 256
    code_stride: int = 1024                     # ar_mel_length_compression

    @property
    def hop(self) -> int:
        p = 1
        for r in self.up_rates:
            p *= r
        return p

    def z_frames(self, n_latents: int, speed: float = 1.0) -> int:
        """Length after the two linear interpolations (hifigan_decoder.py:787-800):
        floor(floor(T*4.0) * 24000/22050) with torch's float rule.  A speaking rate other than 1 first time-scales the T
        latents to floor(T * ls) frames, ls = 1 / speed with the speed rounded to float32 (what the engine receives)."""
        import math
        if speed != 1.0:
            n_latents = int(math.floor(n_latents * speed_scale(speed)))
        t1 = int(math.floor(n_latents * (self.code_stride / self.output_hop_length)))
        return int(math.floor(t1 * (self.output_sample_rate / self.input_sample_rate)))

    def n_samples(self, n_latents: int, speed: float = 1.0) -> int:
        return self.z_frames(n_latents, speed) * self.hop


SPEED_MIN, SPEED_MAX = 0.25, 4.0     # speaking-rate range (that of OpenAI's /v1/audio/speech)
NUM_BEAMS_MAX = 8                   # beams per chunk (TTSRequest.num_beams, xtts_submit_beams)


def speed_scale(speed: float) -> float:
    """The time scale of a speaking rate, ls = 1 / speed, from the float32 value every layer receives (Xtts.inference:
    length_scale = 1 / speed)."""
    import numpy as np
    return 1.0 / float(np.float32(speed))


@dataclass
class CondDims:
    n_mels: int = 80
    cond_blocks: int = 6          # ConditioningEncoder attn_blocks
    perceiver_depth: int = 2
    perceiver_heads: int = 8
    perceiver_dim_head: int = 64
    perceiver_ff_mult: int = 4
    spk_layers: Tuple[int, ...] = (3, 4, 6, 3)
    spk_filters: Tuple[int, ...] = (32, 64, 128, 256)
    spk_mels: int = 64
    spk_proj: int = 512


@dataclass
class XTTSDims:
    gpt: GPTDims = field(default_factory=GPTDims)
    voc: VocoderDims = field(default_factory=VocoderDims)
    cond: CondDims = field(default_factory=CondDims)

    @staticmethod
    def full() -> "XTTSDims":
        return XTTSDims()

    @staticmethod
    def small() -> "XTTSDims":
        """A tiny geometry with the same structure, for CPU-fast parity tests."""
        g = GPTDims(hidden=128, layers=2, heads=2, ff=512, n_text_tokens=97,
                    n_audio_tokens=130, start_audio_token=128, stop_audio_token=129,
                    max_audio_tokens=48, max_text_tokens=30, n_cond_latents=32)
        v = VocoderDims(in_dim=128, init_ch=64, d_vector=32)
        c = CondDims(spk_layers=(1, 1, 1, 1), spk_filters=(8, 16, 32, 64), spk_proj=32,
                     cond_blocks=2, perceiver_depth=1, perceiver_heads=2)
        return XTTSDims(g, v, c)

    @staticmethod
    def from_reference_configs(core_cfg: dict, gpt_cfg: dict | None = None) -> "XTTSDims":
        """Geometry from the two config.json files the reference's converter writes
        (`utils/checkpoint_converter.py:117-223`: `core_xttsv2/config.json` and `gpt/config.json`; the core file also
        embeds the GPT one under "gpt_config").  Keys the files do not carry keep the class defaults, exactly like the
        reference's XTTSConfig / XTTSGPTConfig (`config/xttsv2_config.py:237-301`, `config/xttsv2_gpt_config.py:133-229`);
        the HiFi-GAN layout is not configurable there either (`hifigan_decoder.py:698-723`)."""
        g = dict(core_cfg.get("gpt_config") or {})
        g.update(gpt_cfg or {})
        d = GPTDims()
        gd = GPTDims(
            hidden=int(g.get("hidden_size", d.hidden)), layers=int(g.get("num_hidden_layers", d.layers)),
            heads=int(g.get("num_attention_heads", d.heads)), ff=int(g.get("n_inner", 4 * int(g.get("hidden_size", d.hidden)))),
            n_text_tokens=int(g.get("number_text_tokens", g.get("vocab_size", d.n_text_tokens))),
            n_audio_tokens=int(g.get("num_audio_tokens", d.n_audio_tokens)),
            start_audio_token=int(g.get("start_audio_token", d.start_audio_token)),
            stop_audio_token=int(g.get("stop_audio_token", d.stop_audio_token)),
            max_audio_tokens=int(g.get("max_audio_tokens", d.max_audio_tokens)),
            max_text_tokens=int(g.get("max_text_tokens", d.max_text_tokens)),
            ln_eps=float(g.get("layer_norm_epsilon", d.ln_eps)), activation=str(g.get("activation_function", d.activation)))
        if gd.hidden != gd.heads * 64:
            raise ValueError(f"hidden_size {gd.hidden} / num_attention_heads {gd.heads}: the kernels need 64-wide heads")
        if gd.activation != "gelu_new":
            raise ValueError(f"activation_function {gd.activation!r} is not supported (gelu_new only)")
        v = VocoderDims()
        ac = core_cfg.get("audio_config") or {}
        vd = VocoderDims(
            in_dim=int(core_cfg.get("decoder_input_dim", gd.hidden)), d_vector=int(core_cfg.get("d_vector_dim", v.d_vector)),
            input_sample_rate=int(core_cfg.get("input_sample_rate", ac.get("sample_rate", v.input_sample_rate))),
            output_sample_rate=int(core_cfg.get("output_sample_rate", ac.get("output_sample_rate", v.output_sample_rate))),
            output_hop_length=int(core_cfg.get("output_hop_length", ac.get("hop_length", v.output_hop_length))),
            code_stride=int(core_cfg.get("gpt_code_stride_len", v.code_stride)))
        return XTTSDims(gd, vd, CondDims(spk_proj=vd.d_vector))

    def to_json(self) -> dict:
        return asdict(self)

    @staticmethod
    def from_json(d: dict) -> "XTTSDims":
        g = GPTDims(**d["gpt"])
        vd = dict(d["voc"])
        for k in ("up_rates", "up_kernels", "rb_kernels", "rb_dilations"):
            vd[k] = tuple(vd[k])
        cd = dict(d["cond"])
        for k in ("spk_layers", "spk_filters"):
            cd[k] = tuple(cd[k])
        return XTTSDims(g, VocoderDims(**vd), CondDims(**cd))
