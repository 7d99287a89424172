"""ctypes binding of ``libxtts_b200.so`` (C ABI: ``include/xtts_b200.h``).

No torch types cross this boundary: numpy arrays in host memory in, numpy arrays out.
The library is CUDA-only; creating an engine without an sm_90 GPU raises ``NativeError``
(there is no CPU fallback — parity claims depend on that).
"""
from __future__ import annotations

import ctypes as C
import hashlib
import math
import os
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np

from .config import SPEED_MAX, SPEED_MIN, XTTSDims

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libxtts_b200.so")

PRECISION_FP32 = 0
PRECISION_BF16 = 1
PRECISION_FP16 = 2
ERR_INVALID = -1
ERR_CANCELLED = -5


class NativeError(RuntimeError):
    def __init__(self, msg: str, code: int = 0):
        super().__init__(msg)
        self.code = code            # the XTTS_ERR_* the call returned (0 when not from a call)


class XttsConfig(C.Structure):
    _fields_ = [
        ("device", C.c_int32), ("precision", C.c_int32), ("max_batch", C.c_int32), ("max_speakers", C.c_int32),
        ("hidden", C.c_int32), ("layers", C.c_int32), ("heads", C.c_int32), ("ff", C.c_int32),
        ("n_text_tokens", C.c_int32), ("n_audio_tokens", C.c_int32), ("start_audio_token", C.c_int32),
        ("stop_audio_token", C.c_int32), ("max_audio_tokens", C.c_int32), ("max_text_tokens", C.c_int32),
        ("n_cond_latents", C.c_int32), ("ln_eps", C.c_float),
        ("voc_in_dim", C.c_int32), ("voc_init_ch", C.c_int32), ("voc_n_up", C.c_int32),
        ("voc_up_rates", C.c_int32 * 4), ("voc_up_kernels", C.c_int32 * 4), ("voc_n_rb", C.c_int32),
        ("voc_rb_kernels", C.c_int32 * 4), ("voc_rb_dilations", C.c_int32 * 4), ("d_vector", C.c_int32),
        ("code_stride", C.c_int32), ("output_hop_length", C.c_int32), ("input_sample_rate", C.c_int32),
        ("output_sample_rate", C.c_int32),
        ("n_mels", C.c_int32), ("cond_blocks", C.c_int32), ("perceiver_depth", C.c_int32),
        ("perceiver_heads", C.c_int32), ("perceiver_dim_head", C.c_int32), ("perceiver_ff_mult", C.c_int32),
        ("spk_layers", C.c_int32 * 4), ("spk_filters", C.c_int32 * 4), ("spk_mels", C.c_int32), ("spk_proj", C.c_int32),
    ]


class XttsBeam(C.Structure):
    _fields_ = [("num_beams", C.c_int32), ("length_penalty", C.c_float), ("do_sample", C.c_int32)]


class XttsBeamState(C.Structure):
    _fields_ = [("run_score", C.c_float * 8), ("fin_score", C.c_float * 8), ("fin_valid", C.c_int32 * 8),
                ("fin_step", C.c_int32 * 8), ("fin_beam", C.c_int32 * 8), ("fin_tok", C.c_int32 * 8),
                ("heur_unsat", C.c_int32), ("done", C.c_int32), ("sel_parent", C.c_int32 * 8), ("sel_tok", C.c_int32 * 8),
                ("n_copy", C.c_int32), ("copy_src", C.c_int32 * 8), ("copy_dst", C.c_int32 * 8), ("copy_ntok", C.c_int32 * 8),
                ("n_free", C.c_int32), ("n_pages", C.c_int32 * 8)]


class XttsSampling(C.Structure):
    _fields_ = [("temperature", C.c_float), ("top_p", C.c_float), ("repetition_penalty", C.c_float),
                ("top_k", C.c_int32), ("max_tokens", C.c_int32), ("stop_token", C.c_int32),
                ("seed", C.c_uint64), ("seq_seed", C.c_int32), ("vocode", C.c_int32), ("priority", C.c_int32),
                ("early_tokens", C.c_int32)]


class XttsResult(C.Structure):
    _fields_ = [("seq_id", C.c_uint64), ("status", C.c_int32), ("n_tokens", C.c_int32), ("n_samples", C.c_int32),
                ("n_prompt_rows", C.c_int32), ("t_submit", C.c_double), ("t_first_token", C.c_double),
                ("t_done", C.c_double)]


class XttsStats(C.Structure):
    _fields_ = [("kernel_launches", C.c_uint64), ("decode_steps", C.c_uint64), ("prefill_rows", C.c_uint64),
                ("tokens_generated", C.c_uint64), ("samples_generated", C.c_uint64),
                ("gpt_ms", C.c_double), ("vocoder_ms", C.c_double), ("cond_ms", C.c_double),
                ("hbm_bytes_weights", C.c_uint64)]


class XttsEnhanceConfig(C.Structure):
    _fields_ = [("sample_rate", C.c_int32), ("normalize", C.c_int32), ("trim_silence", C.c_int32),
                ("remove_noise", C.c_int32), ("enhance_speech", C.c_int32), ("vad_frame_length", C.c_int32),
                ("noise_reduce_frames", C.c_int32), ("vad_threshold", C.c_float), ("noise_reduce_margin", C.c_float),
                ("enhance_amount", C.c_float), ("target_lufs", C.c_float)]

    @classmethod
    def of(cls, cfg) -> "XttsEnhanceConfig":
        """From any object with the AudioPreprocessingConfig field names (requests.py)."""
        c = cls()
        for name, typ in cls._fields_:
            v = getattr(cfg, name)
            setattr(c, name, float(v) if typ is C.c_float else int(v))
        return c


class XttsFlacInfo(C.Structure):
    _fields_ = [("sample_rate", C.c_int32), ("channels", C.c_int32), ("bits_per_sample", C.c_int32),
                ("min_block", C.c_int32), ("max_block", C.c_int32), ("total_samples", C.c_int64),
                ("md5", C.c_uint8 * 16)]


def flac_md5(samples: np.ndarray, bits_per_sample: int) -> bytes:
    """The MD5 FLAC's STREAMINFO carries: samples [C, N] interleaved, little-endian, ceil(bps / 8) bytes each."""
    nb = (bits_per_sample + 7) // 8
    inter = np.ascontiguousarray(np.asarray(samples).T)
    if nb in (1, 2, 4):
        return hashlib.md5(inter.astype({1: "<i1", 2: "<i2", 4: "<i4"}[nb]).tobytes()).digest()
    return hashlib.md5(inter.astype("<i4").view(np.uint8).reshape(-1, 4)[:, :nb].tobytes()).digest()


class XttsKernelProfile(C.Structure):
    _fields_ = [("n", C.c_int32), ("name", (C.c_char * 32) * 16), ("ms", C.c_double * 16), ("flops", C.c_double * 16),
                ("bytes", C.c_double * 16), ("launches", C.c_uint64 * 16)]


# every symbol include/xtts_b200.h declares (checked by tests/test_abi.py against the header text)
ABI_SYMBOLS = [
    "xtts_last_error", "xtts_version", "xtts_create", "xtts_destroy", "xtts_load_weight", "xtts_finalize_weights",
    "xtts_set_speaker", "xtts_get_speaker", "xtts_condition", "xtts_enhance", "xtts_change_speed", "xtts_resample", "xtts_encode_flac", "xtts_decode_flac", "xtts_submit", "xtts_submit_speed", "xtts_submit_beams", "xtts_debug_beam_step", "xtts_cancel", "xtts_poll",
    "xtts_fetch", "xtts_set_option", "xtts_get_stats", "xtts_sync", "xtts_get_kernel_profile", "xtts_device_timer", "xtts_vocode",
    "xtts_vocode_window", "xtts_vocode_speed", "xtts_gpt_prefill", "xtts_gpt_teacher_forced",
    "xtts_debug_gemm", "xtts_debug_sample_slots", "xtts_debug_trace",
    "xtts_debug_attn_decode", "xtts_debug_attn_prefill", "xtts_debug_splitk_ln", "xtts_debug_conv_tc",
    "xtts_debug_ln_gemm", "xtts_debug_norms", "xtts_debug_kv_write", "xtts_debug_build_rows", "xtts_debug_build_decode_rows",
    "xtts_debug_cond",
]

# flag bits of xtts_debug_gemm / xtts_debug_ln_gemm (include/xtts_b200.h)
GEMM_GELU, GEMM_OUT16, GEMM_INPLACE, GEMM_PDL = 1, 2, 4, 8

# op codes of xtts_debug_cond (XTTS_COND_* in include/xtts_b200.h)
COND_OPS = ("FRAME_WINDOW", "POWER", "MEL_LOG", "PREEMPHASIS", "INSTNORM_T", "GROUPNORM", "GEGLU", "RMSNORM_ACCUM", "CONV2D",
            "CHANNEL_MEAN", "SE_GATE", "SE_APPLY", "TRANSPOSE", "RELU_BN_ROWS", "ASP", "L2NORM", "GEMV", "MEL22", "MEL16")
COND_OP = {name: i for i, name in enumerate(COND_OPS)}

_lib = None


def load_library(path: Optional[str] = None):
    """dlopen the library and declare prototypes.  Raises NativeError if it was not built."""
    global _lib
    if _lib is not None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise NativeError(f"{p} not found: run `python -m auralis_b200.build` (no CPU fallback exists)")
    lib = C.CDLL(p)
    vp, i32, i64, f32p, i32p = C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_float), C.POINTER(C.c_int32)
    lib.xtts_last_error.restype = C.c_char_p
    lib.xtts_version.restype = C.c_char_p
    lib.xtts_create.argtypes = [C.POINTER(XttsConfig), C.POINTER(vp)]
    lib.xtts_destroy.argtypes = [vp]
    lib.xtts_load_weight.argtypes = [vp, C.c_char_p, f32p, C.POINTER(i64), i32]
    lib.xtts_finalize_weights.argtypes = [vp]
    lib.xtts_set_speaker.argtypes = [vp, i32, f32p, f32p]
    lib.xtts_get_speaker.argtypes = [vp, i32, f32p, f32p]
    lib.xtts_condition.argtypes = [vp, i32, f32p, i64, f32p, i64, i32, i32]
    lib.xtts_enhance.argtypes = [vp, f32p, i64, C.POINTER(XttsEnhanceConfig), f32p, i64, C.POINTER(i64)]
    lib.xtts_change_speed.argtypes = [vp, f32p, i64, C.c_double, f32p, i64, C.POINTER(i64)]
    lib.xtts_resample.argtypes = [vp, f32p, i64, i32, i32, f32p, i64, C.POINTER(i64)]
    u8p = C.POINTER(C.c_uint8)
    lib.xtts_encode_flac.argtypes = [vp, C.POINTER(C.c_int16), i64, i32, u8p, u8p, i64, C.POINTER(i64)]
    lib.xtts_decode_flac.argtypes = [vp, u8p, i64, i32p, i64, C.POINTER(XttsFlacInfo)]
    lib.xtts_submit.argtypes = [vp, C.c_uint64, i32p, i32, i32, C.POINTER(XttsSampling)]
    lib.xtts_submit_speed.argtypes = [vp, C.c_uint64, i32p, i32, i32, C.POINTER(XttsSampling), C.c_float]
    lib.xtts_submit_beams.argtypes = [vp, C.c_uint64, i32p, i32, i32, C.POINTER(XttsSampling), C.c_float, C.POINTER(XttsBeam)]
    lib.xtts_cancel.argtypes = [vp, C.c_uint64]
    lib.xtts_poll.argtypes = [vp, C.POINTER(XttsResult), i32]
    lib.xtts_fetch.argtypes = [vp, C.c_uint64, i32p, f32p, f32p]
    lib.xtts_set_option.argtypes = [vp, C.c_char_p, i64]
    lib.xtts_get_stats.argtypes = [vp, C.POINTER(XttsStats)]
    lib.xtts_sync.argtypes = [vp]
    lib.xtts_get_kernel_profile.argtypes = [vp, C.POINTER(XttsKernelProfile)]
    lib.xtts_device_timer.argtypes = [vp, i32, C.POINTER(C.c_double)]
    lib.xtts_vocode.argtypes = [vp, f32p, i32, i32, f32p, i32p, C.c_char_p, f32p, i64]
    lib.xtts_vocode_window.argtypes = [vp, f32p, i32, i32, i32, i32, f32p]
    lib.xtts_vocode_speed.argtypes = [vp, f32p, i32, i32, C.c_float, i32, i32, f32p, i32p]
    lib.xtts_gpt_prefill.argtypes = [vp, i32p, i32, i32, i32p, i32, f32p, f32p, f32p]
    lib.xtts_gpt_teacher_forced.argtypes = [vp, i32p, i32, i32, i32p, i32, C.POINTER(XttsSampling), f32p, f32p, i32p]
    lib.xtts_debug_gemm.argtypes = [vp, i32, f32p, f32p, f32p, f32p, f32p, i32, i32, i32, i32, i32, f32p]
    lib.xtts_debug_sample_slots.argtypes = [vp, i32, i32, i32p, i32, f32p, i32, C.POINTER(XttsSampling), i32, i32, i32p,
                                            i32p, i32p, i32p, i32p, C.POINTER(C.c_uint8), i32p, i32p]
    lib.xtts_debug_trace.argtypes = [vp, i32, C.POINTER(C.c_uint64), i32]
    lib.xtts_debug_attn_decode.argtypes = [vp, i32, i32, i32, i32p, i32, i32p, i32p, i32, i32, vp, vp, f32p, f32p]
    lib.xtts_debug_attn_prefill.argtypes = [vp, i32, i32, i32p, i32, i32, C.c_float, f32p, i64, i32, i32, f32p, i64, i32, i32,
                                            i64, i64, f32p, i32]
    lib.xtts_debug_splitk_ln.argtypes = [vp, i32, i32, i32, i32, i32, f32p, f32p, f32p, f32p, f32p, f32p, f32p]
    lib.xtts_debug_conv_tc.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, i32p, f32p, f32p, f32p, i32, f32p, f32p, i32,
                                       C.c_float, C.c_float, i32, f32p, f32p]
    u32p = C.POINTER(C.c_uint32)
    lib.xtts_debug_ln_gemm.argtypes = [vp, i32, i32, i32, i32, i32, f32p, f32p, f32p, f32p, f32p, f32p, i32, f32p, f32p, i32p, u32p]
    lib.xtts_debug_norms.argtypes = [vp, i32, i32, i32, f32p, i32, i32p, f32p, f32p, f32p, f32p, f32p, f32p, i32, i32, i32p, i32p,
                                     i32p]
    lib.xtts_debug_kv_write.argtypes = [vp, i32, i32, i32, f32p, i32p, i32p, i32, i32p, i32p, i32, i32, vp, vp]
    lib.xtts_debug_build_rows.argtypes = [vp, i32, i32, f32p, i32, f32p, i32, f32p, i32, f32p, i32, f32p, i32, i32p, i32, f32p]
    lib.xtts_debug_build_decode_rows.argtypes = [vp, i32, f32p, i32, f32p, i32, i32, i32p, i32, i32p, i32p, f32p, u32p, i32, i32]
    lib.xtts_debug_beam_step.argtypes = [vp, i32, i32, i32, i32, C.POINTER(XttsSampling), C.POINTER(XttsBeam), i32, i32, f32p,
                                         i32p, i32p, i32p, u32p, i32, i32p, i32, i32p, i32, i32p, C.POINTER(XttsBeamState),
                                         vp, vp, f32p]
    lib.xtts_debug_cond.argtypes = [vp, i32, i32p, i32, f32p, i32, C.POINTER(f32p), C.POINTER(i64), i32, f32p, i64]
    for s in ABI_SYMBOLS:
        if s not in ("xtts_last_error", "xtts_version"):
            getattr(lib, s).restype = C.c_int
    _lib = lib
    return lib


def _f32(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32))


def _i32(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, dtype=np.int32))


def atoms_lpad(L: int) -> int:
    """Rows per plane of an fp16 atom image holding a signal of L steps (atoms_lpad in csrc/conv1d_tc.cu): a 64-row head
    pad, the signal plus at least one zero row rounded up to 512, a 64-row tail pad."""
    return 64 + -(-(L + 1) // 512) * 512 + 64


def _fp(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_float))


def _ip(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_int32))


def make_config(dims: XTTSDims, device: int = 0, precision: int = PRECISION_FP32, max_batch: int = 64,
                max_speakers: int = 16) -> XttsConfig:
    g, v, c = dims.gpt, dims.voc, dims.cond
    cfg = XttsConfig()
    cfg.device, cfg.precision, cfg.max_batch, cfg.max_speakers = device, precision, max_batch, max_speakers
    cfg.hidden, cfg.layers, cfg.heads, cfg.ff = g.hidden, g.layers, g.heads, g.ff
    cfg.n_text_tokens, cfg.n_audio_tokens = g.n_text_tokens, g.n_audio_tokens
    cfg.start_audio_token, cfg.stop_audio_token = g.start_audio_token, g.stop_audio_token
    cfg.max_audio_tokens, cfg.max_text_tokens, cfg.n_cond_latents = g.max_audio_tokens, g.max_text_tokens, g.n_cond_latents
    cfg.ln_eps = g.ln_eps
    cfg.voc_in_dim, cfg.voc_init_ch, cfg.voc_n_up = v.in_dim, v.init_ch, len(v.up_rates)
    for i, (r, k) in enumerate(zip(v.up_rates, v.up_kernels)):
        cfg.voc_up_rates[i], cfg.voc_up_kernels[i] = r, k
    cfg.voc_n_rb = len(v.rb_kernels)
    for i, k in enumerate(v.rb_kernels):
        cfg.voc_rb_kernels[i] = k
    for i, d in enumerate(v.rb_dilations):
        cfg.voc_rb_dilations[i] = d
    cfg.d_vector = v.d_vector
    cfg.code_stride, cfg.output_hop_length = v.code_stride, v.output_hop_length
    cfg.input_sample_rate, cfg.output_sample_rate = v.input_sample_rate, v.output_sample_rate
    cfg.n_mels, cfg.cond_blocks, cfg.perceiver_depth = c.n_mels, c.cond_blocks, c.perceiver_depth
    cfg.perceiver_heads, cfg.perceiver_dim_head, cfg.perceiver_ff_mult = c.perceiver_heads, c.perceiver_dim_head, c.perceiver_ff_mult
    for i in range(4):
        cfg.spk_layers[i], cfg.spk_filters[i] = c.spk_layers[i], c.spk_filters[i]
    cfg.spk_mels, cfg.spk_proj = c.spk_mels, c.spk_proj
    return cfg


@dataclass
class Sampling:
    temperature: float = 0.75
    top_p: float = 0.85
    top_k: int = 50
    repetition_penalty: float = 5.0
    max_tokens: int = 605
    stop_token: int = 1025
    seed: int = 0
    seq_seed: int = 0
    vocode: bool = True
    priority: int = 0
    early_tokens: int = 0          # > 0: stream the chunk's audio as partial results, first piece after n tokens (include/xtts_b200.h)
    speed: float = 1.0             # speaking rate in [0.25, 4] (xtts_submit_speed; passed beside the struct, which cannot grow)
    num_beams: int = 1             # > 1: beam search over this many beams (xtts_submit_beams), with the two fields below
    length_penalty: float = 1.0
    do_sample: bool = True

    def c(self) -> XttsSampling:
        s = XttsSampling()
        s.temperature, s.top_p, s.repetition_penalty = self.temperature, self.top_p, self.repetition_penalty
        s.top_k, s.max_tokens, s.stop_token = self.top_k, self.max_tokens, self.stop_token
        s.seed, s.seq_seed, s.vocode = self.seed, self.seq_seed, 1 if self.vocode else 0
        s.priority = self.priority
        s.early_tokens = max(0, int(self.early_tokens))
        return s


class NativeEngine:
    """One engine = one GPU.  Thin, allocation-free wrapper over the C ABI."""

    def __init__(self, dims: XTTSDims, device: int = 0, precision: int = PRECISION_FP32, max_batch: int = 64,
                 max_speakers: int = 16):
        self.lib = load_library()
        self.dims = dims
        self.cfg = make_config(dims, device, precision, max_batch, max_speakers)
        self.precision = precision
        self.max_batch = max_batch
        h = C.c_void_p()
        rc = self.lib.xtts_create(C.byref(self.cfg), C.byref(h))
        if rc != 0:
            raise NativeError(f"xtts_create failed ({rc}): {self.lib.xtts_last_error().decode()}")
        self.h = h

    def _chk(self, rc: int, what: str):
        if rc != 0:
            raise NativeError(f"{what} failed ({rc}): {self.lib.xtts_last_error().decode()}", rc)

    def close(self):
        if getattr(self, "h", None):
            self.lib.xtts_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- weights
    def load_state(self, *states: Dict[str, "object"]):
        for st in states:
            for name, t in st.items():
                a = t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
                a = _f32(a)
                shape = (C.c_int64 * max(1, a.ndim))(*a.shape) if a.ndim else (C.c_int64 * 1)(1)
                self._chk(self.lib.xtts_load_weight(self.h, name.encode(), _fp(a), shape, max(1, a.ndim) if a.ndim else 1),
                          f"load_weight({name})")
        self._chk(self.lib.xtts_finalize_weights(self.h), "finalize_weights")

    # ---- speakers
    def set_speaker(self, slot: int, cond_latents, d_vector):
        c, g = _f32(cond_latents).reshape(-1), _f32(d_vector).reshape(-1)
        assert c.size == self.dims.gpt.n_cond_latents * self.dims.gpt.hidden and g.size == self.dims.voc.d_vector
        self._chk(self.lib.xtts_set_speaker(self.h, slot, _fp(c), _fp(g)), "set_speaker")

    def get_speaker(self, slot: int) -> Tuple[np.ndarray, np.ndarray]:
        c = np.empty((self.dims.gpt.n_cond_latents, self.dims.gpt.hidden), np.float32)
        g = np.empty((self.dims.voc.d_vector,), np.float32)
        self._chk(self.lib.xtts_get_speaker(self.h, slot, _fp(c), _fp(g)), "get_speaker")
        return c, g

    def condition(self, slot: int, wav22k, wav16k, gpt_cond_len: int = 30, gpt_cond_chunk_len: int = 4):
        a, b = _f32(wav22k).reshape(-1), _f32(wav16k).reshape(-1)
        self._chk(self.lib.xtts_condition(self.h, slot, _fp(a), a.size, _fp(b), b.size, gpt_cond_len, gpt_cond_chunk_len),
                  "condition")

    def enhance(self, wav, cfg) -> np.ndarray:
        """xtts_enhance: the reference's speaker-file enhancer (VAD trim, spectral gating, clarity, loudness) and its
        16-bit write/read, on the GPU.  `wav` is mono at `cfg.sample_rate`; `cfg` has AudioPreprocessingConfig's
        fields.  Raises NativeError with code ERR_INVALID where the reference's enhancer would fail."""
        a = _f32(wav).reshape(-1)
        out = np.empty((a.size,), np.float32)
        n_out = C.c_int64(0)
        self._chk(self.lib.xtts_enhance(self.h, _fp(a), a.size, C.byref(XttsEnhanceConfig.of(cfg)), _fp(out), out.size,
                                        C.byref(n_out)), "enhance")
        return out[: n_out.value]

    def change_speed(self, wav, rate: float) -> np.ndarray:
        """xtts_change_speed: the reference's TTSOutput.change_speed body (librosa phase-vocoder time stretch, then peak
        normalisation) on the GPU; rate > 1 is faster.  -> float32 [512 * (ceil((1 + n // 512) / rate) - 1)].  Raises
        NativeError with code ERR_INVALID where the reference raises (rate not finite or <= 0, a non-finite sample, an
        empty result)."""
        a = _f32(wav).reshape(-1)
        rate = float(rate)
        n_out = C.c_int64(0)
        frames = math.ceil((1 + a.size // 512) / rate) if math.isfinite(rate) and rate > 0 else 1
        cap = 512 * (frames - 1) if frames <= 1 << 22 else 0          # longer results are rejected by the call
        out = np.empty((max(cap, 1),), np.float32)
        self._chk(self.lib.xtts_change_speed(self.h, _fp(a), a.size, rate, _fp(out), cap, C.byref(n_out)), "change_speed")
        return out[: n_out.value]

    def resample(self, wav, orig_sr: int, new_sr: int) -> np.ndarray:
        """xtts_resample: torchaudio.functional.resample(wav, orig_sr, new_sr) with its defaults, on the GPU, for mono
        float32 audio -> float32 [ceil(new' n / orig')] (the rates over their gcd).  orig_sr == new_sr returns the samples
        unchanged.  Raises NativeError with code ERR_INVALID for a rate outside 1 .. 1048575 or a non-finite sample."""
        a = _f32(wav).reshape(-1)
        orig_sr, new_sr = int(orig_sr), int(new_sr)
        cap = 0                                                           # bad rates are rejected by the call
        if 0 < orig_sr < 1 << 20 and 0 < new_sr < 1 << 20:
            g = math.gcd(orig_sr, new_sr)
            cap = -(-(new_sr // g) * a.size // (orig_sr // g))
        out = np.empty((max(cap, 1),), np.float32)
        n_out = C.c_int64(0)
        self._chk(self.lib.xtts_resample(self.h, _fp(a), a.size, orig_sr, new_sr, _fp(out), cap, C.byref(n_out)), "resample")
        return out[: n_out.value]

    def encode_flac(self, pcm_i16, sample_rate: int, md5: Optional[bytes] = None) -> bytes:
        """xtts_encode_flac: a lossless FLAC stream of mono int16 samples, encoded on the GPU.  `md5` is the 16-byte MD5
        of the samples as little-endian bytes for STREAMINFO, or None (zeros, "not computed").  Raises NativeError with
        code ERR_INVALID for a sample rate outside 1 .. 1048575."""
        a = np.ascontiguousarray(pcm_i16).reshape(-1)
        if a.dtype != np.int16:
            raise TypeError(f"encode_flac takes int16 samples, not {a.dtype}")
        if md5 is not None and len(md5) != 16:
            raise ValueError("md5 must be 16 bytes")
        digest = None if md5 is None else (C.c_uint8 * 16).from_buffer_copy(bytes(md5))
        out = np.empty((42 + -(-a.size // 4096) * 8211,), np.uint8)       # no frame is larger than VERBATIM
        n_out = C.c_int64(0)
        u8p = C.POINTER(C.c_uint8)
        self._chk(self.lib.xtts_encode_flac(self.h, a.ctypes.data_as(C.POINTER(C.c_int16)), a.size, int(sample_rate),
                                            digest, out.ctypes.data_as(u8p), out.size, C.byref(n_out)), "encode_flac")
        return out[: n_out.value].tobytes()

    def decode_flac(self, data) -> Tuple[np.ndarray, int, int]:
        """xtts_decode_flac: a whole FLAC stream (bytes), decoded losslessly on the GPU -> (int32 [channels, samples],
        sample rate, bits per sample); each sample is the signed integer the stream codes.  Sizes the output from the
        call's own report (a stream whose STREAMINFO leaves the total at 0 is decoded twice), then checks STREAMINFO's
        MD5 when it is set.  Raises NativeError with code ERR_INVALID for a stream that breaks the format or fails a
        check, the MD5 included."""
        buf = np.frombuffer(bytes(data), np.uint8)
        u8p = C.POINTER(C.c_uint8)
        info = XttsFlacInfo()
        out = np.empty((0, 0), np.int32)
        rc = self.lib.xtts_decode_flac(self.h, buf.ctypes.data_as(u8p), buf.size, None, 0, C.byref(info))
        need = info.channels * info.total_samples
        if rc == ERR_INVALID and need > 0:          # the output did not fit: allocate what the call reported
            out = np.empty((info.channels, info.total_samples), np.int32)
            rc = self.lib.xtts_decode_flac(self.h, buf.ctypes.data_as(u8p), buf.size, _ip(out), out.size, C.byref(info))
        self._chk(rc, "decode_flac")
        out = out.reshape(info.channels, info.total_samples)
        md5 = bytes(info.md5)
        if md5 != bytes(16) and flac_md5(out, info.bits_per_sample) != md5:
            raise NativeError("decode_flac failed: MD5 mismatch", ERR_INVALID)
        return out, int(info.sample_rate), int(info.bits_per_sample)

    # ---- generation
    def submit(self, seq_id: int, text_ids, speaker_slot: int, sp: Sampling):
        t = _i32(text_ids)
        cs = sp.c()
        nb = int(getattr(sp, "num_beams", 1))
        if nb > 1:
            bm = XttsBeam(nb, float(sp.length_penalty), 1 if sp.do_sample else 0)
            self._chk(self.lib.xtts_submit_beams(self.h, seq_id, _ip(t), t.size, speaker_slot, C.byref(cs),
                                                 float(getattr(sp, "speed", 1.0)), C.byref(bm)), "submit")
            return
        self._chk(self.lib.xtts_submit_speed(self.h, seq_id, _ip(t), t.size, speaker_slot, C.byref(cs),
                                             float(getattr(sp, "speed", 1.0))), "submit")

    def debug_beam_step(self, kv_type: int, heads: int, layers: int, sp: Sampling, first: bool, advance: int, logits,
                        n_gen, ctx_len, seen, block_tables, pool, hist, state: XttsBeamState, kpool, vpool):
        """xtts_debug_beam_step: one beam step (logprob, select, reorder, partial-page copy) on caller arrays, updated in
        place: n_gen, ctx_len int32 [nb]; seen uint32 [nb][ceil(V/32)]; block_tables int32 [nb][max_pages]; pool int32
        [nb * max_pages]; hist int32 [cap][8][2]; state; kpool / vpool raw bytes [layers][n_pages][page].  Returns
        (last_tok [nb], scores [nb][V])."""
        nb = int(sp.num_beams)
        lg = _f32(logits)
        V = lg.shape[-1]
        for a, dt in ((n_gen, np.int32), (ctx_len, np.int32), (seen, np.uint32), (block_tables, np.int32), (pool, np.int32),
                      (hist, np.int32)):
            assert a.dtype == dt and a.flags.c_contiguous
        last = np.zeros(nb, np.int32)
        scores = np.zeros((nb, V), np.float32)
        page = heads * 32 * 64 * (4 if kv_type == 0 else 2)
        n_pages = kpool.nbytes // (layers * page)
        bm = XttsBeam(nb, float(sp.length_penalty), 1 if sp.do_sample else 0)
        cs = sp.c()
        self._chk(self.lib.xtts_debug_beam_step(
            self.h, kv_type, heads, layers, V, C.byref(cs), C.byref(bm), int(first), advance, _fp(lg), _ip(n_gen), _ip(ctx_len),
            _ip(last), seen.ctypes.data_as(C.POINTER(C.c_uint32)), block_tables.shape[1], _ip(block_tables), n_pages, _ip(pool),
            hist.shape[0], _ip(hist), C.byref(state), kpool.ctypes.data_as(C.c_void_p), vpool.ctypes.data_as(C.c_void_p),
            _fp(scores)), "debug_beam_step")
        return last, scores

    def cancel(self, seq_id: int):
        self._chk(self.lib.xtts_cancel(self.h, seq_id), "cancel")

    def poll(self, timeout_ms: int = 1000) -> Optional[XttsResult]:
        r = XttsResult()
        rc = self.lib.xtts_poll(self.h, C.byref(r), timeout_ms)
        if rc < 0:
            self._chk(rc, "poll")
        return r if rc == 1 else None

    def fetch(self, r: XttsResult, want_wav: bool = True, want_latents: bool = False):
        toks = np.empty((max(1, r.n_tokens),), np.int32)
        wav = np.empty((r.n_samples,), np.float32) if (want_wav and r.n_samples > 0) else None
        lat = np.empty((r.n_tokens, self.dims.gpt.hidden), np.float32) if want_latents else None
        self._chk(self.lib.xtts_fetch(self.h, r.seq_id, _ip(toks), _fp(wav), _fp(lat)), "fetch")
        return toks[: r.n_tokens], wav, lat

    def set_option(self, key: str, value: int):
        self._chk(self.lib.xtts_set_option(self.h, key.encode(), value), f"set_option({key})")

    def stats(self) -> XttsStats:
        s = XttsStats()
        self._chk(self.lib.xtts_get_stats(self.h, C.byref(s)), "get_stats")
        return s

    def sync(self):
        self._chk(self.lib.xtts_sync(self.h), "sync")

    def timer_start(self):
        """CUDA event on the engine stream (call with the engine idle)."""
        self._chk(self.lib.xtts_device_timer(self.h, 0, None), "device_timer(start)")

    def timer_stop_ms(self) -> float:
        """Second event behind everything submitted so far; milliseconds on the device clock since timer_start()."""
        ms = C.c_double(0.0)
        self._chk(self.lib.xtts_device_timer(self.h, 1, C.byref(ms)), "device_timer(stop)")
        return float(ms.value)

    def trace_start(self):
        rc = self.lib.xtts_debug_trace(self.h, 1, None, 0)
        if rc < 0:
            self._chk(rc, "debug_trace(start)")

    def trace_stop(self, cap: int = 1 << 20) -> np.ndarray:
        """-> [n, 4] int64: (ns, kernel id, phase, last-CTA flag) sorted by time; grid size in column 4 of the raw word"""
        buf = np.zeros((cap, 2), np.uint64)
        n = self.lib.xtts_debug_trace(self.h, 0, buf.ctypes.data_as(C.POINTER(C.c_uint64)), cap)
        if n < 0:
            self._chk(n, "debug_trace(stop)")
        b = buf[:n]
        out = np.stack([b[:, 0].astype(np.int64), (b[:, 1] >> np.uint64(32) & np.uint64(0xFF)).astype(np.int64),
                        (b[:, 1] & np.uint64(0xFF)).astype(np.int64), (b[:, 1] >> np.uint64(8) & np.uint64(1)).astype(np.int64),
                        (b[:, 1] >> np.uint64(40)).astype(np.int64)], axis=1)
        return out[np.argsort(out[:, 0], kind="stable")]

    def kernel_profile(self) -> Dict[str, dict]:
        """{family: {ms, flops, bytes, launches}} accumulated since option "profile" was switched on."""
        p = XttsKernelProfile()
        self._chk(self.lib.xtts_get_kernel_profile(self.h, C.byref(p)), "get_kernel_profile")
        out = {}
        for i in range(p.n):
            if p.launches[i]:
                out[bytes(p.name[i]).split(b"\0")[0].decode()] = dict(ms=p.ms[i], flops=p.flops[i], bytes=p.bytes[i],
                                                                    launches=int(p.launches[i]))
        return out

    def run_batch(self, jobs, timeout_s: float = 600.0, want_wav: bool = True, want_latents: bool = False,
                  defer_fetch: bool = False):
        """jobs: iterable of (seq_id, text_ids, speaker_slot, Sampling).  Returns {seq_id: (result, tokens, wav, lat)}.
        defer_fetch: final results stay in the engine (tokens, wav, lat are None) until the caller passes each result to
        fetch() — e.g. to copy the waveforms out of HBM after a timed region."""
        import time
        n = 0
        # batch submit: the scheduler admits nothing until the whole batch is queued, so admission waves (and with
        # them which chunks finish together and share a vocoder launch) do not depend on host timing
        self.set_option("hold_admission", 1)
        try:
            for sid, ids, spk, sp in jobs:
                self.submit(sid, ids, spk, sp)
                n += 1
        finally:
            self.set_option("hold_admission", 0)
        out, partials = {}, {}
        t_end = time.time() + timeout_s
        while len(out) < n:
            r = self.poll(1000)
            if r is None:
                if time.time() > t_end:
                    raise NativeError("run_batch timed out")
                continue
            if r.status < 0:
                self.lib.xtts_fetch(self.h, r.seq_id, None, None, None)      # releases the failed chunk's native buffers
                raise NativeError(f"sequence {r.seq_id} failed ({r.status}): {self.lib.xtts_last_error().decode()}")
            if r.status > 0:                 # partial piece (Sampling.early_tokens): kept, in order, next to the final result
                ptoks, pwav, _ = self.fetch(r, want_wav, False)
                partials.setdefault(r.seq_id, []).append((r, ptoks, pwav))
                continue
            out[r.seq_id] = (r, None, None, None) if defer_fetch else (r, *self.fetch(r, want_wav, want_latents))
        self.last_partials = partials        # {seq_id: [(result, tokens, wav), ...]} of the batch just run, oldest first
        return out


    # ---- synchronous single-stage entry points (parity tests)
    def vocode(self, latents, speaker_slot: int, stage: Optional[str] = None, stage_shape: Optional[Tuple[int, ...]] = None):
        lat = _f32(latents)
        T = lat.shape[0]
        ns = self.dims.voc.n_samples(T)
        wav = np.empty((ns,), np.float32)
        n_out = C.c_int32(0)
        st_arr = np.zeros(stage_shape, np.float32) if stage else None
        self._chk(self.lib.xtts_vocode(self.h, _fp(lat), T, speaker_slot, _fp(wav), C.byref(n_out),
                                       stage.encode() if stage else None, _fp(st_arr), st_arr.size if stage else 0), "vocode")
        assert n_out.value == ns, (n_out.value, ns)
        return (wav, st_arr) if stage else wav

    def vocode_window(self, latents, speaker_slot: int, z0: int, nz: int) -> np.ndarray:
        """z-frames [z0, z0 + nz) of the chunk as a window of its own -> nz * hop samples (include/xtts_b200.h)."""
        lat = _f32(latents)
        wav = np.empty((nz * self.dims.voc.hop,), np.float32)
        self._chk(self.lib.xtts_vocode_window(self.h, _fp(lat), lat.shape[0], speaker_slot, z0, nz, _fp(wav)), "vocode_window")
        return wav

    def vocode_speed(self, latents, speaker_slot: int, speed: float = 1.0, z0: int = 0, nz: int = -1) -> np.ndarray:
        """The vocoder at a speaking rate (xtts_vocode_speed): the whole chunk (nz < 0) -> n_samples(T, speed) samples, or
        z-frames [z0, z0 + nz) of the speed-scaled chunk as a window of its own -> nz * hop samples."""
        lat = _f32(latents)
        T = lat.shape[0]
        ok = SPEED_MIN <= speed <= SPEED_MAX                      # (the library rejects anything else)
        ns = (self.dims.voc.n_samples(T, speed) if ok else 0) if nz < 0 else nz * self.dims.voc.hop
        wav = np.empty((ns,), np.float32)
        n_out = C.c_int32(0)
        self._chk(self.lib.xtts_vocode_speed(self.h, _fp(lat), T, speaker_slot, float(speed), z0, nz, _fp(wav),
                                             C.byref(n_out)), "vocode_speed")
        assert n_out.value == ns, (n_out.value, ns)
        return wav

    def gpt_prefill(self, text_ids, speaker_slot: int, audio_tokens=(), want_hidden: bool = False):
        g = self.dims.gpt
        t, a = _i32(text_ids), _i32(list(audio_tokens))
        n = max(1, a.size)
        rows = g.n_cond_latents + t.size + 1 + max(0, a.size - 1)
        hid = np.empty((rows, g.hidden), np.float32) if want_hidden else None
        logits = np.empty((n, g.n_audio_tokens), np.float32)
        lat = np.empty((n, g.hidden), np.float32)
        self._chk(self.lib.xtts_gpt_prefill(self.h, _ip(t), t.size, speaker_slot, _ip(a) if a.size else None, a.size,
                                            _fp(hid), _fp(logits), _fp(lat)), "gpt_prefill")
        return hid, logits, lat

    def gpt_teacher_forced(self, text_ids, speaker_slot: int, forced_tokens, sp: Sampling):
        g = self.dims.gpt
        t, f = _i32(text_ids), _i32(forced_tokens)
        n = f.size
        logits = np.empty((n, g.n_audio_tokens), np.float32)
        lat = np.empty((n, g.hidden), np.float32)
        sampled = np.empty((n,), np.int32)
        cs = sp.c()
        self._chk(self.lib.xtts_gpt_teacher_forced(self.h, _ip(t), t.size, speaker_slot, _ip(f), n, C.byref(cs),
                                                   _fp(logits), _fp(lat), _ip(sampled)), "gpt_teacher_forced")
        return logits, lat, sampled

    def debug_gemm(self, mode: int, A, W, bias=None, resid=None, gelu: bool = False, iters: int = 0, out16: bool = False,
                   inplace: bool = False, pdl: bool = False):
        """One GEMM launch (xtts_debug_gemm): out16 = 16-bit output (returned widened), inplace = the residual preloaded in
        `out` and passed as both, pdl = programmatic dependent launch.  -> (out [M, N] fp32, ms per timed iteration)."""
        A, W = _f32(A), _f32(W)
        M, K = A.shape
        N = W.shape[0]
        b = _f32(bias) if bias is not None else None
        r = _f32(resid) if resid is not None else None
        out = np.empty((M, N), np.float32)
        ms = C.c_float(0)
        flags = (GEMM_GELU if gelu else 0) | (GEMM_OUT16 if out16 else 0) | (GEMM_INPLACE if inplace else 0) | (GEMM_PDL if pdl else 0)
        self._chk(self.lib.xtts_debug_gemm(self.h, mode, _fp(A), _fp(W), _fp(b), _fp(r), _fp(out), M, N, K,
                                           flags, iters, C.byref(ms)), "debug_gemm")
        return out, ms.value

    LN_GEMM_PLAIN, LN_GEMM_PDL, LN_GEMM_COUNTERS = 0, 1, 2

    def debug_ln_gemm(self, mode: int, launch: int, X, ln_w, ln_b, W, bias=None, resid=None, gelu: bool = False,
                      out16: bool = False):
        """The decode LayerNorm -> GEMM pair (xtts_debug_ln_gemm).  -> (Y [M, K] the 16-bit LN output, out [M, N], the GEMM's
        CTA count, counters [2] after the launch)."""
        X, W, lw, lb = _f32(X), _f32(W), _f32(ln_w), _f32(ln_b)
        M, K = X.shape
        N = W.shape[0]
        b = _f32(bias) if bias is not None else None
        r = _f32(resid) if resid is not None else None
        Y = np.empty((M, K), np.float32)
        out = np.empty((M, N), np.float32)
        n = C.c_int32(0)
        cnt = np.zeros(2, np.uint32)
        flags = (GEMM_GELU if gelu else 0) | (GEMM_OUT16 if out16 else 0)
        self._chk(self.lib.xtts_debug_ln_gemm(self.h, mode, launch, M, N, K, _fp(X), _fp(lw), _fp(lb), _fp(W), _fp(b), _fp(r),
                                              flags, _fp(Y), _fp(out), C.byref(n),
                                              cnt.ctypes.data_as(C.POINTER(C.c_uint32))), "debug_ln_gemm")
        return Y, out, int(n.value), cnt

    def debug_norms(self, out_type: int, X, w1, b1, w2=None, b2=None, M: Optional[int] = None, row_index=None, latents=None,
                    slots=None, lat_pos=None, n_gen=None):
        """LayerNorm (w2 None) or the GPT head norms (xtts_debug_norms).  X [x_rows, H]; latents [n_slots, lat_rows, H] is the
        incoming contents.  -> (Y [M, H] fp32, latents after or None)."""
        x = _f32(X)
        x_rows, H = x.shape
        M = M if M is not None else (len(row_index) if row_index is not None else x_rows)
        Y = np.empty((M, H), np.float32)
        lat = _f32(latents).copy() if latents is not None else None
        n_slots, lat_rows = (lat.shape[0], lat.shape[1]) if lat is not None else (0, 0)
        ri, sl, lp, ng = (_i32(a) if a is not None else None for a in (row_index, slots, lat_pos, n_gen))
        w2a = _f32(w2) if w2 is not None else None
        b2a = _f32(b2) if b2 is not None else None
        self._chk(self.lib.xtts_debug_norms(self.h, out_type, M, H, _fp(x), x_rows, _ip(ri), _fp(_f32(w1)), _fp(_f32(b1)),
                                            _fp(w2a), _fp(b2a), _fp(Y), _fp(lat), n_slots, lat_rows, _ip(sl), _ip(lp), _ip(ng)),
                  "debug_norms")
        return Y, lat

    def debug_kv_write(self, kv_type: int, heads: int, qkv, row_slot, block_tables, kpool, vpool, row_pos=None, ctx_len=None):
        """The prefill's paged-cache write (xtts_debug_kv_write).  kpool / vpool as in debug_attn_decode; ctx_len [n_slots]
        (n_slots = rows of block_tables).  -> (kpool after, vpool after)."""
        q, rs, bt = _f32(qkv), _i32(row_slot), _i32(block_tables)
        rp = _i32(row_pos) if row_pos is not None else None
        ctx = _i32(ctx_len) if ctx_len is not None else None
        dt = self.KV_DTYPES[kv_type]
        k = np.ascontiguousarray(kpool, dtype=dt).copy()
        v = np.ascontiguousarray(vpool, dtype=dt).copy()
        assert k.shape == v.shape and k.shape[1] == heads and bt.ndim == 2
        self._chk(self.lib.xtts_debug_kv_write(self.h, kv_type, heads, rs.size, _fp(q), _ip(rs), _ip(rp), bt.shape[0], _ip(ctx),
                                               _ip(bt), bt.shape[1], k.shape[0], k.ctypes.data, v.ctypes.data), "debug_kv_write")
        return k, v

    def debug_build_rows(self, rows, text_emb, text_pos, wte, wpe, spk_cond):
        """Prompt row build (xtts_debug_build_rows): rows [n, 4] = (kind, a, b, c); spk_cond [n_spk, n_cond, H].  -> X [n, H]."""
        r = _i32(rows).reshape(-1, 4)
        te, tp, a, p, s = (_f32(t) for t in (text_emb, text_pos, wte, wpe, spk_cond))
        H = te.shape[1]
        X = np.empty((r.shape[0], H), np.float32)
        self._chk(self.lib.xtts_debug_build_rows(self.h, H, s.shape[1], _fp(te), te.shape[0], _fp(tp), tp.shape[0], _fp(a), a.shape[0],
                                                 _fp(p), p.shape[0], _fp(s), s.shape[0], _ip(r), r.shape[0], _fp(X)),
                  "debug_build_rows")
        return X

    def debug_build_decode_rows(self, active, last_tok, n_gen, wte, wpe, counters=None, n_flags: int = 0):
        """Decode row build (xtts_debug_build_decode_rows): last_tok / n_gen [n_slots]; counters (uint32, incoming contents)
        whose first n_flags words the kernel zeroes.  -> (X [M, H], counters after or None)."""
        act, lt, ng = _i32(active), _i32(last_tok), _i32(n_gen)
        a, p = _f32(wte), _f32(wpe)
        H = a.shape[1]
        X = np.empty((act.size, H), np.float32)
        cnt = np.ascontiguousarray(counters, dtype=np.uint32).copy() if counters is not None else None
        self._chk(self.lib.xtts_debug_build_decode_rows(self.h, H, _fp(a), a.shape[0], _fp(p), p.shape[0], act.size, _ip(act), lt.size,
                                                        _ip(lt), _ip(ng), _fp(X),
                                                        cnt.ctypes.data_as(C.POINTER(C.c_uint32)) if cnt is not None else None,
                                                        n_flags, cnt.size if cnt is not None else 0), "debug_build_decode_rows")
        return X, cnt

    def debug_sample(self, logits, seen, sp: Sampling, step: int = 0):
        """Row b of logits [B, V] sampled as slot b with sp and seq_seed sp.seq_seed + b at step `step`; seen [B, V] (0/1)
        or None.  -> the drawn tokens [B]."""
        lg = _f32(logits)
        Bn, V = lg.shape
        sps = [Sampling(**{**sp.__dict__, "seq_seed": sp.seq_seed + b}) for b in range(Bn)]
        st = self.debug_sample_slots(V, lg, np.arange(Bn), sps, n_gen=np.full(Bn, step), cap=step + 1,
                                     seen=np.zeros((Bn, V), np.uint8) if seen is None else seen)
        return st["last_tok"]

    SAMPLE_STATE = ("n_gen", "ctx_len", "finished", "last_tok", "seen", "tokens", "sampled")

    def debug_sample_slots(self, V: int, logits, active, sps, n_gen=None, ctx_len=None, finished=None, last_tok=None,
                           seen=None, tokens=None, sampled=None, cap: Optional[int] = None, advance_ctx: int = 0,
                           forced=None):
        """One launch of the fused sampler (include/xtts_b200.h).  logits [M, ld]; active [M]; sps: one Sampling per slot.
        State arrays default to zeros (tokens / sampled to -1, with `cap` columns); n_slots = len(sps).
        -> {name: array after the launch} for every name in SAMPLE_STATE."""
        lg, act = _f32(logits), _i32(active)
        n = len(sps)
        if cap is None:
            cap = tokens.shape[1] if tokens is not None else 1
        z = lambda a, fill=0: _i32(a).copy() if a is not None else np.full(n, fill, np.int32)
        st = dict(n_gen=z(n_gen), ctx_len=z(ctx_len), finished=z(finished), last_tok=z(last_tok, -1))
        st["seen"] = (np.ascontiguousarray(seen, dtype=np.uint8).copy() if seen is not None
                      else np.zeros((n, V), np.uint8))
        for k, a in (("tokens", tokens), ("sampled", sampled)):
            st[k] = _i32(a).copy() if a is not None else np.full((n, max(cap, 0)), -1, np.int32)
        f = _i32(forced) if forced is not None else None
        for k, a in [("seen", st["seen"]), ("tokens", st["tokens"]), ("sampled", st["sampled"]), ("forced", f)]:
            if a is not None and a.size != n * (V if k == "seen" else max(cap, 0)):
                raise ValueError(f"{k} has {a.size} elements for {n} slots")
        cs = (XttsSampling * max(n, 1))(*[s.c() for s in sps])
        M = act.size
        ld = lg.shape[1] if lg.ndim == 2 else V
        self._chk(self.lib.xtts_debug_sample_slots(self.h, V, M, _ip(act), n, _fp(lg), ld, cs, cap, advance_ctx, _ip(f),
                                                   _ip(st["n_gen"]), _ip(st["ctx_len"]), _ip(st["finished"]),
                                                   _ip(st["last_tok"]), st["seen"].ctypes.data_as(C.POINTER(C.c_uint8)),
                                                   _ip(st["tokens"]), _ip(st["sampled"])), "debug_sample_slots")
        return st

    # KV type code of xtts_debug_attn_decode -> numpy dtype of the raw pool elements (bf16 as its uint16 bit pattern)
    KV_DTYPES = {0: np.float32, 1: np.uint16, 2: np.float16}

    def debug_attn_decode(self, kv_type: int, heads: int, qkv, active, ctx_len, block_tables, kpool, vpool):
        """One decode-attention launch under the current options.  kpool / vpool: [n_pages, heads, 32 * 64] raw cache
        elements in the device layout (include/xtts_b200.h), dtype KV_DTYPES[kv_type].  -> (out [M, heads*64] fp32,
        kpool after, vpool after)."""
        q, act, ctx, bt = _f32(qkv), _i32(active), _i32(ctx_len), _i32(block_tables)
        dt = self.KV_DTYPES[kv_type]
        k = np.ascontiguousarray(kpool, dtype=dt).copy()
        v = np.ascontiguousarray(vpool, dtype=dt).copy()
        assert k.shape == v.shape and k.shape[1] == heads and bt.ndim == 2 and bt.shape[0] == ctx.size
        M = act.size
        out = np.empty((M, heads * 64), np.float32)
        self._chk(self.lib.xtts_debug_attn_decode(self.h, kv_type, heads, M, _ip(act), ctx.size, _ip(ctx), _ip(bt), bt.shape[1],
                                                  k.shape[0], k.ctypes.data, v.ctypes.data, _fp(q), _fp(out)),
                  "debug_attn_decode")
        return out, k, v

    def debug_attn_prefill(self, out_type: int, heads: int, seqs, causal: bool, scale: float, q, q_row_stride: int,
                           q_head_stride: int, kv, kv_row_stride: int, kv_head_stride: int, k_off: int, v_off: int,
                           out_rows: int):
        """One prefill-attention launch.  seqs: [(q_start, nq, kv_start, nk)]; q / kv: flat fp32 buffers addressed with the
        strides (include/xtts_b200.h).  -> out [out_rows, heads*64] fp32 (NaN where no sequence writes)."""
        s, qq, kk = _i32(seqs).reshape(-1, 4), _f32(q).reshape(-1), _f32(kv).reshape(-1)
        out = np.empty((out_rows, heads * 64), np.float32)
        self._chk(self.lib.xtts_debug_attn_prefill(self.h, out_type, heads, _ip(s), s.shape[0], 1 if causal else 0, scale,
                                                   _fp(qq), qq.size, q_row_stride, q_head_stride, _fp(kk), kk.size,
                                                   kv_row_stride, kv_head_stride, k_off, v_off, _fp(out), out_rows),
                  "debug_attn_prefill")
        return out

    def debug_splitk_ln(self, mode: int, A, W, bias, X, splits: int, ln_w=None, ln_b=None):
        """Split-K 16-bit GEMM + fused residual / LayerNorm (mode 1 bf16, 2 fp16).  -> (X + bias + A.W^T, LN of it or None)."""
        A, W, b = _f32(A), _f32(W), _f32(bias)
        x = _f32(X).copy()
        M, K = A.shape
        N = W.shape[0]
        lw = _f32(ln_w) if ln_w is not None else None
        lb = _f32(ln_b) if ln_b is not None else None
        y = np.empty((M, N), np.float32) if lw is not None else None
        self._chk(self.lib.xtts_debug_splitk_ln(self.h, mode, M, N, K, splits, _fp(A), _fp(W), _fp(b), _fp(x), _fp(lw),
                                                _fp(lb), _fp(y)), "debug_splitk_ln")
        return x, y

    CONV_STORE, CONV_ACCUM = 0, 1

    def debug_conv_tc(self, x, w, up: int = 0, dil: int = 1, item_len=None, bias=None, cbias=None, resid=None,
                      mode: int = 0, slope_out: float = 0.1, scale16: float = 1.0, max_ctas: int = 0, out32=None,
                      out16=None):
        """One launch of the fast-mode vocoder convolution (include/xtts_b200.h).  x [batch, Cin, L]; w [Cout, Cin, K]
        (up 0, Conv1d) or [Cin, Cout, 2 * up] (ConvTranspose1d); cbias [batch, stride].  out32 [batch, Cout, Lout] and
        out16 [batch, Cout / 8, atoms_lpad(Lout), 8] are the incoming contents (accumulate base, sentinels); None = not
        produced.  -> (out32, out16) after the launch."""
        x, w = _f32(x), _f32(w)
        B, Cin, L = x.shape
        Cout, K = (w.shape[1], w.shape[2]) if up else (w.shape[0], w.shape[2])
        if w.shape[0 if up else 1] != Cin:
            raise ValueError(f"weight {w.shape} does not take {Cin} input channels")
        Lout = L * up if up else L
        il = _i32(item_len) if item_len is not None else None
        cb = _f32(cbias) if cbias is not None else None
        r = _f32(resid) if resid is not None else None
        b = _f32(bias) if bias is not None else None
        o32 = _f32(out32).copy() if out32 is not None else None
        o16 = _f32(out16).copy() if out16 is not None else None
        for name, a, n in [("item_len", il, B), ("bias", b, Cout), ("resid", r, B * Cout * Lout),
                           ("out32", o32, B * Cout * Lout), ("out16", o16, B * Cout * atoms_lpad(Lout))]:
            if a is not None and a.size != n:
                raise ValueError(f"{name} has {a.size} elements, expected {n}")
        if cb is not None and (cb.ndim != 2 or cb.shape[0] != B):
            raise ValueError(f"cbias must be [batch, stride], got {cb.shape}")
        self._chk(self.lib.xtts_debug_conv_tc(self.h, up, Cin, Cout, K, dil, B, L, _ip(il), _fp(w), _fp(b), _fp(cb),
                                              cb.shape[1] if cb is not None else 0, _fp(x), _fp(r), mode, slope_out,
                                              scale16, max_ctas, _fp(o32), _fp(o16)), "debug_conv_tc")
        return o32, o16

    def debug_cond(self, op, dims, inputs=(), out=None, out_len: Optional[int] = None, scal=()):
        """One conditioning kernel (xtts_debug_cond).  op: a name of COND_OPS or its code; inputs: arrays, flattened to fp32;
        out: the incoming contents (the base of the in-place ops), else out_len floats of NaN.  -> out after, flat fp32."""
        code = COND_OP[op] if isinstance(op, str) else int(op)
        d = _i32(dims).reshape(-1)
        s = _f32(scal).reshape(-1)
        ins = [_f32(a).reshape(-1) for a in inputs]
        o = _f32(out).reshape(-1).copy() if out is not None else np.full(int(out_len), np.nan, np.float32)
        ptrs = (C.POINTER(C.c_float) * max(len(ins), 1))(*[_fp(a) for a in ins])
        lens = (C.c_int64 * max(len(ins), 1))(*[a.size for a in ins])
        self._chk(self.lib.xtts_debug_cond(self.h, code, _ip(d), d.size, _fp(s) if s.size else None, s.size, ptrs, lens,
                                           len(ins), _fp(o), o.size), "debug_cond")
        return o
