"""CPU: the speaker-reference enhancer (`TTSRequest.enhance_speech`).  The repo oracle against the reference's own
enhancer module (librosa / pyloudnorm restated and injected), the restatements against published values, and the host
logic around `xtts_enhance` with a fake native layer."""
import asyncio
import hashlib
import os
import sys
import threading
import wave
from dataclasses import asdict

import numpy as np
import pytest

from oracle import enhance_oracle as E
from oracle import ref_import

GOLD = os.path.join(os.path.dirname(__file__), "golden")
sys.path.insert(0, GOLD)
import make_enhance_golden as G          # noqa: E402

live = pytest.mark.skipif(not ref_import.available(), reason="reference tree not mounted")
pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")      # the gating stage's 0/0 is reference behaviour


# ---------------------------------------------------------------------------------------------------- oracle vs reference
@live
@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_matches_reference_goldens(name):
    from oracle import ref_enhance
    gold = G.golden_codes(name)
    x, cfg = G.case_input(name), G.case_config(name)
    ours = E.process(x, cfg)
    ref = ref_enhance.process(x, **asdict(cfg))
    assert ours.shape == ref.shape == gold.shape
    assert np.abs(ours - ref).max() <= 1e-6
    # the stored 16-bit codes: within 1e-6 of full scale of rounding the oracle's output to the nearest code
    assert np.abs(np.asarray(ours, np.float64) * 32767.0 - gold).max() <= 0.5 + 1e-6 * 32767


@live
@pytest.mark.parametrize("seed,sr,silence,over", [
    (101, 22050, None, {}),
    (102, 22050, (0.5, 1.5), {"noise_reduce_frames": 7, "noise_reduce_margin": 1.5}),
    (103, 16000, None, {"vad_frame_length": 256, "vad_threshold": 0.5}),       # VAD energy curve longer than the mel one
    (104, 24000, (2.0, 2.9), {"enhance_amount": 0.3, "target_lufs": -14.0, "trim_silence": False}),
])
def test_oracle_matches_reference_fresh(seed, sr, silence, over):
    from oracle import ref_enhance
    x = E.synthetic_input(3.1, sr, seed, silence)
    cfg = E.EnhanceConfig(**{"sample_rate": sr, **over})
    ours, ref = E.process(x, cfg), ref_enhance.process(x, **asdict(cfg))
    assert ours.shape == ref.shape
    np.testing.assert_allclose(ours, ref, rtol=0, atol=1e-6)


def test_golden_file_is_small_and_complete():
    z = np.load(os.path.join(GOLD, "enhance_reference.npz"))
    assert set(G.CASES) <= set(z.files)
    assert all(z[n].dtype == np.int16 for n in G.CASES)
    assert os.path.getsize(os.path.join(GOLD, "enhance_reference.npz")) < 256 * 1024


# ---------------------------------------------------------------------------------------------------- restatements
@pytest.mark.parametrize("n", [4096, 10000, 22050 + 7])
def test_istft_inverts_stft(n):
    x = np.random.default_rng(n).standard_normal(n).astype(np.float32) * 0.3
    y = E.librosa.istft(E.librosa.stft(x))
    assert y.shape == (512 * (n // 512),)
    assert np.abs(y - x[: y.size]).max() < 1e-6


def test_high_shelf_48k_matches_bs1770():
    """ITU-R BS.1770-4 Table 1 (stage 1 pre-filter at 48 kHz)."""
    (b, a), _ = E.kweighting(48000)
    np.testing.assert_allclose(b, [1.53512485958697, -2.69169618940638, 1.19839281085285], atol=1e-3)
    np.testing.assert_allclose(a, [1.0, -1.69065929318241, 0.73248077421585], atol=1e-3)


@pytest.mark.parametrize("sr", [48000, 22050])
def test_full_scale_997hz_sine_is_minus_3_lufs(sr):
    x = np.sin(2 * np.pi * 997 * np.arange(5 * sr) / sr)
    assert abs(E.Meter(sr).integrated_loudness(x) - (-3.01)) < 0.1


@pytest.mark.parametrize("n", [2, 3, 130, 4097, 66150, 1323000])
def test_linspace_is_index_times_step(n):
    """The VAD kernel's index map: np.linspace(0, 1, n)[i] == i * (1 / (n - 1)), last point exactly 1."""
    i = np.arange(n, dtype=np.float64)
    want = i * (1.0 / (n - 1))
    want[-1] = 1.0
    np.testing.assert_array_equal(np.linspace(0, 1, n), want)


def test_reference_failure_conditions():
    cfg = E.EnhanceConfig()
    with pytest.raises(E.ParameterError):
        E.enhance(E.synthetic_input(0.18, 22050, 1), cfg)                  # shorter than one VAD frame (4096)
    with pytest.raises(ValueError):
        E.enhance(E.synthetic_input(0.3, 22050, 1), cfg)                   # shorter than one 400 ms loudness block
    with pytest.raises(ValueError):
        E.enhance(np.zeros(22050, np.float32), E.EnhanceConfig(trim_silence=False))     # every block below -70 LUFS


# ---------------------------------------------------------------------------------------------------- host logic
class _FakeNative:
    def __init__(self, dims, fail=None):
        self.dims, self.fail = dims, fail
        self.enhance_calls, self.cond_inputs = [], []
        self.slots = {}

    def enhance(self, wav, cfg):
        from auralis_b200 import native
        self.enhance_calls.append((wav.size, cfg))
        if self.fail is not None:
            raise native.NativeError("enhance failed (%d): too short" % self.fail, self.fail)
        return np.asarray(wav, np.float32)[: 512 * (wav.size // 512)] * 0.5

    def condition(self, slot, w22, w16, *a):
        self.cond_inputs.append(np.asarray(w22).copy())
        self.slots[slot] = (np.full((self.dims.gpt.n_cond_latents, self.dims.gpt.hidden), float(np.abs(w22).sum()), np.float32),
                            np.ones(self.dims.voc.d_vector, np.float32))

    def get_speaker(self, slot):
        return self.slots[slot]

    def set_speaker(self, slot, c, g):
        self.slots[slot] = (c, g)


def _engine(fail=None):
    from auralis_b200.config import XTTSDims
    from auralis_b200.engine import XTTSv2Engine
    from auralis_b200.speakers import SpeakerSlots
    from auralis_b200.text import XTTSTokenizer
    dims = XTTSDims.small()
    eng = object.__new__(XTTSv2Engine)
    eng.dims, eng.max_speakers = dims, 4
    eng.native = _FakeNative(dims, fail)
    eng.natives = [eng.native]
    eng._spk = SpeakerSlots(4)
    eng._spks = [eng._spk]
    eng._spk_arrays = {}
    eng.tokenizer = XTTSTokenizer(dims.gpt.n_text_tokens, dims.gpt.max_text_tokens)
    eng.mel_eos_token_id = dims.gpt.stop_audio_token
    eng.early_emit_tokens = 0
    eng._wlock, eng._id_lock = threading.Lock(), threading.Lock()
    return eng


def _wav_file(tmp_path, name, seconds=1.0):
    x = E.synthetic_input(seconds, 22050, 5)
    p = tmp_path / name
    with wave.open(str(p), "wb") as w:
        w.setnchannels(1); w.setsampwidth(2); w.setframerate(22050)
        w.writeframes((x * 32767).astype(np.int16).tobytes())
    return str(p)


def _run(coro):
    return asyncio.new_event_loop().run_until_complete(coro)


def _old_key(paths, *params):
    hk = hashlib.sha256()
    for p in paths:
        st = os.stat(p)
        hk.update(f"{p}|{st.st_size}|{st.st_mtime_ns}".encode())
    hk.update("|".join(str(v) for v in params).encode())
    return hk.hexdigest()


def test_default_request_does_not_enhance_and_keeps_the_key(tmp_path):
    from auralis_b200 import TTSRequest
    f = _wav_file(tmp_path, "a.wav")
    eng = _engine()
    req = TTSRequest(text="hello there", speaker_files=[f], language="en")
    _run(eng.get_generation_context(req))
    assert eng.native.enhance_calls == []
    assert list(eng._spk_arrays) == [_old_key([f], 60, 30, 4, False, 22050)]


def test_enhanced_key_differs_from_plain_and_between_configs(tmp_path):
    from auralis_b200 import TTSRequest
    from auralis_b200.requests import AudioPreprocessingConfig
    f = _wav_file(tmp_path, "a.wav")
    eng = _engine()
    for req in (TTSRequest(text="hi", speaker_files=[f], language="en"),
                TTSRequest(text="hi", speaker_files=[f], language="en", enhance_speech=True),
                TTSRequest(text="hi", speaker_files=[f], language="en", enhance_speech=True,
                           audio_config=AudioPreprocessingConfig(target_lufs=-23.0))):
        _run(eng.get_generation_context(req))
    assert len(eng._spk_arrays) == 3
    assert len(eng.native.enhance_calls) == 2
    assert eng.native.enhance_calls[1][1].target_lufs == -23.0
    # the enhanced audio (the fake halves it) is what was conditioned
    assert np.allclose(eng.native.cond_inputs[1], eng.native.cond_inputs[0][: eng.native.cond_inputs[1].size] * 0.5, atol=1e-6)


def test_single_str_speaker_file_is_not_enhanced(tmp_path):
    from auralis_b200 import TTSRequest
    f = _wav_file(tmp_path, "a.wav")
    eng = _engine()
    req = TTSRequest(text="hi", speaker_files=f, language="en", enhance_speech=True)
    assert req.enhance_config() is None
    _run(eng.get_generation_context(req))
    assert eng.native.enhance_calls == []


def test_invalid_enhance_falls_back_with_one_warning(tmp_path):
    from auralis_b200 import TTSRequest, native
    f = _wav_file(tmp_path, "a.wav")
    eng = _engine(fail=native.ERR_INVALID)
    req = TTSRequest(text="hi", speaker_files=[f], language="en", enhance_speech=True)
    with pytest.warns(RuntimeWarning) as rec:
        _run(eng.get_generation_context(req))
    assert len([w for w in rec if "enhance_speech" in str(w.message)]) == 1
    plain = _engine()
    _run(plain.get_generation_context(TTSRequest(text="hi", speaker_files=[f], language="en")))
    np.testing.assert_array_equal(eng.native.cond_inputs[0], plain.native.cond_inputs[0])


def test_other_enhance_errors_propagate(tmp_path):
    from auralis_b200 import TTSRequest, native
    f = _wav_file(tmp_path, "a.wav")
    eng = _engine(fail=-2)
    with pytest.raises(native.NativeError):
        _run(eng.get_generation_context(TTSRequest(text="hi", speaker_files=[f], language="en", enhance_speech=True)))


def test_request_no_longer_warns_and_copy_carries_audio_config(recwarn):
    from auralis_b200 import TTSRequest
    from auralis_b200.requests import AudioPreprocessingConfig
    ac = AudioPreprocessingConfig(sample_rate=16000, vad_threshold=0.05, noise_reduce_frames=10, target_lufs=-20.0)
    r = TTSRequest(text="hi", speaker_files=["a.wav"], language="en", enhance_speech=True, audio_config=ac)
    assert not [w for w in recwarn if "enhance" in str(w.message)]
    c = r.copy()
    assert c.enhance_speech and asdict(c.audio_config) == asdict(ac)
    assert asdict(AudioPreprocessingConfig()) == asdict(E.EnhanceConfig())      # the reference's defaults


def test_enhance_config_struct_layout():
    import ctypes
    from auralis_b200 import native
    assert ctypes.sizeof(native.XttsEnhanceConfig) == 11 * 4
    c = native.XttsEnhanceConfig.of(E.EnhanceConfig(enhance_amount=0.5))
    assert (c.sample_rate, c.vad_frame_length, c.noise_reduce_frames, c.normalize) == (22050, 4096, 25, 1)
    assert abs(c.enhance_amount - 0.5) < 1e-7 and abs(c.target_lufs + 18.0) < 1e-6
