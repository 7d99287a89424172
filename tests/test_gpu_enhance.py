"""GPU: `xtts_enhance` (TTSRequest.enhance_speech) against the goldens the reference's own enhancer module produced and
against the repo oracle (oracle/enhance_oracle.py) stage by stage, its boundaries, determinism, and the end-to-end
conditioning path through TTS.generate_speech.

Tolerance: the output is 16-bit PCM (rint(x * 32767) / 32768), so a value that differs from the reference by less than
the fp32 STFT error can still round to the neighbouring code: one LSB (1/32768).  On top of that the fp32 DFT-by-GEMM
STFTs (2048-term sums, forward and inverse) and the fp32 frame sums differ from numpy's fp64 FFTs by a few 1e-6 of
full scale: STFT_ERR = 2e-5 (0.66 LSB).  A flipped VAD decision or loudness gate would move samples by orders of
magnitude more than this, so a pass also means identical decisions; the inputs' distance from every threshold is
asserted, not assumed."""
import os
import sys
import wave
from dataclasses import asdict

import numpy as np
import pytest

from oracle import enhance_oracle as E

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]
GOLD = os.path.join(os.path.dirname(__file__), "golden")
sys.path.insert(0, GOLD)
import make_enhance_golden as G          # noqa: E402

LSB = 1.0 / 32768
STFT_ERR = 2e-5
TOL = LSB + STFT_ERR
_OFF = dict(trim_silence=False, remove_noise=False, enhance_speech=False, normalize=False)
STAGES = {"vad": {**_OFF, "trim_silence": True}, "gate": {**_OFF, "remove_noise": True},
          "clarity": {**_OFF, "enhance_speech": True}, "loudness": {**_OFF, "normalize": True}}


def _margins(x, cfg):
    """Asserts every VAD frame decision is >= 1e-3 from the threshold and every finite loudness block >= 0.1 LU from
    both gates (oracle intermediates); returns the oracle's taps."""
    taps = {}
    E.process(x, cfg, taps)
    if "vad" in taps:
        assert np.abs(np.abs(taps["vad"]) - cfg.vad_threshold).min() >= 1e-3
    if "blocks" in taps:
        b = taps["blocks"][np.isfinite(taps["blocks"])]
        for g in taps["gates"]:
            assert np.abs(b - g).min() >= 0.1, g
    return taps


@pytest.mark.parametrize("name", list(G.CASES))
def test_enhance_matches_reference_goldens(engine_small, name):
    x, cfg = G.case_input(name), G.case_config(name)
    taps = _margins(x, cfg)
    out = engine_small.enhance(x, cfg)
    want = G.golden_codes(name).astype(np.float32) / 32768       # the reference's 16-bit file, read back
    assert out.shape == want.shape
    err = np.abs(out - want).max()
    print(name, "max err", err, "LSB", err / LSB)
    assert err <= TOL
    if G.CASES[name][3] is not None:                          # a span of exact silence
        # the gating stage's NaN samples: present in the reference, zeroed by the clarity stage's nan_to_num; every sample
        # the oracle leaves exactly 0 is exactly 0 here too
        assert np.isnan(taps["after_gate"]).sum() > 15000
        zero = taps["after_clarity"] == 0
        assert zero.sum() > 10000
        assert np.all(out[zero] == 0)


@pytest.mark.parametrize("stage", list(STAGES))
@pytest.mark.parametrize("seconds", [5.0, 60.0, 75.0])
def test_each_stage_matches_oracle(engine_small, stage, seconds):
    """75 s is longer than max_ref_length: the reference enhances the whole file before truncating."""
    x = E.synthetic_input(seconds, 22050, 42)
    cfg = E.EnhanceConfig(**STAGES[stage])
    _margins(x, cfg)
    out, want = engine_small.enhance(x, cfg), E.enhance(x, cfg)
    assert out.shape == want.shape
    assert np.abs(out - want).max() <= TOL, np.abs(out - want).max()


def test_all_stages_long_with_silence(engine_small):
    x = E.synthetic_input(60.0, 22050, 42, silence=(20.0, 22.0))
    cfg = E.EnhanceConfig()
    _margins(x, cfg)
    out, want = engine_small.enhance(x, cfg), E.enhance(x, cfg)
    assert np.abs(out - want).max() <= TOL


def _invalid(eng, x, cfg):
    from auralis_b200 import native
    with pytest.raises(native.NativeError) as ei:
        eng.enhance(x, cfg)
    assert ei.value.code == native.ERR_INVALID


def test_boundaries(engine_small):
    x = E.synthetic_input(2.0, 22050, 7)
    vad = E.EnhanceConfig(**STAGES["vad"])
    for n in (4096, 4097):                                   # one VAD frame and just above
        out, want = engine_small.enhance(x[:n], vad), E.enhance(x[:n], vad)
        assert np.abs(out - want).max() <= TOL
    _invalid(engine_small, x[:4095], vad)
    loud = E.EnhanceConfig(**STAGES["loudness"])
    for n in (8820, 8821):                                   # 0.4 s at 22.05 kHz and just above
        out, want = engine_small.enhance(x[:n], loud), E.enhance(x[:n], loud)
        assert np.abs(out - want).max() <= TOL
    _invalid(engine_small, x[:8819], loud)
    gate = E.EnhanceConfig(**STAGES["gate"])
    for n in (512 * 10 + 3, 512 * 24 - 1):                  # 11 and 24 STFT frames: fewer than noise_reduce_frames
        out, want = engine_small.enhance(x[:n], gate), E.enhance(x[:n], gate)
        assert out.shape == want.shape and np.abs(out - want).max() <= TOL
    _invalid(engine_small, np.zeros(22050, np.float32), E.EnhanceConfig(**STAGES["loudness"]))   # below the -70 LUFS gate
    bad = x.copy(); bad[100] = np.nan
    _invalid(engine_small, bad, E.EnhanceConfig())
    _invalid(engine_small, x, E.EnhanceConfig(noise_reduce_frames=0))


def test_deterministic(engine_small):
    x = E.synthetic_input(5.0, 22050, 3, silence=(1.0, 2.0))
    a = engine_small.enhance(x, E.EnhanceConfig())
    b = engine_small.enhance(x, E.EnhanceConfig())
    assert a.tobytes() == b.tobytes()


def test_time_counts_as_conditioning(engine_small):
    before = engine_small.stats().cond_ms
    engine_small.enhance(E.synthetic_input(5.0, 22050, 3), E.EnhanceConfig())
    assert engine_small.stats().cond_ms > before


# ---------------------------------------------------------------------------------------------------- end to end
def _write_wav(path, x, sr=22050):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1); w.setsampwidth(2); w.setframerate(sr)
        w.writeframes((np.clip(x, -1, 1) * 32767).astype(np.int16).tobytes())
    return str(path)


@pytest.fixture(scope="module")
def tts(tmp_path_factory, dims_small, state_small):
    from auralis_b200 import TTS
    from auralis_b200.weights import save_model_dir
    d = tmp_path_factory.mktemp("model")
    save_model_dir(str(d), dims_small, state_small[0], state_small[1])
    t = TTS(scheduler_max_concurrency=8).from_pretrained(str(d), precision="fp32", max_concurrency=4)
    yield t
    t.loop.run_until_complete(t.shutdown())


def _condition_like_engine(ne, slot, audios):
    """What get_audio_conditioning does with the loaded (here: given) audio of a list of speaker files."""
    from auralis_b200.engine import _resample
    gs = []
    for a in audios:
        ne.condition(slot, a, _resample(a, 22050, 16000), 30, 4)
        gs.append(ne.get_speaker(slot)[1])
    ne.condition(slot, np.concatenate(audios), _resample(audios[0], 22050, 16000), 30, 4)
    c, _ = ne.get_speaker(slot)
    return c, np.mean(np.stack(gs), axis=0)


def test_generate_speech_conditions_on_enhanced_audio(tts, tmp_path):
    from auralis_b200 import TTSRequest
    from auralis_b200.engine import load_audio
    files = [_write_wav(tmp_path / "a.wav", E.synthetic_input(3.0, 22050, 21, silence=(1.0, 1.8))),
             _write_wav(tmp_path / "b.wav", E.synthetic_input(2.5, 22050, 22))]
    eng = tts.tts_engine
    req = TTSRequest(text="A short sentence to speak.", speaker_files=files, language="en", temperature=0.0,
                     enhance_speech=True)
    out = tts.generate_speech(req)
    assert out.array.size > 0
    n_keys = len(eng._spk_arrays)
    cond, g = tts.loop.run_until_complete(eng.get_audio_conditioning(files, 60, 30, 4, enhance=req.audio_config))
    assert len(eng._spk_arrays) == n_keys                    # the request's own conditioning, from the cache
    cfg = E.EnhanceConfig(**asdict(req.audio_config))
    audios = [E.enhance(load_audio(f, 22050), cfg) for f in files]
    rc, rg = _condition_like_engine(eng.native, eng.max_speakers - 1, audios)
    cond, g = np.asarray(cond)[0], np.asarray(g).reshape(-1)
    assert np.abs(cond - rc).max() < 2e-3 * max(1.0, np.abs(rc).max()), np.abs(cond - rc).max()
    assert np.abs(g - rg).max() < 2e-4, np.abs(g - rg).max()


def test_plain_request_conditioning_is_unchanged(tts, tmp_path):
    from auralis_b200 import TTSRequest
    from auralis_b200.engine import load_audio
    files = [_write_wav(tmp_path / "c.wav", E.synthetic_input(2.0, 22050, 23)),
             _write_wav(tmp_path / "d.wav", E.synthetic_input(2.2, 22050, 24))]
    eng = tts.tts_engine
    req = TTSRequest(text="Another short sentence.", speaker_files=files, language="en", temperature=0.0)
    tts.generate_speech(req)
    cond, g = tts.loop.run_until_complete(eng.get_audio_conditioning(files, 60, 30, 4))
    rc, rg = _condition_like_engine(eng.native, eng.max_speakers - 1, [load_audio(f, 22050) for f in files])
    assert np.asarray(cond)[0].tobytes() == rc.tobytes()
    assert np.asarray(g).reshape(-1).tobytes() == rg.astype(np.float32).tobytes()
