"""CPU: the public façade (`auralis_b200.TTS` / `TTSRequest` / `TTSOutput`) against the REFERENCE's own classes
(`auralis.core.tts.TTS` etc.).  Both are driven by the same fake engine — per chunk one waveform whose values encode
(request text length, chunk index), earlier chunks finishing LATER — and must return the same audio in the same order for:
one-shot generation, streaming, several chunks, the 100 000-character request split (`split_requests`), a prepared speaker
(`prepare_for_streaming_generation`), the async API, and a failing chunk.  What the reference's classes returned in every
case is stored in tests/golden/facade_reference.npz (made by tests/golden/make_facade_golden.py, which imports them
unmodified through oracle/ref_facade.py and runs the `case_*` functions below on them)."""
import asyncio
import io
import json
import os
import wave

import numpy as np
import pytest

import auralis_b200 as ours

pytestmark = pytest.mark.timeout(120)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "facade_reference.npz")
GENERATE_CHARS = [5, 55, 200]
LOAD_AUDIO_CASES = [(48000, 2), (22050, 1), (16000, 1), (44100, 2)]


def make_engine(ns_output, cond_config, fail_at=None):
    """A fake engine speaking the plugin API (`models/base.py:57-224`); `ns_output` is the TTSOutput class of the side under
    test, so each façade receives its own output type."""

    class Engine:
        def __init__(self):
            self.cond_calls = 0

        @property
        def conditioning_config(self):
            return cond_config

        async def get_audio_conditioning(self, speaker_files, *a, **k):
            self.cond_calls += 1
            return np.full((1, 32, 8), 0.5, np.float32), np.full((1, 4, 1), 0.25, np.float32)

        async def get_generation_context(self, request, gpt_cond_latent=None, speaker_embeddings=None):
            if gpt_cond_latent is None:
                gpt_cond_latent, speaker_embeddings = await self.get_audio_conditioning(request.speaker_files)
            n = max(1, len(request.text) // 10)

            async def gen(i):
                await asyncio.sleep(0.003 * (n - i))
                if fail_at == i:
                    raise RuntimeError(f"chunk {i} exploded")
                yield (len(request.text), i)
            return [gen(i) for i in range(n)], [f"{request.request_id}_{i}" for i in range(n)], speaker_embeddings, [gpt_cond_latent] * n

        async def process_tokens_to_speech(self, generator, speaker_embeddings, multimodal_data=None, request=None):
            assert speaker_embeddings is not None and multimodal_data is not None
            async for (L, i) in generator:
                yield ns_output(array=np.full(3 + i, float(1000 * L + i), np.float32), token_length=i + 1,
                                start_time=getattr(request, "start_time", None))

        async def shutdown(self):
            pass
    return Engine()


class Side:
    """One façade: `make_tts(conc, fail_at)` -> a TTS driven by the fake engine; Req / Out = its request / output classes."""

    def __init__(self, make_tts, Req, Out):
        self.make_tts, self.Req, self.Out = make_tts, Req, Out


def ours_side():
    from auralis_b200.base import ConditioningConfig as CC
    return Side(lambda conc=4, fail_at=None: ours.TTS(scheduler_max_concurrency=conc).from_engine(
        make_engine(ours.TTSOutput, CC(True, True), fail_at=fail_at)), ours.TTSRequest, ours.TTSOutput)


# ---- the cases: each runs one scenario on one side and returns plain data (lists, numbers, strings)
def case_generate_speech(side, n_chars):
    out = side.make_tts().generate_speech(side.Req(text="x" * n_chars, speaker_files=["s.wav"], language="en"))
    return [np.asarray(out.array).tolist(), out.sample_rate]


def case_streaming(side):
    chunks = list(side.make_tts().generate_speech(side.Req(text="y" * 64, speaker_files=["s.wav"], language="en", stream=True)))
    return [[np.asarray(c.array).tolist(), c.token_length] for c in chunks]


def case_split(side):
    tts = side.make_tts()
    parts = tts.split_requests(side.Req(text="z" * 250_035, speaker_files=["s.wav"], language="en"), max_length=100_000)
    lens = [len(p.text) for p in parts]
    assert len({p.request_id for p in parts}) == len(parts)
    # and the audio of a (smaller) split request is the concatenation of its parts, in order
    tts = side.make_tts()
    tts.split_requests = lambda request, max_length=100000, _f=type(tts).split_requests: _f(request, 30)
    out = tts.generate_speech(side.Req(text="w" * 75, speaker_files=["s.wav"], language="en"))
    return [lens, np.asarray(out.array).tolist()]


def case_prepared_speaker_and_async(side):
    tts = side.make_tts()
    Req = side.Req
    fn = tts.loop.run_until_complete(tts.prepare_for_streaming_generation(Req(text="q" * 40, speaker_files=["s.wav"], language="en")))
    calls = tts.tts_engine.cond_calls

    async def go():
        a = await tts.generate_speech_async(Req(text="q" * 40, speaker_files=["s.wav"], language="en", context_partial_function=fn))
        gen = await tts.generate_speech_async(Req(text="q" * 30, speaker_files=["s.wav"], language="en", stream=True,
                                                  context_partial_function=fn))
        b = [np.asarray(c.array).tolist() async for c in gen]
        return [np.asarray(a.array).tolist(), b]
    res = tts.loop.run_until_complete(go())
    assert tts.tts_engine.cond_calls == calls                  # the prepared conditioning is reused, not recomputed
    return res


def case_failing_chunk(side):
    try:
        side.make_tts(fail_at=1).generate_speech(side.Req(text="x" * 30, speaker_files=["s.wav"], language="en"))
    except Exception as e:      # noqa: BLE001 — the type is what is compared
        return [type(e).__name__, str(e)]
    return None


def case_request_defaults(side):
    r = side.Req(text="hi", speaker_files=["a.wav"])
    fields = {f: getattr(r, f) for f in ("temperature", "top_p", "top_k", "repetition_penalty", "length_penalty", "do_sample",
                                         "max_ref_length", "gpt_cond_len", "gpt_cond_chunk_len", "stream", "enhance_speech",
                                         "load_sample_rate", "sound_norm_refs", "language")}
    try:
        side.Req(text="hi", speaker_files=["a.wav"], language="klingon")
        rejected = None
    except ValueError:
        rejected = "ValueError"
    return [fields, rejected]


def case_output_helpers(side):
    """TTSOutput: bytes constructor (int16 + fade-in), combine_outputs, pcm encodings, resample, get_info, from_tensor."""
    import torch
    Out = side.Out
    rng = np.random.RandomState(1)
    x = (rng.rand(4800).astype(np.float32) * 1.9 - 0.95)
    pcm = (rng.randint(-30000, 30000, size=600)).astype(np.int16).tobytes()
    a, b, c = Out(array=x.copy()), Out(array=x[::-1].copy()), Out(array=pcm)
    comb = Out.combine_outputs([a, b, c])
    rs = a.resample(16000)
    try:
        a.to_bytes("ogg")
        ogg = None
    except ValueError:
        ogg = "ValueError"
    return {"from_bytes": np.asarray(c.array), "comb": np.asarray(comb.array), "comb_sr": comb.sample_rate,
            "pcm2": a.to_bytes("pcm", 2).hex(), "pcm4": a.to_bytes("pcm", 4).hex(), "pcm1": a.to_bytes("pcm", 1).hex(),
            "rs": np.asarray(rs.array), "rs_sr": rs.sample_rate, "info": a.get_info(), "ogg": ogg,
            "ft": np.asarray(Out.from_tensor(torch.from_numpy(x)[None], 22050).array), "tensor": a.to_tensor().numpy()}


def wav_bytes(sr, nch, seconds=0.25, seed=0):
    rng = np.random.RandomState(seed)
    x = (rng.rand(int(sr * seconds), nch) * 1.6 - 0.8)
    buf = io.BytesIO()
    with wave.open(buf, "wb") as w:
        w.setnchannels(nch); w.setsampwidth(2); w.setframerate(sr)
        w.writeframes((x * 32767).astype(np.int16).tobytes())
    return buf.getvalue()


def randomised_cases():
    """30 random (length, stream, failing chunk, scheduler concurrency) cases"""
    rng = np.random.RandomState(2024)
    out = []
    for _ in range(30):
        n_chars = int(rng.randint(1, 140))
        stream = bool(rng.randint(2))
        n_chunks = max(1, n_chars // 10)
        fail_at = int(rng.randint(n_chunks)) if rng.rand() < 0.25 else None
        conc = int(rng.choice([1, 2, 5, 16]))
        out.append((n_chars, stream, fail_at, conc))
    return out


def case_randomised(side, n_chars, stream, fail_at, conc):
    tts = side.make_tts(conc, fail_at)
    try:
        out = tts.generate_speech(side.Req(text="r" * n_chars, speaker_files=["s.wav"], language="en", stream=stream))
        if stream:
            return ["ok", [np.asarray(c.array).tolist() for c in out]]
        return ["ok", np.asarray(out.array).tolist()]
    except Exception as e:      # noqa: BLE001
        return ["err", type(e).__name__, str(e)]


def record(side):
    """Every case on one side -> {name: JSON string or array} (the golden file's content)"""
    rec = {f"generate_{n}": case_generate_speech(side, n) for n in GENERATE_CHARS}
    rec.update(streaming=case_streaming(side), split=case_split(side), prepared=case_prepared_speaker_and_async(side),
               failing=case_failing_chunk(side), defaults=case_request_defaults(side),
               randomised=[case_randomised(side, *c) for c in randomised_cases()])
    out = {k: json.dumps(v) for k, v in rec.items()}
    for k, v in case_output_helpers(side).items():
        out["helpers_" + k] = v if isinstance(v, np.ndarray) else json.dumps(v)
    return out


@pytest.fixture(scope="module")
def ref():
    """What the reference's classes returned: {name: decoded JSON value or array}"""
    with np.load(GOLDEN) as z:
        return {k: (z[k] if z[k].dtype.kind != "U" else json.loads(str(z[k]))) for k in z.files}


def _same(got, want):
    return json.loads(json.dumps(got)) == want


@pytest.mark.parametrize("n_chars", GENERATE_CHARS)
def test_generate_speech_same_audio(ref, n_chars):
    got = case_generate_speech(ours_side(), n_chars)
    assert _same(got, ref[f"generate_{n_chars}"]) and got[1] == 24000


def test_streaming_same_chunks_in_same_order(ref):
    got = case_streaming(ours_side())
    assert _same(got, ref["streaming"]) and len(got) == 6


def test_long_request_is_split_like_the_reference(ref):
    got = case_split(ours_side())
    assert _same(got, ref["split"]) and got[0] == [100_000, 100_000, 50_035]


def test_prepared_speaker_and_async_api(ref):
    assert _same(case_prepared_speaker_and_async(ours_side()), ref["prepared"])


def test_failing_chunk_raises_the_same_error(ref):
    got = case_failing_chunk(ours_side())
    assert _same(got, ref["failing"]) and got == ["RuntimeError", "chunk 1 exploded"]


def test_request_defaults_and_validation_match(ref):
    got = case_request_defaults(ours_side())
    for f, v in ref["defaults"][0].items():
        assert got[0][f] == v, f
    assert got[1] == ref["defaults"][1] == "ValueError"


def test_output_helpers_match(ref):
    """TTSOutput: bytes constructor (int16 + fade-in), combine_outputs, pcm encodings, resample, get_info, from_tensor."""
    got = case_output_helpers(ours_side())
    for k, v in got.items():
        want = ref["helpers_" + k]
        if isinstance(v, np.ndarray):
            np.testing.assert_array_equal(v, want, err_msg=k)
        else:
            assert _same(v, want), k
    assert got["ogg"] == "ValueError"


def test_load_audio_matches_the_reference_pipeline(ref, tmp_path):
    """common/utilities.py:72-97 (mono mix, torchaudio resample, clip; the golden was made with `torchaudio.load` replaced by a
    stdlib WAV reader): same samples as `auralis_b200.engine.load_audio` for a 48 kHz stereo 16-bit file, a 22.05 kHz mono
    one and in-memory bytes."""
    from auralis_b200.engine import load_audio
    for sr, nch in LOAD_AUDIO_CASES:
        b = wav_bytes(sr, nch, seed=sr)
        want = ref[f"load_audio_{sr}_{nch}"]
        got = load_audio(b, 22050)
        assert got.dtype == np.float32 and got.shape == want.shape
        np.testing.assert_allclose(got, want, atol=1e-6, rtol=0)
        f = tmp_path / f"a{sr}.wav"
        f.write_bytes(b)
        np.testing.assert_allclose(load_audio(str(f), 22050), want, atol=1e-6, rtol=0)
    # IEEE-float WAV (what the reference's own TTSOutput.save writes) is accepted as a speaker reference too
    x = (np.random.RandomState(5).rand(4000).astype(np.float32) * 1.2 - 0.6)
    ours.TTSOutput(array=x, sample_rate=22050).save(tmp_path / "f32.wav")
    np.testing.assert_array_equal(load_audio(str(tmp_path / "f32.wav"), 22050), x)


def test_randomised_requests_same_results(ref):
    """30 random (length, stream, failing chunk, scheduler concurrency) cases: both façades return the same audio in the same
    pieces, or fail with the same error."""
    side = ours_side()
    for case, (c, want) in enumerate(zip(randomised_cases(), ref["randomised"])):
        got = json.loads(json.dumps(case_randomised(side, *c)))
        if want[0] == "err" and c[1]:
            assert got[0] == "err" and got[1:] == want[1:], (case, got, want)
        else:
            assert got == want, (case, c)
