"""Golden results of the reference's own façade classes (auralis.core.tts.TTS, TTSRequest, TTSOutput, imported unmodified by
oracle/ref_facade.py) in every case of tests/test_facade_vs_reference.py, plus the reference's `load_audio`
(common/utilities.py, lifted by source, `torchaudio.load` replaced by a stdlib WAV reader).

    python tests/golden/make_facade_golden.py          (needs the reference source tree, see oracle/ref_import.py)
"""
import ast
import importlib
import io
import os
import sys
import types
import wave

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_facade, ref_import  # noqa: E402
from test_facade_vs_reference import LOAD_AUDIO_CASES, Side, make_engine, record, wav_bytes  # noqa: E402


def reference_side():
    ref = ref_facade.load()
    CC = importlib.import_module("auralis.models.base").ConditioningConfig

    def make_tts(conc=4, fail_at=None):
        r = ref.TTS(scheduler_max_concurrency=conc)
        r._ensure_event_loop()
        r.tts_engine = make_engine(ref.TTSOutput, CC(speaker_embeddings=True, gpt_like_decoder_conditioning=True), fail_at=fail_at)
        return r
    return Side(make_tts, ref.TTSRequest, ref.TTSOutput)


def reference_load_audio(rec):
    import torch
    import torchaudio

    def fake_load(src):
        f = io.BytesIO(src) if isinstance(src, (bytes, bytearray)) else str(src)
        with wave.open(f, "rb") as w:
            nch, sr, raw = w.getnchannels(), w.getframerate(), w.readframes(w.getnframes())
        a = torch.from_numpy(np.frombuffer(raw, dtype="<i2").astype(np.float32) / 32768.0).reshape(-1, nch).t().contiguous()
        return a, sr
    path = os.path.join(ref_import.REF_SRC, "auralis", "common", "utilities.py")
    tree = ast.parse(open(path).read())
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "load_audio"]
    ns = {"torch": torch, "torchaudio": types.SimpleNamespace(load=fake_load, functional=torchaudio.functional)}
    exec(compile(ast.Module(body=fn, type_ignores=[]), path, "exec"), ns)
    for sr, nch in LOAD_AUDIO_CASES:
        rec[f"load_audio_{sr}_{nch}"] = ns["load_audio"](wav_bytes(sr, nch, seed=sr), 22050)[0].numpy()


def main():
    rec = record(reference_side())
    reference_load_audio(rec)
    out = os.path.join(HERE, "facade_reference.npz")
    np.savez_compressed(out, **rec)
    print(f"{out}: {len(rec)} entries, {os.path.getsize(out)} bytes")


if __name__ == "__main__":
    main()
