"""Times FLAC decoding on the GPU (`XTTSv2Engine.decode_flac`, i.e. xtts_decode_flac plus the host MD5 check) against
the sequential Python oracle (oracle/flac_stream.decode) on the same host, for a 30 s 44.1 kHz stereo 16-bit speaker
reference and for 10 and 60 min of mono 24 kHz audio.  The GPU time is the median wall time of the call, H2D and D2H
included; the MD5 share is the hashlib part of it.  The oracle is given the expected samples, which lets it check
predicted subframes vectorised instead of sample by sample (its result is the same); it runs once on the long inputs.
Then the decode's share of `get_audio_conditioning` on the 30 s reference, from its FLAC file.  Prints the card name
and power limit with the numbers.

    python tools/flac_decode_probe.py [--reps 5]
"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _median_ms(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    from auralis_b200 import TTS, native
    from auralis_b200.config import XTTSDims
    from auralis_b200.engine import XTTSv2Engine
    from auralis_b200.weights import save_model_dir, synth_state
    from oracle import enhance_oracle as E
    from oracle import flac_stream as S
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"card: {q}")
    with tempfile.TemporaryDirectory() as tmp:
        dims = XTTSDims.small()
        gs, cs = synth_state(dims, 1234)
        save_model_dir(tmp, dims, gs, cs)
        engine = XTTSv2Engine.from_pretrained(tmp, precision="fp32", max_concurrency=4)
        tts = TTS(scheduler_max_concurrency=4).from_engine(engine)
        try:
            def ref30(seed):
                x = S.signal(2, 44100 * 30, 16, seed, level=0.4)
                n = x.shape[1]
                fr = [S.Frame(4096, S.MID_SIDE, [S.Sub("LPC", order=8, shift=12)] * 2) for _ in range(n // 4096)]
                return x, S.write_stream(x, 16, 44100, fr + [S.Frame(n % 4096, S.MID_SIDE)]).data

            cases = [("30 s 44.1 kHz stereo", *ref30(1))]
            for minutes in (10, 60):
                pcm = (np.clip(E.synthetic_input(60.0 * minutes, 24000, 42), -1, 1) * 32767).astype(np.int16)
                cases.append((f"{minutes} min 24 kHz mono", pcm[None], engine.encode_flac(pcm, 24000, native.flac_md5(pcm[None], 16))))
            print(f"{'input':>22} {'MB':>7} {'gpu call ms':>12} {'md5 ms':>8} {'oracle ms':>11} {'speed-up':>9}", flush=True)
            for name, pcm, data in cases:
                got = engine.decode_flac(data)[0]
                assert np.array_equal(got, pcm)
                call = _median_ms(lambda: engine.decode_flac(data), args.reps)
                md5 = _median_ms(lambda: native.flac_md5(got, 16), args.reps)
                orc = _median_ms(lambda: S.decode(data, expect=pcm), args.reps if pcm.size < 5e6 else 1)
                print(f"{name:>22} {len(data) / 1e6:7.2f} {call:12.2f} {md5:8.2f} {orc:11.1f} {orc / call:8.0f}x", flush=True)

            # the decode's share of conditioning on the 30 s reference (fresh streams: no speaker-cache hits)
            conds, decs = [], []
            for seed in range(2, 2 + args.reps):
                _, data = ref30(seed)
                path = os.path.join(tmp, f"ref{seed}.flac")
                with open(path, "wb") as f:
                    f.write(data)
                t0 = time.perf_counter()
                tts.loop.run_until_complete(engine.get_audio_conditioning(path, 60, 30, 4))
                conds.append(time.perf_counter() - t0)
                decs.append(_median_ms(lambda: engine.decode_flac(data), 1) / 1e3)
            c, dd = float(np.median(conds)) * 1e3, float(np.median(decs)) * 1e3
            print(f"get_audio_conditioning (30 s 44.1 kHz stereo FLAC, small engine): {c:.1f} ms, of which the decode "
                  f"{dd:.2f} ms ({dd / c:.1%})")
        finally:
            tts.loop.run_until_complete(tts.shutdown())


if __name__ == "__main__":
    main()
