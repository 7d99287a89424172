"""Golden records for the live text comparisons of tests/test_text_golden.py and tests/test_zh_textnorm.py: seeded
random inputs and what the reference's own functions return for them —
  * `multilingual_cleaners` of 15 languages on 60 random strings each and `split_sentence` on 20 random texts
    (config/tokenizer.py, imported unmodified by oracle/ref_text.py; num2words = oracle.ref_text.marker_num2words),
  * zh_num2words `TextNorm` on 3 000 fuzzed Chinese sentences and the tokenizer's zh cleaner chain on 300 more
    (tests/zh_fixture.py generates them).

    python tests/golden/make_text_live_golden.py          (needs the reference source tree, see oracle/ref_import.py)
"""
import gzip
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_text  # noqa: E402
from zh_fixture import load_reference_zh, sentences  # noqa: E402

LANGS = ["en", "es", "fr", "de", "it", "pt", "pl", "ar", "zh", "cs", "ru", "nl", "tr", "hu", "ko"]
OUT = os.path.join(HERE, "text_live_reference.json.gz")


def main():
    ref = ref_text.load()
    rng = random.Random(7)
    alphabet = "abc dr. mr. sr. st. co. 1 2 3 12 1.234 5,50 $ £ € % & # @ ° º ª th st er e . , ; ! ?".split(" ")
    cleaners = []
    for lang in LANGS:
        for _ in range(60):
            s = " ".join(rng.choice(alphabet) for _ in range(rng.randint(1, 14)))
            if rng.random() < 0.5:
                s = s.replace(" ", "", rng.randint(0, 4))
            cleaners.append([lang, s, ref.multilingual_cleaners(s, lang)])
    split = []
    for _ in range(20):
        n = rng.randint(3, 30)
        s = " ".join(rng.choice(["Short one.", "A somewhat longer sentence, with a clause; and more - much more - to say about it all", "Why?",
                                 "Numbers like 1.5 do not end sentences.", "Ellipsis... then more!"]) for _ in range(n))
        lim = rng.choice([40, 82, 166, 250])
        split.append([s, lim, ref.split_sentence(s, "en", lim)])
    norm = load_reference_zh().TextNorm()
    rec = {"source": "reference tokenizer.py and zh_num2words.py, imported unmodified; num2words = oracle.ref_text.marker_num2words",
           "cleaners": cleaners, "split_sentence": split,
           "zh_normalize": [[s, norm(s)] for s in sentences(3000, 99)],
           "zh_cleaners": [[s, ref.multilingual_cleaners(s, "zh")] for s in sentences(300, 7)]}
    with gzip.open(OUT, "wt", encoding="utf-8", compresslevel=9) as f:
        json.dump(rec, f, ensure_ascii=False, separators=(",", ":"))
    print(f"{OUT}: {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
