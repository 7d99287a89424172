"""CPU: the Chinese normaliser (auralis_b200/zh_textnorm.py) against the reference's own `zh_num2words` — golden records
(tests/golden/zh_textnorm.json) and fuzzed sentences (tests/golden/text_live_reference.json.gz)."""
import gzip
import json
import os

from auralis_b200 import textnorm as T
from auralis_b200 import zh_textnorm as Z
from zh_fixture import sentences

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "zh_textnorm.json")
LIVE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "text_live_reference.json.gz")


def test_golden_records_from_the_reference():
    rec = json.load(open(GOLD, encoding="utf-8"))
    assert len(rec["sentences"]) >= 400 and len(rec["numbers"]) >= 150
    for r in rec["sentences"]:
        assert Z.normalize(r["in"]) == r["out"], r["in"]
    for r in rec["numbers"]:
        assert Z.num2chn(r["in"]) == r["cardinal"], r["in"]
        assert Z.num2chn(r["in"], alt_two=False, use_units=False) == r["digits"], r["in"]


def test_examples():
    assert Z.normalize("我有2个苹果和12.5%的股份") == "我有二个苹果和百分之十二点五的股份"
    assert Z.normalize("2023年10月5日，价格是3.50元") == "二零二三年十月五日,价格是三点五零元"
    assert Z.normalize("电话13812345678或010-12345678") == "电话一三八一二三四五六七八或零一零一二三四五六七八"
    assert Z.normalize("1/3的人 202 10500 P2P") == "三分之一的人 两百零二 一零五零零 P2P"
    # through the cleaner pipeline: lowercase, zh numbers + punctuation, zh symbol words, whitespace
    assert T.multilingual_cleaners("价格 5£ 和 3°, 共12个!", "zh") == "价格 五 英镑 和 三 度 , 共十二个,"


def test_live_fuzz_against_the_reference_module():
    """3 000 fuzzed sentences through zh_num2words.TextNorm and 300 through the reference tokenizer's whole zh cleaner chain
    (tests/zh_fixture.py generates them; the reference's outputs are in tests/golden/text_live_reference.json.gz)."""
    with gzip.open(LIVE, "rt", encoding="utf-8") as f:
        rec = json.load(f)
    assert len(rec["zh_normalize"]) >= 3000 and len(rec["zh_cleaners"]) >= 300
    assert [s for s, _ in rec["zh_normalize"]] == sentences(3000, 99)        # the stored inputs are the fixture's
    for s, want in rec["zh_normalize"]:
        assert Z.normalize(s) == want, s
    for s, want in rec["zh_cleaners"]:
        assert T.multilingual_cleaners(s, "zh") == want, s
