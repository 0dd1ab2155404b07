"""The XZ oracle (oracle/xz.c) against the reference's own fixtures (tests/golden/xz/, the cases of xz_test.dart), Python's
lzma on valid streams, CRC-64 / SHA-256 known answers, and the reference's quirks.  CPU only."""
import hashlib
import json
import lzma
import os
import random

import pytest

import oracle_lib as orc
import xz_build as xb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "xz")
MAN = json.load(open(os.path.join(GOLD, "manifest.json")))


def gold(name):
    return open(os.path.join(GOLD, name), "rb").read()


@pytest.mark.parametrize("name", sorted(MAN["decode"]))
def test_fixture_decodes(name):
    want = MAN["decode"][name]
    expect = gold(want["expected"]) if "expected" in want else want["text"].encode()
    for verify in (False, True):
        st, out = xb.decode(gold(name), verify)
        assert (st, out) == (orc.OK, expect)


def test_cat_jpg():
    st, out = xb.decode(gold("cat.jpg.xz"))
    assert st == orc.OK and out == open(os.path.join(ROOT, "tests", "golden", "cat.jpg"), "rb").read()


@pytest.mark.parametrize("name,check,text", [(n, c, t) for n, (c, t) in MAN["encode"].items()])
def test_encoder_matches_fixture(name, check, text):
    assert xb.encode(text.encode(), check) == gold(name)


def test_known_answers():
    assert xb.crc64(b"123456789") == 0x995DC9BBDF1939FA
    assert xb.crc64(b"") == 0
    for n in (0, 1, 55, 56, 63, 64, 65, 1000):
        d = bytes(random.Random(n).randbytes(n))
        assert xb.sha256(d) == hashlib.sha256(d).digest()


TEXT = b"".join(b"line %d: the quick brown fox jumps over the lazy dog %d\n" % (i, i * i % 977) for i in range(4000))


@pytest.mark.parametrize("preset", range(10))
@pytest.mark.parametrize("check", [lzma.CHECK_NONE, lzma.CHECK_CRC32, lzma.CHECK_CRC64, lzma.CHECK_SHA256])
def test_presets_and_checks_against_lzma(preset, check):
    c = lzma.compress(TEXT, preset=preset, check=check)
    assert xb.decode(c, True) == (orc.OK, TEXT)


@pytest.mark.parametrize("lc,lp,pb", [(0, 0, 0), (3, 0, 2), (4, 0, 2), (0, 4, 0), (1, 3, 3), (2, 2, 1), (3, 1, 0)])
def test_props_against_lzma(lc, lp, pb):
    c = xb.container([(xb.raw_lzma2(TEXT, lc=lc, lp=lp, pb=pb), TEXT)])
    assert xb.decode(c, True) == (orc.OK, TEXT)


@pytest.mark.parametrize("bs", [1 << 20, 50000, 4096, 241])
def test_blocks(bs):
    data = TEXT[:241000] if bs == 241 else TEXT
    c = xb.xz_blocks(data, bs, check="crc32")
    assert lzma.decompress(c) == data
    assert xb.decode(c, True) == (orc.OK, data)


def test_incompressible_gives_stored_chunks():
    data = random.Random(7).randbytes(300000)
    raw = xb.raw_lzma2(data)
    assert any(c < 0x80 for c, _, _ in xb.chunks(raw))
    assert xb.decode(xb.container([(raw, data)]), True) == (orc.OK, data)


def test_pb4_throws_where_lzma_accepts():
    c = xb.container([(xb.raw_lzma2(TEXT, pb=4), TEXT)])
    assert lzma.decompress(c) == TEXT
    assert xb.decode(c)[0] == orc.THROW


def test_encoder_over_64k_is_not_valid_xz():
    data = bytes(random.Random(3).randbytes(70000))
    enc = xb.encode(data, 2)
    assert enc[24:27] == bytes([1, ((70000 - 1) >> 8) & 0xFF, (70000 - 1) & 0xFF])
    with pytest.raises(lzma.LZMAError):
        lzma.decompress(enc)


def test_verify_catches_wrong_checks_only_when_asked():
    for check in ("crc32", "crc64"):
        bad = xb.container([(xb.raw_lzma2(TEXT), TEXT)], check=check, bad_check=True)
        assert xb.decode(bad, False) == (orc.OK, TEXT)
        assert xb.decode(bad, True) == (orc.FALSE, TEXT)


def test_trimmed_dictionary_against_lzma():
    """dictionary byte 0 (4 KiB): trimDictionary runs after every chunk of a many-chunk stream"""
    r = random.Random(23)
    words = [bytes(r.randbytes(r.randrange(2, 9))) for _ in range(3000)]
    plain = b" ".join(r.choice(words) for _ in range(110000))
    raw = xb.raw_lzma2(plain, preset=1, dict_size=4096)
    assert len(xb.chunks(raw)) > 3
    c = xb.container([(raw, plain)], dict_byte=0)
    assert lzma.decompress(c) == plain
    assert xb.decode(c, True) == (orc.OK, plain)
