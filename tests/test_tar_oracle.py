"""The TAR oracle (oracle/tar.c) against the reference's own expectations: the header table and named cases of
test/tar_test.dart, transcribed in tests/golden/tar/reference_table.json, over the reference's fixtures."""
import gzip
import hashlib
import json
import os

import pytest

import oracle_tar as ot

GOLD = os.path.join(os.path.dirname(__file__), "golden")
TAR = os.path.join(GOLD, "tar")
TABLE = json.load(open(os.path.join(TAR, "reference_table.json")))
KEYS = {"Name": "name", "Mode": "mode", "Uid": "uid", "Gid": "gid", "Size": "size", "Linkname": "link", "ModTime": "mtime",
        "Typeflag": "type_flag", "Uname": "uname", "Gname": "gname", "Devmajor": "devmajor", "Devminor": "devminor"}


def _read(name):
    p = os.path.join(TAR, name)
    return open(p if os.path.exists(p) else os.path.join(GOLD, name), "rb").read()


def test_manifest():
    man = json.load(open(os.path.join(TAR, "manifest.json")))
    files = sorted(f for f in os.listdir(TAR) if f.endswith(".tar"))
    assert files == sorted(k for k in man if not k.startswith("_"))
    for f in files:
        data = _read(f)
        assert (len(data), hashlib.sha256(data).hexdigest()) == (man[f]["size"], man[f]["sha256"]), f


@pytest.mark.parametrize("name", sorted(TABLE["headers"]))
def test_header_table(name):
    """tar_test.dart:297-343: decoder.files has one TarFile per row, and every key a row has matches."""
    st, ms = ot.decode(_read(name))
    rows = TABLE["headers"][name]
    assert st == ot.OK and len(ms) == len(rows)
    for m, row in zip(ms, rows):
        for k, v in row.items():
            assert getattr(m, KEYS[k]) == v, (name, k)


@pytest.mark.parametrize("name", sorted(TABLE["cases"]))
def test_named_cases(name):
    case = TABLE["cases"][name]
    data = _read(name)
    if name.endswith(".gz"):
        data = gzip.decompress(data)
    st, ms = ot.decode(data)
    arch = ot.archive_order(ms)
    assert st == ot.OK and len(arch) == case["archive_length"]
    for i, n in case.get("names", {}).items():
        assert arch[int(i)].name == n
    for i, target in case.get("symlinks", {}).items():
        assert arch[int(i)].link == target


def test_invalid_archive():
    """tar_test.dart:153-160 passes whether or not [1, 2, 3] throws (see the table's note); the source reads it as one
    empty member whose name is the three bytes."""
    case = TABLE["invalid_archive"]
    st, ms = ot.decode(bytes(case["input"]))
    assert st == ot.OK and len(ot.archive_order(ms)) == case["archive_length"]
    assert (ms[0].name, ms[0].size, ms[0].content) == (case["name"], case["size"], b"")


@pytest.mark.parametrize("name", sorted(TABLE["encoder_cases"]))
def test_encoder_cases(name):
    case = TABLE["encoder_cases"][name]
    ents = [dict(e, content=bytes(e["content"]) if "content" in e else None) for e in case["entries"]]
    st, ms = ot.decode(ot.encode(ents))
    arch = ot.archive_order(ms)
    assert st == ot.OK
    if "decoded_names" in case:
        assert [m.name for m in arch] == case["decoded_names"]
    if "decoded_is_symbolic_link" in case:
        assert [bool(m.link) for m in arch] == case["decoded_is_symbolic_link"]
