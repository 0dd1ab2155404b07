"""Tarballs through the device codecs: the compression stage of .tar.gz / .tar.bz2 / .tar.xz on the GPU (one call per
tarball, and one batch call for many shards), TarFileEncoder's device gzip stage, and extract_archive_to_disk on a
decoded tarball -- each checked against the oracle (oracle/tar.c and the codec oracles) and CPython's tarfile."""
import gzip
import io
import lzma
import os
import random
import stat
import tarfile

import pytest

import oracle_lib as orc
import oracle_tar as ot
from test_tar import assert_same, expected_entries, make_tree

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def a():
    import archive_b200
    return archive_b200


def _names(archive):
    return [(f.name, f.is_file, f.content) for f in archive]


def test_test2_tarballs(a):
    """tar_test.dart:231-253: test2.tar, and the same archive behind gzip and bzip2, give 4 members."""
    want = _names(a.TarDecoder().decode_bytes(open(os.path.join(GOLD, "test2.tar"), "rb").read()))
    assert len(want) == 4
    gz = open(os.path.join(GOLD, "test2.tar.gz"), "rb").read()
    bz = open(os.path.join(GOLD, "test2.tar.bz2"), "rb").read()
    assert _names(a.TarDecoder().decode_bytes(a.GZipDecoder().decode_bytes(gz, verify=True))) == want
    assert _names(a.TarDecoder().decode_bytes(a.BZip2Decoder().decode_bytes(bz, verify=True))) == want


def shard_tars(n, seed=11):
    """n small tar archives of text members, written by TarEncoder-independent CPython tarfile (GNU format)."""
    rng = random.Random(seed)
    words = [b"alpha", b"beta", b"gamma", b"delta", b"tar", b"shard", b"\n"]
    out = []
    for s in range(n):
        buf = io.BytesIO()
        with tarfile.open(fileobj=buf, mode="w", format=tarfile.GNU_FORMAT) as tf:
            for k in range(rng.randint(1, 6)):
                body = b" ".join(rng.choice(words) for _ in range(rng.randint(0, 3000)))
                ti = tarfile.TarInfo("shard%03d/%s/member%d.txt" % (s, "x" * rng.choice([1, 120]), k))
                ti.size, ti.mtime = len(body), 1_650_000_000 + k
                tf.addfile(ti, io.BytesIO(body))
        out.append(buf.getvalue())
    return out


@pytest.mark.parametrize("codec", ["gzip", "bzip2", "xz"])
def test_shard_batch(a, codec):
    """One batch call per codec for 64 shards, then TarDecoder per shard: equal to the per-shard single calls and to the
    oracle's reading of the original tar."""
    tars = shard_tars(64)
    if codec == "gzip":
        shards = [orc.gzip_encode(t, 6, mtime=0)[1] for t in tars]
        batch, single = a.gzip_decode_batch(shards, verify=True), [a.GZipDecoder().decode_bytes(z, verify=True) for z in shards]
    elif codec == "bzip2":
        shards = [orc.bzip2_encode(t)[1] for t in tars]
        batch, single = a.bzip2_decode_batch(shards, verify=True), [a.BZip2Decoder().decode_bytes(z, verify=True) for z in shards]
    else:
        shards = [lzma.compress(t, format=lzma.FORMAT_XZ, check=lzma.CHECK_CRC64) for t in tars]
        batch, single = a.xz_decode_batch(shards, verify=True), [a.XZDecoder().decode_bytes(z, verify=True) for z in shards]
    assert [rc for rc, _ in batch] == [0] * len(shards)
    assert [t for _, t in batch] == single == tars
    for (_, t), want in zip(batch, tars):
        arch = a.TarDecoder().decode_bytes(t)
        st, ms = ot.decode(want)
        assert st == ot.OK
        assert [(f.name, f.content) for f in arch] == [(m.name, m.content) for m in ot.archive_order(ms)]
        assert [f.content for f in arch] == [tarfile.open(fileobj=io.BytesIO(want)).extractfile(m).read()
                                             for m in tarfile.open(fileobj=io.BytesIO(want)).getmembers()]


@pytest.mark.parametrize("level", [1, 6])
def test_tar_directory_gzip(a, tmp_path, monkeypatch, level):
    """GZIP: the device gzip of the tar is byte-identical to the oracle's gzip of the oracle's tar of the same sorted
    listing, gzip + tarfile read it back, and the temporary tar is gone."""
    import tempfile
    tmp = tmp_path / "tmp"
    tmp.mkdir()
    monkeypatch.setattr(tempfile, "tempdir", str(tmp))
    root = make_tree(tmp_path / "tree", n_files=20)
    a.TarFileEncoder().tar_directory(str(root), compression=a.TarFileEncoder.GZIP, level=level)
    tgz = (tmp_path / "tree.tar.gz").read_bytes()
    tar = gzip.decompress(tgz)
    assert tar == ot.encode(expected_entries(root, tar))
    mtime = int.from_bytes(tgz[4:8], "little")  # GZipEncoder stamps the wall clock
    assert tgz == orc.gzip_encode(tar, level, mtime=mtime)[1]
    with tarfile.open(str(tmp_path / "tree.tar.gz"), "r:gz") as tf:
        assert sorted(m.name for m in tf.getmembers() if m.isreg()) == sorted(
            "tree/" + os.path.relpath(os.path.join(r, f), root) for r, _, fs in os.walk(root) for f in fs)
    assert os.listdir(tmp) == []
    assert_same(tar)


def test_extract_decoded_tarball(a, tmp_path):
    """extract_archive_to_disk on a decoded .tar.gz: files with their modes; ../ entries and absolute symlinks skipped."""
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.USTAR_FORMAT) as tf:
        for name, mode, body in [("pkg/run.sh", 0o755, b"#!/bin/sh\n"), ("pkg/data.txt", 0o600, b"data"),
                                 ("../escape.txt", 0o644, b"no"), ("pkg/sub/deep.txt", 0o640, b"deep")]:
            ti = tarfile.TarInfo(name)
            ti.size, ti.mode = len(body), mode
            tf.addfile(ti, io.BytesIO(body))
        for name, target in [("pkg/abs", "/etc/passwd"), ("pkg/rel", "data.txt")]:
            ti = tarfile.TarInfo(name)
            ti.type, ti.linkname = tarfile.SYMTYPE, target
            tf.addfile(ti)
    tgz = orc.gzip_encode(buf.getvalue(), 6)[1]
    out = tmp_path / "out"
    a.extract_archive_to_disk(a.TarDecoder().decode_bytes(a.GZipDecoder().decode_bytes(tgz)), str(out))
    assert (out / "pkg/run.sh").read_bytes() == b"#!/bin/sh\n"
    assert stat.S_IMODE(os.stat(out / "pkg/run.sh").st_mode) == 0o755
    assert stat.S_IMODE(os.stat(out / "pkg/data.txt").st_mode) == 0o600
    assert (out / "pkg/sub/deep.txt").read_bytes() == b"deep"
    assert not (tmp_path / "escape.txt").exists()
    assert not os.path.lexists(out / "pkg/abs")
    assert os.readlink(out / "pkg/rel") == "data.txt"
