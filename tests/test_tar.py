"""TarDecoder / TarEncoder / TarFileEncoder(STORE) (archive_b200/tar.py, io.py) against the oracle's restatement of the
reference (oracle/tar.c), member by member and byte for byte, and against CPython's tarfile as an independent reader."""
import io
import os
import tarfile

import pytest

import oracle_tar as ot
from archive_b200 import Archive, ArchiveFile, DartRangeError, InputFileStream, InputMemoryStream, TarDecoder, TarEncoder
from archive_b200 import TarFileEncoder

GOLD = os.path.join(os.path.dirname(__file__), "golden")
TAR = os.path.join(GOLD, "tar")
FIXTURES = sorted(f for f in os.listdir(TAR) if f.endswith(".tar")) + ["../test2.tar"]


def assert_same(data, store_data=True):
    """TarDecoder on `data` equals the oracle: decoder.files field by field, then the Archive in order."""
    st, ms = ot.decode(data, store_data)
    dec = TarDecoder()
    if st == ot.THROW:
        with pytest.raises(DartRangeError):
            dec.decode_bytes(data, store_data=store_data)
        return st, ms
    arch = dec.decode_bytes(data, store_data=store_data)
    assert st == ot.OK
    assert len(dec.files) == len(ms)
    for t, m in zip(dec.files, ms):
        assert (t.filename, t.name_of_linked_file, t.type_flag, t.mode, t.owner_id, t.group_id, t.file_size, t.last_mod_time,
                t.checksum, t.ustar_indicator, t.owner_user_name, t.owner_group_name, t.device_major_number,
                t.device_minor_number, t.raw_content) == \
               (m.name, m.link, m.type_flag, m.mode, m.uid, m.gid, m.size, m.mtime, m.checksum, m.magic, m.uname, m.gname,
                m.devmajor, m.devminor, m.content)
    want = ot.archive_order(ms)
    assert len(arch) == len(want)
    for f, m in zip(arch, want):
        content = (m.content if store_data else None) if m.is_file else None
        assert (f.name, f.is_file, f.content, f.size, f.symbolic_link, f.mode, f.owner_id, f.group_id, f.last_mod_time) == \
               (m.name, m.is_file, content, len(content or b""), m.link, m.mode, m.uid, m.gid, m.mtime)
    return st, ms


# ---- archives ---------------------------------------------------------------------------------------------------------

def _member(tf, name, type=tarfile.REGTYPE, data=b"", **kw):
    ti = tarfile.TarInfo(name)
    ti.type, ti.size, ti.mtime, ti.mode = type, len(data), kw.pop("mtime", 1_700_000_000), kw.pop("mode", 0o644)
    for k, v in kw.items():
        setattr(ti, k, v)
    try:
        tf.addfile(ti, io.BytesIO(data) if type == tarfile.REGTYPE else None)
    except ValueError:  # the format cannot hold it (a V7 / USTAR name too long, ...)
        pass


def generated(fmt, encoding="utf-8"):
    buf = io.BytesIO()
    pax = {"comment": "global"} if fmt == tarfile.PAX_FORMAT else None
    with tarfile.open(fileobj=buf, mode="w", format=fmt, encoding=encoding, pax_headers=pax) as tf:
        for n in (100, 101, 255):
            _member(tf, "n" * (n - 4) + ".txt", data=b"x" * n)
            _member(tf, "d/" + "é" * ((n - 2) // 2), data=b"accent")
        _member(tf, "dir", tarfile.DIRTYPE, mode=0o755)
        _member(tf, "link", tarfile.SYMTYPE, linkname="target/" + "l" * 120)
        _member(tf, "hard", tarfile.LNKTYPE, linkname="n" * 96 + ".txt")
        _member(tf, "fifo", tarfile.FIFOTYPE)
        _member(tf, "chr", tarfile.CHRTYPE, devmajor=4, devminor=7)
        _member(tf, "empty", data=b"")
        for s in (511, 512, 513):
            _member(tf, f"size{s}", data=bytes(range(256)) * 2 + b"z" * (s - 512) if s > 512 else bytes(s))
        _member(tf, "dup", data=b"first")
        _member(tf, "dup", data=b"second, longer")
        _member(tf, "bigid", data=b"ids", uid=1 << 30, gid=5, uname="u" * 20, gname="g")
        _member(tf, "mtime", data=b"t", mtime=0o77777777777)
    return buf.getvalue()


FORMATS = {"gnu": tarfile.GNU_FORMAT, "pax": tarfile.PAX_FORMAT, "ustar": tarfile.USTAR_FORMAT, "v7": tarfile.USTAR_FORMAT}


def _v7(data):
    """A USTAR archive with the magic of every header cleared: the V7 layout tarfile no longer writes."""
    b = bytearray(data)
    for off in range(0, len(b) - 512, 512):
        if b[off + 257:off + 262] == b"ustar":
            b[off + 257:off + 265] = bytes(8)
    return bytes(b)


def header(name, type=b"0", size=0, link=b"", magic=b"ustar\x0000", mode=b"0000644\0", uid=b"0001750\0", size_field=None,
           prefix=b""):
    """A raw 512-byte header (the checksum is filled in but never read back by the reference)."""
    h = bytearray(512)
    h[0:len(name)] = name
    h[100:108] = mode
    h[108:116] = uid
    h[116:124] = b"0001750\0"
    h[124:136] = size_field if size_field is not None else b"%011o\0" % size
    h[136:148] = b"14501113260\0"
    h[156:157] = type
    h[157:157 + len(link)] = link
    h[257:257 + len(magic)] = magic
    h[345:345 + len(prefix)] = prefix
    h[148:156] = b"        "
    h[148:156] = b"%06o\0 " % sum(h)
    return bytes(h)


def body(data):
    return data + bytes(-len(data) % 512)


CRAFTED = {
    "pax_path_linkpath": header(b"PaxHeaders/x", b"x", 57) + body(b"30 path=pax/name\xc3\xa9\n22 linkpath=pax/lnk\n") +
    header(b"short", b"2", link=b"ignored") + bytes(1024),
    "pax_lying_length": header(b"PaxHeaders/y", b"x", 41) + body(b"999 path=lying\n1 ctime=1\nno record here\n") +
    header(b"f", size=3) + body(b"abc") + bytes(1024),
    "pax_unanchored_cr": header(b"PaxHeaders/z", b"X", 40) + body(b"junk 12 path=mid\rtail\n7 linkpath=\xe2\x80\xa8x\n") +
    header(b"g", size=1) + body(b"!") + bytes(1024),
    "pax_global_then_local": header(b"G", b"g", 20) + body(b"20 path=from-global\n") + header(b"plain", size=2) + body(b"ok"),
    "pax_not_utf8": header(b"PaxHeaders/b", b"x", 12) + body(b"12 path=\xff\xfe\n") + header(b"f", size=1) + body(b"1"),
    "longlink_K_sets_name": header(b"././@LongLink", b"K", 9, magic=b"ustar  \0") + body(b"lnk\0after") +
    header(b"real", b"2", link=b"short-target") + bytes(1024),
    "longlink_any_type": header(b"././@LongLink", b"0", 6) + body(b"abc\0de") + header(b"x", size=1) + body(b"1"),
    "base256_uid_size": header(b"b256", size_field=b"\x80" + bytes(7) + b"\x00\x00\x02\x00", uid=b"\x80\x00\x00\x00\x00\x01\x00\x00") +
    body(b"q" * 100) + bytes(1024),
    "dir_with_size": header(b"dir/", b"5", 100) + b"d" * 100 + header(b"after", size=2) + body(b"ok") + bytes(1024),
    "non_utf8_name": header(b"caf\xe9\x1f \x85", size=1, magic=b"") + body(b"1") + bytes(1024),
    "trim_set": header(b"\xe2\x80\x83spaced\xef\xbb\xbf\x0b", size=1, mode=b" 644 \0\0\0") + body(b"1"),
    "octal_grammar": header(b"a", mode=b"0o644\0\0\0", uid=b"+17\0\0\0\0\0") + header(b"b", mode=b"6_44\0\0\0\0",
                                                                                      uid=b"-17\0\0\0\0\0") + bytes(1024),
    "negative_size": header(b"neg", size_field=b"-0000000001\0") + bytes(1024),
    "prefix_joined": header(b"name", prefix=b"some/prefix", size=1) + body(b"p") +
    header(b"gnu", prefix=b"atime-area", magic=b"ustar  \0", size=1) + body(b"g") + bytes(1024),
    "single_zero_then_data": header(b"one", size=1) + body(b"1") + b"\0\x01" + bytes(510),
    "one_byte_left": header(b"one", size=1) + body(b"1") + b"\x07",
}


@pytest.mark.parametrize("name", FIXTURES)
def test_fixtures(name):
    data = open(os.path.join(TAR, name), "rb").read()
    assert_same(data)
    assert_same(data, store_data=False)


@pytest.mark.parametrize("fmt", sorted(FORMATS))
def test_generated(fmt):
    data = generated(FORMATS[fmt])
    if fmt == "v7":
        data = _v7(data)
    st, ms = assert_same(data)
    assert st == ot.OK and len(ms) >= 14
    if fmt != "pax":
        assert_same(data, store_data=False)


def test_generated_non_utf8_names():
    assert_same(generated(tarfile.GNU_FORMAT, encoding="latin-1"))


@pytest.mark.parametrize("name", sorted(CRAFTED))
def test_crafted(name):
    assert_same(CRAFTED[name])
    assert_same(CRAFTED[name], store_data=False)


def test_crafted_outcomes():
    """The quirks the crafted archives are there for, stated outright."""
    a = TarDecoder().decode_bytes(CRAFTED["pax_path_linkpath"])
    assert (a.files[0].name, a.files[0].symbolic_link) == ("pax/nameé", "pax/lnk")
    assert TarDecoder().decode_bytes(CRAFTED["pax_lying_length"]).files[0].name == "lying"
    a = TarDecoder().decode_bytes(CRAFTED["pax_unanchored_cr"])
    assert (a.files[0].name, a.files[0].symbolic_link) == ("mid", "")
    assert TarDecoder().decode_bytes(CRAFTED["pax_global_then_local"]).files[0].name == "plain"
    with pytest.raises(DartRangeError):
        TarDecoder().decode_bytes(CRAFTED["pax_not_utf8"])
    assert TarDecoder().decode_bytes(CRAFTED["longlink_K_sets_name"]).files[0].name == "lnk"
    d = TarDecoder()
    a = d.decode_bytes(CRAFTED["base256_uid_size"])
    assert (d.files[0].owner_id, d.files[0].file_size, a.files[0].content) == (0, 0, b"")
    assert TarDecoder().decode_bytes(CRAFTED["non_utf8_name"]).files[0].name == "café\x1f"
    d = TarDecoder()
    d.decode_bytes(CRAFTED["trim_set"])
    assert (d.files[0].filename, d.files[0].mode) == ("spaced", 0o644)
    d = TarDecoder()
    d.decode_bytes(CRAFTED["octal_grammar"])
    assert [(t.mode, t.owner_id) for t in d.files] == [(0, 0o17), (0, -0o17)]
    with pytest.raises(DartRangeError):
        TarDecoder().decode_bytes(CRAFTED["negative_size"])
    assert [f.name for f in TarDecoder().decode_bytes(CRAFTED["prefix_joined"])] == ["some/prefix/name", "atime-area/gnu"]
    assert len(TarDecoder().decode_bytes(CRAFTED["single_zero_then_data"])) == 2
    assert len(TarDecoder().decode_bytes(CRAFTED["one_byte_left"])) == 1
    assert [(f.name, f.size) for f in TarDecoder().decode_bytes([1, 2, 3])] == [("\x01\x02\x03", 0)]


def test_truncation():
    """Cut at every header and content boundary of a small archive, and one byte either side of each."""
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.GNU_FORMAT) as tf:
        _member(tf, "a" * 120, data=b"first" * 30)
        _member(tf, "b", data=b"x" * 513)
        _member(tf, "d", tarfile.DIRTYPE)
        _member(tf, "l", tarfile.SYMTYPE, linkname="k" * 130)
    data = buf.getvalue()
    cuts = set()
    for b in list(range(0, len(data), 512)) + [512 + 150, 1536 + 150, 2048 + 513]:
        cuts |= {b - 1, b, b + 1}
    for cut in sorted(c for c in cuts if 0 <= c <= len(data)):
        assert_same(data[:cut])
        assert_same(data[:cut], store_data=False)


def test_decode_stream(tmp_path):
    data = open(os.path.join(TAR, "symlink_tar.tar"), "rb").read()
    want = [(f.name, f.content) for f in TarDecoder().decode_bytes(data)]
    s = InputMemoryStream(b"\x09" * 7 + data)
    s.position = 7
    assert [(f.name, f.content) for f in TarDecoder().decode_stream(s)] == want
    p = tmp_path / "a.tar"
    p.write_bytes(data)
    fs = InputFileStream(str(p))
    dec = TarDecoder()
    assert [(f.name, f.content) for f in dec.decode_stream(fs)] == want and len(dec.files) == 4
    fs.close_sync()


def test_callback_and_duplicates():
    data = generated(tarfile.GNU_FORMAT)
    seen = []
    dec = TarDecoder()
    arch = dec.decode_bytes(data, callback=seen.append)
    assert len(seen) == len(dec.files) > len(arch) == len({t.filename for t in dec.files})  # "dup" twice in files, once here
    assert arch.find("dup").content == b"second, longer"


# ---- encoder ----------------------------------------------------------------------------------------------------------

def _entries():
    out = []
    for n in (99, 100, 101, 300):
        out.append(dict(name="a" * n, content=b"ascii %d" % n))
        out.append(dict(name="é" * n, content=b"latin %d" % n))
        out.append(dict(name="\U0001d11e" * (n // 2) + "z" * (n % 2), content=b"astral"))  # n UTF-16 code units
    out += [dict(name="dir/", is_file=False, mode=0o40755, mtime=5), dict(name="sym", symlink="dir/target", mode=0o120777),
            dict(name="emptylink", symlink=""), dict(name="nodata", content=None, size=7),
            dict(name="short-content", content=b"abc", size=600), dict(name="empty", content=b"")]
    for mode in (0, 0o777, 0o100644, 0o7777777, 0o77777777, 1 << 40, -1):
        out.append(dict(name="mode%o" % abs(mode), content=b"m", mode=mode))
    for mt in (0, (1 << 33) - 1, 1 << 36, -5):
        out.append(dict(name="mtime%d" % mt, content=b"t" * 511, mtime=mt, uid=1 << 21, gid=65534))
    return out


def _archive_file(e):
    f = ArchiveFile(e["name"], e.get("size", len(e.get("content") or b"")), is_file=e.get("is_file", True))
    if f.is_file:
        f.content = e.get("content")
    f.symbolic_link = e.get("symlink")
    f.mode, f.owner_id, f.group_id, f.last_mod_time = e.get("mode", 0o644), e.get("uid", 0), e.get("gid", 0), e.get("mtime", 0)
    return f


def test_encoder_matches_oracle():
    ents = _entries()
    arch = Archive()
    for e in ents:
        arch.add(_archive_file(e))
    got = TarEncoder().encode_bytes(arch)
    assert got == ot.encode(ents)
    assert TarEncoder().encode(list(arch)) == got
    enc = TarEncoder()  # start / add / finish
    enc.start()
    enc.add(arch.files[0])
    assert enc._output.get_bytes() == ot.encode(ents[:1])[:-1024]
    enc.finish()
    assert_same(got)  # whatever the misplaced long-name entries do to the walk, the decoder agrees with the oracle


def test_encoder_round_trip_and_tarfile():
    ents = [dict(name="a" * n, content=bytes(range(256)) * (n // 50)) for n in (1, 99, 100, 101, 300)] + \
           [dict(name="dir/", is_file=False, mode=0o755, mtime=77), dict(name="s", symlink="a", mode=0o777),
            dict(name="m", content=b"x" * 513, mode=0o100600, mtime=1_700_000_000, uid=1000, gid=100)]
    data = TarEncoder().encode_bytes([_archive_file(e) for e in ents])
    back = TarDecoder().decode_bytes(data)
    assert [(f.name, f.is_file, f.content if f.is_file and not f.symbolic_link else None) for f in back] == \
           [(e["name"], e.get("is_file", True), e.get("content")) for e in ents]
    assert [f.mode for f in back] == [e.get("mode", 0o644) for e in ents]
    short = [e for e in ents if len(e["name"]) <= 100]
    with tarfile.open(fileobj=io.BytesIO(TarEncoder().encode_bytes([_archive_file(e) for e in short]))) as tf:
        got = [(m.name.rstrip("/"), m.type, m.mode, m.mtime, m.uid, m.linkname, tf.extractfile(m).read() if m.isreg() else None)
               for m in tf.getmembers()]
    assert got == [(e["name"].rstrip("/"), tarfile.DIRTYPE if e.get("is_file") is False else tarfile.SYMTYPE if "symlink" in e
                    else tarfile.REGTYPE, e.get("mode", 0o644), e.get("mtime", 0), e.get("uid", 0), e.get("symlink", ""),
                    e.get("content")) for e in short]


def test_decoded_archive_reencodes_as_links():
    """TarDecoder sets symbolicLink to '' on every member, and TarEncoder writes any member with a symbolicLink as a link
    with no content: the reference's decode -> encode keeps names but drops every file's content."""
    arch = TarDecoder().decode_bytes(open(os.path.join(TAR, "gnu.tar"), "rb").read())
    st, ms = ot.decode(TarEncoder().encode_bytes(arch))
    assert [(m.name, m.type_flag, m.size) for m in ms] == [("small.txt", "2", 0), ("small2.txt", "2", 0)]


# ---- TarFileEncoder, STORE --------------------------------------------------------------------------------------------

def make_tree(root, n_files=12, seed=3):
    import random
    rng = random.Random(seed)
    for i in range(n_files):
        p = root / ("sub%d" % (i % 3)) / ("deep" if i % 4 == 0 else "") / ("f%02d.bin" % i)
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(bytes(rng.getrandbits(8) for _ in range(rng.choice([0, 1, 511, 512, 513, 3000]))))
        os.chmod(p, rng.choice([0o644, 0o600, 0o755]))
        os.utime(p, (1_600_000_000 + i, 1_600_000_000 + i))
    (root / "empty_dir").mkdir()
    return root


def expected_entries(root, tar_bytes):
    """The entries TarFileEncoder.add_directory hands TarEncoder for `root`, in sorted order.  A directory entry carries the
    time it was added, so those are read back from the archive."""
    st, ms = ot.decode(tar_bytes)
    dir_mtime = {m.name: m.mtime for m in ms if m.type_flag == "5"}
    base = os.path.basename(str(root))
    listing = []
    for r, dirs, files in os.walk(root):
        listing += [(os.path.join(r, d), True) for d in dirs] + [(os.path.join(r, f), False) for f in files]
    ents = []
    for p, is_dir in sorted(listing):
        name = base + "/" + os.path.relpath(p, root).replace(os.sep, "/")
        s = os.stat(p)
        if is_dir:
            ents.append(dict(name=name + "/", is_file=False, mode=s.st_mode, mtime=dir_mtime[name + "/"]))
        else:
            ents.append(dict(name=name, content=open(p, "rb").read(), mode=s.st_mode, mtime=int(s.st_mtime)))
    return ents


def test_tar_directory_store(tmp_path):
    root = make_tree(tmp_path / "tree")
    TarFileEncoder().tar_directory(str(root))
    data = (tmp_path / "tree.tar").read_bytes()
    assert data == ot.encode(expected_entries(root, data))
    with tarfile.open(fileobj=io.BytesIO(data)) as tf:
        names = tf.getnames()
        assert all(tf.extractfile(m).read() == (tmp_path / m.name).read_bytes() for m in tf.getmembers() if m.isreg())
    assert names[0] == "tree/empty_dir" and len(names) == 12 + 7
    TarFileEncoder().tar_directory(str(root), filename=str(tmp_path / "named.tar"),
                                   filter=lambda p, progress: "skip" if p.endswith(".bin") else None)
    assert all(m.name.endswith("/") for m in TarDecoder().decode_bytes((tmp_path / "named.tar").read_bytes()))
