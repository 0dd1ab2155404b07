"""Encrypted ZIP members on the device (b200z_zip_extract_password, b200z_zip_aes_encrypt) against the oracle
(oracle/zip_crypt.c, aes.c, zip_enc_crypt.c) and the reference's encrypted fixtures (tests/golden/zip_crypt/)."""
import ctypes as C
import hashlib
import json
import os
import zlib

import pytest

import oracle_lib as orc
import zip_crypt_build as zb

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "zip_crypt")
MAN = json.load(open(os.path.join(GOLD, "manifest.json")))
# oracle status -> device member statuses: the Dart throws (RangeError: B200Z_U_THROW, or B200Z_U_RANGE from inflate),
# the AES verifier (B200Z_ZIP_BAD_PASSWORD) and MAC (B200Z_ZIP_BAD_MAC) exceptions
ERR = {orc.THROW: (-5, -3), 4: (-22,), 5: (-23,)}


@pytest.fixture(scope="module")
def a():
    import archive_b200
    return archive_b200


def fixture(name):
    return open(os.path.join(GOLD, name), "rb").read()


def device_members(data, password, flags=0):
    """-> [(status, bytes)] of every listed member from ONE b200z_zip_extract_password call"""
    from archive_b200 import _ffi
    L = _ffi.ensure_init()
    st, ents = orc.zip_list(data)
    n = len(ents)
    arr = (_ffi.ZipEntry * n)()
    C.memmove(arr, (orc.ZipEntry * n)(*ents), C.sizeof(arr))
    room = [max(int(e.uncomp_size), int(e.comp_size) * 8 + 64, 1 << 16) for e in ents]
    off, tot = [], 0
    for r in room:
        off.append(tot)
        tot += (r + 63) & ~63
    out = (C.c_uint8 * tot)()
    ol, sts = (C.c_uint64 * n)(), (C.c_int32 * n)()
    addr, zl, keep = _ffi.as_buffer(data)
    rc = L.b200z_zip_extract_password(addr, zl, arr, n, C.addressof(out), tot, (C.c_uint64 * n)(*off), (C.c_uint64 * n)(*room),
                                      ol, sts, flags, password, len(password or b""))
    assert rc == 0, _ffi.last_error()
    return [(sts[i], C.string_at(C.addressof(out) + off[i], min(int(ol[i]), room[i]))) for i in range(n)]


def assert_like_oracle(data, password, flags=0):
    dev = device_members(data, password, flags)
    want = zb.oracle_members(data, password, web_eos=bool(flags & 1))
    assert len(dev) == len(want)
    for i, ((ds, db), (os_, ob)) in enumerate(zip(dev, want)):
        if os_ in ERR:
            assert ds in ERR[os_] and db == ob, (i, ds, os_)
        else:
            # (a data error is a status of the device only: the reference stops and keeps what it has, as the oracle does)
            assert db == ob and ds not in (-5, -22, -23), (i, ds, os_, len(db), len(ob))
    return dev


@pytest.mark.parametrize("name", sorted(MAN["archives"]))
def test_fixtures_decode_with_password(a, name):
    """test/zip_test.dart:546-610 ('zipCrypto', 'aes256', 'password')"""
    spec = MAN["archives"][name]
    data = fixture(name)
    arc = a.ZipDecoder().decode_bytes(data, password=spec["password"])
    assert [f.name for f in arc.files] == spec["members"]
    for f in arc.files:
        body = f.read_bytes()
        assert len(body) == MAN["plaintext"][f.name]["size"]
        assert hashlib.sha256(body).hexdigest() == MAN["plaintext"][f.name]["sha256"]
    if spec["mode"] == "aes":  # the real method comes from the AES record, with or without a password
        for arc2 in (arc, a.ZipDecoder().decode_bytes(data)):
            assert {f.name: f.compression for f in arc2.files} == {"hello.txt": "none", "readme.notzip": "deflate"}
    assert_like_oracle(data, spec["password"].encode())
    # InputFileStream + password, as the 'aes256' test reads it
    from archive_b200.streams import InputFileStream
    inp = InputFileStream(os.path.join(GOLD, name))
    arc = a.ZipDecoder().decode_stream(inp, password=spec["password"])
    inp.close_sync()
    assert [hashlib.sha256(f.read_bytes()).hexdigest() for f in arc.files] == [
        MAN["plaintext"][m]["sha256"] for m in spec["members"]]


@pytest.mark.parametrize("name", sorted(MAN["archives"]))
def test_fixtures_without_password_are_unchanged(a, name):
    data = fixture(name)
    arc = a.ZipDecoder().decode_bytes(data)
    assert all(f.status == -20 and f.content == b"" and f.read_bytes() == b"" for f in arc.files)
    assert all(s == -20 and b == b"" for s, b in device_members(data, None))


def test_fixture_errors(a):
    data = fixture("aes256.zip")
    assert_like_oracle(data, b"wrong")
    assert_like_oracle(data, b"")
    arc = a.ZipDecoder().decode_bytes(data, password="wrong")  # the directory walk does not throw; reading does
    with pytest.raises(a.zip.ArchiveException, match="password error"):
        arc.files[0].read_bytes()
    st, ents = orc.zip_list(data)
    bad = bytearray(data)
    bad[ents[1].data_off + 40] ^= 0x10
    dev = assert_like_oracle(bytes(bad), b"12345")
    assert [s for s, _ in dev] == [0, -23]
    arc = a.ZipDecoder().decode_bytes(bytes(bad), password="12345")
    with pytest.raises(a.zip.ArchiveException, match="macs"):
        arc.files[1].read_bytes()
    # ZipCrypto has no check: a wrong password gives what the cipher gives
    assert_like_oracle(fixture("zipCrypto.zip"), b"54321")
    assert_like_oracle(fixture("password_zipcrypto.zip"), b"")


def mixed_members(big=False):
    from archive_b200 import synth
    txt = synth.text(6 << 20, stream=971).tobytes()
    rnd = os.urandom(300_000)
    ms = [
        zb.Member("s128.txt", txt[:5000], 0, "aes", 1),
        zb.Member("d192.txt", txt[5000:90000], 8, "aes", 2),
        zb.Member("d256.txt", txt[:200_000], 8, "aes", 3, foreign_extra=True),
        zb.Member("b256.bin", txt[:150_000], 12, "aes", 3),
        zb.Member("bzc.bin", txt[7:60_000], 12, "zipcrypto"),
        zb.Member("zc_store.bin", rnd, 0, "zipcrypto"),
        zb.Member("zc_defl.txt", txt[100:123_456], 8, "zipcrypto", dd=True),
        zb.Member("aes_dd.txt", txt[3:33_333], 8, "aes", 1, dd=True),
        zb.Member("empty_aes.txt", b"", 0, "aes", 3),
        zb.Member("empty_zc.txt", b"", 0, "zipcrypto", truncate=0),
        zb.Member("dir/", is_dir=True, method=0, crypt="aes"),
        zb.Member("link", b"target/file", 0, "aes", 3, symlink=True),
        zb.Member("plain.txt", txt[:77_777], 8, None),
        zb.Member("odd_method.bin", rnd[:999], 99, "zipcrypto"),
        zb.Member("odd_extra.txt", txt[:3000], 8, "aes", 3, foreign_extra="odd"),
    ]
    if big:
        ms.append(zb.Member("flushed.txt", txt[:4 << 20], 8, "aes", 3, flush_every=65536))
        ms.append(zb.Member("big_zc.bin", txt[1 << 20:(1 << 20) + (4 << 20)], 8, "zipcrypto"))
        ms.append(zb.Member("big_store.bin", txt[:(4 << 20) + 3], 0, "aes", 2))
    return ms


@pytest.mark.parametrize("flags", [0, 1, 2])  # default, B200Z_ZIP_WEB_EOS, B200Z_ZIP_NO_SPLIT
def test_synthetic_mix_matches_oracle(a, flags):
    data = zb.build(mixed_members(big=flags != 1), b"pa55")
    dev = assert_like_oracle(data, b"pa55", flags)
    assert all(s in (0, 1) for s, _ in dev)


def test_synthetic_mix_through_the_decoder(a):
    ms = mixed_members()
    data = zb.build(ms, b"pa55")
    arc = a.ZipDecoder().decode_bytes(data, password=b"pa55")
    got = {f.name: f for f in arc.files}
    for m in ms:
        if m.is_dir or m.foreign_extra == "odd":  # (the reference does not find that AES record: garbage, as the oracle's)
            continue
        assert got[m.name].read_bytes() == m.data, m.name
    assert got["link"].symbolic_link == "target/file"
    assert got["d192.txt"].compression == "deflate" and got["b256.bin"].compression == "bzip2"


def test_many_small_aes_members(a):
    """key derivation per member: 1000 members of about 1 KiB, all three strengths"""
    ms = [zb.Member(f"m{i}.bin", os.urandom(500 + i % 1100), 8 if i % 3 else 0, "aes", 1 + i % 3) for i in range(1000)]
    data = zb.build(ms, b"k3y")
    dev = assert_like_oracle(data, b"k3y")
    assert [b for _, b in dev] == [m.data for m in ms]


def test_error_members_match_oracle(a):
    txt = bytes(range(256)) * 100
    ms = [zb.Member("ok.txt", txt, 8, "aes", 3),
          zb.Member("badmac.txt", txt, 8, "aes", 3, bad_mac=True),
          zb.Member("short_aes.txt", txt, 0, "aes", 3, truncate=20),
          zb.Member("short_aes128.txt", txt, 0, "aes", 1, truncate=19),
          zb.Member("just_header.txt", b"", 0, "aes", 1),
          zb.Member("short_zc.txt", txt, 0, "zipcrypto", truncate=11),
          zb.Member("other_pw.txt", txt, 8, "aes", 2, password=b"other"),
          zb.Member("other_pw_zc.txt", txt, 8, "zipcrypto", password=b"other")]
    data = zb.build(ms, b"right")
    dev = assert_like_oracle(data, b"right")
    assert [s for s, _ in dev][:7] == [0, -23, -5, -5, 0, -5, -22]
    assert_like_oracle(data, b"")  # the empty password: every AES member throws
    arc = a.ZipDecoder().decode_bytes(data, password="right")
    with pytest.raises(a.zip.ArchiveException):
        arc.find("short_aes.txt").read_bytes()


def test_truncated_aes_extra_field_throws_on_that_member(a):
    """an AES record cut short inside the local extra field: ZipFile.read throws for that member"""
    import struct
    data = bytearray(zb.build([zb.Member("x.txt", b"abc" * 100, 0, "aes", 3), zb.Member("y.txt", b"hello", 0, "aes", 3)], b"p"))
    st, ents = orc.zip_list(bytes(data))
    e = ents[0]
    xl = e.data_off - (e.name_off + e.name_len)
    # the record's last 3 bytes (strength, method) move out of the field: the extra length shrinks by 3
    struct.pack_into("<H", data, e.local_header_off + 28, xl - 3)
    data = bytes(data)
    dev = assert_like_oracle(data, b"p")
    assert dev[0][0] == -5


def test_zip_aes_encrypt_matches_oracle(a):
    from archive_b200 import _ffi
    from archive_b200.zip import aes_encrypt_batch
    payloads = [os.urandom(n) for n in (0, 1, 15, 16, 17, 1000, 70_000, (4 << 20) + 9)]
    salts = [os.urandom(16) for _ in payloads]
    got = aes_encrypt_batch(payloads, salts, b"abc123")
    for p, s, (ct, ver, mac) in zip(payloads, salts, got):
        buf = C.create_string_buffer(p, len(p) or 1)
        v, m = C.create_string_buffer(2), C.create_string_buffer(10)
        orc.L().orc_zip_aes_encrypt(buf, C.c_size_t(len(p)), s, b"abc123", C.c_size_t(6), v, m)
        assert (ct, ver, mac) == (buf.raw[:len(p)], v.raw, m.raw)
    with pytest.raises(_ffi.B200ZError):
        aes_encrypt_batch([b"x"], [bytes(16)], b"")


@pytest.mark.parametrize("layout", ["dir_after_file", "dir_first"])
def test_zip_encoder_password_matches_oracle(a, layout):
    import time
    from archive_b200.zip import ArchiveFile, ZipEncoder, _dos_date, _dos_time
    files = [("a.txt", b"hello world" * 5000, "deflate", 1), ("d/", b"", "deflate", 0), ("b.bin", os.urandom(3000), "none", 1),
             ("c.bz", b"bzip2 " * 999, "bzip2", 1), ("e/", b"", "deflate", 0)]
    if layout == "dir_first":
        files = [files[1], files[0]] + files[2:]
    ents = []
    for name, content, method, is_file in files:
        f = ArchiveFile(name, len(content), is_file=bool(is_file))
        f.content = content if is_file else None
        f.compression = method if is_file else None
        f.mode = 0o644
        ents.append(f)
    salts = [bytes((29 * i + k) & 0xFF for k in range(16)) for i in range(len(files))]
    it = iter([s for s, f in zip(salts, files) if f[3]])
    mt = time.mktime((2021, 1, 2, 3, 4, 6, 0, 0, -1))
    for batch in (False, True):
        it = iter([s for s, f in zip(salts, files) if f[3]])
        got = ZipEncoder(password="abc123", salt=lambda: next(it), batch=batch).encode_bytes(ents, level=6, modified=mt)
        lm = time.localtime(mt)
        arr = (orc.ZipMemberIn * len(files))()
        keep = []
        for i, (name, content, method, is_file) in enumerate(files):
            nb = name.encode()
            keep += [nb, content]
            arr[i] = orc.ZipMemberIn(nb, content, len(content), {"none": 0, "deflate": 1, "bzip2": 2}[method], is_file, 0o644,
                                     _dos_time(lm), _dos_date(lm), None)
        out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
        st = orc.L().orc_zip_encode_password(arr, C.c_size_t(len(files)), 6, b"", b"abc123", C.c_size_t(6), b"".join(salts),
                                             C.byref(out), C.byref(n))
        assert st == orc.OK and got == orc._take(out, n), batch


def test_encode_password_round_trip(a):
    """test/zip_test.dart:625-648 ('encode password')"""
    from archive_b200.zip import ArchiveFile
    f = ArchiveFile("abc.txt", 11)
    f.content = b"hello world"
    data = a.ZipEncoder(password="abc123").encode_bytes([f])
    arc = a.ZipDecoder().decode_bytes(data, password="abc123")
    assert len(arc) == 1 and arc.files[0].read_bytes() == b"hello world"


def test_extract_file_to_disk_with_password(a, tmp_path):
    src = tmp_path / "aes256.zip"
    src.write_bytes(fixture("aes256.zip"))
    a.extract_file_to_disk(str(src), str(tmp_path / "out"), password="12345")
    body = (tmp_path / "out" / "readme.notzip").read_bytes()
    assert hashlib.sha256(body).hexdigest() == MAN["plaintext"]["readme.notzip"]["sha256"]
