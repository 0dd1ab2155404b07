"""The oracle's ZIP encryption (oracle/aes.c, zip_crypt.c, zip_enc_crypt.c) against published known answers, the reference's encrypted
fixtures, CPython's zipfile and the `cryptography` package; and the Python ZipEncoder's password container against the
oracle encoder.  CPU only."""
import ctypes as C
import hashlib
import hmac
import io
import json
import os
import struct
import zipfile

import pytest

import oracle_lib as orc
import zip_crypt_build as zb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "zip_crypt")
MAN = json.load(open(os.path.join(GOLD, "manifest.json")))
BAD_PASSWORD, BAD_MAC = 4, 5


def aes_block(key, block):
    rk = (C.c_uint32 * 60)()
    nr = orc.L().orc_aes_expand(key, len(key), rk)
    out = C.create_string_buffer(16)
    orc.L().orc_aes_encrypt_block(rk, nr, block, out)
    return out.raw


@pytest.mark.parametrize("key,expect", [  # FIPS-197 Appendix C.1-C.3
    (bytes(range(16)), "69c4e0d86a7b0430d8cdb78070b4c55a"),
    (bytes(range(24)), "dda97ca4864cdfe06eaf70a0ec0d7191"),
    (bytes(range(32)), "8ea2b7ca516745bfeafc49904b496089")])
def test_aes_fips197(key, expect):
    assert aes_block(key, bytes.fromhex("00112233445566778899aabbccddeeff")).hex() == expect


@pytest.mark.parametrize("key,msg,expect", [  # RFC 2202 section 3
    (b"\x0b" * 20, b"Hi There", "b617318655057264e28bc0b6fb378c8ef146be00"),
    (b"Jefe", b"what do ya want for nothing?", "effcdf6ae5eb2fa2d27416d5f184df9c259a7c79"),
    (b"\xaa" * 20, b"\xdd" * 50, "125d7342b9ac11cd91a39af48aa17b4f63f175d3"),
    (b"\xaa" * 80, b"Test Using Larger Than Block-Size Key - Hash Key First", "aa4ae5e15272d00e95705637ce8a3b55ed402112"),
    (b"\xaa" * 80, b"Test Using Larger Than Block-Size Key and Larger Than One Block-Size Data",
     "e8e99d0f45237d786d6bbaa7965c7808bbff1a91")])
def test_hmac_sha1_rfc2202(key, msg, expect):
    assert zb.hmac_sha1(key, msg).hex() == expect


def test_pbkdf2_rfc6070_and_hashlib():
    out = C.create_string_buffer(20)
    orc.L().orc_pbkdf2_sha1(b"password", C.c_size_t(8), b"salt", C.c_size_t(4), 1, out, C.c_size_t(20))
    assert out.raw.hex() == "0c60c80f961f0e71f3a9b524af6012062fe037a6"
    orc.L().orc_pbkdf2_sha1(b"password", C.c_size_t(8), b"salt", C.c_size_t(4), 4096, out, C.c_size_t(20))
    assert out.raw.hex() == "4b007901b765489abead49d926f721d065a429c1"
    for n, sl in ((34, 8), (50, 12), (66, 16)):
        salt = os.urandom(sl)
        for pw in (b"12345", b"x" * 70, bytes(range(1, 200))):
            assert zb.pbkdf2(pw, salt, n) == hashlib.pbkdf2_hmac("sha1", pw, salt, 1000, n)


@pytest.mark.parametrize("n", [0, 1, 15, 16, 17, 3 * (1 << 20) + 5])
@pytest.mark.parametrize("ks", [16, 24, 32])
def test_winzip_ctr_against_cryptography(n, ks):
    ciphers = pytest.importorskip("cryptography.hazmat.primitives.ciphers")
    key, data = os.urandom(ks), os.urandom(n)
    # the WinZip counter block: little-endian block number from 1 in bytes 0-3 (a 128-bit little-endian counter, for
    # fewer than 2^32 blocks)
    enc = ciphers.Cipher(ciphers.algorithms.AES(key), ciphers.modes.ECB()).encryptor()
    nb = (n + 15) // 16
    ks_stream = enc.update(b"".join(struct.pack("<I12x", i + 1) for i in range(nb))) if nb else b""
    assert zb.winzip_ctr(key, data) == bytes(a ^ b for a, b in zip(data, ks_stream))


def fixture(name):
    return open(os.path.join(GOLD, name), "rb").read()


@pytest.mark.parametrize("name", sorted(MAN["archives"]))
def test_oracle_decodes_the_fixtures(name):
    spec = MAN["archives"][name]
    data = fixture(name)
    st, ents = orc.zip_list(data)
    assert st == orc.OK and len(ents) == len(spec["members"])
    got = zb.oracle_members(data, spec["password"].encode())
    for e, (s, body) in zip(ents, got):
        nm = data[e.name_off:e.name_off + e.name_len].decode()
        assert nm in spec["members"] and s == orc.OK
        plain = MAN["plaintext"][nm]
        assert len(body) == plain["size"] and hashlib.sha256(body).hexdigest() == plain["sha256"]
        if spec["mode"] == "zipcrypto":
            assert body == zipfile.ZipFile(io.BytesIO(data)).read(nm, pwd=spec["password"].encode())
    # without a password: reported, not decoded (unchanged)
    assert all(s == orc.FALSE and b == b"" for s, b in zb.oracle_members(data, None))


def test_oracle_crypt_info_of_the_fixtures():
    for name, spec in MAN["archives"].items():
        data = fixture(name)
        for e in orc.zip_list(data)[1]:
            mode, strength, method = C.c_uint32(), C.c_uint32(), C.c_uint32()
            assert orc.L().orc_zip_crypt_info(data, C.c_size_t(len(data)), C.byref(e), C.byref(mode), C.byref(strength),
                                              C.byref(method)) == orc.OK
            assert mode.value == (2 if spec["mode"] == "aes" else 1)
            if spec["mode"] == "aes":
                assert e.method == 99 and strength.value == 3 and method.value in (0, 8)


def test_oracle_aes_errors():
    data = fixture("aes256.zip")
    assert {s for s, _ in zb.oracle_members(data, b"wrong")} == {BAD_PASSWORD}
    assert {s for s, _ in zb.oracle_members(data, b"")} == {orc.THROW}
    st, ents = orc.zip_list(data)
    bad = bytearray(data)
    bad[ents[1].data_off + 20] ^= 0x40  # a ciphertext byte
    got = zb.oracle_members(bytes(bad), b"12345")
    assert got[0][0] == orc.OK and got[1] == (BAD_MAC, b"")


def test_oracle_written_zipcrypto_reads_back_through_zipfile():
    text = bytes(range(256)) * 300
    ms = [zb.Member("a.txt", text, 8, "zipcrypto"), zb.Member("b.bin", os.urandom(5000), 0, "zipcrypto"),
          zb.Member("c.txt", b"", 0, "zipcrypto"), zb.Member("d.txt", text[:999], 8, "zipcrypto", dd=True)]
    arc = zb.build(ms, b"secret")
    z = zipfile.ZipFile(io.BytesIO(arc))
    for m, (s, body) in zip(ms, zb.oracle_members(arc, b"secret")):
        assert z.read(m.name, pwd=b"secret") == m.data == body and s == orc.OK


def read_aes_with_cryptography(data: bytes, password: bytes):
    """an independent WinZip AES reader: zipfile for the directory, `cryptography` for the ciphers"""
    ciphers = pytest.importorskip("cryptography.hazmat.primitives.ciphers")
    import zlib
    out = {}
    z = zipfile.ZipFile(io.BytesIO(data))
    for info in z.infolist():
        off = info.header_offset
        fl, el = struct.unpack("<HH", data[off + 26:off + 30])
        ex = data[off + 30 + fl:off + 30 + fl + el]
        p = ex.find(b"\x01\x99\x07\x00")
        strength, method = ex[p + 8], struct.unpack("<H", ex[p + 9:p + 11])[0]
        body = data[off + 30 + fl + el:off + 30 + fl + el + info.compress_size]
        if not body:
            out[info.filename] = b""
            continue
        sl, ks = {1: (8, 16), 2: (12, 24), 3: (16, 32)}[strength]
        dk = hashlib.pbkdf2_hmac("sha1", password, body[:sl], 1000, 2 * ks + 2)
        assert body[sl:sl + 2] == dk[2 * ks:]
        ct, mac = body[sl + 2:-10], body[-10:]
        assert hmac.new(dk[ks:2 * ks], ct, "sha1").digest()[:10] == mac
        # the library's CTR mode counts big-endian: the little-endian counter blocks go through ECB instead
        enc = ciphers.Cipher(ciphers.algorithms.AES(dk[:ks]), ciphers.modes.ECB()).encryptor()
        nb = (len(ct) + 15) // 16
        stream = enc.update(b"".join(struct.pack("<I12x", i + 1) for i in range(nb)))
        plain = bytes(a ^ b for a, b in zip(ct, stream))
        out[info.filename] = zlib.decompress(plain, -15) if method == 8 else plain
    return out


def dos(t=0x21):
    return 0, t


def test_oracle_written_aes_reads_back_through_cryptography():
    text = (b"the quick brown fox jumps over the lazy dog\n" * 2000)
    members = [("x.txt", text, "deflate", 1), ("y.bin", os.urandom(777), "none", 1), ("e.txt", b"", "none", 1)]
    arr, salts = zip_members(members)
    st, arc = zip_encode_password(arr, salts, b"abc123")
    assert st == orc.OK
    got = read_aes_with_cryptography(arc, b"abc123")
    assert got == {"x.txt": text, "y.bin": members[1][1], "e.txt": b""}
    for (name, content, _, _), (s, body) in zip(members, zb.oracle_members(arc, b"abc123")):
        assert s == orc.OK and body == content


def zip_members(members):
    arr = [(name, content, method, bool(is_file), 0o644, 0x1234, 0x5678, None) for name, content, method, is_file in members]
    salts = b"".join(bytes((17 * i + k) & 0xFF for k in range(16)) for i in range(len(members)))
    return arr, salts


def zip_encode_password(members, salts, pw, level=1):
    arr = (orc.ZipMemberIn * max(1, len(members)))()
    keep = []
    for i, (name, content, method, is_file, mode, t, d, cm) in enumerate(members):
        nb = name.encode()
        keep += [nb, content]
        arr[i] = orc.ZipMemberIn(nb, content, len(content), {"none": 0, "deflate": 1, "bzip2": 2}[method], int(is_file), mode, t, d,
                                 None)
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    st = orc.L().orc_zip_encode_password(arr, C.c_size_t(len(members)), level, b"", pw, C.c_size_t(len(pw)), salts,
                                         C.byref(out), C.byref(n))
    return st, orc._take(out, n)


def oracle_encrypt(payloads, salts, pw):
    res = []
    for p, s in zip(payloads, salts):
        buf = C.create_string_buffer(bytes(p), len(p) or 1)
        ver, mac = C.create_string_buffer(2), C.create_string_buffer(10)
        orc.L().orc_zip_aes_encrypt(buf, C.c_size_t(len(p)), s, pw, C.c_size_t(len(pw)), ver, mac)
        res.append((buf.raw[:len(p)], ver.raw, mac.raw))
    return res


def oracle_compress(content, method, level):
    if method == "deflate":
        st, out, crc = orc.deflate(content, level)
        return out, crc
    if method == "bzip2":
        return orc.bzip2_encode(content)[1], orc.crc32(content)
    return bytes(content), orc.crc32(content)


@pytest.mark.parametrize("layout", ["dir_after_file", "dir_first"])
def test_python_zip_encoder_password_matches_the_oracle(layout):
    """ZipEncoder(password=) container bytes, with the device work replaced by oracle stand-ins: every quirk of the
    reference's encoder, including a directory after a file (compressedSize 12, that file's MAC behind the header)."""
    import time
    from archive_b200.zip import ArchiveFile, ZipEncoder
    files = [("a.txt", b"hello world" * 50, "deflate", 1), ("d/", b"", "deflate", 0), ("b.bin", bytes(range(200)), "none", 1),
             ("e/", b"", "deflate", 0)]
    if layout == "dir_first":
        files = [files[1]] + [files[0]] + files[2:]
    ents = []
    for name, content, method, is_file in files:
        f = ArchiveFile(name, len(content), is_file=bool(is_file))
        f.content = content if is_file else None
        f.compression = method if is_file else None
        f.mode = 0o644
        ents.append(f)
    salts = [bytes((17 * i + k) & 0xFF for k in range(16)) for i in range(len(files))]
    it = iter([s for s, (_, _, _, isf) in zip(salts, files) if isf])
    mt = time.mktime((2020, 5, 17, 10, 20, 30, 0, 0, -1))
    got = ZipEncoder(compress=oracle_compress, password="abc123", salt=lambda: next(it), encrypt=oracle_encrypt).encode_bytes(
        ents, level=6, modified=mt)
    from archive_b200.zip import _dos_date, _dos_time
    lm = time.localtime(mt)
    arr = [(name, content, method, bool(is_file), 0o644, _dos_time(lm), _dos_date(lm), None) for name, content, method, is_file in files]
    st, want = zip_encode_password(arr, b"".join(salts), b"abc123", level=6)
    assert st == orc.OK and got == want
    # the quirk itself: what ZipFile.read sees for the directories
    st, listed = orc.zip_list(want)
    for (name, _, _, is_file), e in zip(files, listed):
        assert e.method == 99 and e.flags & 1
        if not is_file:
            assert e.comp_size == (0 if layout == "dir_first" and name == "d/" else 12)


def test_python_password_bytes_are_dart_code_units():
    from archive_b200.zip import password_bytes
    assert password_bytes("12345") == b"12345"
    assert password_bytes("pä€") == bytes([0x70, 0xE4, 0xAC])
    assert password_bytes("\U0001F600") == bytes([0x3D, 0x00])  # a surrogate pair: two code units
    assert password_bytes(b"\xff\x00") == b"\xff\x00" and password_bytes(None) is None
