"""TEST INFRASTRUCTURE: builders of encrypted ZIP archives for the zip_crypt tests, on top of the oracle's ciphers
(oracle/aes.c).  The reference only writes AES-256 (oracle/zip_enc_crypt.c restates that); these write what it READS as well:
AES-128/192/256 and ZipCrypto members, stored / deflate / bzip2, data descriptors, foreign extra fields ahead of the AES
record, directories and symlinks."""
import ctypes as C
import struct
import zlib

import oracle_lib as orc

SALT_LEN = {1: 8, 2: 12, 3: 16}


def pbkdf2(pw: bytes, salt: bytes, n: int) -> bytes:
    out = C.create_string_buffer(n)
    orc.L().orc_pbkdf2_sha1(pw, C.c_size_t(len(pw)), salt, C.c_size_t(len(salt)), 1000, out, C.c_size_t(n))
    return out.raw


def hmac_sha1(key: bytes, msg: bytes) -> bytes:
    out = C.create_string_buffer(20)
    orc.L().orc_hmac_sha1(key, C.c_size_t(len(key)), msg, C.c_size_t(len(msg)), out)
    return out.raw


def winzip_ctr(key: bytes, data: bytes) -> bytes:
    buf = C.create_string_buffer(bytes(data), len(data) or 1)
    orc.L().orc_winzip_ctr(key, len(key), buf, C.c_size_t(len(data)))
    return buf.raw[:len(data)]


def zipcrypto_encrypt(pw: bytes, data: bytes) -> bytes:
    out = C.create_string_buffer(len(data) or 1)
    orc.L().orc_zipcrypto_encrypt(pw, C.c_size_t(len(pw)), bytes(data), C.c_size_t(len(data)), out)
    return out.raw[:len(data)]


def aes_payload(pw: bytes, salt: bytes, data: bytes, strength: int = 3, bad_mac: bool = False) -> bytes:
    ks = {1: 16, 2: 24, 3: 32}[strength]
    dk = pbkdf2(pw, salt, 2 * ks + 2)
    ct = winzip_ctr(dk[:ks], data)
    mac = hmac_sha1(dk[ks:2 * ks], ct)[:10]
    if bad_mac:
        mac = bytes([mac[0] ^ 1]) + mac[1:]
    return salt + dk[2 * ks:] + ct + mac


def compress(data: bytes, method: int, flush_every: int = 0) -> bytes:
    if method == 8:
        c = zlib.compressobj(6, zlib.DEFLATED, -15)
        if not flush_every:
            return c.compress(data) + c.flush()
        parts = []
        for i in range(0, len(data), flush_every):
            parts.append(c.compress(data[i:i + flush_every]) + c.flush(zlib.Z_FULL_FLUSH))
        return b"".join(parts) + c.flush()
    if method == 12:
        import bz2
        return bz2.compress(data, 9)
    return bytes(data)


class Member:
    """one entry of a test archive.  crypt: None | 'zipcrypto' | 'aes'; strength 1/2/3 for AES."""

    def __init__(self, name, data=b"", method=8, crypt="aes", strength=3, is_dir=False, symlink=False, dd=False,
                 foreign_extra=False, flush_every=0, salt=None, bad_mac=False, truncate=None, password=None):
        self.__dict__.update(locals())
        del self.__dict__["self"]


def build(members, password: bytes) -> bytes:
    """a ZIP archive in the layout ZipEncoder writes, with each member encrypted as asked"""
    out, cd = bytearray(), bytearray()
    for i, m in enumerate(members):
        pw = m.password if m.password is not None else password
        payload = compress(m.data, m.method, m.flush_every) if not m.is_dir else b""
        crc = zlib.crc32(m.data) & 0xFFFFFFFF
        flags, method, extra = 0x800, m.method, b""
        if m.foreign_extra == "odd":  # an extended-timestamp record of 9 bytes: the reference's word-by-word walk then
            extra += struct.pack("<HHBI", 0x5455, 5, 1, 0x5F5E1000)  # steps over the AES id -> read as ZipCrypto
        elif m.foreign_extra:  # an NTFS times record (as in the reference's aes256.zip), walked word by word
            extra += struct.pack("<HHIHHQQQ", 0x000A, 32, 0, 1, 24, 0x01D4893DDAF3AD00, 0x01D8EA7E677E028C, 0x01D4893DDAF3AD00)
        if m.crypt == "zipcrypto" and not m.is_dir:
            flags |= 1
            # the check byte: high byte of the CRC, or of the DOS time when a data descriptor follows (the time is 0 here)
            header = bytes((7 * i + k) & 0xFF for k in range(11)) + bytes([0 if m.dd else crc >> 24])
            payload = zipcrypto_encrypt(pw, header + payload)
        elif m.crypt == "aes":
            flags |= 1
            extra += struct.pack("<HHH2sBH", 0x9901, 7, 2, b"AE", m.strength, m.method)
            method = 99
            if not m.is_dir:
                salt = m.salt or bytes((31 * i + 5 * k + 1) & 0xFF for k in range(SALT_LEN[m.strength]))
                payload = aes_payload(pw, salt, payload, m.strength, m.bad_mac)
        if m.truncate is not None:
            payload = payload[:m.truncate]
        if m.dd:
            flags |= 8
        name = m.name.encode()
        pos = len(out)
        out += struct.pack("<IHHHHHIIIHH", 0x04034B50, 20, flags, method, 0, 0x21, 0 if m.dd else crc,
                           0 if m.dd else len(payload), 0 if m.dd else len(m.data), len(name), len(extra))
        out += name + extra + payload
        if m.dd:
            out += struct.pack("<IIII", 0x08074B50, crc, len(payload), len(m.data))
        ver_made = (3 << 8) | 20 if m.symlink else 20
        attr = (0o120777 << 16) if m.symlink else ((0o40755 << 16) | 0x10 if m.is_dir else 0o100644 << 16)
        cd += struct.pack("<IHHHHHHIIIHHHHHII", 0x02014B50, ver_made, 20, flags, method, 0, 0x21, crc, len(payload),
                          len(m.data), len(name), 0, 0, 0, 0, attr, pos)
        cd += name
    cd_pos = len(out)
    out += cd
    out += struct.pack("<IHHHHIIH", 0x06054B50, 0, 0, len(members), len(members), len(cd), cd_pos, 0)
    return bytes(out)


def oracle_members(data: bytes, password, web_eos=False):
    """-> [(status, bytes)] of every listed member, from the oracle"""
    st, ents = orc.zip_list(data)
    assert st == orc.OK
    res = []
    for e in ents:
        out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
        pw = password
        s = orc.L().orc_zip_member_password(data, C.c_size_t(len(data)), C.byref(e), int(web_eos), pw,
                                            C.c_size_t(len(pw or b"")), C.byref(out), C.byref(n))
        res.append((s, orc._take(out, n)))
    return res
