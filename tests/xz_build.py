"""TEST INFRASTRUCTURE: oracle bindings for the XZ codec (oracle/xz.c) and a writer of .xz containers around Python `lzma`
FORMAT_RAW LZMA2 data: block count and size, check type, header size fields, chunk edits, and seeded damage."""
import ctypes as C
import lzma
import random
import struct
import zlib

import oracle_lib as orc

CHECK_FLAGS = {"none": 0, "crc32": 1, "crc64": 4, "sha256": 0xA}


def decode(data: bytes, verify=False):
    """-> (status, output) of the reference's XZDecoder().decodeBytes"""
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    st = orc.L().orc_xz_decode(bytes(data), C.c_size_t(len(data)), int(verify), C.byref(out), C.byref(n))
    return st, orc._take(out, n)


def encode(data: bytes, check=2):
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    st = orc.L().orc_xz_encode(bytes(data), C.c_size_t(len(data)), int(check), C.byref(out), C.byref(n))
    assert st == orc.OK
    return orc._take(out, n)


def crc64(data: bytes) -> int:
    orc.L().orc_crc64.restype = C.c_uint64
    return orc.L().orc_crc64(bytes(data), C.c_size_t(len(data)), C.c_uint64(0))


def sha256(data: bytes) -> bytes:
    d = C.create_string_buffer(32)
    orc.L().orc_sha256(bytes(data), C.c_size_t(len(data)), d)
    return d.raw


def _mbi(v: int) -> bytes:
    out = bytearray()
    while v >= 0x80:
        out.append(0x80 | (v & 0x7F))
        v >>= 7
    out.append(v)
    return bytes(out)


def _pad4(b: bytes) -> bytes:
    return b + bytes(-len(b) % 4)


def raw_lzma2(data: bytes, preset=6, lc=None, lp=None, pb=None, dict_size=None) -> bytes:
    f = {"id": lzma.FILTER_LZMA2, "preset": preset}
    for k, v in (("lc", lc), ("lp", lp), ("pb", pb), ("dict_size", dict_size)):
        if v is not None:
            f[k] = v
    return lzma.compress(data, format=lzma.FORMAT_RAW, filters=[f])


def chunks(raw: bytes):
    """LZMA2 data -> [(control, header bytes, payload bytes)] up to (not including) the end marker"""
    out, p = [], 0
    while raw[p] != 0:
        c = raw[p]
        if c & 0x80:
            hl = 6 if (c >> 5) & 3 >= 2 else 5
            cs = (raw[p + 3] << 8 | raw[p + 4]) + 1
            out.append((c, raw[p:p + hl], raw[p + hl:p + hl + cs]))
            p += hl + cs
        else:
            u = (raw[p + 1] << 8 | raw[p + 2]) + 1
            out.append((c, raw[p:p + 3], raw[p + 3:p + 3 + u]))
            p += 3 + u
    return out


def join(chs) -> bytes:
    return b"".join(h + d for _, h, d in chs) + b"\x00"


def container(blocks, check="crc64", sizes=(False, False), dict_byte=0x16, bad_check=False) -> bytes:
    """blocks: [(lzma2 data incl. end marker, uncompressed bytes)] -> one .xz stream (like liblzma's container);
    bad_check: every block check is inverted"""
    flags = CHECK_FLAGS[check]
    sf = bytes([0, flags])
    out = bytearray(b"\xfd7zXZ\x00" + sf + struct.pack("<I", zlib.crc32(sf)))
    recs = []
    for data, plain in blocks:
        szf = (_mbi(len(data)) if sizes[0] else b"") + (_mbi(len(plain)) if sizes[1] else b"")
        body = bytes([(0x40 if sizes[0] else 0) | (0x80 if sizes[1] else 0)]) + szf + b"\x21\x01" + bytes([dict_byte])
        hlen = (len(body) + 1 + 4 + 3) // 4 * 4
        hdr = bytes([hlen // 4 - 1]) + body
        hdr = hdr + bytes(hlen - 4 - len(hdr))
        blk = hdr + struct.pack("<I", zlib.crc32(hdr)) + data
        unpadded = len(blk)
        blk = _pad4(blk)
        if check == "crc32":
            ck = struct.pack("<I", zlib.crc32(plain))
        elif check == "crc64":
            ck = struct.pack("<Q", crc64(plain))
        elif check == "sha256":
            ck = sha256(plain)
        else:
            ck = b""
        if bad_check:
            ck = bytes(b ^ 0xFF for b in ck)
        out += blk + ck
        recs.append((unpadded + len(ck), len(plain)))
    idx = b"\x00" + _mbi(len(recs)) + b"".join(_mbi(u) + _mbi(n) for u, n in recs)
    idx = _pad4(idx)
    out += idx + struct.pack("<I", zlib.crc32(idx))
    ft = struct.pack("<I", (len(idx) + 4) // 4 - 1) + sf
    out += struct.pack("<I", zlib.crc32(ft)) + ft + b"YZ"
    return bytes(out)


def xz_blocks(data: bytes, block_size: int, check="crc64", **kw) -> bytes:
    """liblzma-style multi-block stream: every block is an independent LZMA2 stream (its first chunk resets)"""
    blocks = [(raw_lzma2(data[o:o + block_size], **kw), data[o:o + block_size]) for o in range(0, len(data), block_size)]
    return container(blocks, check=check)


def flip_bits(data: bytes, seed: int, n: int = 1) -> bytes:
    r = random.Random(seed)
    b = bytearray(data)
    for _ in range(n):
        i = r.randrange(len(b))
        b[i] ^= 1 << r.randrange(8)
    return bytes(b)
