"""K12 (inflate_chunked.cuh) on the device: large single DEFLATE streams through Inflate, GZipDecoder and ZLibDecoder at the
built-in chunk size, checked against Python's zlib.  The threshold is lowered to 1 MiB of compressed input so that streams
of 16 MiB and more of output take K12; the largest case runs at the built-in threshold.  The statistics hook must show
that the chunked path, not the fallback, produced every clean stream that is not made of stored blocks.  The CPU tier (tests/test_inflate_chunked_emul.py) covers the edge cases
with forced small chunks; this file also runs a few of them at full size."""
import ctypes as C
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MiB = 1 << 20
LOW = 1 * MiB  # K12 threshold for these tests (compressed bytes)


@pytest.fixture(scope="module")
def a():
    import archive_b200
    return archive_b200


@pytest.fixture(scope="module")
def L(a):
    from archive_b200 import _ffi
    _ffi.ensure_init()
    lib = _ffi.lib()
    lib.b200z_debug_inflate_chunked_set(C.c_ulonglong(LOW), C.c_ulonglong(0))
    yield lib
    lib.b200z_debug_inflate_chunked_set(C.c_ulonglong(0), C.c_ulonglong(0))


def stats(L):
    s = (C.c_ulonglong * 6)()
    L.b200z_debug_inflate_chunked_stats(s)
    return dict(zip(("regions", "chunks", "redo", "merged", "fell_back", "ran"), list(s)))


def text(n, stream=4):
    from archive_b200 import synth
    return synth.text(n, stream=stream).tobytes()


def raw(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy)
    return c.compress(data) + c.flush()


@pytest.mark.parametrize("size,thresh", [(16 * MiB, LOW), (64 * MiB, LOW), (256 * MiB, 0)])
def test_inflate_text(a, L, size, thresh):
    plain = text(size)
    comp = raw(plain) + b"\0\0"
    L.b200z_debug_inflate_chunked_set(C.c_ulonglong(thresh), C.c_ulonglong(0))
    try:
        out = a.Inflate(comp, uncompressed_size=len(plain) + 4096).get_bytes()
    finally:
        L.b200z_debug_inflate_chunked_set(C.c_ulonglong(LOW), C.c_ulonglong(0))
    st = stats(L)
    assert out == plain
    assert st["ran"] == 1 and st["fell_back"] == 0, st


def test_gzip_and_zlib(a, L):
    plain = text(48 * MiB, stream=5)
    c = zlib.compressobj(6, zlib.DEFLATED, 31)
    gz = c.compress(plain) + c.flush()
    assert a.GZipDecoder().decode_bytes(gz) == plain
    st = stats(L)
    assert st["ran"] == 1 and st["fell_back"] == 0, st
    zz = zlib.compress(plain, 9)
    assert a.ZLibDecoder().decode_bytes(zz) == plain
    st = stats(L)
    assert st["ran"] == 1 and st["fell_back"] == 0, st


def test_random_and_stored(a, L):
    rnd = np.random.default_rng(9).integers(0, 256, 40 * MiB, dtype=np.uint8).tobytes()
    assert a.Inflate(raw(rnd) + b"\0\0", uncompressed_size=len(rnd) + 4096).get_bytes() == rnd
    st = stats(L)
    assert st["ran"] == 1 and st["fell_back"] == 1, st  # mostly stored blocks: left to the exact path
    plain = text(24 * MiB, stream=6)
    assert a.Inflate(raw(plain, 0) + b"\0\0", uncompressed_size=len(plain) + 4096).get_bytes() == plain


@pytest.mark.parametrize("strategy", [zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE])
def test_strategies(a, L, strategy):
    plain = text(24 * MiB, stream=7)
    assert a.Inflate(raw(plain, 6, strategy) + b"\0\0", uncompressed_size=len(plain) + 4096).get_bytes() == plain


def test_many_members_and_damage(a, L):
    plain = text(32 * MiB, stream=8)
    parts = [plain[i:i + 256 * 1024] for i in range(0, len(plain), 256 * 1024)]
    blob = b"".join(zlib.compress(p, 6, 31) for p in parts)  # unhinted gzip members
    assert a.GZipDecoder().decode_bytes(blob) == plain
    # a damaged stream: whatever the exact path gives (here checked against the exact path itself)
    comp = bytearray(raw(plain[:20 * MiB]))
    comp[len(comp) // 2] ^= 0x10
    def run():
        try:
            r = a.Inflate(bytes(comp), uncompressed_size=21 * MiB)
            return r.get_bytes(), r.status
        except Exception as e:  # a throw of the reference
            return type(e).__name__, str(e)

    got = run()
    L.b200z_debug_inflate_chunked_set(C.c_ulonglong(1 << 62), C.c_ulonglong(0))
    try:
        assert got == run()
    finally:
        L.b200z_debug_inflate_chunked_set(C.c_ulonglong(LOW), C.c_ulonglong(0))


def test_members_reaching_into_previous_output(a, L):
    # each member is compressed with the output before it as a preset dictionary: the first chunk's markers of every
    # member resolve into the members in front of it
    plain = text(24 * MiB, stream=11)
    parts = [plain[i:i + 8 * MiB] for i in range(0, len(plain), 8 * MiB)]
    blob, prev = b"", b""
    for p in parts:
        co = zlib.compressobj(6, zlib.DEFLATED, -15, 8, zlib.Z_DEFAULT_STRATEGY, zdict=prev[-32768:] if prev else b"\0")
        body = co.compress(p) + co.flush()
        blob += b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff" + body + zlib.crc32(p).to_bytes(4, "little") + \
            len(p).to_bytes(4, "little")
        prev += p
    assert a.GZipDecoder().decode_bytes(blob) == plain
    st = stats(L)
    assert st["ran"] == 1 and st["fell_back"] == 0, st  # (the last member)
