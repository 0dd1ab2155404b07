"""K12 (inflate_chunked.cuh): one DEFLATE stream decoded by many chunks, on the emulated library (the whole product library
compiled for the host, tests/host_emul/build_emu_lib.py).  The chunk size is forced down to a few KiB through the test hook
so that every stream has dozens of chunks.  Each case is decoded twice by the same library -- through K12, and with the
threshold out of reach so that the exact single-unit path runs -- and the two results must be identical (status, bytes,
input used); valid streams are also checked against Python's zlib and the oracle.  The statistics hook tells which path
produced the result."""
import ctypes as C
import os
import random
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "host_emul"))
sys.path.insert(0, os.path.dirname(HERE))

import deflate_craft as dc  # noqa: E402
import oracle_lib as orc  # noqa: E402
from archive_b200 import synth  # noqa: E402

OFF = 1 << 62  # a threshold no stream reaches: the exact path


class Lib:
    def __init__(self, path):
        self.L = C.CDLL(path)
        assert self.L.b200z_init(0, 0) == 0

    def set(self, thresh, chunk=0):
        self.L.b200z_debug_inflate_chunked_set(C.c_ulonglong(thresh), C.c_ulonglong(chunk))

    def stats(self):
        a = (C.c_ulonglong * 6)()
        self.L.b200z_debug_inflate_chunked_stats(a)
        return dict(zip(("regions", "chunks", "redo", "merged", "fell_back", "ran"), list(a)))

    def inflate(self, data, cap=None):
        cap = cap if cap is not None else 8 * len(data) + (1 << 16)
        out = C.create_string_buffer(max(cap, 1))
        n, used, ust = C.c_size_t(), C.c_size_t(), C.c_int32()
        rc = self.L.b200z_inflate_raw(data, C.c_size_t(len(data)), out, C.c_size_t(cap), C.byref(n), C.byref(used), C.byref(ust))
        return rc, out.raw[:n.value], used.value, ust.value

    def gzip(self, data, cap):
        out = C.create_string_buffer(cap)
        n = C.c_size_t()
        rc = self.L.b200z_gzip_decode(data, C.c_size_t(len(data)), 0, out, C.c_size_t(cap), C.byref(n))
        return rc, out.raw[:min(n.value, cap)]

    def zlib(self, data, cap):
        out = C.create_string_buffer(cap)
        n = C.c_size_t()
        rc = self.L.b200z_zlib_decode(data, C.c_size_t(len(data)), 0, 0, out, C.c_size_t(cap), C.byref(n))
        return rc, out.raw[:min(n.value, cap)]


@pytest.fixture(scope="module")
def E():
    import build_emu_lib
    lib = Lib(build_emu_lib.build())
    yield lib
    lib.set(0, 0)


def both(E, fn, chunk=4096, thresh=16384):
    E.set(OFF)
    ref = fn()
    E.set(thresh, chunk)
    got = fn()
    st = E.stats()
    E.set(OFF)
    assert got == ref
    return got, st


def raw(data, level=6, wbits=15, mem=8, strategy=zlib.Z_DEFAULT_STRATEGY, flush_every=0, flush=zlib.Z_SYNC_FLUSH):
    c = zlib.compressobj(level, zlib.DEFLATED, -wbits, mem, strategy)
    if not flush_every:
        return c.compress(data) + c.flush()
    out = []
    for i in range(0, len(data), flush_every):
        out.append(c.compress(data[i:i + flush_every]))
        out.append(c.flush(flush))
    return b"".join(out) + c.flush()


TEXT = synth.text(400_000, stream=3).tobytes()


def check_clean(E, comp, plain, chunk=4096, thresh=16384):
    # two bytes of padding: the reference stops short when the last code of a stream lies in its last maxCodeLength
    # bits (DESIGN.md K1, Q1); test_final_block_in_last_bytes covers that case on its own
    data = comp + b"\0\0"
    (rc, out, used, ust), st = both(E, lambda: E.inflate(data, cap=len(plain) + 4096), chunk=chunk, thresh=thresh)
    assert rc == 0 and ust == 0 and out == plain and used == len(comp)
    assert orc.inflate(data)[1:] == (plain, len(comp))
    return st


@pytest.mark.parametrize("level,wbits,mem", [(1, 15, 8), (6, 15, 8), (9, 15, 9), (6, 9, 8), (6, 12, 1), (9, 10, 1),
                                             (3, 15, 2), (6, 15, 5)])
def test_text_levels(E, level, wbits, mem):
    comp = raw(TEXT, level, wbits, mem)
    st = check_clean(E, comp, TEXT, chunk=2048, thresh=65536)
    assert st["ran"] == 1 and st["fell_back"] == 0 and st["chunks"] >= 3, st


def test_stored_level0_and_random(E):
    # streams of stored blocks stay on the exact path (it moves a stored block as one run); the result is the same
    st = check_clean(E, raw(TEXT[:100_000], 0), TEXT[:100_000], chunk=8192)
    assert st["fell_back"] == 1, st
    rnd = np.random.default_rng(5).integers(0, 256, 120_000, dtype=np.uint8).tobytes()
    check_clean(E, raw(rnd, 6), rnd, chunk=8192)
    # text and random data in turns: dynamic and stored blocks, the stored ones decoded by the chunks
    mix = b"".join(TEXT[i * 30_000:(i + 1) * 30_000] + rnd[i * 8_000:(i + 1) * 8_000] for i in range(12))
    st = check_clean(E, raw(mix, 6), mix, chunk=4096, thresh=65536)
    assert st["fell_back"] == 0 and st["chunks"] >= 4, st


def test_fixed_huffman_only_rle(E):
    check_clean(E, raw(TEXT, 6, strategy=zlib.Z_FIXED), TEXT)  # the finder sees no fixed block: merged, then the exact path
    st = check_clean(E, raw(TEXT, 6, strategy=zlib.Z_HUFFMAN_ONLY), TEXT, chunk=8192)
    assert st["fell_back"] == 0, st
    st = check_clean(E, raw(TEXT, 6, strategy=zlib.Z_RLE), TEXT)
    assert st["fell_back"] == 0, st


@pytest.mark.parametrize("flush", [zlib.Z_SYNC_FLUSH, zlib.Z_BLOCK, zlib.Z_FULL_FLUSH])
def test_flushed_every_few_hundred_bytes(E, flush):
    check_clean(E, raw(TEXT[:60_000], 6, flush_every=300, flush=flush), TEXT[:60_000])


def test_repetitive_markers_through_many_chunks(E):
    # long-range repeats in many small blocks (memLevel 1): symbols copied from markers, and markers of markers
    rng = random.Random(3)
    plain = bytearray((TEXT[:700] * 600)[:400_000])
    for i in range(0, len(plain), 40):
        plain[i] = rng.randrange(256)
    plain = bytes(plain)
    st = check_clean(E, raw(plain, 9, mem=1), plain, chunk=1024, thresh=8192)
    assert st["ran"] == 1 and st["fell_back"] == 0 and st["chunks"] >= 8, st


def test_distance_32768_across_chunk_edge(E):
    rng = random.Random(7)
    head = bytes(rng.randrange(256) for _ in range(32768))
    plain = TEXT[:60_000] + head + head[:258] * 3 + TEXT[60_000:110_000] + head[:258] + TEXT[:258]
    st = check_clean(E, raw(plain, 9), plain, chunk=2048)
    assert st["ran"] == 1 and st["fell_back"] == 0, st


def seg(data, level=9):
    """data as a raw DEFLATE piece on its own: dynamic blocks, none final, then zlib's empty stored block"""
    c = zlib.compressobj(level, zlib.DEFLATED, -15)
    return c.compress(data) + c.flush(zlib.Z_SYNC_FLUSH)


def test_short_chunks_and_false_candidate(E):
    # stored blocks whose payload is a whole valid non-final dynamic block: the finder takes it for a block start, the
    # chunk decoded from there is not on the chain and is redone
    u = dc.Unit()
    for i in range(30):
        for k in range(3):
            part = TEXT[(3 * i + k) * 4000:(3 * i + k + 1) * 4000]
            u.w.raw(seg(part))
            u.plain += part
        u.stored(seg(TEXT[300_000 + i * 1000:300_000 + (i + 1) * 1000]) + TEXT[i * 300:(i + 1) * 300])
    u.stored(b"end", final=True)
    comp, plain = u.w.getvalue(), bytes(u.plain)
    st = check_clean(E, comp, plain, chunk=2048)
    assert st["ran"] == 1 and st["fell_back"] == 0 and st["chunks"] >= 8, st


def test_final_block_in_last_bytes(E):
    # no padding: whatever the reference makes of a last code in the last bits (Q1), K12 must give the same
    for level in (1, 6, 9):
        comp = raw(TEXT, level)
        got, _ = both(E, lambda: E.inflate(comp, cap=len(TEXT) + 4096))
        st, oout, used = orc.inflate(comp)
        assert got[1] == oout and got[2] == used


def test_out_cap_one_short(E):
    comp = raw(TEXT, 6)
    (rc, out, used, ust), st = both(E, lambda: E.inflate(comp + b"\0\0", cap=len(TEXT) - 1))
    assert ust == -2 and st["fell_back"] == 1
    (rc, out, used, ust), st = both(E, lambda: E.inflate(comp + b"\0\0", cap=len(TEXT)))
    assert out == TEXT and st["fell_back"] == 0


def test_bitflips_and_truncations(E):
    comp = raw(TEXT[:80_000], 6)
    rng = random.Random(11)
    for _ in range(12):
        b = bytearray(comp)
        p = rng.randrange(len(b))
        b[p] ^= 1 << rng.randrange(8)
        both(E, lambda: E.inflate(bytes(b)))
    for cut in (len(comp) - 1, len(comp) - 7, len(comp) // 2, 5000):
        both(E, lambda: E.inflate(comp[:cut]))


def gz(data, level=6):
    c = zlib.compressobj(level, zlib.DEFLATED, 31)
    return c.compress(data) + c.flush()


def test_gzip_members_hinted_and_unhinted(E):
    a, b, c = TEXT[:70_000], TEXT[70_000:120_000], TEXT[120_000:]
    blob = gz(a) + b"".join(synth.gzip_members(np.frombuffer(b, np.uint8), workers=1)) + gz(c)
    (rc, out), st = both(E, lambda: E.gzip(blob, len(TEXT) + 100))
    assert rc == 0 and out == TEXT == orc.gzip_decode(blob)[1]


def test_members_reaching_into_previous_output(E):
    # each member is compressed with the preceding output as a preset dictionary: its first chunk's markers resolve into
    # the members before it
    parts = [TEXT[i:i + 40_000] for i in range(0, 160_000, 40_000)]
    blob, prev = b"", b""
    for p in parts:
        co = zlib.compressobj(6, zlib.DEFLATED, -15, 8, zlib.Z_DEFAULT_STRATEGY, zdict=prev[-32768:] if prev else b"\0")
        body = co.compress(p) + co.flush()
        blob += b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff" + body + zlib.crc32(p).to_bytes(4, "little") + \
            (len(p) & 0xffffffff).to_bytes(4, "little")
        prev += p
    (rc, out), st = both(E, lambda: E.gzip(blob, len(TEXT) + 100), chunk=1024, thresh=4096)
    assert rc == 0 and out == b"".join(parts) == orc.gzip_decode(blob)[1]
    assert st["ran"] == 1 and st["fell_back"] == 0, st  # (the last member's call)


def test_many_small_members_regions_bounded(E):
    parts = [TEXT[i:i + 6000] for i in range(0, 60_000, 6000)]
    blob = b"".join(gz(p) for p in parts)
    (rc, out), st = both(E, lambda: E.gzip(blob, len(TEXT) + 100), chunk=1024, thresh=2048)
    assert rc == 0 and out == b"".join(parts)
    assert st["regions"] <= 4, st


def test_zlib_stream(E):
    comp = zlib.compress(TEXT, 6)
    (rc, out), st = both(E, lambda: E.zlib(comp, len(TEXT) + 100))
    assert rc == 0 and out == TEXT == orc.zlib_decode(comp)[1]
    assert st["ran"] == 1 and st["fell_back"] == 0, st


def test_small_out_cap_band(E):
    # caps whose workspace is just above K12's fixed part: the exact path's NOSPC, and no pool carved past the workspace
    comp = raw(TEXT, 6) + b"\0\0"
    for cap in list(range(15_900, 16_500, 3)) + [20_000, 65_536]:
        (rc, out, used, ust), st = both(E, lambda: E.inflate(comp, cap=cap))
        assert ust == -2 and st["fell_back"] == 1, (cap, st)
