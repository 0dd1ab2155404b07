"""The device BZip2 encoder's multi-stream driver (bz2e::encode_streams, archive_b200/csrc/bzip2_enc_*) on the CUDA
execution-model emulation: many streams in one pass, each starting on its own 4 KiB input tile, with blocks of different
streams in one block batch.  Every stream must equal the oracle's encodeBytes of that stream alone, decode with libbz2,
and its CRC-32 must equal zlib's.

The cases are the places where one stream can leak into the next: RLE1 runs that end a stream and start the next with the
same byte (a driver whose run scan crossed the boundary would merge them), empty and 1-byte streams, tile edges, the block
cut, a periodic block (serial sort) next to text blocks, block batches that hold the end of one stream and the start of
the next, and repeated or overlapping input ranges."""
import bz2
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest

import bz2_stream as bs
import oracle_lib as orc

_LIB = None
CUT = 899982  # the longest stream of distinct-neighbour bytes that is one block


def lib():
    global _LIB
    if _LIB is None:
        emul = os.path.join(orc.ROOT, "tests", "host_emul")
        csrc = os.path.join(orc.ROOT, "archive_b200", "csrc")
        src = os.path.join(emul, "bz2enc_multi_emul.cpp")
        so = os.path.join(emul, "libbz2enc_multi_emul.so")
        deps = [src, os.path.join(emul, "cuda_emu.h")] + [
            os.path.join(csrc, f) for f in os.listdir(csrc) if f.startswith("bzip2_enc")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
            subprocess.run(["g++", "-O2", "-g", "-fPIC", "-shared", "-std=c++17", "-I", emul, "-I", csrc, src, "-o", so],
                           check=True)
        _LIB = C.CDLL(so)
    return _LIB


def encode_multi(buf: bytes, ranges, max_batch=0):
    """Streams buf[off:off + len] for (off, len) in ranges, in one pass -> (list of (payload, crc32), stats)."""
    n = len(ranges)
    off = np.array([r[0] for r in ranges], dtype=np.uint64)
    ln = np.array([r[1] for r in ranges], dtype=np.uint64)
    cap = sum(L + L // 32 + 8192 + 320 for _, L in ranges) + 16
    out = np.zeros(cap, dtype=np.uint8)
    out_off, out_len = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint64)
    crc = np.zeros(n, dtype=np.uint32)
    st = np.zeros(5, dtype=np.uint32)
    src = np.frombuffer(buf if buf else b"\0", dtype=np.uint8)
    p = lambda a: C.c_void_p(a.ctypes.data)
    rc = lib().emu_bzip2_encode_multi(p(src), p(off), p(ln), C.c_size_t(n), C.c_uint32(max_batch), p(out), p(out_off),
                                      p(out_len), p(crc), p(st))
    assert rc == 0
    res = [(out[int(out_off[i]):int(out_off[i] + out_len[i])].tobytes(), int(crc[i])) for i in range(n)]
    return res, [int(x) for x in st]


def check_streams(streams, max_batch=0):
    """Encode `streams` packed back to back; every one must be the oracle's bytes and carry zlib's CRC-32."""
    buf = b"".join(streams)
    ranges, at = [], 0
    for s in streams:
        ranges.append((at, len(s)))
        at += len(s)
    return check_ranges(buf, ranges, max_batch)


def check_ranges(buf, ranges, max_batch=0):
    res, st = encode_multi(buf, ranges, max_batch)
    assert st[0] == sum(len(bs.parse(z).blocks) for z, _ in res)  # blocks of all streams
    for k, ((o, L), (z, crc)) in enumerate(zip(ranges, res)):
        data = buf[o:o + L]
        assert z == orc.bzip2_encode(data)[1], f"stream {k} ({L} bytes)"
        assert bz2.decompress(z) == data, k
        assert crc == zlib.crc32(data), k
    return res, st


def text(n, seed):
    from archive_b200 import synth
    return synth.text(n, stream=seed).tobytes() if n else b""


def norun(n, seed):
    r = np.random.default_rng(seed)
    a = np.cumsum(r.integers(1, 255, n)) % 256
    return a.astype(np.uint8).tobytes()


@pytest.mark.parametrize("tail,head", [(200, 300), (3, 1), (254, 1), (255, 1), (256, 1), (255, 300), (4, 4)])
@pytest.mark.parametrize("a_len", [None, 8192])
def test_run_across_stream_boundary(tail, head, a_len):
    """A ends in `tail` x 'a' and B starts with `head` x 'a': two runs, one per stream (RLE1 threshold 4, chunks of 255).
    With a_len 8192, A ends on a tile edge, so B's first byte sits right behind A's last one in the staged input."""
    a = text((a_len or 5000 + tail) - tail, 1) + b"a" * tail
    b = b"a" * head + text(3000, 2)
    check_streams([a, b, b"a" * tail, b"a" * head, b"a" * 7])


def test_runs_across_tiles_and_streams():
    """Streams of one byte value whose lengths straddle the 4 KiB tile: a merged run would span the padding."""
    check_streams([b"a" * 4095, b"a" * 4096, b"a" * 4097, b"a" * 1, b"a" * 8193, b"b" * 300, b"b" * 5])


def test_empty_and_one_byte_streams():
    check_streams([b"", text(2000, 3), b"", b"x", b"", b"", b"", text(1500, 4), b"y", b"", b"z" * 1, b""])
    check_streams([b"", b"", b""])
    check_streams([b"q"])


def test_tile_edge_lengths():
    check_streams([text(4095, 5), text(4096, 6), text(4097, 7), text(1, 8), text(8192, 9)])


def test_stream_at_block_cut():
    """A stream exactly at the block cut is one block; one byte more takes two."""
    a = norun(CUT, 10)
    res, st = check_streams([b"ab", a, a + a[:1], b"c"])
    assert [len(bs.parse(z).blocks) for z, _ in res] == [1, 1, 2, 1]


def test_multi_block_stream_between_tiny_ones():
    big = text(2_400_000, 11)
    res, st = check_streams([b"t", big, b"u" * 10, text(700, 12)])
    assert len(bs.parse(res[1][0]).blocks) == 3


def test_periodic_stream_in_a_text_batch():
    """A periodic stream needs the serial sort; it shares the block batch with text streams."""
    per = b"abc" * 20000
    res, st = check_streams([text(30000, 13), per, text(20000, 14), text(9000, 15)])
    assert st[0] == 4 and st[1] == 1 and st[4] == 1


@pytest.mark.parametrize("max_batch", [1, 2, 3])
def test_batches_split_across_streams(max_batch):
    """With 1, 2 or 3 blocks per batch, a batch holds the end of one stream and the start of the next, and the 3-block
    stream's blocks span batches: bit positions and combined CRCs carry across batches per stream."""
    streams = [text(1200, 16), text(2_000_000, 17), b"a" * 900, b"a" * 1000, text(5000, 18), b"", b"abc" * 9000]
    res, st = check_streams(streams, max_batch)
    assert st[0] == 1 + 3 + 1 + 1 + 1 + 1 and len(bs.parse(res[1][0]).blocks) == 3
    assert st[4] == -(-st[0] // max_batch)


def test_repeated_and_overlapping_ranges():
    buf = text(20000, 19) + b"a" * 600 + text(9000, 20)
    ranges = [(0, 20000), (0, 20000), (19000, 1600), (19500, 1100), (20000, 600), (20100, 500), (5, 29595), (0, 0)]
    check_ranges(buf, ranges)


def test_many_small_streams():
    r = np.random.default_rng(21)
    streams = [text(int(r.integers(0, 9000)), 100 + k) for k in range(40)]
    check_streams(streams, 7)
