"""b200z_bzip2_encode_batch and the bzip2 members of ZipEncoder(batch=True): every stream of a batch must come out exactly
as b200z_bzip2_encode gives it alone (rc, out_len, bytes) and as the oracle's BZip2Encoder restatement gives it
(oracle/bzip2_enc.c), whatever its neighbours in the input, in the block batches and in the device groups are."""
import bz2
import ctypes as C
import glob
import io
import os
import random
import time
import zipfile
import zlib

import pytest

import bz2_stream as bs
import oracle_lib as orc

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
from archive_b200._ffi import E_ARG, E_NOSPC  # noqa: E402


@pytest.fixture(scope="module")
def L():
    from archive_b200 import _ffi
    lib = _ffi.ensure_init()
    lib.b200z_debug_bzip2_encode_batch_set.argtypes = [C.c_uint]
    lib.b200z_debug_bzip2_encode_group_set.argtypes = [C.c_uint]
    lib.b200z_debug_bzip2_encode_batch_stats.argtypes = [C.c_void_p]
    yield lib
    lib.b200z_debug_bzip2_encode_batch_set(0)
    lib.b200z_debug_bzip2_encode_group_set(0)


def stats(L):
    s = (C.c_ulonglong * 5)()
    L.b200z_debug_bzip2_encode_batch_stats(s)
    return tuple(s)  # streams, device groups, block batches, blocks, serially sorted blocks of the last call


def single(L, data, room=None):
    """b200z_bzip2_encode alone -> (rc, out_len, bytes; None on E_NOSPC)"""
    room = L.b200z_bzip2_bound(len(data)) if room is None else room
    buf = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data or b"\0")
    out = (C.c_uint8 * max(room, 1))()
    n = C.c_size_t(0)
    rc = L.b200z_bzip2_encode(C.addressof(buf), len(data), C.addressof(out), room, C.byref(n))
    return rc, n.value, (None if rc == E_NOSPC else C.string_at(C.addressof(out), n.value))


def batch(L, data, offs, lens, rooms=None, with_crc=True):
    """b200z_bzip2_encode_batch over ranges of `data` -> ([(rc, out_len, bytes)], [crc32] or None)"""
    n = len(offs)
    rooms = rooms or [L.b200z_bzip2_bound(x) for x in lens]
    buf = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data or b"\0")
    out_off, tot = [], 0
    for r in rooms:
        out_off.append(tot)
        tot += r
    out = (C.c_uint8 * max(tot, 1))()
    a64 = lambda v: (C.c_uint64 * max(n, 1))(*v)
    ol, rc, crc = (C.c_uint64 * max(n, 1))(), (C.c_int32 * max(n, 1))(), (C.c_uint32 * max(n, 1))()
    r = L.b200z_bzip2_encode_batch(C.addressof(buf), a64(offs), a64(lens), n, C.addressof(out), a64(out_off), a64(rooms), ol,
                                   crc if with_crc else None, rc)
    assert r == 0, L.b200z_last_error()
    got = [(rc[i], ol[i], None if rc[i] == E_NOSPC else C.string_at(C.addressof(out) + out_off[i], ol[i])) for i in range(n)]
    return got, (list(crc[:n]) if with_crc else None)


def packed(streams):
    offs, pos = [], 0
    for s in streams:
        offs.append(pos)
        pos += len(s)
    return b"".join(streams), offs, [len(s) for s in streams]


def check_ranges(L, data, offs, lens, alone=True):
    got, crcs = batch(L, data, offs, lens)
    assert stats(L)[0] == len(offs)
    for i, (o, n) in enumerate(zip(offs, lens)):
        src = data[o:o + n]
        assert got[i][0] == 0, (i, got[i][:2])
        assert got[i][2] == orc.bzip2_encode(src)[1], (i, n)
        assert crcs[i] == zlib.crc32(src), i
        if alone:
            assert got[i] == single(L, src), i
    return got


def check(L, streams, alone=True):
    return check_ranges(L, *packed(streams), alone=alone)


def text(n, seed):
    from archive_b200 import synth
    return synth.text(n, stream=seed).tobytes() if n else b""


def catalogue():
    """the edge catalogue of tests/test_bzip2_enc_batch_emul.py, as lists of streams"""
    t = lambda n, s: text(n, s)
    for a_len in (None, 8192):  # 8192: A ends on a tile edge, right in front of B in the staged input
        for tail, head in ((200, 300), (3, 1), (254, 1), (255, 1), (256, 1)):
            yield [t((a_len or 5000 + tail) - tail, 1) + b"a" * tail, b"a" * head + t(3000, 2), b"a" * tail]
    yield [b"a" * 4095, b"a" * 4096, b"a" * 4097, b"a", b"a" * 8193]
    yield [b"", t(2000, 5), b"", b"x", b"", b"", b"", t(1500, 6), b"y", b""]
    yield [t(4095, 7), t(4096, 8), t(4097, 9)]
    yield [b"t", t(2_400_000, 10), b"u" * 10, t(700, 11)]


def test_catalogue(L):
    for streams in catalogue():
        check(L, streams)


def test_stream_at_the_block_cut(L):
    import numpy as np
    r = np.random.default_rng(12)
    a = (np.cumsum(r.integers(1, 255, 899982)) % 256).astype(np.uint8).tobytes()
    got = check(L, [b"ab", a, a + a[:1], b"c"])
    assert [len(bs.parse(z).blocks) for _, _, z in got] == [1, 1, 2, 1]


def test_periodic_stream_in_a_text_batch(L):
    check(L, [text(30000, 13), b"abc" * 20000, text(20000, 14), text(9000, 15)], alone=False)
    assert stats(L) == (4, 1, 1, 4, 1)


@pytest.mark.parametrize("max_batch", [1, 2, 3])
def test_block_batch_caps(L, max_batch):
    streams = [text(1200, 16), text(2_000_000, 17), b"a" * 900, b"a" * 1000, text(5000, 18), b"", b"abc" * 9000]
    L.b200z_debug_bzip2_encode_batch_set(max_batch)
    try:
        check(L, streams, alone=False)
        st = stats(L)
    finally:
        L.b200z_debug_bzip2_encode_batch_set(0)
    assert st[3] == 8 and st[2] == -(-8 // max_batch) and st[4] == 1


def test_repeated_and_overlapping_ranges(L):
    data = text(20000, 19) + b"a" * 600 + text(9000, 20)
    rng = [(0, 20000), (0, 20000), (19000, 1600), (19500, 1100), (20000, 600), (20100, 500), (5, 29595), (0, 0)]
    check_ranges(L, data, [o for o, _ in rng], [n for _, n in rng])


def test_golden_fixtures_shuffled_with_duplicates(L):
    files = [os.path.join(G, "cat.jpg"), os.path.join(G, "test2.tar")] + sorted(
        f for f in glob.glob(os.path.join(G, "zip", "*")) if os.path.isfile(f))
    items = [open(f, "rb").read() for f in files]
    items = items + items[:3]
    random.Random(21).shuffle(items)
    check(L, items)


def test_output_rooms(L):
    streams = [text(7000, 22), text(9000, 23), text(3000, 24)]
    need = [len(orc.bzip2_encode(s)[1]) for s in streams]
    data, offs, lens = packed(streams)
    got, _ = batch(L, data, offs, lens, rooms=[need[0], need[1] - 1, need[2]])
    assert got[1][:2] == (E_NOSPC, need[1])
    for i in (0, 2):
        assert got[i] == (0, need[i], orc.bzip2_encode(streams[i])[1])
    got, _ = batch(L, data, offs, lens, rooms=need)
    assert [g[0] for g in got] == [0, 0, 0]


def test_arguments(L):
    streams = [text(3000, 25), b"", text(100, 26)]
    data, offs, lens = packed(streams)
    got, crcs = batch(L, data, offs, lens, with_crc=False)
    assert crcs is None and [g[2] for g in got] == [orc.bzip2_encode(s)[1] for s in streams]
    buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
    out = (C.c_uint8 * 100000)()
    a64 = lambda v: (C.c_uint64 * 3)(*v)
    ol, rc = (C.c_uint64 * 3)(), (C.c_int32 * 3)()
    assert L.b200z_bzip2_encode_batch(C.addressof(buf), a64(offs), a64(lens), 3, C.addressof(out), a64([0, 30000, 30001]),
                                      a64([30001, 100, 100]), ol, None, rc) == E_ARG  # slots 0 and 1 overlap
    assert L.b200z_bzip2_encode_batch(C.addressof(buf), None, a64(lens), 3, C.addressof(out), a64([0, 1, 2]),
                                      a64([1, 1, 1]), ol, None, rc) == E_ARG
    assert L.b200z_bzip2_encode_batch(None, None, None, 0, None, None, None, None, None, None) == 0


def test_device_groups(L):
    streams = [text(20000 + 997 * k, 30 + k) for k in range(9)] + [b"", b"a" * 5000]
    ref = check(L, streams, alone=False)
    for cap in (1, 2, 4):
        L.b200z_debug_bzip2_encode_group_set(cap)
        try:
            got, _ = batch(L, *packed(streams))
            st = stats(L)
        finally:
            L.b200z_debug_bzip2_encode_group_set(0)
        assert got == ref and st[1] == -(-len(streams) // cap)


def test_launches_do_not_grow_with_streams(L):
    base = text(60000, 40)
    streams = [b"%08d" % k + base for k in range(256)]
    data, offs, lens = packed(streams)
    single(L, streams[0])
    n0 = L.b200z_launch_count()
    one = single(L, streams[0])
    n1 = L.b200z_launch_count()
    got, _ = batch(L, data, offs, lens)
    n2 = L.b200z_launch_count()
    assert stats(L) == (256, 1, 1, 256, 0)
    assert n2 - n1 <= 2 * (n1 - n0), (n2 - n1, n1 - n0)
    assert got[0] == one
    for i in (1, 100, 255):
        assert got[i][2] == orc.bzip2_encode(streams[i])[1]


def test_large_stream_among_small_ones(L):
    big = text(20 << 20, 41)
    r = random.Random(42)
    streams = [text(r.randrange(0, 6000), 500 + k) for k in range(500)]
    streams.insert(250, big)
    got = check(L, streams, alone=False)
    crcs, combined = bs.scan_headers(got[250][2])
    assert len(crcs) > 20 and bs.fold_crcs(crcs) == combined


def _archive(n_bz=300):
    from archive_b200.zip import Archive, ArchiveFile
    arc = Archive()
    t0 = int(time.mktime((2024, 5, 17, 13, 37, 42, 0, 0, -1)))
    r = random.Random(43)
    for i in range(n_bz):
        body = text(r.randrange(0, 20000), 600 + i) if i % 7 else b"a" * r.randrange(0, 600)
        f = ArchiveFile(f"bz/{i:03d}.txt", len(body))
        f.content, f.compression, f.last_mod_time, f.mode = body, "bzip2", t0 + 2 * i, 0o100644
        arc.add(f)
        if i % 50 == 0:
            g = ArchiveFile(f"d/{i}.txt", 5000)
            g.content, g.compression, g.last_mod_time, g.mode = text(5000, 900 + i), ("none" if i % 100 else None), t0, 0o100644
            arc.add(g)
            d = ArchiveFile(f"dir{i}/", 0, is_file=False)
            d.last_mod_time, d.mode = t0, 0o40755
            arc.add(d)
    return arc


def test_zip_encoder_batch(L):
    from archive_b200.zip import ZipDecoder, ZipEncoder, _dos_date, _dos_time
    arc = _archive()
    one = ZipEncoder().encode_bytes(arc, level=6)
    many = ZipEncoder(batch=True).encode_bytes(arc, level=6)
    assert many == one
    members = []
    for f in arc.files:
        lm = time.localtime(f.last_mod_time)
        name = f.name + ("/" if not f.is_file and not f.name.endswith("/") else "")
        members.append((name, f.content or b"", (f.compression or "deflate") if f.is_file else "deflate", f.is_file, f.mode,
                        _dos_time(lm), _dos_date(lm), None))
    st, ref = orc.zip_encode(members, level=6)
    assert st == orc.OK and many == ref
    z = zipfile.ZipFile(io.BytesIO(many))
    back = ZipDecoder().decode_bytes(many)
    for f in arc.files:
        if f.is_file:
            assert z.read(f.name) == f.content
    assert [f.content for f in back.files if f.is_file] == [f.content for f in arc.files if f.is_file]


def test_zip_encoder_batch_with_password(L):
    from archive_b200.zip import ZipDecoder, ZipEncoder
    arc = _archive(60)
    salts = lambda: iter(bytes([k % 251]) * 16 for k in range(10 ** 6))
    s1, s2 = salts(), salts()
    one = ZipEncoder(password="pa55", salt=lambda: next(s1)).encode_bytes(arc, level=6)
    many = ZipEncoder(password="pa55", salt=lambda: next(s2), batch=True).encode_bytes(arc, level=6)
    assert many == one
    back = ZipDecoder().decode_bytes(many, password="pa55")
    assert [f.content for f in back.files if f.is_file] == [f.content for f in arc.files if f.is_file]


def test_bzip2_encode_batch_python(L):
    import archive_b200 as a
    items = [text(3000, 50), b"", b"a" * 1000, bytes(range(256))]
    got = a.bzip2_encode_batch(items)
    assert got == [(orc.bzip2_encode(x)[1], zlib.crc32(x)) for x in items]
    assert a.bzip2_encode_batch([]) == []
    assert bz2.decompress(got[0][0]) == items[0]
