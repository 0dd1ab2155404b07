"""b200z_bzip2_decode_batch and the bzip2 members of b200z_zip_extract: every stream of a batch must come out exactly as
b200z_bzip2_decode gives it alone (rc, out_len, bytes) and as the oracle's BZip2Decoder.decodeStream restatement gives it
(oracle/bzip2_dec.c), whatever its neighbours in the input buffer, in the output and in the device groups are."""
import bz2
import ctypes as C
import glob
import io
import os
import random
import zipfile

import pytest

import oracle_lib as orc
import zip_crypt_build as zb

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
E_NOSPC, E_DATA, E_THROW = -3, -4, -5
TO_ORC = {0: orc.OK, E_DATA: orc.FALSE, E_THROW: orc.THROW}
U_DONE, U_STOP, U_NOSPC, U_THROW = 0, -1, -2, -5


@pytest.fixture(scope="module")
def L():
    from archive_b200 import _ffi
    lib = _ffi.ensure_init()
    lib.b200z_debug_bz2_batch_set.argtypes = [C.c_uint]
    lib.b200z_debug_bz2_batch_stats.argtypes = [C.c_void_p]
    yield lib
    lib.b200z_debug_bz2_batch_set(0)


def stats(L):
    s = (C.c_ulonglong * 3)()
    L.b200z_debug_bz2_batch_stats(s)
    return tuple(s)  # streams, device groups, blocks of the last call


def room_for(z):
    """an output room that holds what the stream decodes to (the oracle's bytes, verify off) and a little more"""
    return len(orc.bzip2_decode(z, verify=False)[1]) + 4096


def single(L, z, room, verify):
    """b200z_bzip2_decode alone -> (rc, out_len, bytes of the slot up to out_len; None on E_NOSPC)"""
    buf = (C.c_uint8 * max(len(z), 1)).from_buffer_copy(z or b"\0")
    out = (C.c_uint8 * max(room, 1))()
    n = C.c_size_t(0)
    rc = L.b200z_bzip2_decode(C.addressof(buf), len(z), int(verify), C.addressof(out), room, C.byref(n))
    return rc, n.value, (None if rc == E_NOSPC else C.string_at(C.addressof(out), n.value))


def batch(L, data, offs, lens, rooms, verify):
    """b200z_bzip2_decode_batch over ranges of `data` -> [(rc, out_len, bytes)] as single() gives them"""
    n = len(offs)
    buf = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data or b"\0")
    out_off, tot = [], 0
    for r in rooms:
        out_off.append(tot)
        tot += r
    out = (C.c_uint8 * max(tot, 1))()
    a64 = lambda v: (C.c_uint64 * max(n, 1))(*v)
    ol, rc = (C.c_uint64 * max(n, 1))(), (C.c_int32 * max(n, 1))()
    r = L.b200z_bzip2_decode_batch(C.addressof(buf), a64(offs), a64(lens), n, int(verify), C.addressof(out), a64(out_off),
                                   a64(rooms), ol, rc)
    assert r == 0, L.b200z_last_error()
    return [(rc[i], ol[i], None if rc[i] == E_NOSPC else C.string_at(C.addressof(out) + out_off[i], ol[i])) for i in range(n)]


def packed(streams):
    """the streams back to back, no gap -> (data, offsets, lengths)"""
    offs, pos = [], 0
    for z in streams:
        offs.append(pos)
        pos += len(z)
    return b"".join(streams), offs, [len(z) for z in streams]


def check(L, streams, verify_modes=(False, True), rooms=None):
    rooms = rooms or [room_for(z) for z in streams]
    data, offs, lens = packed(streams)
    for verify in verify_modes:
        got = batch(L, data, offs, lens, rooms, verify)
        assert stats(L)[0] == len(streams)
        for i, z in enumerate(streams):
            alone = single(L, z, rooms[i], verify)
            assert got[i] == alone, (i, verify, got[i][:2], alone[:2])
            if got[i][0] == E_NOSPC:
                continue
            ost, oout = orc.bzip2_decode(z, verify=verify)
            assert TO_ORC[got[i][0]] == ost, (i, verify, got[i][0], ost)
            assert ost == orc.THROW or got[i][2] == oout, (i, verify)
    return got


def fixtures():
    return sorted(glob.glob(os.path.join(G, "**", "*.bz2"), recursive=True))


def test_fixtures_shuffled_with_duplicates(L):
    names = fixtures()
    assert len(names) >= 10
    zs = [open(p, "rb").read() for p in names]
    rng = random.Random(7)
    streams = zs + [rng.choice(zs) for _ in range(len(zs))]
    rng.shuffle(streams)
    check(L, streams)


def _text(rng, n):
    words = [bytes(rng.choice(b"abcdefghij klmnop") for _ in range(rng.randrange(1, 9))) for _ in range(300)]
    out = bytearray()
    while len(out) < n:
        out += rng.choice(words) + b" "
    return bytes(out[:n])


def test_levels_and_multi_block_streams(L):
    rng = random.Random(11)
    streams = [bz2.compress(_text(rng, rng.randrange(1000, 60000)), lv) for lv in range(1, 10)]
    streams += [bz2.compress(_text(rng, 250000), 1), bz2.compress(_text(rng, 450000), 2),
                bz2.compress(bytes(rng.randrange(256) for _ in range(120000)), 1)]  # 3, 3 and 2 blocks
    streams.insert(4, streams[-3])
    check(L, streams)


def test_edge_streams(L):
    rng = random.Random(5)
    z = bz2.compress(_text(rng, 150000), 1)
    z9 = bz2.compress(_text(rng, 20000), 9)
    eos = z.rfind(b"\x17\x72\x45\x38\x50\x90")
    streams = [b"", b"B", b"BZ", b"BZh", b"BZh9", b"BZh0", b"BZx9" + z[4:], b"BZhA" + z[4:], b"XZh9" + z[4:],
               z + z9, z9 + b"trailing junk" * 3, z9 + b"\0" * 7]
    blk = z.find(b"\x31\x41\x59\x26\x53\x59", 4)
    for cut in sorted({5, 6, 9, 10, 12, 14, 20, blk + 2, blk + 8, len(z) // 2, len(z) - 12, eos if eos > 0 else 30, len(z) - 7,
                       len(z) - 3, len(z) - 1}):
        streams.append(z[:cut])  # inside the header, inside a magic, inside a CRC, mid-block, in the stream's last bytes
    check(L, streams)


def test_damage_seeds(L):
    """the damage kinds and seed of tests/test_zz_bzip2_damaged_gpu.py, all streams of a round in one batch"""
    rng = random.Random(0xB200)
    for r in range(24):
        k = r % 3
        if k == 0:
            src = bytes(rng.randrange(rng.choice([3, 7, 256])) for _ in range(rng.randrange(200, 30000)))
        elif k == 1:
            src = b"".join(bytes([rng.randrange(3)]) * rng.choice([1, 2, 4, 5, 255, 256, 1000]) for _ in range(rng.randrange(1, 400)))
        else:
            src = bytes(rng.randrange(256) for _ in range(rng.randrange(1, 40))) * rng.randrange(1, 2000)
        z = bz2.compress(src, rng.choice([1, 1, 9]))
        streams = [z]
        for _ in range(8):
            bad = bytearray(z)
            kind = rng.randrange(4)
            if kind == 0:
                for _k in range(rng.choice([1, 1, 2, 5])):
                    bad[rng.randrange(4, len(bad))] ^= 1 << rng.randrange(8)
            elif kind == 1:
                p = rng.randrange(4, len(bad))
                bad[p:p + rng.randrange(1, 9)] = bytes(rng.randrange(256) for _ in range(rng.randrange(1, 9)))
            elif kind == 2:
                bad = bad[:rng.randrange(0, len(bad))]
            else:
                if len(bad) > 14:
                    bad[14] |= 0x80
                if rng.random() < 0.5 and len(bad) > 30:
                    bad[rng.randrange(15, len(bad))] ^= 1 << rng.randrange(8)
            streams.append(bytes(bad))
        check(L, streams)


def test_truncated_stream_followed_by_a_valid_one(L):
    """Bytes behind a stream's end are the next stream's here: a read past the end must still be the reference's
    RangeError (or its earlier `false`), exactly as for the stream staged alone."""
    rng = random.Random(3)
    z = bz2.compress(_text(rng, 200000), 1)
    nxt = bz2.compress(_text(rng, 30000), 9)
    streams = []
    for cut in range(8, len(z), max(1, len(z) // 40)):
        streams += [z[:cut], nxt]
    for cut in range(len(z) - 24, len(z)):
        streams += [z[:cut], nxt]
    got = check(L, streams)
    assert {g[0] for g in got[0::2]} & {E_THROW, E_DATA}


def test_overlapping_and_repeated_input_ranges(L):
    rng = random.Random(9)
    a = bz2.compress(_text(rng, 50000), 9)
    b = bz2.compress(_text(rng, 70000), 3)
    data = a + b
    offs = [0, len(a), 0, 2, len(a), 0]
    lens = [len(a), len(b), len(a), len(a), len(b) - 5, len(data)]
    rooms = [200000] * len(offs)
    got = batch(L, data, offs, lens, rooms, True)
    for i in range(len(offs)):
        z = data[offs[i]:offs[i] + lens[i]]
        assert got[i] == single(L, z, rooms[i], True), i


def test_output_rooms(L):
    rng = random.Random(13)
    streams = [bz2.compress(_text(rng, n), 9) for n in (40000, 41000, 42000, 43000, 150000)]
    need = [len(orc.bzip2_decode(z)[1]) for z in streams]
    rooms = [need[0], need[1] - 1, 0, need[3] + 100, need[4]]
    data, offs, lens = packed(streams)
    for verify in (False, True):
        got = batch(L, data, offs, lens, rooms, verify)
        for i, z in enumerate(streams):
            assert got[i] == single(L, z, rooms[i], verify), i
        assert got[1][:2] == (E_NOSPC, need[1]) and got[2][:2] == (E_NOSPC, need[2])
        assert [g[0] for g in got] == [0, E_NOSPC, E_NOSPC, 0, 0]
        assert got[0][2] == orc.bzip2_decode(streams[0])[1] and got[3][2] == orc.bzip2_decode(streams[3])[1]


def test_device_groups(L):
    rng = random.Random(17)
    streams = [bz2.compress(_text(rng, rng.randrange(1000, 90000)), 1) for _ in range(14)]
    streams += [bz2.compress(_text(rng, 250000), 1), bz2.compress(_text(rng, 40000), 1)]
    rooms = [room_for(z) for z in streams]
    data, offs, lens = packed(streams)
    blocks = []
    for z in streams:
        single(L, z, room_for(z), False)
        blocks.append(stats(L)[2])
    assert all(b >= 1 for b in blocks) and blocks[14] >= 3
    for verify in (False, True):
        L.b200z_debug_bz2_batch_set(0)
        want = batch(L, data, offs, lens, rooms, verify)
        assert stats(L) == (len(streams), 1, sum(blocks))
        for cap in (1, 3, 64):
            L.b200z_debug_bz2_batch_set(cap)
            got = batch(L, data, offs, lens, rooms, verify)
            groups, cur = 0, None
            for b in blocks:  # consecutive streams while their blocks fit the cap; a larger stream alone
                if cur is None or cur + b > cap:
                    groups, cur = groups + 1, b
                else:
                    cur += b
            assert got == want and stats(L) == (len(streams), groups, sum(blocks)), (cap, stats(L), groups)
    L.b200z_debug_bz2_batch_set(0)
    assert batch(L, b"", [], [], [], False) == [] and stats(L) == (0, 0, 0)


def test_streams_share_launches(L):
    """512 one-block streams take as many launches as one stream (plus a small constant): they are batched"""
    rng = random.Random(19)
    streams = [bz2.compress(b"%d " % i + _text(rng, 3000), 1) for i in range(512)]
    rooms = [8192] * len(streams)
    L.b200z_debug_bz2_batch_set(0)
    c0 = L.b200z_launch_count()
    one = batch(L, streams[0], [0], [len(streams[0])], rooms[:1], False)
    c1 = L.b200z_launch_count()
    assert stats(L) == (1, 1, 1)
    data, offs, lens = packed(streams)
    got = batch(L, data, offs, lens, rooms, False)
    c2 = L.b200z_launch_count()
    assert stats(L) == (512, 1, 512)
    assert (c2 - c1) <= (c1 - c0) + 8, (c1 - c0, c2 - c1)
    assert got[0] == one[0] and all(g[0] == 0 for g in got)
    assert got[77][2] == bz2.decompress(streams[77])


def test_python_batch(L):
    import archive_b200 as a
    rng = random.Random(23)
    streams = [bz2.compress(_text(rng, rng.randrange(0, 30000)), rng.randrange(1, 10)) for _ in range(20)]
    streams += [bytes(300000), b"BZh9", b"BZh", b"nope"]
    streams[-4] = bz2.compress(bytes(300000), 9)  # decodes to far more than BZip2Decoder's first room: grown and retried
    for verify in (False, True):
        got = a.bzip2_decode_batch(streams, verify=verify)
        for z, (rc, out) in zip(streams, got):
            ost, oout = orc.bzip2_decode(z, verify=verify)
            assert TO_ORC[rc] == ost and (ost == orc.THROW or out == oout)
    assert a.bzip2_decode_batch([]) == []


# ---- ZIP archives: every bzip2 member in one batch ----
def device_members(L, data, rooms=None, password=None):
    """-> [(status, out_len, bytes)] of every listed member from ONE b200z_zip_extract_password call"""
    from archive_b200 import _ffi
    st, ents = orc.zip_list(data)
    assert st == orc.OK
    n = len(ents)
    arr = (_ffi.ZipEntry * n)()
    C.memmove(arr, (orc.ZipEntry * n)(*ents), C.sizeof(arr))
    rooms = rooms or [max(int(e.uncomp_size), 1) for e in ents]
    off, tot = [], 0
    for r in rooms:
        off.append(tot)
        tot += (r + 63) & ~63
    out = (C.c_uint8 * max(tot, 1))()
    ol, sts = (C.c_uint64 * n)(), (C.c_int32 * n)()
    buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
    rc = L.b200z_zip_extract_password(C.addressof(buf), len(data), arr, n, C.addressof(out), max(tot, 1), (C.c_uint64 * n)(*off),
                                      (C.c_uint64 * n)(*rooms), ol, sts, 0, password, len(password or b""))
    assert rc == 0, L.b200z_last_error()
    return ents, [(sts[i], ol[i], C.string_at(C.addressof(out) + off[i], min(ol[i], rooms[i]))) for i in range(n)]


def assert_bzip2_members_like_oracle(L, data, password=None, rooms=None):
    ents, dev = device_members(L, data, rooms, password)
    want = zb.oracle_members(data, password) if password else [orc.zip_member(data, e) for e in ents]
    for i, (e, (ds, dl, db), (os_, ob)) in enumerate(zip(ents, dev, want)):
        if rooms and dl > rooms[i]:
            assert ds == U_NOSPC and dl == len(ob), (i, ds, dl, len(ob))
            continue
        assert db == ob, (i, ds, os_, len(db), len(ob))
        if e.method == 12:
            assert ds == {orc.OK: U_DONE, orc.FALSE: U_STOP, orc.THROW: U_THROW}[os_] and dl == len(ob), (i, ds, os_)
    return dev


def _zip_mixed(n_members, seed):
    rng = random.Random(seed)
    bio = io.BytesIO()
    with zipfile.ZipFile(bio, "w") as zf:
        for i in range(n_members):
            size = rng.choice([0, 1, 100, 3000, 20000, 70000, rng.randrange(150000, 400000)])
            body = _text(rng, size) if rng.random() < 0.8 else bytes(rng.randrange(256) for _ in range(size // 4))
            ct = rng.choice([zipfile.ZIP_BZIP2] * 6 + [zipfile.ZIP_STORED, zipfile.ZIP_DEFLATED])
            zf.writestr(zipfile.ZipInfo("m%03d.txt" % i), body, compress_type=ct)
    return bio.getvalue()


def test_zip_archive_with_many_bzip2_members(L):
    data = _zip_mixed(300, 29)
    dev = assert_bzip2_members_like_oracle(L, data)
    ents = orc.zip_list(data)[1]
    n_bz = sum(1 for e in ents if e.method == 12 and e.has_data)
    assert n_bz > 150 and stats(L)[0] == n_bz  # one batch for all of them
    import archive_b200 as a
    arc = a.ZipDecoder().decode_bytes(data)
    zf = zipfile.ZipFile(io.BytesIO(data))
    for f in arc:
        assert f.content == zf.read(f.name), f.name


def test_zip_bzip2_fixtures(L):
    for p in (os.path.join(G, "zip_bzip2.zip"), os.path.join(G, "zip", "zip_bzip2.zip")):
        data = open(p, "rb").read()
        assert_bzip2_members_like_oracle(L, data)
        assert stats(L)[0] == sum(1 for e in orc.zip_list(data)[1] if e.method == 12 and e.has_data)


def test_encrypted_bzip2_members(L):
    rng = random.Random(31)
    txt = [_text(rng, n) for n in (0, 5000, 60000, 200000)]
    members = [zb.Member("p%d.txt" % i, t, 12, None) for i, t in enumerate(txt)]
    members += [zb.Member("z%d.txt" % i, t, 12, "zipcrypto") for i, t in enumerate(txt)]
    members += [zb.Member("a%d.txt" % i, t, 12, "aes", 1 + i % 3) for i, t in enumerate(txt)]
    members += [zb.Member("d.txt", txt[2], 8, "aes"), zb.Member("s.txt", txt[1], 0, "zipcrypto"),
                zb.Member("cut.txt", txt[3], 12, "zipcrypto", truncate=3000)]
    data = zb.build(members, b"pa55")
    dev = assert_bzip2_members_like_oracle(L, data, password=b"pa55")
    assert stats(L)[0] == sum(1 for m in members if m.method == 12)


def test_zip_member_room_one_byte_short(L):
    data = _zip_mixed(40, 37)
    ents = orc.zip_list(data)[1]
    rooms = [max(int(e.uncomp_size), 1) for e in ents]
    short = [i for i, e in enumerate(ents) if e.method == 12 and e.uncomp_size > 1000][:2]
    for i in short:
        rooms[i] = int(ents[i].uncomp_size) - 1
    dev = assert_bzip2_members_like_oracle(L, data, rooms=rooms)
    for i in short:
        assert dev[i][0] == U_NOSPC and dev[i][1] == ents[i].uncomp_size
