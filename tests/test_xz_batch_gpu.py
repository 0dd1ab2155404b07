"""b200z_xz_decode_batch / b200z_xz_encode_batch: every stream of a batch must come out exactly as b200z_xz_decode /
b200z_xz_encode give it alone (rc, out_len, bytes) and as the oracle's restatement of the reference gives it (oracle/xz.c),
whatever its neighbours in the input buffer, in the output and in the device groups are."""
import ctypes as C
import glob
import hashlib
import lzma
import os
import random

import pytest

import oracle_lib as orc
import xz_build as xb

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "xz")
E_ARG, E_NOSPC, E_DATA, E_THROW = -2, -3, -4, -5
RC = {orc.OK: 0, orc.FALSE: E_DATA, orc.THROW: E_THROW}
TEXT = b"".join(b"line %d: the quick brown fox jumps over the lazy dog %d\n" % (i, i * i % 977) for i in range(1500))


@pytest.fixture(scope="module")
def L():
    from archive_b200 import _ffi
    lib = _ffi.ensure_init()
    lib.b200z_debug_xz_batch_set.argtypes = [C.c_uint]
    lib.b200z_debug_xz_batch_stats.argtypes = [C.c_void_p]
    yield lib
    lib.b200z_debug_xz_batch_set(0)


def stats(L):
    s = (C.c_ulonglong * 3)()
    L.b200z_debug_xz_batch_stats(s)
    return tuple(s)  # streams, device groups, runs of the last decode call


def bound(L, z):
    buf = (C.c_uint8 * max(len(z), 1)).from_buffer_copy(z or b"\0")
    return L.b200z_xz_bound(C.addressof(buf), len(z))


def single(L, z, cap, verify):
    """b200z_xz_decode alone -> (rc, out_len, bytes of the slot up to out_len; None on E_NOSPC)"""
    buf = (C.c_uint8 * max(len(z), 1)).from_buffer_copy(z or b"\0")
    out = (C.c_uint8 * max(cap, 1))()
    n = C.c_size_t(0)
    rc = L.b200z_xz_decode(C.addressof(buf), len(z), int(verify), C.addressof(out), cap, C.byref(n))
    return rc, n.value, (None if rc == E_NOSPC else C.string_at(C.addressof(out), n.value))


def a64(v):
    return (C.c_uint64 * max(len(v), 1))(*v)


def slots(caps):
    offs, tot = [], 0
    for c in caps:
        offs.append(tot)
        tot += c
    return offs, tot


def batch(L, data, offs, lens, caps, verify):
    """b200z_xz_decode_batch over ranges of `data` -> [(rc, out_len, bytes)] as single() gives them"""
    n = len(offs)
    buf = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data or b"\0")
    out_off, tot = slots(caps)
    out = (C.c_uint8 * max(tot, 1))()
    ol, rc = (C.c_uint64 * max(n, 1))(), (C.c_int32 * max(n, 1))()
    r = L.b200z_xz_decode_batch(C.addressof(buf), a64(offs), a64(lens), n, int(verify), C.addressof(out), a64(out_off),
                                a64(caps), ol, rc)
    assert r == 0, L.b200z_last_error()
    return [(rc[i], ol[i], None if rc[i] == E_NOSPC else C.string_at(C.addressof(out) + out_off[i], ol[i])) for i in range(n)]


def packed(streams):
    """the streams back to back, no gap -> (data, offsets, lengths)"""
    offs, pos = [], 0
    for z in streams:
        offs.append(pos)
        pos += len(z)
    return b"".join(streams), offs, [len(z) for z in streams]


def check(L, streams, verify_modes=(False, True), caps=None, ranges=None):
    """every stream against b200z_xz_decode alone and against the oracle; `ranges` = (data, offs, lens) reads the
    streams from other places of one buffer (streams[i] must be data[offs[i]:offs[i] + lens[i]])"""
    caps = caps or [bound(L, z) for z in streams]
    data, offs, lens = ranges or packed(streams)
    seen = set()
    for verify in verify_modes:
        got = batch(L, data, offs, lens, caps, verify)
        check.stats = stats(L)
        assert check.stats[0] == len(streams)
        for i, z in enumerate(streams):
            alone = single(L, z, caps[i], verify)
            assert got[i] == alone, (i, verify, got[i][:2], alone[:2])
            if got[i][0] == E_NOSPC:
                continue
            st, want = xb.decode(z, verify)
            seen.add(st)
            assert got[i][0] == RC[st], (i, verify, got[i][0], st)
            assert st == orc.THROW or got[i][2] == want, (i, verify)
    return seen


def _trim_corpus(seed=23, words=3000, count=40000):
    r = random.Random(seed)
    ws = [bytes(r.randbytes(r.randrange(2, 9))) for _ in range(words)]
    return b" ".join(r.choice(ws) for _ in range(count))


def _global_model_stream(n):
    raw = bytearray(xb.raw_lzma2(TEXT[:n], lc=4, lp=0, pb=2))
    raw[5] = 2 * 45 + 0 * 9 + 8  # lc = 8: lc + lp > 4, the model lives in a global slot
    return xb.container([(bytes(raw), TEXT[:n])])


def test_fixtures_shuffled_with_duplicates_and_shared_ranges(L):
    zs = [open(p, "rb").read() for p in sorted(glob.glob(os.path.join(GOLD, "*.xz")))]
    assert len(zs) >= 9
    rng = random.Random(7)
    streams = zs + [rng.choice(zs) for _ in range(len(zs))]
    rng.shuffle(streams)
    assert check(L, streams) == {orc.OK}
    # repeated and overlapping ranges of one buffer: a range read twice, and ranges that run on into the next stream
    # (the bytes behind a stream's footer are ignored)
    data, offs, lens = packed(streams)
    offs2, lens2, views = [], [], []
    for i in range(len(streams)):
        for o, n in ((offs[i], lens[i]), (offs[i], lens[i]), (offs[i], len(data) - offs[i])):
            offs2.append(o)
            lens2.append(n)
            views.append(data[o:o + n])
    check(L, views, ranges=(data, offs2, lens2))


def test_mixed_streams_in_one_batch(L):
    rng = random.Random(3)
    streams = []
    for preset in (0, 1, 6, 9):
        for ck in (lzma.CHECK_NONE, lzma.CHECK_CRC32, lzma.CHECK_CRC64, lzma.CHECK_SHA256):
            streams.append(lzma.compress(TEXT[:rng.randrange(1, len(TEXT))], preset=preset, check=ck))
    for lc, lp, pb in ((0, 0, 0), (4, 0, 2), (0, 4, 1), (1, 3, 3), (2, 2, 0)):
        streams.append(xb.container([(xb.raw_lzma2(TEXT, lc=lc, lp=lp, pb=pb), TEXT)], check="crc32"))
    streams += [_global_model_stream(8000), _global_model_stream(20000), _global_model_stream(3000)]  # several global slots
    for check_kind in ("crc32", "crc64", "sha256", "none"):
        streams.append(xb.xz_blocks((TEXT * 3)[:200000], 200, check=check_kind))  # 1000 blocks
        streams.append(xb.xz_blocks(TEXT[:30000], 30000, check=check_kind))  # 1 block
    rand = random.Random(5).randbytes(150000)
    streams.append(xb.container([(xb.raw_lzma2(rand), rand)], check="crc64"))  # stored chunks
    streams.append(xb.container([(xb.join([(2, b"\x02\x00\x04", b"hello")] + xb.chunks(xb.raw_lzma2(TEXT))),
                                  b"hello" + TEXT)]))
    plain = _trim_corpus()
    for lc, lp, pb in ((3, 0, 2), (0, 2, 0), (3, 1, 3)):
        raw = xb.raw_lzma2(plain, preset=1, lc=lc, lp=lp, pb=pb, dict_size=4096)
        streams.append(xb.container([(raw, plain)], dict_byte=0))
        streams.append(xb.container([(xb.raw_lzma2(plain, preset=1, lc=lc, lp=lp, pb=pb), plain)], dict_byte=0))
    chs = xb.chunks(xb.raw_lzma2(plain, preset=1, dict_size=4096))
    for k in (2, 3):
        c, h, d = chs[k]
        for props in (2 * 45 + 1 * 9 + 3, 0 * 45 + 0 * 9 + 3, 4 * 45 + 3):
            hh = bytes([(c & 0x1F) | 0xC0]) + h[1:5] + bytes([props])
            streams.append(xb.container([(xb.join(chs[:k] + [(0xC0, hh, d)] + chs[k + 1:]), plain)], dict_byte=0))
    rng.shuffle(streams)
    seen = check(L, streams)
    assert orc.OK in seen and orc.THROW in seen
    assert check.stats[1] == 1 and check.stats[2] > 4000  # the runs of every stream in one group


def _damaged(good):
    out = [good[:k] for k in range(0, len(good), max(1, len(good) // 25))]
    out += [xb.flip_bits(good, seed, 1 + seed % 3) for seed in range(30)]
    for pos in (8, 12 + 8, len(good) - 12 - 2, len(good) - 10):
        b = bytearray(good)
        b[pos] ^= 0x40
        out.append(bytes(b))
    out.append(xb.container([(xb.raw_lzma2(TEXT, pb=4), TEXT)]))
    for ck in ("crc32", "crc64"):
        out.append(xb.container([(xb.raw_lzma2(TEXT), TEXT)], check=ck, bad_check=True))
    chs = xb.chunks(xb.raw_lzma2(TEXT))
    c, h, d = chs[0]
    ulen = ((c & 0x1F) << 16 | h[1] << 8 | h[2]) + 1
    for k in (1, 3, 7, 20):  # declared sizes that end inside a match
        u = ulen - k - 1
        hh = bytes([(c & 0xE0) | (u >> 16), (u >> 8) & 0xFF, u & 0xFF]) + h[3:]
        out.append(xb.container([(xb.join([(c, hh, d)]), TEXT[:-k])]))
    return out


def test_damaged_streams_between_good_ones(L):
    good = xb.xz_blocks(TEXT * 2, 30000, check="crc64")
    goods = [lzma.compress(TEXT[:n], check=lzma.CHECK_CRC32) for n in (100, 5000, 40000)] + [good]
    streams = []
    for k, z in enumerate(_damaged(good)):
        streams += [goods[k % len(goods)], z]
    streams.append(goods[0])
    seen = check(L, streams)
    assert {orc.OK, orc.FALSE, orc.THROW} <= seen


def test_size_edges(L):
    z1, z2 = lzma.compress(TEXT), lzma.compress(TEXT[:999])
    empty = lzma.compress(b"")
    streams = [b"", z1, empty, b"", z2, open(os.path.join(GOLD, "empty.xz"), "rb").read(), z1]
    check(L, streams)
    # one room one byte short: E_NOSPC with the bound for that stream only; room 0 for a stream that needs some
    caps = [bound(L, z) for z in streams]
    caps[1] -= 1
    caps[4] = 0
    data, offs, lens = packed(streams)
    got = batch(L, data, offs, lens, caps, True)
    assert got[1] == (E_NOSPC, len(TEXT), None) and got[4] == (E_NOSPC, 999, None)
    assert got[6] == (0, len(TEXT), TEXT)
    for i in (0, 2, 3, 5):
        assert got[i] == single(L, streams[i], caps[i], True)
    check(L, streams, caps=caps)
    # n == 0
    assert L.b200z_xz_decode_batch(None, None, None, 0, 1, None, None, None, None, None) == 0


def test_argument_errors_write_nothing(L):
    z = lzma.compress(TEXT)
    buf = (C.c_uint8 * len(z)).from_buffer_copy(z)
    cap = bound(L, z)
    out = (C.c_uint8 * (2 * cap))(*([0xAB] * (2 * cap)))
    ol, rc = (C.c_uint64 * 2)(7, 7), (C.c_int32 * 2)(9, 9)

    def call(offs, lens, oo, cc, **kw):
        a = dict(in_off=a64(offs), in_len=a64(lens), out_off=a64(oo), caps=a64(cc), ol=ol, rc=rc)
        a.update(kw)
        return L.b200z_xz_decode_batch(C.addressof(buf), a["in_off"], a["in_len"], 2, 1, C.addressof(out), a["out_off"],
                                       a["caps"], a["ol"], a["rc"])

    for k in ("in_off", "in_len", "out_off", "caps", "ol", "rc"):
        assert call([0, 0], [len(z)] * 2, [0, cap], [cap, cap], **{k: None}) == E_ARG
    assert call([0, 2 ** 64 - 4], [len(z), 8], [0, cap], [cap, cap]) == E_ARG  # input range wraps
    assert call([0, 0], [len(z)] * 2, [0, 2 ** 64 - 4], [cap, 8]) == E_ARG  # output range wraps
    assert call([0, 0], [len(z)] * 2, [0, cap - 1], [cap, cap]) == E_ARG  # output slots overlap
    assert bytes(out) == b"\xab" * (2 * cap) and list(ol) == [7, 7] and list(rc) == [9, 9]
    assert call([0, 0], [len(z)] * 2, [0, cap], [cap, cap]) == 0
    assert list(rc) == [0, 0] and bytes(out) == TEXT + b"\xab" * (cap - len(TEXT)) + TEXT + b"\xab" * (cap - len(TEXT))


def test_forced_device_groups(L):
    rng = random.Random(9)
    streams = [xb.xz_blocks(TEXT[:rng.randrange(1, 20000)], rng.choice([500, 4000, 20000]),
                            check=rng.choice(["crc32", "crc64", "none"])) for _ in range(9)]
    streams.insert(4, _global_model_stream(5000))
    streams.insert(7, xb.container([(xb.raw_lzma2(TEXT, pb=4), TEXT)]))
    data, offs, lens = packed(streams)
    caps = [bound(L, z) for z in streams]
    L.b200z_debug_xz_batch_set(0)
    want = batch(L, data, offs, lens, caps, True)
    assert stats(L)[:2] == (len(streams), 1)
    try:
        for g in (1, 2, 3):
            L.b200z_debug_xz_batch_set(g)
            assert batch(L, data, offs, lens, caps, True) == want
            assert stats(L)[:2] == (len(streams), -(-len(streams) // g))
    finally:
        L.b200z_debug_xz_batch_set(0)
    for i, z in enumerate(streams):
        assert want[i] == single(L, z, caps[i], True)


def test_launch_count_does_not_grow_with_streams(L):
    counts = []
    for n in (64, 128):
        streams = [lzma.compress(TEXT[:1000 + 37 * i], check=lzma.CHECK_CRC32) for i in range(n)]
        data, offs, lens = packed(streams)
        caps = [bound(L, z) for z in streams]
        before = L.b200z_launch_count()
        got = batch(L, data, offs, lens, caps, True)
        counts.append(L.b200z_launch_count() - before)
        assert stats(L) == (n, 1, n)
        assert all(g == (0, 1000 + 37 * i, TEXT[:1000 + 37 * i]) for i, g in enumerate(got))
    assert counts[0] <= 4 and counts[1] == counts[0], counts


def test_python_decode_batch():
    import archive_b200 as a
    zs = [lzma.compress(TEXT[:n]) for n in (0, 10, 30000)] + [xb.container([(xb.raw_lzma2(TEXT, pb=4), TEXT)]), b"junk"]
    got = a.xz_decode_batch(zs, verify=True)
    assert got[:3] == [(0, b""), (0, TEXT[:10]), (0, TEXT[:30000])]
    assert got[3][0] == E_THROW and got[4] == (E_DATA, b"")
    assert a.xz_decode_batch([]) == []


# ---- encode ----
SIZES = [0, 6, 65536, 65537, 300000]


def single_enc(L, data, check, cap=None):
    buf = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data or b"\0")
    cap = L.b200z_xz_encode_bound(len(data)) if cap is None else cap
    out = (C.c_uint8 * max(cap, 1))()
    n = C.c_size_t(0)
    rc = L.b200z_xz_encode(C.addressof(buf), len(data), check, C.addressof(out), cap, C.byref(n))
    return rc, n.value, (C.string_at(C.addressof(out), n.value) if rc == 0 else None)


def batch_enc(L, data, offs, lens, caps, check):
    n = len(offs)
    buf = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data or b"\0")
    out_off, tot = slots(caps)
    out = (C.c_uint8 * max(tot, 1))()
    ol, rc = (C.c_uint64 * max(n, 1))(), (C.c_int32 * max(n, 1))()
    r = L.b200z_xz_encode_batch(C.addressof(buf), a64(offs), a64(lens), n, check, C.addressof(out), a64(out_off), a64(caps),
                                ol, rc)
    assert r == 0, L.b200z_last_error()
    return [(rc[i], ol[i], C.string_at(C.addressof(out) + out_off[i], ol[i]) if rc[i] == 0 else None) for i in range(n)]


def _inputs(seed):
    rng = random.Random(seed)
    ins = [rng.randbytes(n) for n in SIZES] + [TEXT[:n] for n in SIZES]
    rng.shuffle(ins)
    return ins


@pytest.mark.parametrize("check", [0, 1, 2, 3])
def test_encode_mixed_sizes(L, check):
    ins = _inputs(check)
    data, offs, lens = packed(ins)
    caps = [L.b200z_xz_encode_bound(len(d)) for d in ins]
    got = batch_enc(L, data, offs, lens, caps, check)
    for i, d in enumerate(ins):
        assert got[i] == single_enc(L, d, check)
        assert got[i][2] == xb.encode(d, check)
    # repeated ranges: every input twice, the second time from the same bytes
    got2 = batch_enc(L, data, offs + offs, lens + lens, caps + caps, check)
    assert got2 == got + got


def test_sha256_digests(L):
    ins = _inputs(11) + [os.urandom(n) for n in (1, 55, 56, 63, 64, 119, 120, 128, 1000)]
    data, offs, lens = packed(ins)
    got = batch_enc(L, data, offs, lens, [L.b200z_xz_encode_bound(len(d)) for d in ins], 3)
    for d, (rc, n, z) in zip(ins, got):
        assert rc == 0
        if not d:
            continue
        after = 27 + len(d) + 1  # stream header 12, block header 12, chunk header 3, the bytes, the end marker
        dig = z[after + (-after % 4):][:32]
        assert dig == hashlib.sha256(d).digest() == xb.sha256(d)


def test_encode_short_room_and_arguments(L):
    ins = _inputs(4)
    data, offs, lens = packed(ins)
    caps = [L.b200z_xz_encode_bound(len(d)) for d in ins]
    need = [len(xb.encode(d, 2)) for d in ins]
    caps[2], caps[5] = need[2] - 1, 0
    got = batch_enc(L, data, offs, lens, caps, 2)
    for i, d in enumerate(ins):
        if i in (2, 5):
            assert got[i] == (E_NOSPC, need[i], None) == single_enc(L, d, 2, caps[i])
        else:
            assert got[i] == (0, need[i], xb.encode(d, 2))
    buf = (C.c_uint8 * 1)()
    out = (C.c_uint8 * 64)(*([0xAB] * 64))
    ol, rc = (C.c_uint64 * 1)(), (C.c_int32 * 1)()
    assert L.b200z_xz_encode_batch(C.addressof(buf), a64([0]), a64([0]), 1, 4, C.addressof(out), a64([0]), a64([64]), ol,
                                   rc) == E_ARG
    assert L.b200z_xz_encode_batch(C.addressof(buf), a64([0]), None, 1, 2, C.addressof(out), a64([0]), a64([64]), ol, rc) == E_ARG
    assert bytes(out) == b"\xab" * 64
    assert L.b200z_xz_encode_batch(None, None, None, 0, 2, None, None, None, None, None) == 0


def test_round_trip_through_the_batches():
    """The reference's own decoder does not take back every stream its encoder writes (the encoder's index records a
    block size the decoder does not find for many lengths): each stream must decode as the oracle decodes it, and those
    the oracle takes back must give the input."""
    import archive_b200 as a
    rng = random.Random(8)
    ins = [TEXT[:n] for n in (0, 1, 2, 3, 4, 5, 700, 4096, 65536)] + [rng.randbytes(n) for n in (3, 6, 40000, 65535)]
    ok = 0
    for check in (a.XZCheck.none, a.XZCheck.crc32, a.XZCheck.crc64, a.XZCheck.sha256):
        enc = a.xz_encode_batch(ins, check=check)
        assert enc == [a.XZEncoder().encode_bytes(d, check=check) for d in ins]
        got = a.xz_decode_batch(enc, verify=True)
        for d, z, (rc, out) in zip(ins, enc, got):
            st, want = xb.decode(z, True)
            assert rc == RC[st] and (st == orc.THROW or out == want)
            if st == orc.OK:
                assert out == d
                ok += 1
    assert ok >= 8
