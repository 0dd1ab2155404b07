"""b200z_gzip_decode_batch / b200z_zlib_decode_batch / b200z_gzip_encode_batch / b200z_zlib_encode_batch: every stream of a
batch must come out exactly as the single call gives it alone (rc, out_len, bytes) and as the oracle's restatement of the
reference gives it, whatever its neighbours in the input buffer, in the output, in the rounds and in the device groups are."""
import ctypes as C
import glob
import gzip as pygzip
import os
import random
import struct
import zlib

import pytest

import oracle_lib as orc

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
E_ARG, E_NOSPC, E_DATA, E_THROW = -2, -3, -4, -5
RC = {orc.OK: 0, orc.FALSE: E_DATA, orc.THROW: E_THROW}
VERIFY, RAW = 1, 2  # B200Z_GZIP_VERIFY, B200Z_GZIP_RAW


@pytest.fixture(scope="module")
def L():
    from archive_b200 import _ffi
    lib = _ffi.ensure_init()
    lib.b200z_debug_gzip_batch_set.argtypes = [C.c_uint]
    lib.b200z_debug_gzip_batch_stats.argtypes = [C.c_void_p]
    yield lib
    lib.b200z_debug_gzip_batch_set(0)


def stats(L):
    s = (C.c_ulonglong * 6)()
    L.b200z_debug_gzip_batch_stats(s)
    return dict(zip(("streams", "groups", "rounds", "units", "k12_offered", "k12_accepted"), s))


def text(n, stream=7):
    from archive_b200 import synth
    return synth.text(n, stream=stream).tobytes()


def a64(v):
    return (C.c_uint64 * max(len(v), 1))(*v)


def buf(b):
    return (C.c_uint8 * max(len(b), 1)).from_buffer_copy(b or b"\0")


def single(L, gz, z, cap, verify, raw=False):
    """the single call alone -> (rc, out_len, bytes of the slot up to out_len; None on E_NOSPC)"""
    src = buf(z)
    out = (C.c_uint8 * max(cap, 1))()
    n = C.c_size_t(0)
    if gz:
        rc = L.b200z_gzip_decode(C.addressof(src), len(z), verify, C.addressof(out), cap, C.byref(n))
    else:
        rc = L.b200z_zlib_decode(C.addressof(src), len(z), verify, int(raw), C.addressof(out), cap, C.byref(n))
    return rc, n.value, (None if rc == E_NOSPC else C.string_at(C.addressof(out), min(n.value, cap)))


def batch(L, gz, data, offs, lens, caps, verify, raw=False):
    """one decode batch over ranges of `data` -> [(rc, out_len, bytes)] as single() gives them"""
    n = len(offs)
    src = buf(data)
    out_off, tot = [], 0
    for c in caps:
        out_off.append(tot)
        tot += c
    out = (C.c_uint8 * max(tot, 1))()
    ol, rc = (C.c_uint64 * max(n, 1))(), (C.c_int32 * max(n, 1))()
    if gz:
        r = L.b200z_gzip_decode_batch(C.addressof(src), a64(offs), a64(lens), n, verify, C.addressof(out), a64(out_off), a64(caps), ol, rc)
    else:
        r = L.b200z_zlib_decode_batch(C.addressof(src), a64(offs), a64(lens), n, verify, int(raw), C.addressof(out), a64(out_off),
                                      a64(caps), ol, rc)
    assert r == 0, L.b200z_last_error()
    return [(rc[i], ol[i], None if rc[i] == E_NOSPC else C.string_at(C.addressof(out) + out_off[i], min(ol[i], caps[i])))
            for i in range(n)]


def packed(streams):
    offs, pos = [], 0
    for s in streams:
        offs.append(pos)
        pos += len(s)
    return b"".join(streams), offs, [len(s) for s in streams]


def room(z):
    return 4 * len(z) + 1024


def check(L, gz, streams, verify=0, raw=False, caps=None, oracle=True, data=None, offs=None, lens=None):
    if data is None:
        data, offs, lens = packed(streams)
    caps = caps or [room(data[o:o + n]) for o, n in zip(offs, lens)]
    got = batch(L, gz, data, offs, lens, caps, verify, raw)
    for i, (o, n) in enumerate(zip(offs, lens)):
        z = data[o:o + n]
        want = single(L, gz, z, caps[i], verify, raw)
        assert got[i] == want, (i, got[i][:2], want[:2])
        if oracle and want[0] != E_NOSPC:
            if gz:
                st, ob = orc.gzip_decode(z, verify=bool(verify & VERIFY), raw=bool(verify & RAW))
            else:
                st, ob = orc.zlib_decode(z, verify=bool(verify), raw=raw)
            assert RC[st] == want[0], (i, st, want[0])
            if want[0] == 0:
                assert ob == want[2], i
    return got


def member(chunk, level=6, zdict=None, hint=False, strategy=zlib.Z_DEFAULT_STRATEGY, isize=None):
    co = (zlib.compressobj(level, zlib.DEFLATED, -15, 9, strategy, zdict) if zdict
          else zlib.compressobj(level, zlib.DEFLATED, -15, 9, strategy))
    body = co.compress(chunk) + co.flush()
    trailer = struct.pack("<II", zlib.crc32(chunk), len(chunk) if isize is None else isize)
    if hint:
        total = 10 + 2 + 6 + len(body) + 8
        return (b"\x1f\x8b\x08\x04" + bytes(4) + b"\x00\xff" + struct.pack("<H", 6) + b"BC" + struct.pack("<HH", 2, total - 1)
                + body + trailer)
    return b"\x1f\x8b\x08\x00" + bytes(4) + b"\x00\xff" + body + trailer


def chained(data, cuts, hint=False):
    """members whose matches reach into the output of the members before them (preset dictionary = that output)"""
    ms, done = [], b""
    for lo, hi in cuts:
        ms.append(member(data[lo:hi], zdict=done[-32768:] or None, hint=hint))
        done += data[lo:hi]
    return b"".join(ms)


def golden():
    return [open(p, "rb").read() for p in sorted(glob.glob(os.path.join(GOLD, "*.gz")))]


# ---------------------------------------------------------------- decode


def test_golden_shuffled_duplicates_and_overlapping_ranges(L):
    g = golden()
    assert g
    rnd = random.Random(1)
    streams = g * 3
    rnd.shuffle(streams)
    check(L, True, streams)
    # repeated and overlapping ranges of one buffer: the same file twice, and ranges that run into the next file
    data, offs, lens = packed(g)
    o2 = offs + offs + [offs[0] + 3] + offs[:-1]
    l2 = lens + lens + [lens[0] - 3] + [lens[i] + min(50, lens[i + 1]) for i in range(len(g) - 1)]
    check(L, True, None, data=data, offs=o2, lens=l2)


def test_single_member_mixed_sizes_levels_and_block_kinds(L):
    t = text(300000)
    streams = []
    for i, n in enumerate([0, 1, 100, 4000, 70000, 200000]):
        for level in range(10):
            st = [zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY][(i + level) % 3]
            streams.append(member(t[i * 1000:i * 1000 + n], level=level, strategy=st))
    streams.append(pygzip.compress(t[:50000], 9, mtime=0))
    streams.append(b"")
    random.Random(2).shuffle(streams)
    got = check(L, True, streams)
    assert all(r[0] == 0 for r in got)
    st = stats(L)
    assert st["streams"] == len(streams) and st["groups"] == 1 and st["rounds"] == 1


def test_bgzf_hinted_runs_with_a_lying_hint(L):
    t = text(200000, stream=3)
    good = b"".join(member(t[i:i + 20000], hint=True) for i in range(0, 100000, 20000))
    lie = (b"".join(member(t[i:i + 20000], hint=True) for i in range(0, 40000, 20000))
           + member(t[40000:60000], hint=True, isize=12345)
           + b"".join(member(t[i:i + 20000], hint=True) for i in range(60000, 100000, 20000)))
    mixed = good + member(t[:30000]) + good  # a hinted run, an unhinted member, a hinted run
    check(L, True, [good, lie, mixed, lie, good])


def test_members_that_reach_into_earlier_members(L):
    t = text(90000, stream=50)
    cuts = [(0, 20000), (15000, 40000), (30000, 60000), (100, 9000), (50000, 90000)]
    reach = chained(t, cuts)
    reach_h = chained(t, cuts, hint=True)
    plain = [member(t[i:i + 7000]) for i in range(0, 70000, 7000)]
    got = check(L, True, plain[:3] + [reach] + plain[3:] + [reach_h, reach])
    assert got[3][0] == 0 and got[3][2] == b"".join(t[lo:hi] for lo, hi in cuts)
    # one round per unhinted member of `reach`; the hinted copy's members reach back, fail their run and are redone one by one
    assert stats(L)["rounds"] >= len(cuts)


def test_gzip_falls_back_to_zlib(L):
    t = text(40000, stream=9)
    z = zlib.compress(t, 6)
    le = z[:-4] + struct.pack("<I", zlib.adler32(t))  # the gzip fall-back reads a little-endian Adler-32
    rawd = zlib.compress(t, 6)[2:-4]
    for verify in (0, VERIFY, RAW, VERIFY | RAW):
        check(L, True, [z, le, rawd, member(t[:5000]), le + le], verify=verify, oracle=verify & RAW == 0)


def test_zlib_multi_stream_verify_adler_and_commit_late(L):
    t = text(120000, stream=11)
    s = [zlib.compress(t[i:i + 15000], 1 + i // 15000) for i in range(0, 120000, 15000)]
    bad_adler = s[0][:-1] + bytes([s[0][-1] ^ 1])
    bad_hdr = s[1] + b"\x78\x00" + s[2]  # a bad FCHECK after a good stream: the good one never reaches the output
    fdict = s[2] + b"\x78\xbb\x00\x00\x00\x01" + s[3]
    method = s[3] + b"\x77\x9c" + s[4]
    streams = [b"".join(s), bad_adler + s[1], s[0] + bad_adler, bad_hdr, fdict, method, s[5], b"", s[6][:1], s[7][:-2]]
    for verify in (0, 1):
        check(L, False, streams, verify=verify)
    check(L, False, [x[2:-4] for x in s] + [s[0][2:-4] + s[1][2:-4]], raw=True)


def test_truncated_and_damaged_streams_packed_before_good_ones(L):
    t = text(60000, stream=13)
    good = member(t[:30000])
    zl = zlib.compress(t[:30000])
    streams = []
    for cut in (1, 5, 11, 200, len(good) - 9, len(good) - 1):
        streams += [good[:cut], good]
    dam = bytearray(good)
    dam[40] ^= 0xff
    streams += [bytes(dam), good, b"", good, b"\x1f", good, good + b"\x1f\x8b", good]
    check(L, True, streams)
    zs = []
    for cut in (1, 2, 9, len(zl) - 3):
        zs += [zl[:cut], zl]
    check(L, False, zs + [b""], verify=1)


def test_short_output_rooms(L):
    t = text(100000, stream=17)
    cuts = [(0, 20000), (10000, 30000), (5000, 40000)]
    streams = [member(t[:40000]), chained(t, cuts), b"".join(member(t[i:i + 10000], hint=True) for i in range(0, 40000, 10000)),
               zlib.compress(t[:40000]), zlib.compress(t[:9000]) * 3]
    for caps in ([0] * 5, [1] * 5, [39999, 40000, 39999, 0, 100], [20000] * 5, [70000, 80000, 30000, 0, 18000]):
        check(L, True, streams[:3], caps=caps[:3], oracle=False)
        check(L, False, streams[3:], caps=caps[3:], oracle=False, verify=1)


def test_argument_errors_write_nothing(L):
    z = member(b"hello" * 100)
    src = buf(z + z)
    out = (C.c_uint8 * 4096)(*([0xa5] * 4096))
    ol, rc = (C.c_uint64 * 2)(7, 7), (C.c_int32 * 2)(9, 9)
    base = C.addressof(src)
    ok = dict(offs=a64([0, len(z)]), lens=a64([len(z)] * 2), oo=a64([0, 2048]), caps=a64([2048, 2048]))
    cases = [
        dict(offs=None),
        dict(lens=None),
        dict(oo=None),
        dict(caps=None),
        dict(offs=a64([0, 2 ** 64 - 4])),
        dict(caps=a64([2048, 2 ** 64 - 1])),
        dict(oo=a64([0, 1000])),  # overlapping slots
    ]
    for c in cases:
        a = dict(ok, **c)
        r = L.b200z_gzip_decode_batch(base, a["offs"], a["lens"], 2, 0, C.addressof(out), a["oo"], a["caps"], ol, rc)
        assert r == E_ARG
        r = L.b200z_zlib_decode_batch(base, a["offs"], a["lens"], 2, 0, 0, C.addressof(out), a["oo"], a["caps"], ol, rc)
        assert r == E_ARG
        r = L.b200z_gzip_encode_batch(base, a["offs"], a["lens"], 2, 6, 0, C.addressof(out), a["oo"], a["caps"], ol, rc)
        assert r == E_ARG
        r = L.b200z_zlib_encode_batch(base, a["offs"], a["lens"], 2, 6, 15, 0, C.addressof(out), a["oo"], a["caps"], ol, rc)
        assert r == E_ARG
        assert bytes(out) == b"\xa5" * 4096 and list(ol) == [7, 7] and list(rc) == [9, 9]
    for level, wb in ((-1, 15), (10, 15), (6, 8), (6, 16)):
        r = L.b200z_zlib_encode_batch(base, ok["offs"], ok["lens"], 2, level, wb, 0, C.addressof(out), ok["oo"], ok["caps"], ol, rc)
        assert r == E_ARG
    for level in (-1, 10):
        r = L.b200z_gzip_encode_batch(base, ok["offs"], ok["lens"], 2, level, 0, C.addressof(out), ok["oo"], ok["caps"], ol, rc)
        assert r == E_ARG
    assert bytes(out) == b"\xa5" * 4096 and list(ol) == [7, 7] and list(rc) == [9, 9]
    for fn in (L.b200z_gzip_decode_batch,):
        assert fn(None, None, None, 0, 0, None, None, None, None, None) == 0
    assert L.b200z_zlib_decode_batch(None, None, None, 0, 0, 0, None, None, None, None, None) == 0
    assert L.b200z_gzip_encode_batch(None, None, None, 0, 6, 0, None, None, None, None, None) == 0
    assert L.b200z_zlib_encode_batch(None, None, None, 0, 6, 15, 0, None, None, None, None, None) == 0


def test_forced_device_groups(L):
    t = text(100000, stream=19)
    streams = [member(t[i * 3000:i * 3000 + 1000 + 700 * i]) for i in range(20)]
    streams[7] = chained(t, [(0, 8000), (4000, 12000)])
    streams[11] = zlib.compress(t[:5000])  # falls back to zlib
    L.b200z_debug_gzip_batch_set(3)
    try:
        check(L, True, streams, verify=VERIFY)
        st = stats(L)
        assert st["groups"] == 7 and st["streams"] == 20
    finally:
        L.b200z_debug_gzip_batch_set(0)


def test_k12_member_beside_small_ones(L):
    L.b200z_debug_inflate_chunked_set(C.c_ulonglong(256 << 10), C.c_ulonglong(0))
    try:
        t = text(2 << 20, stream=23)
        big = member(t, level=6)
        assert len(big) > 256 << 10
        small = [member(t[i:i + 5000]) for i in range(0, 50000, 5000)]
        # a K12-sized member behind a small one in an unhinted stream: it reaches into its predecessor's output (hist > 0)
        later = chained(t, [(0, 40000), (40000, 2 << 20)])
        assert len(later) - len(small[0]) > 256 << 10
        got = check(L, True, small[:5] + [big] + small[5:] + [zlib.compress(t), later], oracle=False)
        assert got[5][2] == t and got[-1][2] == t
        st = stats(L)
        # the member, the zlib stream the gzip call falls back to (as alone), and the later member
        assert st["k12_offered"] == 3 and st["k12_accepted"] == 3, st
        check(L, False, [zlib.compress(t)] + [zlib.compress(s) for s in (t[:1000], t[:3000])], verify=1, oracle=False)
        st = stats(L)
        assert st["k12_offered"] == 1 and st["k12_accepted"] == 1, st
    finally:
        L.b200z_debug_inflate_chunked_set(C.c_ulonglong(0), C.c_ulonglong(0))


def test_finished_streams_offer_nothing_in_later_rounds(L):
    """A stream that fails in one round has no unit in any later one, while its neighbours go on for more rounds: the
    large units K12 sees are exactly those of the streams still running."""
    t = text(400000, stream=41)
    small = zlib.compress(t[:3000])
    large = zlib.compress(t[:400000], 9)
    assert len(large) > 100000
    good = small + large  # two rounds, the second one K12-sized
    bad = zlib.compress(t[:2000])[:-2]  # truncated Adler-32: ends in round 1
    L.b200z_debug_inflate_chunked_set(C.c_ulonglong(4096), C.c_ulonglong(0))
    try:
        got = check(L, False, [good, bad, good] + [bad] * 20 + [good], verify=1, oracle=False)
        assert [g[0] for g in got] == [0, E_THROW, 0] + [E_THROW] * 20 + [0]
        st = stats(L)
        # each good stream offers its first zlib stream (its view runs to the end of its input, as alone) and its second
        assert st["rounds"] == 2 and st["k12_offered"] == 6 and st["k12_accepted"] == 6, st
        gz = member(t[:3000]) + member(t[:400000], level=9)
        bad_gz = member(t[:2000])[:-3]  # truncated trailer: ends in round 1
        got = check(L, True, [gz, bad_gz] * 6, oracle=False)
        assert [g[0] for g in got] == [0, E_THROW] * 6
        st = stats(L)
        # the small member is followed by a member header within the threshold: only the large ones are offered
        assert st["rounds"] == 2 and st["k12_offered"] == 6 and st["k12_accepted"] == 6, st
    finally:
        L.b200z_debug_inflate_chunked_set(C.c_ulonglong(0), C.c_ulonglong(0))
    # many rounds beside streams that fail in the first one (the multi-stream input takes 8 rounds)
    s = [zlib.compress(t[i:i + 15000]) for i in range(0, 120000, 15000)]
    got = check(L, False, [b"".join(s)] + [s[0][:-2]] * 20, verify=1)
    assert got[0][0] == 0 and stats(L)["rounds"] == 8


def test_launch_count_does_not_grow_with_the_stream_count(L):
    t = text(200000, stream=29)
    counts = []
    for n in (8, 64):
        streams = [member(t[i * 2000:i * 2000 + 2000]) for i in range(n)]
        data, offs, lens = packed(streams)
        l0 = L.b200z_launch_count()
        got = batch(L, True, data, offs, lens, [room(s) for s in streams], 0)
        counts.append(L.b200z_launch_count() - l0)
        assert [g[2] for g in got] == [t[i * 2000:i * 2000 + 2000] for i in range(n)]
    assert counts[0] == counts[1], counts
    counts = []
    for n in (8, 64):
        streams = [zlib.compress(t[i * 2000:i * 2000 + 2000]) for i in range(n)]
        data, offs, lens = packed(streams)
        l0 = L.b200z_launch_count()
        batch(L, False, data, offs, lens, [room(s) for s in streams], 1)
        counts.append(L.b200z_launch_count() - l0)
    assert counts[0] == counts[1], counts


def test_python_decode_batches(L):
    import archive_b200 as a
    t = text(50000, stream=31)
    streams = [member(t[:i * 5000]) for i in range(8)] + [b"".join(member(t[i:i + 9000], hint=True) for i in range(0, 45000, 9000))]
    got = a.gzip_decode_batch(streams, verify=True)
    assert [g[0] for g in got] == [0] * 9
    assert [g[1] for g in got] == [t[:i * 5000] for i in range(8)] + [t[:45000]]
    big = zlib.compress(bytes(300000))  # 1000:1: the first room (4n + 1024) is too small, the retry fits
    got = a.zlib_decode_batch([big, zlib.compress(t)], verify=True)
    assert got == [(0, bytes(300000)), (0, t)]


# ---------------------------------------------------------------- encode


def encode_batch(L, gz, contents, caps, level, wb=15, raw=False, mtime=0):
    data, offs, lens = packed(contents)
    src = buf(data)
    out_off, tot = [], 0
    for c in caps:
        out_off.append(tot)
        tot += c
    out = (C.c_uint8 * max(tot, 1))()
    n = len(contents)
    ol, rc = (C.c_uint64 * max(n, 1))(), (C.c_int32 * max(n, 1))()
    if gz:
        r = L.b200z_gzip_encode_batch(C.addressof(src), a64(offs), a64(lens), n, level, mtime, C.addressof(out), a64(out_off), a64(caps),
                                      ol, rc)
    else:
        r = L.b200z_zlib_encode_batch(C.addressof(src), a64(offs), a64(lens), n, level, wb, int(raw), C.addressof(out), a64(out_off),
                                      a64(caps), ol, rc)
    assert r == 0, L.b200z_last_error()
    return [(rc[i], ol[i], None if rc[i] else C.string_at(C.addressof(out) + out_off[i], ol[i])) for i in range(n)]


def encode_single(L, gz, x, cap, level, wb=15, raw=False, mtime=0):
    src = buf(x)
    out = (C.c_uint8 * max(cap, 1))()
    n = C.c_size_t(0)
    if gz:
        rc = L.b200z_gzip_encode(C.addressof(src), len(x), level, mtime, C.addressof(out), cap, C.byref(n))
    else:
        rc = L.b200z_zlib_encode(C.addressof(src), len(x), level, wb, int(raw), C.addressof(out), cap, C.byref(n))
    return rc, n.value, None if rc else C.string_at(C.addressof(out), n.value)


def contents():
    t = text(150000, stream=37)
    return [b"", b"a", t[:100], t[:5000], bytes(70000), t[7000:100000], t[:33000]]


@pytest.mark.parametrize("level", range(10))
def test_encode_every_level(L, level):
    cs = contents()
    for gz in (True, False):
        caps = [L.b200z_deflate_bound(len(x)) + 18 for x in cs]
        got = encode_batch(L, gz, cs, caps, level, mtime=0x01020304)
        for x, g, cap in zip(cs, got, caps):
            assert g == encode_single(L, gz, x, cap, level, mtime=0x01020304)
            want = orc.gzip_encode(x, level, mtime=0x01020304) if gz else orc.zlib_encode(x, level)
            assert g[2] == want[1]


@pytest.mark.parametrize("wb", range(9, 16))
def test_encode_window_bits_and_raw(L, wb):
    cs = contents()
    for raw in (False, True):
        for level in (1, 6):
            caps = [L.b200z_deflate_bound(len(x)) + 18 for x in cs]
            got = encode_batch(L, False, cs, caps, level, wb=wb, raw=raw)
            for x, g, cap in zip(cs, got, caps):
                assert g == encode_single(L, False, x, cap, level, wb=wb, raw=raw)
                assert g[2] == orc.zlib_encode(x, level, window_bits=wb, raw=raw)[1]


def test_encode_short_rooms(L):
    cs = contents()
    for gz in (True, False):
        full = encode_batch(L, gz, cs, [L.b200z_deflate_bound(len(x)) + 18 for x in cs], 6)
        for delta in (0, -1):
            caps = [max(0, f[1] + delta) for f in full]
            caps[0] = 0
            got = encode_batch(L, gz, cs, caps, 6)
            for x, g, cap in zip(cs, got, caps):
                assert g == encode_single(L, gz, x, cap, 6)
            assert [g[0] for g in got][1:] == [0 if delta == 0 else E_NOSPC] * (len(cs) - 1)


def test_encode_round_trip_through_the_decode_batches(L):
    import archive_b200 as a
    cs = contents() * 2
    for level in (0, 1, 6, 9):
        gz = a.gzip_encode_batch(cs, level=level, mtime=5)
        assert gz == [a.GZipEncoder().encode_bytes(x, level=level, mtime=5) for x in cs]
        assert a.gzip_decode_batch(gz, verify=True) == [(0, x) for x in cs]
        zl = a.zlib_encode_batch(cs, level=level, window_bits=12)
        assert zl == [a.ZLibEncoder().encode_bytes(x, level=level, window_bits=12) for x in cs]
        assert a.zlib_decode_batch(zl, verify=True) == [(0, x) for x in cs]
        rw = a.zlib_encode_batch(cs, level=level, raw=True)
        assert a.zlib_decode_batch(rw, raw=True) == [(0, x) for x in cs]
