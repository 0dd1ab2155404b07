"""TEST INFRASTRUCTURE: the archives and the extraction harness shared by tests/test_zip_chunked_emul.py (the emulated library)
and tests/test_zip_chunked_gpu.py (the device).  Large ZIP members go through K12 inside b200z_zip_extract; every archive
is extracted twice by the same library -- with K12, and with its threshold out of reach so that every member takes the
exact path -- and the statuses, out_len and bytes of every member must be identical, and equal to the oracle's bytes
for every member that decodes.  The extraction mirrors archive_b200/zip.py's ZipDecoder._extract, including its retry
with more room after B200Z_U_NOSPC."""
import ctypes as C
import io
import struct
import zipfile
import zlib

import oracle_lib as orc
import zip_crypt_build as zcb
from archive_b200._ffi import ZipEntry

OFF = 1 << 62  # a K12 threshold no member reaches: the exact path
U_DONE, U_NOSPC = 0, -2
WEB_EOS = 1


class Harness:
    def __init__(self, L, thresh, chunk):
        self.L, self.thresh, self.chunk = L, thresh, chunk

    def set(self, thresh, chunk=0):
        self.L.b200z_debug_inflate_chunked_set(C.c_ulonglong(thresh), C.c_ulonglong(chunk))

    def caps(self, max_streams=0, max_pages=0):
        self.L.b200z_debug_zip_chunked_set(C.c_uint(max_streams), C.c_uint(max_pages))

    def stats(self):
        a, m = (C.c_ulonglong * 5)(), (C.c_double * 3)()
        self.L.b200z_debug_zip_chunked_stats(a, m)
        return dict(zip(("offered", "accepted", "fell_back", "rounds", "batches"), list(a)))

    def entries(self, data):
        cnt = C.c_size_t(0)
        assert self.L.b200z_zip_list(data, C.c_size_t(len(data)), None, C.c_size_t(0), C.byref(cnt)) == 0
        ents = (ZipEntry * max(1, cnt.value))()
        assert self.L.b200z_zip_list(data, C.c_size_t(len(data)), ents, C.c_size_t(cnt.value), C.byref(cnt)) == 0
        return ents, cnt.value

    def extract(self, data, flags=0, password=None):
        """-> ([(status, out_len, bytes)] per entry, [stats of every b200z_zip_extract call])"""
        ents, n = self.entries(data)
        room = [max(ents[i].hint_uncomp_size, ents[i].uncomp_size, 1) if ents[i].has_data else 0 for i in range(n)]
        res, calls = [None] * n, []
        todo = list(range(n))
        while todo:
            m = len(todo)
            sub = (ZipEntry * m)(*[ents[i] for i in todo])
            off, tot = [], 0
            for i in todo:
                off.append(tot)
                tot += (room[i] + 63) & ~63
            out = (C.c_uint8 * max(tot, 1))()
            out_len, st = (C.c_uint64 * m)(), (C.c_int32 * m)()
            rc = self.L.b200z_zip_extract_password(
                data, C.c_size_t(len(data)), sub, C.c_size_t(m), C.cast(out, C.c_void_p), C.c_size_t(max(tot, 1)),
                (C.c_uint64 * m)(*off), (C.c_uint64 * m)(*[room[i] for i in todo]), out_len, st, C.c_uint32(flags),
                password, C.c_size_t(len(password or b"")))
            assert rc == 0, rc
            calls.append(self.stats())
            again = []
            for k, i in enumerate(todo):
                if st[k] == U_NOSPC and room[i] < (1 << 32) - 64:
                    room[i] = min(max(room[i] * 4, int(out_len[k]), int(ents[i].comp_size) * 4), (1 << 32) - 64)
                    again.append(i)
                    continue
                res[i] = (st[k], int(out_len[k]), C.string_at(C.addressof(out) + off[k], min(int(out_len[k]), room[i])))
            todo = again
        return res, calls

    def both(self, data, flags=0, password=None, oracle=True):
        """extract through K12 and through the exact path; the results must be identical (and match the oracle)"""
        self.set(OFF)
        ref, _ = self.extract(data, flags, password)
        self.set(self.thresh, self.chunk)
        try:
            got, calls = self.extract(data, flags, password)
        finally:
            self.set(OFF)
        assert [r[:2] for r in got] == [r[:2] for r in ref]
        for i, (g, r) in enumerate(zip(got, ref)):
            assert g[2] == r[2], i
        if oracle:
            want = zcb.oracle_members(data, password, web_eos=bool(flags & WEB_EOS)) if password else None
            st, ents = orc.zip_list(data)
            assert st == orc.OK
            for i, e in enumerate(ents):
                if got[i][0] != U_DONE or not e.has_data:
                    continue
                ob = want[i][1] if password else orc.zip_member(data, e, web_eos=bool(flags & WEB_EOS))[1]
                assert got[i][2] == ob, i
        return got, calls


def raw(data, level=6, flush_every=0, flush=zlib.Z_SYNC_FLUSH):
    c = zlib.compressobj(level, zlib.DEFLATED, -15)
    if not flush_every:
        return c.compress(data) + c.flush()
    out = []
    for i in range(0, len(data), flush_every):
        out.append(c.compress(data[i:i + flush_every]))
        out.append(c.flush(flush))
    return b"".join(out) + c.flush()


def build(members):
    """members: [(name, payload, method, crc, usize)] or (name, None) for a directory -> a ZIP archive (local headers
    with sizes, central directory, end record), payloads written exactly as given"""
    out, cd = bytearray(), bytearray()
    for name, *rest in members:
        nb = name.encode()
        if rest[0] is None:
            payload, method, crc, usize = b"", 0, 0, 0
            attr = (0o40755 << 16) | 0x10
        else:
            payload, method, crc, usize = rest
            attr = 0o100644 << 16
        pos = len(out)
        out += struct.pack("<IHHHHHIIIHH", 0x04034B50, 20, 0x800, method, 0, 0x21, crc, len(payload), usize, len(nb), 0)
        out += nb + payload
        cd += struct.pack("<IHHHHHHIIIHHHHHII", 0x02014B50, 20, 20, 0x800, method, 0, 0x21, crc, len(payload), usize,
                          len(nb), 0, 0, 0, 0, attr, pos)
        cd += nb
    cd_pos = len(out)
    out += cd
    out += struct.pack("<IHHHHIIH", 0x06054B50, 0, 0, len(members), len(members), len(cd), cd_pos, 0)
    return bytes(out)


def deflated(name, plain, level=6, **kw):
    return (name, raw(plain, level, **kw), 8, zlib.crc32(plain) & 0xFFFFFFFF, len(plain))


def mixed(text, big, small):
    """large deflate members of `big` bytes of text between small deflate, stored, empty, bzip2 and directory entries"""
    import bz2
    t = lambda i, n: text[(i * 7919) % (len(text) - n):][:n]
    s = t(1, small)
    return build([
        deflated("a.txt", t(0, big)),
        deflated("small.txt", s),
        ("stored.bin", s[:5000], 0, zlib.crc32(s[:5000]) & 0xFFFFFFFF, 5000),
        ("dir/", None),
        deflated("b.txt", t(2, big), level=9),
        ("empty.txt", b"", 8, 0, 0),
        ("s.bz2", bz2.compress(s, 9), 12, zlib.crc32(s) & 0xFFFFFFFF, len(s)),
        deflated("c.txt", t(3, big), level=1),
        ("empty_stored", b"", 0, 0, 0),
        deflated("tail.txt", s[:3000]),
    ])


def zipfile_archive(members):
    """[(name, bytes)] -> an archive written by Python's zipfile (deflate, level 6: no flush points)"""
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w", compression=zipfile.ZIP_DEFLATED, compresslevel=6) as z:
        for name, body in members:
            z.writestr(name, body)
    return buf.getvalue()


def zero_sizes(data):
    """the same archive with every uncompressed size field set to 0, in the central directory and the local headers: the
    output room starts at one byte and grows after B200Z_U_NOSPC"""
    b = bytearray(data)
    p = 0
    while True:
        p = b.find(b"PK\x01\x02", p)
        if p < 0:
            break
        b[p + 24:p + 28] = b"\0" * 4
        p += 4
    p = 0
    while True:
        p = b.find(b"PK\x03\x04", p)
        if p < 0:
            break
        b[p + 22:p + 26] = b"\0" * 4
        p += 4
    return bytes(b)


# ---- the cases; `text` is synthetic text, `big` the size of a large member's text (its compressed size must reach the
# threshold under test), `small` that of a small one ----
def case_mixed(H, text, big, small, web_eos):
    got, calls = H.both(mixed(text, big, small), flags=WEB_EOS if web_eos else 0)
    st = calls[-1]
    # K12 takes every large member the exact path decodes to its end; under web_eos a member whose last code lies in its
    # last bits stops short on the exact path (SURVEY Q1), and K12 leaves it to the exact path
    done = sum(got[i][0] == U_DONE for i in (0, 4, 7))
    assert st["offered"] == 3 and st["accepted"] == done and st["fell_back"] == 3 - done, st
    assert done == 3 or web_eos
    return got


def case_final_code_in_last_bits(H, text, big, web_eos):
    # non-final dynamic blocks, then a final fixed block that ends the member: its last code (end-of-block, 7 bits) lies
    # in the member's last 9 bits, where the pure-Dart Inflate stops short (SURVEY Q1) -- unless the look-ahead pad lets
    # it read on.  K12 must give what the exact path gives either way.
    import deflate_craft as dc
    plain = text[:big]
    u = dc.Unit()
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    u.w.raw(c.compress(plain) + c.flush(zlib.Z_SYNC_FLUSH))
    u.plain += plain
    u.fixed(final=True)
    u.literals(b"the end")
    u.match(10, 1000)  # (a reach behind the sync-flush point: the flush-point split keeps the member whole)
    u.eob()
    body = u.w.getvalue()
    full = bytes(u.plain)
    data = build([(f"q{web_eos}", body, 8, zlib.crc32(full) & 0xFFFFFFFF, len(full)), deflated("after", text[:2000])])
    got, calls = H.both(data, flags=WEB_EOS if web_eos else 0)
    assert calls[-1]["offered"] == 1, calls
    if not web_eos:
        assert got[0][0] == U_DONE and got[0][2] == full and calls[-1]["accepted"] == 1, calls
    return got


def case_bitflip(H, text, big, small):
    data = bytearray(mixed(text, big, small))
    st, ents = orc.zip_list(bytes(data))
    e = ents[4]  # b.txt
    data[e.data_off + e.comp_size // 2] ^= 0x08
    got, calls = H.both(bytes(data))
    st = calls[-1]
    assert st["offered"] == 3 and st["accepted"] >= 2, st  # the other two members of its batch are still accepted
    return got


def case_room_one_short_and_zero_sizes(H, text, big):
    a, b = text[:big], text[big:2 * big]
    ma, mb = deflated("a", a), deflated("b", b)
    data = build([ma[:4] + (len(a) - 1,), mb])
    got, calls = H.both(data)
    assert got[0][0] == U_DONE and got[0][2] == a, got[0][:2]  # NOSPC, then the retry with more room
    assert len(calls) == 2 and calls[0]["offered"] == 2 and calls[0]["accepted"] == 1 and calls[1]["accepted"] == 1, calls
    got, calls = H.both(zero_sizes(build([ma, mb])))
    assert [g[2] for g in got] == [a, b]
    assert sum(c["accepted"] for c in calls) == 2, calls


def case_random_declined(H, text, big, nrand):
    import numpy as np
    rnd = np.random.default_rng(5).integers(0, 256, nrand, dtype=np.uint8).tobytes()
    data = build([deflated("rnd", rnd), deflated("t", text[:big])])
    got, calls = H.both(data)
    st = calls[-1]
    assert st["offered"] == 2 and st["accepted"] == 1 and st["fell_back"] == 1, st  # stored blocks: the exact path


def case_flush_points(H, text, n, every):
    # Z_SYNC_FLUSH points: candidates of the flush-point split that the sizing pass rejects (the window continues), so the
    # member stays whole and goes to K12.  Z_FULL_FLUSH points: the member is split, its pieces are units of the batch.
    sync = raw(text[:n], 6, flush_every=every, flush=zlib.Z_SYNC_FLUSH)
    full = raw(text[n:2 * n], 6, flush_every=every, flush=zlib.Z_FULL_FLUSH)
    assert len(sync) >= 256 << 10 and len(full) >= 256 << 10  # (what the split looks at)
    data = build([("sync", sync, 8, zlib.crc32(text[:n]) & 0xFFFFFFFF, n),
                  ("full", full, 8, zlib.crc32(text[n:2 * n]) & 0xFFFFFFFF, n)])
    got, calls = H.both(data)
    st = calls[-1]
    assert st["offered"] == 1 and st["accepted"] == 1, st
    assert [g[2] for g in got] == [text[:n], text[n:2 * n]]


def case_encrypted(H, text, big, small):
    pw = b"k12 secret"
    members = [zcb.Member("aes.txt", text[:big], 8, "aes"), zcb.Member("small", text[:small], 8, "zipcrypto"),
               zcb.Member("zc.txt", text[big:2 * big], 8, "zipcrypto"), zcb.Member("d/", is_dir=True, crypt=None),
               zcb.Member("plain.txt", text[2 * big:3 * big], 8, None)]
    data = zcb.build(members, pw)
    got, calls = H.both(data, password=pw)
    st = calls[-1]
    assert st["offered"] == 3 and st["accepted"] == 3, st
    assert got[0][2] == text[:big] and got[2][2] == text[big:2 * big]


def case_zip_chunks(H, text, big, small, n_chunks):
    import os
    parts = []
    for i in range(6):
        s = text[i * small:(i + 1) * small]
        parts += [deflated(f"s{i}", s), ("st%d" % i, s[:999], 0, zlib.crc32(s[:999]) & 0xFFFFFFFF, 999)]
        if i % 2 == 0:
            parts.append(deflated(f"big{i}", text[i * big // 3:i * big // 3 + big]))
    data = build(parts)
    old = os.environ.get("B200Z_ZIP_CHUNKS")
    os.environ["B200Z_ZIP_CHUNKS"] = str(n_chunks)
    try:
        got, calls = H.both(data)
    finally:
        if old is None:
            del os.environ["B200Z_ZIP_CHUNKS"]
        else:
            os.environ["B200Z_ZIP_CHUNKS"] = old
    assert calls[-1]["accepted"] == 3, calls


def case_pool_cap(H, text, big, small, heavy, max_pages):
    # a member with far more output than its neighbours (`heavy`) needs far more pages: capped pools make it run out and
    # fall back on its own, the others in its batch are still accepted
    comp = heavy
    data = build([deflated("a", text[:big]), deflated("rep", comp), deflated("b", text[big:2 * big]),
                  deflated("s", text[:small])])
    H.caps(max_pages=max_pages)
    try:
        got, calls = H.both(data)
    finally:
        H.caps()
    st = calls[-1]
    assert st["offered"] == 3 and st["accepted"] == 2 and st["fell_back"] == 1, st
    assert got[1][2] == comp


def case_one_stream_per_batch(H, text, big, small):
    data = mixed(text, big, small)
    H.caps(max_streams=1)
    try:
        _, calls = H.both(data)
    finally:
        H.caps()
    assert calls[-1]["batches"] == 3 and calls[-1]["accepted"] == 3, calls
    _, calls = H.both(data)
    assert calls[-1]["batches"] == 1, calls
