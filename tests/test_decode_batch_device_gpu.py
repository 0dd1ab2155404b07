"""b200z_{gzip,zlib,bzip2,xz}_decode_batch_to_device: the decode batches with their output slots in device memory.

Every stream must come out of the device call exactly as it comes out of the host batch with the same arguments (rc,
out_len and the slot's bytes) and as the oracle's restatement of the reference gives it; nothing outside the slots may be
written (every such byte keeps the guard value 0xA5), whatever the slots' order, gaps and alignment, and whatever the
device groups are.  The same tests run on an H100 (torch CUDA tensors, on a side stream) and on the emulated library with
B200Z_EMU_TESTS=1 (numpy arrays as device memory; its ASan build then checks that k_copy_slots reads and writes nothing
outside the documented buffers).  Bit-exact: byte work has no tolerance."""
import bz2
import ctypes as C
import glob
import gzip as pygzip
import lzma
import os
import random
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest

import oracle_lib as orc
import xz_build as xb

EMU = os.environ.get("B200Z_EMU_TESTS") == "1"
GOLD = os.path.join(os.path.dirname(__file__), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, E_NODEVICE, E_ARG, E_NOSPC, E_DATA, E_THROW = 0, -1, -2, -3, -4, -5
RC = {orc.OK: OK, orc.FALSE: E_DATA, orc.THROW: E_THROW}
GUARD = 0xA5
VERIFY, RAW = 1, 2  # B200Z_GZIP_VERIFY, B200Z_GZIP_RAW
CODECS = ("gzip", "zlib", "bzip2", "xz")
gpu = pytest.mark.gpu
needs_device = pytest.mark.needs_device


# ------------------------------------------------------------------ device buffers, on either tier
class Device:
    """Device memory of the library's device: torch CUDA tensors used on a side stream on the GPU; numpy arrays on the
    emulated library, whose device memory is host memory and whose launches finish before they return."""

    def __init__(self):
        from archive_b200 import _ffi
        self.L = _ffi.ensure_init()
        self.torch = None
        if not EMU:
            import torch
            self.torch = torch
            self.stream = torch.cuda.Stream()

    def full(self, n, fill=GUARD):
        if self.torch is None:
            return np.full(max(n, 1), fill, np.uint8)
        with self.torch.cuda.stream(self.stream):
            return self.torch.full((max(n, 1),), fill, dtype=self.torch.uint8, device="cuda")

    def ptr(self, d):
        return d.ctypes.data if self.torch is None else d.data_ptr()

    def get(self, d):
        return d.copy() if self.torch is None else d.cpu().numpy()

    def handle(self):
        return None if self.torch is None else self.stream.cuda_stream


@pytest.fixture(scope="module")
def D():
    d = Device()
    L = d.L
    for hook in ("gzip", "bz2", "xz"):
        getattr(L, f"b200z_debug_{hook}_batch_set").argtypes = [C.c_uint]
        getattr(L, f"b200z_debug_{hook}_batch_stats").argtypes = [C.c_void_p]
    yield d
    for hook in ("gzip", "bz2", "xz"):
        getattr(L, f"b200z_debug_{hook}_batch_set")(0)


def a64(v):
    return (C.c_uint64 * max(len(v), 1))(*v)


def host_buf(b):
    return (C.c_uint8 * max(len(b), 1)).from_buffer_copy(b or b"\0")


def call(L, codec, to_dev, data_addr, offs, lens, n, out_addr, out_offs, caps, out_len, rc, verify, raw=0, stream=None):
    args = [data_addr, offs, lens, n, verify] + ([raw] if codec == "zlib" else []) + [out_addr, out_offs, caps, out_len, rc]
    name = f"b200z_{codec}_decode_batch"
    return getattr(L, name + "_to_device")(*args, stream) if to_dev else getattr(L, name)(*args)


def packed(streams):
    data, offs, lens = b"", [], []
    for z in streams:
        offs.append(len(data))
        lens.append(len(z))
        data += z
    return data, offs, lens


def layout(caps, mode, rng):
    """out_off of every slot: 'packed' back to back in order; 'scattered' in reverse order, with gaps, at odd offsets"""
    offs, pos = [0] * len(caps), 0
    order = range(len(caps)) if mode == "packed" else reversed(range(len(caps)))
    for i in order:
        if mode != "packed":
            pos += rng.randrange(1, 40) | 1
        offs[i] = pos
        pos += caps[i]
    return offs, pos + (0 if mode == "packed" else 23)


def pair(D, codec, data, offs, lens, caps, verify, raw=0, mode="scattered", lead=13, seed=1):
    """The host batch and the device batch on the same arguments -> [(rc, out_len, bytes)], after checking that both agree
    and that the device call wrote nothing outside its slots.  The device slots start `lead` bytes into a larger
    allocation."""
    L, n = D.L, len(lens)
    out_offs, extent = layout(caps, mode, random.Random(seed))
    src = host_buf(data)
    io, il, oo, cc = a64(offs), a64(lens), a64(out_offs), a64(caps)
    h_out = (C.c_uint8 * max(extent, 1))()
    h_len, h_rc = (C.c_uint64 * max(n, 1))(), (C.c_int32 * max(n, 1))()
    assert call(L, codec, False, C.addressof(src), io, il, n, C.addressof(h_out), oo, cc, h_len, h_rc, verify, raw) == OK
    d = D.full(lead + extent + 29)
    d_len, d_rc = (C.c_uint64 * max(n, 1))(), (C.c_int32 * max(n, 1))()
    r = call(L, codec, True, C.addressof(src), io, il, n, D.ptr(d) + lead, oo, cc, d_len, d_rc, verify, raw, D.handle())
    assert r == OK, L.b200z_last_error()
    got = D.get(d)
    hb = np.frombuffer(h_out, np.uint8)
    inside = np.zeros(len(got), bool)
    res = []
    for i in range(n):
        assert (d_rc[i], d_len[i]) == (h_rc[i], h_len[i]), (codec, i, d_rc[i], d_len[i], h_rc[i], h_len[i])
        o = out_offs[i]
        inside[lead + o:lead + o + caps[i]] = True
        k = min(d_len[i], caps[i])
        if d_rc[i] != E_NOSPC:
            assert bytes(got[lead + o:lead + o + k]) == bytes(hb[o:o + k]), (codec, i)
        res.append((d_rc[i], d_len[i], bytes(got[lead + o:lead + o + k])))
    assert (got[~inside] == GUARD).all(), (codec, "bytes outside the slots were written")
    return res


def oracle(codec, z, verify, raw=0):
    if codec == "gzip":
        return orc.gzip_decode(z, verify=bool(verify & VERIFY), raw=bool(verify & RAW))
    if codec == "zlib":
        return orc.zlib_decode(z, verify=bool(verify), raw=bool(raw))
    if codec == "bzip2":
        return orc.bzip2_decode(z, verify=bool(verify))
    return xb.decode(z, bool(verify))


def check(D, codec, streams, verify=0, raw=0, caps=None, ranges=None, use_oracle=True, modes=("scattered", "packed")):
    """every stream through the device call against the host batch (pair) and the oracle; `ranges` = (data, offs, lens)
    reads the streams from other places of one buffer (streams[i] == data[offs[i]:offs[i] + lens[i]])"""
    caps = caps or [room(D.L, codec, z) for z in streams]
    data, offs, lens = ranges or packed(streams)
    for mode in modes:
        got = pair(D, codec, data, offs, lens, caps, verify, raw, mode)
        if not use_oracle:
            continue
        for i, z in enumerate(streams):
            if got[i][0] == E_NOSPC:
                continue
            st, want = oracle(codec, z, verify, raw)[:2]
            assert got[i][0] == RC[st], (codec, i, got[i][0], st)
            assert st == orc.THROW or got[i][2] == want, (codec, i)
    return got


def room(L, codec, z):
    """a room that holds what the stream decodes to"""
    if codec == "xz":
        return L.b200z_xz_bound(host_buf(z), len(z))
    st, out = oracle(codec, z, 0)[:2]
    return len(out) + 64


def text(n, stream=7):
    from archive_b200 import synth
    return synth.text(n, stream=stream).tobytes()


def member(chunk, level=6, hint=False, zdict=None):
    co = (zlib.compressobj(level, zlib.DEFLATED, -15, 9, zlib.Z_DEFAULT_STRATEGY, zdict) if zdict
          else zlib.compressobj(level, zlib.DEFLATED, -15))
    body = co.compress(chunk) + co.flush()
    trailer = struct.pack("<II", zlib.crc32(chunk), len(chunk))
    if hint:
        total = 10 + 2 + 6 + len(body) + 8
        return (b"\x1f\x8b\x08\x04" + bytes(4) + b"\x00\xff" + struct.pack("<H", 6) + b"BC" + struct.pack("<HH", 2, total - 1)
                + body + trailer)
    return b"\x1f\x8b\x08\x00" + bytes(4) + b"\x00\xff" + body + trailer


def damaged(good, rng, k=6):
    out = [good[:c] for c in sorted(rng.sample(range(1, len(good)), k))]
    for _ in range(k):
        b = bytearray(good)
        b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
        out.append(bytes(b))
    return out


# ------------------------------------------------------------------ corpora, one per codec
def corpus(codec):
    rng = random.Random(hash(codec) & 0xffff)
    t = text(300000, stream=31)
    if codec == "gzip":
        golden = [open(p, "rb").read() for p in sorted(glob.glob(os.path.join(GOLD, "*.gz")))]
        good = [member(t[:40000]), member(t[:120000], hint=True) + member(t[5000:9000], hint=True),  # hinted run
                member(t[:7000]) + member(t[7000:30000], zdict=t[:7000]) + member(t[30000:31000]),  # multi-member, reaching back
                zlib.compress(t[:50000]),  # no gzip header: the zlib fall-back
                pygzip.compress(t[:200000], 9)]
        return golden + good, good
    if codec == "zlib":
        s = [zlib.compress(t[i:i + 20000], 1 + i // 40000) for i in range(0, 160000, 20000)]
        good = [b"".join(s[:4]), s[4], s[5] + s[6], zlib.compress(t, 9)]
        return good + [s[0][:-1] + bytes([s[0][-1] ^ 1]) + s[1], s[2] + b"\x78\x00" + s[3]], good
    if codec == "bzip2":
        golden = [open(p, "rb").read() for p in sorted(glob.glob(os.path.join(GOLD, "**", "*.bz2"), recursive=True))]
        good = [bz2.compress(t[:30000], 1), bz2.compress(t, 1),  # 3 blocks
                bz2.compress(bytes(rng.randrange(256) for _ in range(150000)), 1)]  # 2 blocks
        return golden + good, good
    golden = [open(p, "rb").read() for p in sorted(glob.glob(os.path.join(GOLD, "xz", "*.xz")))]
    good = [lzma.compress(t[:n], check=ck) for n, ck in ((100, lzma.CHECK_NONE), (5000, lzma.CHECK_CRC32),
                                                         (70000, lzma.CHECK_CRC64), (40000, lzma.CHECK_SHA256))]
    good += [xb.xz_blocks(t[:200000], 30000, check="crc64"), xb.xz_blocks(t[:60000], 60000, check="crc32")]
    return golden + good, good


@gpu
@pytest.mark.parametrize("codec", CODECS)
def test_fixtures_shuffled_with_duplicates_and_shared_ranges(D, codec):
    streams, good = corpus(codec)
    rng = random.Random(3)
    order = streams + rng.sample(streams, len(streams) // 2)
    rng.shuffle(order)
    for v in (0, 1):  # (1 is B200Z_GZIP_VERIFY for gzip)
        check(D, codec, order, verify=v)
    # duplicate and overlapping input ranges: every stream read from one shared buffer
    data, offs, lens = packed(good)
    streams2 = good + [good[0], good[-1]]
    offs2, lens2 = offs + [offs[0], offs[-1]], lens + [lens[0], lens[-1]]
    check(D, codec, streams2, ranges=(data, offs2, lens2), modes=("scattered",))


@gpu
@pytest.mark.parametrize("codec", CODECS)
def test_damaged_and_truncated_streams_between_good_ones(D, codec):
    streams, good = corpus(codec)
    rng = random.Random(17)
    mixed = []
    for g in good[:3]:
        for bad in damaged(g, rng):
            mixed += [bad, g]
    for v in (0, 1):
        check(D, codec, mixed, verify=v, modes=("scattered",))


@gpu
def test_zlib_raw_and_gzip_raw_streams(D):
    t = text(60000, stream=5)
    raws = [zlib.compress(t[i:i + 9000])[2:-4] for i in range(0, 54000, 9000)]
    check(D, "zlib", raws + [raws[0] + raws[1]], raw=1, modes=("scattered",))
    check(D, "gzip", [member(t[:9000])[10:-8], raws[1], member(t[:3000])], verify=RAW, use_oracle=False, modes=("scattered",))


@gpu
@pytest.mark.parametrize("codec", CODECS)
def test_rooms_too_small(D, codec):
    streams, good = corpus(codec)
    caps = [room(D.L, codec, z) for z in good]
    small = [max(c // 3, 0) for c in caps]
    small[1] = 0
    got = check(D, codec, good, caps=[s if i % 2 else c for i, (s, c) in enumerate(zip(small, caps))])
    assert any(r[0] == E_NOSPC for r in got), got


@gpu
@needs_device
def test_gzip_stream_of_16_mib_compressed_goes_through_k12(D):
    """K12 (the whole-GPU decode of one large DEFLATE stream) delivers through the device sink as well."""
    L = D.L
    L.b200z_debug_gzip_batch_stats.argtypes = [C.c_void_p]
    big_text = text(48 << 20, stream=29)
    big = member(big_text)
    assert len(big) >= 16 << 20, len(big)
    small = [member(big_text[i:i + 30000]) for i in range(0, 150000, 30000)]
    streams = small[:2] + [big] + small[2:]
    caps = [room(L, "gzip", z) for z in streams]
    caps[2] = 2 * len(big_text)
    got = check(D, "gzip", streams, caps=caps, use_oracle=False, modes=("scattered",))
    s = (C.c_ulonglong * 6)()
    L.b200z_debug_gzip_batch_stats(s)
    assert s[4] == s[5] == 1, list(s)  # K12 was offered the large member and decoded it
    assert got[2][0] == OK and got[2][2] == big_text


@gpu
def test_k12_with_a_lowered_threshold(D):
    """The same on both tiers, with K12's threshold lowered so that a 2 MiB member takes it."""
    L = D.L
    L.b200z_debug_inflate_chunked_set(C.c_ulonglong(256 << 10), C.c_ulonglong(0))
    try:
        t = text(2 << 20, stream=23)
        big = member(t)
        small = [member(t[i:i + 5000]) for i in range(0, 20000, 5000)]
        got = check(D, "gzip", small[:2] + [big] + small[2:] + [zlib.compress(t)], use_oracle=False, modes=("scattered",))
        s = (C.c_ulonglong * 6)()
        L.b200z_debug_gzip_batch_stats(s)
        assert s[5] == 2, list(s)
        assert got[2][2] == t and got[-1][2] == t
    finally:
        L.b200z_debug_inflate_chunked_set(C.c_ulonglong(0), C.c_ulonglong(0))


@gpu
@pytest.mark.parametrize("codec", CODECS)
def test_large_slots_at_every_alignment(D, codec):
    """Slots larger than one k_copy_slots piece (64 KiB) at every destination offset modulo 16, against the group
    buffer's alignment: the vector path, the shifted-vector path and the byte heads and tails."""
    t = text(200000, stream=3)
    enc = {"gzip": lambda b: member(b), "zlib": zlib.compress, "bzip2": lambda b: bz2.compress(b, 1),
           "xz": lambda b: lzma.compress(b, check=lzma.CHECK_CRC32)}[codec]
    streams = [enc(t[i * 1000:i * 1000 + 70000 + 13 * i]) for i in range(16)]
    caps = [room(D.L, codec, z) for z in streams]
    data, offs, lens = packed(streams)
    for lead in range(16):
        got = pair(D, codec, data, offs, lens, caps, 0, lead=lead, seed=lead)
        assert all(g[0] == OK for g in got)
        assert [g[2] for g in got] == [t[i * 1000:i * 1000 + 70000 + 13 * i] for i in range(16)]


# ------------------------------------------------------------------ device groups and launches
def _groups(L, codec):
    hook = {"gzip": "gzip", "zlib": "gzip", "bzip2": "bz2", "xz": "xz"}[codec]
    s = (C.c_ulonglong * 6)()
    getattr(L, f"b200z_debug_{hook}_batch_stats")(s)
    return s[1]


def _set_groups(L, codec, cap):
    hook = {"gzip": "gzip", "zlib": "gzip", "bzip2": "bz2", "xz": "xz"}[codec]
    getattr(L, f"b200z_debug_{hook}_batch_set")(cap)


def _launches(D, codec, streams, caps, to_dev):
    L, n = D.L, len(streams)
    data, offs, lens = packed(streams)
    out_offs, extent = layout(caps, "scattered", random.Random(5))
    src = host_buf(data)
    out = D.full(extent) if to_dev else (C.c_uint8 * extent)()
    addr = D.ptr(out) if to_dev else C.addressof(out)
    ol, rc = (C.c_uint64 * n)(), (C.c_int32 * n)()
    before = L.b200z_launch_count()
    assert call(L, codec, to_dev, C.addressof(src), a64(offs), a64(lens), n, addr, a64(out_offs), a64(caps), ol, rc, 0, 0,
                D.handle()) == OK
    assert all(r == OK for r in rc[:n])
    return L.b200z_launch_count() - before, _groups(L, codec)


@gpu
@pytest.mark.parametrize("codec", CODECS)
def test_forced_device_groups_and_launch_count(D, codec):
    """Small device groups give the same results; the device sink adds one launch per group, whatever the number of
    streams."""
    L = D.L
    t = text(100000, stream=19)
    enc = {"gzip": lambda b: member(b), "zlib": zlib.compress, "bzip2": lambda b: bz2.compress(b, 1),
           "xz": lambda b: lzma.compress(b, check=lzma.CHECK_CRC64)}[codec]
    streams = [enc(t[i * 997:i * 997 + 3000 + 211 * i]) for i in range(24)]
    caps = [room(L, codec, z) for z in streams]
    whole = check(D, codec, streams, modes=("scattered",))
    # bzip2 groups are capped by blocks (one per stream here), the others by streams
    _set_groups(L, codec, 5)
    try:
        assert check(D, codec, streams, modes=("scattered",)) == whole
        host, g_host = _launches(D, codec, streams, caps, False)
        dev, g_dev = _launches(D, codec, streams, caps, True)
        assert g_host == g_dev == 5, (g_host, g_dev)
        assert dev - host == g_dev, (dev, host, g_dev)
    finally:
        _set_groups(L, codec, 0)
    for k in (6, 24):  # one group: one more launch than the host batch, for 6 streams as for 24
        host, _ = _launches(D, codec, streams[:k], caps[:k], False)
        dev, g = _launches(D, codec, streams[:k], caps[:k], True)
        assert g == 1 and dev - host == 1, (k, dev, host)


# ------------------------------------------------------------------ argument errors
@gpu
@pytest.mark.parametrize("codec", CODECS)
def test_argument_errors_write_nothing(D, codec):
    L = D.L
    good = corpus(codec)[1][:2]
    data, offs, lens = packed(good)
    caps = [room(L, codec, z) for z in good]
    src = host_buf(data)
    d = D.full(sum(caps) + 64)

    def attempt(offs_, lens_, oo, cc, base=None, null=None):
        n = len(lens_)
        ol = (C.c_uint64 * n)(*([77] * n))
        rc = (C.c_int32 * n)(*([77] * n))
        arrs = [a64(offs_), a64(lens_), a64(oo), a64(cc), ol, rc]
        if null is not None:
            arrs[null] = None
        r = call(L, codec, True, C.addressof(src), arrs[0], arrs[1], n, D.ptr(d) if base is None else base, arrs[2], arrs[3],
                 arrs[4], arrs[5], 0, 0, D.handle())
        if r == E_ARG:
            assert list(ol) == [77] * n and list(rc) == [77] * n
        return r

    oo = [0, caps[0]]
    assert attempt(offs, lens, oo, caps) == OK
    d = D.full(sum(caps) + 64)
    for null in range(6):
        assert attempt(offs, lens, oo, caps, null=null) == E_ARG
    assert attempt([2**64 - 4, offs[1]], [8, lens[1]], oo, caps) == E_ARG  # wrapping input range
    assert attempt(offs, lens, [2**64 - 4, caps[0]], [8, caps[1]]) == E_ARG  # wrapping output range
    assert attempt(offs, lens, [0, caps[0] - 1], caps) == E_ARG  # overlapping slots
    assert attempt(offs, lens, oo, caps, base=0) == E_ARG  # no output buffer
    pinned = L.b200z_host_alloc(sum(caps) + 64)  # host memory, page-locked: not device memory
    try:
        C.memset(pinned, GUARD, sum(caps) + 64)
        assert attempt(offs, lens, oo, caps, base=pinned) == E_ARG
        assert C.string_at(pinned, sum(caps) + 64) == bytes([GUARD]) * (sum(caps) + 64)
    finally:
        L.b200z_host_free(pinned)
    assert (D.get(d) == GUARD).all()
    # no room at all: the base is never looked at
    assert attempt(offs, lens, [0, 0], [0, 0], base=0) == OK
    assert attempt([], [], [], []) == OK


@gpu
@needs_device
@pytest.mark.parametrize("codec", CODECS)
def test_pageable_host_pointer_is_an_argument_error(D, codec):
    L = D.L
    good = corpus(codec)[1][:1]
    data, offs, lens = packed(good)
    caps = [room(L, codec, good[0])]
    host = np.full(caps[0], GUARD, np.uint8)
    ol, rc = (C.c_uint64 * 1)(), (C.c_int32 * 1)()
    r = call(L, codec, True, C.addressof(host_buf(data)), a64(offs), a64(lens), 1, host.ctypes.data, a64([0]), a64(caps), ol,
             rc, 0, 0, D.handle())
    assert r == E_ARG and (host == GUARD).all()


# ------------------------------------------------------------------ ordering (GPU only)
@gpu
@needs_device
@pytest.mark.parametrize("codec", CODECS)
def test_decoded_bytes_win_over_earlier_work_on_the_callers_stream(D, codec):
    """A fill of the output buffer enqueued on the caller's stream behind a long kernel, right before the call: the
    library's stream waits for it, so the decoded bytes land after the fill."""
    import torch
    L = D.L
    good = corpus(codec)[1]
    data, offs, lens = packed(good)
    caps = [room(L, codec, z) for z in good]
    out_offs, extent = layout(caps, "packed", random.Random(1))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d = torch.zeros(extent, dtype=torch.uint8, device="cuda")
        torch.cuda._sleep(200_000_000)  # ~0.1 s of spinning on s
        d.fill_(0x5A)
    n = len(good)
    ol, rc = (C.c_uint64 * n)(), (C.c_int32 * n)()
    src = host_buf(data)
    assert call(L, codec, True, C.addressof(src), a64(offs), a64(lens), n, d.data_ptr(), a64(out_offs), a64(caps), ol, rc, 0, 0,
                s.cuda_stream) == OK
    got = d.cpu().numpy()  # (the call has returned: the bytes are in place, readable from any stream)
    for i, z in enumerate(good):
        assert rc[i] == OK
        assert bytes(got[out_offs[i]:out_offs[i] + ol[i]]) == oracle(codec, z, 0)[1], (codec, i)


# ------------------------------------------------------------------ the Python API
@gpu
@needs_device
def test_python_decode_batches_to_a_cuda_device():
    import torch
    import archive_b200 as a
    streams = {c: corpus(c)[0] for c in CODECS}
    t = text(400000, stream=2)
    streams["gzip"] = streams["gzip"] + [member(bytes(3 << 20))]  # its first room (4n + 1024) is too small: retried
    streams["zlib"] = streams["zlib"] + [zlib.compress(bytes(2 << 20)), zlib.compress(t)]
    fns = {"gzip": a.gzip_decode_batch, "zlib": a.zlib_decode_batch, "bzip2": a.bzip2_decode_batch, "xz": a.xz_decode_batch}
    side = torch.cuda.Stream()
    for codec, fn in fns.items():
        want = fn(streams[codec])
        with torch.cuda.stream(side):
            torch.cuda._sleep(50_000_000)  # work already queued on the current stream
            got = fn(streams[codec], device="cuda")
        assert len(got) == len(want)
        total = torch.zeros((), dtype=torch.int64, device="cuda")
        for (rc, tens), (hrc, hbytes) in zip(got, want):
            assert rc == hrc
            assert tens.dtype == torch.uint8 and tens.dim() == 1 and tens.is_cuda and tens.numel() == len(hbytes)
            total += tens.to(torch.int64).sum()  # used on another stream with no synchronisation
            assert bytes(tens.cpu().numpy()) == hbytes, codec
        assert int(total) == sum(sum(b) for _, b in want)
        assert fn([], device="cuda") == []
    with pytest.raises(ValueError):
        a.gzip_decode_batch(streams["gzip"][:1], device="cpu")
    with pytest.raises(ValueError):
        a.xz_decode_batch(streams["xz"][:1], device=torch.device("cuda", torch.cuda.device_count() + 3))


# ------------------------------------------------------------------ without a device
def test_entry_points_report_no_device_and_write_nothing():
    """In a process that has no device (b200z_init never succeeds), every *_to_device entry point returns
    B200Z_E_NODEVICE and writes nothing."""
    prog = r"""
import ctypes as C, sys
sys.path.insert(0, sys.argv[1])
from archive_b200 import _ffi
L = _ffi.lib()
assert L.b200z_init(0, 0) == _ffi.E_NODEVICE
data = (C.c_uint8 * 16)(*b"\x1f\x8b\x08\x00" + bytes(12))
a = lambda *v: (C.c_uint64 * len(v))(*v)
out = (C.c_uint8 * 64)(*([0xA5] * 64))
for codec in ("gzip", "zlib", "bzip2", "xz"):
    ol, rc = a(7, 7), (C.c_int32 * 2)(7, 7)
    args = [data, a(0, 4), a(16, 8), 2, 0] + ([0] if codec == "zlib" else []) + [out, a(0, 32), a(32, 32), ol, rc, None]
    assert getattr(L, "b200z_%s_decode_batch_to_device" % codec)(*args) == _ffi.E_NODEVICE, codec
    assert list(ol) == [7, 7] and list(rc) == [7, 7] and bytes(out) == b"\xa5" * 64, codec
print("ok")
"""
    env = {k: v for k, v in os.environ.items() if k not in ("B200Z_LIB", "B200Z_EMU_TESTS")}
    env["CUDA_VISIBLE_DEVICES"] = ""
    r = subprocess.run([sys.executable, "-c", prog, ROOT], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stdout + r.stderr
