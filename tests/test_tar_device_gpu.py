"""b200z_tar_walk_device, TarDecoder.decode_bytes(device=) and tar_decode_batch: the TAR member walk on the device.

The walk's records must equal a restatement of the host walk's position arithmetic (TarDecoder._decode over TarFile.read
with storeData) and the oracle's content ranges (oracle/tar.c); the Python device path must give, member by member, what
the host TarDecoder gives for the same bytes, and raise where it raises.  The C-level tests run on an H100 (torch CUDA
tensors on a side stream) and on the emulated library with B200Z_EMU_TESTS=1 (numpy arrays as device memory); the tests
of the Python API need torch CUDA tensors (needs_device)."""
import ctypes as C
import io
import lzma
import os
import random
import subprocess
import sys
import tarfile

import numpy as np
import pytest

import oracle_lib as orc
import oracle_tar as ot
from test_decode_batch_device_gpu import GUARD, Device, a64
from test_tar import CRAFTED, FIXTURES, FORMATS, TAR, _member, _v7, body, generated, header
from test_tar_gpu import shard_tars

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, E_NODEVICE, E_ARG, E_NOSPC, E_DATA, E_THROW = 0, -1, -2, -3, -4, -5
gpu = pytest.mark.gpu
needs_device = pytest.mark.needs_device
MEMBER = np.dtype([(f, "<u8") for f in ("header_off", "content_off", "content_len")] +
                  [("size", "<i8"), ("header_len", "<u4"), ("pad_", "<u4")])


@pytest.fixture(scope="module")
def D():
    return Device()


# ------------------------------------------------------------------ the archives
def truncation_cuts():
    """Every cut of test_tar.test_truncation."""
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.GNU_FORMAT) as tf:
        _member(tf, "a" * 120, data=b"first" * 30)
        _member(tf, "b", data=b"x" * 513)
        _member(tf, "d", tarfile.DIRTYPE)
        _member(tf, "l", tarfile.SYMTYPE, linkname="k" * 130)
    data = buf.getvalue()
    cuts = set()
    for b in list(range(0, len(data), 512)) + [512 + 150, 1536 + 150, 2048 + 513]:
        cuts |= {b - 1, b, b + 1}
    return [data[:c] for c in sorted(c for c in cuts if 0 <= c <= len(data))]


def corpus():
    """name -> archive bytes: every fixture, every crafted archive, the generated formats and every truncation."""
    out = {f"fixture/{n}": open(os.path.join(TAR, n), "rb").read() for n in FIXTURES}
    out.update({f"crafted/{n}": v for n, v in CRAFTED.items()})
    for fmt in sorted(FORMATS):
        g = generated(FORMATS[fmt])
        out[f"generated/{fmt}"] = _v7(g) if fmt == "v7" else g
    out["generated/latin1"] = generated(tarfile.GNU_FORMAT, encoding="latin-1")
    for i, t in enumerate(truncation_cuts()):
        out[f"cut/{i:02d}"] = t
    return out


_WS_UTF8 = ["\t", "\n", "\x0b", "\x0c", "\r", " ", "\x85", "\xa0", "\u1680"] + [chr(c) for c in range(0x2000, 0x200b)] + \
           ["\u2028", "\u2029", "\u202f", "\u205f", "\u3000", "\ufeff"]


def size_fields():
    """Size fields (12 bytes, NUL-filled when shorter) for the table: every trimmed form on both sides in valid UTF-8 and
    in Latin-1, signs, 12 digits with no NUL, NULs inside, digits 8 and 9, base-256, empty fields and near misses."""
    fs = []
    for w in _WS_UTF8:
        e = w.encode("utf-8")
        fs += [e + b"17" + e, e + b"17", b"17" + e, e + e + b"5" if len(e) < 4 else e + b"5"]
    for w in (b"\x85", b"\xa0"):  # Latin-1: the field is not valid UTF-8
        fs += [w + b"17" + w, w + b" 21\t" + w, b"\xff" + w + b"3", w + b"17\xff", b"\xc2" + w + b"17"]
    fs += [b"\xff\xe2\x80\x8017", b"\xc2\xa017\xff", b"17\xe2\x80", b"\xc0\xa017", b"\xed\xa0\x8017", b"\xf4\x90\x80\x8017",
           b"\xf0\x9d\x84\x9e17", b"\xe2\x80\x8b17", b"\x1c17", b"17\x1f", b"\x00\xe2\x80\x80"]
    fs += [b"+17", b"-0", b"+0", b"-", b"+", b"--1", b"+-1", b" -1 ", b"-17", b"-000000000001", b"\t-1\xe3\x80\x80",
           b"000000001750", b"777777777777", b"000000000001", b"17\x0034", b"\x0017", b"1 7", b"18", b"9", b"0o17", b"1_7",
           b"\x80" + bytes(7) + b"\x00\x00\x02\x00", b"\xff" * 12, bytes(12), b" " * 12, b"", b"\xef\xbb\xbf" * 4, b"0" * 11 + b" "]
    return [f[:12] + bytes(12 - len(f[:12])) for f in fs]


def size_archive(field):
    """One member with `field` as its size field, 40 content bytes, a second member, two zero blocks."""
    return header(b"sized", size_field=field) + b"\x01" * 40 + header(b"second", size=3) + body(b"abc") + bytes(1024)


# ------------------------------------------------------------------ the walk, restated on the host
def ref_walk(data):
    """The positions TarDecoder._decode walks through with storeData (tar.py: _host_walk over TarFile.read) -> (rc,
    [(header_off, header_len, content_off, content_len, size)])."""
    from archive_b200.tar import TarFile, _parse_int
    L, pos, out = len(data), 0, []
    while pos < L:
        if L - pos < 2 or (data[pos] == 0 and data[pos + 1] == 0):
            break
        hl = min(512, L - pos)
        h = data[pos:pos + hl]
        size = _parse_int(h[124:136])
        if size < 0:
            return E_THROW, out
        co = pos + hl
        cl = min(size, L - co)
        out.append((pos, hl, co, cl, size))
        pos = co + cl
        if TarFile.from_header(h).is_file and size > 0 and size % 512:
            pos = min(pos + 512 - size % 512, L)
    return OK, out


def oracle_ranges(data):
    """(status, [(content_off, content_len)]) of TarDecoder.files as oracle/tar.c reads them."""
    n, cap = C.c_size_t(), max(1024, len(data) // 512 + 2)
    arr = (ot._Member * cap)()
    strs, slen = C.POINTER(C.c_uint8)(), C.c_size_t()
    st = ot.L().orc_tar_decode(data, C.c_size_t(len(data)), 1, arr, C.c_size_t(cap), C.byref(n), C.byref(strs), C.byref(slen))
    ot.L().orc_free(strs)
    assert n.value <= cap
    return st, [(m.content_off, m.content_len) for m in arr[:n.value]]


# ------------------------------------------------------------------ the C call
def walk(D, archives, cap=None, seed=1, stream=True):
    """b200z_tar_walk_device over `archives`, placed in one device buffer in shuffled order at odd offsets with guarded
    gaps -> (r, n_total, [(rc, records, headers)]).  The guard around the archives must survive."""
    L = D.L
    rng = random.Random(seed)
    order = list(range(len(archives)))
    rng.shuffle(order)
    offs, at = [0] * len(archives), 0
    for i in order:
        at += rng.randrange(1, 40)
        offs[i] = at
        at += len(archives[i])
    img = np.full(at + 64, GUARD, np.uint8)
    for i, a in enumerate(archives):
        img[offs[i]:offs[i] + len(a)] = np.frombuffer(a, np.uint8)
    d = D.full(len(img))
    if D.torch is None:
        d[:] = img
    else:
        with D.torch.cuda.stream(D.stream):
            d.copy_(D.torch.from_numpy(img))
    n = len(archives)
    if cap is None:
        cap = sum(len(a) // 512 + 1 for a in archives)
    recs = np.zeros(max(cap, 1), MEMBER)
    hdrs = np.full(max(cap, 1) * 512, 0x77, np.uint8)
    first, count = (C.c_uint64 * max(n, 1))(*([99] * max(n, 1))), (C.c_uint64 * max(n, 1))(*([99] * max(n, 1)))
    rc, total = (C.c_int32 * max(n, 1))(*([99] * max(n, 1))), C.c_size_t(12345)
    r = L.b200z_tar_walk_device(D.ptr(d), a64(offs), a64([len(a) for a in archives]), n, recs.ctypes.data, hdrs.ctypes.data,
                                cap, first, count, rc, C.byref(total), D.handle() if stream else None)
    assert (D.get(d) == img).all()  # the archives are read, never written
    if r != OK:
        assert list(first)[:n] == [99] * n and list(count)[:n] == [99] * n and list(rc)[:n] == [99] * n
        assert (recs == np.zeros(1, MEMBER)).all() and (hdrs == 0x77).all()
        return r, total.value, None
    out = []
    for i in range(n):
        k0, k1 = first[i], first[i] + count[i]
        out.append((rc[i], recs[k0:k1], [hdrs[512 * k:512 * k + 512].tobytes() for k in range(k0, k1)]))
    return r, total.value, out


def check_walk(data, rc, recs, hdrs):
    """One archive's records against the restated walk, its headers against the bytes, its files against the oracle."""
    from archive_b200.tar import LONG_LINK, TarFile
    want_rc, want = ref_walk(data)
    assert rc == want_rc
    got = [(int(m["header_off"]), int(m["header_len"]), int(m["content_off"]), int(m["content_len"]), int(m["size"]))
           for m in recs]
    assert got == want
    for (ho, hl, *_), h in zip(want, hdrs):
        assert h == data[ho:ho + hl] + bytes(512 - hl)
    st, ranges = oracle_ranges(data)
    if rc == E_THROW:  # (the oracle also throws in the loop, at a PAX block that is not UTF-8)
        assert st == ot.THROW
    files = []
    for (ho, hl, co, cl, size), h in zip(want, hdrs):
        tf = TarFile.from_header(h[:hl])
        if tf.filename == LONG_LINK or tf.type_flag in ("g", "G", "x", "X"):
            continue
        files.append((co, cl))
    assert (files if st == ot.OK else files[:len(ranges)]) == ranges


@gpu
def test_walk_matches_the_host_walk_and_the_oracle(D):
    arch = corpus()
    names = sorted(arch)
    r, total, out = walk(D, [arch[k] for k in names])
    assert r == OK and total == sum(len(recs) for _, recs, _ in out)
    for k, (rc, recs, hdrs) in zip(names, out):
        check_walk(arch[k], rc, recs, hdrs)
    assert out[names.index("crafted/negative_size")][0] == E_THROW


@gpu
def test_size_field_table(D):
    fields = size_fields()
    archives = [size_archive(f) for f in fields]
    r, total, out = walk(D, archives, seed=3)
    assert r == OK
    from archive_b200.tar import _parse_int
    for f, a, (rc, recs, hdrs) in zip(fields, archives, out):
        check_walk(a, rc, recs, hdrs)
        if rc == OK:
            assert int(recs[0]["size"]) == _parse_int(f), f
    sizes = {f: _parse_int(f) for f in fields}
    # the table reaches every branch: trimmed forms, Latin-1, signs, rejects and a negative size
    assert sizes["\u3000".encode() + b"17" + "\u3000".encode() + bytes(4)] == 0o17
    assert sizes[b"777777777777"] == 0o777777777777 and sizes[b"17\x0034" + bytes(7)] == 0o17
    assert any(rc == E_THROW for rc, _, _ in out) and sum(rc == E_THROW for rc, _, _ in out) == sum(v < 0 for v in sizes.values())


@gpu
def test_empty_and_tiny_archives(D):
    archives = [b"", b"\x07", b"\0\0", b"a", b"ab", bytes(1024), header(b"x", size=1)[:200], b""]
    r, total, out = walk(D, archives)
    assert r == OK
    for a, (rc, recs, hdrs) in zip(archives, out):
        check_walk(a, rc, recs, hdrs)
    assert [len(recs) for _, recs, _ in out] == [0, 0, 0, 0, 1, 0, 1, 0]
    r, total, out = walk(D, [])
    assert r == OK and total == 0


def tiny_members(n):
    """n members of one byte each, every one its own name, then two zero blocks."""
    one = header(b"m", size=1)
    return b"".join(b"m%05d" % i + one[6:] + body(b"%c" % (65 + i % 26)) for i in range(n)) + bytes(1024)


@gpu
def test_many_tiny_members_bound_nospc_and_retry(D):
    data = tiny_members(20000)
    bound = len(data) // 512 + 1
    r, total, out = walk(D, [data], cap=bound)
    assert r == OK and total == 20000 and len(out[0][1]) == 20000
    check_walk(data, *out[0])
    r, total, out = walk(D, [data, tiny_members(10)], cap=19999)  # one short: nothing but n_total is written
    assert r == E_NOSPC and total == 20010 and out is None
    r, total2, out = walk(D, [data, tiny_members(10)], cap=total)
    assert r == OK and total2 == 20010 and [len(x[1]) for x in out] == [20000, 10]


def empty_members(n):
    """n members of size 0, one header each and no end marker: as dense as the record bound allows."""
    one = header(b"e", size=0)
    return b"".join(b"e%05d" % i + one[6:] for i in range(n))


def raw_walk(D, archives):
    """b200z_tar_walk_device over archives packed back to back -> (first, count, rc, records, headers) as returned."""
    data = b"".join(archives)
    d = D.full(len(data))
    if D.torch is None:
        d[:] = np.frombuffer(data, np.uint8)
    else:
        with D.torch.cuda.stream(D.stream):
            d.copy_(D.torch.frombuffer(bytearray(data), dtype=D.torch.uint8))
    n = len(archives)
    offs = list(np.cumsum([0] + [len(a) for a in archives])[:-1])
    cap = sum(len(a) // 512 + 1 for a in archives)
    recs, hdrs = np.zeros(cap, MEMBER), np.zeros(cap * 512, np.uint8)
    first, count, rc, total = (C.c_uint64 * n)(), (C.c_uint64 * n)(), (C.c_int32 * n)(), C.c_size_t()
    assert D.L.b200z_tar_walk_device(D.ptr(d), a64([int(o) for o in offs]), a64([len(a) for a in archives]), n, recs.ctypes.data,
                                     hdrs.ctypes.data, cap, first, count, rc, C.byref(total), D.handle()) == OK
    return list(first), list(count), list(rc), recs[:total.value], hdrs[:total.value * 512]


@gpu
def test_layout_is_archive_order_on_every_call(D):
    """first[] is the exclusive prefix sum of count[], and two calls give the same arrays, however the warps finish:
    300 archives of different lengths, a dense one whose records span several copy pieces, and empty ones."""
    rng = random.Random(9)
    archives = [tiny_members(rng.randrange(0, 40)) for _ in range(300)]
    archives[17] = empty_members(5000)  # 5000 records: 200 KB of records in 4 pieces
    archives[200] = b""
    a = raw_walk(D, archives)
    b = raw_walk(D, archives)
    first, count = a[0], a[1]
    assert first == [int(x) for x in np.cumsum([0] + count)[:-1]]
    assert count[17] == 5000 and count[200] == 0
    assert a[:3] == b[:3] and (a[3] == b[3]).all() and (a[4] == b[4]).all()
    for i, arch in enumerate(archives):
        recs = a[3][first[i]:first[i] + count[i]]
        hdrs = [a[4][512 * k:512 * k + 512].tobytes() for k in range(first[i], first[i] + count[i])]
        check_walk(arch, a[2][i], recs, hdrs)


def _launches(D, archives):
    before = D.L.b200z_launch_count()
    r, _, _ = walk(D, archives)
    assert r == OK
    return D.L.b200z_launch_count() - before


@gpu
def test_launch_count_does_not_grow(D):
    one = tiny_members(10)
    counts = [_launches(D, [one]), _launches(D, [one] * 1024), _launches(D, [tiny_members(20000)])]
    assert counts == [2, 2, 2]  # k_tar_walk and one k_copy_slots
    assert _launches(D, [b"", bytes(1024)]) == 1  # no member: nothing to gather


@gpu
def test_argument_errors_write_nothing(D):
    L = D.L
    data = tiny_members(3)
    d = D.full(len(data) + 64)
    if D.torch is None:
        d[:len(data)] = np.frombuffer(data, np.uint8)
    else:
        with D.torch.cuda.stream(D.stream):
            d[:len(data)].copy_(D.torch.frombuffer(bytearray(data), dtype=D.torch.uint8))

    def attempt(base, offs, lens, null=None, cap=16):
        n = len(lens)
        recs = np.zeros(max(cap, 1), MEMBER)
        hdrs = np.full(max(cap, 1) * 512, 0x77, np.uint8)
        arrs = [a64(offs), a64(lens), (C.c_uint64 * n)(*([9] * n)), (C.c_uint64 * n)(*([9] * n)), (C.c_int32 * n)(*([9] * n))]
        total = C.c_size_t(4321)
        args = [base, arrs[0], arrs[1], n, recs.ctypes.data, hdrs.ctypes.data, cap, arrs[2], arrs[3], arrs[4], C.byref(total),
                D.handle()]
        if null is not None:
            args[null] = None
        r = L.b200z_tar_walk_device(*args)
        if r == E_ARG:
            assert [list(a) for a in arrs[2:]] == [[9] * n] * 3 and total.value == 4321
            assert (recs == np.zeros(1, MEMBER)).all() and (hdrs == 0x77).all()
        return r

    lens = [len(data)]
    assert attempt(D.ptr(d), [0], lens) == OK
    for null in (1, 2, 4, 5, 7, 8, 9, 10):
        assert attempt(D.ptr(d), [0], lens, null=null) == E_ARG, null
    assert attempt(D.ptr(d), [0], lens, null=4, cap=0) == E_NOSPC  # cap 0 allows null record arrays
    assert attempt(D.ptr(d), [2**64 - 8], [16]) == E_ARG  # a wrapping range
    assert attempt(0, [0], lens) == E_ARG  # no base
    pinned = L.b200z_host_alloc(len(data))  # page-locked host memory: not device memory
    try:
        C.memmove(pinned, data, len(data))
        assert attempt(pinned, [0], lens) == E_ARG
        # the check covers every archive, not the base alone: a pinned archive reached by a pointer difference
        assert attempt(D.ptr(d), [0, (pinned - D.ptr(d)) % 2**64], [len(data), len(data)]) == E_ARG
    finally:
        L.b200z_host_free(pinned)
    assert attempt(0, [0, 0], [0, 0]) == OK  # empty archives: the base is never looked at
    assert attempt(None, [], []) == OK


@gpu
@needs_device
def test_pageable_host_archive_is_an_argument_error(D):
    data = np.frombuffer(tiny_members(3), np.uint8).copy()
    recs, hdrs = np.zeros(16, MEMBER), np.full(16 * 512, 0x77, np.uint8)
    first, count, rc, total = (C.c_uint64 * 1)(9), (C.c_uint64 * 1)(9), (C.c_int32 * 1)(9), C.c_size_t(4321)
    r = D.L.b200z_tar_walk_device(data.ctypes.data, a64([0]), a64([len(data)]), 1, recs.ctypes.data, hdrs.ctypes.data, 16, first,
                                  count, rc, C.byref(total), D.handle())
    assert r == E_ARG and (first[0], count[0], rc[0], total.value) == (9, 9, 9, 4321) and (hdrs == 0x77).all()


@gpu
@needs_device
def test_walk_runs_after_earlier_work_on_the_callers_stream(D):
    """The archive is written on the caller's stream behind a long kernel, right before the call: the walk sees it."""
    import torch
    data = tiny_members(50)
    s = torch.cuda.Stream()
    src = torch.frombuffer(bytearray(data), dtype=torch.uint8).to("cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        d = torch.zeros(len(data), dtype=torch.uint8, device="cuda")
        torch.cuda._sleep(200_000_000)  # ~0.1 s of spinning on s
        d.copy_(src)
    recs, hdrs = np.zeros(128, MEMBER), np.zeros(128 * 512, np.uint8)
    first, count, rc, total = (C.c_uint64 * 1)(), (C.c_uint64 * 1)(), (C.c_int32 * 1)(), C.c_size_t()
    assert D.L.b200z_tar_walk_device(d.data_ptr(), a64([0]), a64([len(data)]), 1, recs.ctypes.data, hdrs.ctypes.data, 128, first,
                                     count, rc, C.byref(total), s.cuda_stream) == OK
    assert (rc[0], count[0]) == (OK, 50)
    check_walk(data, rc[0], recs[:50], [hdrs[512 * k:512 * k + 512].tobytes() for k in range(50)])


# ------------------------------------------------------------------ the Python API
def _b(x):
    return x if x is None or isinstance(x, (bytes, bytearray)) else bytes(x.cpu().numpy())


def assert_same_decode(data, got, dec):
    """The device decode (`got`, the decoder `dec` that made it, or the DartRangeError it gave) equals the host TarDecoder
    member by member."""
    import archive_b200 as a
    host = a.TarDecoder()
    try:
        want = host.decode_bytes(data)
    except a.DartRangeError:
        assert isinstance(got, a.DartRangeError), "the host walk throws, the device walk does not"
        return
    assert not isinstance(got, Exception), got
    assert len(dec.files) == len(host.files)
    for t, h in zip(dec.files, host.files):
        assert (t.filename, t.name_of_linked_file, t.type_flag, t.mode, t.owner_id, t.group_id, t.file_size, t.last_mod_time,
                t.checksum, t.ustar_indicator, t.owner_user_name, t.owner_group_name, t.is_file, _b(t.raw_content)) == \
               (h.filename, h.name_of_linked_file, h.type_flag, h.mode, h.owner_id, h.group_id, h.file_size, h.last_mod_time,
                h.checksum, h.ustar_indicator, h.owner_user_name, h.owner_group_name, h.is_file, h.raw_content)
    assert len(got) == len(want)
    for f, w in zip(got, want):
        assert (f.name, f.symbolic_link, f.mode, f.owner_id, f.group_id, f.last_mod_time, f.is_file, f.size) == \
               (w.name, w.symbolic_link, w.mode, w.owner_id, w.group_id, w.last_mod_time, w.is_file, w.size)
        if f.is_file:
            assert f.content.is_cuda and f.content.dtype == _torch().uint8
            assert _b(f.content) == w.content
        else:
            assert f.content is None and w.content is None


def _torch():
    import torch
    return torch


@gpu
@needs_device
def test_decode_bytes_on_the_device_equals_the_host():
    import archive_b200 as a
    torch = _torch()
    cases = dict(corpus())
    cases.update({f"size/{i:02d}": size_archive(f) for i, f in enumerate(size_fields())})
    for name, data in sorted(cases.items()):
        dec = a.TarDecoder()
        try:
            got = dec.decode_bytes(data, device="cuda")
        except a.DartRangeError as e:
            got = e
        assert_same_decode(data, got, dec)
        dec2 = a.TarDecoder()  # a CUDA tensor is walked where it is
        t = torch.frombuffer(bytearray(data), dtype=torch.uint8).to("cuda") if data else torch.empty(0, dtype=torch.uint8, device="cuda")
        try:
            got2 = dec2.decode_bytes(t, device="cuda")
        except a.DartRangeError as e:
            got2 = e
        assert_same_decode(data, got2, dec2)
    seen, host_seen = [], []
    a.TarDecoder().decode_bytes(generated(tarfile.GNU_FORMAT), device="cuda", callback=seen.append)
    a.TarDecoder().decode_bytes(generated(tarfile.GNU_FORMAT), callback=host_seen.append)
    assert [f.name for f in seen] == [f.name for f in host_seen] and len(seen) > 14
    dec = a.TarDecoder()  # anything bytes() takes, as on the host path
    assert_same_decode(bytes([1, 2, 3]), dec.decode_bytes([1, 2, 3], device="cuda"), dec)
    with pytest.raises(ValueError):
        a.TarDecoder().decode_bytes(CRAFTED["dir_with_size"], device="cuda", store_data=False)
    with pytest.raises(ValueError):
        a.TarDecoder().decode_bytes(CRAFTED["dir_with_size"], device="cpu")


def _compress(codec, t):
    if codec == "gzip":
        return orc.gzip_encode(t, 6, mtime=0)[1]
    if codec == "bzip2":
        return orc.bzip2_encode(t)[1]
    return lzma.compress(t, format=lzma.FORMAT_XZ, check=lzma.CHECK_CRC64)


def batch_shards(codec):
    """64 shards: generated GNU shards (LongLink names), PAX, crafted archives, duplicates, a damaged shard (partial
    output walked) and a shard whose walk throws."""
    tars = shard_tars(52, seed=5) + [generated(tarfile.PAX_FORMAT), CRAFTED["pax_path_linkpath"], CRAFTED["dir_with_size"],
                                     CRAFTED["longlink_K_sets_name"], CRAFTED["negative_size"], CRAFTED["pax_not_utf8"]]
    shards = [t if codec is None else _compress(codec, t) for t in tars]
    shards += [shards[3], shards[3], shards[-2]]  # duplicates
    damaged = bytearray(shards[7])
    if codec is None:
        damaged = damaged[:700]
    else:
        damaged = damaged[:len(damaged) * 2 // 3]
    shards.append(bytes(damaged))
    shards += [shards[0], shards[10]]
    assert len(shards) == 64
    return shards


def assert_same_batch(got, want, decoded):
    assert len(got) == len(want)
    import archive_b200 as a
    for (rc, g), (hrc, w), data in zip(got, want, decoded):
        assert rc == hrc
        if isinstance(w, a.DartRangeError):
            assert isinstance(g, a.DartRangeError)
            continue
        assert not isinstance(g, Exception)
        assert len(g) == len(w)
        for f, h in zip(g, w):
            assert (f.name, f.symbolic_link, f.mode, f.owner_id, f.group_id, f.last_mod_time, f.is_file, f.size) == \
                   (h.name, h.symbolic_link, h.mode, h.owner_id, h.group_id, h.last_mod_time, h.is_file, h.size)
            assert _b(f.content) == h.content


@gpu
@needs_device
@pytest.mark.parametrize("codec", ["gzip", "bzip2", "xz", None])
def test_tar_decode_batch_equals_the_host_batch(codec):
    import archive_b200 as a
    torch = _torch()
    shards = batch_shards(codec)
    want = a.tar_decode_batch(shards, compression=codec, verify=True)
    if codec is None:
        decoded = shards
    else:
        fn = {"gzip": a.gzip_decode_batch, "bzip2": a.bzip2_decode_batch, "xz": a.xz_decode_batch}[codec]
        decoded = [t for _, t in fn(shards, verify=True)]
        assert any(rc != OK for rc, _ in want)  # the damaged shard
    for (rc, w), t in zip(want, decoded):  # the host batch is TarDecoder on each decoded shard
        try:
            ref = a.TarDecoder().decode_bytes(t)
        except a.DartRangeError:
            assert isinstance(w, a.DartRangeError)
            continue
        assert [(f.name, f.content) for f in w] == [(f.name, f.content) for f in ref]
    assert sum(isinstance(w, a.DartRangeError) for _, w in want) >= 3
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)  # work already queued on the current stream
        got = a.tar_decode_batch(shards, compression=codec, verify=True, device="cuda")
    assert_same_batch(got, want, decoded)
    assert a.tar_decode_batch([], compression=codec, device="cuda") == []


@gpu
@needs_device
def test_tar_decode_batch_of_cuda_tensor_shards():
    """Plain shards already on the device, each its own allocation, mixed with host shards: walked where they are."""
    import archive_b200 as a
    torch = _torch()
    shards = batch_shards(None)
    want = a.tar_decode_batch(shards)
    tens = [torch.frombuffer(bytearray(s), dtype=torch.uint8).to("cuda") if s else torch.empty(0, dtype=torch.uint8, device="cuda")
            for s in shards]
    mixed = [t if i % 3 else s for i, (s, t) in enumerate(zip(shards, tens))]
    for inp in (tens, mixed):
        got = a.tar_decode_batch(inp, device="cuda")
        assert_same_batch(got, want, shards)
    for i, (rc, arch) in enumerate(a.tar_decode_batch(tens, device="cuda")):
        if not isinstance(arch, Exception):
            for f in arch:
                if f.is_file and f.content.numel():  # a view into the shard's own tensor, not a copy
                    assert tens[i].data_ptr() <= f.content.data_ptr() < tens[i].data_ptr() + tens[i].numel()
    with pytest.raises(ValueError):
        a.tar_decode_batch([tens[0].to(torch.int32)], device="cuda")
    with pytest.raises(ValueError):
        a.tar_decode_batch(shards[:1], compression="zstd")


@gpu
@needs_device
def test_tar_decode_batch_many_tiny_members():
    """A shard of 20 000 one-byte members is past the first records guess: the call retries once, sized exactly."""
    import archive_b200 as a
    data = tiny_members(20000)
    got = a.tar_decode_batch([data, tiny_members(5)], device="cuda")
    want = a.tar_decode_batch([data, tiny_members(5)])
    assert_same_batch(got, want, [data, tiny_members(5)])
    assert len(got[0][1]) == 20000 and got[0][1].files[-1].content.numel() == 1


# ------------------------------------------------------------------ without a device
def test_walk_reports_no_device_and_writes_nothing():
    """In a process that has no device (b200z_init never succeeds), b200z_tar_walk_device returns B200Z_E_NODEVICE and
    writes nothing."""
    prog = r"""
import ctypes as C, sys
sys.path.insert(0, sys.argv[1])
from archive_b200 import _ffi
L = _ffi.lib()
assert L.b200z_init(0, 0) == _ffi.E_NODEVICE
data = (C.c_uint8 * 1024)()
a = lambda *v: (C.c_uint64 * len(v))(*v)
recs = (_ffi.TarMember * 4)()
hdrs = (C.c_uint8 * 2048)(*([0xA5] * 2048))
first, count, rc, total = a(7, 7), a(7, 7), (C.c_int32 * 2)(7, 7), C.c_size_t(7)
assert L.b200z_tar_walk_device(data, a(0, 512), a(512, 512), 2, recs, hdrs, 4, first, count, rc, C.byref(total), None) == _ffi.E_NODEVICE
assert list(first) == [7, 7] and list(count) == [7, 7] and list(rc) == [7, 7] and total.value == 7
assert bytes(hdrs) == b"\xa5" * 2048 and all(r.header_off == 0 and r.size == 0 for r in recs)
print("ok")
"""
    env = {k: v for k, v in os.environ.items() if k not in ("B200Z_LIB", "B200Z_EMU_TESTS")}
    env["CUDA_VISIBLE_DEVICES"] = ""
    r = subprocess.run([sys.executable, "-c", prog, ROOT], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stdout + r.stderr
