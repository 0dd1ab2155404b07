"""b200z_zip_extract_to_device: ZIP members extracted straight into device memory, with each member's CRC-32 computed there.

Every member must come out of the device call exactly as it comes out of b200z_zip_extract_password with the same
arguments (status, out_len and the bytes d_out[out_off .. + min(out_len, room)) unless the member ran out of room), and as the oracle's restatement of the
reference gives it; nothing outside the slots may be written (every such byte keeps the guard value 0xA5), whatever the
slots' order, gaps and alignment; crc32[i] is zlib.crc32 of the delivered bytes.  The same tests run on an H100 (torch
CUDA tensors, on a side stream) and on the emulated library with B200Z_EMU_TESTS=1 (numpy arrays as device memory; its
ASan build then checks that nothing outside the documented buffers is read or written)."""
import bz2
import ctypes as C
import glob
import hashlib
import json
import os
import random
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest

import oracle_lib as orc
import zip_chunked_cases as zcc
import zip_crypt_build as zcb
from archive_b200._ffi import ZipEntry

EMU = os.environ.get("B200Z_EMU_TESTS") == "1"
GOLD = os.path.join(os.path.dirname(__file__), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, E_NODEVICE, E_ARG = 0, -1, -2
U_DONE, U_NOSPC = 0, -2
ZIP_ENCRYPTED = -20
WEB_EOS, NO_SPLIT = 1, 2
GUARD = 0xA5
gpu = pytest.mark.gpu
needs_device = pytest.mark.needs_device


class Device:
    """Device memory of the library's device: torch CUDA tensors used on a side stream on the GPU; numpy arrays on the
    emulated library, whose device memory is host memory and whose launches finish before they return."""

    def __init__(self):
        from archive_b200 import _ffi
        self.L = _ffi.ensure_init()
        self.L.b200z_debug_zip_out_bytes.restype = C.c_uint64
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
    return Device()


def a64(v):
    return (C.c_uint64 * max(len(v), 1))(*v)


def entries(L, data):
    cnt = C.c_size_t(0)
    assert L.b200z_zip_list(data, len(data), None, 0, C.byref(cnt)) == OK
    ents = (ZipEntry * max(1, cnt.value))()
    assert L.b200z_zip_list(data, len(data), ents, cnt.value, C.byref(cnt)) == OK
    return ents, cnt.value


def rooms_of(ents, n):
    """the first rooms ZipDecoder gives (archive_b200/zip.py)"""
    return [max(int(ents[i].hint_uncomp_size), int(ents[i].uncomp_size), 1) if ents[i].has_data else 0 for i in range(n)]


def layout(rooms, mode, rng):
    """out_off of every slot: 'packed' back to back in order; 'scattered' in reverse order, with odd gaps"""
    offs, pos = [0] * len(rooms), 0
    order = range(len(rooms)) if mode == "packed" else reversed(range(len(rooms)))
    for i in order:
        if mode != "packed":
            pos += rng.randrange(1, 40) | 1
        offs[i] = pos
        pos += rooms[i]
    return offs, pos + (0 if mode == "packed" else 23)


def pair(D, data, rooms=None, flags=0, password=None, mode="scattered", lead=13, seed=1, shift=0, with_crc=True):
    """The host call and the device call on the same arguments -> [(status, out_len, bytes, crc)], after checking that both
    agree, that the device call wrote nothing outside its slots, and that every CRC is that of the delivered bytes.  The
    device slots start `lead` bytes into a larger allocation, and `shift` bytes behind the base the call is given."""
    L = D.L
    ents, n = entries(L, data)
    rooms = rooms_of(ents, n) if rooms is None else rooms
    offs, extent = layout(rooms, mode, random.Random(seed))
    offs = [o + shift for o in offs]
    extent += shift
    pw, pwl = (password, len(password)) if password is not None else (None, 0)
    h_out = (C.c_uint8 * max(extent, 1))()
    h_len, h_st = (C.c_uint64 * n)(), (C.c_int32 * n)()
    oo, rr = a64(offs), a64(rooms)
    r = L.b200z_zip_extract_password(data, len(data), ents, n, C.addressof(h_out), max(extent, 1), oo, rr, h_len, h_st, flags,
                                     pw, pwl)
    assert r == OK, L.b200z_last_error()
    host_out_bytes = L.b200z_debug_zip_out_bytes()
    d = D.full(lead + extent + 29)
    d_len, d_st, crc = (C.c_uint64 * n)(), (C.c_int32 * n)(), (C.c_uint32 * n)()
    r = L.b200z_zip_extract_to_device(data, len(data), ents, n, D.ptr(d) + lead, max(extent, 1), oo, rr, d_len, d_st,
                                      crc if with_crc else None, flags, pw, pwl, D.handle())
    assert r == OK, L.b200z_last_error()
    assert L.b200z_debug_zip_out_bytes() == host_out_bytes
    got = D.get(d)
    hb = np.frombuffer(h_out, np.uint8)
    inside = np.zeros(len(got), bool)
    res = []
    for i in range(n):
        assert (d_st[i], d_len[i]) == (h_st[i], h_len[i]), (i, d_st[i], d_len[i], h_st[i], h_len[i])
        o = offs[i]
        inside[lead + o:lead + o + rooms[i]] = True
        k = min(d_len[i], rooms[i])
        b = bytes(got[lead + o:lead + o + k])
        if d_st[i] != U_NOSPC:  # (the slot of a member out of room holds unspecified bytes, on the host as well)
            assert b == bytes(hb[o:o + k]), i
        if d_st[i] == ZIP_ENCRYPTED:  # not decoded: the slot is untouched
            assert (got[lead + o:lead + o + rooms[i]] == GUARD).all(), i
        if with_crc:
            assert crc[i] == (0 if d_st[i] == U_NOSPC else zlib.crc32(b)), (i, crc[i])
        res.append((d_st[i], d_len[i], b, crc[i] if with_crc else None))
    assert (got[~inside] == GUARD).all(), "bytes outside the slots were written"
    return res


def text(n, stream=7):
    from archive_b200 import synth
    return synth.text(n, stream=stream).tobytes()


# ------------------------------------------------------------------ fixtures
def _fixtures():
    out = [(os.path.basename(p), None) for p in sorted(glob.glob(os.path.join(GOLD, "zip", "*.zip")))]
    man = json.load(open(os.path.join(GOLD, "zip_crypt", "manifest.json")))
    for name, a in sorted(man["archives"].items()):
        out += [("zip_crypt/" + name, None), ("zip_crypt/" + name, a["password"])]
    return out


@gpu
@pytest.mark.parametrize("name,password", _fixtures())
def test_fixtures_equal_the_host_call_and_the_oracle(D, name, password):
    path = os.path.join(GOLD, name if "/" in name else os.path.join("zip", name))
    data = open(path, "rb").read()
    pw = None if password is None else password.encode()
    ents, n = entries(D.L, data)
    for mode in ("scattered", "packed"):
        got = pair(D, data, password=pw, mode=mode)
        for i in range(n):
            e = ents[i]
            st, _, b, crc = got[i]
            if not e.has_data or st != U_DONE:
                continue
            if not (e.flags & 1):
                assert b == orc.zip_member(data, e)[1], (name, i)
            if e.crc32 or not (e.flags & 1):  # (AE-2 AES members store no CRC)
                assert crc == e.crc32, (name, i)  # what ZipFile.verifyCrc32 compares
    if password is not None:
        man = json.load(open(os.path.join(GOLD, "zip_crypt", "manifest.json")))
        want = zcb.oracle_members(data, pw)
        for i in range(n):
            assert (got[i][0], got[i][2]) == (want[i][0], want[i][1]) or got[i][0] != U_DONE, (name, i)
            nm = data[ents[i].name_off:ents[i].name_off + ents[i].name_len].decode()
            if nm in man["plaintext"]:
                assert hashlib.sha256(got[i][2]).hexdigest() == man["plaintext"][nm]["sha256"], (name, nm)
    else:
        man = json.load(open(os.path.join(GOLD, "zip", "manifest.json"))).get(name, {})
        sha = {w["name"]: w["sha256"] for w in man.get("entries") or [] if w.get("sha256")}
        for i in range(n):
            nm = data[ents[i].name_off:ents[i].name_off + ents[i].name_len].decode("utf-8", "replace")
            if nm in sha and got[i][0] == U_DONE:
                assert hashlib.sha256(got[i][2]).hexdigest() == sha[nm], (name, nm)


# ------------------------------------------------------------------ a synthetic mix of every member kind
def _mix(t):
    pw = b"s3cret"
    M = zcb.Member
    s = t[:20000]
    members = [
        M("stored.bin", s[:7000], method=0, crypt=None),
        M("small.txt", s, crypt=None),
        M("flushed.txt", t[:1 << 20], crypt=None, flush_every=64 << 10),  # full-flush points: the split path
        M("k12.txt", t[1 << 20:(1 << 20) + (3 << 19)], crypt=None),  # no flush points: K12 with the lowered threshold
        M("s.bz2", s, method=12, crypt=None),
        M("unknown.bin", s[:3000], method=5, crypt=None),  # read as stored
        M("empty.txt", b"", crypt=None),
        M("empty_stored", b"", method=0, crypt=None),
        M("dir/", is_dir=True, crypt=None),
        M("zc.txt", s[:9000], crypt="zipcrypto"),
        M("aes.txt", s[:11000], crypt="aes"),
        M("aes128.bin", s[:5000], method=0, crypt="aes", strength=1),
        M("aes_bz2", s[:6000], method=12, crypt="aes"),
        M("bad_mac.txt", s[:4000], crypt="aes", bad_mac=True),
        M("short_aes", s[:100], crypt="aes", truncate=20),
        M("other_pw.txt", s[:3000], crypt="aes", password=b"other"),
        M("tail.txt", s[:1500], crypt=None),
    ]
    data = bytearray(zcb.build(members, pw))
    # one more member whose local header is gone (has_data == 0): the stored member's signature is broken
    p = data.find(b"PK\x03\x04")
    data[p:p + 4] = b"PK\x03\x05"
    return bytes(data), pw


@pytest.fixture(scope="module")
def mix():
    return _mix(text(3 << 20, stream=11))


@pytest.fixture
def k12_low(D):
    D.L.b200z_debug_inflate_chunked_set(C.c_ulonglong(256 << 10), C.c_ulonglong(0))
    yield
    D.L.b200z_debug_inflate_chunked_set(C.c_ulonglong(0), C.c_ulonglong(0))


@gpu
@pytest.mark.parametrize("flags", [0, WEB_EOS, NO_SPLIT])
def test_synthetic_mix_of_every_member_kind(D, mix, k12_low, flags):
    data, pw = mix
    ents, n = entries(D.L, data)
    assert ents[0].has_data == 0
    rooms = rooms_of(ents, n)
    short = [r - 1 if r > 1 and i % 3 == 1 else r for i, r in enumerate(rooms)]  # every third room one byte short
    for password in (None, pw):
        assert any(g[0] == U_NOSPC for g in pair(D, data, short, flags, password))
        got = pair(D, data, rooms, flags, password)
        if password is not None:
            want = zcb.oracle_members(data, password, web_eos=bool(flags & WEB_EOS))
            for i, (st, ln, b, crc) in enumerate(got):
                if st == U_DONE:
                    assert b == want[i][1], i
    # a NULL crc32 changes nothing else
    assert [g[:3] for g in pair(D, data, rooms, flags, pw, with_crc=False)] == [g[:3] for g in got]
    # size fields that lie: rooms of one byte
    pair(D, zcc.zero_sizes(data), None, flags, pw)


@gpu
def test_b200z_zip_chunks_gives_the_same_results(D, mix, k12_low, monkeypatch):
    data, pw = mix
    one = pair(D, data, password=pw)
    monkeypatch.setenv("B200Z_ZIP_CHUNKS", "8")
    assert pair(D, data, password=pw) == one


@gpu
def test_layouts_packed_and_at_every_lead(D):
    t = text(400000, stream=3)
    data = zcc.build([zcc.deflated(f"m{i}", t[i * 1000:i * 1000 + 70000 + 13 * i]) for i in range(12)] +
                     [(f"s{i}", t[i:i + 70001 + i], 0, zlib.crc32(t[i:i + 70001 + i]), 70001 + i) for i in range(4)])
    for lead in range(16):
        got = pair(D, data, mode="packed" if lead % 2 else "scattered", lead=lead, seed=lead)
        assert all(g[0] == U_DONE for g in got)


@gpu
@needs_device
def test_slots_deep_inside_a_large_allocation(D):
    """Slots 1 GiB into the buffer: the library's own output buffer is sized by the slots' span, not their end."""
    t = text(1 << 20, stream=9)
    data = zcc.build([zcc.deflated(f"m{i}", t[i << 16:(i + 2) << 16]) for i in range(8)])
    got = pair(D, data, shift=1 << 30)
    assert all(g[0] == U_DONE for g in got)
    span = sum(len(g[2]) for g in got) + 8 * 40 + 23
    assert D.L.b200z_debug_zip_out_bytes() <= span + 64


# ------------------------------------------------------------------ launches
@gpu
def test_launch_count_does_not_grow_with_members(D):
    s = text(300000, stream=13)
    diffs = []
    for m in (16, 1024):
        mem = []
        for i in range(m):
            c = s[(i * 211) % 200000:][:100 + i % 300]
            mem.append(zcc.deflated(f"d{i}", c) if i % 2 else (f"s{i}", c, 0, zlib.crc32(c), len(c)))
        mem += [(f"b{i}", bz2.compress(s[:5000 * (i + 1)], 9), 12, zlib.crc32(s[:5000 * (i + 1)]), 5000 * (i + 1)) for i in range(2)]
        data = zcc.build(mem)
        L = D.L
        ents, n = entries(L, data)
        rooms = rooms_of(ents, n)
        offs, extent = layout(rooms, "packed", random.Random(0))
        h = (C.c_uint8 * extent)()
        d = D.full(extent)
        ol, st, crc = (C.c_uint64 * n)(), (C.c_int32 * n)(), (C.c_uint32 * n)()
        c0 = L.b200z_launch_count()
        assert L.b200z_zip_extract(data, len(data), ents, n, C.addressof(h), extent, a64(offs), a64(rooms), ol, st, 0) == OK
        c1 = L.b200z_launch_count()
        assert L.b200z_zip_extract_to_device(data, len(data), ents, n, D.ptr(d), extent, a64(offs), a64(rooms), ol, st, crc, 0,
                                             None, 0, D.handle()) == OK
        c2 = L.b200z_launch_count()
        assert all(x == U_DONE for x in st)
        diffs.append((c2 - c1) - (c1 - c0))
    assert diffs[0] == diffs[1] and diffs[0] >= 2, diffs  # k_copy_slots, BZip2's delivery, one CRC launch


# ------------------------------------------------------------------ argument errors and ordering
@gpu
def test_argument_errors_write_nothing(D):
    L = D.L
    t = text(50000, stream=5)
    data = zcc.build([zcc.deflated("a", t[:20000]), ("b", t[:3000], 0, zlib.crc32(t[:3000]), 3000)])
    ents, n = entries(L, data)
    rooms = rooms_of(ents, n)
    offs = [0, rooms[0]]
    cap = sum(rooms)
    d = D.full(cap + 64)

    def attempt(base=None, null=None, offs_=offs, cap_=cap):
        ol, st, crc = (C.c_uint64 * n)(*[77] * n), (C.c_int32 * n)(*[77] * n), (C.c_uint32 * n)(*[77] * n)
        arrs = [ents, a64(offs_), a64(rooms), ol, st]
        if null is not None:
            arrs[null] = None
        r = L.b200z_zip_extract_to_device(data, len(data), arrs[0], n, D.ptr(d) if base is None else base, cap_, arrs[1],
                                          arrs[2], arrs[3], arrs[4], crc, 0, None, 0, D.handle())
        if r != OK:
            assert list(ol) == [77] * n and list(st) == [77] * n and list(crc) == [77] * n
        return r

    for null in range(5):
        assert attempt(null=null) == E_ARG
    assert attempt(offs_=[0, cap - rooms[1] + 1]) == E_ARG  # the second slot ends past out_cap
    assert attempt(cap_=cap - 1) == E_ARG
    assert attempt(base=0) == E_ARG
    pinned = L.b200z_host_alloc(cap + 64)  # host memory, page-locked: not device memory
    try:
        C.memset(pinned, GUARD, cap + 64)
        assert attempt(base=pinned) == E_ARG
        assert C.string_at(pinned, cap + 64) == bytes([GUARD]) * (cap + 64)
    finally:
        L.b200z_host_free(pinned)
    assert (D.get(d) == GUARD).all()
    assert attempt() == OK


@gpu
@needs_device
def test_extracted_bytes_land_after_earlier_work_on_the_callers_stream(D):
    import torch
    L = D.L
    t = text(300000, stream=17)
    data = zcc.build([zcc.deflated(f"m{i}", t[i * 30000:(i + 1) * 30000]) for i in range(8)])
    ents, n = entries(L, data)
    rooms = rooms_of(ents, n)
    offs, extent = layout(rooms, "packed", random.Random(1))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d = torch.zeros(extent, dtype=torch.uint8, device="cuda")
        torch.cuda._sleep(200_000_000)  # ~0.1 s of spinning on s
        d.fill_(0x5A)
    ol, st = (C.c_uint64 * n)(), (C.c_int32 * n)()
    assert L.b200z_zip_extract_to_device(data, len(data), ents, n, d.data_ptr(), extent, a64(offs), a64(rooms), ol, st, None,
                                         0, None, 0, s.cuda_stream) == OK
    got = d.cpu().numpy()
    for i in range(n):
        assert st[i] == U_DONE and bytes(got[offs[i]:offs[i] + ol[i]]) == t[i * 30000:(i + 1) * 30000], i


# ------------------------------------------------------------------ the Python API
@gpu
@needs_device
def test_python_decode_bytes_to_a_cuda_device(mix, k12_low):
    import torch
    import archive_b200 as a
    from archive_b200.zip import ArchiveException
    cases = [(open(p, "rb").read(), None) for p in sorted(glob.glob(os.path.join(GOLD, "zip", "*.zip")))]
    man = json.load(open(os.path.join(GOLD, "zip_crypt", "manifest.json")))
    cases += [(open(os.path.join(GOLD, "zip_crypt", nm), "rb").read(), v["password"]) for nm, v in sorted(man["archives"].items())]
    data, pw = mix
    cases += [(data, pw), (zcc.zero_sizes(data), pw)]  # the second: every room starts at one byte and grows
    side = torch.cuda.Stream()
    for data, password in cases:
        want = a.ZipDecoder().decode_bytes(data, password=password)
        with torch.cuda.stream(side):
            torch.cuda._sleep(20_000_000)
            got = a.ZipDecoder().decode_bytes(data, password=password, device="cuda")
        assert [f.name for f in got] == [f.name for f in want]
        for g, w in zip(got, want):
            assert (g.mode, g.symbolic_link, g.crc32, g.status, g.is_file) == (w.mode, w.symbolic_link, w.crc32, w.status, w.is_file)
            if not w.is_file:
                continue
            try:
                wb = w.read_bytes()
            except ArchiveException:
                with pytest.raises(ArchiveException):
                    g.read_bytes()
                with pytest.raises(ArchiveException):
                    g.verify_crc32()
                continue
            gb = g.read_bytes()
            assert gb.is_cuda and gb.dtype == torch.uint8 and bytes(gb.cpu().numpy()) == wb, g.name
            assert g.verify_crc32() == w.verify_crc32() == (zlib.crc32(wb) == w.crc32), g.name
    sym = a.ZipDecoder().decode_bytes(open(os.path.join(GOLD, "zip", "symlink.zip"), "rb").read(), device="cuda")
    assert sym.files[0].symbolic_link == "../target"
    with pytest.raises(ArchiveException):  # a symlink that does not decrypt throws during the walk, as on the host
        a.ZipDecoder().decode_bytes(zcb.build([zcb.Member("l", b"../t", symlink=True)], b"pw"), password="wrong", device="cuda")
    with pytest.raises(ValueError):
        a.ZipDecoder().decode_bytes(cases[0][0], device="cpu")
    with pytest.raises(ValueError):
        a.ZipDecoder().decode_bytes(cases[0][0], device=torch.device("cuda", torch.cuda.device_count() + 3))


# ------------------------------------------------------------------ without a device
def test_entry_point_reports_no_device_and_writes_nothing():
    """In a process that has no device (b200z_init never succeeds), b200z_zip_extract_to_device returns B200Z_E_NODEVICE
    and writes nothing."""
    prog = r"""
import ctypes as C, sys
sys.path.insert(0, sys.argv[1])
from archive_b200 import _ffi
L = _ffi.lib()
assert L.b200z_init(0, 0) == _ffi.E_NODEVICE
ents = (_ffi.ZipEntry * 2)()
ents[0].has_data = ents[1].has_data = 1
data = (C.c_uint8 * 16)()
a = lambda *v: (C.c_uint64 * len(v))(*v)
out = (C.c_uint8 * 64)(*([0xA5] * 64))
ol, st, crc = a(7, 7), (C.c_int32 * 2)(7, 7), (C.c_uint32 * 2)(7, 7)
r = L.b200z_zip_extract_to_device(data, 16, ents, 2, out, 64, a(0, 32), a(32, 32), ol, st, crc, 0, None, 0, None)
assert r == _ffi.E_NODEVICE, r
assert list(ol) == [7, 7] and list(st) == [7, 7] and list(crc) == [7, 7] and bytes(out) == b"\xa5" * 64
print("ok")
"""
    env = {k: v for k, v in os.environ.items() if k not in ("B200Z_LIB", "B200Z_EMU_TESTS")}
    env["CUDA_VISIBLE_DEVICES"] = ""
    r = subprocess.run([sys.executable, "-c", prog, ROOT], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stdout + r.stderr
