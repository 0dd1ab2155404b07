"""b200z_inflate_batch_device against the oracle, on both inflate kernels (k_inflate_fast, and the exact pair
k_inflate_decode + k_inflate_expand that B200Z_FAST=0 leaves everything to).

The device entry point differs from b200z_inflate_batch in what the caller owns: the input buffer (no padding beyond
the documented round_up(max(in_off + in_len), 16)), the output layout (any order, gaps, unaligned slots, a base inside
a larger allocation), the workspace (sized by b200z_inflate_workspace_bytes, uninitialised, reused) and the stream.
These tests vary each of them.  The same tests run on an H100 (torch CUDA tensors, on a side stream) and on the
emulated library with B200Z_EMU_TESTS=1 (numpy arrays as device memory; its ASan build then checks that no kernel
reads or writes outside the documented buffers).  Bit-exact: byte/integer work has no tolerance."""
import os
import random
import zlib

import numpy as np
import pytest

import oracle_lib as orc

pytestmark = pytest.mark.gpu

EMU = os.environ.get("B200Z_EMU_TESTS") == "1"
E_ARG = -2
U_NOSPC = -2
GUARD = 0xA5
# k_inflate_fast's eligibility limits (inflate_fast.cuh, namespace fp)
MIN_IN, IN_CAP, WIN = 192, 30720, 65536


# ------------------------------------------------------------------ device buffers, on either tier
class Backend:
    """Where a batch's "device" buffers live: torch CUDA tensors, used on a side stream, on the GPU; numpy arrays on
    the emulated library, whose device memory is host memory and whose launches finish before they return."""

    _TORCH = {np.dtype(np.uint8): "uint8", np.dtype(np.int32): "int32", np.dtype(np.uint32): "int32",
              np.dtype(np.uint64): "int64"}

    def __init__(self):
        from archive_b200 import _ffi
        self.ffi = _ffi
        self.L = _ffi.ensure_init()
        self.torch = None
        self.stream = None
        if not EMU:
            import torch
            self.torch = torch
            self.stream = torch.cuda.Stream()

    def put(self, a, stream=None):
        """An exact-size device copy of the numpy array `a` (16-byte aligned)."""
        a = np.ascontiguousarray(a)
        if self.torch is None:
            d = self._np_aligned(a.nbytes).view(a.dtype)
            d[...] = a.reshape(-1)
            return d
        if not a.flags.writeable:
            a = a.copy()  # (torch does not take read-only arrays)
        t = self.torch
        with t.cuda.stream(stream or self.stream):
            d = t.from_numpy(a.reshape(-1).view(getattr(np, self._TORCH[a.dtype]))).to("cuda")
        return (d, a.dtype)

    def full(self, n, dtype, fill, stream=None):
        """n elements of `dtype`; fill None = uninitialised."""
        dtype = np.dtype(dtype)
        if self.torch is None:
            d = self._np_aligned(n * dtype.itemsize).view(dtype)
            if fill is not None:
                d[...] = np.array(fill).astype(dtype)
            return d
        t = self.torch
        with t.cuda.stream(stream or self.stream):
            d = t.empty(n, dtype=getattr(t, self._TORCH[dtype]), device="cuda")
            if fill is not None:
                d.fill_(int(np.array(fill).astype(dtype).view(getattr(np, self._TORCH[dtype]))))
        return (d, dtype)

    def ptr(self, d):
        return d.ctypes.data if self.torch is None else d[0].data_ptr()

    def get(self, d):
        """Host copy.  The caller has synchronised the stream the batch ran on."""
        if self.torch is None:
            return d.copy()
        return d[0].cpu().numpy().view(d[1])

    def handle(self, stream=None):
        if self.torch is None:
            return None
        return (stream or self.stream).cuda_stream

    def sync(self, stream=None):
        if self.torch is not None:
            (stream or self.stream).synchronize()

    @staticmethod
    def _np_aligned(nbytes):
        a = np.empty(max(nbytes, 1), np.uint8)
        if a.ctypes.data % 16:  # (allocators on x86-64 return 16-byte aligned blocks; otherwise give up the exact end)
            a = np.empty(nbytes + 16, np.uint8)
            k = (-a.ctypes.data) % 16
            a = a[k:k + max(nbytes, 1)]
        return a[:nbytes] if nbytes else a[:0]


@pytest.fixture(scope="module")
def B():
    return Backend()


# ------------------------------------------------------------------ a batch, its call and its results
def pad16(x):
    return (x + 15) & ~15


class Batch:
    """Input units packed into one buffer that ends exactly at the documented minimum, plus an output layout."""

    def __init__(self, units, caps, in_off=None, out_off=None, extent=None, rng=None, leads=None, garbage=True):
        rng = rng or random.Random(1)
        n = len(units)
        self.units = units
        self.caps = np.array(caps, dtype=np.uint32)
        if in_off is None:
            blob = bytearray()
            in_off = np.zeros(n, dtype=np.uint64)
            for i, u in enumerate(units):
                lead = leads[i] if leads is not None else rng.randrange(16)
                gap = pad16(len(blob)) + lead - len(blob)
                blob += bytes(rng.getrandbits(8) for _ in range(gap)) if garbage else bytes(gap)
                in_off[i] = len(blob)
                blob += u
            blob += bytes(rng.getrandbits(8) for _ in range(pad16(len(blob)) - len(blob)))
            self.blob = bytes(blob)
        else:
            self.blob = None  # set by the caller
        self.in_off = np.asarray(in_off, dtype=np.uint64)
        self.in_len = np.array([len(u) for u in units], dtype=np.uint32)
        if out_off is None:
            out_off = np.zeros(n, dtype=np.uint64)
            out_off[1:] = np.cumsum(self.caps.astype(np.uint64))[:-1]
        self.out_off = np.asarray(out_off, dtype=np.uint64)
        ends = self.out_off + self.caps.astype(np.uint64)
        self.extent = int(ends.max()) if extent is None and n else int(extent or 0)


class Result:
    def __init__(self, rc, err, status, out_len, used, out, base, batch):
        self.rc, self.err, self.status, self.out_len, self.used = rc, err, status, out_len, used
        self.out, self.base, self.batch = out, base, batch

    def unit(self, i):
        o = self.base + int(self.batch.out_off[i])
        return int(self.status[i]), self.out[o:o + int(self.out_len[i])].tobytes(), int(self.used[i])

    def units(self):
        return [self.unit(i) for i in range(len(self.status))]


class Pending:
    pass


def enqueue(B, b, *, ws=None, ws_bytes=None, ws_fill=None, stream=None, null_stream=False, base=0, tail=0):
    """Enqueue one b200z_inflate_batch_device call; `base` bytes of the output allocation lie in front of d_out_base
    and `tail` behind the extent, all filled with GUARD like every gap of the layout."""
    L = B.L
    n = len(b.in_len)
    p = Pending()
    p.b, p.base, p.stream = b, base, stream
    p.d_in = B.put(np.frombuffer(b.blob, dtype=np.uint8), stream)
    p.d_in_off, p.d_in_len = B.put(b.in_off, stream), B.put(b.in_len, stream)
    p.d_out_off, p.d_out_cap = B.put(b.out_off, stream), B.put(b.caps, stream)
    p.d_out = B.full(base + b.extent + tail, np.uint8, GUARD, stream)
    p.d_status = B.full(n, np.int32, -99, stream)
    p.d_len = B.full(n, np.uint32, 0xFFFFFFFF, stream)
    p.d_used = B.full(n, np.uint32, 0xFFFFFFFF, stream)
    if ws is None:
        if ws_bytes is None:
            ws_bytes = L.b200z_inflate_workspace_bytes(n, len(b.blob), b.extent)
        ws = B.full(ws_bytes, np.uint8, ws_fill, stream)
    p.ws = ws
    if null_stream:
        B.sync(stream)  # the uploads above ran on the side stream; the library's own stream does not wait for it
    h = None if null_stream else B.handle(stream)
    p.rc = L.b200z_inflate_batch_device(B.ptr(p.d_in), B.ptr(p.d_in_off), B.ptr(p.d_in_len), B.ptr(p.d_out) + base,
                                        B.ptr(p.d_out_off), B.ptr(p.d_out_cap), B.ptr(p.d_len), B.ptr(p.d_status),
                                        B.ptr(p.d_used), n, B.ptr(ws), ws_bytes, h)
    p.err = B.ffi.last_error() if p.rc else ""
    return p


def collect(B, p, synced=False):
    if not synced:
        B.sync(p.stream)
    r = Result(p.rc, p.err, B.get(p.d_status), B.get(p.d_len), B.get(p.d_used), B.get(p.d_out), p.base, p.b)
    if r.rc == 0:
        check_guards(r)
    return r


def run(B, b, **kw):
    return collect(B, enqueue(B, b, **kw))


def check_guards(r):
    """Every output byte outside the units' [out_off, out_off + out_cap) slots is unchanged, and no unit reports
    more bytes than its cap."""
    b = r.batch
    assert (r.out_len <= b.caps).all()
    d = np.zeros(len(r.out) + 1, dtype=np.int64)
    st = r.base + b.out_off.astype(np.int64)
    np.add.at(d, st, 1)
    np.add.at(d, st + b.caps.astype(np.int64), -1)
    outside = np.cumsum(d)[:-1] == 0
    bad = np.nonzero(outside & (r.out != GUARD))[0]
    assert len(bad) == 0, f"bytes outside every slot were written, first at {bad[:8]}"


def both_kernels(monkeypatch, fn):
    """fn() under B200Z_FAST=1 and =0; every unit must give the same status, out_len, in_used and bytes."""
    res = {}
    for f in ("1", "0"):
        monkeypatch.setenv("B200Z_FAST", f)
        res[f] = fn()
    a, z = res["1"], res["0"]
    assert a.rc == z.rc == 0, (a.err, z.err)
    same_results(a, z)
    return a


def same_results(a, z):
    for name in ("status", "out_len", "used"):
        diff = np.nonzero(getattr(a, name) != getattr(z, name))[0]
        assert len(diff) == 0, (name, diff[:8], getattr(a, name)[diff[:8]], getattr(z, name)[diff[:8]])
    for i in range(len(a.status)):
        assert a.unit(i)[1] == z.unit(i)[1], i


def check_vs_oracle(units, caps, res, oracle=None, clean=False):
    """The oracle's comparison rules of test_inflate_gpu.py; clean=True also requires the oracle to decode the unit."""
    seen = set()
    for i, u in enumerate(units):
        ost, oout, oused = oracle[i] if oracle is not None else orc.inflate(u)
        st, out, used = res.unit(i)
        seen.add((st, ost))
        if clean:
            assert ost == orc.OK, i
        if st == U_NOSPC:  # the cap was reached: a prefix of what the oracle decodes
            assert oout[:len(out)] == out, i
            if ost == orc.OK:
                assert len(oout) > caps[i], (i, len(oout), caps[i])
        elif ost == orc.OK:
            if st in (0, 1, -1):
                assert out == oout, i
                if st == 0:
                    assert used == oused, (i, used, oused)
            else:
                assert not clean and st in (-3, -4) and oout[:len(out)] == out, (i, st)
        elif ost == orc.RUNAWAY:
            assert st == -4, (i, st)
        else:
            assert st in (-3, -4, -5), (i, st)
    return seen


# ------------------------------------------------------------------ inputs
def corpus(rng, n):
    words = [bytes(rng.choice(b"etaoinshrdlu") for _ in range(rng.randint(2, 9))) for _ in range(300)]
    b = bytearray()
    while len(b) < n:
        b += rng.choice(words) + b" "
    return bytes(b[:n])


def raw_deflate(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, mem=8):
    co = zlib.compressobj(level, zlib.DEFLATED, -15, mem, strategy)
    return co.compress(data) + co.flush()


def mixed_units(rng, n, sizes):
    """Stored, fixed, dynamic, Huffman-only and RLE units, with sync / full flush points, random and zero text, and
    sometimes trailing garbage or nothing at all after the final block (the reference's short-read quirk Q1)."""
    units = []
    for it in range(n):
        t = corpus(rng, rng.choice(sizes))
        if it % 7 == 0:
            t = bytes(rng.getrandbits(8) for _ in range(len(t) // 4))
        if it % 11 == 0:
            t = b"\0" * len(t)
        co = zlib.compressobj(rng.choice([0, 1, 6, 9]), zlib.DEFLATED, -15, rng.choice([1, 8, 9]),
                              rng.choice([zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE]))
        h = len(t) // 2
        z = co.compress(t[:h]) + co.flush(rng.choice([zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH, zlib.Z_NO_FLUSH])) + \
            co.compress(t[h:]) + co.flush()
        units.append(z + rng.choice([b"", b"", b"\0\0", b"trailing garbage"]))
    return units


def oracle_caps(rng, units, slack=(0, 0, 5)):
    oracle = [orc.inflate(u) for u in units]
    return oracle, [len(o[1]) + rng.choice(slack) for o in oracle]


# ------------------------------------------------------------------ 1. mixed corpus
def test_mixed_corpus_vs_oracle(B, monkeypatch):
    rng = random.Random(17)
    units = mixed_units(rng, 120 if EMU else 300, [0, 1, 2, 3, 100, 191, 192, 5000, 30000, 65536, 70000])
    oracle, caps = oracle_caps(rng, units)
    b = Batch(units, caps, rng=rng)
    r = both_kernels(monkeypatch, lambda: run(B, b))
    seen = check_vs_oracle(units, caps, r, oracle, clean=True)
    assert (0, orc.OK) in seen and (-1, orc.OK) in seen


def test_tiny_batches(B, monkeypatch):
    """Batches whose whole output is a few bytes (or none) run with exactly b200z_inflate_workspace_bytes."""
    hello = raw_deflate(b"hello world")
    for units in ([hello], [b"\x03\x00"], [hello, hello], [b"\x03\x00"] * 3, [raw_deflate(b"x" * 75)]):
        oracle = [orc.inflate(u) for u in units]
        caps = [len(o[1]) for o in oracle]
        b = Batch(units, caps)
        r = both_kernels(monkeypatch, lambda: run(B, b))
        check_vs_oracle(units, caps, r, oracle, clean=True)
    r = run(B, Batch([hello], [11]))
    assert r.unit(0) == (0, b"hello world", len(hello))


# ------------------------------------------------------------------ 2. batch sizes that change the decode geometry
def small_pool(rng, k=48):
    pool = []
    for i in range(k):
        t = corpus(rng, rng.choice([0, 1, 5, 40, 120, 300]))
        pool.append(raw_deflate(t, rng.choice([0, 1, 6, 9]), rng.choice([zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED])))
    pool.append(b"\x03\x00")
    return pool


@pytest.mark.parametrize("n", [1, 2, 31, 33, 1583, 1584, 1585, 3169, 6337, 12673])
def test_batch_geometry_exact_pair(B, monkeypatch, n):
    """launch_inflate sizes streams per warp against 132 x 12 target warps and gives each stream 32 / upw lanes
    (capped at 8): these batch sizes cross those steps and leave partly filled tail warps."""
    monkeypatch.setenv("B200Z_FAST", "0")
    rng = random.Random(n)
    pool = small_pool(rng)
    po = [orc.inflate(u) for u in pool]
    pick = [rng.randrange(len(pool)) for _ in range(n)]
    units = [pool[k] for k in pick]
    oracle = [po[k] for k in pick]
    caps = [len(o[1]) + (i % 3 == 0) for i, o in enumerate(oracle)]
    r = run(B, Batch(units, caps, rng=rng))
    assert r.rc == 0, r.err
    check_vs_oracle(units, caps, r, oracle, clean=True)


# ------------------------------------------------------------------ 3. k_inflate_fast's eligibility edges
def test_fast_eligibility_in_len_edges(B, monkeypatch):
    """The same stream followed by trailing bytes, so that in_len crosses MIN_IN and (at leads 0, 1 and 15)
    the IN_CAP limit on the 16-byte rounded input, which includes the unit's lead."""
    rng = random.Random(3)
    small = raw_deflate(b"".join(rng.choice([b"alpha ", b"beta ", b"gamma "]) for _ in range(120)), 9)
    assert len(small) < MIN_IN - 1
    big = raw_deflate(bytes(rng.choice(b"abcdefghijklmnop") for _ in range(52000)), 9)
    assert IN_CAP - 15 - 16 - 16 > len(big) > IN_CAP // 2, len(big)
    units, leads = [], []
    for il in (MIN_IN - 1, MIN_IN, MIN_IN + 1):
        units.append(small + bytes(rng.getrandbits(8) for _ in range(il - len(small))))
        leads.append(rng.randrange(16))
    for lead in (0, 1, 15):
        for il in range(IN_CAP - lead - 16, IN_CAP - lead + 2):
            units.append(big + bytes(rng.getrandbits(8) for _ in range(il - len(big))))
            leads.append(lead)
    oracle, caps = oracle_caps(rng, units, slack=(0,))
    b = Batch(units, caps, rng=rng, leads=leads)
    assert all(int(o) % 16 == ld for o, ld in zip(b.in_off, leads))
    r = both_kernels(monkeypatch, lambda: run(B, b))
    check_vs_oracle(units, caps, r, oracle, clean=True)
    assert (r.status == 0).all()


def test_fast_eligibility_cap_edges(B, monkeypatch):
    """A 65 536-byte output under caps of 65535 (full), 65536 (the fast kernel's window) and 65537 (too big for
    it), and smaller outputs under exact caps and caps with slack."""
    rng = random.Random(4)
    t64 = corpus(rng, WIN)
    units, caps = [], []
    for strat in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED):
        z = raw_deflate(t64, 6, strat)
        for cap in (WIN - 1, WIN, WIN + 1, WIN + 4096):
            units.append(z)
            caps.append(cap)
    for size in (1, 15, 16, 17, 4095, 4096, 40000):
        z = raw_deflate(corpus(rng, size), 6)
        z += bytes(max(0, MIN_IN - len(z)))  # long enough for the fast kernel
        for slack in (0, 1, 16, 1000):
            units.append(z)
            caps.append(size + slack)
        units.append(z)
        caps.append(size - 1)
    oracle = [orc.inflate(u) for u in units]
    b = Batch(units, caps, rng=rng)
    r = both_kernels(monkeypatch, lambda: run(B, b))
    check_vs_oracle(units, caps, r, oracle, clean=True)
    for i, (ost, oout, _) in enumerate(oracle):
        assert int(r.status[i]) == (U_NOSPC if caps[i] < len(oout) else 0), i


# ------------------------------------------------------------------ 4. layouts
def test_layout_permuted_gapped_unaligned_inner_base(B, monkeypatch):
    """Slots in an order unrelated to the units, with guard-filled gaps between them, at every offset mod 16, behind
    a d_out_base that sits inside a larger allocation."""
    rng = random.Random(5)
    units = mixed_units(rng, 60 if EMU else 160, [0, 1, 100, 191, 5000, 20000, 65536])
    oracle, caps = oracle_caps(rng, units)
    n = len(units)
    order = list(range(n))
    rng.shuffle(order)
    out_off = np.zeros(n, dtype=np.uint64)
    pos = 0
    for k, u in enumerate(order):
        pos += rng.choice([0, 1, 7, 100])
        pos += (k % 16 - pos) % 16  # slot k of the layout starts at k mod 16
        out_off[u] = pos
        pos += caps[u]
    b = Batch(units, caps, out_off=out_off, rng=rng)
    assert {int(o) % 16 for o in out_off} == set(range(16))
    r = both_kernels(monkeypatch, lambda: run(B, b, base=4096 + 5, tail=333))
    check_vs_oracle(units, caps, r, oracle, clean=True)


def test_layout_bench_two_rank_chunks(B, monkeypatch):
    """bench.py's layout at world = 2, rank 1, four chunks: a chunk's units land at rank * cb of a world * cb window
    (the other rank's half is a gap), d_out_base moves by chunk and out_off is relative to it, and the workspace is
    sized by the window's extent.  One workspace serves every chunk, alternating the kernels."""
    from archive_b200 import synth
    unit, world, rank, nch = 4096, 2, 1, 4
    n = 64 if EMU else 512
    upc, cb = n // nch, n // nch * unit
    w = synth.gzip_workload(n, unit, stream0=11, keep_text=True)
    blob, moff = w["blob"], w["member_off"]
    in_off = (moff[:-1] + 18).astype(np.uint64)
    in_len = (moff[1:] - moff[:-1] - 18).astype(np.uint32)
    units = [blob[int(o):int(o) + int(ln)].tobytes() for o, ln in zip(in_off, in_len)]
    out_off = np.array([rank * cb + (u % upc) * unit for u in range(upc)], dtype=np.uint64)
    caps = [unit] * upc
    ws_bytes = B.L.b200z_inflate_workspace_bytes(upc, len(blob), world * cb)
    ws = B.full(ws_bytes, np.uint8, None)
    full = bytearray()
    for c in range(nch):
        b = Batch(units[c * upc:(c + 1) * upc], caps, in_off=in_off[c * upc:(c + 1) * upc], out_off=out_off,
                  extent=world * cb)
        b.blob = bytes(blob) + bytes((-len(blob)) % 16)
        monkeypatch.setenv("B200Z_FAST", "1" if c % 2 == 0 else "0")
        r = run(B, b, ws=ws, ws_bytes=ws_bytes, base=c * world * cb, tail=(nch - 1 - c) * world * cb)
        assert r.rc == 0, r.err
        assert (r.status == 0).all() and (r.used + 8 == b.in_len).all()
        full += r.out[c * world * cb + rank * cb:c * world * cb + (rank + 1) * cb].tobytes()
    assert bytes(full) == w["text"].tobytes()


def test_layout_shared_input(B, monkeypatch):
    """Entries that point at the same compressed bytes decode the same output into their own slots."""
    rng = random.Random(6)
    z = raw_deflate(corpus(rng, 30000))
    small = raw_deflate(corpus(rng, 50))
    blob = bytes(3) + z + bytes(5) + small
    blob += bytes((-len(blob)) % 16)
    in_off = [3, 3, len(z) + 8, 3, len(z) + 8]
    units = [blob[o:o + (len(z) if o == 3 else len(small))] for o in in_off]
    oracle, caps = oracle_caps(rng, units, slack=(0, 1))
    b = Batch(units, caps, in_off=in_off)
    b.blob = blob
    r = both_kernels(monkeypatch, lambda: run(B, b))
    check_vs_oracle(units, caps, r, oracle, clean=True)


# ------------------------------------------------------------------ 5. workspace
def test_workspace_contents_do_not_matter(B, monkeypatch):
    rng = random.Random(7)
    units = mixed_units(rng, 48 if EMU else 120, [0, 1, 100, 191, 192, 5000, 65536])
    oracle, caps = oracle_caps(rng, units)
    b = Batch(units, caps, rng=rng)
    ref = both_kernels(monkeypatch, lambda: run(B, b, ws_fill=0x00))
    check_vs_oracle(units, caps, ref, oracle, clean=True)
    for fill in (0xFF, None):
        same_results(ref, both_kernels(monkeypatch, lambda: run(B, b, ws_fill=fill)))


def test_workspace_reused_across_kernels(B, monkeypatch):
    """One workspace of exactly b200z_inflate_workspace_bytes, no slack, serves consecutive calls that alternate
    the kernels, as bench.py's timed steps do; each call starts from what the previous one left in it."""
    rng = random.Random(8)
    batches = []
    for k in range(4):
        units = mixed_units(rng, 40 if EMU else 100, [0, 100, 192, 5000, 65536])
        oracle, caps = oracle_caps(rng, units)
        batches.append((units, caps, oracle, Batch(units, caps, rng=rng)))
    n = max(len(b.in_len) for *_, b in batches)
    ext = max(b.extent for *_, b in batches)
    ws_bytes = B.L.b200z_inflate_workspace_bytes(n, 0, ext)
    ws = B.full(ws_bytes, np.uint8, 0xFF)
    first = []
    for rep in range(2):
        for k, (units, caps, oracle, b) in enumerate(batches):
            monkeypatch.setenv("B200Z_FAST", str((k + rep) % 2))
            wsb = B.L.b200z_inflate_workspace_bytes(len(units), 0, b.extent)
            r = run(B, b, ws=ws, ws_bytes=wsb)
            assert r.rc == 0, r.err
            check_vs_oracle(units, caps, r, oracle, clean=True)
            if rep == 0:
                first.append(r)
            else:
                same_results(first[k], r)


def test_workspace_one_byte_short(B):
    """A workspace one byte smaller than the least any batch of n units needs is refused before anything is
    enqueued: the status array keeps what the caller put there."""
    for n in (1, 5, 300):
        units = [raw_deflate(b"abc")] * n
        b = Batch(units, [3] * n)
        least = B.L.b200z_inflate_workspace_bytes(n, 0, 0)
        r = run(B, b, ws_bytes=least - 1)
        assert r.rc == E_ARG and "workspace" in r.err
        assert (r.status == -99).all() and (r.out_len == 0xFFFFFFFF).all() and (r.out == GUARD).all()
        r = run(B, b, ws_bytes=B.L.b200z_inflate_workspace_bytes(n, 0, b.extent))
        assert r.rc == 0 and (r.status == 0).all() and r.unit(n - 1)[1] == b"abc"


# ------------------------------------------------------------------ 6. sizing sweep
SWEEP_N = [1, 2, 7, 64, 1000]


@pytest.mark.parametrize("n", SWEEP_N)
def test_workspace_sizing_sweep(B, n):
    """n empty units whose caps add up to the extent E run with exactly b200z_inflate_workspace_bytes(n, in, E),
    for every E up to 4096 and seeded larger ones: the library must find in that workspace an extent >= E."""
    rng = random.Random(n)
    extents = list(range(4097)) + [rng.randrange(4097, 1 << 24) for _ in range(64)]
    if EMU and n >= 64:  # (the emulated library decodes every unit on the CPU: a sample of the same extents)
        extents = list(range(0, 160)) + extents[160::101]
    st0, _, used0 = orc.inflate(b"\x03\x00")
    assert st0 == orc.OK
    blob = np.frombuffer(bytes(pad16(2 * n)), dtype=np.uint8).copy()
    blob[0:2 * n:2] = 3
    d_in = B.put(blob)
    d_in_off = B.put(np.arange(n, dtype=np.uint64) * 2)
    d_in_len = B.put(np.full(n, 2, dtype=np.uint32))
    caps = np.zeros((len(extents), n), dtype=np.uint32)
    for k, e in enumerate(extents):
        caps[k] = e // n
        caps[k, :e % n] += 1
    offs = np.zeros_like(caps, dtype=np.uint64)
    offs[:, 1:] = np.cumsum(caps, axis=1, dtype=np.uint64)[:, :-1]
    assert (caps.sum(axis=1, dtype=np.uint64) == np.array(extents, dtype=np.uint64)).all()
    d_caps, d_offs = B.put(caps), B.put(offs)
    d_status = B.full(caps.size, np.int32, -99)
    d_len = B.full(caps.size, np.uint32, 0xFFFFFFFF)
    d_used = B.full(caps.size, np.uint32, 0xFFFFFFFF)
    d_out = B.full(max(extents) + 1, np.uint8, GUARD)
    rcs = []
    for k, e in enumerate(extents):
        wsb = B.L.b200z_inflate_workspace_bytes(n, len(blob), e)
        ws = B.full(wsb, np.uint8, None)
        at = k * n
        rc = B.L.b200z_inflate_batch_device(B.ptr(d_in), B.ptr(d_in_off), B.ptr(d_in_len), B.ptr(d_out),
                                            B.ptr(d_offs) + 8 * at, B.ptr(d_caps) + 4 * at, B.ptr(d_len) + 4 * at,
                                            B.ptr(d_status) + 4 * at, B.ptr(d_used) + 4 * at, n, B.ptr(ws), wsb,
                                            B.handle())
        rcs.append((e, rc, B.ffi.last_error() if rc else ""))
    B.sync()
    bad = [x for x in rcs if x[1] != 0]
    assert not bad, f"{len(bad)} of {len(extents)} extents refused, first {bad[:3]}"
    status, out_len, used = B.get(d_status), B.get(d_len), B.get(d_used)
    assert (status == 0).all() and (out_len == 0).all() and (used == used0).all()
    assert (B.get(d_out) == GUARD).all()


# ------------------------------------------------------------------ 7. streams
@pytest.mark.needs_device
def test_two_streams_in_flight(B):
    """Two batches with workspaces of their own, enqueued on two streams before either is synchronised, give what
    each gives alone."""
    import torch
    from archive_b200 import synth
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    bs = []
    for k in range(2):
        w = synth.gzip_workload(256, 65536, stream0=20 + k)
        blob, moff = w["blob"], w["member_off"]
        in_off = (moff[:-1] + 18).astype(np.uint64)
        units = [blob[int(a) + 18:int(z)].tobytes() for a, z in zip(moff[:-1], moff[1:])]
        b = Batch(units, [65536] * 256, in_off=in_off)
        b.blob = bytes(blob) + bytes((-len(blob)) % 16)
        bs.append(b)
    alone = [run(B, b) for b in bs]
    p1 = enqueue(B, bs[0], stream=s1)
    p2 = enqueue(B, bs[1], stream=s2)
    both = [collect(B, p1), collect(B, p2)]
    for a, z in zip(alone, both):
        assert a.rc == z.rc == 0
        assert (a.status == 0).all()
        same_results(a, z)


@pytest.mark.needs_device
def test_null_stream(B):
    """cuda_stream = NULL runs on the library's own stream; a device-wide synchronise then covers it."""
    import torch
    rng = random.Random(9)
    units = mixed_units(rng, 100, [0, 100, 5000, 65536])
    oracle, caps = oracle_caps(rng, units)
    b = Batch(units, caps, rng=rng)
    p = enqueue(B, b, null_stream=True)
    torch.cuda.synchronize()
    r = collect(B, p, synced=True)
    assert r.rc == 0, r.err
    check_vs_oracle(units, caps, r, oracle, clean=True)
    same_results(r, run(B, b))


# ------------------------------------------------------------------ 8. bench.py's config-2 shape
def test_config2_shape(B, monkeypatch):
    """bench.py's workload at test size: synth.gzip_workload members of 64 KiB, units at the 18-byte header, the
    8-byte trailer inside in_len.  Every unit's output hashes to its trailer's CRC-32 and length."""
    from archive_b200 import synth
    n = 64 if EMU else 1024
    w = synth.gzip_workload(n, 65536, stream0=0)
    blob, moff = w["blob"], w["member_off"]
    in_off = (moff[:-1] + 18).astype(np.uint64)
    units = [blob[int(a) + 18:int(z)].tobytes() for a, z in zip(moff[:-1], moff[1:])]
    b = Batch(units, [65536] * n, in_off=in_off)
    b.blob = bytes(blob) + bytes((-len(blob)) % 16)
    r = both_kernels(monkeypatch, lambda: run(B, b))
    assert (r.status == 0).all() and (r.out_len == 65536).all()
    assert (r.used + 8 == b.in_len).all()
    for i, u in enumerate(units):
        out = r.unit(i)[1]
        assert zlib.crc32(out) == int.from_bytes(u[-8:-4], "little"), i
        assert len(out) == int.from_bytes(u[-4:], "little"), i
    for i in random.Random(10).sample(range(n), 8):
        ost, oout, oused = orc.inflate(units[i])
        assert ost == orc.OK and r.unit(i) == (0, oout, oused), i


# ------------------------------------------------------------------ 9. bad data
def test_bad_data_vs_oracle(B, monkeypatch):
    rng = random.Random(23)
    units, base = [], []
    for it in range(8 if EMU else 12):
        t = corpus(rng, rng.randint(1, 4000))
        base.append(raw_deflate(t, rng.choice([0, 1, 6, 9]), rng.choice([0, 4])))
    for z in base:
        for cut in range(0, len(z), max(1, len(z) // 25)):
            units.append(z[:cut])
        for _ in range(25):
            zz = bytearray(z)
            zz[rng.randrange(len(zz))] ^= 1 << rng.randrange(8)
            units.append(bytes(zz))
    for _ in range(100):
        units.append(bytes(rng.getrandbits(8) for _ in range(rng.randint(1, 300))))
    big = raw_deflate(corpus(rng, 60000))  # long enough for the fast kernel to take, then give back
    for _ in range(12):
        zz = bytearray(big)
        zz[rng.randrange(len(zz))] ^= 1 << rng.randrange(8)
        units.append(bytes(zz))
    units = [u for u in units if len(u) > 0]
    caps = [1 << 16] * len(units)
    b = Batch(units, caps, rng=rng)
    r = both_kernels(monkeypatch, lambda: run(B, b))
    seen = check_vs_oracle(units, caps, r)
    assert (0, 0) in seen and (-1, 0) in seen
