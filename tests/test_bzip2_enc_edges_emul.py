"""Edge catalogue of the device BZip2 encoder (archive_b200/csrc/bzip2_enc_*.{cu,inl}) on the CUDA execution-model
emulation.  Every case must give the oracle's bytes, decode with libbz2, and pass the table check of tests/bz2_stream.py
(each table's code lengths are those of its symbol counts under the final selectors), which does not use the oracle.

Each case also asserts, from the parsed stream, the edge it is there for, so that an input which drifts off its edge fails
instead of passing quietly:
  - table count: nmtf on both sides of 200 / 600 / 1200 / 2400, and more tables than symbols (k_h_tables);
  - alphabet: nInUse 1, 2, 255, 256 and in-use maps with gaps;
  - the 17-bit length limit: tables whose unlimited code is deeper than 17 (the halving retry) and one exactly 17 deep;
  - selectors: counts around the 12 384 split of the staged selectors, the largest count, look-backs past a thread's own
    run, tables never selected, nmtf around multiples of 50 and of 2000 (the emission tiles);
  - MTF chunks of 2048 symbols: zero runs placed exactly at chunk edges, symbols absent for many chunks, first seen late;
  - RLE1 runs around 4 KiB input tiles and 128-byte sub-tiles (k_e_*);
  - a batch mixing periodic blocks (k_serial_sort) with random and text blocks, and the same input in several batches.
tests/test_bzip2_enc_edges_gpu.py runs the same catalogue on the device."""
import bz2
import ctypes as C
import functools
import os
import random
import subprocess

import numpy as np
import pytest

import bz2_stream as bs
import oracle_lib as orc

TS = 2048  # MTF chunk (symbols)
TI = 4096  # input tile (bytes)
SUB = 128  # input sub-tile


# ---------------------------------------------------------------------------------------------------------------------
# sources
# ---------------------------------------------------------------------------------------------------------------------
def norun(alphabet, n, seed):
    """Random bytes over `alphabet` with no two neighbours equal: RLE1 leaves them as they are."""
    a = np.frombuffer(bytes(alphabet), np.uint8)
    r = np.random.default_rng(seed)
    idx = np.cumsum(r.integers(1, len(a), n)) % len(a)
    return a[idx].tobytes()


def skewed(seed, nsym, n, ratio):
    """i.i.d. symbols k = 0..nsym-1 with p(k) proportional to ratio^-k."""
    p = ratio ** -np.arange(nsym, dtype=np.float64)
    r = np.random.default_rng(seed)
    return (r.choice(nsym, size=n, p=p / p.sum()) + 0x61).astype(np.uint8).tobytes()


def letters(n, seed, k=16):
    r = random.Random(seed)
    return bytes(0x61 + r.randrange(k) for _ in range(n))


def short_runs(alphabet, n, seed):
    """Runs of 1 to 3 equal bytes cycling through `alphabet` (no RLE1 run length bytes): nInUse == len(alphabet)."""
    r = random.Random(seed)
    out = bytearray()
    i = 0
    while len(out) < n:
        out += bytes([alphabet[i % len(alphabet)]]) * r.randint(1, 3)
        i += 1 + (r.randrange(len(alphabet) - 1) if len(alphabet) > 2 else 0)
    return bytes(out[:n])


def text(n, seed):
    from archive_b200 import synth
    return synth.text(n, stream=seed).tobytes()


def last_column_input(seq: bytes) -> bytes:
    """An input whose last column ends with `seq`.  Token i is seq[i], 0xF0 and a 3-byte key of i (bytes 0x80..0xEF):
    the rotations that start with 0xF0 sort last, in token order, and each is preceded by seq[i].  So the last M = len(seq)
    rows of the block's last column are seq, rows 4M .. 5M - 1, and no RLE1 run reaches 4."""
    m = len(seq)
    i = np.arange(m)
    tok = np.empty((m, 5), np.uint8)
    tok[:, 0] = np.frombuffer(seq, np.uint8)
    tok[:, 1] = 0xF0
    tok[:, 2] = 0x80 + i // (112 * 112)
    tok[:, 3] = 0x80 + (i // 112) % 112
    tok[:, 4] = 0x80 + i % 112
    return tok.tobytes()


@functools.lru_cache(maxsize=None)
def oracle(data: bytes) -> bytes:
    st, z = orc.bzip2_encode(data)
    assert st == orc.OK
    return z


def nmtf_of(data: bytes) -> int:
    s = bs.parse(oracle(data))
    assert len(s.blocks) == 1
    return s.blocks[0].nmtf


def prefix_with_nmtf(src: bytes, target: int) -> bytes:
    """The shortest prefix of `src` whose single block has nmtf == target (a bisection on the length, then a walk)."""
    lo, hi = 1, len(src)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if nmtf_of(src[:mid]) < target:
            lo = mid
        else:
            hi = mid
    for n in range(max(1, lo - 64), min(len(src), hi + 256)):
        if nmtf_of(src[:n]) == target:
            return src[:n]
    raise AssertionError("no prefix reaches nmtf %d" % target)


# ---------------------------------------------------------------------------------------------------------------------
# edge claims, checked on the parsed stream of every encoder (oracle, emulation, device)
# ---------------------------------------------------------------------------------------------------------------------
def zero_runs(pos):
    a = np.asarray(pos, dtype=np.int64)
    z = np.concatenate([[0], (a == 0).astype(np.int8), [0]])
    d = np.diff(z)
    return list(zip(np.nonzero(d == 1)[0].tolist(), np.nonzero(d == -1)[0].tolist()))


def lookback_past_run(b: bs.Block) -> bool:
    """Some thread of the selector MTF (512 threads, ceil(nSel/512) selectors each) finds a table it needs for its start
    list only before the previous thread's run."""
    per = (b.n_sel + 511) // 512
    sel = b.selectors
    for lo in range(per, b.n_sel, per):
        seen = set(sel[max(0, lo - per):lo])
        if any(t in sel[:max(0, lo - per)] and t not in seen for t in range(b.n_groups)):
            return True
    return False


def n_groups_is(*want):
    def claim(s, chk):
        assert [b.n_groups for b in s.blocks] == list(want)
    return claim


def nmtf_is(want, groups):
    def claim(s, chk):
        assert len(s.blocks) == 1 and s.blocks[0].nmtf == want and s.blocks[0].n_groups == groups
    return claim


def in_use_is(n, groups=None, gaps=None):
    def claim(s, chk):
        b = s.blocks[0]
        assert b.n_in_use == n
        if groups is not None:
            assert b.n_groups == groups
        if gaps is not None:  # 16-byte ranges with a gap
            ranges = [set(range(16 * i, 16 * i + 16)) for i in range(16)]
            assert sum(1 for r in ranges if not r <= set(b.in_use)) == gaps
    return claim


def retry_runs(s, chk):
    assert any(any(c.retried) for c in chk)


def depth_17_no_retry(s, chk):
    assert max(chk[0].depths) == 17 and not any(chk[0].retried)


def n_sel_is(want):
    def claim(s, chk):
        assert s.blocks[0].n_sel == want
    return claim


def max_n_sel(s, chk):
    assert max(b.n_sel for b in s.blocks) == 18000


def lookback(s, chk):
    assert any(lookback_past_run(b) for b in s.blocks)


def unused_table(s, chk):
    assert any(any(c.unused) for c in chk)


# zero runs of the MTF positions placed in the controlled tail of the last column (last_column_input):
# (length, where) with where "end" = the run ends at a chunk edge, "start" = starts at one, "cross" = straddles one
ZR_PLAN = ([(L, "cross") for L in (2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257,
                                    511, 512, 513, 1023, 1024, 1025, 2047, 2048, 2049)]
           + [(L, w) for L in (1, 2, 3, 4, 7, 8, 9, 255, 256, 257) for w in ("end", "start")]
           + [(2048, "start"), (4096, "start"), (2047, "end"), (5000, "cross")])
ZR_EOB = 100


@functools.lru_cache(maxsize=None)
def zero_run_layout():
    """-> (input, planned zero runs as [start, end) rows, rows of the rare symbols)"""
    m = 80 * TS  # 5m bytes: one block
    base = 4 * m  # first row of the controlled tail
    seq = bytearray()
    runs = []
    letter = 0

    def put(n):  # n equal letters; the letter alternates between runs
        nonlocal letter
        seq.extend([b"AB"[letter]] * n)
        letter ^= 1

    edge = base + TS
    for L, where in ZR_PLAN:
        while True:
            start = {"end": edge - L, "start": edge, "cross": edge - L // 2}[where]
            if start - base - 1 >= len(seq):
                break
            edge += TS
        while len(seq) < start - base - 1:
            put(1)
        # a letter run of L + 1 gives L zeros after its first symbol
        runs.append((start, start + L))
        put(L + 1)
        edge = (runs[-1][1] // TS + 1) * TS
    while len(seq) < m - ZR_EOB - 1:
        put(1)
    runs.append((base + len(seq) + 1, base + m))
    put(m - len(seq))
    assert len(seq) == m and runs[-2][1] < base + m - 3 * TS

    def free_row(r):  # the first row from r on that holds a filler letter
        while any(a - 1 <= r <= b for a, b in runs):
            r += 1
        return r

    # 'D' early and again 6 chunks later; 'C' once, in the last chunk but one
    d0 = free_row(base + 3 * TS)
    rare = {b"D": (d0, free_row(d0 + 6 * TS)), b"C": (free_row(base + m - 2 * TS + 11),)}
    for ch, rows in rare.items():
        for r in rows:
            seq[r - base] = ch[0]
    return last_column_input(bytes(seq)), runs, rare


def zero_runs_placed(s, chk):
    _, runs, rare = zero_run_layout()
    b = s.blocks[0]
    pos = bs.mtf_positions(b)
    got = set(zero_runs(pos))
    for r in runs:
        assert r in got, r
    assert runs[-1][1] == len(pos)  # a zero run up to EOB
    # the edges the plan claims
    assert any(a % TS == 0 for a, _ in runs) and any(e % TS == 0 for _, e in runs[:-1])
    assert any(e // TS - (a + TS - 1) // TS >= 2 for a, e in runs)  # covers two whole chunks
    col = bs.last_column(b)
    sym = {ch: b.in_use.index(ch[0]) for ch in rare}
    d_rows = [i for i, v in enumerate(col) if v == sym[b"D"]]
    assert d_rows == list(rare[b"D"]) and d_rows[1] // TS - d_rows[0] // TS > 4  # absent for more than 3 whole chunks
    c_rows = [i for i, v in enumerate(col) if v == sym[b"C"]]
    assert c_rows == list(rare[b"C"]) and c_rows[0] // TS >= len(col) // TS - 2 >= 100  # first seen late


SEL12384, SEL12385 = 619154, 619204  # prefixes of the seeded random source found by a bisection with the oracle


# ---------------------------------------------------------------------------------------------------------------------
# the catalogue: name -> (input builder, claim)
# ---------------------------------------------------------------------------------------------------------------------
def groups_for(nmtf):
    return 2 if nmtf < 200 else 3 if nmtf < 600 else 4 if nmtf < 1200 else 5 if nmtf < 2400 else 6


def _threshold_cases():
    out = {}
    for t in (200, 600, 1200, 2400):
        groups = groups_for(t - 1)
        src = letters(4 * t, seed=t)
        out["groups_%d_below" % t] = (functools.partial(prefix_with_nmtf, src, t - 1), nmtf_is(t - 1, groups))
        out["groups_%d_at" % t] = (functools.partial(prefix_with_nmtf, src, t), nmtf_is(t, groups + 1))
    for k in (1050, 2000, 4000):  # emission tiles of 2000 symbols, groups of 50
        src = letters(3 * k, seed=k, k=64)
        for d in (-1, 0, 1):
            out["nmtf_%d%+d" % (k, d)] = (functools.partial(prefix_with_nmtf, src, k + d), nmtf_is(k + d, groups_for(k + d)))
    return out


CASES = {
    **_threshold_cases(),
    # more tables than symbols in the alphabet (alpha = nInUse + 2 < nGroups); a block over one symbol never has more
    # than a few MTF values (nmtf <= 1 + log2 of the run), so nInUse 1 stays at 2 tables
    "tables_gt_alpha_2": (lambda: short_runs(b"ab", 60000, 1), in_use_is(2, groups=6)),
    "tables_gt_alpha_3": (lambda: short_runs(b"abc", 20000, 2), in_use_is(3, groups=6)),
    "in_use_1_run3": (lambda: b"zzz", in_use_is(1, groups=2)),
    "in_use_1_zero4": (lambda: bytes(4), in_use_is(1, groups=2)),  # RLE1: 0 0 0 0 and run length byte 0
    "in_use_2": (lambda: norun(b"\x00\xff", 5000, 3), in_use_is(2)),
    "in_use_255": (lambda: norun(bytes(v for v in range(256) if v != 0x41), 40000, 4), in_use_is(255, gaps=1)),
    "in_use_256": (lambda: norun(range(256), 40000, 5), in_use_is(256, gaps=0)),
    "in_use_gaps_every_range": (lambda: norun(bytes(v for v in range(256) if v % 16 not in (3, 12)), 40000, 6),
                                in_use_is(224, gaps=16)),
    "in_use_gaps_one_range": (lambda: norun(bytes(v for v in range(256) if v not in (0x70, 0x75, 0x7F)), 40000, 7),
                              in_use_is(253, gaps=1)),
    # the 17-bit limit: unlimited depths of 18 (the halving retry) and exactly 17 (no retry)
    "length_retry_a": (lambda: skewed(1, 40, 899000, 1.7), retry_runs),
    "length_retry_b": (lambda: skewed(1, 40, 899000, 1.6), retry_runs),
    "length_depth_17": (lambda: skewed(1, 24, 899000, 1.8), depth_17_no_retry),
    # selectors staged in two shared arrays split at 12 384, and the most one block allows
    "n_sel_12384": (lambda: bytes(np.random.default_rng(12384).integers(0, 256, 700000, dtype=np.uint8))[:SEL12384],
                    n_sel_is(12384)),
    "n_sel_12385": (lambda: bytes(np.random.default_rng(12384).integers(0, 256, 700000, dtype=np.uint8))[:SEL12385],
                    n_sel_is(12385)),
    "n_sel_max": (lambda: bytes(np.random.default_rng(18000).integers(0, 256, 950000, dtype=np.uint8)), max_n_sel),
    "selector_lookback": (lambda: text(300000, 11)[:150000] + norun(range(32, 128), 150000, 12), lookback),
    "unused_tables": (lambda: letters(3000, 13, k=4) + norun(range(256), 400, 14), unused_table),
    # MTF chunks: zero runs at chunk edges, a symbol absent for 6 chunks, one first seen in the last chunk but one
    "mtf_zero_runs": (lambda: zero_run_layout()[0], zero_runs_placed),
}


# RLE1 runs around the front end's 4 KiB input tiles and 128-byte sub-tiles (k_e_tile_info / k_e_tile_pre / k_e_tile_emit)
RLE_LENGTHS = (3, 4, 5, 255, 256, 259)


def rle_at_edges(period, spacing, seed):
    """Runs of every length in RLE_LENGTHS starting at e - k (k = 0..5) for edges e = multiples of `period`, then runs
    that end on the last byte before an edge, over a background without runs."""
    slots = [e for e in range(spacing, 1 << 30, spacing) if e % period == 0 and (period == TI or e % TI)]
    plan = [(e - k, L) for (L, k), e in zip([(L, k) for L in RLE_LENGTHS for k in range(6)], slots)]
    plan += [(e - L, L) for L, e in zip(RLE_LENGTHS, slots[len(plan):])]
    buf = bytearray(norun(range(0x20, 0x7F), plan[-1][0] + 2 * spacing, seed))
    for i, (s, L) in enumerate(plan):
        buf[s:s + L] = bytes([0x80 + i % 64]) * L
    return bytes(buf)


def runs_only(n, seed):
    r = random.Random(seed)
    out = bytearray()
    while len(out) < n:
        out += bytes([r.randrange(256)]) * r.choice((1, 2, 3, 4, 5, r.randrange(1, 300)))
    return bytes(out[:n])


def one_block(s, chk):
    assert len(s.blocks) == 1


CASES.update({
    "rle_tile_edges": (lambda: rle_at_edges(TI, TI, 21), one_block),
    "rle_subtile_edges": (lambda: rle_at_edges(SUB, 512, 22), one_block),
    **{"runs_len_%d" % n: (functools.partial(runs_only, n, n), one_block) for n in (4095, 4096, 4097, 8191, 8192, 8193)},
})


@functools.lru_cache(maxsize=None)
def case_input(name) -> bytes:
    return CASES[name][0]()


@functools.lru_cache(maxsize=8)
def _checked(data: bytes, z: bytes):
    assert bz2.decompress(z) == data
    return bs.check_stream(z)


def check(data: bytes, z: bytes, claim=None):
    """Byte identity with the oracle, a libbz2 round trip and the table check; then the case's own claim."""
    assert z == oracle(data)
    s, chk = _checked(data, z)
    if claim is not None:
        claim(s, chk)
    return s, chk


@pytest.mark.parametrize("name", list(CASES))
def test_edge_case(name):
    data = case_input(name)
    rc, z, _ = orc.emul_bzip2_encode(data)
    assert rc == 0
    check(data, z, CASES[name][1])


# ---------------------------------------------------------------------------------------------------------------------
# a batch of random, periodic, text, periodic and random blocks, in one batch and in several
# ---------------------------------------------------------------------------------------------------------------------
BLOCK = 899_982  # bytes of a block of runs of length 1: 899 981 RLE1 bytes plus the byte that closes the last run


def dedup_text(n, seed) -> bytes:
    t = np.frombuffer(text(n * 2, seed), np.uint8)
    t = t[np.concatenate([[True], t[1:] != t[:-1]])][:n]
    assert len(t) == n
    return t.tobytes()


def join_blocks(parts) -> bytes:
    """Every byte differs from the one before it, so each part but the last is exactly one block of BLOCK bytes and a
    periodic part starts on its period."""
    for i, (a, b) in enumerate(zip(parts, parts[1:])):
        assert len(a) == BLOCK and a[-1] != b[0]
    return b"".join(parts)


@functools.lru_cache(maxsize=None)
def mixed_input() -> bytes:
    """random | abc.. (period 3) | text | a short xy.. (period 2)"""
    return join_blocks([norun(range(0x80, 0x100), BLOCK, 32), b"abc" * (BLOCK // 3), dedup_text(BLOCK, 31),
                        b"xy" * 20_000])


MIXED_PERIODIC = 2


@functools.lru_cache(maxsize=None)
def batches_input() -> bytes:
    """random | text | random | random | a short pq.. (period 2): five blocks, the last one periodic"""
    return join_blocks([norun(range(0x80, 0x100), BLOCK, 34), dedup_text(BLOCK, 35), norun(range(0x80, 0x100), BLOCK, 36),
                        norun(range(0x80, 0x100), BLOCK, 37), b"pq" * 20_000])


def test_mixed_batch():
    """k_serial_sort re-sorts only the blocks whose rotations stay tied (the whole block of period 3 here keeps every
    doubling round busy to the end); the others keep the doubling sort's order."""
    data = mixed_input()
    rc, z, st = orc.emul_bzip2_encode(data)
    assert rc == 0
    s, _ = check(data, z)
    assert st[0] == len(s.blocks) == 4
    assert st[1] == MIXED_PERIODIC and 1 <= st[1] < st[0]


_BATCH_LIB = None


def emul_encode_batch(data: bytes, max_batch: int):
    """The encoder on the emulation with at most `max_batch` blocks per batch (0: the built-in plan), from
    tests/host_emul/bz2enc_batch_emul.cpp, rebuilt here when it or the encoder sources change.
    -> (rc, output, stats[n_blocks, n_serial_blocks, rounds, _])"""
    global _BATCH_LIB
    if _BATCH_LIB is None:
        emul = os.path.join(orc.ROOT, "tests", "host_emul")
        csrc = os.path.join(orc.ROOT, "archive_b200", "csrc")
        src = os.path.join(emul, "bz2enc_batch_emul.cpp")
        so = os.path.join(emul, "libbz2enc_batch_emul.so")
        deps = [src, os.path.join(emul, "cuda_emu.h")] + [
            os.path.join(csrc, f) for f in os.listdir(csrc) if f.startswith("bzip2_enc")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
            subprocess.run(["g++", "-O2", "-g", "-fPIC", "-shared", "-std=c++17", "-I", emul, "-I", csrc, src, "-o", so],
                           check=True)
        _BATCH_LIB = C.CDLL(so)
    cap = len(data) + len(data) // 32 + 8192
    out = (C.c_uint8 * (cap + 16))()
    n = C.c_size_t()
    st = (C.c_uint32 * 4)()
    rc = _BATCH_LIB.emu_bzip2_encode_batch(data, C.c_size_t(len(data)), out, C.c_size_t(cap), C.byref(n), st,
                                           C.c_uint32(max_batch))
    return rc, bytes(out[:n.value]), list(st)


@pytest.mark.parametrize("max_batch", [1, 2, 3, 0])
def test_several_batches(max_batch):
    """EncState (bit position, combined CRC) carried across batches (0: the built-in plan, one batch).  With 2 blocks per
    batch the last batch holds only the periodic block, behind a batch of plain ones; with 3 the last batch is partial."""
    data = batches_input()
    rc, z, st = emul_encode_batch(data, max_batch)
    assert rc == 0
    s, _ = check(data, z)
    assert st[0] == len(s.blocks) == 5 and st[1] == 1


# ---------------------------------------------------------------------------------------------------------------------
# fuzz: seeded inputs from the generators above, 0 to 2 MB
# ---------------------------------------------------------------------------------------------------------------------
def fuzz_input(seed: int) -> bytes:
    r = random.Random(seed)
    n = int(2 ** (21 * r.random() ** 4)) - 1
    kind = r.randrange(8)
    if kind == 0:
        return letters(n, seed, k=r.choice((2, 4, 16, 64)))
    if kind == 1:
        return norun(range(r.randrange(1, 64), 256), n, seed) if n else b""
    if kind == 2:
        return skewed(seed, r.randrange(2, 40), n, r.uniform(1.3, 2.5))
    if kind == 3:
        return short_runs(b"abcd"[:r.randrange(2, 5)], n, seed)
    if kind == 4:
        return text(n, seed) if n else b""
    if kind == 5:
        return runs_only(n, seed)
    if kind == 6:
        m = max(1, n // 5)
        return last_column_input(bytes(r.choice(b"AAAAB") for _ in range(m)))
    return fuzz_input(seed * 7 + 1)[: n // 2] + fuzz_input(seed * 7 + 2)[: n // 2]


N_FUZZ = 150


def test_fuzz():
    ran = 0
    for seed in range(N_FUZZ):
        data = fuzz_input(seed)
        rc, z, _ = orc.emul_bzip2_encode(data)
        assert rc == 0, seed
        check(data, z)
        ran += 1
    assert ran == N_FUZZ
