"""Edge catalogue of the device Deflate encoder's per-block stage (archive_b200/csrc/deflate_kernels.cu: k_defl_cut places
the block cuts, k_defl_block_trees builds the three Huffman trees and picks the block kind) on the CUDA execution-model
emulation.  Every case, at every level it runs, must give the oracle's bytes, have the emulation's token and block counts
equal to the stream's, decode to the input through tests/deflate_stream.py and pass that file's table check: each
block's code lengths, header and size are those the restated tree builder makes of the block's own histograms.

Each case also asserts, from the parsed stream, the edge it is there for, so that an input which drifts off its edge
fails instead of passing quietly:
  - the 15-bit limit: lit/len and distance trees whose depth without the limit is 15 (no repair), 16 and 18 (overflow 6,
    the repair loop runs three times); the 18-deep lit/len tree again at window bits 12;
  - small trees: no matches, exactly one distance code (0, 1, 2, 29), EOB plus one literal, the empty input;
  - block-kind ties: static at static_lenb == opt_lenb, dynamic at static_lenb == opt_lenb + 1, stored at
    stored_len + 4 == min(opt_lenb, static_lenb), not stored one byte later;
  - _scanTree's run codes at their limits, in the lit/len and in the distance part;
  - block cuts: the heuristic cut at 8192 tokens (levels above 2), full cuts at 16383 tokens, final blocks of 16382,
    16383 (the last pending literal keeps it in one block at levels 4-9) and 16384 tokens.
tests/test_deflate_enc_edges_gpu.py runs the same catalogue on the device.

The designed inputs are back-to-back matches copied from a random history with no repeated 3-byte string.  Each copy's
source is the latest position with its hash (15 bits, as the encoder's default memory level gives), is inserted in the
hash chains at every level, and neither that match nor the one a position later can be longer than designed -- so the
encoder's tokens are the designed ones at every level, which the parsed histograms then confirm."""
import functools
import random

import pytest

import deflate_stream as ds
import oracle_lib as orc

LEVELS = (1, 3, 4, 6, 9)
MAX_DIST = {15: 32768 - 262, 12: 4096 - 262, 9: 512 - 262}


# ---------------------------------------------------------------------------------------------------------------------
# construction
# ---------------------------------------------------------------------------------------------------------------------
def unique_history(n: int, seed: int, alphabet=range(256)) -> bytes:
    """n random bytes over `alphabet` with no 3-byte string twice: the encoder can only code them as literals."""
    r = random.Random(seed)
    alphabet = list(alphabet)
    out, seen, misses = bytearray(r.choice(alphabet) for _ in range(2)), set(), 0
    while len(out) < n:
        b = r.choice(alphabet)
        g = (out[-2], out[-1], b)
        if g not in seen:
            seen.add(g)
            out.append(b)
            misses = 0
        else:
            misses += 1
            if misses > 64 * len(alphabet):
                raise ValueError("the alphabet has no 3-byte string left to extend with")
    return bytes(out[:n])


def no_repeated_3(d: bytes) -> bool:
    return len({d[i:i + 3] for i in range(len(d) - 2)}) == max(len(d) - 2, 0)


def copies(hist: bytes, toks, max_dist: int, seed: int) -> bytes:
    """`hist` followed by one match per (length, (dmin, dmax)) of `toks`, in order (see the module docstring)."""
    r = random.Random(seed)
    data = bytearray(hist)
    hv = lambda i: ((data[i] << 10) ^ (data[i + 1] << 5) ^ data[i + 2]) & 0x7FFF
    last = {hv(i): i for i in range(len(data) - 2)}
    hashed = bytearray(b"\1" * len(data))  # inserted in the hash chains at every level (levels 1-3 skip long matches)
    prev = None
    for length, (dlo, dhi) in toks:
        p = len(data)
        dhi = min(dhi, max_dist, p - 1, 4096 if length == 3 else p)
        for _ in range(20000):
            d = r.randint(max(dlo, length), dhi)
            s = p - d
            if not hashed[s] or last.get(hv(s)) != s:
                continue
            if prev is None and p >= 2:  # after literals: no match may start one or two bytes early
                edge = bytes(data[p - 2:p]) + bytes(data[s:s + 2])
                if data[s - 1] == data[p - 1] or edge[:3] in data[:p] or edge[1:] in data[:p]:
                    continue
            if prev:
                pp, pl = prev
                cur = bytes(data[pp:p]) + bytes(data[s:s + 2])
                if cur[:pl + 1] in data[max(0, pp - max_dist):p - 1] or cur[1:pl + 2] in data[max(0, pp + 1 - max_dist):p]:
                    continue
            break
        else:
            raise AssertionError("no source for a designed match")
        data += data[s:s + length]
        hashed += b"\1" * length if length <= 4 else b"\1" + b"\0" * (length - 1)
        for i in range(max(p - 2, 0), p + length - 2):
            last[hv(i)] = i
        prev = (p, length)
    return bytes(data)


def chain(k: int, margin: float):
    """k counts, increasing, each larger than the sum of all but the previous one by 1 + margin of that sum: the
    Huffman tree of such counts is a chain k - 1 deep, whatever the tie-break."""
    c = [1, 1, 1]
    while len(c) < k:
        s = sum(c[:-1])
        c.append(s + 1 + int(margin * s))
    return c[:k]


# lit/len: EOB (count 1) and k - 1 length codes; distance: k distance codes
DEPTH_PLANS = {15: (16, 0.5), 16: (17, 0.3), 18: (19, 0.05)}


def full_block(c):
    """the counts with the largest raised so that they fill one block of 16383 tokens"""
    return c[:-1] + [c[-1] + 16383 - sum(c)]


@functools.lru_cache(maxsize=None)
def litlen_depth_input(depth: int, wbits: int = 15, segment=None) -> bytes:
    """segment 0 / 1: the history over bytes 0x00-0x7f / 0x80-0xff and the designed matches filling one block of
    16383 tokens, so that segments of the two alphabets can follow one another without matches across them"""
    k, margin = DEPTH_PLANS[depth]
    c = chain(k, margin)[1:]  # the first count is EOB's
    if segment is not None:
        c = full_block(c)
    toks = []
    for i, x in enumerate(sorted(c, reverse=True)):  # the most frequent codes are the shortest lengths
        toks += [(ds.LEN_BASE[i], (1, 1 << 15))] * x
    random.Random(depth).shuffle(toks)
    alphabet = range(256) if segment is None else range(128 * segment, 128 * segment + 128)
    hist = unique_history(16383, 10 + depth, alphabet)
    return copies(hist, toks, MAX_DIST[wbits], depth)


@functools.lru_cache(maxsize=None)
def dist_depth_input(depth: int, segment=None) -> bytes:
    k, margin = DEPTH_PLANS[depth]
    c = chain(k, margin)
    if segment is not None:
        c = full_block(c)
    codes = list(range(30 - len(c), 30))
    toks = []
    for code, x in zip(codes, sorted(c)):
        toks += [(4, (ds.DIST_BASE[code], ds.DIST_BASE[code] + (1 << ds.DIST_EXTRA[code]) - 1))] * x
    random.Random(depth).shuffle(toks)
    alphabet = range(256) if segment is None else range(128 * segment, 128 * segment + 128)
    return copies(unique_history(2 * 16383, 20 + depth, alphabet), toks, MAX_DIST[15], depth)


# ---------------------------------------------------------------------------------------------------------------------
# the check
# ---------------------------------------------------------------------------------------------------------------------
def encode(data: bytes, level: int, wbits: int = 15):
    rc, out, stats = orc.emul_deflate_raw(data, level, wbits)
    assert rc == 0, rc
    return out, stats


def check(data: bytes, z: bytes, level: int, wbits: int = 15, stats=None):
    """-> (Stream, plans).  The oracle's bytes, the input back, the table check; with the emulation's stats, its token
    and block counts."""
    st, ref, _ = orc.deflate(data, level, wbits)
    assert st == orc.OK and z == ref, (len(data), level, wbits, len(z), len(ref))
    s, plans = ds.check_stream(z, data, 1 << wbits)
    if stats is not None:
        assert stats[1] == len(s.blocks), (stats, len(s.blocks))
        if not any(b.btype == 0 for b in s.blocks):  # (a stored block's tokens are not in the stream)
            assert stats[0] == s.ntok, (stats, s.ntok)
    return s, plans


def run(data: bytes, level: int, wbits: int = 15):
    z, stats = encode(data, level, wbits)
    return check(data, z, level, wbits, stats)


def coded(s, plans):
    return [(b, p) for b, p in zip(s.blocks, plans) if p is not None]


# ---------------------------------------------------------------------------------------------------------------------
# edge claims: each takes (Stream, plans, level) and asserts on the parsed stream
# ---------------------------------------------------------------------------------------------------------------------
def litlen_depth(want):
    def claim(s, plans, level):
        b, p = coded(s, plans)[-1]
        assert b.btype == 2 and sum(b.lit_hist[:256]) == 0, "the designed block: dynamic, matches only"
        assert p.lt.depth == want and max(b.ll_lens) == min(want, 15), (p.lt.depth, max(b.ll_lens))
        assert (p.lt.overflow > 0) == (want > 15) and (want != 18 or p.lt.overflow >= 3), p.lt.overflow
        return p.lt.depth
    return claim


def dist_depth(want):
    def claim(s, plans, level):
        b, p = coded(s, plans)[-1]
        assert b.btype == 2 and sum(b.lit_hist[:256]) == 0, "the designed block: dynamic, matches only"
        assert p.dt.depth == want and max(b.d_lens) == min(want, 15), (p.dt.depth, max(b.d_lens))
        assert (p.dt.overflow > 0) == (want > 15) and b.hdist == 30, (p.dt.overflow, b.hdist)
        if want == 18:
            assert p.dt.overflow >= 3
        return p.dt.depth
    return claim


CASES = {}


def case(name, make, claim, levels=LEVELS, wbits=15):
    CASES[name] = (make, claim, levels, wbits)


for _d in (15, 16, 18):
    case(f"litlen_depth_{_d}", functools.partial(litlen_depth_input, _d), litlen_depth(_d))
    case(f"dist_depth_{_d}", functools.partial(dist_depth_input, _d), dist_depth(_d))
for _w in (12,):
    case(f"litlen_depth_18_wbits{_w}", functools.partial(litlen_depth_input, 18, _w), litlen_depth(18), wbits=_w)


# small trees -------------------------------------------------------------------------------------------------------
def lit_block(n, seed, alphabet=range(0x61, 0x71)):
    return unique_history(n, seed, alphabet)


def with_pattern(pattern: bytes, n=400, seed=3):
    """letters with no repeated 3-byte string, `pattern` (bytes outside their alphabet) in the middle"""
    d = lit_block(n, seed)
    return d[:n // 2] + pattern + d[n // 2:]


def far_copy():
    """one 40-byte copy at distance 25 000 (distance code 29) after literals only"""
    d = unique_history(25_100, 29, range(0x40, 0x80))
    return d + d[100:140]


def no_matches(s, plans, level):
    for b, p in coded(s, plans):
        assert b.matches == 0 and p.dt.lens[:2] == [1, 1] and p.dt.max_code == 1
        if b.btype == 2:
            assert b.hdist == 2 and b.d_lens == [1, 1]
    assert any(b.btype == 2 for b in s.blocks)


def one_dist_code(code):
    want = {0: [1, 1], 1: [0, 1, 1], 2: [1, 0, 1], 29: [1] + [0] * 28 + [1]}[code]  # padded to two codes

    def claim(s, plans, level):
        b, p = [(b, p) for b, p in coded(s, plans) if b.matches][-1]
        assert [c for c in range(30) if b.dist_hist[c]] == [code], b.dist_hist
        assert b.btype == 2 and b.d_lens == want, (b.btype, b.d_lens)
    return claim


def eob_plus_one_literal(s, plans, level):
    (b, p), = coded(s, plans)
    assert [c for c in range(286) if b.lit_hist[c]] == [0x61, 256] and b.ntok == 2
    assert [c for c in range(286) if p.lt.lens[c]] == [0x61, 256] and p.lt.max_code == 256 and p.dt.max_code == 1


def empty(s, plans, level):
    (b, p), = coded(s, plans)
    assert b.btype == 1 and b.ntok == 0 and b.end_bit - b.first_bit == 10
    assert [c for c in range(286) if p.lt.lens[c]] == [0, 256]  # EOB padded with code 0


case("no_matches", functools.partial(lit_block, 3000, 1), no_matches)
case("one_dist_code_0", functools.partial(with_pattern, b"\xf0" * 20), one_dist_code(0))
case("one_dist_code_1", functools.partial(with_pattern, b"\xf0\xf1" * 10), one_dist_code(1))
case("one_dist_code_2", functools.partial(with_pattern, b"\xf0\xf1\xf2" * 7), one_dist_code(2))
# (levels 1-3 also find a second, shorter match there: their chains are 4 to 32 long)
case("one_dist_code_29", far_copy, one_dist_code(29), levels=(4, 6, 9))
case("eob_plus_one_literal", lambda: b"aa", eob_plus_one_literal)
case("empty", lambda: b"", empty)


# block-kind ties: literals only (no 3-byte string twice), so the tokens are the input's bytes at every level.  Found by
# a seeded search over (seed, alphabet size, first byte, length) with the restated tree builder.
TIES = {"static_tie": (444, 16, 73, 33), "dynamic_by_one": (247, 24, 86, 41), "stored_tie": (0, 128, 107, 21),
        "not_stored_by_one": (44, 128, 29, 91)}


def tie_input(name):
    seed, k, lo, n = TIES[name]
    return unique_history(n, seed, range(lo, lo + k))


def tie(name):
    def claim(s, plans, level):
        d = s.data
        assert no_repeated_3(d) and len(s.blocks) == 1
        lh = [0] * ds.L_CODES
        for x in d:
            lh[x] += 1
        p = ds.plan(lh, [0] * ds.D_CODES)
        b = s.blocks[0]
        if b.btype:
            assert b.ntok == len(d) and plans[0].opt_len == p.opt_len
        m = min(p.opt_lenb, p.static_lenb)
        if name == "static_tie":
            assert b.btype == 1 and p.static_lenb == p.opt_lenb
        elif name == "dynamic_by_one":
            assert b.btype == 2 and p.static_lenb == p.opt_lenb + 1
        elif name == "stored_tie":
            assert b.btype == 0 and len(d) + 4 == m
        else:
            assert b.btype != 0 and len(d) + 4 == m + 1
    return claim


for _n in TIES:
    case(_n, functools.partial(tie_input, _n), tie(_n))


# block cuts ---------------------------------------------------------------------------------------------------------
def text(n, seed):
    from archive_b200 import synth
    return synth.text(n, stream=seed).tobytes()


def compressible_literals():
    """two fresh letters, then a 30-byte copy: fewer matches than half the tokens, and under half the input's size"""
    r = random.Random(81)
    d = bytearray(unique_history(20_000, 81, range(0x40, 0x80)))
    while len(d) < 150_000:
        d += bytes(r.randrange(0x40, 0x80) for _ in range(2))
        s = len(d) - r.randint(1000, 30_000)
        d += d[s:s + 30]
    return bytes(d)


def heuristic_cut(s, plans, level):
    nt = [b.ntok for b in s.blocks]
    if level > 2:
        assert 8192 in nt[:-1], nt
    else:
        assert 8192 not in nt and set(nt[:-1]) == {16383}, nt


def final_block(n_final):
    """literal-only inputs (64 letters: dynamic blocks) of 16383 + n_final bytes: one token per byte"""
    def claim(s, plans, level):
        nt = [b.ntok for b in s.blocks]
        assert all(b.btype == 2 for b in s.blocks if b.ntok > 1) and nt[0] == 16383, nt
        want = {16382: [16382], 16383: [16383] if level >= 4 else [16383, 0], 16384: [16383, 1]}[n_final]
        assert nt[1:] == want, (level, nt)  # at levels 4-9 the last literal is pending: the cut it asks for is dropped
    return claim


case("heuristic_cut_8192", compressible_literals, heuristic_cut, levels=(2, 3, 4, 6, 9))
for _n in (16382, 16383, 16384):
    case(f"final_block_{_n}", functools.partial(lit_block, 16383 + _n, 40, range(0x40, 0x80)), final_block(_n))


# _scanTree runs -------------------------------------------------------------------------------------------------------
def runs_input(first: int, dist_codes, seed: int) -> bytes:
    """Literals (no 3-byte string twice) over a set that starts at byte `first` and has gaps of 3, 10 and 11 values and
    ten neighbours, all in one block with the 4-byte matches that follow, 64 per distance code of `dist_codes`: equal counts, equal code lengths."""
    lits = [first, first + 4, first + 15, first + 27] + list(range(first + 28, first + 38)) + list(range(first + 40, first + 110))
    r = random.Random(seed)
    hist = unique_history(16_300, seed, lits)
    toks = [(4, (ds.DIST_BASE[c], ds.DIST_BASE[c] + (1 << ds.DIST_EXTRA[c]) - 1)) for c in dist_codes for _ in range(64)]
    r.shuffle(toks)
    return copies(hist, toks, MAX_DIST[15], seed)


def runs_claim(first, ll_want, d_want):
    def claim(s, plans, level):
        assert [b.btype for b in s.blocks] == [2, 2]  # the literals, then the matches
        ll = {x for b in s.blocks for x in b.runs_ll}
        dd = {x for b in s.blocks for x in b.runs_d}
        for want, got, part in ((ll_want, ll, "lit/len"), (d_want, dd, "distance")):
            assert set(want) <= got, (part, sorted(set(want) - got), got)
        hs = [b.header_syms for b in s.blocks]
        assert any(h[i] == (18, 138) and h[i + 1] == (0, 0) for h in hs for i in range(len(h) - 1)) == (first == 139)
    return claim


RUNS_A = (138, list(range(6, 13)) + [16, 27])  # distance zeros: 0-5, 13-15, 17-26
RUNS_B = (139, list(range(6, 13)) + list(range(24, 28)))  # distance zeros: 0-5, 13-23
case("scan_runs_a", functools.partial(runs_input, *RUNS_A, 61),
     runs_claim(138, [(18, 138), (17, 3), (17, 10), (18, 11), (16, 3)], [(17, 6), (17, 10), (17, 3)]))
case("scan_runs_b", functools.partial(runs_input, *RUNS_B, 62),
     runs_claim(139, [(18, 138), (17, 3), (17, 10), (18, 11), (16, 3), (16, 4), (16, 6)], [(17, 6), (18, 11)]))


def parts(b):
    """a dynamic block's code-length symbols, split into the lit/len part and the distance part"""
    n, i, h = 0, 0, b.header_syms
    while n < b.hlit:
        n += h[i][1] or 1
        i += 1
    return h[:i], h[i:]


def runs_exact_input(seed=64) -> bytes:
    """Literals in groups of 3, 4, 5, 6 and 10 neighbouring byte values and three single ones, a gap after each, every
    one 250 times, and one more literal 249 times (no 3-byte string twice); then 500 matches of 4 bytes per distance
    code 9-24.  The 249 pairs with EOB, so the other 31 literals and one node make 32 equal subtrees under the length
    code's 8000: every literal is 6 bits long, every distance code 4 -- groups of equal lengths, as designed."""
    lh = [0] * 256
    lh[0x20] = 249
    v = 0x41
    for g in (3, 4, 5, 6, 10, 1, 1, 1):
        for x in range(v, v + g):
            lh[x] = 250
        v += g + 1
    hist = histogram_sequence(lh, seed)
    toks = [(4, (ds.DIST_BASE[c], ds.DIST_BASE[c] + (1 << ds.DIST_EXTRA[c]) - 1)) for c in range(9, 25) for _ in range(500)]
    random.Random(seed).shuffle(toks)
    return copies(hist, toks, MAX_DIST[15], seed)


def repeats(s, plans, level):
    (b, p), = coded(s, plans)
    ll, dd = parts(b)
    for part, h in (("lit/len", ll), ("distance", dd)):
        pairs = list(zip(h, h[1:]))
        # a run of 7 equal lengths after a different one: the length, then 16 for the other six
        assert any(x[0] < 16 and x[0] and y == (16, 6) for x, y in pairs), (part, h)
        # the same length goes on: 16 straight after 16, no length before it (curlen == prevlen)
        assert any(x == (16, 6) and y[0] == 16 for x, y in pairs), (part, h)
    assert {(16, 3), (16, 4), (16, 5), (16, 6)} <= set(b.runs_ll), b.runs_ll


case("scan_repeats", runs_exact_input, repeats)


# the 7-bit limit of the bit-length tree: literals only, with a histogram found by a seeded search with the restated
# builder -- Zipf-like counts over a random set of byte values, so that the counts of the code-length values grow
# like a chain.  (A search checked by the reader: no 3-byte string twice, so the tokens are the input's bytes.)
def zipf_histogram(seed):
    r = random.Random(seed)
    nsym, n, a = r.randint(120, 256), r.randint(3000, 16000), r.uniform(0.6, 2.5)
    w = [1 / (i + 1) ** a for i in range(nsym)]
    f = [max(1, round(n * x / sum(w))) for x in w]
    lh = [0] * 256
    for v, x in zip(r.sample(range(256), nsym), f):
        lh[v] = x
    return lh


def histogram_sequence(lh, seed) -> bytes:
    """the bytes of histogram `lh` in an order with no 3-byte string twice"""
    r = random.Random(seed)
    seq = [v for v in range(256) for _ in range(lh[v])]
    r.shuffle(seq)
    seen = set()
    for i in range(2, len(seq)):
        for _ in range(200):
            g = (seq[i - 2], seq[i - 1], seq[i])
            if g not in seen:
                break
            j = r.randrange(i, len(seq))
            seq[i], seq[j] = seq[j], seq[i]
        else:
            raise AssertionError("no order without a repeated 3-byte string")
        seen.add(g)
    return bytes(seq)


BL_SEEDS = {7: 23, 9: 145}  # the bit-length tree's depth without the limit


@functools.lru_cache(maxsize=None)
def bitlen_input(depth):
    return histogram_sequence(zipf_histogram(BL_SEEDS[depth]), BL_SEEDS[depth])


def bitlen_depth(want):
    def claim(s, plans, level):
        (b, p), = coded(s, plans)
        assert b.btype == 2 and b.matches == 0 and b.ntok == len(s.data)
        assert p.blt.depth == want and max(b.bl_lens) == 7, (p.blt.depth, b.bl_lens)
        assert (p.blt.overflow > 0) == (want > 7), p.blt.overflow
        return p.blt.depth
    return claim


for _w in (15, 12, 9):
    for _d in BL_SEEDS:
        case(f"bitlen_depth_{_d}" + ("" if _w == 15 else f"_wbits{_w}"), functools.partial(bitlen_input, _d),
             bitlen_depth(_d), wbits=_w)


# the heuristic cut's match test (matches < last_lit / 2 at 8192 tokens): a block of 16383 literals, then a block that
# starts with 4096 or 4097 more literals and goes on with long matches -- so 4096 or 4095 of its first 8192 tokens are
# matches, and they cover enough bytes for the size test to hold
@functools.lru_cache(maxsize=None)
def matches_at_8192_input(n_matches):
    hist = unique_history(16383 + 8192 - n_matches, 70)
    r = random.Random(71)
    toks = [(r.choice([4, 4, 10, 17]), (1, 1 << 15)) for _ in range(14000)]
    return copies(hist, toks, MAX_DIST[15], 72)


def matches_at_8192(n_matches):
    def claim(s, plans, level):
        b = s.blocks[1]
        assert s.blocks[0].nbytes == 16383 and sum(b.lit_hist[:256]) == 8192 - n_matches  # block 0: 16383 literals
        if level > 2 and n_matches < 4096:
            assert b.ntok == 8192 and b.matches == n_matches, (b.ntok, b.matches)
        else:  # 4096 is not fewer than half: the block runs on to the full cut
            assert b.ntok == 16383 and b.matches_8192 == n_matches, (b.ntok, b.matches_8192)
    return claim


for _m in (4095, 4096):
    case(f"matches_{_m}_at_8192", functools.partial(matches_at_8192_input, _m), matches_at_8192(_m), levels=(2, 3, 4, 6, 9))


@pytest.mark.parametrize("name", list(CASES))
def test_edge_case(name):
    make, claim, levels, wbits = CASES[name]
    data = make()
    for level in levels:
        s, plans = run(data, level, wbits)
        claim(s, plans, level)


def fuzz_input(seed: int) -> bytes:
    """literals from a random alphabet mixed with copies of geometric length and distance"""
    r = random.Random(seed)
    n = r.choice([0, 1, 100, 3000, r.randrange(1, 300_000)])
    k = r.choice([4, 16, 64, 256])
    p_match, mean_len, mean_dist = r.uniform(0.05, 0.9), r.choice([4, 8, 30, 120]), r.choice([8, 200, 5000])
    d = bytearray()
    while len(d) < n:
        if d and r.random() < p_match:
            dist = min(len(d), 1 + int(r.expovariate(1 / mean_dist)))
            ln = min(258, 3 + int(r.expovariate(1 / mean_len)))
            for _ in range(ln):
                d.append(d[-dist])
        else:
            d.append(r.randrange(k))
    return bytes(d[:n])


def deep_fuzz_input(seed: int) -> bytes:
    """a designed block of matches with a random chain of counts (16 to 19 codes, random margin), lengths or distances"""
    r = random.Random(seed)
    c = chain(r.randint(16, 19), r.uniform(0.0, 0.08))
    c[-1] += r.randrange(200)
    if r.random() < 0.5:
        toks = [(ds.LEN_BASE[i], (1, 1 << 15)) for i, x in enumerate(sorted(c[1:], reverse=True)) for _ in range(x)]
        hist = unique_history(16383, seed)
    else:
        toks = [(4, (ds.DIST_BASE[k], ds.DIST_BASE[k] + (1 << ds.DIST_EXTRA[k]) - 1))
                for k, x in zip(range(30 - len(c), 30), sorted(c)) for _ in range(x)]
        hist = unique_history(2 * 16383, seed)
    r.shuffle(toks)
    return copies(hist, toks, MAX_DIST[15], seed)


def test_fuzz():
    r = random.Random(0xF00D)
    n_blocks = n_dyn = n_repaired = 0
    for seed in range(100):
        data = fuzz_input(seed) if seed % 10 else deep_fuzz_input(seed)
        level, wbits = r.choice([1, 2, 3, 4, 5, 6, 7, 8, 9]), r.choice([15, 15, 9, 12, 14])
        if seed % 10 == 0:
            wbits = 15
        s, plans = run(data, level, wbits)
        n_blocks += len(s.blocks)
        n_dyn += sum(b.btype == 2 for b in s.blocks)
        n_repaired += sum(1 for p in plans if p and (p.lt.overflow or p.dt.overflow or p.blt.overflow))
    assert n_blocks >= 80 and n_dyn >= 40 and n_repaired >= 8, (n_blocks, n_dyn, n_repaired)


def test_reached_depths():
    """The deepest trees the catalogue makes, before the limit: lit/len 18, distance 18 (the 15-bit repair runs),
    bit-length 9 (the 7-bit repair runs)."""
    got = {}
    for name, kind in (("litlen_depth_18", "lt"), ("dist_depth_18", "dt"), ("litlen_depth_18_wbits12", "lt"),
                       ("bitlen_depth_9", "blt")):
        make, claim, levels, wbits = CASES[name]
        s, plans = run(make(), 6, wbits)
        got[name] = getattr(coded(s, plans)[-1][1], kind).depth
    assert got == {"litlen_depth_18": 18, "dist_depth_18": 18, "litlen_depth_18_wbits12": 18, "bitlen_depth_9": 9}, got


def test_reader_rejects():
    """The stream reader is part of the check: it must refuse what a decoder refuses."""
    z = orc.deflate(text(20_000, 4), 6)[1]
    ds.parse(z)
    assert ds.parse(b"\x01\x05\x00\xfa\xff" + b"x" * 5).data == b"x" * 5
    # a byte after the final block, set padding bits after it or before a stored block's LEN, a truncated stream
    for bad in (z + b"\0", z[:-1] + bytes([z[-1] | 0x80]) if z[-1] < 0x80 else None, b"\x09\x05\x00\xfa\xff" + b"x" * 5,
                b"\x05\x00", b"\x03"):
        if bad is None:
            continue
        with pytest.raises(ds.StreamError):
            ds.parse(bad)
    # a distance past the start of the output: static block, literal 'a', match length 3 at distance 2
    with pytest.raises(ds.StreamError):
        ds.parse(_static_stream([("lit", 0x61), ("match", 3, 2)]))
    ds.parse(_static_stream([("lit", 0x61), ("match", 3, 1)]))
    # an over-subscribed and an incomplete lit/len code
    with pytest.raises(ds.StreamError, match="over-subscribed"):
        ds._table([1, 1, 1], "x")
    with pytest.raises(ds.StreamError, match="incomplete"):
        ds._table([1, 2], "x")
    ds._table([1], "distance", one_code_ok=True)
    with pytest.raises(ds.StreamError, match="incomplete"):
        ds._table([1], "lit/len")


def _static_stream(toks) -> bytes:
    """a final static block of `toks`, written bit by bit"""
    out = [1, 1, 0]  # BFINAL, BTYPE = 01

    def code(sym):
        ln = ds.STATIC_LL[sym]
        c = [0x30 + sym, 0x190 + sym - 144, sym - 256, 0xC0 + sym - 280][(sym >= 144) + (sym >= 256) + (sym >= 280)]
        out.extend((c >> (ln - 1 - i)) & 1 for i in range(ln))

    for t in toks:
        if t[0] == "lit":
            code(t[1])
        else:
            lc = ds.length_code(t[1])
            code(lc)
            out.extend((t[1] - ds.LEN_BASE[lc - 257]) >> i & 1 for i in range(ds.LEN_EXTRA[lc - 257]))
            dc = ds.dist_code(t[2])
            out.extend((dc >> (4 - i)) & 1 for i in range(5))
            out.extend((t[2] - ds.DIST_BASE[dc]) >> i & 1 for i in range(ds.DIST_EXTRA[dc]))
    code(256)
    out += [0] * (-len(out) % 8)
    return bytes(sum(out[i + j] << j for j in range(8)) for i in range(0, len(out), 8))
