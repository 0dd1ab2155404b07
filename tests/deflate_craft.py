"""Hand-built DEFLATE streams (RFC 1951) for the inflate tests -- TEST INFRASTRUCTURE, never the product path.

zlib's encoder writes a narrow slice of DEFLATE (Huffman-optimal code sets, HLIT <= 286, HDIST <= 30, at least two
distance codes, complete code-length codes, length 258 only as code 285).  The reference decoder (inflate.dart,
_huffman_table.dart; oracle/inflate.c) accepts much more.  This writer emits any of it: explicit code-length lists of any
size, incomplete and over-subscribed sets, explicit HLIT / HDIST / HCLEN and code-length op lists, every length and
distance code with any extra bits, stored blocks with free LEN / NLEN, reserved block types, BFINAL under control.

`Unit` tracks the plaintext a decoder should produce and whether the stream stays inside what zlib itself accepts
(`zlib_ok`); a zlib-compatible stream must decompress under Python's zlib to that plaintext, which checks this writer
independently of the decoders under test."""
import random
import struct
import zlib
from fractions import Fraction

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227,
            258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32  # the writer can emit codes 30 / 31; the reference's fixed table has 30 entries (holes)
REPEAT = {16: (2, 3, 6), 17: (3, 3, 10), 18: (7, 11, 138)}  # op -> (extra bits, least, most repeats)


class BitWriter:
    """LSB-first bit packing: bits gather in a small Python int and leave 8 bytes at a time; Huffman codes go out
    MSB-first."""

    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.k = 0  # bits in acc

    @property
    def n(self):
        return 8 * len(self.out) + self.k

    def bits(self, value, n):
        assert 0 <= value < (1 << n) or n == 0 and value == 0, (value, n)
        self.acc |= value << self.k
        self.k += n
        if self.k >= 64:
            self.out += (self.acc & 0xFFFFFFFFFFFFFFFF).to_bytes(8, "little")
            self.acc >>= 64
            self.k -= 64

    def code(self, code, length):
        self.bits(int(format(code, f"0{length}b")[::-1], 2) if length else 0, length)

    def align(self):
        self.bits(0, (-self.k) % 8)

    def raw(self, data: bytes):
        assert self.k % 8 == 0
        self.out += self.acc.to_bytes(self.k // 8, "little") + bytes(data)
        self.acc = 0
        self.k = 0

    def getvalue(self) -> bytes:
        return bytes(self.out) + self.acc.to_bytes((self.k + 7) // 8, "little")


def canonical(lengths):
    """Canonical codes of RFC 1951 3.2.2 for any length list (incomplete or over-subscribed sets included: an
    over-subscribed set gets codes that overflow their length, and must not be written).  None for length 0."""
    count = [0] * 17
    for l in lengths:
        count[l] += 1
    count[0] = 0
    nxt, code = [0] * 17, 0
    for l in range(1, 17):
        code = (code + count[l - 1]) << 1
        nxt[l] = code
    out = []
    for l in lengths:
        if l:
            out.append(nxt[l])
            nxt[l] += 1
        else:
            out.append(None)
    return out


def kraft(lengths):
    return sum((Fraction(1, 1 << l) for l in lengths if l), Fraction(0))


def sub_entries(lengths, root):
    """Second-level table entries a two-level decoder with `root`-bit root tables allocates for this set: one block of
    2^(longest - root) entries for every root prefix that codes longer than `root` share (inflate_fast.cuh)."""
    deepest = {}
    for l, c in zip(lengths, canonical(lengths)):
        if l > root:
            p = c >> (l - root)
            deepest[p] = max(deepest.get(p, 0), l)
    return sum(1 << (m - root) for m in deepest.values())


def _fill(rng, units, depth, count):
    """`count` leaf lengths (<= depth) whose Kraft sum is units / 2^depth: binary decomposition, then random splits."""
    leaves = [depth - b for b in range(units.bit_length()) if units >> b & 1]
    assert len(leaves) <= count, "too few symbols for the space"
    while len(leaves) < count:
        cand = [i for i, l in enumerate(leaves) if l < depth]
        if not cand:
            break
        i = rng.choice(cand)
        leaves[i] += 1
        leaves.append(leaves[i])
    return leaves


def complete_lengths(rng, n, maxlen, forced=None, must=(), count=None, zero=()):
    """A random Kraft-complete length list for n symbols, codes no longer than maxlen.  `forced` = {symbol: length} is
    kept; the symbols in `must` get a length, those in `zero` none; `count` = how many symbols get one (default
    random)."""
    forced = dict(forced or {})
    lens = [0] * n
    for s, l in forced.items():
        lens[s] = l
    left = (1 << maxlen) - sum(1 << (maxlen - l) for l in forced.values())
    assert left >= 0, "forced lengths over-subscribe the set"
    free = [s for s in range(n) if s not in forced and s not in zero]
    if left == 0:
        return lens
    least = bin(left).count("1")
    most = min(len(free), left)
    if count is None:
        count = rng.randint(max(least, len([s for s in must if s not in forced])), most)
    leaves = _fill(rng, left, maxlen, count)
    pick = [s for s in must if s not in forced]
    rest = [s for s in free if s not in pick]
    rng.shuffle(rest)
    syms = (pick + rest)[:len(leaves)]
    rng.shuffle(leaves)
    for s, l in zip(syms, leaves):
        lens[s] = l
    return lens


def prefix_lengths(rng, n, root, k, maxlen=15, must=(), extra_splits=0):
    """A complete set whose codes longer than `root` bits lie under exactly k root prefixes (the tail of the canonical
    code space); one of them reaches maxlen.  Short codes fill the other 2^root - k prefixes."""
    short_units = (1 << root) - k
    long_units = k << (maxlen - root)
    # long part: k subtrees of depth >= root + 1, one chain down to maxlen
    longs = [root + 1] * (2 * k)
    l = root + 1
    while l < maxlen:  # turn one leaf into a chain
        longs.remove(l)
        longs += [l + 1, l + 1]
        l += 1
    for _ in range(extra_splits):
        cand = [i for i, x in enumerate(longs) if x < maxlen]
        if not cand:
            break
        i = rng.choice(cand)
        longs[i] += 1
        longs.append(longs[i])
    assert sum(1 << (maxlen - x) for x in longs) == long_units
    shorts = _fill(rng, short_units, root, min(n - len(longs), short_units)) if short_units else []
    assert len(shorts) + len(longs) <= n, "alphabet too small for this shape"
    lens = [0] * n
    order = [s for s in must] + [s for s in range(n) if s not in must]
    rest = order[len(must):]
    rng.shuffle(rest)
    order = list(must) + rest
    rng.shuffle(shorts)
    rng.shuffle(longs)
    for s, x in zip(order, shorts + longs):
        lens[s] = x
    assert kraft(lens) == 1
    return lens


def rle_ops(seq):
    """The code-length op list of a length sequence: literal lengths, (16, n), (17, n), (18, n) -- greedy, as zlib."""
    ops, i = [], 0
    while i < len(seq):
        l = seq[i]
        run = 1
        while i + run < len(seq) and seq[i + run] == l:
            run += 1
        if l == 0 and run >= 3:
            r = min(run, 138)
            ops.append((18, r) if r >= 11 else (17, r))
            i += r
            continue
        ops.append(l)
        i += 1
        run -= 1
        while run >= 3:
            r = min(run, 6)
            ops.append((16, r))
            i += r
            run -= r
    return ops


def ops_to_lens(ops, num):
    """The lengths the reference's _decode (inflate.dart:345-401) makes of an op list: 16 repeats the previous
    length, which a 17 / 18 run resets to 0.  A code-length-code hole ("hole") gives a 0 and consumes no bits, so every
    later read meets it again: the rest are 0.  None when a run passes `num`."""
    out, prev = [], 0
    for o in ops:
        if o == "hole":
            return out + [0] * (num - len(out))
        if isinstance(o, int):
            out.append(o)
            prev = o
            continue
        s, r = o
        out += [prev if s == 16 else 0] * r
        if s != 16:
            prev = 0
        if len(out) > num:
            return None
    return out


def cl_for(ops):
    """A complete code-length code over the op symbols used (balanced: as zlib requires, complete; a single used
    symbol gets a partner of the same length)."""
    used = sorted({o if isinstance(o, int) else o[0] for o in ops})
    if len(used) == 1:
        used.append(0 if used[0] else 1)
    k = (len(used) - 1).bit_length()
    short = (1 << k) - len(used)  # this many symbols one bit shorter
    lens = [0] * 19
    for j, s in enumerate(used):
        lens[s] = k - 1 if j < short else k
    return lens


class Unit:
    """One DEFLATE stream under construction, with the plaintext a reference decoder produces from it."""

    def __init__(self):
        self.w = BitWriter()
        self.plain = bytearray()
        self.zlib_ok = True
        self.blocks = 0
        self.lit = self.dist = None

    # ---------------------------------------------------------------- block headers
    def _header(self, final, btype):
        self.w.bits(1 if final else 0, 1)
        self.w.bits(btype, 2)
        self.blocks += 1

    def stored(self, data=b"", final=False, length=None, nlen=None):
        """A stored block; LEN defaults to len(data) and NLEN to ~LEN.  The plaintext grows by `data` only when LEN
        matches it (the caller owns the meaning of anything else)."""
        self._header(final, 0)
        self.w.align()
        ln = len(data) if length is None else length
        nl = (~ln & 0xffff) if nlen is None else nlen
        if nl != (~ln & 0xffff):
            self.zlib_ok = False
        self.w.bits(ln, 16)
        self.w.bits(nl, 16)
        self.w.raw(bytes(data))
        if ln == len(data):
            self.plain += data

    def fixed(self, final=False):
        self._header(final, 1)
        self._tables(FIXED_LIT, FIXED_DIST)

    def dynamic(self, lit_lens, dist_lens, final=False, cl_lens=None, ops=None, hclen=None):
        """A dynamic block.  HLIT = len(lit_lens), HDIST = len(dist_lens).  `ops` = the code-length op list (ints
        0..15, (16|17|18, repeats)); default rle_ops.  `cl_lens` = the 19 code-length-code lengths; default cl_for.
        `hclen` defaults to the least that carries every nonzero cl length."""
        hlit, hdist = len(lit_lens), len(dist_lens)
        assert 257 <= hlit <= 288 and 1 <= hdist <= 32
        if ops is None:
            ops = rle_ops(list(lit_lens) + list(dist_lens))
        if cl_lens is None:
            cl_lens = cl_for(ops)
        if hclen is None:
            hclen = max([4] + [i + 1 for i, s in enumerate(CL_ORDER) if cl_lens[s]])
        self._header(final, 2)
        self.w.bits(hlit - 257, 5)
        self.w.bits(hdist - 1, 5)
        self.w.bits(hclen - 4, 4)
        for i in range(hclen):
            self.w.bits(cl_lens[CL_ORDER[i]], 3)
        clc = canonical(cl_lens)
        for o in ops:
            if o == "hole":  # a read of a code-length-code hole: no bits, the next data bits are its bits
                continue
            s, r = (o, None) if isinstance(o, int) else o
            self.w.code(clc[s], cl_lens[s])
            if r is not None:
                nx, lo, _ = REPEAT[s]
                self.w.bits(r - lo, nx)
        self._check_zlib(lit_lens, dist_lens, cl_lens, ops, hclen)
        self._tables(lit_lens, dist_lens)

    def _check_zlib(self, lit_lens, dist_lens, cl_lens, ops, hclen):
        def ok_set(lens):  # zlib's inflate_table: complete, or a single code of length 1
            k = kraft(lens)
            return k == 1 or (k == Fraction(1, 2) and max(lens) == 1)
        first = ops[0] if ops else None
        if (len(lit_lens) > 286 or len(dist_lens) > 30 or kraft(cl_lens) != 1 or not ok_set(lit_lens)
                or not (ok_set(dist_lens) or not any(dist_lens)) or lit_lens[256] == 0
                or "hole" in ops or (isinstance(first, tuple) and first[0] == 16)):
            self.zlib_ok = False

    def _tables(self, lit_lens, dist_lens):
        self.lit = (list(lit_lens), canonical(lit_lens))
        self.dist = (list(dist_lens), canonical(dist_lens))

    def reserved(self, final=False):
        self._header(final, 3)
        self.zlib_ok = False

    # ---------------------------------------------------------------- symbols
    def sym(self, s):
        """Lit/len symbol s, as a raw code (no plaintext tracking)."""
        lens, codes = self.lit
        assert lens[s], f"lit/len symbol {s} has no code"
        self.w.code(codes[s], lens[s])
        if s > 285:
            self.zlib_ok = False

    def dsym(self, d):
        lens, codes = self.dist
        assert lens[d], f"distance symbol {d} has no code"
        self.w.code(codes[d], lens[d])
        if d > 29:
            self.zlib_ok = False

    def lit_byte(self, b):
        self.sym(b)
        self.plain.append(b)

    def literals(self, data):
        for b in data:
            self.lit_byte(b)

    def eob(self):
        self.sym(256)

    def length_part(self, length, code=None):
        """The lit/len symbol and extra bits of a match length; code 284 writes 258 as 227 + 31."""
        if code is None:
            code = 285 if length == 258 else max(c for c in range(257, 285) if LEN_BASE[c - 257] <= length)
        x = length - LEN_BASE[code - 257]
        assert 0 <= x < (1 << LEN_EXTRA[code - 257]) or (code == 284 and x == 31), (length, code)
        if code == 284 and x == 31:
            self.zlib_ok = False
        self.sym(code)
        self.w.bits(x, LEN_EXTRA[code - 257])

    def match(self, length, dist, len_code=None):
        """A (length, distance) pair copied from the plaintext so far (distance <= its length)."""
        assert 1 <= dist <= len(self.plain) and dist <= 32768, (dist, len(self.plain))
        self.length_part(length, len_code)
        d = max(c for c in range(30) if DIST_BASE[c] <= dist)
        self.dsym(d)
        self.w.bits(dist - DIST_BASE[d], DIST_EXTRA[d])
        for _ in range(length):
            self.plain.append(self.plain[-dist])

    def copy_plain(self, length, dist):
        """Track a copy the decoder makes without writing anything (a distance read from a hole: distance 1)."""
        for _ in range(length):
            self.plain.append(self.plain[-dist])

    def bits(self, v, n):
        self.w.bits(v, n)

    def align(self):
        self.w.align()

    def data(self) -> bytes:
        return self.w.getvalue()

    def lit_syms(self):
        """Literal bytes that have a code in the current block."""
        return [s for s in range(256) if self.lit[0][s]]

    def dist_syms(self):
        return [d for d in range(min(30, len(self.dist[0]))) if self.dist[0][d]]


# ---------------------------------------------------------------- whole units
def zlib_inflate(raw: bytes):
    """Python's zlib on a raw stream -> (output, reached the final block)."""
    d = zlib.decompressobj(-15)
    return d.decompress(raw) + d.flush(), d.eof


def random_symbols(u: Unit, rng, n_out, match_frac=0.3, long_first=False):
    """Literals and matches drawn from the current block's codes until ~n_out plaintext bytes were added.  Matches
    use only distance codes the block has and distances the plaintext allows."""
    lits = u.lit_syms()
    lens = [c for c in range(257, min(286, len(u.lit[0]))) if u.lit[0][c]]
    dsyms = u.dist_syms()
    if long_first:  # frequent symbols with long codes
        lits.sort(key=lambda s: -u.lit[0][s])
        lits = lits[:max(1, len(lits) // 3)] * 3 + lits
    target = len(u.plain) + n_out
    while len(u.plain) < target:
        if lens and dsyms and rng.random() < match_frac and len(u.plain) > 0:
            lc = rng.choice(lens)
            lo = LEN_BASE[lc - 257]
            ln = 258 if lc == 285 else lo + rng.randrange(1 << LEN_EXTRA[lc - 257])
            ok = [d for d in dsyms if DIST_BASE[d] <= min(len(u.plain), 32768)]
            if ok:
                d = rng.choice(ok)
                hi = min(len(u.plain), 32768, DIST_BASE[d] + (1 << DIST_EXTRA[d]) - 1)
                u.match(ln, rng.randint(DIST_BASE[d], hi), lc)
                continue
        u.lit_byte(rng.choice(lits))


def gzip_member(raw: bytes, plain: bytes, hint: bool) -> bytes:
    """A gzip member around a raw DEFLATE unit, laid out as synth.gzip_member (with or without the BGZF 'BC' size
    hint), trailer = CRC-32 and size of `plain`."""
    trailer = struct.pack("<II", zlib.crc32(plain) & 0xffffffff, len(plain) & 0xffffffff)
    if hint:
        total = 10 + 2 + 6 + len(raw) + 8
        assert total <= 65536
        hdr = b"\x1f\x8b\x08\x04" + b"\0\0\0\0" + b"\x00\xff" + struct.pack("<H", 6) + b"BC" + struct.pack("<HH", 2, total - 1)
        return hdr + raw + trailer
    return b"\x1f\x8b\x08\x00" + b"\0\0\0\0" + b"\x00\xff" + raw + trailer


def zip_of(units):
    """A .zip whose deflated members are the given (name, raw, plain) units (synth.zip_from_deflated)."""
    from archive_b200 import synth
    return synth.zip_from_deflated([(n, r, zlib.crc32(p) & 0xffffffff, len(p)) for n, r, p in units])
