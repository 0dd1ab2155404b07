"""TEST INFRASTRUCTURE: an independent reader of raw DEFLATE streams and a restatement of the zlib-lineage tree builder.

`parse(stream, window)` reads a raw DEFLATE stream (RFC 1951) without zlib or the oracle.  For every block it returns BFINAL,
BTYPE and the block's first and end bit; for a stored block LEN; for a dynamic block HLIT, HDIST, HCLEN, the bit-length code
lengths, the lit/len and distance code lengths and the run-length symbols (16, 17, 18 with their repeat counts) of the
lit/len part and of the distance part; for static and dynamic blocks the token count, the lit/len histogram (EOB = 1), the
distance-code histogram and the sum of distance extra bits.  Every block knows which bytes of the output it decodes to.
It rejects over-subscribed and incomplete codes (except a distance code of one code, which RFC 1951 allows), distances
beyond the window or the output, non-zero padding bits and bytes after the final block.

`build_tree(freq, kind)` restates the encoder's _buildTree / _genBitlen (deflate.dart; zlib's trees.c is the same
algorithm): a heap ordered by frequency, then by depth; trees with fewer than two used codes padded to two; code lengths
limited to 15 bits (7 for the bit-length tree) with the overflow repair.  It returns the limited lengths, the depth the
tree had before the limit and the overflow count.  `plan(lit_hist, dist_hist)` adds _scanTree, the bit-length tree,
max_blindex, opt_len and static_len; `check_block(block, w_size)` asserts that a parsed block is what that plan makes of
its own histograms.
"""
from dataclasses import dataclass, field

L_CODES, D_CODES, BL_CODES, MAX_BITS, MAX_BL_BITS, HEAP_SIZE = 286, 30, 19, 15, 7, 2 * 286 + 1
MIN_LOOKAHEAD = 258 + 3 + 1
BL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
DIST_EXTRA = [0, 0, 0, 0] + [k for k in range(1, 14) for _ in (0, 1)]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
BL_EXTRA = [0] * 16 + [2, 3, 7]
STATIC_LL = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
STATIC_D = [5] * 30


def length_code(length: int) -> int:
    """lit/len symbol (257..285) of a match length 3..258"""
    if length == 258:
        return 285
    return 257 + max(i for i in range(28) if LEN_BASE[i] <= length)


def dist_code(dist: int) -> int:
    return max(i for i in range(30) if DIST_BASE[i] <= dist)


class StreamError(ValueError):
    pass


class BitReader:
    def __init__(self, data: bytes):
        self.data = data + b"\0" * 8
        self.n = len(data) * 8
        self.pos = 0

    def peek(self, k: int) -> int:  # k <= 25
        p = self.pos
        return (int.from_bytes(self.data[p >> 3:(p >> 3) + 4], "little") >> (p & 7)) & ((1 << k) - 1)

    def bits(self, k: int) -> int:
        v = self.peek(k)
        self.pos += k
        if self.pos > self.n:
            raise StreamError("read past the end of the stream")
        return v


def _table(lens, what: str, one_code_ok=False):
    """Canonical decode table: index by the next `width` stream bits (LSB first) -> (symbol, length)."""
    width = max(lens) if lens else 0
    if width == 0:
        raise StreamError(f"{what}: no codes")
    count = [0] * (width + 1)
    for ln in lens:
        if ln:
            count[ln] += 1
    left = 1
    for b in range(1, width + 1):
        left = (left << 1) - count[b]
        if left < 0:
            raise StreamError(f"{what}: over-subscribed code")
    if left > 0 and not (one_code_ok and sum(count) == 1 and width == 1):
        raise StreamError(f"{what}: incomplete code")
    nxt, code = [0] * (width + 2), 0
    for b in range(1, width + 1):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    tab = [None] * (1 << width)
    for s, ln in enumerate(lens):
        if not ln:
            continue
        c = nxt[ln]
        nxt[ln] += 1
        r = int(format(c, f"0{ln}b")[::-1], 2)
        for hi in range(0, 1 << width, 1 << ln):
            tab[r | hi] = (s, ln)
    return tab, width


def _sym(br: BitReader, tab):
    t, w = tab
    e = t[br.peek(w)]
    if e is None:
        raise StreamError("no such code")
    br.pos += e[1]
    if br.pos > br.n:
        raise StreamError("read past the end of the stream")
    return e[0]


@dataclass
class Block:
    bfinal: int
    btype: int
    first_bit: int
    end_bit: int = 0
    out0: int = 0  # the bytes [out0, out1) of the output
    out1: int = 0
    stored_len: int = 0  # LEN of a stored block
    hlit: int = 0
    hdist: int = 0
    hclen: int = 0
    bl_lens: list = field(default_factory=list)  # by symbol 0..18
    ll_lens: list = field(default_factory=list)  # HLIT entries
    d_lens: list = field(default_factory=list)  # HDIST entries
    runs_ll: list = field(default_factory=list)  # (16 | 17 | 18, repeat count) of the lit/len part
    runs_d: list = field(default_factory=list)  # ... of the distance part
    header_syms: list = field(default_factory=list)  # every code-length symbol with its extra bits, both parts
    ntok: int = 0  # literals + matches (EOB not counted)
    lit_hist: list = field(default_factory=lambda: [0] * L_CODES)
    dist_hist: list = field(default_factory=lambda: [0] * D_CODES)
    dist_extra: int = 0  # sum of distance extra bits
    matches_8192: int = -1  # matches among the block's first 8192 tokens (-1: fewer tokens); the heuristic cut reads it

    @property
    def nbytes(self) -> int:
        return self.out1 - self.out0

    @property
    def matches(self) -> int:
        return sum(self.dist_hist)


@dataclass
class Stream:
    blocks: list
    data: bytes

    @property
    def ntok(self) -> int:
        return sum(b.ntok for b in self.blocks)


def _read_header(br: BitReader, b: Block):
    b.hlit, b.hdist, b.hclen = br.bits(5) + 257, br.bits(5) + 1, br.bits(4) + 4
    if b.hlit > 286 or b.hdist > 30:
        raise StreamError("HLIT / HDIST out of range")
    bl = [0] * BL_CODES
    for i in range(b.hclen):
        bl[BL_ORDER[i]] = br.bits(3)
    b.bl_lens = bl
    tab = _table(bl, "bit-length code")
    lens = []
    while len(lens) < b.hlit + b.hdist:
        s = _sym(br, tab)
        if s < 16:
            lens.append(s)
            b.header_syms.append((s, 0))
            continue
        if s == 16:
            if not lens:
                raise StreamError("repeat with no previous length")
            k, v = 3 + br.bits(2), lens[-1]
        elif s == 17:
            k, v = 3 + br.bits(3), 0
        else:
            k, v = 11 + br.bits(7), 0
        b.header_syms.append((s, k))
        (b.runs_ll if len(lens) < b.hlit else b.runs_d).append((s, k))
        lens += [v] * k
    if len(lens) > b.hlit + b.hdist:
        raise StreamError("code lengths run past HLIT + HDIST")
    # (a run across the lit/len / distance border is legal; the encoder never makes one, and check_block would see it)
    b.ll_lens, b.d_lens = lens[:b.hlit], lens[b.hlit:]
    if b.ll_lens[256] == 0:
        raise StreamError("no end-of-block code")
    return _table(b.ll_lens, "lit/len code"), _table(b.d_lens, "distance code", one_code_ok=True)


_STATIC = None


def parse(stream: bytes, window: int = 32768) -> Stream:
    global _STATIC
    if _STATIC is None:
        _STATIC = (_table(STATIC_LL, "static lit/len"), _table([5] * 32, "static distance"))
    br, out, blocks = BitReader(stream), bytearray(), []
    while True:
        b = Block(bfinal=br.bits(1), btype=0, first_bit=br.pos - 1)
        b.btype = br.bits(2)
        b.out0 = len(out)
        if b.btype == 3:
            raise StreamError("block type 3")
        if b.btype == 0:
            pad = (-br.pos) & 7
            if br.bits(pad):
                raise StreamError("non-zero padding before a stored block")
            ln, nln = br.bits(16), br.bits(16)
            if ln != (~nln & 0xFFFF):
                raise StreamError("LEN / NLEN mismatch")
            p = br.pos >> 3
            if p + ln > len(stream):
                raise StreamError("stored block past the end")
            out += stream[p:p + ln]
            br.pos += 8 * ln
            b.stored_len = ln
        else:
            lt, dt = _STATIC if b.btype == 1 else _read_header(br, b)
            lh, dh = b.lit_hist, b.dist_hist
            nt = 0
            while True:
                if nt == 8192:
                    b.matches_8192 = sum(dh)
                nt += 1
                s = _sym(br, lt)
                lh[s] += 1
                if s < 256:
                    out.append(s)
                    continue
                if s == 256:
                    break
                if s > 285:
                    raise StreamError("lit/len symbol 286 / 287")
                c = s - 257
                ln = LEN_BASE[c] + br.bits(LEN_EXTRA[c])
                dc = _sym(br, dt)
                if dc >= 30:
                    raise StreamError("distance symbol 30 / 31")
                dh[dc] += 1
                b.dist_extra += DIST_EXTRA[dc]
                d = DIST_BASE[dc] + br.bits(DIST_EXTRA[dc])
                if d > window or d > len(out):
                    raise StreamError(f"distance {d} beyond the window / output")
                if d >= ln:
                    out += out[len(out) - d:len(out) - d + ln]
                else:
                    for _ in range(ln):
                        out.append(out[-d])
            b.ntok = sum(lh) - 1
        b.out1 = len(out)
        b.end_bit = br.pos
        blocks.append(b)
        if b.bfinal:
            break
    pad = (-br.pos) & 7
    if br.bits(pad):
        raise StreamError("non-zero padding after the final block")
    if br.pos != br.n:
        raise StreamError("bytes after the final block")
    return Stream(blocks, bytes(out))


# ---------------------------------------------------------------------------------------------------------------------
# the tree builder, restated
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class Tree:
    lens: list  # limited code lengths, one per symbol of the alphabet
    max_code: int  # the largest code with a length, padding included
    depth: int  # the deepest leaf without the length limit
    overflow: int  # nodes the limit cut, as gen_bitlen counts them (internal nodes included)
    opt_bits: int  # sum of freq * (length + extra bits) after the repair, minus one per padding code
    static_bits: int  # the same with the fixed code lengths, minus the fixed length of every padding code


def build_tree(freq, kind: int, max_length=None) -> Tree:
    """kind 0: lit/len (length extra bits from code 257), 1: distance, 2: bit-length.  max_length: 15, or 7 for kind 2."""
    elems = (L_CODES, D_CODES, BL_CODES)[kind]
    if max_length is None:
        max_length = MAX_BL_BITS if kind == 2 else MAX_BITS
    base = 257 if kind == 0 else 0
    extra = (LEN_EXTRA, DIST_EXTRA, BL_EXTRA)[kind]
    stree = (STATIC_LL, STATIC_D, None)[kind]
    f = list(freq[:elems]) + [0] * (elems + 1)
    f += [0] * (2 * elems + 1 - len(f))
    dad, ln, dep = [0] * len(f), [0] * len(f), [0] * len(f)
    heap = [0] * HEAP_SIZE
    opt = stat = 0
    hl, hmax, max_code = 0, HEAP_SIZE, -1

    def smaller(n, m):  # frequency first, then depth: the subtree that is less deep goes first
        return f[n] < f[m] or (f[n] == f[m] and dep[n] <= dep[m])

    def down(k):
        v, j = heap[k], k << 1
        while j <= hl:
            if j < hl and smaller(heap[j + 1], heap[j]):
                j += 1
            if smaller(v, heap[j]):
                break
            heap[k] = heap[j]
            k, j = j, j << 1
        heap[k] = v

    for n in range(elems):
        if f[n]:
            hl += 1
            heap[hl] = max_code = n
    # at least two codes: the first missing of 0, 1, 2 above max_code, else code 0
    while hl < 2:
        if max_code < 2:
            max_code += 1
            node = max_code
        else:
            node = 0
        hl += 1
        heap[hl] = node
        f[node] = 1
        dep[node] = 0
        opt -= 1
        if stree:
            stat -= stree[node]
    for n in range(hl // 2, 0, -1):
        down(n)
    node = elems
    while True:
        n = heap[1]
        heap[1] = heap[hl]
        hl -= 1
        down(1)
        m = heap[1]
        hmax -= 1
        heap[hmax] = n
        hmax -= 1
        heap[hmax] = m
        f[node] = f[n] + f[m]
        dep[node] = max(dep[n], dep[m]) + 1
        dad[n] = dad[m] = node
        heap[1] = node
        node += 1
        down(1)
        if hl < 2:
            break
    hmax -= 1
    heap[hmax] = heap[1]
    # gen_bitlen: lengths from the root down, the limit applied on the way, then the overflow repair
    bl_count = [0] * (MAX_BITS + 1)
    udepth = [0] * len(f)
    ln[heap[hmax]] = 0
    overflow = depth = 0
    for h in range(hmax + 1, HEAP_SIZE):
        n = heap[h]
        bits = ln[dad[n]] + 1
        udepth[n] = udepth[dad[n]] + 1
        if bits > max_length:
            bits = max_length
            overflow += 1
        ln[n] = bits
        if n > max_code:
            continue
        depth = max(depth, udepth[n])
        bl_count[bits] += 1
        xb = extra[n - base] if n >= base else 0
        opt += f[n] * (bits + xb)
        if stree:
            stat += f[n] * (stree[n] + xb)
    h, overflow0 = HEAP_SIZE, overflow
    if overflow:
        while True:
            bits = max_length - 1
            while bl_count[bits] == 0:
                bits -= 1
            bl_count[bits] -= 1  # a leaf moves one level down, taking an overflowed leaf as its brother
            bl_count[bits + 1] += 2
            bl_count[max_length] -= 1
            overflow -= 2
            if overflow <= 0:
                break
        for bits in range(max_length, 0, -1):
            n = bl_count[bits]
            while n:
                h -= 1
                m = heap[h]
                if m > max_code:
                    continue
                if ln[m] != bits:
                    opt += (bits - ln[m]) * f[m]
                    ln[m] = bits
                n -= 1
    lens = [ln[n] if n <= max_code and f[n] else 0 for n in range(elems)]
    return Tree(lens, max_code, depth, overflow0, opt, stat)


def scan_runs(lens, max_code):
    """_scanTree / _sendTree: the code-length symbols of lens[0..max_code] -> [(symbol, repeat count or 0)]."""
    out = []
    prevlen, nextlen, count = -1, lens[0], 0
    max_count, min_count = (138, 3) if nextlen == 0 else (7, 4)
    for n in range(max_code + 1):
        cur = nextlen
        nextlen = lens[n + 1] if n + 1 <= max_code else -1  # the guard entry past max_code
        count += 1
        if count < max_count and cur == nextlen:
            continue
        if count < min_count:
            out += [(cur, 0)] * count
        elif cur != 0:
            if cur != prevlen:
                out.append((cur, 0))
                count -= 1
            out.append((16, count))
        elif count <= 10:
            out.append((17, count))
        else:
            out.append((18, count))
        count, prevlen = 0, cur
        if nextlen == 0:
            max_count, min_count = 138, 3
        elif cur == nextlen:
            max_count, min_count = 6, 3
        else:
            max_count, min_count = 7, 4
    return out


@dataclass
class Plan:
    lt: Tree
    dt: Tree
    blt: Tree
    runs: list  # code-length symbols of both parts
    max_blindex: int
    opt_len: int
    static_len: int

    @property
    def opt_lenb(self) -> int:
        return (self.opt_len + 3 + 7) >> 3

    @property
    def static_lenb(self) -> int:
        return (self.static_len + 3 + 7) >> 3


def plan(lit_hist, dist_hist, bl_limit=MAX_BL_BITS) -> Plan:
    """The trees, bit-length tree and sizes _flushBlock computes for a block with these histograms (EOB counted once)."""
    lh = list(lit_hist)
    lh[256] = 1
    lt = build_tree(lh, 0)
    dt = build_tree(dist_hist, 1)
    runs = scan_runs(lt.lens, lt.max_code) + scan_runs(dt.lens, dt.max_code)
    blf = [0] * BL_CODES
    for s, _ in runs:
        blf[s] += 1
    blt = build_tree(blf, 2, bl_limit)
    mb = BL_CODES - 1
    while mb >= 3 and blt.lens[BL_ORDER[mb]] == 0:
        mb -= 1
    opt = lt.opt_bits + dt.opt_bits + blt.opt_bits + 3 * (mb + 1) + 5 + 5 + 4
    return Plan(lt, dt, blt, runs, mb, opt, lt.static_bits + dt.static_bits)


def check_block(b: Block, w_size: int = 32768) -> Plan | None:
    """The table check of one parsed block: None for a stored block, else the plan of its histograms, which must be
    the block as coded -- the three trees' lengths, HLIT / HDIST / HCLEN, every code-length symbol, the block's size in
    bits and its kind."""
    if b.btype == 0:
        return None
    p = plan(b.lit_hist, b.dist_hist)
    size = b.end_bit - b.first_bit
    if b.btype == 2:
        assert b.hlit == p.lt.max_code + 1 and b.hdist == p.dt.max_code + 1 and b.hclen == p.max_blindex + 1, \
            ((b.hlit, b.hdist, b.hclen), (p.lt.max_code + 1, p.dt.max_code + 1, p.max_blindex + 1))
        assert b.ll_lens == p.lt.lens[:b.hlit] and b.d_lens == p.dt.lens[:b.hdist], "code lengths"
        assert b.bl_lens == p.blt.lens, ("bit-length code lengths", b.bl_lens, p.blt.lens)
        assert b.header_syms == p.runs, "code-length symbols"
        assert size == 3 + p.opt_len, (size, 3 + p.opt_len)
        assert p.static_lenb > p.opt_lenb, ("dynamic block", p.static_lenb, p.opt_lenb)
    else:
        assert size == 3 + p.static_len, (size, 3 + p.static_len)
        assert p.static_lenb <= p.opt_lenb, ("static block", p.static_lenb, p.opt_lenb)
    if b.nbytes + 4 <= min(p.opt_lenb, p.static_lenb):
        # stored would be smaller: only a block whose start has slid out of the window may be coded otherwise
        assert b.nbytes >= w_size - MIN_LOOKAHEAD, ("stored was smaller", b.nbytes, p.opt_lenb, p.static_lenb)
    return p


def check_stream(stream: bytes, data: bytes, w_size: int = 32768):
    """parse + the input back + the table check of every block -> (Stream, [Plan | None])"""
    s = parse(stream, w_size)
    assert s.data == data, "the stream does not decode to the input"
    return s, [check_block(b, w_size) for b in s.blocks]
