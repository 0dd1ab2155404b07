"""TEST INFRASTRUCTURE: an independent reader of BZh streams and a check of their coding tables.

`parse(stream)` reads a whole "BZh9" stream without inverting the BWT.  For every block it returns the block CRC, origPtr,
the in-use map, nGroups, nSelectors, the selectors (MTF undone), every table's code lengths and the MTF/RUNA/RUNB symbols
up to and including EOB; for the stream, the combined CRC.

`hb_lengths(freq, max_len)` restates _hbMakeCodeLengths (bzip2_encoder.dart:747-864) with the length limit as a parameter
(None: no limit).  `check_tables(block)` recounts each table's symbols under the block's final selectors and asserts that
the limited code lengths of those counts are the lengths in the stream.  This holds exactly for the reference's encoder:
its last refinement round fixes the selectors and computes the lengths from the same counts.  It does not need the oracle.
"""
from dataclasses import dataclass, field

G_SIZE = 50
MAX_LEN = 17


class BitReader:
    def __init__(self, data: bytes):
        self.data = data
        self.pos = 0
        self.nbits = len(data) * 8
        # 32-bit big-endian window at every byte offset (bits past the end read as zero)
        pad = data + b"\0\0\0\0"
        self.win = [int.from_bytes(pad[i:i + 4], "big") for i in range(len(data) + 1)]

    def bits(self, n: int) -> int:
        v = 0
        while n > 0:
            take = min(n, 24)
            v = (v << take) | self.peek(take)
            self.pos += take
            n -= take
        if self.pos > self.nbits:
            raise ValueError("read past the end of the stream")
        return v

    def peek(self, n: int) -> int:  # n <= 25
        p = self.pos
        return ((self.win[p >> 3] << (p & 7)) & 0xFFFFFFFF) >> (32 - n)


@dataclass
class Block:
    crc: int
    orig_ptr: int
    in_use: list  # the byte values present in the block, increasing
    n_groups: int
    n_sel: int
    selectors: list  # table of every group of 50 symbols, MTF undone
    lens: list  # lens[t][v]: code length of symbol v in table t
    syms: list = field(default_factory=list)  # MTF values, RUNA = 0, RUNB = 1, ..., EOB last

    @property
    def n_in_use(self) -> int:
        return len(self.in_use)

    @property
    def alpha(self) -> int:
        return self.n_in_use + 2

    @property
    def nmtf(self) -> int:
        return len(self.syms)


@dataclass
class Stream:
    blocks: list
    combined_crc: int
    n_bytes: int


def _decode_table(lens):
    """Canonical codes of _hbAssignCodes (:866-878) -> lookup over MAX_LEN-bit windows: (symbol << 5) | length."""
    tab = [0] * (1 << MAX_LEN)
    vec = 0
    for n in range(min(lens), max(lens) + 1):
        for s, l in enumerate(lens):
            if l == n:
                lo = vec << (MAX_LEN - n)
                hi = (vec + 1) << (MAX_LEN - n)
                tab[lo:hi] = [(s << 5) | n] * (hi - lo)
                vec += 1
        vec <<= 1
    return tab


def parse(stream: bytes) -> Stream:
    r = BitReader(stream)
    if r.bits(32) != 0x425A6839:
        raise ValueError("not a BZh9 stream")
    blocks = []
    combined = 0
    while True:
        magic = r.bits(48)
        if magic == 0x177245385090:
            crc = r.bits(32)
            if crc != combined:
                raise ValueError("combined CRC %08x, blocks give %08x" % (crc, combined))
            break
        if magic != 0x314159265359:
            raise ValueError("bad block magic %012x" % magic)
        bcrc = r.bits(32)
        if r.bits(1):
            raise ValueError("randomised block")
        orig_ptr = r.bits(24)
        m16 = r.bits(16)
        in_use = []
        for i in range(16):
            if m16 & (0x8000 >> i):
                w = r.bits(16)
                in_use += [i * 16 + j for j in range(16) if w & (0x8000 >> j)]
        if not in_use:
            raise ValueError("empty in-use map")
        alpha = len(in_use) + 2
        n_groups = r.bits(3)
        n_sel = r.bits(15)
        if not 2 <= n_groups <= 6 or n_sel < 1:
            raise ValueError("nGroups %d, nSelectors %d" % (n_groups, n_sel))
        order = list(range(n_groups))
        selectors = []
        for _ in range(n_sel):
            j = 0
            while r.bits(1):
                j += 1
                if j >= n_groups:
                    raise ValueError("selector MTF value out of range")
            v = order.pop(j)
            order.insert(0, v)
            selectors.append(v)
        lens = []
        for _ in range(n_groups):
            cur = r.bits(5)
            tl = []
            for _ in range(alpha):
                while r.bits(1):
                    cur += -1 if r.bits(1) else 1
                if not 1 <= cur <= 20:
                    raise ValueError("code length %d" % cur)
                tl.append(cur)
            lens.append(tl)
        tables = [_decode_table(tl) for tl in lens]
        eob = alpha - 1
        syms = []
        win, peekmask = r.win, (1 << MAX_LEN) - 1
        pos = r.pos
        g = 0
        while True:
            if g >= n_sel:
                raise ValueError("symbols beyond the last selector")
            tab = tables[selectors[g]]
            done = False
            for _ in range(G_SIZE):
                e = tab[(((win[pos >> 3] << (pos & 7)) & 0xFFFFFFFF) >> (32 - MAX_LEN)) & peekmask]
                if e == 0:
                    raise ValueError("invalid code")
                pos += e & 31
                s = e >> 5
                syms.append(s)
                if s == eob:
                    done = True
                    break
            g += 1
            if done:
                break
        r.pos = pos
        if g != n_sel:
            raise ValueError("EOB in group %d of %d" % (g, n_sel))
        blocks.append(Block(bcrc, orig_ptr, in_use, n_groups, n_sel, selectors, lens, syms))
        combined = (((combined << 1) | (combined >> 31)) & 0xFFFFFFFF) ^ bcrc
    if r.pos > r.nbits or (r.nbits - r.pos) >= 8:
        raise ValueError("stream length: %d bits read of %d" % (r.pos, r.nbits))
    return Stream(blocks, combined, len(stream))


def hb_lengths(freq, max_len=MAX_LEN):
    """_hbMakeCodeLengths (bzip2_encoder.dart:747-864); max_len None: no limit, a single pass."""
    alpha = len(freq)
    weight = [0] * (2 * alpha + 2)
    parent = [0] * (2 * alpha + 2)
    for i in range(alpha):
        weight[i + 1] = (freq[i] if freq[i] else 1) << 8
    while True:
        heap = [0] * (alpha + 2)
        weight[0] = 0
        parent[0] = -2
        n_nodes, n_heap = alpha, 0

        def up(z):
            tmp = heap[z]
            while weight[tmp] < weight[heap[z >> 1]]:
                heap[z] = heap[z >> 1]
                z >>= 1
            heap[z] = tmp

        def down(z):
            tmp = heap[z]
            while True:
                y = z << 1
                if y > n_heap:
                    break
                if y < n_heap and weight[heap[y + 1]] < weight[heap[y]]:
                    y += 1
                if weight[tmp] < weight[heap[y]]:
                    break
                heap[z] = heap[y]
                z = y
            heap[z] = tmp

        for i in range(1, alpha + 1):
            parent[i] = -1
            n_heap += 1
            heap[n_heap] = i
            up(n_heap)
        while n_heap > 1:
            n1 = heap[1]
            heap[1] = heap[n_heap]
            n_heap -= 1
            down(1)
            n2 = heap[1]
            heap[1] = heap[n_heap]
            n_heap -= 1
            down(1)
            n_nodes += 1
            parent[n1] = parent[n2] = n_nodes
            w1, w2 = weight[n1], weight[n2]
            weight[n_nodes] = ((w1 & ~0xFF) + (w2 & ~0xFF)) | (1 + max(w1 & 0xFF, w2 & 0xFF))
            parent[n_nodes] = -1
            n_heap += 1
            heap[n_heap] = n_nodes
            up(n_heap)
        lens = []
        for i in range(1, alpha + 1):
            j, k = 0, i
            while parent[k] >= 0:
                k = parent[k]
                j += 1
            lens.append(j)
        if max_len is None or max(lens) <= max_len:
            return lens
        for i in range(1, alpha + 1):
            weight[i] = (1 + (weight[i] >> 8) // 2) << 8


def mtf_positions(b: Block):
    """The move-to-front positions of the block's last column (RUNA/RUNB expanded to zeros, EOB dropped)."""
    out = []
    run, k = 0, 0
    for s in b.syms[:-1]:
        if s < 2:
            run += (s + 1) << k
            k += 1
            continue
        if run:
            out.extend([0] * run)
            run, k = 0, 0
        out.append(s - 1)
    out.extend([0] * run)
    return out


def last_column(b: Block):
    """The block's last column as indices into the in-use map (MTF undone; the BWT is not inverted)."""
    order = list(range(b.n_in_use))
    col = []
    for p in mtf_positions(b):
        v = order.pop(p)
        order.insert(0, v)
        col.append(v)
    return col


def table_freqs(b: Block):
    """Symbols coded with each table under the block's final selectors."""
    freq = [[0] * b.alpha for _ in range(b.n_groups)]
    for g, t in enumerate(b.selectors):
        f = freq[t]
        for s in b.syms[g * G_SIZE:(g + 1) * G_SIZE]:
            f[s] += 1
    return freq


@dataclass
class TableCheck:
    depths: list  # per table: depth of the code without the length limit
    retried: list  # per table: the halving retry ran (depth without the limit > 17)
    unused: list  # per table: never selected


def check_tables(b: Block) -> TableCheck:
    assert b.n_sel == (b.nmtf + G_SIZE - 1) // G_SIZE, (b.n_sel, b.nmtf)
    assert b.syms[-1] == b.alpha - 1 and all(s < b.alpha - 1 for s in b.syms[:-1])
    assert b.n_groups == (2 if b.nmtf < 200 else 3 if b.nmtf < 600 else 4 if b.nmtf < 1200 else 5 if b.nmtf < 2400 else 6)
    depths, retried = [], []
    freqs = table_freqs(b)
    for t, f in enumerate(freqs):
        assert hb_lengths(f, MAX_LEN) == b.lens[t], "table %d: lengths are not those of its symbol counts" % t
        d = max(hb_lengths(f, None))
        depths.append(d)
        retried.append(d > MAX_LEN)
    return TableCheck(depths, retried, [t not in set(b.selectors) for t in range(b.n_groups)])


def check_stream(stream: bytes) -> tuple:
    """Parse and check every block's tables -> (Stream, [TableCheck per block])."""
    s = parse(stream)
    return s, [check_tables(b) for b in s.blocks]


def _find_bits(stream: bytes, pattern: bytes):
    """Bit offsets of `pattern` in `stream`, at any bit alignment."""
    import numpy as np
    a = np.frombuffer(stream + b"\0", np.uint8).astype(np.uint16)
    found = []
    for sh in range(8):
        v = (((a[:-1] << sh) | (a[1:] >> (8 - sh))) & 0xFF).astype(np.uint8)
        cand = np.nonzero(v[:len(v) - len(pattern) + 1] == pattern[0])[0]
        for k in range(1, len(pattern)):
            cand = cand[v[cand + k] == pattern[k]]
        found += (cand * 8 + sh).tolist()
    return sorted(found)


def scan_headers(stream: bytes):
    """For a stream too large to parse in Python: the block CRCs read after every block magic and the combined CRC read
    after the end-of-stream magic.  A false match needs 48 coincident bits.  -> ([block CRC], combined CRC)"""
    def u32(bit):
        v = int.from_bytes(stream[bit // 8:bit // 8 + 5].ljust(5, b"\0"), "big")
        return (v >> (8 - bit % 8)) & 0xFFFFFFFF
    crcs = [u32(p + 48) for p in _find_bits(stream, bytes.fromhex("314159265359"))]
    eos = _find_bits(stream, bytes.fromhex("177245385090"))
    assert len(eos) == 1
    return crcs, u32(eos[0] + 48)


def fold_crcs(crcs) -> int:
    c = 0
    for b in crcs:
        c = (((c << 1) | (c >> 31)) & 0xFFFFFFFF) ^ b
    return c
