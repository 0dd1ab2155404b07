"""The inflate kernels on hand-built DEFLATE streams (tests/deflate_craft.py), on the CUDA execution-model emulation.

Every other inflate test feeds the kernels streams made by zlib, which only ever writes a narrow slice of DEFLATE.  The
reference (inflate.dart, _huffman_table.dart; oracle/inflate.c) accepts much more, and gives some malformed inputs a
defined result.  This catalogue pins each kernel's table construction on that wider slice: HLIT 288 / HDIST 32 with the
extra symbols moving every other code, single-code and incomplete sets, explicit code-length op lists, every length and
distance code at both extra-bit ends, k_inflate_fast's second-level pool at exactly its 384 entries and one allocation
past them, the reference's table holes, and the documented divergences (DESIGN.md section 7), each with an exact
outcome.  The same units run on the GPU in tests/test_inflate_crafted_gpu.py."""
import ctypes as C
import os
import random
import zlib

import pytest

import deflate_craft as dc
import oracle_lib as orc
import test_inflate_fast_emul as tfe
import test_inflate_spec_emul as tse

DONE, EOS, STOP, NOSPC, RANGE, BADCODE, UTHROW = 0, 1, -1, -2, -3, -4, -5
# k_inflate_fast's eligibility (inflate_fast.cuh, namespace fp) and its second-level pool
MIN_IN, IN_CAP, WIN, FAST_SUBN, FAST_LB, FAST_DB = 192, 30720, 65536, 384, 10, 8
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Case:
    """One unit and its exact expected outcome on the exact kernels (k_inflate_decode / k_inflate_expand, and their
    per-stream logic).  kind: "valid" (the reference decodes `plain`), "quirk" (a defined reference result on a
    malformed stream: bit-exact with the oracle), "diverge" (DESIGN.md section 7: `plain` is the output before the
    offending block or symbol).  `fast`: "finish" / "leave" / None (not asserted)."""

    def __init__(self, name, raw, plain, status=DONE, kind="valid", cap=None, ostatus=orc.OK, zlib_ok=False,
                 fast=None, stream_len=None):
        self.name, self.raw, self.plain, self.status, self.kind = name, raw, bytes(plain), status, kind
        self.cap = cap if cap is not None else (max(1, len(plain)) if kind == "valid" else WIN)
        self.ostatus, self.zlib_ok = ostatus, zlib_ok
        self.stream_len = stream_len if stream_len is not None else len(raw)
        if fast is None:
            if kind == "valid":
                fast = "finish" if status in (DONE, EOS) and self.eligible() else None
            else:
                fast = "leave"
        self.fast = fast

    def eligible(self, lead_max=15):
        return MIN_IN <= len(self.raw) and len(self.raw) + lead_max <= IN_CAP and 0 < self.cap <= WIN

    def __repr__(self):
        return self.name


def padded(u, n=MIN_IN + 8):
    """The unit's stream followed by zero bytes (bytes after the final block), at least two and up to n bytes."""
    raw = u.data()
    return raw + bytes(max(2, n - len(raw)))


def valid(name, u, n=MIN_IN + 8, status=DONE, raw=None, **kw):
    s = u.data()
    return Case(name, padded(u, n) if raw is None else raw, u.plain, status, zlib_ok=u.zlib_ok, stream_len=len(s), **kw)


def words(rng, n):
    ws = [bytes(rng.choice(b"etaoinshrdlucmfw") for _ in range(rng.randint(2, 8))) for _ in range(200)]
    b = bytearray()
    while len(b) < n:
        b += rng.choice(ws) + b" "
    return bytes(b[:n])


def grow(u, rng, n):
    """Add about n bytes of non-periodic plaintext to a fixed or dynamic block (long matches with a literal after each)."""
    lits = u.lit_syms()
    if not u.plain:
        u.lit_byte(rng.choice(lits))
    target = len(u.plain) + n
    while len(u.plain) < target:
        u.match(rng.randint(200, 258), rng.randint(1, min(len(u.plain), 32768)))
        u.lit_byte(rng.choice(lits))


def lit_lengths(rng, n=286, maxlen=12, **kw):
    must = set(kw.pop("must", ())) | {256} | set(range(257, min(n, 286)))
    return dc.complete_lengths(rng, n, maxlen, must=sorted(must - set(kw.get("zero", ()))), **kw)


def dist_lengths(rng, n=30, maxlen=9, **kw):
    if n == 1:
        return [1]
    return dc.complete_lengths(rng, n, maxlen, must=[d for d in range(min(n, 30)) if d not in kw.get("zero", ())], **kw)


# ------------------------------------------------------------------ valid for the reference
def fam_single_distance(rng):
    out = []
    for d in (0, 3, 17, 29):
        u = dc.Unit()
        u.fixed()
        u.literals(words(rng, 40))
        hi = dc.DIST_BASE[d] + (1 << dc.DIST_EXTRA[d]) - 1
        if len(u.plain) < hi:
            grow(u, rng, hi - len(u.plain))
        u.eob()
        lit = lit_lengths(rng, 286, 10)
        # incomplete lit/len set: a literal loses its code, which becomes a hole that is never hit
        lit[max(range(256), key=lambda s: lit[s])] = 0
        dist = [0] * d + [1]
        u.dynamic(lit, dist, final=True)
        for x in (0, (1 << dc.DIST_EXTRA[d]) - 1):
            u.match(rng.randint(3, 258), dc.DIST_BASE[d] + x)
            u.lit_byte(rng.choice(u.lit_syms()))
        dc.random_symbols(u, rng, 500)
        u.eob()
        assert dc.kraft(lit) < 1
        out.append(valid(f"single_dist_{d}", u))
    return out


def fam_alphabet_sizes(rng):
    out = []
    for hlit, hdist in ((257, 1), (286, 30), (287, 31), (288, 32), (288, 1), (257, 32), (287, 2)):
        fl = {s: l for s, l in ((286, 3), (287, 4)) if s < hlit}  # shorter than the rest: every other code moves
        fd = {s: l for s, l in ((30, 2), (31, 3)) if s < hdist}
        u = dc.Unit()
        u.stored(words(rng, 30))
        lit = lit_lengths(rng, hlit, 12, forced=fl)
        dist = dist_lengths(rng, hdist, 9, forced=fd) if hdist > 2 else ([1] if hdist == 1 else [1, 1])
        u.dynamic(lit, dist, final=True)
        dc.random_symbols(u, rng, 3000)
        u.eob()
        out.append(valid(f"hlit{hlit}_hdist{hdist}", u))
    return out


def fam_hclen(rng):
    out = []
    # HCLEN 5: only code-length symbols 16, 17, 18, 0 and 8: 255 literals and end-of-block, all 8 bits
    u = dc.Unit()
    lit = [8] * 255 + [0, 8]
    u.dynamic(lit, [0], final=True)
    assert u.w.n and dc.cl_for(dc.rle_ops(lit + [0]))[8]
    u.literals(bytes(rng.randrange(255) for _ in range(600)))
    u.eob()
    out.append(valid("hclen5_all_8", u))
    # HCLEN 19: every code-length length written, the trailing ones 0
    u = dc.Unit()
    u.dynamic(lit_lengths(rng, 286, 11), dist_lengths(rng, 30, 7), final=True, hclen=19)
    dc.random_symbols(u, rng, 2000)
    u.eob()
    out.append(valid("hclen19", u))
    # a code-length code with one used symbol (9, length 1, incomplete): every lit/len and distance length is 9
    u = dc.Unit()
    cl = [0] * 19
    cl[9] = 1
    u.dynamic([9] * 257, [9], final=True, cl_lens=cl, ops=[9] * 258)
    u.literals(bytes(rng.randrange(256) for _ in range(700)))
    u.eob()
    out.append(valid("cl_single_symbol", u))
    return out


def _crosses(ops, at):
    """True when one run op of `ops` covers lengths on both sides of index `at`."""
    i = 0
    for o in ops:
        r = 1 if isinstance(o, int) else o[1]
        if not isinstance(o, int) and i < at < i + r:
            return True
        i += r
    return False


def fam_cl_ops(rng):
    out = []

    def unit(name, lit, dist, ops, check=None):
        assert dc.ops_to_lens(ops, len(lit) + len(dist)) == lit + dist, name
        if check:
            assert check(ops), name
        u = dc.Unit()
        u.fixed()
        u.literals(words(rng, 50))
        u.eob()
        u.dynamic(lit, dist, ops=ops, final=True)
        dc.random_symbols(u, rng, 2500)
        u.eob()
        out.append(valid(name, u))

    # 16 as the first op: it repeats prev = 0
    lit, dist = lit_lengths(rng, 286, 11, zero={0, 1, 2}), dist_lengths(rng, 30, 8)
    unit("op16_first", lit, dist, [(16, 3)] + dc.rle_ops(lit[3:] + dist))
    # 16 right after a 17 and right after an 18: it repeats 0, not the length before the run
    z = set(range(11, 17)) | set(range(21, 35))
    lit, dist = lit_lengths(rng, 286, 11, zero=z, must=[10, 20]), dist_lengths(rng, 30, 8)
    seq = lit + dist
    ops = dc.rle_ops(seq[:11]) + [(17, 3), (16, 3)] + dc.rle_ops(seq[17:21]) + [(18, 11), (16, 3)] + dc.rle_ops(seq[35:])
    unit("op16_after_17_and_18", lit, dist, ops)
    # runs of 16, 17 and 18 across the lit/len -> distance boundary
    lit = lit_lengths(rng, 286, 12, forced={283: 6, 284: 6, 285: 6})
    dist = dist_lengths(rng, 30, 8, forced={0: 6, 1: 6, 2: 6})
    unit("op16_across", lit, dist, dc.rle_ops(lit + dist), lambda o: _crosses(o, 286))
    lit = lit_lengths(rng, 286, 12, zero=set(range(281, 286)))
    dist = dist_lengths(rng, 30, 8, zero={0, 1, 2})
    unit("op17_across", lit, dist, dc.rle_ops(lit + dist), lambda o: _crosses(o, 286) and (17, 8) in o)
    lit = lit_lengths(rng, 286, 12, zero=set(range(273, 286)))
    dist = dist_lengths(rng, 30, 8, zero={0, 1, 2, 3, 4})
    unit("op18_across", lit, dist, dc.rle_ops(lit + dist), lambda o: _crosses(o, 286) and (18, 18) in o)
    # 16, 17 and 18 at their most repeats
    f = {s: 9 for s in range(170, 177)}
    f.update({169: 8, 177: 10})
    lit = lit_lengths(rng, 286, 12, zero=set(range(138)) | set(range(150, 160)), forced=f, must=[149, 160])
    dist = dist_lengths(rng, 30, 8)
    unit("op_max_repeats", lit, dist, dc.rle_ops(lit + dist),
         lambda o: (18, 138) in o and (17, 10) in o and (16, 6) in o)
    return out


def fam_every_code(rng):
    out = []
    u = dc.Unit()
    lit = lit_lengths(rng, 286, 12)
    u.dynamic(lit, dist_lengths(rng, 30, 10), final=True)
    u.literals(bytes(rng.choice(u.lit_syms()) for _ in range(100)))
    u.match(20, len(u.plain))  # a distance equal to the output position: reaches byte 0
    for c in range(257, 286):
        for ln in sorted({dc.LEN_BASE[c - 257], dc.LEN_BASE[c - 257] + (1 << dc.LEN_EXTRA[c - 257]) - 1}):
            u.match(ln, rng.randint(1, len(u.plain)), c)
    while len(u.plain) < 32768 + 300:
        u.match(258, rng.randint(1, min(len(u.plain), 32768)))
        u.lit_byte(rng.choice(u.lit_syms()))
    for d in range(30):
        for x in (0, (1 << dc.DIST_EXTRA[d]) - 1):
            u.match(rng.randint(3, 40), dc.DIST_BASE[d] + x)
    u.match(258, 32768)
    u.match(3, 32768)
    u.eob()
    out.append(valid("every_code_min_max_extra", u))
    # length 258 as 284 + 31 extra bits, in a dynamic and in a fixed block
    u = dc.Unit()
    u.fixed()
    u.literals(words(rng, 300))
    for k in range(20):
        u.match(258, rng.randint(1, len(u.plain)), 284 if k % 2 else 285)
    u.eob()
    u.dynamic(lit_lengths(rng, 286, 12), dist_lengths(rng, 30, 9), final=True)
    for k in range(20):
        u.match(258, rng.randint(1, min(32768, len(u.plain))), 284 if k % 2 else 285)
        u.lit_byte(rng.choice(u.lit_syms()))
    u.eob()
    assert not u.zlib_ok
    out.append(valid("len258_as_284_plus_31", u))
    return out


def fam_random_sets(rng, n=6):
    out = []
    for k in range(n):
        u = dc.Unit()
        u.dynamic(lit_lengths(rng, 286, 15), dist_lengths(rng, 30, 15), final=True)
        dc.random_symbols(u, rng, rng.choice([1500, 4000, 9000]), match_frac=rng.choice([0.05, 0.3]), long_first=True)
        u.eob()
        out.append(valid(f"random_sets_15_{k}", u))
    return out


def pool_sets(rng, over):
    """Lit/len and distance sets whose codes longer than k_inflate_fast's 10-bit / 8-bit roots take exactly FAST_SUBN
    second-level entries (over=False), or one 2-entry allocation more (over=True).  The distance codes longer than
    8 bits are one chain 9..15, 15 under one prefix (128 entries); the lit/len ones a chain 11..15, 15 and seven
    prefixes of 32 fifteen-bit codes (256 entries)."""
    dist = [0] * 30
    ds = list(range(30))
    rng.shuffle(ds)
    for s, l in zip(ds, [1, 2, 3, 4, 5, 6, 7, 8] + [9, 10, 11, 12, 13, 14, 15, 15]):
        dist[s] = l
    longs = [11, 12, 13, 14, 15, 15] + [15] * 224
    shorts = [10] * 2 + [9] * 4 + [8] * 4 + [7] * 6 + [6] * 6 + [5] * 4  # 26 symbols ...
    units = (1 << 10) - 8 - sum(1 << (10 - l) for l in shorts)
    shorts += [10 - b for b in range(11) if units >> b & 1]  # ... plus what fills the root space
    if over:  # one 10-bit code becomes two 11-bit codes: one more prefix, of 2 entries, in front of the others
        shorts.remove(10)
        longs += [11, 11]
    lit = [0] * 286
    syms = list(range(286))
    rng.shuffle(syms)
    syms.remove(256)
    syms = [256] + syms
    for s, l in zip(syms, sorted(shorts) + longs):
        lit[s] = l
    assert dc.kraft(lit) == 1 and dc.kraft(dist) == 1
    return lit, dist


def fam_pool(rng):
    out = []
    for over in (False, True):
        lit, dist = pool_sets(rng, over)
        ent = dc.sub_entries(lit, FAST_LB) + dc.sub_entries(dist, FAST_DB)
        assert ent == FAST_SUBN + (2 if over else 0), ent
        u = dc.Unit()
        u.dynamic(lit, dist, final=True)
        dc.random_symbols(u, rng, 3000, match_frac=0.15)
        u.eob()
        out.append(valid("pool_over_by_one_allocation" if over else "pool_exactly_384", u,
                         fast="leave" if over else "finish"))
    return out


def fam_multiblock(rng):
    out = []
    for junk in (False, True):
        u = dc.Unit()
        u.stored(b"", nlen=0x1234 if junk else None)  # LEN 0 (with junk NLEN): an empty stored block
        u.fixed()
        u.eob()  # EOB-only blocks of every type
        u.dynamic(lit_lengths(rng, 286, 9), dist_lengths(rng, 30, 6))
        u.eob()
        u.stored(words(rng, 120))
        u.fixed()
        u.literals(words(rng, 200))
        dc.random_symbols(u, rng, 1500)
        u.eob()
        u.dynamic(lit_lengths(rng, 286, 13), dist_lengths(rng, 30, 11))
        dc.random_symbols(u, rng, 2000)
        u.eob()
        u.dynamic(lit_lengths(rng, 288, 15, forced={287: 2}), [0] * 5 + [1])
        dc.random_symbols(u, rng, 1000)
        u.eob()
        u.stored(b"", final=True, nlen=0x00FF if junk else None)
        tail = bytes(rng.getrandbits(8) for _ in range(40))  # bytes after the final block
        out.append(valid(f"multiblock_{'junk_nlen' if junk else 'clean'}", u, raw=u.data() + tail))
    # a stored block of LEN 65535 between two Huffman blocks
    u = dc.Unit()
    u.fixed()
    u.literals(words(rng, 1))
    u.eob()
    u.stored(bytes(rng.getrandbits(8) for _ in range(65535)))
    u.fixed(final=True)
    u.eob()
    out.append(valid("stored_65535", u, cap=65536))
    # the last block is not final: the input ends at a block boundary (B200Z_U_EOS)
    u = dc.Unit()
    u.dynamic(lit_lengths(rng, 286, 12), dist_lengths(rng, 30, 9))
    dc.random_symbols(u, rng, 3000)
    u.eob()
    u.fixed()
    dc.random_symbols(u, rng, 500)
    u.eob()
    u.stored(words(rng, 100))
    out.append(valid("last_block_not_final", u, status=EOS, raw=u.data()))
    return out


# ------------------------------------------------------------------ reference quirks with a defined result
def fixed_with_prefix(rng, n=200):
    u = dc.Unit()
    u.stored(words(rng, n))
    u.fixed(final=True)
    u.literals(words(rng, 20))
    return u


def fam_quirks(rng):
    out = []
    # fixed block, distance codes 30 / 31: holes of the reference's 30-entry table -> distance 1 from zero bits; the
    # hole's 5 bits then start the next lit/len code (a 9-bit literal 11110xxxx / 11111xxxx)
    for code, lo in ((30, 224), (31, 240)):
        u = fixed_with_prefix(rng)
        ln = rng.randint(3, 258)
        u.length_part(ln)
        u.copy_plain(ln, 1)
        u.lit_byte(rng.randint(lo, lo + 15))
        u.literals(words(rng, 30))
        u.eob()
        out.append(Case(f"fixed_dist_hole_{code}", padded(u), u.plain, DONE, "quirk"))
    # ... and a hole whose 5 bits are the last of the input: the next lit/len code is a short read (B200Z_U_STOP)
    u = fixed_with_prefix(rng)
    while (u.w.n + 7) % 8 > 3:  # after the 7-bit length code fewer than 9 bits must remain
        u.lit_byte(rng.choice(b"abc"))
    u.length_part(3)
    u.copy_plain(3, 1)
    u.bits(0b01111, 5)  # stream order 1, 1, 1, 1, 0: code 30
    assert len(u.data()) * 8 - u.w.n + 5 < 9 + 5
    out.append(Case("fixed_dist_hole_at_end", u.data(), u.plain, STOP, "quirk"))
    # the unused bit of a single-code distance tree (code 5 = "0"; a "1" is a hole: distance 1, no bits)
    u = dc.Unit()
    u.stored(words(rng, 200))
    u.dynamic(lit_lengths(rng, 286, 10), [0] * 5 + [1], final=True)
    lens, codes = u.lit
    one = [s for s in u.lit_syms() if codes[s] >> (lens[s] - 1)]  # literals whose code starts with a 1 bit
    for k in range(8):
        ln = rng.randint(3, 258)
        u.length_part(ln)
        u.copy_plain(ln, 1)
        u.lit_byte(rng.choice(one))
        u.match(rng.randint(3, 30), rng.choice([7, 8]))  # and the code's own "0" with its extra bit
    u.eob()
    out.append(Case("single_dist_unused_bit", padded(u), u.plain, DONE, "quirk"))
    # a code-length-code hole: length 0 from no bits, so every later length is 0 too, and the block's first code
    # starts with the hole's bits
    cl = [0] * 19
    cl[0] = cl[1] = cl[2] = 2  # codes 00, 01, 10; 11 is a hole
    lit = [0] * 65 + [2, 2] + [0] * 189 + [1]  # end of block "0", 'A' "10", 'B' "11"
    ops = [0] * 65 + [2, 2] + [0] * 189 + [1, "hole"]
    u = dc.Unit()
    u.stored(words(rng, 200))
    u.dynamic(lit + [0] * 29, [0] * 30, final=True, cl_lens=cl, ops=ops)
    u.lit_byte(66)
    u.literals(bytes(rng.choice(b"AB") for _ in range(300)))
    u.eob()
    assert dc.ops_to_lens(ops, 316) == lit + [0] * 59
    out.append(Case("cl_code_hole", padded(u), u.plain, DONE, "quirk"))
    # lit/len symbols 286 / 287 and dynamic distance symbols 30 / 31, decoded: the reference stops (B200Z_U_STOP)
    for s in (286, 287):
        u = dc.Unit()
        u.stored(words(rng, 200))
        u.dynamic(lit_lengths(rng, 288, 11, forced={286: 5, 287: 6}), dist_lengths(rng, 30, 8), final=True)
        dc.random_symbols(u, rng, 300)
        plain = bytes(u.plain)
        u.sym(s)
        u.literals(bytes(u.lit_syms()[:5]))  # never decoded
        u.eob()
        out.append(Case(f"litlen_symbol_{s}", padded(u), plain, STOP, "quirk"))
    for d in (30, 31):
        u = dc.Unit()
        u.stored(words(rng, 200))
        u.dynamic(lit_lengths(rng, 286, 11), dist_lengths(rng, 32, 8, forced={30: 4, 31: 5}), final=True)
        dc.random_symbols(u, rng, 300)
        plain = bytes(u.plain)
        u.length_part(10)
        u.dsym(d)
        u.literals(bytes(u.lit_syms()[:5]))  # never decoded
        u.eob()
        out.append(Case(f"dist_symbol_{d}", padded(u), plain, STOP, "quirk"))
    # a 16 / 17 / 18 run past HLIT + HDIST: RangeError in the reference (B200Z_U_THROW), output before the block
    for op in (16, 17, 18):
        lit, dist = lit_lengths(rng, 286, 11), dist_lengths(rng, 30, 8)
        seq = lit + dist
        ops = dc.rle_ops(seq[:-2]) + [(op, dc.REPEAT[op][1] + 2)]
        assert dc.ops_to_lens(ops, len(seq)) is None
        u = dc.Unit()
        u.stored(words(rng, 200))
        u.dynamic(lit, dist, ops=ops, final=True)
        plain = bytes(u.plain)
        u.bits(rng.getrandbits(32), 32)
        out.append(Case(f"op{op}_run_past_end", padded(u), plain, UTHROW, "quirk", ostatus=orc.THROW))
    # a distance one byte beyond the output position: RangeError (B200Z_U_RANGE) with the output before the match
    for blk in ("fixed", "dynamic"):
        u = dc.Unit()
        u.stored(words(rng, 200))
        if blk == "fixed":
            u.fixed(final=True)
        else:
            u.dynamic(lit_lengths(rng, 286, 11), dist_lengths(rng, 30, 10), final=True)
        u.literals(bytes(rng.choice(u.lit_syms()) for _ in range(50)))
        plain = bytes(u.plain)
        dist = len(plain) + 1
        u.length_part(5)
        d = max(c for c in range(30) if dc.DIST_BASE[c] <= dist)
        u.dsym(d)
        u.bits(dist - dc.DIST_BASE[d], dc.DIST_EXTRA[d])
        u.eob()
        out.append(Case(f"distance_beyond_output_{blk}", padded(u), plain, RANGE, "quirk", ostatus=orc.THROW))
    return out


# ------------------------------------------------------------------ documented divergences (DESIGN.md section 7)
def fam_divergences(rng):
    out = []
    for which in ("litlen", "dist", "cl"):
        u = dc.Unit()
        u.stored(words(rng, 200))
        plain = bytes(u.plain)
        lit, dist = lit_lengths(rng, 286, 11), dist_lengths(rng, 30, 8)
        cl = None
        if which == "litlen":
            lit[rng.choice([s for s in range(256) if not lit[s]] or [0])] = max(lit)  # one code too many
            lit[0] = lit[0] or 3
        elif which == "dist":
            dist = [1, 1, 1] + dist[3:]
        else:
            cl = [0] * 19
            for s in (0, 8, 9, 16):  # four one-bit codes
                cl[s] = 1
        u.dynamic(lit, dist, final=True, cl_lens=cl, ops=None if cl is None else [8] * 286 + [1] * 30)
        u.bits(rng.getrandbits(64), 64)
        out.append(Case(f"oversubscribed_{which}", padded(u), plain, BADCODE, "diverge", ostatus=None))
    # a lit/len hole that is hit: the reference emits literal 0 for ever (RUNAWAY here)
    u = dc.Unit()
    u.stored(words(rng, 200))
    lit = lit_lengths(rng, 286, 10)
    codes = dc.canonical(lit)
    last = max((s for s in range(286) if lit[s] and s != 256), key=lambda s: (lit[s], codes[s]))
    ln, cd = lit[last], codes[last]
    lit[last] = 0  # the last canonical code becomes a hole
    u.dynamic(lit, dist_lengths(rng, 30, 8), final=True)
    dc.random_symbols(u, rng, 200)
    plain = bytes(u.plain)
    u.w.code(cd, ln)
    u.eob()
    out.append(Case("litlen_hole_hit", padded(u), plain, BADCODE, "diverge", ostatus=orc.RUNAWAY))
    return out


# ------------------------------------------------------------------ k_inflate_fast's eligibility edges
def edge_variants(family):
    """A family's first valid final unit again: its input padded to 192 and to 30720 bytes (lead 0), and under caps of
    len(out) - 1 (output full) and 65536."""
    out = []
    for c in family:
        if c.kind != "valid" or c.status != DONE or len(c.plain) > WIN:
            continue
        s = c.raw[:c.stream_len]
        for n in (MIN_IN, IN_CAP):
            if c.stream_len + 2 <= n:
                out.append(Case(f"{c.name}@in{n}", s + bytes(n - len(s)), c.plain, zlib_ok=c.zlib_ok, stream_len=len(s),
                                fast=c.fast if c.fast == "leave" else "finish"))
        if c.plain:
            v = Case(f"{c.name}@cap-1", c.raw, c.plain, NOSPC, cap=len(c.plain) - 1, stream_len=c.stream_len)
            v.fast = "leave" if v.eligible() else None
            out.append(v)
        out.append(Case(f"{c.name}@cap65536", c.raw, c.plain, cap=WIN, stream_len=c.stream_len,
                        fast=c.fast if c.fast == "leave" else None))
        return out
    return out


def catalogue():
    rng = random.Random(2024)
    cases = []
    for fam in (fam_single_distance, fam_alphabet_sizes, fam_hclen, fam_cl_ops, fam_every_code, fam_random_sets,
                fam_pool, fam_multiblock):
        f = fam(rng)
        cases += f + edge_variants(f)
    cases += fam_quirks(rng) + fam_divergences(rng)
    assert len({c.name for c in cases}) == len(cases)
    return cases


# ------------------------------------------------------------------ seeded fuzz of valid streams
def fuzz_unit(rng, k):
    u = dc.Unit()
    nb = rng.randint(1, 6)
    budget = rng.choice([200, 1000, 5000, 20000, 65536])
    for b in range(nb):
        final = b == nb - 1
        share = rng.randint(0, max(0, (budget - len(u.plain)) // (nb - b)))
        kind = rng.randrange(3)
        if kind == 0:
            u.stored(bytes(rng.getrandbits(8) for _ in range(min(share, 3000))), final=final)
            continue
        if kind == 1:
            u.fixed(final=final)
        else:
            single = rng.random() < 0.25
            d = rng.randrange(30)
            dist = [0] * d + [1] if single else dist_lengths(rng, rng.randint(1, 30), rng.randint(5, 15))
            lit = lit_lengths(rng, rng.randint(257, 286), rng.randint(9, 15), must=[rng.randrange(256)])
            u.dynamic(lit, dist, final=final)
        if share:
            dc.random_symbols(u, rng, share, match_frac=rng.choice([0.0, 0.2, 0.5]), long_first=rng.random() < 0.5)
        u.eob()
    pad = rng.choice([2, 8, MIN_IN])
    return valid(f"fuzz_{k}", u, n=len(u.data()) + pad)


def fuzz(n, seed):
    rng = random.Random(seed)
    return [fuzz_unit(rng, k) for k in range(n)]


# ------------------------------------------------------------------ checks
def check_exact(c, st, out, used, oracle=None):
    """The exact kernels' outcome for case c: (status, bytes, in_used) against the case and the oracle."""
    ost, oout, oused = oracle if oracle is not None else orc.inflate(c.raw)
    assert st == c.status, (c, st)
    if c.status == NOSPC:
        assert len(out) <= c.cap and c.plain.startswith(out), c
        return
    if c.kind == "valid":
        assert ost == orc.OK and oout == c.plain, (c, ost)
        assert out == c.plain, c
        assert used == oused, (c, used, oused)
    elif c.kind == "quirk":
        assert ost == c.ostatus, (c, ost)
        assert out == oout == c.plain, c
        if st == DONE:
            assert used == oused, (c, used, oused)
    else:
        if c.ostatus is not None:
            assert ost == c.ostatus, (c, ost)
        assert out == c.plain, c
        assert oout.startswith(c.plain), c


@pytest.fixture(scope="module")
def cases():
    return catalogue()


@pytest.fixture(scope="module")
def fuzzed():
    return fuzz(300, 77)


def test_catalogue_covers_what_it_claims(cases):
    names = {c.name for c in cases}
    for need in ("pool_exactly_384", "pool_over_by_one_allocation", "hlit288_hdist32", "fixed_dist_hole_30",
                 "fixed_dist_hole_31", "cl_code_hole", "litlen_hole_hit", "last_block_not_final"):
        assert need in names
    assert sum(c.zlib_ok for c in cases) >= 15
    # the fast-kernel expectations are not vacuous: every unit asserted either way is one the kernel looks at
    for c in cases:
        if c.fast is not None:
            assert c.eligible() or c.name.endswith("@in30720"), c
    assert sum(c.fast == "finish" for c in cases) >= 40


def test_zlib_compatible_units_round_trip(cases, fuzzed):
    n = 0
    for c in cases + fuzzed:
        if c.zlib_ok and c.kind == "valid" and c.status != NOSPC:
            out, eof = dc.zlib_inflate(c.raw)
            assert out == c.plain, c
            assert eof == (c.status == DONE), c
            n += 1
    assert n >= 150


def test_exact_decoder_logic(cases, fuzzed):
    """tests/host_emul's build of inflate_decode.cuh's per-stream decode against the case and the oracle."""
    for c in cases + fuzzed:
        st, out, used, _ = orc.emul_inflate(c.raw, c.cap)
        check_exact(c, st, out, used)


def fast_outcomes(units, **kw):
    got = tfe.run_fast([c.raw for c in units], [c.cap for c in units], **kw)
    finished = 0
    for c, g in zip(units, got):
        if c.fast == "finish":
            assert g is not None, f"{c}: left by k_inflate_fast"
        elif c.fast == "leave":
            assert g is None, f"{c}: finished by k_inflate_fast, status {g[2]}"
        if g is not None:
            finished += 1
            check_exact(c, g[2], g[0], g[3])
            assert g[1] == len(g[0])
    return finished


def test_fast_kernel(cases):
    """k_inflate_fast finishes every clean eligible unit with the exact result, and leaves every quirk, every
    divergence, the pool one allocation past its 384 entries and every unit whose output passes its cap."""
    at_lead0 = [c for c in cases if "@in" in c.name]
    rest = [c for c in cases if "@in" not in c.name]
    assert fast_outcomes(rest) == sum(c.fast == "finish" for c in rest) >= 35
    assert fast_outcomes(at_lead0, misalign=False) == sum(c.fast == "finish" for c in at_lead0) >= 8
    assert any(c.name.endswith("@in192") for c in at_lead0) and any(c.name.endswith("@in30720") for c in at_lead0)


def test_fast_kernel_fuzz(fuzzed):
    want = sum(c.fast == "finish" for c in fuzzed)
    assert want >= 150
    assert fast_outcomes(fuzzed) == want


def test_fast_kernel_pool_boundary(cases):
    pool = [c for c in cases if c.name in ("pool_exactly_384", "pool_over_by_one_allocation")]
    got = tfe.run_fast([c.raw for c in pool], [c.cap for c in pool])
    assert [g is not None for g in got] == [True, False]
    st, out, _ = got[0][2], got[0][0], got[0][3]
    assert st == DONE and out == pool[0].plain


def test_fast_kernel_lz77_by_blocks(cases, monkeypatch):
    """The same units through k_inflate_fast built with -DFP_LZBLK=1 (its LZ77 pass by 2 KiB blocks)."""
    monkeypatch.setattr(tfe, "_E", C.CDLL(os.path.join(ROOT, "tests", "host_emul", "libinflate_emul_lzblk.so")))
    rest = [c for c in cases if "@in" not in c.name]
    assert fast_outcomes(rest) == sum(c.fast == "finish" for c in rest)


def test_multi_lane_exact_kernels(cases, fuzzed):
    """k_inflate_decode with helper lanes + k_inflate_expand: the same as one lane per stream, and that is the exact
    outcome."""
    units = cases + fuzzed
    ref = tse.same_as_one_lane([c.raw for c in units], [c.cap for c in units], "crafted")
    for i, c in enumerate(units):
        check_exact(c, ref[2][i], ref[0][i], ref[3][i])
