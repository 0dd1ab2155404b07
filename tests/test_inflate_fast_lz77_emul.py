"""k_inflate_fast's LZ77 pass on the CUDA execution-model emulation, on hand-built DEFLATE streams whose matches stress
its copy turns: runs of 258 at short distances (a run that overlaps itself doubles its stride), hundreds of matches ready
at once with lengths from 3 to 258, short matches back to back, chains of matches deeper than the benchmark text's 42,
distance 32 768, matches that end in the ragged tail of a unit's store, and a unit that falls back after a clean block.
Every other unit must be finished by the fast kernel and give the oracle's bytes, out_len, status and in_used; the unit
that falls back must be left untouched.  The same streams run on the GPU in tests/test_inflate_fast_lz77_gpu.py."""
import random

import deflate_craft as dc
from test_inflate_fast_emul import check_against_oracle, run_fast

MIN_IN = 192  # shorter units are not k_inflate_fast's


def _unit(rng, lead=400):
    """A fixed-code final block that opens with `lead` random literals (so the unit is long enough for the fast kernel)."""
    u = dc.Unit()
    u.fixed(final=True)
    u.literals(bytes(rng.randrange(256) for _ in range(lead)))
    return u


def _done(u):
    u.eob()
    raw = u.data()
    assert MIN_IN <= len(raw) <= 30000, len(raw)
    return raw + bytes(8), bytes(u.plain)


def long_runs(rng):
    """Runs of 258 at short distances, several in a row (each overlaps itself and reads the run before it)."""
    out = []
    for d in (1, 2, 3, 7, 31, 33):
        u = _unit(rng)
        for k in range(12):
            u.match(258, d)
            if k % 4 == 3:
                u.literals(bytes(rng.randrange(256) for _ in range(rng.randrange(1, 5))))
        out.append(_done(u))
    return out


def many_ready(rng):
    """Hundreds of matches that all read the literal prefix: every look finds its match ready, and a turn holds matches
    of every length from 3 to 258."""
    out = []
    for lens in ((3, 4, 5, 6, 7), (3, 258, 4, 131, 5, 64), tuple(range(3, 40))):
        u = _unit(rng, 2000)
        for k in range(600):
            ln = lens[k % len(lens)] if k % 3 else rng.randrange(3, 259)
            u.match(ln, rng.randrange(ln, 1900) if ln < 1900 else 1900)
        out.append(_done(u))
    return out


def short_neighbours(rng):
    """Short matches back to back, overlapping and not, at distances that read the matches just before them."""
    u = _unit(rng)
    for _ in range(1500):
        ln = rng.choice((3, 4, 5))
        u.match(ln, rng.choice((1, 2, 3, ln, 5, 9, 100, 380)))
    return [_done(u)]


def deep_chains(rng):
    """Chains of matches that each read the one before: 200 deep, and 120 deep with overlapping runs."""
    out = []
    u = _unit(rng, 300)
    for _ in range(200):
        u.match(16, 16)
    out.append(_done(u))
    u = _unit(rng, 300)
    for k in range(120):
        u.match(20 + k % 7, 13 + k % 5)
        u.literals(bytes([rng.randrange(256)]))
    out.append(_done(u))
    return out


def far(rng):
    """Matches at distance 32 768 (and just short of it), after 33 KB of varied output."""
    u = _unit(rng, 600)
    while len(u.plain) < 33000:
        u.literals(bytes(rng.randrange(256) for _ in range(5)))
        ln = rng.randrange(20, 259)
        u.match(ln, rng.randrange(ln + 1, min(len(u.plain), 32768) + 1))
    for ln in (3, 258, 17, 258):
        u.match(ln, 32768)
        u.match(ln, 32767)
        u.literals(bytes([rng.randrange(256)]))
    return [_done(u)]


def ragged_ends(rng):
    """Units whose output ends in a match, at every length modulo 16, so the last match ends in the ragged tail of the
    store (the tests run every unit at two window alignments)."""
    out = []
    for r in range(16):
        u = _unit(rng, 300)
        while (len(u.plain) + 40) % 16 != r:
            u.lit_byte(rng.randrange(256))
        u.match(40, rng.choice((1, 3, 33, 250)))
        out.append(_done(u))
    return out


def falls_back(rng):
    """A unit whose first block is clean and whose second block is of the reserved type: the fast kernel leaves it."""
    u = dc.Unit()
    u.fixed()
    u.literals(bytes(rng.randrange(256) for _ in range(400)))
    for _ in range(20):
        u.match(258, rng.choice((1, 7, 300)))
    u.eob()
    u.reserved(final=True)
    u.bits(0, 16)
    return u.data() + bytes(8), bytes(u.plain)


def cases():
    rng = random.Random(77)
    units = []
    for make in (long_runs, many_ready, short_neighbours, deep_chains, far, ragged_ends):
        units += make(rng)
    return units


def test_lz77_copy_turns_against_oracle():
    units = cases()
    raws = [r for r, _ in units]
    caps = [len(p) for _, p in units]
    for misalign in (True, False):
        got = check_against_oracle(raws, caps, must_finish=len(raws), misalign=misalign)
        assert [g[0] for g in got] == [p for _, p in units]


def test_unit_that_falls_back_is_left():
    rng = random.Random(78)
    bad, plain = falls_back(rng)
    good = long_runs(rng)[:2]
    got = run_fast([good[0][0], bad, good[1][0]], [len(good[0][1]), 65536, len(good[1][1])])
    assert got[1] is None
    assert got[0][0] == good[0][1] and got[2][0] == good[1][1]
