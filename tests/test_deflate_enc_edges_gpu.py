"""The Deflate encoder's edge catalogue (tests/test_deflate_enc_edges_emul.py) on the device: through Deflate
(b200z_deflate_raw) and through one b200z_deflate_batch call of the whole catalogue per level, where levels 1-3 take the
multi-member k_defl_fast_batch.  Every stream must be the oracle's, decode to its input through tests/deflate_stream.py,
pass the table check and keep each case's own edge claim.  Also one input of about 64 MiB made of the designed segments,
whose hundreds of repaired trees are built by concurrent k_defl_block_trees CTAs."""
import ctypes as C
import time
import zlib

import pytest

import deflate_stream as ds
import oracle_lib as orc
import test_deflate_enc_edges_emul as cases

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]


@pytest.fixture(scope="module")
def a():
    import archive_b200
    return archive_b200


@pytest.mark.parametrize("name", list(cases.CASES))
def test_edge_case(a, name):
    make, claim, levels, wbits = cases.CASES[name]
    data = make()
    for level in levels:
        z = a.Deflate(data, level=level, window_bits=wbits).get_bytes()
        s, plans = cases.check(data, z, level, wbits)
        claim(s, plans, level)


@pytest.mark.parametrize("lanes", ["1", None])
def test_catalogue_in_one_batch(a, monkeypatch, lanes):
    from archive_b200.zip import deflate_batch
    if lanes is None:
        monkeypatch.delenv("B200Z_DEFLATE_LANES", raising=False)
    else:
        monkeypatch.setenv("B200Z_DEFLATE_LANES", lanes)
    by_wbits = {}
    for name, (make, claim, levels, wbits) in cases.CASES.items():
        by_wbits.setdefault(wbits, []).append((name, make(), claim, levels))
    for wbits, items in by_wbits.items():
        for level in (1, 2, 3, 4, 6, 9):
            got = deflate_batch([d for _, d, _, _ in items], level, wbits)
            for (name, data, claim, levels), (z, crc) in zip(items, got):
                assert crc == zlib.crc32(data), name
                s, plans = cases.check(data, z, level, wbits)
                if level in levels:
                    claim(s, plans, level)


@pytest.mark.needs_device
def test_64_mib_of_repaired_trees(a):
    """Levels 1 and 6 both give the oracle's stream, which zlib decodes.  The designed tokens are the same at both
    levels, so the pure-Python reader (about a minute for this input) reads the level-6 stream only: every designed
    block must run the 15-bit repair."""
    # every segment is whole blocks (a literal history, then one designed block of 16383 tokens); neighbours use
    # disjoint byte sets, so no match crosses from one into the next and every designed block stays as designed
    segs = [cases.litlen_depth_input(18, segment=0), cases.dist_depth_input(18, segment=1),
            cases.litlen_depth_input(16, segment=0), cases.dist_depth_input(16, segment=1)]
    parts, n = [], 0
    while n < 64 << 20:
        parts.append(segs[len(parts) % 4])
        n += len(parts[-1])
    data = b"".join(parts)
    orc.L().orc_set_runaway_limit(C.c_int64(1 << 40))  # (a 64 MiB input is no runaway)
    try:
        for level in (1, 6):
            z = a.Deflate(data, level=level).get_bytes()
            st, ref, _ = orc.deflate(data, level)
            assert st == orc.OK and z == ref, level
            assert zlib.decompress(z, -15) == data, level
    finally:
        orc.L().orc_set_runaway_limit(C.c_int64(1 << 24))
    t = time.time()
    s = ds.parse(z)
    assert s.data == data
    repaired = 0
    for b in s.blocks:
        p = ds.check_block(b)
        if p is not None and (p.lt.overflow or p.dt.overflow):
            repaired += 1
    print(f"{len(s.blocks)} blocks, {repaired} repaired, read and checked in {time.time() - t:.1f} s")
    assert repaired > 100 and repaired == len(parts), (repaired, len(parts))
