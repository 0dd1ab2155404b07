"""The hand-built DEFLATE catalogue of tests/test_inflate_crafted_emul.py, and a larger seeded fuzz of valid hand-built
streams, through every inflate entry point of the library against the oracle: b200z_inflate_batch_device on both
kernels (k_inflate_fast, and the exact pair B200Z_FAST=0 leaves everything to), b200z_inflate_batch, Inflate on one
stream, GZipDecoder / GZipDecoderWeb on members with and without the BGZF size hint, and ZipDecoder's batch extraction.
Runs on an H100 and, with B200Z_EMU_TESTS=1, on the emulated library."""
import random

import pytest

import deflate_craft as dc
import oracle_lib as orc
from test_inflate_crafted_emul import DONE, EOS, catalogue, check_exact, fuzz
from test_inflate_device_gpu import EMU, Backend, Batch, both_kernels, check_guards, run
from test_inflate_gpu import inflate_batch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def B():
    return Backend()


@pytest.fixture(scope="module")
def a():
    import archive_b200
    return archive_b200


@pytest.fixture(scope="module")
def units():
    return catalogue() + fuzz(300 if EMU else 2000, 78)


def clean(units):
    """Valid units that end with their final block, once per stream: the framing tests' members."""
    seen, out = set(), []
    for c in units:
        s = c.raw[:c.stream_len]
        if c.kind == "valid" and c.status == DONE and "@" not in c.name and s not in seen:
            seen.add(s)
            out.append(c)
    return out


def test_device_batch_both_kernels(B, monkeypatch, units):
    """Both kernels give the same results, touch nothing outside the slots, and give each case's exact outcome.  The
    units padded to 30720 bytes sit at lead 0, where k_inflate_fast still takes them."""
    rng = random.Random(3)
    leads = [0 if c.name.endswith("@in30720") else rng.randrange(16) for c in units]
    b = Batch([c.raw for c in units], [c.cap for c in units], rng=rng, leads=leads)
    r = both_kernels(monkeypatch, lambda: run(B, b))
    check_guards(r)
    for i, c in enumerate(units):
        check_exact(c, *r.unit(i))


def test_host_batch(units):
    res = inflate_batch([c.raw for c in units], [c.cap for c in units])
    for c, (st, out, used) in zip(units, res):
        check_exact(c, st, out, used)


def test_inflate_one_stream(a, units):
    """Inflate(bytes) on every stream the reference decodes without a throw: the oracle's bytes."""
    seen = set()
    for c in units:
        if c.raw in seen or c.kind == "diverge" or c.status not in (DONE, EOS, -1):
            continue
        seen.add(c.raw)
        ost, oout, _ = orc.inflate(c.raw)
        assert ost == orc.OK
        assert a.Inflate(c.raw).get_bytes() == oout, c


@pytest.mark.parametrize("hint", [True, False])
def test_gzip_members(a, units, hint):
    """The clean units as gzip streams of members (with or without the 'BC' size hint where it fits), each stream
    under 8 MiB of output (the oracle stops a decode at 16 MiB)."""
    groups, cur, size = [], [], 0
    for c in clean(units):
        if cur and size + len(c.plain) > 8 << 20:
            groups.append(cur)
            cur, size = [], 0
        cur.append(c)
        size += len(c.plain)
    groups.append(cur)
    for cs in groups:
        blob = b"".join(dc.gzip_member(c.raw[:c.stream_len], c.plain, hint and c.stream_len + 26 <= 65536) for c in cs)
        want = b"".join(c.plain for c in cs)
        st, oout = orc.gzip_decode(blob)
        assert st == orc.OK and oout == want
        assert a.GZipDecoder().decode_bytes(blob) == want
        assert a.GZipDecoderWeb().decode_bytes(blob, verify=True) == want


def test_zip_batch_extraction(a, units):
    cs = clean(units)
    z = dc.zip_of([(f"m{i:04d}.bin", c.raw[:c.stream_len], c.plain) for i, c in enumerate(cs)])
    got = {f.name: f.content for f in a.ZipDecoder().decode_bytes(z).files}
    assert len(got) == len(cs)
    for i, c in enumerate(cs):
        assert got[f"m{i:04d}.bin"] == c.plain, c
