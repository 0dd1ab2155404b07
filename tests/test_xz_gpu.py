"""XZDecoder / XZEncoder / getCrc64 on the device (b200z_xz_decode, b200z_xz_encode, b200z_crc64) against the oracle
(oracle/xz.c): identical status, out_len and bytes on valid streams, chunk edits and damage."""
import ctypes as C
import lzma
import os
import random
import tarfile

import pytest

import oracle_lib as orc
import xz_build as xb

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "xz")
# the oracle's status -> b200z return code
RC = {orc.OK: 0, orc.FALSE: -4, orc.THROW: -5}
TEXT = b"".join(b"line %d: the quick brown fox jumps over the lazy dog %d\n" % (i, i * i % 977) for i in range(4000))


def device(data: bytes, verify=False, cap=None):
    from archive_b200 import _ffi
    L = _ffi.ensure_init()
    addr, n, keep = _ffi.as_buffer(bytes(data))
    bound = L.b200z_xz_bound(addr, n)
    cap = bound if cap is None else cap
    out = (C.c_uint8 * max(cap, 1))()
    got = C.c_size_t(0)
    rc = L.b200z_xz_decode(addr, n, int(verify), C.addressof(out), cap, C.byref(got))
    return rc, bytes(out[:min(got.value, cap)]) if rc != -3 else got.value


def same(data: bytes, verify=False):
    st, want = xb.decode(data, verify)
    rc, got = device(data, verify)
    if st == orc.THROW:
        assert rc == -5
        return st
    assert (rc, got) == (RC[st], want)
    return st


@pytest.mark.parametrize("name", sorted(f for f in os.listdir(GOLD) if f.endswith(".xz")))
def test_fixtures(name):
    for verify in (False, True):
        assert same(open(os.path.join(GOLD, name), "rb").read(), verify) == orc.OK


@pytest.mark.parametrize("preset", [0, 1, 6, 9])
@pytest.mark.parametrize("check", [lzma.CHECK_NONE, lzma.CHECK_CRC32, lzma.CHECK_CRC64, lzma.CHECK_SHA256])
def test_lzma_streams(preset, check):
    assert same(lzma.compress(TEXT, preset=preset, check=check), True) == orc.OK


@pytest.mark.parametrize("lc,lp,pb", [(0, 0, 0), (4, 0, 2), (0, 4, 1), (1, 3, 3), (2, 2, 0)])
def test_props(lc, lp, pb):
    assert same(xb.container([(xb.raw_lzma2(TEXT, lc=lc, lp=lp, pb=pb), TEXT)]), True) == orc.OK


def test_large_lc_uses_global_model():
    # liblzma writes only lc + lp <= 4; the props byte is rewritten to lc = 8 (the model then needs 393 KB): the bytes
    # differ from the input, but the oracle and the device must agree
    raw = bytearray(xb.raw_lzma2(TEXT[:20000], lc=4, lp=0, pb=2))
    assert raw[0] == 0xE0
    raw[5] = 2 * 45 + 0 * 9 + 8  # lc = 8
    same(xb.container([(bytes(raw), TEXT[:20000])]))


@pytest.mark.parametrize("nblocks", [1, 7, 1000])
def test_blocks(nblocks):
    data = (TEXT * 3)[: 2000 * nblocks]
    bs = max(1, len(data) // nblocks)
    for check in ("crc32", "crc64", "sha256", "none"):
        assert same(xb.xz_blocks(data, bs, check=check), True) == orc.OK


def test_incompressible_and_size_fields():
    data = random.Random(5).randbytes(300000)
    assert same(xb.container([(xb.raw_lzma2(data), data)], sizes=(True, True)), True) == orc.OK


def test_pb4_throws():
    assert same(xb.container([(xb.raw_lzma2(TEXT, pb=4), TEXT)])) == orc.THROW


def test_chunk_edits():
    r = random.Random(11)
    words = [bytes(r.randbytes(r.randrange(2, 9))) for _ in range(4000)]
    PLAIN = b" ".join(r.choice(words) for _ in range(120000))
    raw = xb.raw_lzma2(PLAIN, preset=1)
    chs = xb.chunks(raw)
    assert len(chs) > 3
    # a block whose first chunk does not reset the dictionary (reset 3 -> reset 2, and -> reset 0)
    for new in (0xC0, 0x80):
        c0, h0, d0 = chs[0]
        h = bytes([(c0 & 0x1F) | new]) + h0[1:] if new == 0xC0 else bytes([(c0 & 0x1F) | new]) + h0[1:5]
        same(xb.container([(xb.join([(new, h, d0)] + chs[1:]), PLAIN)]))
    # a stored chunk without an earlier reset (control 2 first), then the LZMA chunks
    same(xb.container([(xb.join([(2, b"\x02\x00\x04", b"hello")] + chs), b"hello" + PLAIN)]))
    # a props change without a dictionary reset: the second chunk gets reset 2 with other props
    c1, h1, d1 = chs[1]
    h = bytes([(c1 & 0x1F) | 0xC0]) + h1[1:5] + bytes([2 * 45 + 1 * 9 + 3])
    same(xb.container([(xb.join([chs[0], (0xC0, h, d1)] + chs[2:]), PLAIN)]))
    # a read past a chunk's compressed bytes: its compressed size cut to 8
    c, h, d = chs[1]
    h = h[:3] + bytes([0, 7]) + h[5:]
    assert same(xb.container([(xb.join([chs[0], (c, h, d[:8])] + chs[2:]), PLAIN)])) == orc.THROW
    # control 3: false with the chunks before it
    assert same(xb.container([(xb.join(chs[:2])[:-1] + b"\x03" + xb.join(chs[2:]), PLAIN)])) == orc.FALSE


def test_verify_on_and_off():
    for check in ("crc32", "crc64"):
        bad = xb.container([(xb.raw_lzma2(TEXT), TEXT)], check=check, bad_check=True)
        assert same(bad, False) == orc.OK
        assert same(bad, True) == orc.FALSE


def test_damage():
    good = xb.xz_blocks(TEXT * 2, 60000, check="crc64")
    seen = set()
    for k in range(0, len(good), max(1, len(good) // 150)):
        seen.add(same(good[:k], True))
    for seed in range(150):
        seen.add(same(xb.flip_bits(good, seed, 1 + seed % 3), seed % 2 == 0))
    # header / index / footer CRCs
    for pos in (8, 12 + 8, len(good) - 12 - 2, len(good) - 10):
        b = bytearray(good)
        b[pos] ^= 0x40
        seen.add(same(bytes(b), True))
    assert {orc.FALSE, orc.THROW} <= seen


def test_out_cap_one_short():
    data = lzma.compress(TEXT)
    rc, need = device(data, cap=len(TEXT) - 1)
    assert rc == -3 and need == len(TEXT)
    assert device(data, cap=len(TEXT)) == (0, TEXT)


def test_classes_and_throw():
    import archive_b200 as a
    assert a.XZDecoder().decode_bytes(lzma.compress(TEXT)) == TEXT
    with pytest.raises(a.DartRangeError):
        a.XZDecoder().decode_bytes(xb.container([(xb.raw_lzma2(TEXT, pb=4), TEXT)]))
    assert a.get_crc64(b"123456789") == 0x995DC9BBDF1939FA
    big = random.Random(2).randbytes(1 << 20)
    assert a.get_crc64(big) == xb.crc64(big)


@pytest.mark.parametrize("n", [0, 6, 65536, 65537, 300000])
def test_encoder_identity(n):
    import archive_b200 as a
    data = random.Random(n).randbytes(n)
    for check in (a.XZCheck.none, a.XZCheck.crc32, a.XZCheck.crc64, a.XZCheck.sha256):
        assert a.XZEncoder().encode_bytes(data, check=check) == xb.encode(data, check)


def test_file_streams_and_tar_xz(tmp_path):
    import io as _io
    import archive_b200 as a
    src = tmp_path / "in.xz"
    src.write_bytes(xb.xz_blocks(TEXT, 30000))
    inp, out = a.InputFileStream(str(src)), a.OutputFileStream(str(tmp_path / "out.bin"))
    assert a.XZDecoder().decode_stream(inp, out) is True
    inp.close_sync()
    out.close_sync()
    assert (tmp_path / "out.bin").read_bytes() == TEXT
    plain = tmp_path / "plain.bin"
    plain.write_bytes(TEXT[:1000])
    inp, out = a.InputFileStream(str(plain)), a.OutputFileStream(str(tmp_path / "enc.xz"))
    a.XZEncoder().encode_stream(inp, out, check=a.XZCheck.crc32)
    inp.close_sync()
    out.close_sync()
    assert (tmp_path / "enc.xz").read_bytes() == xb.encode(TEXT[:1000], 1)
    buf = _io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w") as t:
        ti = tarfile.TarInfo("a.txt")
        ti.size = len(TEXT)
        t.addfile(ti, _io.BytesIO(TEXT))
    for name in ("x.tar.xz", "y.txz"):
        (tmp_path / name).write_bytes(lzma.compress(buf.getvalue()))
        got = a.extract_file_to_disk(str(tmp_path / name), str(tmp_path / ("o" + name)))
        assert len(got) == 1 and open(got[0], "rb").read() == buf.getvalue()


@pytest.mark.needs_device
def test_256mib_in_1mib_blocks():
    from archive_b200 import synth
    data = synth.text(256 << 20, stream=3).tobytes()
    raws = [xb.raw_lzma2(data[o:o + (1 << 20)], preset=1) for o in range(0, len(data), 1 << 20)]
    c = xb.container([(r, data[i << 20:(i + 1) << 20]) for i, r in enumerate(raws)], check="crc64")
    rc, out = device(c, True)
    assert rc == 0 and out == data


def test_overshoot_is_a_throw():
    """A chunk whose declared size ends inside a match: the reference lets the match finish when its dictionary list has
    room (and then yields more than declared) and throws otherwise; the device always reports a throw (DESIGN.md 7)."""
    chs = xb.chunks(xb.raw_lzma2(TEXT))
    assert len(chs) == 1 and chs[0][0] >= 0xE0
    c, h, d = chs[0]
    ulen = ((c & 0x1F) << 16 | h[1] << 8 | h[2]) + 1
    overshoots = 0
    for k in range(1, 60):
        u = ulen - k - 1
        hh = bytes([(c & 0xE0) | (u >> 16), (u >> 8) & 0xFF, u & 0xFF]) + h[3:]
        s = xb.container([(xb.join([(c, hh, d)]), TEXT[:-k])])
        st, want = xb.decode(s)
        rc, got = device(s)
        if st == orc.THROW or len(want) > len(TEXT) - k:
            overshoots += 1
            assert rc == -5
        else:
            assert (rc, got) == (RC[st], want)
    assert overshoots > 0


def _trim_corpus():
    r = random.Random(23)
    words = [bytes(r.randbytes(r.randrange(2, 9))) for _ in range(3000)]
    return b" ".join(r.choice(words) for _ in range(110000))


@pytest.mark.parametrize("lc,lp,pb", [(3, 0, 2), (0, 2, 0), (3, 1, 3)])
def test_trimmed_dictionary(lc, lp, pb):
    """A 4 KiB dictionary (dictionary byte 0): trimDictionary moves the dictionary after every chunk, so the chunks'
    dictionary positions, posState and the reach check all run on trimmed positions."""
    plain = _trim_corpus()
    raw = xb.raw_lzma2(plain, preset=1, lc=lc, lp=lp, pb=pb, dict_size=4096)
    assert len(xb.chunks(raw)) > 3
    assert same(xb.container([(raw, plain)], dict_byte=0), True) == orc.OK
    # distances made for an 8 MiB dictionary reach before the trimmed dictionary's start
    far = xb.raw_lzma2(plain, preset=1, lc=lc, lp=lp, pb=pb)
    assert same(xb.container([(far, plain)], dict_byte=0)) == orc.THROW


def test_props_change_after_trim():
    plain = _trim_corpus()
    chs = xb.chunks(xb.raw_lzma2(plain, preset=1, dict_size=4096))
    for k in (2, 3):
        c, h, d = chs[k]
        for props in (2 * 45 + 1 * 9 + 3, 0 * 45 + 0 * 9 + 3, 4 * 45 + 3):
            hh = bytes([(c & 0x1F) | 0xC0]) + h[1:5] + bytes([props])
            same(xb.container([(xb.join(chs[:k] + [(0xC0, hh, d)] + chs[k + 1:]), plain)], dict_byte=0))
