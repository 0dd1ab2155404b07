"""The BZip2 encoder's edge catalogue (tests/test_bzip2_enc_edges_emul.py) on the device, through BZip2Encoder: the
oracle's bytes, a libbz2 round trip, the table check of tests/bz2_stream.py and each case's own edge claim.  Also inputs
split into several batches, by the test hook b200z_debug_bzip2_encode_batch_set and, above 256 blocks, by the built-in
plan; and an output buffer one byte short."""
import bz2
import ctypes as C

import pytest

import bz2_stream as bs
import oracle_lib as orc
import test_bzip2_enc_edges_emul as cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def a():
    import archive_b200
    return archive_b200


@pytest.fixture
def lib(a):
    from archive_b200 import _ffi
    _ffi.ensure_init()
    L = _ffi.lib()
    yield L
    L.b200z_debug_bzip2_encode_batch_set(C.c_uint(0))


def enc(a, data):
    return a.BZip2Encoder().encode_bytes(data)


@pytest.mark.parametrize("name", list(cases.CASES))
def test_edge_case(a, name):
    data = cases.case_input(name)
    cases.check(data, enc(a, data), cases.CASES[name][1])


def test_mixed_batch(a):
    data = cases.mixed_input()
    s, _ = cases.check(data, enc(a, data))
    assert len(s.blocks) == 4


@pytest.mark.parametrize("max_batch", [1, 2, 3])
def test_several_batches(a, lib, max_batch):
    lib.b200z_debug_bzip2_encode_batch_set(C.c_uint(max_batch))
    for data in (cases.batches_input(), cases.mixed_input()):
        cases.check(data, enc(a, data))


@pytest.mark.needs_device
def test_more_than_256_blocks(a):
    """The built-in plan codes at most 256 blocks per batch: 240 MiB of text is about 280 blocks.  The oracle's output
    cap for runaway decodes (16 MiB, set by oracle_lib) is lifted for this call: the encoder entry point does not catch
    the cap's exit, and its 70 MB output is no runaway."""
    from archive_b200 import synth
    src = synth.text(240 << 20, stream=500).tobytes()
    z = enc(a, src)
    crcs, combined = bs.scan_headers(z)
    assert len(crcs) > 256
    assert bs.fold_crcs(crcs) == combined
    orc.L().orc_set_runaway_limit(C.c_int64(1 << 40))
    try:
        st, ref = orc.bzip2_encode(src)
    finally:
        orc.L().orc_set_runaway_limit(C.c_int64(1 << 24))
    assert st == orc.OK and z == ref
    assert bz2.decompress(z) == src


def test_out_cap_one_byte_short(a, lib):
    from archive_b200 import _ffi
    data = cases.case_input("length_retry_a")
    need = len(orc.bzip2_encode(data)[1])
    out = (C.c_uint8 * need)()
    n = C.c_size_t(0)
    assert lib.b200z_bzip2_encode(data, len(data), C.addressof(out), need - 1, C.byref(n)) == _ffi.E_NOSPC
    assert n.value == need
    assert lib.b200z_bzip2_encode(data, len(data), C.addressof(out), need, C.byref(n)) == _ffi.OK
    assert n.value == need and bytes(out) == orc.bzip2_encode(data)[1]
