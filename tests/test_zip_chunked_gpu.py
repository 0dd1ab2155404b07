"""K12 inside b200z_zip_extract on the device: the cases of tests/test_zip_chunked_emul.py at the built-in chunk size, with
the threshold lowered to 1 MiB of compressed input so that members of a few MiB of text take K12; and one archive written
by Python's zipfile with three members of more than 16 MiB compressed each, at the built-in threshold, checked against
zlib.  Every archive of the shared cases is extracted through K12 and through the exact path; the results must be
identical and match the oracle (tests/zip_chunked_cases.py).  With B200Z_EMU_TESTS=1 the same cases run on the emulated
library, except the one at the built-in threshold."""
import ctypes as C
import os
import zlib

import pytest

import zip_chunked_cases as zc

pytestmark = pytest.mark.gpu
EMU = os.environ.get("B200Z_EMU_TESTS") == "1"
MiB = 1 << 20
LOW = 1 * MiB  # K12 threshold for these tests (compressed bytes)
BIG, SMALL = 3_200_000, 100_000  # text of a large member (about 1.2 MiB compressed) and of a small one
# pages per pool: more than a BIG member takes in any region (110 fail it), fewer than the member of 3 * BIG needs (135 do
# not); page use is deterministic (it depends on the chunks' outputs, not on their order)
POOL_CAP = 122


@pytest.fixture(scope="module")
def text():
    from archive_b200 import synth
    return synth.text(12 * MiB, stream=21).tobytes()


@pytest.fixture(scope="module")
def H():
    from archive_b200 import _ffi
    L = _ffi.ensure_init()
    h = zc.Harness(L, LOW, 0)
    yield h
    h.set(0, 0)
    h.caps()


@pytest.mark.parametrize("web_eos", [False, True])
def test_mixed_members(H, text, web_eos):
    zc.case_mixed(H, text, BIG, SMALL, web_eos)


@pytest.mark.parametrize("web_eos", [False, True])
def test_final_code_in_last_bits(H, text, web_eos):
    zc.case_final_code_in_last_bits(H, text, BIG, web_eos)


def test_bitflip_spares_the_batch(H, text):
    zc.case_bitflip(H, text, BIG, SMALL)


def test_room_one_short_and_zero_sizes(H, text):
    zc.case_room_one_short_and_zero_sizes(H, text, BIG)


def test_random_declined(H, text):
    zc.case_random_declined(H, text, BIG, 2 * MiB)


def test_flush_points(H, text):
    zc.case_flush_points(H, text, BIG, 256 << 10)


def test_encrypted(H, text):
    zc.case_encrypted(H, text, BIG, SMALL)


@pytest.mark.parametrize("n_chunks", [1, 3, 64])
def test_zip_chunks(H, text, n_chunks):
    zc.case_zip_chunks(H, text, BIG, SMALL, n_chunks)


def test_pool_cap(H, text):
    # three times the text of its neighbours: three times their pages
    zc.case_pool_cap(H, text, BIG, SMALL, text[2 * BIG:5 * BIG], POOL_CAP)


def test_one_stream_per_batch(H, text):
    zc.case_one_stream_per_batch(H, text, BIG, SMALL)


@pytest.mark.skipif(EMU, reason="members of 45 MiB: too slow for the emulated library")
def test_three_members_at_builtin_threshold(H, text):
    import archive_b200 as a
    from archive_b200 import synth
    big = synth.text(3 * 45 * MiB, stream=22).tobytes()
    parts = [(f"m{i}.txt", big[i * 45 * MiB:(i + 1) * 45 * MiB]) for i in range(3)]
    data = zc.zipfile_archive(parts + [("small.txt", text[:SMALL])])
    H.set(0, 0)
    arc = a.ZipDecoder().decode_bytes(data)
    st = H.stats()
    import zipfile
    import io
    with zipfile.ZipFile(io.BytesIO(data)) as z:
        infos = z.infolist()
        assert all(i.compress_size >= 16 * MiB for i in infos[:3])
    assert [f.name for f in arc.files] == [p[0] for p in parts] + ["small.txt"]
    for f, (name, body) in zip(arc.files, parts + [("small.txt", text[:SMALL])]):
        assert f.content == body and zlib.crc32(f.content) == f.crc32, name
    assert st["offered"] == 3 and st["accepted"] == 3 and st["batches"] == 1, st
