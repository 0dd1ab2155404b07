"""K12 inside b200z_zip_extract: large ZIP members decoded by many chunks, as one batch of streams, on the emulated library
(the whole product library compiled for the host, tests/host_emul/build_emu_lib.py).  The threshold is lowered to 16 KiB
of compressed input and the chunk size to 4 KiB through the test hook, so that members of about 100 KiB of text take K12
with a dozen chunks each.  Every archive is extracted through K12 and through the exact path by the same library; the
results must be identical and match the oracle (tests/zip_chunked_cases.py).  The statistics hook tells which members
K12 took."""
import ctypes as C
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "host_emul"))
sys.path.insert(0, os.path.dirname(HERE))

import zip_chunked_cases as zc  # noqa: E402
from archive_b200 import synth  # noqa: E402

THRESH, CHUNK = 16 << 10, 4 << 10
TEXT = synth.text(2_000_000, stream=12).tobytes()
BIG, SMALL = 120_000, 6_000


@pytest.fixture(scope="module")
def H():
    import build_emu_lib
    L = C.CDLL(build_emu_lib.build())
    assert L.b200z_init(0, 0) == 0
    h = zc.Harness(L, THRESH, CHUNK)
    yield h
    h.set(0, 0)
    h.caps()


@pytest.mark.parametrize("web_eos", [False, True])
def test_mixed_members(H, web_eos):
    zc.case_mixed(H, TEXT, BIG, SMALL, web_eos)


@pytest.mark.parametrize("web_eos", [False, True])
def test_final_code_in_last_bits(H, web_eos):
    zc.case_final_code_in_last_bits(H, TEXT, BIG, web_eos)


def test_bitflip_spares_the_batch(H):
    zc.case_bitflip(H, TEXT, BIG, SMALL)


def test_room_one_short_and_zero_sizes(H):
    zc.case_room_one_short_and_zero_sizes(H, TEXT, BIG)


def test_random_declined(H):
    zc.case_random_declined(H, TEXT, BIG, 60_000)


def test_flush_points(H):
    zc.case_flush_points(H, TEXT, 800_000, 30_000)


def test_encrypted(H):
    zc.case_encrypted(H, TEXT, BIG, SMALL)


@pytest.mark.parametrize("n_chunks", [1, 3, 64])
def test_zip_chunks(H, n_chunks):
    zc.case_zip_chunks(H, TEXT, BIG, SMALL, n_chunks)


def test_pool_cap(H):
    # a block repeated within the window: 2 MB of output from 26 KB
    zc.case_pool_cap(H, TEXT, BIG, SMALL, TEXT[:20_000] * 100, 32)


def test_one_stream_per_batch(H):
    zc.case_one_stream_per_batch(H, TEXT, BIG, SMALL)
