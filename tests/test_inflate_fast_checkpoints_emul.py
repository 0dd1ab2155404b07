"""k_inflate_fast's checkpoint counts (archive_b200/csrc/inflate_fast.cuh), on the CUDA execution-model emulation.

A lane that decodes from a guessed offset records, at the first token boundary it marks in each 32-bit word of its bitmap
row, how many bytes it has counted so far.  When the true parse meets the lane, the bytes before the meeting point are
then counted from that word's checkpoint -- the meeting point itself, or a few symbols before it -- instead of from the
guessed offset.  A block whose room in the window cannot hold the counts counts every false start from its guessed
offset.  These tests build the kernel with -DFP_DEBUG, whose counters tell which of the three ways each false start was
counted, and check that every way is taken on units checked byte for byte against the oracle.  Builds with a slip in
what the checkpoints record or how they are read must fail the same checks."""
import ctypes as C
import os
import random
import shutil
import subprocess
import zlib

import pytest

import test_inflate_fast_emul as tfe

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "archive_b200", "csrc")
EMUL = os.path.join(ROOT, "tests", "host_emul")
WRAPPER = """#include "inflate_emul.cpp"
extern "C" void emu_fast_dbg_counts(unsigned long *o) {
  o[0] = fp::fp_dbg_restarts;
  o[1] = fp::fp_dbg_ck_exact;
  o[2] = fp::fp_dbg_ck_walk;
  o[3] = fp::fp_dbg_ck_full;
  fp::fp_dbg_restarts = fp::fp_dbg_ck_exact = fp::fp_dbg_ck_walk = fp::fp_dbg_ck_full = 0;
}
"""


def _compile(workdir, emul_dir):
    src = os.path.join(workdir, "fast_dbg.cpp")
    with open(src, "w") as f:
        f.write(WRAPPER)
    so = os.path.join(workdir, "libfast_dbg.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-DFP_DEBUG", "-I", emul_dir, src, "-o", so], check=True)
    return C.CDLL(so)


@pytest.fixture(scope="module")
def dbg_lib(tmp_path_factory):
    return _compile(str(tmp_path_factory.mktemp("fast_dbg")), EMUL)


# Slips in what the checkpoints record or how they are read, each applied to a copy of the sources: the checks below
# must catch every one.  (old text, new text, occurrences)
MUTATIONS = {
    "count_read_off_by_one": [("f = ck[tid * bms + j];", "f = ck[tid * bms + j] + 1u;", 1)],
    "count_written_off_by_one": [("FP_STS16(c.s_ck + ((rel >> 5) << 1), acc);", "FP_STS16(c.s_ck + ((rel >> 5) << 1), acc + 1u);", 1),
                                 ("= (uint16_t)G;", "= (uint16_t)(G + 1u);", 1)],
    "every_mark_overwrites_the_count": [("if (old == 0u && c.s_ck != NONE)", "if (c.s_ck != NONE)", 1),
                                        ("if (bw == 0u && ck)", "if (ck)", 1)],
}


@pytest.fixture(scope="module", params=sorted(MUTATIONS))
def mutant_lib(request, tmp_path_factory):
    d = str(tmp_path_factory.mktemp("fast_mut"))
    csrc = os.path.join(d, "archive_b200", "csrc")
    emul = os.path.join(d, "tests", "host_emul")
    shutil.copytree(CSRC, csrc, ignore=shutil.ignore_patterns("*.o"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(d, "include"))
    os.makedirs(emul)
    for f in ("inflate_emul.cpp", "cuda_emu.h"):
        shutil.copy(os.path.join(EMUL, f), emul)
    path = os.path.join(csrc, "inflate_fast.cuh")
    s = open(path).read()
    for old, new, n in MUTATIONS[request.param]:
        assert s.count(old) == n, old
        s = s.replace(old, new)
    open(path, "w").write(s)
    return _compile(d, emul)


def counts(lib):
    o = (C.c_ulong * 4)()
    lib.emu_fast_dbg_counts(o)
    return dict(zip(("restarts", "exact", "walk", "full"), o))


def run(lib, monkeypatch, units, caps, must_finish):
    monkeypatch.setattr(tfe, "_E", lib)
    counts(lib)
    tfe.check_against_oracle(units, caps, must_finish=must_finish)
    return counts(lib)


def bench_text(seed, n):
    """n units of 64 KiB of the benchmark's text"""
    from archive_b200 import synth
    t = synth.text(n * 65536, stream=seed)
    return [t[i * 65536:(i + 1) * 65536].tobytes() for i in range(n)]


def text_units(seed, n, mem=9):
    return [tfe.deflate(p, 6, mem) + bytes(8) for p in bench_text(seed, n)]


def test_met_exactly_at_a_checkpoint_and_between_two(dbg_lib, monkeypatch):
    """Units of the benchmark's shape: lanes are met both exactly at a checkpoint and a few symbols after one, and every
    block has room for the checkpoints."""
    units = text_units(11, 4)
    got = run(dbg_lib, monkeypatch, units, [65536] * len(units), must_finish=len(units))
    assert got["exact"] > 0 and got["walk"] > 0, got
    assert got["full"] == 0, got


def test_many_small_blocks_with_restarts(dbg_lib, monkeypatch):
    """Many blocks per unit (memLevel 1): small blocks make lanes restart in pass A (a false parse runs into the
    end-of-block code), and the restarted lanes' counts are the ones their new parse recorded."""
    units = text_units(12, 3, mem=1)
    got = run(dbg_lib, monkeypatch, units, [65536] * len(units), must_finish=len(units))
    assert got["restarts"] > 0 and got["exact"] + got["walk"] > 0, got


def late_block_without_room(seed):
    """48 KiB of text, a full flush, then 16 KiB of skewed bytes that compress by less than 1.5: the last blocks start
    with three quarters of the window written, and their many lanes need all of the rest for the bitmaps"""
    rng = random.Random(seed)
    text = bench_text(seed, 1)[0][:49152]
    noise = bytes(min(255, int(abs(rng.gauss(0, 20)))) for _ in range(16384))
    co = zlib.compressobj(6, zlib.DEFLATED, -15)
    return co.compress(text) + co.flush(zlib.Z_FULL_FLUSH) + co.compress(noise) + co.flush() + bytes(8)


def test_late_block_without_room_counts_from_the_guessed_offset(dbg_lib, monkeypatch):
    """A block whose room in the window cannot hold the checkpoints counts its false starts from the guessed offset;
    the text blocks before it in the same unit use the checkpoints."""
    units = [late_block_without_room(s) for s in (21, 22)]
    assert all(len(u) <= 30720 - 16 for u in units)
    got = run(dbg_lib, monkeypatch, units, [65536] * len(units), must_finish=len(units))
    assert got["full"] > 0, got
    assert got["exact"] + got["walk"] > 0, got


def test_binary_and_fixed_code_units(dbg_lib, monkeypatch):
    """Codes of other shapes (fixed Huffman, a few-symbol alphabet, skewed binary) through the same counts, with lanes
    that restart in pass A."""
    rng = random.Random(13)
    units, caps = [], []
    for strat, p in zip((zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE), bench_text(14, 3)):
        p = p[:50000]
        units.append(tfe.deflate(p, 6, 9, strat) + bytes(8))
        caps.append(len(p))
    p = bytes(rng.choice(b"abc") for _ in range(60000))
    units.append(tfe.deflate(p) + bytes(8))
    caps.append(len(p))
    p = bytes(min(255, int(abs(rng.gauss(0, 40)))) for _ in range(60000))
    units.append(tfe.deflate(p, 9) + bytes(8))
    caps.append(len(p))
    fits = sum(1 for u in units if 192 <= len(u) <= 30720 - 16)
    got = run(dbg_lib, monkeypatch, units, caps, must_finish=fits)
    assert got["restarts"] > 0 and got["exact"] + got["walk"] > 0, got


def test_checkpoint_slips_are_caught(mutant_lib, monkeypatch):
    units = text_units(11, 2)
    with pytest.raises(AssertionError):
        run(mutant_lib, monkeypatch, units, [65536] * len(units), must_finish=len(units))
