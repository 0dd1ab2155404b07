"""The streams of tests/test_inflate_fast_lz77_emul.py (k_inflate_fast's LZ77 pass) on the GPU: through
b200z_inflate_batch_device with k_inflate_fast and with the exact pair alone, which must agree, against the oracle,
with every unit at both window alignments."""
import random

import pytest

import oracle_lib as orc
from test_inflate_device_gpu import Backend, Batch, both_kernels, check_guards, check_vs_oracle, run
from test_inflate_fast_lz77_emul import cases, falls_back, long_runs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def B():
    return Backend()


def test_lz77_copy_turns_against_oracle(B, monkeypatch):
    rng = random.Random(79)
    units = cases() + long_runs(rng)[:1]
    fb = len(units) // 2
    units.insert(fb, falls_back(rng))
    raws = [r for r, _ in units]
    for shift in (0, 5):  # every other output slot moves by `shift` bytes: the windows' offsets modulo 16 change
        caps = [len(p) + shift * (i % 2) for i, (_, p) in enumerate(units)]
        caps[fb] = 65536
        b = Batch(raws, caps, rng=rng)
        r = both_kernels(monkeypatch, lambda: run(B, b))
        check_guards(r)
        check_vs_oracle(raws, caps, r)
        for i, (raw, plain) in enumerate(units):
            if i != fb:
                ost, oout, oused = orc.inflate(raw)
                assert ost == orc.OK and oout == plain, i
                assert r.unit(i) == (0, plain, oused), i
