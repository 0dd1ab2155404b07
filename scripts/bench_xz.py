"""XZDecoder / XZEncoder on the device: host-to-host time, k_xz_lzma time (CUDA events), GB/s of output and the run
count, with the oracle (oracle/xz.c, a C restatement of the reference, one host core) beside it.  Every workload is checked
for parity before it is timed; each line names the GPU and its power limit.

  python scripts/bench_xz.py [--mib 256] [--reps 3] [--oracle]

Streams are made with Python's lzma at preset 1 (a block per process, all host cores), around the repository's own .xz
container writer (tests/xz_build.py)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _raw(chunk):
    import xz_build as xb
    return xb.raw_lzma2(chunk, preset=1)


def make_stream(data: bytes, block: int) -> bytes:
    import xz_build as xb
    parts = [data[o:o + block] for o in range(0, len(data), block)]
    with ProcessPoolExecutor() as ex:
        raws = list(ex.map(_raw, parts))
    return xb.container(list(zip(raws, parts)), check="crc64")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True).stdout.strip().splitlines()[0]
        name, pl = [x.strip() for x in q.split(",")]
        return name, pl
    except Exception:
        return "unknown", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--oracle", action="store_true", help="also time the oracle on one host core (every decode workload)")
    a = ap.parse_args()
    import numpy as np
    import archive_b200 as arc
    import xz_build as xb
    from archive_b200 import _ffi, synth
    L = _ffi.ensure_init()
    dbg = L.b200z_debug_xz
    dbg.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_uint32)]
    name, pl = gpu_info()
    n = a.mib << 20
    text = synth.text(n, stream=1).tobytes()
    rand = np.random.default_rng(1).integers(0, 256, n, dtype=np.uint8).tobytes()
    work = [(f"text {a.mib} MiB in 1 MiB blocks", text, 1 << 20), (f"text {a.mib} MiB in 24 MiB blocks", text, 24 << 20),
            ("text 64 MiB, one block", text[:64 << 20], 64 << 20), (f"random {a.mib} MiB in 24 MiB blocks", rand, 24 << 20)]
    for label, data, block in work:
        stream = make_stream(data, block)
        addr, sn, keep = _ffi.as_buffer(stream)
        cap = L.b200z_xz_bound(addr, sn)
        out = (C.c_uint8 * cap)()
        got = C.c_size_t(0)
        rc = L.b200z_xz_decode(addr, sn, 1, C.addressof(out), cap, C.byref(got))
        assert rc == 0 and got.value == len(data) and C.string_at(out, got.value) == data, f"{label}: parity"
        best, kms, runs = 1e9, C.c_double(), C.c_uint32()
        for _ in range(a.reps):
            t0 = time.perf_counter()
            L.b200z_xz_decode(addr, sn, 1, C.addressof(out), cap, C.byref(got))
            best = min(best, time.perf_counter() - t0)
            dbg(C.byref(kms), C.byref(runs))
        rec = {"workload": "xz decode " + label, "gpu": name, "power_limit": pl, "compressed_bytes": sn, "runs": runs.value,
               "host_to_host_s": round(best, 4), "k_xz_lzma_ms": round(kms.value, 2),
               "GBps_output_host_to_host": round(len(data) / best / 1e9, 3),
               "GBps_output_k_xz_lzma": round(len(data) / (kms.value / 1e3) / 1e9, 3) if kms.value else None}
        if a.oracle:
            t0 = time.perf_counter()
            st, o = xb.decode(stream, True)
            assert st == 0 and o == data
            rec["oracle_restatement_1core_s"] = round(time.perf_counter() - t0, 3)
        print(json.dumps(rec), flush=True)
    for check, cname in ((2, "crc64"), (3, "sha256")):
        data = text[:256 << 20]  # the encoder workload is 256 MiB at every --mib
        want_tail = xb.encode(data, check)
        enc = arc.XZEncoder().encode_bytes(data, check=check)
        assert enc == want_tail, f"encode {cname}: parity"
        best = 1e9
        for _ in range(a.reps):
            t0 = time.perf_counter()
            arc.XZEncoder().encode_bytes(data, check=check)
            best = min(best, time.perf_counter() - t0)
        print(json.dumps({"workload": f"xz encode {len(data) >> 20} MiB {cname}", "gpu": name, "power_limit": pl,
                          "host_to_host_s": round(best, 4), "GBps_input": round(len(data) / best / 1e9, 3)}), flush=True)


if __name__ == "__main__":
    main()
