"""K12 (DESIGN.md): one large DEFLATE stream decoded by many chunks, against the exact single-unit path, in the same process.

Workloads: one gzip member of synth.text at level 6 (sizes on both sides of the threshold), random data, and a file of many
unhinted 256 KiB members.  For each, the library as built (--thresh 0) or with the threshold forced to --thresh compressed
bytes, and the exact path (threshold out of reach) are timed alternately, host to host, best of --reps after a warm-up;
every output is checked against zlib.  The chunked run also reports K12's kernel times from CUDA events (block finder,
chunk decodes over all rounds, windows + emit) and its statistics.  Prints the card and its power limit, then one JSON
line per workload.

  python scripts/bench_inflate_stream.py [--sizes 1,4,16,64,256] [--reps 3]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import archive_b200 as a  # noqa: E402
from archive_b200 import _ffi, synth  # noqa: E402

MiB = 1 << 20
OFF = 1 << 62


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,4,16,64,256")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--thresh", type=int, default=0, help="K12 threshold in compressed bytes (0: the built-in one)")
    ap.add_argument("--random-mib", type=int, default=64)
    ap.add_argument("--members-mib", type=int, default=32)
    args = ap.parse_args()
    _ffi.ensure_init()
    L = _ffi.lib()
    print("card:", card(), flush=True)

    def stats():
        s = (C.c_ulonglong * 6)()
        L.b200z_debug_inflate_chunked_stats(s)
        return dict(zip(("regions", "chunks", "redo", "merged", "fell_back", "ran"), list(s)))

    def kernel_ms():
        m = (C.c_double * 3)()
        L.b200z_debug_inflate_chunked_ms(m)
        return [round(v, 2) for v in m]

    def bench(name, blob, plain, decode):
        res = {}
        for mode, th in (("chunked", args.thresh), ("exact", OFF)):
            L.b200z_debug_inflate_chunked_set(C.c_ulonglong(th), C.c_ulonglong(0))
            assert decode(blob) == plain, (name, mode)  # warm-up, checked
        best = {"chunked": 1e9, "exact": 1e9}
        st = km = None
        for _ in range(args.reps):
            for mode, th in (("chunked", args.thresh), ("exact", OFF)):
                L.b200z_debug_inflate_chunked_set(C.c_ulonglong(th), C.c_ulonglong(0))
                t0 = time.perf_counter()
                out = decode(blob)
                dt = time.perf_counter() - t0
                if mode == "chunked":
                    st = stats()
                    km = kernel_ms()
                assert out == plain
                best[mode] = min(best[mode], dt)
        L.b200z_debug_inflate_chunked_set(C.c_ulonglong(0), C.c_ulonglong(0))
        res = {"workload": name, "out_MiB": round(len(plain) / MiB, 2), "in_MiB": round(len(blob) / MiB, 2),
               "chunked_ms": round(best["chunked"] * 1e3, 2), "exact_ms": round(best["exact"] * 1e3, 2),
               "speedup": round(best["exact"] / best["chunked"], 2), "last_chunked_stats": st, "kernel_ms_find_decode_resolve": km}
        print(json.dumps(res), flush=True)

    gz = a.GZipDecoder()
    for s in [int(x) for x in args.sizes.split(",")]:
        plain = synth.text(s * MiB, stream=9).tobytes()
        c = zlib.compressobj(6, zlib.DEFLATED, 31)
        blob = c.compress(plain) + c.flush()
        bench(f"gzip_text_l6_{s}MiB", blob, plain, gz.decode_bytes)
    if args.random_mib:
        rnd = np.random.default_rng(1).integers(0, 256, args.random_mib * MiB, dtype=np.uint8).tobytes()
        c = zlib.compressobj(6, zlib.DEFLATED, 31)
        bench(f"gzip_random_{args.random_mib}MiB", c.compress(rnd) + c.flush(), rnd, gz.decode_bytes)
    if args.members_mib:
        plain = synth.text(args.members_mib * MiB, stream=10).tobytes()
        blob = b"".join(zlib.compress(plain[i:i + 256 * 1024], 6, 31) for i in range(0, len(plain), 256 * 1024))
        bench(f"gzip_256KiB_members_{args.members_mib}MiB", blob, plain, gz.decode_bytes)


if __name__ == "__main__":
    main()
