"""K12 inside b200z_zip_extract (DESIGN.md "K12", "ZIP container"): large ZIP members decoded by many chunks, as one batch
of streams, against the exact path, in the same process.

Workloads (archives written by Python's zipfile at level 6, so no flush points):
  - one member of 256 MiB of synth.text;
  - 8 members of 64 MiB each;
  - 256 members of 4 MiB each (below the threshold: the path is unchanged);
  - and, for the single-stream case, bench_inflate_stream.py's 64 MiB gzip member through GZipDecoder.
For each, the library as built and with the K12 threshold out of reach are timed alternately, host to host
(ZipDecoder().decode_bytes), best of --reps after a warm-up; every output is checked against the input zipfile compressed.
The ZIP runs also time "every large member in one K12 batch" against "one member per batch" (the test hook that caps the
streams of a batch), and report the K12 batch's kernel times from CUDA events (block finder, chunk decodes over all
rounds, windows + emit) and its statistics.  Prints the card and its power limit, then one JSON line per workload.

  python scripts/bench_zip_large.py [--reps 3] [--only one256,eight64,many4,gzip64]
"""
import argparse
import ctypes as C
import io
import json
import os
import subprocess
import sys
import time
import zipfile
import zlib

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
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", default="one256,eight64,many4,gzip64")
    args = ap.parse_args()
    L = _ffi.ensure_init()
    print("card:", card(), flush=True)

    def zstats():
        s, m = (C.c_ulonglong * 5)(), (C.c_double * 3)()
        L.b200z_debug_zip_chunked_stats(s, m)
        return dict(zip(("offered", "accepted", "fell_back", "rounds", "batches"), list(s))), [round(v, 2) for v in m]

    def set_mode(mode):
        L.b200z_debug_inflate_chunked_set(C.c_ulonglong(OFF if mode == "exact" else 0), C.c_ulonglong(0))
        L.b200z_debug_zip_chunked_set(C.c_uint(1 if mode == "per_member" else 0), C.c_uint(0))

    def bench(name, blob, want, decode, modes):
        for mode in modes:  # warm-up, checked
            set_mode(mode)
            assert decode(blob) == want, (name, mode)
        best = {m: 1e9 for m in modes}
        info = {}
        for _ in range(args.reps):
            for mode in modes:
                set_mode(mode)
                t0 = time.perf_counter()
                out = decode(blob)
                dt = time.perf_counter() - t0
                if mode != "exact" and name != "gzip64":
                    info[mode] = zstats()
                assert out == want, (name, mode)
                best[mode] = min(best[mode], dt)
        set_mode("built")
        res = {"workload": name, "out_MiB": round(sum(len(w) for w in want) / MiB, 2), "in_MiB": round(len(blob) / MiB, 2)}
        for m in modes:
            res[f"{m}_ms"] = round(best[m] * 1e3, 2)
        res["speedup_vs_exact"] = round(best["exact"] / best["built"], 2)
        if "per_member" in best:
            res["batch_vs_per_member"] = round(best["per_member"] / best["built"], 2)
        for m, (st, km) in info.items():
            res[f"{m}_stats"] = st
            res[f"{m}_kernel_ms_find_decode_resolve"] = km
        print(json.dumps(res), flush=True)

    def zip_of(parts):
        buf = io.BytesIO()
        with zipfile.ZipFile(buf, "w", compression=zipfile.ZIP_DEFLATED, compresslevel=6) as z:
            for i, p in enumerate(parts):
                z.writestr(f"m{i}.txt", p)
        return buf.getvalue()

    def unzip(blob):
        return [f.content for f in a.ZipDecoder().decode_bytes(blob).files]

    only = set(args.only.split(","))
    for name, n, size in (("one256", 1, 256 * MiB), ("eight64", 8, 64 * MiB), ("many4", 256, 4 * MiB)):
        if name not in only:
            continue
        text = synth.text(n * size, stream=30).tobytes()
        parts = [text[i * size:(i + 1) * size] for i in range(n)]
        blob = zip_of(parts)
        bench(name, blob, parts, unzip, ("built", "exact") if n == 1 or size < 16 * MiB else ("built", "per_member", "exact"))
    if "gzip64" in only:  # single-stream K12 (bench_inflate_stream.py's 64 MiB workload)
        plain = synth.text(64 * MiB, stream=9).tobytes()
        c = zlib.compressobj(6, zlib.DEFLATED, 31)
        blob = c.compress(plain) + c.flush()
        bench("gzip64", blob, [plain], lambda b: [a.GZipDecoder().decode_bytes(b)], ("exact", "built"))
        m = (C.c_double * 3)()
        L.b200z_debug_inflate_chunked_ms(m)
        print(json.dumps({"workload": "gzip64", "last_kernel_ms_find_decode_resolve": [round(v, 2) for v in m]}), flush=True)


if __name__ == "__main__":
    main()
