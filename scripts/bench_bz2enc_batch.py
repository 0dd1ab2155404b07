"""Many BZip2 encodes: one b200z_bzip2_encode_batch call against a loop of b200z_bzip2_encode over the same streams, a ZIP
of those streams as bzip2 members through ZipEncoder(batch=True) against batch=False, and one 256 MiB stream through
b200z_bzip2_encode (the batch of one), optionally against another build of the library in the same run.  Host to host,
with every output compared; launches are the library's launch counter.  The card's name and power limit are read in the
same run.  One JSON line per measurement.

  python scripts/bench_bz2enc_batch.py [--streams 4096] [--size 65536] [--reps 3] [--other-lib PATH] [--alt 3]

--other-lib names another libb200z.so (for example one built from an earlier commit): the 256 MiB single stream is then
timed alternately in child processes of this library and of that one, --alt times each, and the outputs are compared."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def many(L, n, size, reps):
    from archive_b200 import _ffi, synth
    src = np.concatenate([synth.text(size, stream=1000 + i) for i in range(n)])
    off = np.arange(n, dtype=np.uint64) * size
    ln = np.full(n, size, dtype=np.uint64)
    cap = L.b200z_bzip2_bound(size)
    ocap = np.full(n, cap, dtype=np.uint64)
    ooff = np.arange(n, dtype=np.uint64) * cap
    out = np.empty(n * cap, dtype=np.uint8)
    olen, crc, rc = np.zeros(n, np.uint64), np.zeros(n, np.uint32), np.zeros(n, np.int32)
    p = lambda a: a.ctypes.data

    def batch():
        _ffi.check(L.b200z_bzip2_encode_batch(p(src), p(off), p(ln), n, p(out), p(ooff), p(ocap), p(olen), p(crc), p(rc)))
        assert not rc.any()

    one = np.empty(cap, dtype=np.uint8)
    zl = C.c_size_t(0)
    singles = [None] * n

    def loop(k=n):
        for i in range(k):
            assert L.b200z_bzip2_encode(src.ctypes.data + i * size, size, one.ctypes.data, cap, C.byref(zl)) == 0
            singles[i] = one[:zl.value].tobytes()

    res = {}
    for name, fn, warm in (("batch", batch, batch), ("loop", loop, lambda: loop(64))):
        warm()
        ts, launches = [], 0
        for _ in range(reps if name == "batch" else 1):
            l0 = L.b200z_launch_count()
            t0 = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t0)
            launches = L.b200z_launch_count() - l0
        res[name] = {"best_s": round(min(ts), 4), "times_s": [round(t, 4) for t in ts], "launches": launches}
    st = (C.c_ulonglong * 5)()
    batch()
    L.b200z_debug_bzip2_encode_batch_stats(st)
    same = all(out[int(ooff[i]):int(ooff[i] + olen[i])].tobytes() == singles[i] for i in range(n))
    import zlib
    crc_ok = all(int(crc[i]) == zlib.crc32(src[i * size:(i + 1) * size].tobytes()) for i in range(0, n, max(1, n // 64)))
    return {"workload": f"{n} x {size} B synth.text", "in_MiB": n * size / 2**20, "out_MiB": round(float(olen.sum()) / 2**20, 2),
            **res, "speedup": round(res["loop"]["best_s"] / res["batch"]["best_s"], 2), "stats": list(st),
            "identical_to_single_calls": same, "crc32_ok": crc_ok}, src


def zip_workload(src, n, size, reps):
    from archive_b200.zip import Archive, ArchiveFile, ZipEncoder
    arc = Archive()
    for i in range(n):
        f = ArchiveFile(f"m/{i:05d}.txt", size)
        f.content, f.compression, f.last_mod_time, f.mode = src[i * size:(i + 1) * size].tobytes(), "bzip2", 1715953062, 0o100644
        arc.add(f)
    res, blobs = {}, {}
    for name, enc in (("batch", ZipEncoder(batch=True)), ("one_by_one", ZipEncoder())):
        ts = []
        for _ in range(reps if name == "batch" else 1):
            t0 = time.perf_counter()
            blobs[name] = enc.encode_bytes(arc, level=6)
            ts.append(time.perf_counter() - t0)
        res[name] = {"best_s": round(min(ts), 3), "times_s": [round(t, 3) for t in ts]}
    return {"workload": f"ZipEncoder, {n} bzip2 members of {size} B", **res,
            "speedup": round(res["one_by_one"]["best_s"] / res["batch"]["best_s"], 2),
            "archives_equal": blobs["batch"] == blobs["one_by_one"], "archive_MiB": round(len(blobs["batch"]) / 2**20, 2)}


CHILD = r"""
import ctypes as C, hashlib, json, os, sys, time
sys.path.insert(0, sys.argv[1])
from archive_b200 import _ffi, synth
L = _ffi.ensure_init()
m = 256 << 20
src = synth.text(m, stream=500)
h_in = L.b200z_host_alloc(m); C.memmove(h_in, src.ctypes.data, m)
cap = L.b200z_bzip2_bound(m); h_out = L.b200z_host_alloc(cap); ol = C.c_size_t(0)
ts = []
for i in range(4):
    t0 = time.perf_counter(); rc = L.b200z_bzip2_encode(h_in, m, h_out, cap, C.byref(ol)); ts.append(time.perf_counter() - t0)
    assert rc == 0, _ffi.last_error()
print(json.dumps({"times_s": ts[1:], "out": ol.value, "sha": hashlib.sha256(C.string_at(h_out, ol.value)).hexdigest()}))
"""


def single_256(other, alt):
    libs = {"this": os.path.join(ROOT, "archive_b200", "libb200z.so")}
    if other:
        libs["other"] = os.path.abspath(other)
    runs = {k: [] for k in libs}
    outs = {}
    for _ in range(alt):
        for k, lib in libs.items():
            env = dict(os.environ, B200Z_LIB=lib)
            r = subprocess.run([sys.executable, "-c", CHILD, ROOT], capture_output=True, text=True, env=env, check=True)
            d = json.loads(r.stdout.strip().splitlines()[-1])
            runs[k] += d["times_s"]
            outs[k] = (d["out"], d["sha"])
    res = {"workload": "one 256 MiB synth.text stream, b200z_bzip2_encode (pinned buffers)", "alternations": alt}
    for k, ts in runs.items():
        res[k] = {"best_s": round(min(ts), 4), "median_s": round(float(np.median(ts)), 4),
                  "spread_s": round(max(ts) - min(ts), 4), "times_s": [round(t, 4) for t in ts]}
    if other:
        res["identical_output"] = outs["this"] == outs["other"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--size", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--other-lib", default=None)
    ap.add_argument("--alt", type=int, default=3)
    a = ap.parse_args()
    from archive_b200 import _ffi
    L = _ffi.ensure_init()
    L.b200z_debug_bzip2_encode_batch_stats.argtypes = [C.c_void_p]
    print(json.dumps({"card": card()}), flush=True)
    r, src = many(L, a.streams, a.size, a.reps)
    print(json.dumps(r), flush=True)
    print(json.dumps(zip_workload(src, a.streams, a.size, max(1, a.reps - 1))), flush=True)
    print(json.dumps(single_256(a.other_lib, a.alt)), flush=True)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
