"""Many BZip2 streams: one b200z_bzip2_decode_batch call against a loop of b200z_bzip2_decode over the same streams, and a
ZIP of many bzip2 members through ZipDecoder().decode_bytes.  Host to host, best of --reps after a checked warm-up; every
output is compared with its source.  The card's name, power limit and SM clock are read in the same run, and the K7 / K8
kernel times of one batch call come from torch.profiler in a separate, untimed call.  One JSON line per measurement.

  python scripts/bench_bz2_batch.py [--reps 5] [--zip-only]

--zip-only times just the ZIP workload: with PYTHONPATH pointing at another checkout it measures that checkout's library
on the same archive, for a comparison in the same GPU session."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
import zlib

import numpy as np

sys.path.insert(0, os.getcwd())
from archive_b200 import _ffi, synth  # noqa: E402

K7 = ("k_bz2_entropy",)  # k_bz2_entropy, k_bz2_entropy_fast, k_bz2_entropy_literal
K8 = ("k_bz2_expand", "k_bz2_chunk", "k_bz2_build_tt", "k_bz2_walk", "k_bz2_periodic", "k_bz2_rle", "k_bz2_offsets", "k_bz2_rand")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def streams(L, n, size, stream0):
    """n synth.text streams of `size` bytes, each compressed to one BZh9 stream by the device encoder"""
    srcs, zs = [], []
    cap = L.b200z_bzip2_bound(size)
    zbuf = np.empty(cap, dtype=np.uint8)
    zl = C.c_size_t(0)
    for i in range(n):
        t = synth.text(size, stream=stream0 + i)
        assert L.b200z_bzip2_encode(t.ctypes.data, size, zbuf.ctypes.data, cap, C.byref(zl)) == 0, _ffi.last_error()
        srcs.append(t.tobytes())
        zs.append(zbuf[:zl.value].tobytes())
    return srcs, zs


def best_of(fn, reps):
    fn()  # warm-up (its outputs are checked by the caller)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return min(ts), ts


def batch_workload(L, name, srcs, zs, reps):
    n = len(zs)
    data = b"".join(zs)
    h_in = L.b200z_host_alloc(len(data))
    C.memmove(h_in, data, len(data))
    in_off = np.zeros(n, dtype=np.uint64)
    in_off[1:] = np.cumsum([len(z) for z in zs])[:-1]
    in_len = np.array([len(z) for z in zs], dtype=np.uint64)
    rooms = np.array([len(s) + 1024 for s in srcs], dtype=np.uint64)
    out_off = np.zeros(n, dtype=np.uint64)
    out_off[1:] = np.cumsum(rooms)[:-1]
    total_out = int(rooms.sum())
    h_out = L.b200z_host_alloc(total_out)
    out_len = np.zeros(n, dtype=np.uint64)
    rc = np.zeros(n, dtype=np.int32)
    p = lambda a: a.ctypes.data

    def one_batch():
        r = L.b200z_bzip2_decode_batch(h_in, p(in_off), p(in_len), n, 1, h_out, p(out_off), p(rooms), p(out_len), p(rc))
        assert r == 0, _ffi.last_error()

    ol = C.c_size_t(0)

    def loop():
        for i in range(n):
            r = L.b200z_bzip2_decode(h_in + int(in_off[i]), int(in_len[i]), 1, h_out + int(out_off[i]), int(rooms[i]), C.byref(ol))
            assert r == 0, _ffi.last_error()

    def check():
        ok = True
        for i in range(n):
            ok = ok and zlib.crc32(C.string_at(h_out + int(out_off[i]), len(srcs[i]))) == zlib.crc32(srcs[i])
        return ok

    one_batch()
    ok_batch = bool((rc == 0).all()) and [int(v) for v in out_len] == [len(x) for x in srcs] and check()
    st = (C.c_ulonglong * 3)()
    L.b200z_debug_bz2_batch_stats(st)
    c0 = L.b200z_launch_count()
    t_batch, ts_b = best_of(one_batch, reps)
    launches_batch = (L.b200z_launch_count() - c0) // (reps + 1)
    ok_batch = ok_batch and check()
    C.memset(h_out, 0, total_out)
    loop()
    ok_loop = check()
    c0 = L.b200z_launch_count()
    t_loop, ts_l = best_of(loop, reps)
    launches_loop = (L.b200z_launch_count() - c0) // (reps + 1)
    ok_loop = ok_loop and check()
    # kernel times of one batch call (a separate call under the profiler: tracing slows the host)
    k7 = k8 = None
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            one_batch()
            torch.cuda.synchronize()
        k7 = k8 = 0.0
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            if any(k in e.key for k in K7):
                k7 += us / 1e3
            elif any(k in e.key for k in K8):
                k8 += us / 1e3
    except Exception as ex:  # noqa: BLE001 (the timings above stand without the kernel split)
        print(json.dumps({"profiler": "not measured", "why": repr(ex)[:200]}))
    out_bytes = sum(len(s) for s in srcs)
    res = {"workload": name, "streams": n, "in_bytes": len(data), "out_bytes": out_bytes,
           "batch_ms": round(t_batch * 1e3, 2), "loop_ms": round(t_loop * 1e3, 2), "speedup": round(t_loop / t_batch, 2),
           "batch_GBps": round(out_bytes / t_batch / 1e9, 3), "loop_GBps": round(out_bytes / t_loop / 1e9, 3),
           "batch_runs_ms": [round(t * 1e3, 2) for t in ts_b], "loop_runs_ms": [round(t * 1e3, 2) for t in ts_l],
           "launches_per_call": {"batch": launches_batch, "loop": launches_loop},
           "batch_stats": {"streams": st[0], "device_groups": st[1], "blocks": st[2]},
           "k7_ms": None if k7 is None else round(k7, 2), "k8_ms": None if k8 is None else round(k8, 2),
           "outputs_equal_sources": {"batch": ok_batch, "loop": ok_loop}}
    L.b200z_host_free(h_in)
    L.b200z_host_free(h_out)
    return res


def zip_workload(L, srcs, zs, reps):
    import struct
    import archive_b200 as a
    out, cd = bytearray(), bytearray()
    for i, (s, z) in enumerate(zip(srcs, zs)):
        nb = b"m%05d.txt" % i
        crc = zlib.crc32(s)
        off = len(out)
        out += struct.pack("<IHHHHHIIIHH", 0x04034b50, 46, 0, 12, 0, 0x21, crc, len(z), len(s), len(nb), 0) + nb + z
        cd += struct.pack("<IHHHHHHIIIHHHHHII", 0x02014b50, 0x031e, 46, 0, 12, 0, 0x21, crc, len(z), len(s), len(nb), 0, 0, 0, 0,
                          0o100644 << 16, off) + nb
    cd_off = len(out)
    out += cd
    out += struct.pack("<IHHHHIIH", 0x06054b50, 0, 0, len(zs), len(zs), len(cd), cd_off, 0)
    data = bytes(out)
    arc = a.ZipDecoder().decode_bytes(data)
    ok = len(arc) == len(srcs) and all(f.content == srcs[i] for i, f in enumerate(arc))
    t, ts = best_of(lambda: a.ZipDecoder().decode_bytes(data), reps)
    out_bytes = sum(len(s) for s in srcs)
    return {"workload": f"ZipDecoder().decode_bytes: {len(zs)} bzip2 members of 64 KiB", "lib": _ffi.LIB_PATH,
            "zip_bytes": len(data), "out_bytes": out_bytes, "best_ms": round(t * 1e3, 2), "GBps": round(out_bytes / t / 1e9, 3),
            "runs_ms": [round(x * 1e3, 2) for x in ts], "outputs_equal_sources": ok}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--zip-only", action="store_true")
    args = ap.parse_args()
    L = _ffi.ensure_init()
    print(json.dumps({"card": card()}))
    srcs, zs = streams(L, 4096, 64 << 10, 1000)
    if not args.zip_only:
        L.b200z_debug_bz2_batch_stats.argtypes = [C.c_void_p]
        print(json.dumps(batch_workload(L, "4096 x 64 KiB synth.text, BZh9 (one block each)", srcs, zs, args.reps)))
    print(json.dumps(zip_workload(L, srcs, zs, args.reps)))
    if not args.zip_only:
        big_s, big_z = streams(L, 64, 8 << 20, 9000)
        print(json.dumps(batch_workload(L, "64 x 8 MiB synth.text, BZh9 (10 blocks each)", big_s, big_z, args.reps)))
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
