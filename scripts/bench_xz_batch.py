"""Many XZ streams in one call against a loop of single calls, host to host on one GPU.  Every output is checked before
anything is timed; each line names the GPU and its power limit.

  python scripts/bench_xz_batch.py [--n 2048] [--kib 64] [--enc-n 4096] [--reps 3]

Decode: n single-block streams made by Python's lzma at preset 1 (CRC-64 checks, the xz default) from synth.text, decoded
with verify on by one b200z_xz_decode_batch call and by a loop of b200z_xz_decode.  Encode: enc-n inputs of kib KiB by one
b200z_xz_encode_batch call and by a loop of b200z_xz_encode, with sha256 and with crc64 checks."""
import argparse
import ctypes as C
import json
import lzma
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True).stdout.strip().splitlines()[0]
        name, pl = [x.strip() for x in q.split(",")]
        return name, pl
    except Exception:
        return "unknown", "unknown"


def _xz1(data):
    return lzma.compress(data, preset=1)


def packed(items):
    """-> (ctypes buffer, in_off, in_len) with the items back to back"""
    n = len(items)
    off, ln = (C.c_uint64 * n)(), (C.c_uint64 * n)()
    pos = 0
    for i, b in enumerate(items):
        off[i], ln[i] = pos, len(b)
        pos += len(b)
    buf = (C.c_uint8 * max(pos, 1)).from_buffer_copy(b"".join(items) or b"\0")
    return buf, off, ln


def slots(caps):
    n = len(caps)
    off, cap = (C.c_uint64 * n)(), (C.c_uint64 * n)(*caps)
    tot = 0
    for i, c in enumerate(caps):
        off[i] = tot
        tot += c
    return (C.c_uint8 * max(tot, 1))(), off, cap


def best_of(reps, fn):
    best = 1e9
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        best = min(best, time.perf_counter() - t0)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2048, help="decode: streams")
    ap.add_argument("--kib", type=int, default=64, help="bytes of every stream's content, KiB")
    ap.add_argument("--enc-n", type=int, default=4096, help="encode: inputs")
    ap.add_argument("--reps", type=int, default=3, help="batch calls timed (best of); a loop of single calls runs once")
    a = ap.parse_args()
    import xz_build as xb
    from archive_b200 import _ffi, synth
    L = _ffi.ensure_init()
    L.b200z_debug_xz.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_uint32)]
    name, pl = gpu_info()
    sz = a.kib << 10
    text = synth.text(max(a.n, a.enc_n) * sz, stream=2).tobytes()

    # ---- decode ----
    parts = [text[i * sz:(i + 1) * sz] for i in range(a.n)]
    with ProcessPoolExecutor() as ex:
        streams = list(ex.map(_xz1, parts, chunksize=64))
    in_buf, in_off, in_len = packed(streams)
    base = C.addressof(in_buf)
    caps = [L.b200z_xz_bound(base + in_off[i], in_len[i]) for i in range(a.n)]
    out, out_off, cap = slots(caps)
    out_len, rc = (C.c_uint64 * a.n)(), (C.c_int32 * a.n)()

    def dec_batch():
        assert L.b200z_xz_decode_batch(base, in_off, in_len, a.n, 1, C.addressof(out), out_off, cap, out_len, rc) == 0

    l0 = L.b200z_launch_count()
    dec_batch()
    launches = L.b200z_launch_count() - l0
    for i in range(a.n):
        assert rc[i] == 0 and C.string_at(C.addressof(out) + out_off[i], out_len[i]) == parts[i], f"decode batch: stream {i}"
    ms, runs = C.c_double(), C.c_uint32()
    L.b200z_debug_xz(C.byref(ms), C.byref(runs))
    t_batch = best_of(a.reps, dec_batch)
    L.b200z_debug_xz(C.byref(ms), C.byref(runs))
    one = C.c_size_t(0)

    def dec_loop():
        for i in range(a.n):
            r = L.b200z_xz_decode(base + in_off[i], in_len[i], 1, C.addressof(out) + out_off[i], caps[i], C.byref(one))
            assert r == 0 and one.value == len(parts[i])

    C.memset(C.addressof(out), 0, len(out))
    l0 = L.b200z_launch_count()
    t_loop = best_of(1, dec_loop)
    loop_launches = L.b200z_launch_count() - l0
    for i in range(a.n):
        assert C.string_at(C.addressof(out) + out_off[i], len(parts[i])) == parts[i], f"decode loop: stream {i}"
    print(json.dumps({"workload": f"xz decode {a.n} single-block streams of {a.kib} KiB (lzma preset 1, crc64, verify)",
                      "gpu": name, "power_limit": pl, "compressed_bytes": len(in_buf), "runs": runs.value,
                      "batch_s": round(t_batch, 4), "batch_k_xz_lzma_ms": round(ms.value, 2), "batch_launches": launches,
                      "loop_of_single_calls_s": round(t_loop, 3), "loop_launches": loop_launches,
                      "speedup": round(t_loop / t_batch, 1), "GBps_output_batch": round(a.n * sz / t_batch / 1e9, 3),
                      "outputs_checked": a.n}), flush=True)

    # ---- encode ----
    ins = [text[i * sz:(i + 1) * sz] for i in range(a.enc_n)]
    in_buf, in_off, in_len = packed(ins)
    base = C.addressof(in_buf)
    caps = [L.b200z_xz_encode_bound(sz)] * a.enc_n
    out, out_off, cap = slots(caps)
    out_len, rc = (C.c_uint64 * a.enc_n)(), (C.c_int32 * a.enc_n)()
    for check, cname in ((3, "sha256"), (2, "crc64")):
        def enc_batch():
            assert L.b200z_xz_encode_batch(base, in_off, in_len, a.enc_n, check, C.addressof(out), out_off, cap, out_len,
                                           rc) == 0

        l0 = L.b200z_launch_count()
        enc_batch()
        launches = L.b200z_launch_count() - l0
        got = [C.string_at(C.addressof(out) + out_off[i], out_len[i]) for i in range(a.enc_n)]
        for i in range(a.enc_n):
            assert rc[i] == 0 and got[i] == xb.encode(ins[i], check), f"encode batch {cname}: input {i}"
        t_batch = best_of(a.reps, enc_batch)

        def enc_loop():
            for i in range(a.enc_n):
                r = L.b200z_xz_encode(base + in_off[i], in_len[i], check, C.addressof(out) + out_off[i], caps[i], C.byref(one))
                assert r == 0

        C.memset(C.addressof(out), 0, len(out))
        l0 = L.b200z_launch_count()
        t_loop = best_of(1, enc_loop)
        loop_launches = L.b200z_launch_count() - l0
        for i in range(a.enc_n):
            assert C.string_at(C.addressof(out) + out_off[i], len(got[i])) == got[i], f"encode loop {cname}: input {i}"
        print(json.dumps({"workload": f"xz encode {a.enc_n} inputs of {a.kib} KiB, {cname}", "gpu": name, "power_limit": pl,
                          "batch_s": round(t_batch, 4), "batch_launches": launches, "loop_of_single_calls_s": round(t_loop, 3),
                          "loop_launches": loop_launches, "speedup": round(t_loop / t_batch, 1),
                          "GBps_input_batch": round(a.enc_n * sz / t_batch / 1e9, 3), "outputs_checked": a.enc_n}),
              flush=True)


if __name__ == "__main__":
    main()
