"""Many gzip / zlib streams in one call against a loop of single calls, host to host on one GPU.  Every output is checked
before anything is timed; each line names the GPU and its power limit.

  python scripts/bench_gzip_batch.py [--n 4096] [--kib 64] [--enc-n 4096] [--reps 3]

Decode: n unhinted single-member gzip streams (what `gzip` and Python's gzip write: no size hint) of kib KiB of
synth.text at level 6, by one b200z_gzip_decode_batch call and by a loop of b200z_gzip_decode; then the same data as zlib
streams with verify on, by b200z_zlib_decode_batch and a loop of b200z_zlib_decode.  Encode: enc-n inputs of kib KiB at
levels 6 and 1, as gzip and as zlib, by one batch call and by a loop of single calls."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True).stdout.strip().splitlines()[0]
        name, pl = [x.strip() for x in q.split(",")]
        return name, pl
    except Exception:
        return "unknown", "unknown"


def packed(items):
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
    best = None
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--kib", type=int, default=64)
    ap.add_argument("--enc-n", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from archive_b200 import _ffi, synth
    L = _ffi.ensure_init()
    name, pl = gpu_info()
    unit = args.kib << 10
    text = synth.text(max(args.n, args.enc_n) * unit, stream=3).tobytes()
    plain = [text[i * unit:(i + 1) * unit] for i in range(args.n)]

    # ---- decode: unhinted gzip, then zlib with verify
    for kind in ("gzip", "zlib"):
        if kind == "gzip":
            streams = [synth.gzip_member(p, 6, hint=False) for p in plain]
        else:
            streams = [zlib.compress(p, 6) for p in plain]
        buf, off, ln = packed(streams)
        caps = [4 * len(s) + 1024 for s in streams]
        out, oo, cap = slots(caps)
        ol, rc = (C.c_uint64 * args.n)(), (C.c_int32 * args.n)()
        base = C.addressof(buf)

        def run_batch():
            if kind == "gzip":
                r = L.b200z_gzip_decode_batch(base, off, ln, args.n, 0, C.addressof(out), oo, cap, ol, rc)
            else:
                r = L.b200z_zlib_decode_batch(base, off, ln, args.n, 1, 0, C.addressof(out), oo, cap, ol, rc)
            assert r == 0, L.b200z_last_error()

        n1 = C.c_size_t(0)

        def run_loop():
            for i in range(args.n):
                if kind == "gzip":
                    r = L.b200z_gzip_decode(base + off[i], ln[i], 0, C.addressof(out) + oo[i], cap[i], C.byref(n1))
                else:
                    r = L.b200z_zlib_decode(base + off[i], ln[i], 1, 0, C.addressof(out) + oo[i], cap[i], C.byref(n1))
                assert r == 0 and n1.value == unit, (i, r, L.b200z_last_error())

        def check():
            for i in range(args.n):
                assert C.string_at(C.addressof(out) + oo[i], unit) == plain[i], i

        run_batch()
        assert all(rc[i] == 0 and ol[i] == unit for i in range(args.n))
        check()
        C.memset(C.addressof(out), 0, sum(caps))
        run_loop()
        check()
        l0 = L.b200z_launch_count()
        run_batch()
        launches = L.b200z_launch_count() - l0
        tb = best_of(args.reps, run_batch)
        tl = best_of(1, run_loop)
        print(json.dumps({"workload": f"{kind}_decode", "streams": args.n, "kib": args.kib, "verify": kind == "zlib",
                          "batch_s": round(tb, 4), "loop_s": round(tl, 3), "batch_launches": launches,
                          "speedup": round(tl / tb, 1), "gpu": name, "power_limit": pl}), flush=True)

    # ---- encode
    contents = [text[i * unit:(i + 1) * unit] for i in range(args.enc_n)]
    buf, off, ln = packed(contents)
    base = C.addressof(buf)
    caps = [L.b200z_deflate_bound(unit) + 18] * args.enc_n
    for kind in ("gzip", "zlib"):
        for level in (6, 1):
            out, oo, cap = slots(caps)
            ol, rc = (C.c_uint64 * args.enc_n)(), (C.c_int32 * args.enc_n)()

            def run_batch():
                if kind == "gzip":
                    r = L.b200z_gzip_encode_batch(base, off, ln, args.enc_n, level, 0, C.addressof(out), oo, cap, ol, rc)
                else:
                    r = L.b200z_zlib_encode_batch(base, off, ln, args.enc_n, level, 15, 0, C.addressof(out), oo, cap, ol, rc)
                assert r == 0, L.b200z_last_error()

            lout, loo, _ = slots(caps)
            lol = [0] * args.enc_n
            n1 = C.c_size_t(0)

            def run_loop():
                for i in range(args.enc_n):
                    if kind == "gzip":
                        r = L.b200z_gzip_encode(base + off[i], unit, level, 0, C.addressof(lout) + loo[i], caps[i], C.byref(n1))
                    else:
                        r = L.b200z_zlib_encode(base + off[i], unit, level, 15, 0, C.addressof(lout) + loo[i], caps[i], C.byref(n1))
                    assert r == 0
                    lol[i] = n1.value

            run_batch()
            run_loop()
            for i in range(args.enc_n):
                assert rc[i] == 0 and ol[i] == lol[i], i
                z = C.string_at(C.addressof(out) + oo[i], ol[i])
                assert z == C.string_at(C.addressof(lout) + loo[i], lol[i]), i
                if i % 64 == 0:
                    assert zlib.decompress(z, 31 if kind == "gzip" else 15) == contents[i], i
            tb = best_of(args.reps, run_batch)
            tl = best_of(1, run_loop)
            print(json.dumps({"workload": f"{kind}_encode", "inputs": args.enc_n, "kib": args.kib, "level": level,
                              "batch_s": round(tb, 4), "loop_s": round(tl, 3), "speedup": round(tl / tb, 1), "gpu": name,
                              "power_limit": pl}), flush=True)


if __name__ == "__main__":
    main()
