"""Encrypted ZIP extraction, host to host through b200z_zip_extract_password (one JSON line per workload):
  a  256 x 4 MiB deflate members with full flushes every 64 KiB, AES-256
  b  100 000 x 1 KiB AES-256 members (bound by key derivation)
  c  one 1 GiB stored AES-256 member (bound by the serial MAC chain)
  d  256 x 4 MiB deflate members, ZipCrypto (one serial chain per member)
For each: best host-to-host time of --reps calls after a warm-up, the CUDA-event times of the PBKDF2 / CTR / MAC /
ZipCrypto kernels of the best call, the unencrypted b200z_zip_extract of the same members in the same run, and the oracle
on all host cores (one pass) as the CPU line.  The archives are built here: AES payloads through b200z_zip_aes_encrypt,
ZipCrypto through the oracle.  Usage: python scripts/bench_zip_crypt.py [--only abcd] [--scale 1.0] [--reps 3]"""
import argparse
import ctypes as C
import json
import os
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import oracle_lib as orc  # noqa: E402
import zip_crypt_build as zb  # noqa: E402
from archive_b200 import _ffi, synth  # noqa: E402
from archive_b200.zip import ZipDecoder, aes_encrypt_batch  # noqa: E402

PW = b"bench-password"


def flushed_deflate(body, every):
    c = zlib.compressobj(1, zlib.DEFLATED, -15)
    return b"".join(c.compress(body[i:i + every]) + c.flush(zlib.Z_FULL_FLUSH) for i in range(0, len(body), every)) + c.flush()


def archive(payloads, sizes, crcs, methods, crypt):
    """payloads already encrypted (or plain when crypt is None)"""
    import struct
    out, cd = bytearray(), bytearray()
    for i, (p, usize, crc, m) in enumerate(zip(payloads, sizes, crcs, methods)):
        name = b"m%06d" % i
        flags, method, extra = 0x800, m, b""
        if crypt:
            flags |= 1
        if crypt == "aes":
            extra = struct.pack("<HHH2sBH", 0x9901, 7, 1, b"AE", 3, m)
            method = 99
        pos = len(out)
        out += struct.pack("<IHHHHHIIIHH", 0x04034B50, 20, flags, method, 0, 0x21, crc, len(p), usize, len(name), len(extra))
        out += name + extra + p
        cd += struct.pack("<IHHHHHHIIIHHHHHII", 0x02014B50, 20, 20, flags, method, 0, 0x21, crc, len(p), usize, len(name),
                          len(extra), 0, 0, 0, 0o100644 << 16, pos) + name + extra
    cd_pos = len(out)
    n = len(payloads)
    out += cd
    if n > 0xFFFF:  # zip64 end records, as ZipEncoder writes them (zip_encoder.dart:470-484)
        eocd64 = len(out)
        out += struct.pack("<IQHHIIQQQQ", 0x06064B50, 0x2C, 0x2D, 0x2D, 0, 0, n, n, len(cd), cd_pos)
        out += struct.pack("<IIQI", 0x07064B50, 0, eocd64, 1)
        out += struct.pack("<IHHHHIIH", 0x06054B50, 0, 0xFFFF, 0xFFFF, 0xFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0)
    else:
        out += struct.pack("<IHHHHIIH", 0x06054B50, 0, 0, n, n, len(cd), cd_pos, 0)
    return bytes(out)


def build(kind, scale):
    txt = synth.text(4 << 20, stream=991).tobytes()
    if kind in "ad":
        n, size = max(1, int(256 * scale)), 4 << 20
        bodies = [txt[(i * 4099) % 65536:] + txt[:(i * 4099) % 65536] for i in range(n)]
        comp = [flushed_deflate(b, 65536) for b in bodies[:8]]
        comp = [comp[i % 8] for i in range(n)]
        bodies = [bodies[i % 8] for i in range(n)]
        methods = [8] * n
    elif kind == "b":
        n = max(1, int(100_000 * scale))
        bodies = [txt[(i * 997) % ((4 << 20) - 1024):][:1024] for i in range(n)]
        comp, methods = bodies, [0] * n
    else:
        size = int((1 << 30) * scale)
        bodies = [(txt * (size // len(txt) + 1))[:size]]
        comp, methods = bodies, [0]
    crcs = [zlib.crc32(b) & 0xFFFFFFFF for b in bodies]
    sizes = [len(b) for b in bodies]
    plain = archive(comp, sizes, crcs, methods, None)
    if kind == "d":
        enc = [zb.zipcrypto_encrypt(PW, bytes(12) + c) for c in comp[:8]]
        enc = [enc[i % 8] for i in range(len(comp))]
        return plain, archive(enc, sizes, crcs, methods, "zipcrypto"), bodies
    salts = [os.urandom(16) for _ in comp]
    sealed = aes_encrypt_batch(comp, salts, PW)
    enc = [s + v + ct + m for s, (ct, v, m) in zip(salts, sealed)]
    return plain, archive(enc, sizes, crcs, methods, "aes"), bodies


def listing(data):
    ents, n = ZipDecoder().list(data)  # b200z_zip_list (host only)
    return ents, [ents[i] for i in range(n)]


def extract(data, listed, password):
    L = _ffi.ensure_init()
    arr, ents = listed
    n = len(ents)
    room = [int(e.uncomp_size) + 64 for e in ents]
    off, tot = [], 0
    for r in room:
        off.append(tot)
        tot += (r + 63) & ~63
    out = L.b200z_host_alloc(tot)
    ol, st = (C.c_uint64 * n)(), (C.c_int32 * n)()
    addr, zl, keep = _ffi.as_buffer(data)
    o64, r64 = (C.c_uint64 * n)(*off), (C.c_uint64 * n)(*room)
    t0 = time.perf_counter()
    rc = L.b200z_zip_extract_password(addr, zl, arr, n, out, tot, o64, r64, ol, st, 0, password, len(password or b""))
    dt = time.perf_counter() - t0
    assert rc == 0, _ffi.last_error()
    ok = all(s in (0, 1) for s in st)
    first = C.string_at(out + off[0], int(ol[0]))
    L.b200z_host_free(out)
    return dt, ok, first


def kernel_ms():
    v = (C.c_double * 4)()
    _ffi.lib().b200z_debug_zip_crypt_ms(v)
    return dict(zip(("pbkdf2", "ctr", "mac", "zipcrypto"), [round(x, 3) for x in v]))


def oracle_all_cores(data, ents, password):
    def one(e):
        out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
        s = orc.L().orc_zip_member_password(data, C.c_size_t(len(data)), C.byref(e), 0, password, C.c_size_t(len(password)),
                                            C.byref(out), C.byref(n))
        orc.L().orc_free(out)
        return s
    t0 = time.perf_counter()
    with ThreadPoolExecutor(os.cpu_count()) as ex:
        sts = list(ex.map(one, ents))
    return time.perf_counter() - t0, all(s == 0 for s in sts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="abcd")
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import torch
    dev = torch.cuda.get_device_name(0)
    try:
        import subprocess
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                               text=True).stdout.strip().splitlines()[0]
    except Exception:
        power = "unknown"
    for kind in a.only:
        plain, enc, bodies = build(kind, a.scale)
        pents, eents = listing(plain), listing(enc)
        extract(enc, eents, PW)
        extract(plain, pents, None)
        best, best_k = None, None
        for _ in range(a.reps):
            dt, ok, first = extract(enc, eents, PW)
            assert ok and first == bodies[0], kind
            if best is None or dt < best:
                best, best_k = dt, kernel_ms()
        pbest = min(extract(plain, pents, None)[0] for _ in range(a.reps))
        cpu = oracle_all_cores(enc, eents[1], PW) if not a.no_cpu else (None, True)
        out_bytes = sum(len(b) for b in bodies)
        print(json.dumps({"workload": kind, "members": len(eents[1]), "archive_bytes": len(enc), "output_bytes": out_bytes,
                          "encrypted_s": round(best, 4), "encrypted_GBps": round(out_bytes / best / 1e9, 3),
                          "unencrypted_s": round(pbest, 4), "kernels_ms": best_k,
                          "oracle_all_cores_s": None if cpu[0] is None else round(cpu[0], 3), "oracle_ok": cpu[1],
                          "host_cores": os.cpu_count(),
                          "device": dev, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
