"""ZIP extraction into host memory against the same extraction into device memory (b200z_zip_extract_to_device).

  python scripts/bench_zip_to_device.py [--reps 5] [--scale 1.0] [--out DIR]

Workloads (--scale shrinks the member counts for a rehearsal):
  config 5       1024 x 4 MiB synth.text, deflate level 6, a full flush every 64 KiB (SURVEY.md 8d config 5);
  k12            8 x 64 MiB synth.text, deflate level 6 without flush points (each member goes through K12);
  bzip2          256 x 1 MiB synth.text, BZh9;
  aes256         64 x 4 MiB synth.text, deflate level 1, AES-256 (ZipEncoder(password:)), extracted with the password.
Per workload, best of --reps after a warm-up:
  host_s         b200z_zip_extract_password into page-locked host slots (b200z_host_alloc);
  host_upload_s  the same, then the slots copied to a CUDA tensor (what a torch user had to do before);
  device_s       b200z_zip_extract_to_device into a CUDA tensor on torch's current stream, with the member CRC-32s.
Every member of the device call is compared with the host call (status, out_len, bytes) and its CRC with the header's
before anything is timed.  The k_copy_slots and k_crc_tiles times come from a separate torch.profiler run of one device
call, so that tracing does not slow the timed calls.  Slots start at 16-byte boundaries, as ZipDecoder(device=...) lays
them out.  Each line names the GPU and its power limit, read in the same run."""
import argparse
import bz2
import ctypes as C
import json
import os
import struct
import subprocess
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, pl = [x.strip() for x in q.split(",")]
    return name, pl


def best_of(reps, fn):
    fn()  # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return min(ts), ts


def zip_archive(members):
    """[(name, payload, method, crc, size)] -> a ZIP archive (local headers with sizes, central directory, end record)"""
    out, cd = bytearray(), bytearray()
    for name, payload, method, crc, size in members:
        nb = name.encode()
        pos = len(out)
        out += struct.pack("<IHHHHHIIIHH", 0x04034B50, 20, 0x800, method, 0, 0x21, crc, len(payload), size, len(nb), 0)
        out += nb + payload
        cd += struct.pack("<IHHHHHHIIIHHHHHII", 0x02014B50, 20, 20, 0x800, method, 0, 0x21, crc, len(payload), size, len(nb),
                          0, 0, 0, 0, 0o100644 << 16, pos)
        cd += nb
    cd_pos = len(out)
    out += cd + struct.pack("<IHHHHIIH", 0x06054B50, 0, 0, len(members), len(members), len(cd), cd_pos, 0)
    return bytes(out)


class Workload:
    def __init__(self, L, data, password):
        import torch
        from archive_b200 import _ffi
        self.L, self.torch = L, torch
        self.pw = password
        self.h_in = L.b200z_host_alloc(len(data))
        self.zlen = len(data)
        C.memmove(self.h_in, data, len(data))
        cnt = C.c_size_t(0)
        assert L.b200z_zip_list(self.h_in, self.zlen, None, 0, C.byref(cnt)) == 0
        self.n = cnt.value
        self.ents = (_ffi.ZipEntry * self.n)()
        assert L.b200z_zip_list(self.h_in, self.zlen, self.ents, self.n, C.byref(cnt)) == 0
        self.room = np.array([e.uncomp_size for e in self.ents], np.uint64)
        rooms = (self.room + 15) & ~np.uint64(15)
        self.out_off = np.zeros(self.n, np.uint64)
        self.out_off[1:] = np.cumsum(rooms)[:-1]
        self.extent = int(rooms.sum())
        self.h_out = L.b200z_host_alloc(self.extent)
        self.h_view = np.ctypeslib.as_array((C.c_uint8 * self.extent).from_address(self.h_out))
        self.h_tensor = torch.from_numpy(self.h_view)
        self.d_out = torch.empty(self.extent, dtype=torch.uint8, device="cuda")
        self.d_up = torch.empty(self.extent, dtype=torch.uint8, device="cuda")
        self.out_len = np.zeros(self.n, np.uint64)
        self.st = np.zeros(self.n, np.int32)
        self.crc = np.zeros(self.n, np.uint32)

    def _args(self, out_addr):
        p = lambda a: a.ctypes.data
        return [self.h_in, self.zlen, self.ents, self.n, out_addr, self.extent, p(self.out_off), p(self.room), p(self.out_len),
                p(self.st)]

    def _pw(self):
        return (self.pw, len(self.pw)) if self.pw is not None else (None, 0)

    def host(self):
        r = self.L.b200z_zip_extract_password(*self._args(self.h_out), 0, *self._pw())
        assert r == 0, self.L.b200z_last_error()

    def host_upload(self):
        self.host()
        self.d_up.copy_(self.h_tensor, non_blocking=True)
        self.torch.cuda.current_stream().synchronize()

    def device(self):
        s = self.torch.cuda.current_stream().cuda_stream or 1  # (cudaStreamLegacy for the legacy default stream)
        r = self.L.b200z_zip_extract_to_device(*self._args(self.d_out.data_ptr()), self.crc.ctypes.data, 0, *self._pw(), s)
        assert r == 0, self.L.b200z_last_error()

    def check(self):
        """the device call gives what the host call gives (status, out_len, bytes), and every CRC is the header's"""
        self.host()
        h_st, h_len = self.st.copy(), self.out_len.copy()
        assert (h_st == 0).all(), np.unique(h_st)
        self.d_up.copy_(self.h_tensor)
        self.d_out.zero_()
        self.device()
        assert (self.st == h_st).all() and (self.out_len == h_len).all()
        for i in range(self.n):
            o, k = int(self.out_off[i]), int(self.out_len[i])
            assert self.torch.equal(self.d_out[o:o + k], self.d_up[o:o + k]), i
            assert self.crc[i] == self.ents[i].crc32 or (self.pw is not None and self.ents[i].crc32 == 0), i
        return int(h_len.sum())

    def kernel_ms(self):
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            self.device()
            self.torch.cuda.synchronize()
        ka = prof.key_averages()
        res = {}
        for k in ("k_copy_slots", "k_crc_tiles"):
            res[k] = (sum(e.device_time_total for e in ka if k in e.key) / 1000.0, sum(e.count for e in ka if k in e.key))
        return res

    def free(self):
        self.L.b200z_host_free(self.h_in)
        self.L.b200z_host_free(self.h_out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="member counts times this (a rehearsal at a small size)")
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/bench_zip_to_device.jsonl")
    a = ap.parse_args()
    import torch
    import archive_b200 as ab
    from archive_b200 import _ffi, synth
    L = _ffi.ensure_init()
    name, pl = gpu_info()
    cnt = lambda k: max(1, int(k * a.scale))
    pool = ThreadPoolExecutor(32)

    def deflated(n, size, stream, flush):
        txt = synth.text(n * size, stream=stream)

        def comp(i):
            b = txt[i * size:(i + 1) * size].tobytes()
            z = synth.deflate_raw_flushed(b, 65536) if flush else synth.deflate_raw(b)
            return (f"m{i:05d}.txt", z, 8, zlib.crc32(b), size)
        return zip_archive(list(pool.map(comp, range(n))))

    def bzipped(n, size, stream):
        txt = synth.text(n * size, stream=stream)

        def comp(i):
            b = txt[i * size:(i + 1) * size].tobytes()
            return (f"b{i:05d}.txt", bz2.compress(b, 9), 12, zlib.crc32(b), size)
        return zip_archive(list(pool.map(comp, range(n))))

    def aes(n, size, stream, pw):
        txt = synth.text(n * size, stream=stream)
        arc = []
        for i in range(n):
            f = ab.ArchiveFile(f"a{i:05d}.txt", size)
            f.content = txt[i * size:(i + 1) * size].tobytes()
            arc.append(f)
        return ab.ZipEncoder(batch=True, password=pw).encode_bytes(arc, level=1, modified=0)

    def workloads():  # (label, archive, password)
        yield f"config 5: {cnt(1024)} x 4 MiB synth.text, deflate 6, full flush every 64 KiB", deflated(cnt(1024), 4 << 20, 700, True), None
        yield f"k12: {cnt(8)} x 64 MiB synth.text, deflate 6, no flush points", deflated(cnt(8), 64 << 20, 710, False), None
        yield f"bzip2: {cnt(256)} x 1 MiB synth.text, BZh9", bzipped(cnt(256), 1 << 20, 720), None
        yield f"aes256: {cnt(64)} x 4 MiB synth.text, deflate 1, AES-256", aes(cnt(64), 4 << 20, 730, b"bench-pw"), b"bench-pw"

    lines = []
    for label, data, pw in workloads():
        w = Workload(L, data, pw)
        del data
        out_bytes = w.check()

        def fresh():  # every timed phase starts from released library buffers: no phase inherits another's reservations
            L.b200z_shutdown()
            assert L.b200z_init(_ffi._inited_device, 0) == 0
            torch.cuda.empty_cache()

        fresh()
        th, _ = best_of(a.reps, w.host)
        fresh()
        tu, _ = best_of(a.reps, w.host_upload)
        fresh()
        td, tds = best_of(a.reps, w.device)
        k = w.kernel_ms()
        line = {"workload": label, "members": w.n, "out_bytes": out_bytes, "host_s": round(th, 4), "host_upload_s": round(tu, 4),
                "device_s": round(td, 4), "device_all_s": [round(t, 4) for t in tds],
                "host_over_device": round(th / td, 2), "host_upload_over_device": round(tu / td, 2),
                "k_copy_slots_ms": round(k["k_copy_slots"][0], 3), "k_copy_slots_launches": k["k_copy_slots"][1],
                "k_copy_slots_share": round(k["k_copy_slots"][0] * 1e-3 / td, 4),
                "k_crc_tiles_ms": round(k["k_crc_tiles"][0], 3), "k_crc_tiles_launches": k["k_crc_tiles"][1],
                "k_crc_tiles_share": round(k["k_crc_tiles"][0] * 1e-3 / td, 4), "gpu": name, "power_limit": pl}
        print(json.dumps(line), flush=True)
        lines.append(line)
        w.free()
        del w
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_zip_to_device.jsonl"), "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
