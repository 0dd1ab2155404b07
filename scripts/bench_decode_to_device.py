"""Decode batches into host memory against the same batches into device memory (b200z_*_decode_batch_to_device).

  python scripts/bench_decode_to_device.py [--reps 5] [--out DIR]

Workloads are those of bench_gzip_batch.py, bench_bz2_batch.py and bench_xz_batch.py: 4096 x 64 KiB synth.text as
unhinted gzip members (level 6) and as zlib streams (verify), 4096 x 64 KiB and 64 x 8 MiB as BZh9 streams, 2048 x 64 KiB
as XZ (preset 1).  Per workload, best of --reps after a warm-up:
  host_s         the host batch into page-locked host slots (b200z_host_alloc);
  host_upload_s  the same, then the slots copied to a CUDA tensor (what a torch user had to do before);
  device_s       the *_to_device batch into a CUDA tensor on torch's current stream (returns with the bytes in place).
Every output of the device call is compared with the host batch's (rc, out_len, bytes) before anything is timed.  The
k_copy_slots time comes from a separate torch.profiler run of one device call (CUDA kernel records), so that tracing
does not slow the timed calls.  Slots start at 16-byte boundaries in both, as archive_b200's device=... calls lay them
out.  Each line names the GPU and its power limit, read in the same run."""
import argparse
import ctypes as C
import json
import lzma
import os
import subprocess
import sys
import time
import zlib
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, pl = [x.strip() for x in q.split(",")]
    return name, pl


def _xz1(data):
    return lzma.compress(data, preset=1)


def best_of(reps, fn):
    fn()  # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return min(ts), ts


class Workload:
    def __init__(self, L, codec, streams, caps, verify):
        import torch
        self.L, self.codec, self.n, self.verify = L, codec, len(streams), verify
        data = b"".join(streams)
        self.h_in = L.b200z_host_alloc(len(data))
        C.memmove(self.h_in, data, len(data))
        lens = np.array([len(s) for s in streams], np.uint64)
        self.in_off = np.zeros(self.n, np.uint64)
        self.in_off[1:] = np.cumsum(lens)[:-1]
        self.in_len = lens
        self.cap = np.array(caps, np.uint64)
        rooms = (self.cap + 15) & ~np.uint64(15)
        self.out_off = np.zeros(self.n, np.uint64)
        self.out_off[1:] = np.cumsum(rooms)[:-1]
        self.extent = int(rooms.sum())
        self.h_out = L.b200z_host_alloc(self.extent)
        self.h_view = np.ctypeslib.as_array((C.c_uint8 * self.extent).from_address(self.h_out))
        self.d_out = torch.empty(self.extent, dtype=torch.uint8, device="cuda")
        self.d_up = torch.empty(self.extent, dtype=torch.uint8, device="cuda")
        self.h_tensor = torch.from_numpy(self.h_view)
        self.out_len = np.zeros(self.n, np.uint64)
        self.rc = np.zeros(self.n, np.int32)
        self.torch = torch

    def _args(self, out_addr):
        p = lambda a: a.ctypes.data
        head = [self.h_in, p(self.in_off), p(self.in_len), self.n, self.verify] + ([0] if self.codec == "zlib" else [])
        return head + [out_addr, p(self.out_off), p(self.cap), p(self.out_len), p(self.rc)]

    def host(self):
        r = getattr(self.L, f"b200z_{self.codec}_decode_batch")(*self._args(self.h_out))
        assert r == 0, self.L.b200z_last_error()

    def host_upload(self):
        self.host()
        self.d_up.copy_(self.h_tensor, non_blocking=True)
        self.torch.cuda.current_stream().synchronize()

    def device(self):
        s = self.torch.cuda.current_stream().cuda_stream or 1  # (cudaStreamLegacy for the legacy default stream)
        r = getattr(self.L, f"b200z_{self.codec}_decode_batch_to_device")(*self._args(self.d_out.data_ptr()), s)
        assert r == 0, self.L.b200z_last_error()

    def check(self):
        """the device call gives what the host batch gives: rc, out_len and every slot's bytes"""
        self.host()
        h_rc, h_len = self.rc.copy(), self.out_len.copy()
        assert (h_rc == 0).all(), np.unique(h_rc)
        self.d_out.fill_(0)
        self.device()
        assert (self.rc == h_rc).all() and (self.out_len == h_len).all()
        got = self.d_out.cpu().numpy()
        for i in range(self.n):
            o, k = int(self.out_off[i]), int(self.out_len[i])
            assert np.array_equal(got[o:o + k], self.h_view[o:o + k]), (self.codec, i)
        return int(h_len.sum())

    def copy_kernel_ms(self):
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            self.device()
            self.torch.cuda.synchronize()
        us = [e.device_time_total for e in prof.key_averages() if "k_copy_slots" in e.key]
        return sum(us) / 1000.0, sum(e.count for e in prof.key_averages() if "k_copy_slots" in e.key)

    def free(self):
        self.L.b200z_host_free(self.h_in)
        self.L.b200z_host_free(self.h_out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/bench_decode_to_device.jsonl")
    a = ap.parse_args()
    import torch
    from archive_b200 import _ffi, synth
    L = _ffi.ensure_init()
    name, pl = gpu_info()
    unit = 64 << 10
    text = synth.text(4096 * unit, stream=3).tobytes()
    plain = [text[i * unit:(i + 1) * unit] for i in range(4096)]

    def bz2_streams(parts):
        data, offs, lens = b"".join(parts), [], []
        pos = 0
        for p in parts:
            offs.append(pos)
            lens.append(len(p))
            pos += len(p)
        caps = [L.b200z_bzip2_bound(n) for n in lens]
        out_off = np.zeros(len(parts), np.uint64)
        out_off[1:] = np.cumsum(caps)[:-1]
        out = np.empty(int(sum(caps)), np.uint8)
        ol, rc = np.zeros(len(parts), np.uint64), np.zeros(len(parts), np.int32)
        src = np.frombuffer(data, np.uint8)
        i_off, i_len, cc = np.array(offs, np.uint64), np.array(lens, np.uint64), np.array(caps, np.uint64)
        p = lambda x: x.ctypes.data
        assert L.b200z_bzip2_encode_batch(p(src), p(i_off), p(i_len), len(parts), p(out), p(out_off), p(cc), p(ol), None,
                                          p(rc)) == 0
        return [out[int(out_off[i]):int(out_off[i] + ol[i])].tobytes() for i in range(len(parts))]

    def workloads():  # (codec, label, streams, output room of each, verify)
        room = [unit + 1024] * 4096
        yield "gzip", "4096 x 64 KiB synth.text, unhinted gzip level 6", [synth.gzip_member(p, 6, hint=False) for p in plain], room, 0
        yield "zlib", "4096 x 64 KiB synth.text, zlib level 6, verify", [zlib.compress(p, 6) for p in plain], room, 1
        yield "bzip2", "4096 x 64 KiB synth.text, BZh9 (one block each)", bz2_streams(plain), room, 0
        big = synth.text(64 * (8 << 20), stream=9000).tobytes()
        yield "bzip2", "64 x 8 MiB synth.text, BZh9 (10 blocks each)", bz2_streams(
            [big[i * (8 << 20):(i + 1) * (8 << 20)] for i in range(64)]), [(8 << 20) + 1024] * 64, 0
        with ProcessPoolExecutor() as ex:
            xs = list(ex.map(_xz1, plain[:2048], chunksize=64))
        yield "xz", "2048 x 64 KiB synth.text, XZ preset 1, verify", xs, [L.b200z_xz_bound(x, len(x)) for x in xs], 1

    lines = []
    for codec, label, streams, caps, verify in workloads():
        w = Workload(L, codec, streams, caps, verify)
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
        k_ms, k_n = w.copy_kernel_ms()
        line = {"workload": label, "codec": codec, "streams": w.n, "out_bytes": out_bytes, "host_s": round(th, 4),
                "host_upload_s": round(tu, 4), "device_s": round(td, 4), "device_all_s": [round(t, 4) for t in tds],
                "host_over_device": round(th / td, 2), "host_upload_over_device": round(tu / td, 2),
                "k_copy_slots_ms": round(k_ms, 3), "k_copy_slots_launches": k_n,
                "k_copy_slots_GBps": round(out_bytes / (k_ms * 1e-3) / 1e9, 1) if k_ms else None,
                "gpu": name, "power_limit": pl}
        print(json.dumps(line), flush=True)
        lines.append(line)
        w.free()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_decode_to_device.jsonl"), "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
