"""Every member of a batch of tarballs as a CUDA tensor, three ways, on one GPU.  Every output is checked against the host
path before anything is timed; each line names the GPU and its power limit, read in the same run.

  python scripts/bench_tar_to_device.py [--shards 1024] [--mib 4] [--codecs gzip,bzip2,xz,none] [--reps 5] [--walk-gib 1]

The workload of scripts/bench_tar.py: `shards` tar archives of about `mib` MiB, members of 4-64 KiB, as .tar.gz (level
6), .tar.bz2, .tar.xz or plain .tar ("none").  Three ways to get every file's content on the device:
  device:     tar_decode_batch(device="cuda"): the codec's *_decode_batch_to_device (or one upload of the plain shards),
              one b200z_tar_walk_device call, each content a view into the decoded buffer;
  one_upload: the host batch, TarDecoder per shard on the host, then every content packed and uploaded in one copy;
  per_member: the host batch, TarDecoder per shard on the host, then one upload per member.
First, k_tar_walk alone (its device time between CUDA events the library records around the launch) on one plain tar of `walk_gib` GiB with
members of 1-4 KiB, walked where it lies on the device."""
import argparse
import json
import os
import random
import sys
import time
from concurrent.futures import ProcessPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_tar import compress, gpu_info, make_shard  # noqa: E402


def best_of(reps, fn):
    import torch
    best = None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best or 1e9, time.perf_counter() - t0)
    return best


def contents(results):
    """[(name, content)] of every shard's archive, in order."""
    return [[(f.name, f.content) for f in arch] for _, arch in results]


def way_device(a, shards, codec):
    return contents(a.tar_decode_batch(shards, compression=codec, device="cuda"))


def _host(a, shards, codec):
    return contents(a.tar_decode_batch(shards, compression=codec))


def way_one_upload(a, shards, codec):
    import torch
    host = _host(a, shards, codec)
    flat = [c for arch in host for _, c in arch if c is not None]
    buf = torch.frombuffer(bytearray(b"".join(flat)), dtype=torch.uint8).to("cuda")
    out, at = [], 0
    for arch in host:
        row = []
        for name, c in arch:
            if c is not None:
                row.append((name, buf[at:at + len(c)]))
                at += len(c)
            else:
                row.append((name, None))
        out.append(row)
    return out


def way_per_member(a, shards, codec):
    import torch
    return [[(name, None if c is None else torch.frombuffer(bytearray(c), dtype=torch.uint8).to("cuda") if c else
              torch.empty(0, dtype=torch.uint8, device="cuda")) for name, c in arch] for arch in _host(a, shards, codec)]


def same(got, want):
    """Names and contents equal, the device contents compared in one copy back per shard."""
    import torch
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert [n for n, _ in g] == [n for n, _ in w]
        gc = [c for _, c in g if c is not None]
        wc = [c for _, c in w if c is not None]
        assert [c.numel() for c in gc] == [len(c) for c in wc]
        if gc:
            assert torch.cat(gc).cpu().numpy().tobytes() == b"".join(wc)


def walk_tar(gib, seed=3):
    """One plain tar of about `gib` GiB: members of 1-4 KiB, each header written directly (ustar-free V7 fields)."""
    rng = random.Random(seed)
    pattern = bytes(rng.getrandbits(8) | 1 for _ in range(8192))  # no zero bytes: every header is found by its size only
    parts, total, k = [], 0, 0
    while total < gib << 30:
        n = rng.randint(1 << 10, 4 << 10)
        h = bytearray(512)
        h[0:12] = b"m%011d" % k
        h[100:108] = b"0000644\0"
        h[124:136] = b"%011o\0" % n
        h[156] = 0x30
        parts += [bytes(h), pattern[:n], bytes(-n % 512)]
        total += 512 + n + (-n % 512)
        k += 1
    parts.append(bytes(1024))
    return b"".join(parts), k


def bench_walk(a, gib, reps, gpu, pl):
    import ctypes as C

    import torch
    from archive_b200 import tar as T
    data, k = walk_tar(gib)
    d = torch.frombuffer(bytearray(data), dtype=torch.uint8).to("cuda")
    arch = a.tar_decode_batch([d], device="cuda")[0][1]  # checked against the host walk first
    want = a.TarDecoder().decode_bytes(data)
    assert len(arch) == len(want) == k
    assert torch.cat([f.content for f in arch]).cpu().numpy().tobytes() == b"".join(f.content for f in want)
    del arch, want
    from archive_b200.codecs import _Sink
    sink = _Sink("cuda")
    L = a._ffi.ensure_init()
    L.b200z_debug_tar_walk.argtypes = [C.POINTER(C.c_double)]
    calls = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        first, count, rc, recs, hdrs = T._walk_on_device(sink, [d])
        call_s = time.perf_counter() - t0
        assert count[0] == k and rc[0] == 0
        ms = C.c_double()
        L.b200z_debug_tar_walk(C.byref(ms))  # k_tar_walk of that call, between CUDA events on the library's stream
        calls.append((call_s, ms.value * 1e-3))
    call_s, walk_s = min(c for c, _ in calls), min(w for _, w in calls)
    print(json.dumps({"workload": "k_tar_walk", "tar_bytes": len(data), "members": k, "k_tar_walk_s": round(walk_s, 4),
                      "ns_per_member": round(walk_s / k * 1e9, 1), "tar_walk_device_call_s": round(call_s, 4), "gpu": gpu,
                      "power_limit": pl}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shards", type=int, default=1024)
    ap.add_argument("--mib", type=int, default=4)
    ap.add_argument("--codecs", default="gzip,bzip2,xz,none")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--walk-gib", type=int, default=1)
    args = ap.parse_args()
    import torch
    import archive_b200 as a
    a._ffi.ensure_init()
    torch.cuda.init()
    gpu, pl = gpu_info()
    if args.walk_gib:
        bench_walk(a, args.walk_gib, args.reps, gpu, pl)
    ways = {"device": way_device, "one_upload": way_one_upload, "per_member": way_per_member}
    if args.shards:
        with ProcessPoolExecutor(max(1, min(32, os.cpu_count() or 1))) as pool:
            tars = list(pool.map(make_shard, [(k, args.mib << 20) for k in range(args.shards)]))
            for name in args.codecs.split(","):
                codec = None if name == "none" else name
                shards = tars if codec is None else list(pool.map(compress, [(codec, t) for t in tars], chunksize=4))
                want = _host(a, shards, codec)
                assert sum(len(x) for x in want) > 0
                for way, fn in ways.items():  # every way checked against the host path before anything is timed
                    same(fn(a, shards, codec), want)
                del want
                row = {"workload": f"tar_{name}_to_device", "shards": len(shards), "tar_bytes": sum(len(t) for t in tars),
                       "members": sum(len(x) for x in contents(a.tar_decode_batch(tars))), "reps": args.reps}
                for way, fn in ways.items():
                    row[f"{way}_s"] = round(best_of(args.reps, lambda: fn(a, shards, codec)), 4)
                row.update({"gpu": gpu, "power_limit": pl})
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
