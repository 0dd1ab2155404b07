"""Tarballs through the device codecs, host to host on one GPU.  Every output is checked against its input and the oracle
before anything is timed; each line names the GPU and its power limit.

  python scripts/bench_tar.py [--shards 1024] [--mib 4] [--tree-mib 256] [--codecs gzip,bzip2,xz] [--reps 3]

Decode: `shards` tar archives of about `mib` MiB each, their members synth.text samples of 4-64 KiB, compressed as
.tar.gz (level 6), .tar.bz2 and .tar.xz.  Path A is one gzip_decode_batch / bzip2_decode_batch / xz_decode_batch call,
then TarDecoder per shard; path B is a loop of GZipDecoder / BZip2Decoder / XZDecoder + TarDecoder per shard.  The batch
call, the loop of single calls and the tar walk are timed apart.
Encode: TarFileEncoder.tar_directory(compression=GZIP) on a generated tree of about `tree_mib` MiB, with the tar write
(the STORE pass) and the device gzip stage (GZipEncoder file to file) timed apart as well as together."""
import argparse
import bz2
import json
import lzma
import os
import random
import shutil
import subprocess
import sys
import tempfile
import time
import zlib
from concurrent.futures import ProcessPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    return [x.strip() for x in q.split(",")]


def best_of(reps, fn):
    best = None
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        best = min(best or 1e9, time.perf_counter() - t0)
    return best


def make_shard(args):
    """One tar of about `size` bytes: members of 4-64 KiB cut from synth.text, written by TarEncoder."""
    k, size = args
    from archive_b200 import ArchiveFile, TarEncoder, synth
    text = synth.text(size + (64 << 10), stream=100 + k).tobytes()
    rng = random.Random(k)
    files, pos = [], 0
    while pos < size:
        n = rng.randint(4 << 10, 64 << 10)
        f = ArchiveFile("shard%04d/doc%05d.txt" % (k, len(files)), n)
        f.content, f.last_mod_time = text[pos:pos + n], 1_700_000_000
        files.append(f)
        pos += n
    return TarEncoder().encode_bytes(files)


def compress(args):
    codec, data = args
    if codec == "gzip":
        c = zlib.compressobj(6, zlib.DEFLATED, 31)
        return c.compress(data) + c.flush()
    if codec == "bzip2":
        return bz2.compress(data, 9)
    return lzma.compress(data, format=lzma.FORMAT_XZ, check=lzma.CHECK_CRC64, preset=1)


def check_walk(archives, tars):
    import oracle_tar as ot
    for arch, t in zip(archives, tars):
        st, ms = ot.decode(t)
        assert st == ot.OK and [(f.name, f.content) for f in arch] == [(m.name, m.content) for m in ot.archive_order(ms)]


def bench_decode(a, args, gpu, pl, pool):
    tars = list(pool.map(make_shard, [(k, args.mib << 20) for k in range(args.shards)]))
    total = sum(len(t) for t in tars)
    dec = {"gzip": (a.gzip_decode_batch, a.GZipDecoder), "bzip2": (a.bzip2_decode_batch, a.BZip2Decoder),
           "xz": (a.xz_decode_batch, a.XZDecoder)}
    for codec in args.codecs.split(","):
        shards = list(pool.map(compress, [(codec, t) for t in tars], chunksize=4))
        batch_fn, single = dec[codec]
        out = batch_fn(shards)
        assert [rc for rc, _ in out] == [0] * len(shards) and [t for _, t in out] == tars, codec
        loop = [single().decode_bytes(z) for z in shards]
        assert loop == tars, codec
        walked = [a.TarDecoder().decode_bytes(t) for _, t in out]
        check_walk(walked, tars)
        del out, loop, walked
        tb = best_of(args.reps, lambda: batch_fn(shards))
        tl = best_of(1, lambda: [single().decode_bytes(z) for z in shards])
        tw = best_of(args.reps, lambda: [a.TarDecoder().decode_bytes(t) for t in tars])
        print(json.dumps({"workload": f"tar_{codec}_decode", "shards": len(shards), "tar_bytes": total,
                          "compressed_bytes": sum(len(z) for z in shards), "batch_s": round(tb, 4), "loop_s": round(tl, 3),
                          "tar_walk_s": round(tw, 4), "path_a_s": round(tb + tw, 4), "path_b_s": round(tl + tw, 3),
                          "batch_GBps": round(total / tb / 1e9, 2), "gpu": gpu, "power_limit": pl}), flush=True)


def bench_encode(a, args, gpu, pl, work):
    import gzip

    import oracle_lib as orc
    import oracle_tar as ot
    from archive_b200 import synth
    root = os.path.join(work, "tree")
    text = synth.text((args.tree_mib << 20) + (64 << 10), stream=7).tobytes()
    rng = random.Random(5)
    pos, k = 0, 0
    while pos < args.tree_mib << 20:
        n = rng.randint(4 << 10, 64 << 10)
        p = os.path.join(root, "d%02d" % (k % 37), "e%d" % (k % 5), "f%06d.txt" % k)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as fh:
            fh.write(text[pos:pos + n])
        pos, k = pos + n, k + 1
    tar_path, tgz_path = os.path.join(work, "store.tar"), os.path.join(work, "gz.tar.gz")

    def store():
        a.TarFileEncoder().tar_directory(root, filename=tar_path)

    def gz_stage():
        inp, out = a.InputFileStream(tar_path), a.OutputFileStream(tgz_path)
        a.GZipEncoder().encode_stream(inp, out, level=6)
        inp.close_sync()
        out.close_sync()

    def whole():
        a.TarFileEncoder().tar_directory(root, compression=a.TarFileEncoder.GZIP, filename=tgz_path)

    store()
    gz_stage()
    tar = open(tar_path, "rb").read()
    st, ms = ot.decode(tar)
    assert st == ot.OK and sum(1 for m in ms if m.type_flag != "5") == k
    assert all(m.content == open(os.path.join(os.path.dirname(root), m.name), "rb").read() for m in ms if m.type_flag != "5")
    tgz = open(tgz_path, "rb").read()
    assert gzip.decompress(tgz) == tar
    # the oracle's Deflate restatement takes one stream of up to 32 MiB (it crashes on 64 MiB); above that the device
    # gzip is checked on its first 32 MiB of tar, compressed alone, and by the round trip above
    head = tar[:32 << 20]
    gz_head = a.GZipEncoder().encode_bytes(head, level=6, mtime=0)
    assert gz_head == orc.gzip_encode(head, 6, mtime=0)[1]
    if len(tar) <= 32 << 20:
        assert tgz == orc.gzip_encode(tar, 6, mtime=int.from_bytes(tgz[4:8], "little"))[1]
    whole()
    assert [m.name for m in ot.decode(gzip.decompress(open(tgz_path, "rb").read()))[1]] == [m.name for m in ms]
    ts = best_of(args.reps, store)
    tg = best_of(args.reps, gz_stage)
    tt = best_of(args.reps, whole)
    print(json.dumps({"workload": "tar_directory_gzip", "files": k, "tar_bytes": len(tar), "tgz_bytes": len(tgz),
                      "tar_write_s": round(ts, 3), "gzip_stage_s": round(tg, 3), "tar_directory_s": round(tt, 3),
                      "gzip_stage_GBps": round(len(tar) / tg / 1e9, 2), "gpu": gpu, "power_limit": pl}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shards", type=int, default=1024)
    ap.add_argument("--mib", type=int, default=4)
    ap.add_argument("--tree-mib", type=int, default=256)
    ap.add_argument("--codecs", default="gzip,bzip2,xz")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import archive_b200 as a
    a._ffi.ensure_init()
    gpu, pl = gpu_info()
    work = tempfile.mkdtemp(prefix="bench_tar")
    try:
        with ProcessPoolExecutor(max(1, min(32, os.cpu_count() or 1))) as pool:
            if args.shards:
                bench_decode(a, args, gpu, pl, pool)
        if args.tree_mib:
            bench_encode(a, args, gpu, pl, work)
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
