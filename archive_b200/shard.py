"""Multi-GPU partitioning of independent compressed units (SURVEY.md section 8e): contiguous unit ranges per rank,
balanced by compressed bytes, each rank decoding straight into its slice of the final output so that ONE in-place
all-gather (equal slices) or all-gather-v (ragged) reassembles the byte stream in order.  Host logic only."""
from __future__ import annotations

import numpy as np


def split_units(in_len, world: int):
    """-> list of (lo, hi) unit ranges, one per rank, contiguous, balanced by compressed bytes."""
    in_len = np.asarray(in_len, dtype=np.int64)
    n = len(in_len)
    if world <= 1 or n == 0:
        return [(0, n)] + [(n, n)] * (world - 1)
    csum = np.concatenate([[0], np.cumsum(in_len)])
    total = int(csum[-1])
    cuts = [0]
    for r in range(1, world):
        target = total * r // world
        k = int(np.searchsorted(csum, target, side="left"))
        k = min(max(k, cuts[-1]), n)
        cuts.append(k)
    cuts.append(n)
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


def out_slices(out_len, ranges):
    """Byte ranges of each rank's decoded output inside the final stream, given per-unit output sizes."""
    out_len = np.asarray(out_len, dtype=np.int64)
    csum = np.concatenate([[0], np.cumsum(out_len)])
    return [(int(csum[lo]), int(csum[hi])) for lo, hi in ranges]


# ---------------------------------------------------------------------------------------------
# BZip2: blocks sharded over ranks (SURVEY.md 8e, config 4)
# ---------------------------------------------------------------------------------------------
BZ2_EOS, BZ2_RANDOMISED, BZ2_CORRUPT_CYCLE, BZ2_OVERRUN = 1, 2, 4, 8


_BZ2_MAGIC_BLOCK, _BZ2_MAGIC_EOS = bytes.fromhex("314159265359"), bytes.fromhex("177245385090")


def _bz2_short_magic(data, in_len: int, pos: int) -> str:
    """_readBlockType with fewer than 48 bits left (bzip2_decoder.dart:90-111): the six bytes are read one at a time and the
    first one that fits neither magic returns -1 (decodeStream false) BEFORE the missing bytes are asked for (RangeError)."""
    total = in_len * 8
    blk = eos = True
    for i in range(6):
        p = pos + 8 * i
        if p + 8 > total:
            return "throw"
        hi, lo = data[p >> 3], (data[(p >> 3) + 1] if (p >> 3) + 1 < in_len else 0)
        b = (((hi << 8) | lo) >> (8 - (p & 7))) & 0xFF
        blk = blk and b == _BZ2_MAGIC_BLOCK[i]
        eos = eos and b == _BZ2_MAGIC_EOS[i]
        if not blk and not eos:
            return "data"
    return "throw"


def bz2_walk_chain(reports, in_len: int, verify: bool, data=None):
    """Merge the block reports of all ranks and walk them exactly as BZip2Decoder.decodeStream does
    (bzip2_decoder.dart:46-87): the stream is the chain of blocks in which every block starts on the bit where the
    previous one ended, up to the first end-of-stream magic; CRCs are compared only when `verify`.
    reports: iterable of (start_bit, end_bit, out_bytes, crc_calc, crc_stored, status, flags, rank, local_off);
    data: the stream (anything indexable to ints), looked at only when it ends inside a block signature.
    -> (kind, chain, n_out): kind 'ok' | 'data' (decodeStream returns false) | 'throw' (RangeError); chain = the
    reports that make up the output, in order; n_out = bytes of output that are kept."""
    by_start = {}
    for r in reports:
        by_start.setdefault(r[0], r)  # every rank reports the EOS candidates: keep one
    total_bits = in_len * 8
    pos, chain, kind, eos = 32, [], "ok", None
    while True:
        if (pos + 7) // 8 >= in_len:
            break
        if pos + 48 > total_bits:
            kind = _bz2_short_magic(data, in_len, pos) if data is not None else "throw"
            break
        r = by_start.get(pos)
        if r is None:
            kind = "data"
            break
        if pos + 80 > total_bits:
            kind = "throw"
            break
        if r[6] & BZ2_EOS:
            eos = r
            break
        if r[5] == -2:
            kind = "throw"
            break
        if r[5] != 0 or (r[6] & BZ2_RANDOMISED):
            kind = "data"
            break
        chain.append(r)
        pos = r[1]
    n_out, combined, kept = 0, 0, []
    for r in chain:
        if r[6] & BZ2_CORRUPT_CYCLE:
            kind = "data"
            break
        kept.append(r)
        n_out += r[2]
        if r[6] & BZ2_OVERRUN:  # the bytes are written before the reference notices (bzip2_decoder.dart:628-631)
            kind, eos = "data", None
            break
        if verify and r[3] != r[4]:
            kind, eos = "data", None
            break
        combined = (((combined << 1) | (combined >> 31)) & 0xFFFFFFFF) ^ r[3]
    if kind == "ok" and eos is not None and verify and eos[4] != combined:
        kind = "data"
    return kind, kept, n_out


def bzip2_decode_sharded(data, verify: bool = False, group=None, rank=None, world=None, reports_in=None, out_buf=None):
    """Every rank passes the same BZip2 stream; rank r decodes its share of the blocks on its GPU
    (b200z_bzip2_decode_shard), the per-block reports are exchanged (a few dozen bytes per block -- the only collective on
    this path; the decoded bytes stay where they were produced), and every rank derives the same chain.
    -> dict(kind, total, pieces): pieces = [(stream_offset, bytes)] this rank holds of the output."""
    import ctypes as C

    import torch.distributed as dist

    from . import _ffi
    L = _ffi.ensure_init()
    use_dist = rank is None
    if use_dist:
        rank = dist.get_rank(group) if dist.is_initialized() else 0
        world = dist.get_world_size(group) if dist.is_initialized() else 1
    addr, n, keep = _ffi.as_buffer(data)
    cap_blocks = n // 4096 + 64
    blocks = (_ffi.Bz2Block * cap_blocks)()
    # out_buf = (address, capacity) of a caller-owned (ideally pinned: b200z_host_alloc) buffer that is reused across calls
    out_cap = out_buf[1] if out_buf else n * 8 // world + (2 << 20)
    while True:
        out = (C.c_uint8 * out_cap).from_address(out_buf[0]) if out_buf else (C.c_uint8 * out_cap)()
        out_len, nb = C.c_size_t(0), C.c_size_t(0)
        rc = L.b200z_bzip2_decode_shard(addr, n, rank, world, C.addressof(out), out_cap, C.byref(out_len), blocks,
                                        cap_blocks, C.byref(nb))
        if rc == _ffi.E_NOSPC and nb.value > cap_blocks:
            # more block reports than the array holds: highly compressible streams (a 900 kB block of one long run is
            # ~40 bytes) and chance matches of the magic both add candidates
            cap_blocks = nb.value + 64
            blocks = (_ffi.Bz2Block * cap_blocks)()
            continue
        if rc == _ffi.E_NOSPC and out_len.value > out_cap and not out_buf:
            out_cap = out_len.value + 64
            continue
        _ffi.check(rc)
        break
    mine, off = [], 0
    for i in range(nb.value):
        b = blocks[i]
        mine.append((b.start_bit, b.end_bit, b.out_bytes, b.crc_calc, b.crc_stored, b.status, b.flags, rank, off))
        off += b.out_bytes
    if not use_dist:  # the caller plays the other ranks itself (tests): it passes their reports in
        reports = mine + list(reports_in or [])
    elif world > 1:
        gathered = [None] * world
        dist.all_gather_object(gathered, mine, group=group)
        reports = [r for part in gathered for r in part]
    else:
        reports = mine
    kind, chain, n_out = bz2_walk_chain(reports, n, verify, data=(C.c_uint8 * n).from_address(addr) if n else b"")
    pieces, pos = [], 0
    view = memoryview(out)
    for r in chain:
        if r[7] == rank and r[2]:
            if pieces and pieces[-1][0] + len(pieces[-1][1]) == pos and pieces[-1][2] + len(pieces[-1][1]) == r[8]:
                o, v, lo = pieces[-1]
                pieces[-1] = (o, view[lo:lo + len(v) + r[2]], lo)
            else:
                pieces.append((pos, view[r[8]:r[8] + r[2]], r[8]))
        pos += r[2]
    return {"kind": kind, "total": n_out, "pieces": [(o, v) for o, v, _ in pieces], "n_chain": len(chain), "reports": mine}


# ---------------------------------------------------------------------------------------------
# ZIP members sharded over ranks (SURVEY.md 8e, config 5): largest-first bin packing by compressed size
# ---------------------------------------------------------------------------------------------
def pack_members(comp_sizes, world: int):
    """-> list (one per rank) of member indices; greedy largest-first onto the least loaded rank, ties to the lower rank,
    every rank's list in archive order.  Deterministic, so every rank computes the same assignment without talking."""
    order = sorted(range(len(comp_sizes)), key=lambda i: (-int(comp_sizes[i]), i))
    load = [0] * world
    bins = [[] for _ in range(world)]
    for i in order:
        r = min(range(world), key=lambda k: (load[k], k))
        bins[r].append(i)
        load[r] += int(comp_sizes[i]) + 1
    return [sorted(b) for b in bins]


def zip_extract_sharded(data, rank: int, world: int, web_eos: bool = False):
    """Rank `rank` of `world` decodes its share of the archive's members with one b200z_zip_extract call.
    -> (entries, {member index: bytes}) -- the directory is parsed by every rank (host work, no device)."""
    from .zip import ZipDecoder
    dec = ZipDecoder(web_eos=web_eos)
    ents, n = dec.list(data)
    mine = pack_members([ents[i].comp_size if ents[i].has_data else 0 for i in range(n)], world)[rank]
    if not mine:
        return ents, {}
    import ctypes as C
    from . import _ffi
    sub = (_ffi.ZipEntry * len(mine))(*[ents[i] for i in mine])
    contents = dec._extract(data, sub, len(mine))[0]
    return ents, {i: contents[k] for k, i in enumerate(mine)}


# ---------------------------------------------------------------------------------------------
# ZipEncoder members sharded over ranks (SURVEY.md 8f3): a member's payload depends on nothing but its own content
# (zip_encoder.dart:185-259), so every rank compresses a share and ONE exchange of the payloads lets any rank write the
# container -- byte for byte the archive a single rank produces.
# ---------------------------------------------------------------------------------------------
def zip_encode_sharded(archive, level: int = 1, modified=None, comment: str = "", group=None, rank=None, world=None,
                       compress=None, payloads_in=None):
    """ZipEncoder().encode_bytes(archive, ...) with the members' compression spread over the ranks of `group`.
    Members are packed largest-first by content size (pack_members); every rank compresses its share on its own GPU, the
    (payload, crc) pairs are exchanged with one all_gather_object, and every rank assembles the same container.
    Without torch.distributed (`rank` / `world` given explicitly) the call returns this rank's {member index: (payload,
    crc)} and accepts the other ranks' dictionaries as `payloads_in` -- the single-process form the tests drive.
    `compress(content, method, level) -> (payload, crc32)` defaults to the device path (zip._b200_compress)."""
    from .zip import ZipEncoder, _b200_compress
    compress = compress or _b200_compress
    entries = list(archive)
    dist = None
    if rank is None or world is None:
        import torch.distributed as dist
        rank, world = dist.get_rank(group), dist.get_world_size(group)
    sizes = [(e.size if e.is_file else 0) for e in entries]
    mine = pack_members(sizes, world)[rank]
    def level_of(e):  # the member's own level wins (ZipEncoder.level_of, zip_encoder.dart:137-183)
        own = getattr(e, "compress_level", None)
        return own if own is not None else (level if level is not None else 6)

    done = {}
    for i in mine:
        e = entries[i]
        if e.is_file:
            method = e.compression or "deflate"
            done[i] = compress(e.content or b"", method, level_of(e))
    if dist is not None:
        parts = [None] * world
        dist.all_gather_object(parts, done, group=group)
    elif payloads_in is not None:
        parts = [done] + list(payloads_in)
    else:
        return done
    table = {}
    for p in parts:
        table.update(p)
    order = iter(i for i, e in enumerate(entries) if e.is_file)

    def lookup(content, method, level_):  # ZipEncoder asks for the members in archive order
        return table[next(order)]

    return ZipEncoder(compress=lookup).encode_bytes(entries, level=level, modified=modified, comment=comment)
