// inflate_chunked.cuh -- K12: large raw DEFLATE streams, each decoded by many chunks at once (included by inflate_kernels.cu).
//
// A chunk starts at a block boundary guessed inside its slice of the compressed stream and decodes without the 32 KiB of
// output in front of it: its output is 16-bit SYMBOLS, a value < 256 being a byte and 0x8000 | w byte w (0..32767) of the
// window in front of the chunk (a match that copies from such a place copies the marker).  The host proves the chain of
// chunks from the stream's true start and redoes the chunks that started at a wrong guess (b200z_api.cu:
// run_chunked); then k_inflate_windows resolves the last 32 KiB of every chunk in chunk order, straight into the
// output buffer, and k_inflate_emit translates every page of symbols in parallel.  Every kernel works on a batch of
// streams (CkStream): a chunk, a job or a chain entry names its stream, and each stream has its own input, page range and
// "reached too far" flag.  DESIGN.md "K12".
//
// The per-block logic is the exact step's (inflate_decode.cuh: BitReader, parse_tables, build_table, slow_decode) with
// every end-of-input rule of the reference: a chunk reads the stream's input up to its end, not its slice's.
#pragma once
#include "inflate_chunked.h"

namespace b200z {

B200Z_HD void ck_reader(BitReader &br, const uint8_t *in, uint32_t in_len, unsigned long long bit) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(in);
  br.lead = (uint32_t)(a & 15);
  br.w = reinterpret_cast<const uint32_t *>(a - br.lead);
  br.in_len = in_len;
  br.nw = (uint32_t)(((uint64_t)br.lead + br.in_len + 3) >> 2);
  br.seek((uint32_t)(bit >> 3));
  br.drop((int)(bit & 7u));
}
B200Z_HD unsigned long long ck_bitpos(const BitReader &br) {
  return 32ull * br.widx - (unsigned long long)br.cnt - 8ull * br.lead;
}

// Does a block that the exact step would decode start at `bit`?  Stored: LEN == ~NLEN at the next byte boundary and LEN
// fits the input (the host takes the chunk from any start with the same stored header: b200z_api.cu).  Dynamic: a
// header the exact step accepts (no run past HLIT + HDIST, which is a throw), a code for end-of-block, complete codes
// (zlib's single distance code excepted), and a block that decodes to its end.  Only blocks that are not final are
// looked for.  Fixed blocks cannot be told from noise and are not looked for either.  A block this rejects costs a merge
// or a redo, never wrong bytes: every chunk is proven by the chain.
// (A loop, not recursion: the device stack of a recursive function cannot be sized at compile time.)
B200Z_HD bool ck_block_here(const uint8_t *in, uint32_t in_len, unsigned long long bit, uint8_t *lens, uint16_t *lut_l,
                            uint16_t *lut_d, SlowTab &sl, SlowTabD &sd) {
  BitReader br;
  uint32_t type = 0;
  for (int hop = 0;; ++hop) {  // hop 1: the header behind a stored candidate's payload (which may be final)
    ck_reader(br, in, in_len, bit);
    br.refill();
    if (br.rem_bits() < 8 || (hop == 0 && (br.peek(1) & 1u))) return false;  // only blocks that are not final are looked for
    type = br.peek(3) >> 1;
    br.drop(3);
    if (type != 0) break;
    br.drop((int)(br.rem_bits() & 7));
    const long long rem_bytes = br.rem_bits() >> 3;
    if (rem_bytes < 4) return false;
    br.refill();
    const uint32_t len = br.peek(16), nlen = (uint32_t)(br.buf >> 16) & 0xffffu;
    if ((len ^ 0xffffu) != nlen || (long long)len > rem_bytes - 4) return false;
    // LEN == ~NLEN turns up by chance about every 64 KiB of noise: the block behind the payload must begin with a stored
    // or dynamic header too (or the input ends there)
    if (hop > 0) return true;
    bit = 8ull * (br.in_len - (uint32_t)rem_bytes + 4u + len);
    if (bit + 8 >= 8ull * br.in_len) return true;
  }
  if (type != 2) return false;
  if (parse_tables(br, 2, lens, lut_l, lut_d, sl, sd) != 0 || lens[256] == 0) return false;
  // zlib writes complete codes, except a distance code with a single symbol; noise rarely spells one
  {
    uint32_t kl = 0, kd = 0, nd = 0;
    for (int l = 1; l < 16; ++l) {
      kl += (uint32_t)sl.count[l] << (15 - l);
      kd += (uint32_t)sd.count[l] << (15 - l);
      nd += sd.count[l];
    }
    if (kl != 32768u || (kd != 32768u && nd != 1u)) return false;
  }
  // The header alone lets through about one offset in a few thousand of compressed data.  So the block is decoded to its
  // end-of-block symbol (no symbol the exact step stops at on the way) and the next header must not be BTYPE 3.
  const int maxl = sl.maxlen, maxd = sd.maxlen;
  for (uint32_t nsym = 0; nsym < 65536u + 258u; ++nsym) {  // zlib's blocks hold at most 64 Ki symbols
    br.refill();
    if (!br.fast() && br.rem_bits() < maxl) return false;
    const uint32_t e = lut_l[br.peek(LBITS)];
    int nb = e & 15, sym = e >> 4;
    if (nb == 0) {
      nb = slow_decode<LBITS, uint16_t>(br.peek(15), sl.first, sl.count, sl.offs, sl.perm, maxl, &sym);
      if (nb == 0) return false;
    }
    br.drop(nb);
    if (sym < 256) continue;
    if (sym == 256) {
      br.refill();
      return br.rem_bits() < 3 || (br.peek(3) >> 1) != 3u;
    }
    if (sym > 285) return false;
    const int lx = c_len_tab[sym - 257] & 15;
    if (!br.fast() && br.rem_bits() < lx + maxd) return false;
    br.drop(lx);
    br.refill();
    const uint32_t de = lut_d[br.peek(DBITS)];
    int dn = de & 15, dsym = de >> 4;
    if (dn == 0) {
      dn = slow_decode<DBITS, uint8_t>(br.peek(15), sd.first, sd.count, sd.offs, sd.perm, maxd, &dsym);
      if (dn == 0) return false;
    }
    if (dsym > 29) return false;
    br.drop(dn);
    const int dx = c_dist_tab[dsym] & 15;
    if (!br.fast() && br.rem_bits() < dx) return false;
    br.drop(dx);
  }
  return false;
}

// One warp per chunk: bit offsets lo, lo + 1, ... below hi of its stream are tried 32 at a time; the lowest that passes
// wins.
__global__ void __launch_bounds__(32)
k_inflate_find_blocks(const uint8_t *__restrict__ in_base, const CkStream *__restrict__ streams,
                      const CkFind *__restrict__ finds, unsigned long long *__restrict__ cand, uint32_t n) {
  const uint32_t k = blockIdx.x;
  if (k >= n) return;
  const int lane = threadIdx.x & 31;
  uint16_t lut[LUT_HALFWORDS];
  uint8_t lens[320];
  SlowTab sl;
  SlowTabD sd;
  const CkFind fd = finds[k];
  const uint8_t *in = in_base + streams[fd.stream].in_off;
  const uint32_t in_len = streams[fd.stream].in_len;
  const unsigned long long a = fd.lo, b = fd.hi;
  unsigned long long found = CK_NOCAND;
  for (unsigned long long base = a; base < b; base += 32) {
    const unsigned long long o = base + (unsigned long long)lane;
    const bool ok = o < b && ck_block_here(in, in_len, o, lens, lut, lut + (1 << LBITS), sl, sd);
    const unsigned v = __ballot_sync(0xffffffffu, ok);
    if (v) {
      found = base + (unsigned long long)(__ffs((int)v) - 1);
      break;
    }
  }
  if (lane == 0) cand[k] = found;
}

// One lane per chunk: decode from jobs[j].start_bit, block after block, until a block ends at or past stop_bit or a final
// block is done.  Symbols go to 64 KiB pages taken off the stream's page range by its atomic counter
// (page_ctr[stream]); every page records whose it is.
__global__ void __launch_bounds__(32)
k_inflate_chunks(const uint8_t *__restrict__ in_base, const CkStream *__restrict__ streams, const CkJob *__restrict__ jobs,
                 uint32_t n, CkRes *__restrict__ res, uint16_t *__restrict__ pool, CkPage *__restrict__ pinfo,
                 uint32_t *page_ctr) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const CkJob job = jobs[j];
  const CkStream sm = streams[job.stream];
  const uint8_t *in = in_base + sm.in_off;
  const uint32_t in_len = sm.in_len;
  uint16_t lut[LUT_HALFWORDS];
  uint16_t *lut_l = lut, *lut_d = lut + (1 << LBITS);
  uint8_t lens[320];
  SlowTab sl;
  SlowTabD sd;
  BitReader br;
  ck_reader(br, in, in_len, job.start_bit);
  uint32_t nsym = 0, cur = 0, prev = 0;
  int st = 0;
  bool final_block = false;
  int first_type = -1;
  // the next symbol; false when the pool is exhausted
  auto put = [&](uint32_t v) -> bool {
    if ((nsym & (CK_PAGE - 1u)) == 0u) {
      uint32_t p = atomicAdd(page_ctr + job.stream, 1u);
      if (p >= sm.n_pages) return false;
      p += sm.page0;
      CkPage pi;
      pi.slot = job.slot;
      pi.seq = nsym / CK_PAGE;
      pi.gen = job.gen;
      pi.pad = 0;
      pinfo[p] = pi;
      prev = cur;
      cur = p;
    }
    pool[(size_t)cur * CK_PAGE + (nsym & (CK_PAGE - 1u))] = (uint16_t)v;
    nsym++;
    return true;
  };
  // symbol `dist` (1..32768) back: a marker in front of the chunk, else from the current or the previous page
  auto back = [&](uint32_t dist) -> uint32_t {
    if (dist > nsym) return 0x8000u | (CK_PAGE - (dist - nsym));
    const uint32_t q = nsym - dist;
    const uint32_t pg = (q / CK_PAGE) == ((nsym - 1u) / CK_PAGE) ? cur : prev;
    return pool[(size_t)pg * CK_PAGE + (q & (CK_PAGE - 1u))];
  };
  for (;;) {
    // ---- block boundary (the exact step's, inflate_decode.cuh) ----
    if (final_block) { st = CK_FINAL; break; }
    if (ck_bitpos(br) >= job.stop_bit) { st = CK_BOUNDARY; break; }
    br.refill();
    if (br.rem_bits() < 8) { st = B200Z_U_EOS; break; }
    const uint32_t hdr = br.peek(3);
    br.drop(3);
    final_block = hdr & 1u;
    const uint32_t type = hdr >> 1;
    if (first_type < 0) first_type = (int)type;
    if (type == 0) {
      br.drop((int)(br.rem_bits() & 7));
      long long rem_bytes = br.rem_bits() >> 3;
      uint32_t pos = br.in_len - (uint32_t)rem_bytes;
      long long len = -1, nlen;
      if (rem_bytes >= 2) {
        br.refill();
        len = br.peek(16);
        br.drop(16);
        rem_bytes -= 2;
        pos += 2;
      } else {
        rem_bytes = 0;
        pos = br.in_len;
      }
      if (rem_bytes >= 2) {
        br.refill();
        nlen = (long long)br.peek(16) ^ 0xffff;
        br.drop(16);
        rem_bytes -= 2;
        pos += 2;
      } else {
        nlen = -1ll ^ 0xffff;
        rem_bytes = 0;
        pos = br.in_len;
      }
      if ((len != 0 && len != nlen) || len > rem_bytes) { st = B200Z_U_STOP; break; }
      bool full = false;
      for (long long i = 0; i < len && !full; ++i) full = !put(in[pos + i]);
      if (full) { st = CK_POOL; break; }
      br.seek(pos + (uint32_t)(len > 0 ? len : 0));
      continue;
    }
    if (type == 3) { st = B200Z_U_STOP; break; }
    st = parse_tables(br, type, lens, lut_l, lut_d, sl, sd);
    if (st != 0) break;
    const int maxl = sl.maxlen, maxd = sd.maxlen;
    // ---- symbols (_decodeHuffman, the exact step's token loop) ----
    for (;;) {
      br.refill();
      const bool careful = !br.fast();
      if (careful && br.rem_bits() < maxl) { st = U_STOP_SHORT; break; }
      const uint32_t e = lut_l[br.peek(LBITS)];
      int nb = e & 15, sym = e >> 4;
      if (nb == 0) {
        nb = slow_decode<LBITS, uint16_t>(br.peek(15), sl.first, sl.count, sl.offs, sl.perm, maxl, &sym);
        if (nb == 0) { st = B200Z_U_BADCODE; break; }
      }
      br.drop(nb);
      if (sym < 256) {
        if (!put((uint32_t)sym)) { st = CK_POOL; break; }
        continue;
      }
      if (sym == 256) break;
      if (sym > 285) { st = B200Z_U_STOP; break; }
      const uint32_t le = c_len_tab[sym - 257];
      const int lx = le & 15;
      int mlen = (int)(le >> 4);
      if (!careful) {
        mlen += (int)br.peek(lx);
        br.drop(lx);
      } else if (lx) {
        if (br.rem_bits() < lx) mlen -= 1;  // _readBits -> -1 is ADDED to the base (inflate.dart:323)
        else { mlen += (int)br.peek(lx); br.drop(lx); }
      }
      br.refill();
      const bool careful2 = !br.fast();
      if (careful2 && br.rem_bits() < maxd) { st = U_STOP_SHORT; break; }
      const uint32_t de = lut_d[br.peek(DBITS)];
      int dn = de & 15, dsym = de >> 4;
      if (dn == 0) {
        dn = slow_decode<DBITS, uint8_t>(br.peek(15), sd.first, sd.count, sd.offs, sd.perm, maxd, &dsym);
        if (dn == 0) dsym = 0;  // hole in the flat table: (len 0, sym 0) (_huffman_table.dart:22)
      }
      br.drop(dn);
      if (dsym > 29) { st = B200Z_U_STOP; break; }
      const uint32_t dd = c_dist_tab[dsym];
      const int dx = dd & 15;
      int dist = (int)(dd >> 4);
      if (!careful2) {
        dist += (int)br.peek(dx);
        br.drop(dx);
      } else if (dx) {
        if (br.rem_bits() < dx) dist -= 1;
        else { dist += (int)br.peek(dx); br.drop(dx); }
      }
      if (dist <= 0) { st = B200Z_U_RANGE; break; }  // (reach before the allowed history: k_inflate_emit's flag)
      bool full = false;
      int i = 0;
      if (dist >= 8) {  // eight sources at a time: their loads do not wait on each other
        for (; i + 8 <= mlen && !full; i += 8) {
          uint32_t v[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) v[u] = back((uint32_t)dist - (uint32_t)u);
#pragma unroll
          for (int u = 0; u < 8; ++u) full = full || !put(v[u]);
        }
      }
      for (; i < mlen && !full; ++i) full = !put(back((uint32_t)dist));
      if (full) { st = CK_POOL; break; }
    }
    if (st != 0) break;
  }
  CkRes r;
  r.end_bit = ck_bitpos(br);
  r.nsym = nsym;
  r.status = st;
  r.first_stored = first_type == 0;
  r.pad = 0;
  res[j] = r;
}

// Byte of symbol v of a chunk whose output starts at out_off; a marker reads the (already final) output in front of the
// chunk.  A reach before `lo_valid` (the first byte a back-reference of this stream may touch) raises *bad.
__device__ __forceinline__ uint8_t ck_resolve(uint32_t v, const uint8_t *out, unsigned long long out_off,
                                              unsigned long long lo_valid, uint32_t *bad) {
  if (!(v & 0x8000u)) return (uint8_t)v;
  const unsigned long long src = out_off - CK_PAGE + (v & 0x7fffu);
  if (out_off + (v & 0x7fffu) < CK_PAGE + lo_valid) {
    atomicOr(bad, 1u);
    return 0;
  }
  return out[src];
}

// One CTA per stream walks its chain, chain[chain_lo[blockIdx.x] .. chain_lo[blockIdx.x + 1]), in order and writes the
// resolved last 32 KiB of every chunk at its final place: the window of chunk k + 1 is then in the output buffer when
// k + 1 is reached (a chunk shorter than 32 KiB reaches further back, into tails written before it).  Streams write
// disjoint output ranges, so their CTAs do not wait on each other.
constexpr int CK_WIN_THREADS = 256;
constexpr int CK_WIN_PER_THREAD = (int)CK_PAGE / CK_WIN_THREADS;
__global__ void __launch_bounds__(CK_WIN_THREADS)
k_inflate_windows(const CkChain *__restrict__ chain, const uint32_t *__restrict__ chain_lo, const uint32_t *__restrict__ flat,
                  const uint16_t *__restrict__ pool, uint8_t *out, const CkStream *__restrict__ streams, uint32_t *bad) {
  const uint32_t k0 = chain_lo[blockIdx.x], k1 = chain_lo[blockIdx.x + 1];
  for (uint32_t k = k0; k < k1; ++k) {
    const CkChain c = chain[k];
    const unsigned long long lo_valid = streams[c.stream].lo_valid;
    const uint32_t t = c.nsym < CK_PAGE ? c.nsym : CK_PAGE, base = c.nsym - t;
    uint32_t v[CK_WIN_PER_THREAD];
#pragma unroll
    for (int i = 0; i < CK_WIN_PER_THREAD; ++i) {  // all loads first: they do not wait on each other
      const uint32_t x = (uint32_t)i * CK_WIN_THREADS + threadIdx.x;
      const uint32_t q = base + x;
      v[i] = x < t ? pool[(size_t)flat[c.page0 + q / CK_PAGE] * CK_PAGE + (q & (CK_PAGE - 1u))] : 0u;
    }
#pragma unroll
    for (int i = 0; i < CK_WIN_PER_THREAD; ++i) {
      const uint32_t x = (uint32_t)i * CK_WIN_THREADS + threadIdx.x;
      if (x < t) out[c.out_off + base + x] = ck_resolve(v[i], out, c.out_off, lo_valid, bad + c.stream);
    }
    __syncthreads();
  }
}

// One CTA per page of the flat page list (every stream's chain): symbols -> bytes at their final place.  A chunk's last
// 32 KiB are k_inflate_windows' and are left alone here: other CTAs read them as windows.  A reach before the stream's
// allowed history raises that stream's flag only.
__global__ void __launch_bounds__(256)
k_inflate_emit(const CkChain *__restrict__ chain, const uint32_t *__restrict__ flat, const uint32_t *__restrict__ flat_chunk,
               const uint16_t *__restrict__ pool, uint8_t *out, const CkStream *__restrict__ streams, uint32_t *bad) {
  const uint32_t f = blockIdx.x;
  const CkChain c = chain[flat_chunk[f]];
  const unsigned long long lo_valid = streams[c.stream].lo_valid;
  const uint32_t seq = f - c.page0;
  const uint32_t first = seq * CK_PAGE;
  const uint32_t body = c.nsym > CK_PAGE ? c.nsym - CK_PAGE : 0u;  // symbols in front of the tail
  if (first >= body) return;
  const uint32_t cnt = body - first < CK_PAGE ? body - first : CK_PAGE;
  const uint16_t *src = pool + (size_t)flat[f] * CK_PAGE;
  uint8_t *dst = out + c.out_off + first;
  for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x) dst[i] = ck_resolve(src[i], out, c.out_off, lo_valid, bad + c.stream);
}

}  // namespace b200z
