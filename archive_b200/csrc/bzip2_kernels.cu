// bzip2_kernels.cu -- sm_90a BZip2 block decode.
//
// Replaces (reference, paths relative to /root/reference/):
//   lib/src/codecs/bzip2_decoder.dart:90-111    _readBlockType         -> k_bz2_scan      (K6)
//   lib/src/codecs/bzip2_decoder.dart:113-388   _readCompressed part 1 -> k_bz2_entropy_fast / k_bz2_entropy (K7)
//       (symbol map, selectors, code lengths, _hbCreateDecodeTables :774-813, _getMtfVal :732-772,
//        MTF + RUNA/RUNB)
//   lib/src/codecs/bzip2_decoder.dart:397-439   cftab + T^-1            -> k_bz2_expand / k_bz2_chunk_hist /
//                                                                          k_bz2_chunk_scan / k_bz2_build_tt
//   lib/src/codecs/bzip2_decoder.dart:610-727   pointer chase + un-RLE  -> k_bz2_walk_len / _order / _emit,
//                                                                          k_bz2_rle_count / k_bz2_rle_emit
//   lib/src/codecs/bzip2/bzip2.dart:11-14       CRC (0x04c11db7, MSB first) -> inside k_bz2_rle_emit
//
// Shape of the work (DESIGN.md "K6-K8"): the entropy stage is a chain per block (a table switch every 50 symbols + an MTF
// list).  k_bz2_entropy_fast breaks it up for clean blocks -- code look-ups at every bit offset of a window + four-symbol
// jumps leave ~13 dependent hops per group of 50 symbols, move-to-front runs symbolically per group (32 groups at once) and
// is composed across groups, records come from ballots and scans -- and k_bz2_entropy, one warp per block walking every
// symbol, decodes whatever the fast kernel flags, with the reference's verdicts.  Everything after it is data parallel:
// records -> bytes, a stable counting sort builds T, the single cycle of T is cut at ~4096 splitters whose segments are
// walked by threads that take them off a counter, and RLE1 + CRC are scans over a 5-state automaton / an associative
// CRC combine.
#include <stdint.h>
#include <stdlib.h>

#include <algorithm>

#include "b200z_internal.h"
#include "bz2_rnums.h"

namespace b200z {

// ---------------------------------------------------------------------------------------------
// MSB-first bit reader over 32-bit big-endian words (bz2_bit_reader.dart:12-44)
// ---------------------------------------------------------------------------------------------
struct BzBits {
  const uint32_t *w;   // 4-byte aligned base of the whole stream
  uint64_t buf;        // next bit = bit 63
  int cnt;             // valid bits in buf
  uint64_t next_word;  // index of the next word to load
  uint64_t n_words;    // words that contain stream bytes
  uint32_t last_mask;  // bytes of word n_words - 1 that belong to the stream
  // the stream's bytes end at bit end_bit of w: from there on the reader sees zeros, as behind a stream staged on its own,
  // whatever bytes (another stream's) follow in the buffer
  __device__ __forceinline__ void set_end(uint64_t end_bit) {
    const uint64_t nb = end_bit >> 3;
    n_words = (nb + 3) >> 2;
    last_mask = (nb & 3) ? ~0u << (8 * (4 - (uint32_t)(nb & 3))) : ~0u;
  }
  __device__ __forceinline__ uint32_t word(uint64_t i) const {
    const uint32_t v = i < n_words ? __byte_perm(__ldg(w + i), 0, 0x0123) : 0u;
    return i + 1 == n_words ? v & last_mask : v;
  }
  __device__ __forceinline__ void seek(uint64_t bitpos) {
    next_word = bitpos >> 5;
    uint32_t sh = (uint32_t)(bitpos & 31);
    uint32_t v = word(next_word);
    next_word++;
    buf = ((uint64_t)v << 32) << sh;
    cnt = 32 - (int)sh;
  }
  __device__ __forceinline__ void refill() {
    if (cnt <= 32) {
      uint32_t v = word(next_word);
      if ((next_word & 31u) == 0u) asm volatile("prefetch.global.L1 [%0];" ::"l"(w + next_word + 64));
      next_word++;
      buf |= (uint64_t)v << (32 - cnt);
      cnt += 32;
    }
  }
  __device__ __forceinline__ uint32_t get(int n) {  // 1..24 bits
    refill();
    uint32_t x = (uint32_t)(buf >> (64 - n));
    buf <<= n;
    cnt -= n;
    return x;
  }
  __device__ __forceinline__ uint64_t bitpos() const { return next_word * 32 - (uint64_t)cnt; }
};

// ---------------------------------------------------------------------------------------------
// K6: every bit offset is tested for the block magic 0x314159265359 and the end-of-stream magic
// 0x177245385090 (bzip2.dart compressedMagic / eosMagic).  cand = bit position of the magic in `in` | type << 63.
// Over a stream table (a.streams) a magic counts only when it lies wholly inside its stream, each candidate carries its
// stream and the 32 bits behind its magic (the stored CRC), and thread 0 of every stream copies the stream's first 4 and
// last 8 bytes to a.ends (what the host needs of the header and of a truncated block signature).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_bz2_scan(const Bz2Scan a) {
  const uint64_t MAGIC_BLK = 0x314159265359ull, MAGIC_EOS = 0x177245385090ull;
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t si = 0;
  uint64_t off = 0, n_bytes = a.n_bytes, b0 = t * 4;
  if (a.streams) {
    if (t >= a.first_thr[a.n_streams]) return;
    uint32_t lo = 0, hi = a.n_streams;  // the stream whose threads hold t: first_thr[lo] <= t < first_thr[lo + 1]
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) >> 1;
      if (a.first_thr[mid] <= t) lo = mid;
      else hi = mid;
    }
    si = lo;
    off = a.streams[si].off;
    n_bytes = a.streams[si].len;
    b0 = (t - a.first_thr[si]) * 4;
    if (b0 == 0 && a.ends) {
      uint8_t *e = a.ends + (size_t)si * 12;
      for (int i = 0; i < 4; ++i) e[i] = (uint64_t)i < n_bytes ? a.in[off + i] : 0;
      for (int i = 0; i < 8; ++i) e[4 + i] = n_bytes + i >= 8 ? a.in[off + n_bytes + i - 8] : 0;
    }
  }
  if (b0 >= n_bytes) return;
  const uint8_t *in = a.in + off;
  // 11 bytes cover 4 byte offsets x 8 bit shifts x 48 bits
  uint8_t by[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) by[i] = (b0 + i < n_bytes) ? in[b0 + i] : 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (b0 + k + 6 > n_bytes) break;  // fewer than 48 bits left even at shift 0
    uint64_t v = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) v = (v << 8) | by[k + i];
#pragma unroll
    for (int s = 0; s < 8; ++s) {
      uint64_t m = (v << s) >> 16;
      bool blk = m == MAGIC_BLK, eos = m == MAGIC_EOS;
      if (blk || eos) {
        uint64_t bit = (b0 + k) * 8 + s;
        if (bit + 48 <= n_bytes * 8) {
          uint32_t slot = atomicAdd(a.n_cand, 1u);
          if (slot < a.cap) {
            a.cand[slot] = (off * 8 + bit) | (eos ? (1ull << 63) : 0ull);
            if (a.streams) {
              uint64_t c = 0;  // (bytes past the stream's end read 0)
              for (int i = 0; i < 5; ++i) c = (c << 8) | (b0 + k + 6 + i < n_bytes ? in[b0 + k + 6 + i] : 0);
              a.cand_stream[slot] = si;
              a.cand_crc[slot] = (uint32_t)(c >> (8 - s));
            }
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// K7: entropy decode of one block per warp.
// ---------------------------------------------------------------------------------------------
constexpr int BZ_LUT_BITS = 10;
constexpr int BZ_MAX_SEL = 18002;  // bzMaxSelectors (bzip2_decoder.dart:847)

struct BzSmem {
  uint16_t lut[6][1 << BZ_LUT_BITS];  // (sym << 5) | len ; 0 = needs the limit/base walk
  int32_t limit[6][24];
  int32_t base[6][24];
  uint16_t perm[6][258];
  uint8_t len[6][258];
  uint8_t minlen[6];
  uint8_t selector[BZ_MAX_SEL + 2];
  __device__ __forceinline__ void set_sel(int i, uint8_t v) { selector[i] = v; }
  uint32_t mtfw[64];  // the MTF list, 4 entries per word (entry k = byte k%4 of word k/4)
  uint8_t seq2unseq[256];
};

// status per block
#define BZ_OK 0
#define BZ_DATA (-1)    // _readCompressed returned -1 -> decodeStream returns false
#define BZ_THROW (-2)   // the Dart code would have thrown (read past the end / selector overrun)
#define BZ_QUIRK (-3)   // _getMtfVal returned -1 after the first symbol: the reference does not look at that value and goes
                        // on with it (:387, :306) -- k_bz2_entropy_literal decodes such a block the reference's way

// ---- block header (bzip2_decoder.dart:113-257): symbol map, selectors (MTF undone on the fly), code lengths, and
// _hbCreateDecodeTables (:774-813) per table.  One thread; SM is the kernel's shared-memory block (seq2unseq, len, minlen,
// perm, base, limit, set_sel).  Shared by the exact kernel and the fast one. ----
struct BzHdr {
  int n_groups, n_sel, alpha, n_in_use, err;
  uint32_t optr, rnd;
};
template <class SM>
__device__ void bz_parse_header(SM &S, BzBits &br, uint64_t blk_bit, uint64_t total_bits, BzHdr &h) {
  int err = 0;
  uint32_t rnd = 0, optr = 0;
  int n_groups = 0, n_sel = 0, alpha = 0, n_in_use = 0;
  // header: after the 48-bit magic and the 32-bit stored CRC (bzip2_decoder.dart:113-218)
  br.seek(blk_bit + 48 + 32);
  rnd = br.get(1);
  optr = br.get(8);
  optr = (optr << 8) | br.get(8);
  optr = (optr << 8) | br.get(8);
  uint32_t used16 = br.get(16);
  for (int i = 0; i < 16; ++i) {
    if (used16 & (0x8000u >> i)) {
      uint32_t m = br.get(16);
      for (int j = 0; j < 16; ++j)
        if (m & (0x8000u >> j)) S.seq2unseq[n_in_use++] = (uint8_t)(i * 16 + j);
    }
  }
  if (n_in_use == 0) err = BZ_DATA;
  alpha = n_in_use + 2;
  if (!err) {
    n_groups = (int)br.get(3);
    if (n_groups < 2 || n_groups > 6) err = BZ_DATA;
  }
  if (!err) {
    n_sel = (int)br.get(15);
    if (n_sel < 1) err = BZ_DATA;
  }
  if (!err) {
    // (one thread parses up to 18 002 selectors: the run of ones is counted with one clz instead of bit by bit, and the
    // MTF list of the <= 6 tables is six nibbles of a register)
    uint32_t pl = 0x543210u;  // list entry k = nibble k
    for (int i = 0; i < n_sel && !err; ++i) {
      br.refill();
      const int j = __clz((int)~(uint32_t)(br.buf >> 32));  // ones in front of the first zero (:160-167)
      if (j >= n_groups) {
        err = BZ_DATA;
        break;
      }
      br.buf <<= (j + 1);
      br.cnt -= (j + 1);
      if (i >= BZ_MAX_SEL) {  // _selectorMtf[i]: RangeError (bzip2_decoder.dart:168)
        err = BZ_THROW;
        break;
      }
      // undo the selector MTF on the fly (:172-186): same result as the reference's second loop
      const uint32_t sh = 4u * (uint32_t)j;
      const uint32_t tmp = (pl >> sh) & 15u;
      const uint32_t low = pl & ((1u << sh) - 1u);
      pl = (pl & ~((16u << sh) - 1u)) | (low << 4) | tmp;
      S.set_sel(i, (uint8_t)tmp);
      if (br.bitpos() > total_bits) {
        err = BZ_THROW;
        break;
      }
    }
  }
  if (!err) {
    for (int t = 0; t < n_groups && !err; ++t) {
      int c = (int)br.get(5);
      for (int i = 0; i < alpha && !err; ++i) {
        for (;;) {
          if (c < 1 || c > 20) {
            err = BZ_DATA;
            break;
          }
          if (br.get(1) == 0) break;
          if (br.get(1) == 0) c++;
          else c--;
        }
        S.len[t][i] = (uint8_t)c;
      }
      if (br.bitpos() > total_bits) err = BZ_THROW;
    }
  }
  if (!err) {
    // _hbCreateDecodeTables (:774-813) per table
    for (int t = 0; t < n_groups; ++t) {
      int mn = 32, mx = 0;
      for (int i = 0; i < alpha; ++i) {
        int l = S.len[t][i];
        mx = l > mx ? l : mx;
        mn = l < mn ? l : mn;
      }
      S.minlen[t] = (uint8_t)mn;
      for (int i = 0; i < 258; ++i) S.perm[t][i] = 0;  // Int32List(bzMaxAlphaSize) starts zeroed (:234)
      int pp = 0;
      for (int i = mn; i <= mx; i++)
        for (int j = 0; j < alpha; j++)
          if (S.len[t][j] == i) S.perm[t][pp++] = (uint16_t)j;
      int32_t *base = S.base[t], *limit = S.limit[t];
      for (int i = 0; i < 23; i++) base[i] = 0;
      for (int i = 0; i < alpha; i++) base[S.len[t][i] + 1]++;
      for (int i = 1; i < 23; i++) base[i] += base[i - 1];
      for (int i = 0; i < 23; i++) limit[i] = 0;
      int32_t vec = 0;
      for (int i = mn; i <= mx; i++) {
        vec += (base[i + 1] - base[i]);
        limit[i] = vec - 1;
        vec <<= 1;
      }
      for (int i = mn + 1; i <= mx; i++) base[i] = ((limit[i - 1] + 1) << 1) - base[i];
    }
  }
  h.n_groups = n_groups;
  h.n_sel = n_sel;
  h.alpha = alpha;
  h.n_in_use = n_in_use;
  h.err = err;
  h.optr = optr;
  h.rnd = rnd;
}

// The decode LUTs, filled by `nthr` threads.  Entry for a 10-bit prefix = what _getMtfVal's limit/base walk (:747-771)
// decides from those bits alone, so any code-length set (valid or not) decodes exactly as in the reference.
template <class SM>
__device__ void bz_fill_luts(SM &S, int n_groups, int tid, int nthr) {
  for (int t = 0; t < n_groups; ++t) {
    const int mn = S.minlen[t];
    for (int v = tid; v < (1 << BZ_LUT_BITS); v += nthr) {
      uint16_t e = 0;
      for (int zn = mn; zn <= BZ_LUT_BITS; ++zn) {
        if (zn < 1) continue;
        int32_t zvec = v >> (BZ_LUT_BITS - zn);
        if (zvec <= S.limit[t][zn]) {
          int32_t idx = zvec - S.base[t][zn];
          if (idx < 0 || idx >= 258) e = (uint16_t)((0x3ff << 5) | zn);  // data error marker
          else e = (uint16_t)((S.perm[t][idx] << 5) | zn);
          break;
        }
      }
      S.lut[t][v] = e;
    }
  }
}

__global__ void __launch_bounds__(32)
k_bz2_entropy(const uint32_t *__restrict__ words, uint64_t n_bytes, const unsigned long long *__restrict__ blk_bit,
              uint32_t n_blocks, uint32_t nblock_max, uint32_t *__restrict__ rec_val, uint32_t *__restrict__ rec_pos,
              uint32_t *__restrict__ n_rec, uint32_t *__restrict__ nblock_out, uint32_t *__restrict__ orig_ptr,
              uint32_t *__restrict__ randomised, unsigned long long *__restrict__ end_bit, int32_t *__restrict__ status,
              int only_redo, const unsigned long long *__restrict__ blk_end, const uint32_t *__restrict__ blk_lim) {
  extern __shared__ __align__(16) uint8_t smraw[];
  BzSmem &S = *reinterpret_cast<BzSmem *>(smraw);
  const uint32_t b = blockIdx.x;
  if (b >= n_blocks) return;
  if (only_redo && status[b] != -9) return;  // (BZ_REDO) the fast kernel has decoded this block
  const int lane = threadIdx.x;
  const uint64_t total_bits = blk_end ? blk_end[b] : n_bytes * 8;
  const uint32_t lim = blk_lim ? blk_lim[b] : nblock_max;  // the block's own limit; nblock_max is the stride of its arrays
  __shared__ int s_groups, s_alpha, s_err, s_nsel, s_inuse;
  __shared__ uint32_t s_optr, s_rnd;
  __shared__ unsigned long long s_bitpos;

  BzBits br;
  br.w = words;
  br.set_end(total_bits);
  int err = 0;
  uint32_t rnd = 0, optr = 0;
  int n_groups = 0, n_sel = 0, alpha = 0, n_in_use = 0;

  if (lane == 0) {
    BzHdr h;
    bz_parse_header(S, br, blk_bit[b], total_bits, h);
    n_groups = h.n_groups;
    n_sel = h.n_sel;
    alpha = h.alpha;
    n_in_use = h.n_in_use;
    err = h.err;
    optr = h.optr;
    rnd = h.rnd;
    s_groups = n_groups;
    s_alpha = alpha;
    s_err = err;
    s_nsel = n_sel;
    s_inuse = n_in_use;
    s_optr = optr;
    s_rnd = rnd;
    s_bitpos = br.bitpos();
  }
  __syncwarp();
  n_groups = s_groups;
  alpha = s_alpha;
  if (s_err == 0) {
    bz_fill_luts(S, n_groups, lane, 32);
  }
  __syncwarp();
  // From here on EVERY lane walks the same bits with the same tables (shared-memory reads of one address are broadcasts),
  // so the symbol is known to the whole warp without an exchange -- and the move-to-front list, the other serial chain of
  // this stage, lives in the warp's registers: lane l holds entries 8l .. 8l+7 as one 64-bit word, a symbol's position is
  // served by one shuffle and the shift of everything in front of it by another, whatever the position.  (With the list
  // in shared memory a position of 20 cost five dependent read-modify-writes; text sits at 5-10 on average.)  The next
  // symbol's Huffman look-up is issued before the list work of the current one, so the two chains overlap.
  err = s_err;
  n_sel = s_nsel;
  n_in_use = s_inuse;
  optr = s_optr;
  rnd = s_rnd;
  br.seek(s_bitpos);
  const unsigned FULLW = 0xffffffffu;
  uint32_t nrec = 0, nblock = 0;
  if (!err) {
    uint64_t v = 0;  // my eight list entries
    for (int k = 0; k < 8; ++k) v |= (uint64_t)(8 * lane + k) << (8 * k);
    uint32_t front = 0;  // list entry 0 (every lane keeps it)
    const int eob = n_in_use + 1;
    uint32_t *rv = rec_val + (size_t)b * nblock_max;
    uint32_t *rp = rec_pos + (size_t)b * nblock_max;
    uint32_t my_rv = 0, my_rp = 0;  // records leave 32 at a time, lane k carries record k of the group
    int gpos = 0, gno = -1, tsel = 0;
    int run_n = 0;       // number of RUNA/RUNB symbols in the open run
    uint32_t run_es = 0;  // value accumulated so far (es + 1 in the reference's terms)
    // ---- _getMtfVal (:732-772); sets derr instead of returning -1 ----
    int derr = 0;
    auto decode = [&]() -> int {
      if (gpos == 0) {
        gno++;
        if (gno >= n_sel) {
          derr = BZ_DATA;  // reference returns -1 here (then spins to the block limit and fails)
          return 0;
        }
        gpos = 50;
        tsel = S.selector[gno];
      }
      gpos--;
      br.refill();
      uint32_t e = S.lut[tsel][(uint32_t)(br.buf >> (64 - BZ_LUT_BITS))];
      int zn = e & 31;
      int sym = e >> 5;
      if (zn == 0) {
        // code longer than the LUT (or a minLen above it): the reference's walk from LUT_BITS+1 (or minLen) on
        zn = S.minlen[tsel] > BZ_LUT_BITS + 1 ? S.minlen[tsel] : BZ_LUT_BITS + 1;
        for (;;) {
          if (zn > 20) {
            derr = BZ_DATA;
            return 0;
          }
          int32_t zvec = (int32_t)(br.buf >> (64 - zn));
          if (zvec <= S.limit[tsel][zn]) {
            int32_t idx = zvec - S.base[tsel][zn];
            if (idx < 0 || idx >= 258) {
              derr = BZ_DATA;
              return 0;
            }
            sym = S.perm[tsel][idx];
            break;
          }
          zn++;
        }
      } else if (sym == 0x3ff) {
        derr = BZ_DATA;
        return 0;
      }
      br.buf <<= zn;
      br.cnt -= zn;
      return sym;
    };
    auto emit = [&](uint32_t val, uint32_t pos) {
      if ((uint32_t)lane == (nrec & 31u)) {
        my_rv = val;
        my_rp = pos;
      }
      nrec++;
      if ((nrec & 31u) == 0u) {
        rv[nrec - 32u + lane] = my_rv;
        rp[nrec - 32u + lane] = my_rp;
      }
    };
    int sym = decode();
    err = derr;
    while (!err) {
      // the NEXT symbol's Huffman decode does not depend on the list work of this one: start it first so the two
      // dependency chains overlap (a decode error is acted on after this symbol, as in the reference's order)
      const bool more = sym != eob;
      int nsym = 0;
      if (more) nsym = decode();
      // ---- MTF / run-length (:276-388) ----
      if (sym <= 1) {
        if (run_n >= 21) {  // N >= 2*1024*1024 (:291)
          err = BZ_DATA;
          break;
        }
        run_es += (uint32_t)(sym + 1) << run_n;
        run_n++;
      } else {
        if (run_n) {
          if (nblock + run_es > lim) {  // (:313-316)
            err = BZ_DATA;
            break;
          }
          emit((run_es << 8) | S.seq2unseq[front], nblock);
          nblock += run_es;
          run_n = 0;
          run_es = 0;
        }
        if (sym == eob) break;
        if (nblock >= lim) {  // (:326-329)
          err = BZ_DATA;
          break;
        }
        // move entry nn to the front (:331-378 does the same job with its 16x16 blocks)
        const int nn = sym - 1, owner = nn >> 3;
        const uint32_t half = (nn & 4) ? (uint32_t)(v >> 32) : (uint32_t)v;
        const uint32_t uc = (__shfl_sync(FULLW, half, owner) >> ((nn & 3) * 8)) & 0xffu;
        uint32_t carry = __shfl_up_sync(FULLW, (uint32_t)(v >> 56), 1);
        if (lane == 0) carry = uc;
        if (lane < owner) {
          v = (v << 8) | carry;
        } else if (lane == owner) {
          const int sh = (nn & 7) * 8;
          const uint64_t below = v & ((1ull << sh) - 1ull);
          const uint64_t upto = sh == 56 ? ~0ull : ((1ull << (sh + 8)) - 1ull);
          v = (v & ~upto) | (((below << 8) | carry) & upto);
        }
        front = uc;
        emit((1u << 8) | S.seq2unseq[uc], nblock);
        nblock++;
        if ((nrec & 1023u) == 0u && br.bitpos() > total_bits) {
          err = BZ_THROW;
          break;
        }
      }
      if (derr) {
        err = BZ_QUIRK;
        break;
      }
      sym = nsym;
    }
    // the records of the last, partial group
    if ((nrec & 31u) != 0u && (uint32_t)lane < (nrec & 31u)) {
      rv[(nrec & ~31u) + lane] = my_rv;
      rp[(nrec & ~31u) + lane] = my_rp;
    }
    if (!err && optr >= nblock) err = BZ_DATA;  // (:399-402) also covers nblock == 0
  }
  if (lane != 0) return;
  uint64_t endp = err ? s_bitpos : br.bitpos();
  if (!err) endp = br.bitpos();
  if (br.bitpos() > total_bits) err = BZ_THROW;  // some read went past the end: InputStream.readByte throws
  n_rec[b] = nrec;
  nblock_out[b] = nblock;
  orig_ptr[b] = optr;
  randomised[b] = rnd;
  end_bit[b] = endp;
  status[b] = err;
}

// ---------------------------------------------------------------------------------------------
// K7f `k_bz2_entropy_fast`: the entropy stage of a CLEAN block without its serial chain per symbol.
//
// _getMtfVal (:732-772) is a chain of ~700 k dependent table look-ups per 900 kB block, the MTF list (:331-378) a second
// one; the exact kernel above walks both with one warp.  Here a CTA of three warps splits the
// block into batches of 32 selector groups (50 symbols each) and pipelines them, a batch apart:
//   * the WALKER (warp 0) finds where every group starts -- nothing else.  For a group that starts at bit s with table t,
//     lane l looks up the code at each of the bit offsets s + 8l .. s + 8l + 7 (E[b] = the length of the code that would
//     start there: 256 look-ups at once, no chain), then J4[b] = where four symbols from b end (four dependent reads of E,
//     eight independent chains per lane; lengths read 0 behind the window, so a hop from there stays put, and a flag says
//     whether all four hops started inside).  The only serial part left is 12 hops over J4 and two over E per group.  A
//     group longer than the 256-bit window takes another round from where the chain left it.
//   * the DECODER (warp 1), one group per lane: 32 lanes decode their groups' 50 symbols side by side from the start bits
//     (the end-of-block code ends the block: the lowest lane that meets it), and undo move-to-front SYMBOLICALLY as they go:
//     every lane runs against a list that starts as the identity and records which INITIAL position each symbol refers to
//     (word-wise shifts in shared memory); the block's real list is then carried through the 32 groups by composing each
//     lane's permutation (32 lanes gather), which also resolves the references.
//   * the RECORDER (warp 2) takes the batch's resolved symbols as ONE stream, 32 at a time: RUNA/RUNB runs, record indices
//     and block positions are a ballot, a 5-step scan and two shuffles away (a run may straddle passes and batches).
// Output = the block's bytes (the L column of the BWT, K8's input; a run longer than 32 bytes as one of the exact kernel's
// records, which k_bz2_expand turns into bytes).  Anything that is not an ordinary block -- header errors, an invalid code on the
// parse, a run of more than 21 symbols, a block that overflows, selectors that run out, bits past the end of the input,
// origPtr out of range -- sets status BZ_REDO and the exact kernel decodes the block again with the reference's verdicts.
// ---------------------------------------------------------------------------------------------
#define BZ_REDO (-9)
constexpr int BZF_W = 256;  // bits of the walker's window
constexpr int BZF_NT = 96;  // threads: walker, decoder, recorder
constexpr uint32_t BZF_BADSYM = 0x3ffu;
constexpr uint32_t BZF_INLINE_RUN = 32u;  // runs up to this length are written as bytes by the recorder, longer ones as a record

struct BzFast {
  uint16_t lut[6][1 << BZ_LUT_BITS];
  int32_t limit[6][24];
  int32_t base[6][24];
  uint16_t perm[6][258];
  uint8_t len[6][258];
  uint8_t minlen[8];
  uint8_t selp[(BZ_MAX_SEL + 3) / 2 + 3];  // selectors, two per byte
  uint8_t seq2unseq[256];
  __device__ __forceinline__ void set_sel(int i, uint8_t v) {
    const uint8_t c = selp[i >> 1];
    selp[i >> 1] = (i & 1) ? (uint8_t)((c & 0x0fu) | (v << 4)) : (uint8_t)((c & 0xf0u) | v);
  }
  __device__ __forceinline__ int get_sel(int i) const { return (selp[i >> 1] >> ((i & 1) * 4)) & 15; }
  uint8_t EL[BZF_W + 64];  // walker: length of the code that starts at window bit b; 0 behind the window
  uint16_t J4[BZF_W];      // walker: where four symbols from b end | 0x8000 when all four started inside the window
  unsigned long long gstart[2][32];  // a batch: the bit every group starts at
  int ngw[2];                        // groups the walker found for the batch
  uint16_t syms[2][32][50];  // a batch: the symbols of 32 groups (references resolved to move-to-front VALUES | 0x8000)
  uint8_t cnt[2][32];        // symbols in each group of the batch (50; fewer in the block's last group)
  uint32_t mtf[64][32];      // decoder: word w of lane l's symbolic list
  uint8_t cur[256];          // decoder: the block's MTF list at the start of the group being resolved
  int ng[2], last[2];        // groups of the batch that belong to the block; the batch holds the end-of-block code
  int redo;
  unsigned long long end_bit, hdr_bitpos;
  BzHdr hdr;
};
static_assert(sizeof(BzFast) <= 45 * 1024, "five CTAs per SM");

__global__ void __launch_bounds__(BZF_NT)
k_bz2_entropy_fast(const uint32_t *__restrict__ words, uint64_t n_bytes, const unsigned long long *__restrict__ blk_bit,
                   uint32_t n_blocks, uint32_t nblock_max, uint32_t *__restrict__ rec_val, uint32_t *__restrict__ rec_pos,
                   uint32_t *__restrict__ n_rec, uint32_t *__restrict__ nblock_out, uint32_t *__restrict__ orig_ptr,
                   uint32_t *__restrict__ randomised, unsigned long long *__restrict__ end_bit, int32_t *__restrict__ status,
                   uint32_t *__restrict__ fast_flag, uint8_t *__restrict__ sym8, const unsigned long long *__restrict__ blk_end,
                   const uint32_t *__restrict__ blk_lim) {
  __shared__ BzFast S;
  const uint32_t b = blockIdx.x;
  if (b >= n_blocks) return;
  if (fast_flag && threadIdx.x == 0) fast_flag[b] = 0;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned FULLW = 0xffffffffu;
  const uint64_t total_bits = blk_end ? blk_end[b] : n_bytes * 8;
  const uint32_t lim = blk_lim ? blk_lim[b] : nblock_max;  // the block's own limit; nblock_max is the stride of its arrays
  // The walker and the decoder read whole words up to the stream's end without masking the bytes that follow it (another
  // stream's, in a batch): a block is only accepted here when all its symbols end inside the stream, and those symbols
  // do not depend on what follows; a block that reads further is handed to the exact kernel, whose reader sees zeros.
  const uint64_t n_words = ((total_bits >> 3) + 3) >> 2;
  if (tid == 0) {
    BzBits br;
    br.w = words;
    br.set_end(total_bits);
    BzHdr h;
    bz_parse_header(S, br, blk_bit[b], total_bits, h);
    S.hdr = h;
    S.hdr_bitpos = br.bitpos();
    S.end_bit = 0;
    S.redo = (h.err != 0 || br.bitpos() > total_bits) ? 1 : 0;
    S.ngw[0] = S.ngw[1] = 0;
    S.ng[0] = S.ng[1] = 0;
    S.last[0] = S.last[1] = 0;
  }
  __syncthreads();
  if (S.redo) {
    if (tid == 0) status[b] = BZ_REDO;
    return;
  }
  const BzHdr h = S.hdr;
  bz_fill_luts(S, h.n_groups, tid, BZF_NT);
  for (int i = tid; i < 256; i += BZF_NT) S.cur[i] = (uint8_t)i;
  if (tid < 64) S.EL[BZF_W + tid] = 0;
  __syncthreads();

  const uint32_t eob = (uint32_t)h.n_in_use + 1u;
  // walker state (warp 0; the same in every lane)
  uint64_t s = S.hdr_bitpos;  // bit the next group starts at
  int g = 0;                  // its number
  bool walk_done = false;
  // recorder state (warp 2; the same in every lane): what the exact kernel calls nrec, nblock, run_n, run_es, front
  uint32_t st_nrec = 0, st_nblock = 0, st_n = 0, st_v = 0, st_front = 0;
  uint32_t *const rv = rec_val + (size_t)b * nblock_max;
  uint32_t *const rp = rec_pos + (size_t)b * nblock_max;
  uint8_t *const s8 = sym8 + (size_t)b * nblock_max;  // the block's bytes (L of the BWT), written here directly
  auto ldw = [&](uint64_t i) -> uint32_t { return i < n_words ? __byte_perm(__ldg(words + i), 0, 0x0123) : 0u; };

  bool dec_done = false;   // the decoder has met the end-of-block code (in an earlier iteration)
  bool prev_last = false;  // ... and the batch the recorder takes in THIS iteration is the one that holds it
  for (int bt = 0;; ++bt) {
    if (warp == 0) {
      if (walk_done || dec_done) {
        if (lane == 0) S.ngw[bt & 1] = 0;
      } else {
        // ---------------- walker: where the groups of batch bt start ----------------
        const int buf = bt & 1;
        int ngb = 0;
        for (; ngb < 32 && g < h.n_sel; ++ngb, ++g) {
          const int t = S.get_sel(g);
          if (lane == 0) {
            S.gstart[buf][ngb] = s;
            if ((s >> 5) + 96 < n_words) asm volatile("prefetch.global.L1 [%0];" ::"l"(words + (s >> 5) + 96));
          }
          int need = 50;
          while (need > 0) {
            // E over [s, s + 256): my window starts at byte (s >> 3) + lane
            {
              const uint64_t byte0 = (s >> 3) + (uint64_t)lane, w0 = byte0 >> 2;
              const uint32_t bsh = (uint32_t)(byte0 & 3u) * 8u;
              const uint32_t a0 = ldw(w0), a1 = ldw(w0 + 1), a2 = ldw(w0 + 2);
              const uint32_t whi = __funnelshift_l(a1, a0, bsh), wlo = __funnelshift_l(a2, a1, bsh);
              const int o0 = (int)(s & 7u);
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const uint32_t x = __funnelshift_l(wlo, whi, (uint32_t)(o0 + j));  // 32 bits from window bit 8 * lane + j on
                uint32_t zl = S.lut[t][x >> (32 - BZ_LUT_BITS)] & 31u;
                if (zl == 0u) {  // longer than the LUT: the limit / base walk from there on (:747-771); no fit: 1 (the decoder flags it)
                  int zn = S.minlen[t] > BZ_LUT_BITS + 1 ? S.minlen[t] : BZ_LUT_BITS + 1;
                  zl = 1u;
                  for (; zn <= 20; ++zn)
                    if ((int32_t)(x >> (32 - zn)) <= S.limit[t][zn]) {
                      zl = (uint32_t)zn;
                      break;
                    }
                }
                S.EL[8 * lane + j] = (uint8_t)zl;
              }
            }
            __syncwarp();
            // J4: four symbols on from each bit of the window (eight independent chains per lane)
            {
              uint32_t p[8], p3[8];
#pragma unroll
              for (int j = 0; j < 8; ++j) p[j] = 8u * lane + j;
#pragma unroll
              for (int hop = 0; hop < 4; ++hop) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                  if (hop == 3) p3[j] = p[j];
                  p[j] += S.EL[p[j]];
                }
              }
#pragma unroll
              for (int j = 0; j < 8; ++j) S.J4[8 * lane + j] = (uint16_t)(p[j] | (p3[j] < (uint32_t)BZF_W ? 0x8000u : 0u));
            }
            __syncwarp();
            // the chain: four symbols per hop while whole hops fit, single symbols for the rest
            uint32_t pos = 0;
            while (need >= 4 && pos < (uint32_t)BZF_W) {
              const uint32_t j4 = S.J4[pos];
              if (!(j4 & 0x8000u)) break;
              pos = j4 & 0x7fffu;
              need -= 4;
            }
            while (need > 0 && pos < (uint32_t)BZF_W) {
              pos += S.EL[pos];
              need--;
            }
            s += pos;
            __syncwarp();
          }
        }
        if (lane == 0) S.ngw[buf] = ngb;
        if (g >= h.n_sel) walk_done = true;  // (the encoder writes as many selectors as the block has groups)
      }
    } else if (warp == 1) {
      if (bt >= 1 && !dec_done) {
        // ---------------- decoder: batch bt - 1, a group per lane ----------------
        const int wb = (bt - 1) & 1;
        const int ngb = S.ngw[wb];
        const int g0 = (bt - 1) * 32;
        bool lbad = false, saw_eob = false;
        unsigned long long my_end = 0;
        int mycnt = 0, hiw = 0;
        uint16_t *const sy = S.syms[wb][lane];
        if (lane < ngb) {
          const int t = S.get_sel(g0 + lane);
          uint64_t sp = S.gstart[wb][lane];
          for (int k = 0; k < 50; ++k) {
            const uint64_t wi = sp >> 5;
            const uint32_t x = __funnelshift_l(ldw(wi + 1), ldw(wi), (uint32_t)(sp & 31u));  // 32 bits from bit sp on
            uint32_t e = S.lut[t][x >> (32 - BZ_LUT_BITS)];
            if ((e & 31u) == 0u) {  // longer than the LUT: the limit / base walk from there on (:747-771)
              int zn = S.minlen[t] > BZ_LUT_BITS + 1 ? S.minlen[t] : BZ_LUT_BITS + 1;
              e = BZF_BADSYM << 5;
              for (; zn <= 20; ++zn) {
                const int32_t zvec = (int32_t)(x >> (32 - zn));
                if (zvec <= S.limit[t][zn]) {
                  const int32_t idx = zvec - S.base[t][zn];
                  if (idx >= 0 && idx < 258) e = ((uint32_t)S.perm[t][idx] << 5) | (uint32_t)zn;
                  break;
                }
              }
            }
            const uint32_t sym = e >> 5;
            if (sym == BZF_BADSYM) {
              lbad = true;
              break;
            }
            sp += e & 31u;
            if (sym == eob) {
              saw_eob = true;
              my_end = sp;
              break;
            }
            mycnt = k + 1;
            if (sym <= 1u) {
              sy[k] = (uint16_t)sym;
              continue;
            }
            // my group against a list that starts as the identity: the symbol becomes a reference to an initial position
            const uint32_t nn = sym - 1u, wn = nn >> 2, bn = nn & 3u;
            for (; hiw <= (int)wn; ++hiw) S.mtf[hiw][lane] = 0x03020100u + 0x04040404u * (uint32_t)hiw;
            const uint32_t top = S.mtf[wn][lane];
            const uint32_t uc = (top >> (8u * bn)) & 0xffu;
            uint32_t carry = uc;
            for (uint32_t w = 0; w < wn; ++w) {
              const uint32_t tw = S.mtf[w][lane];
              S.mtf[w][lane] = (tw << 8) | carry;
              carry = tw >> 24;
            }
            const uint32_t mlow = bn == 3u ? 0xffffffffu : ((1u << (8u * (bn + 1u))) - 1u);
            S.mtf[wn][lane] = (top & ~mlow) | (((top << 8) | carry) & mlow);
            sy[k] = (uint16_t)(0x8000u | uc);
          }
        }
        // the block ends in the lowest lane that met the end-of-block code; what the lanes above it decoded is not the block's
        const unsigned em = __ballot_sync(FULLW, saw_eob);
        const int el = em ? __ffs((int)em) - 1 : 31;
        const int ngb_eff = em ? el + 1 : ngb;
        if (__ballot_sync(FULLW, lbad && lane <= el && lane < ngb_eff) != 0u) {
          if (lane == 0) S.redo = 1;
        } else if (!em && ngb < 32) {
          if (lane == 0) S.redo = 1;  // the selectors ran out before the end-of-block code
        }
        __syncwarp();
        // the real list, group by group: resolve the group's references, then list'[i] = list[P[i]]
        for (int gi = 0; gi < ngb_eff; ++gi) {
          const int cg = __shfl_sync(FULLW, mycnt, gi);
          const int hib = __shfl_sync(FULLW, hiw, gi) * 4;  // bytes of the group's list that may have moved
          for (int k = lane; k < cg; k += 32) {
            const uint32_t v = S.syms[wb][gi][k];
            if (v & 0x8000u) S.syms[wb][gi][k] = (uint16_t)(0x8000u | S.cur[v & 0xffu]);
          }
          uint8_t nv[8];
#pragma unroll
          for (int m = 0; m < 8; ++m) {
            const int i = lane + 32 * m;
            nv[m] = 0;
            if (i < hib) nv[m] = S.cur[(S.mtf[i >> 2][gi] >> (8 * (i & 3))) & 0xffu];
          }
          __syncwarp();
#pragma unroll
          for (int m = 0; m < 8; ++m) {
            const int i = lane + 32 * m;
            if (i < hib) S.cur[i] = nv[m];
          }
          __syncwarp();
        }
        if (lane < 32) S.cnt[wb][lane] = (uint8_t)mycnt;
        if (lane == 0) {
          S.ng[wb] = ngb_eff;
          S.last[wb] = em ? 1 : 0;
        }
        if (em && lane == el) S.end_bit = my_end;
      }
    } else {
      if (bt >= 2) {
        // ---------------- recorder: batch bt - 2 (:276-388) ----------------
        // The batch's symbols as ONE stream, 32 at a time.  A run symbol adds (sym + 1) << its index in the run; a symbol
        // that is not a run symbol closes the run in front of it (one record, written at the position the run started at)
        // and makes a record of its own.  Everything a lane needs -- its index in the run, the run's value, records and
        // block positions in front of it -- is a ballot, a 5-step scan and two shuffles away.
        const int wb = bt & 1;  // (bt - 2) & 1
        const int ngb = S.ng[wb];
        const bool lastb = prev_last;
        bool lbad = false;
        const int total = ngb ? 50 * (ngb - 1) + (int)S.cnt[wb][ngb - 1] : 0;  // only the block's last group is short
        const uint16_t *const flat = &S.syms[wb][0][0];
        for (int base = 0; base < total; base += 32) {
          const int i = base + lane;
          const bool valid = i < total;
          const uint32_t v = valid ? (uint32_t)flat[i] : 0xffffu;
          const bool isrun = valid && v <= 1u, isnr = valid && v > 1u;
          const unsigned NR = __ballot_sync(FULLW, isnr);
          const unsigned below = NR & ((1u << lane) - 1u);
          const int q = below ? 31 - __clz((int)below) : -1;  // the last symbol below me that is not a run symbol
          const uint32_t before = q < 0 ? st_n + (uint32_t)lane : (uint32_t)(lane - q - 1);  // run symbols right in front of me
          uint32_t a = 0;
          if (isrun) {
            if (before > 20u) lbad = true;  // N >= 2*1024*1024 (:291)
            else a = (v + 1u) << before;
          }
          uint32_t pa = a;  // inclusive scan
#pragma unroll
          for (int dlt = 1; dlt < 32; dlt <<= 1) {
            const uint32_t tsh = __shfl_up_sync(FULLW, pa, dlt);
            if (lane >= dlt) pa += tsh;
          }
          const uint32_t pa_q = __shfl_sync(FULLW, pa, q < 0 ? 0 : q);
          const uint32_t fv = __shfl_sync(FULLW, v & 0xffu, q < 0 ? 0 : q);
          const bool hasrun = isnr && before != 0u;
          // The bytes go straight to the block's byte array (what k_bz2_expand made of the records); only a LONG run stays a
          // record for that kernel (its fill would hold a lane, and the warp with it, for up to 2 M iterations).
          const uint32_t runval = q < 0 ? st_v + pa : pa - pa_q;  // (a is 0 in a closing lane: pa is the sum over what lies below it)
          const bool longrun = hasrun && runval > BZF_INLINE_RUN;
          const unsigned LR = __ballot_sync(FULLW, longrun);
          if (isnr) {
            const uint32_t pos_sym = st_nblock + st_v + pa + (uint32_t)__popc(below);
            if (pos_sym >= lim) {  // (:313-316, :326-329)
              lbad = true;
            } else {
              if (hasrun) {
                const uint32_t rb = S.seq2unseq[q < 0 ? st_front : fv];
                if (longrun) {
                  const uint32_t r = st_nrec + (uint32_t)__popc(LR & ((1u << lane) - 1u));
                  rv[r] = (runval << 8) | rb;
                  rp[r] = pos_sym - runval;
                } else {
                  for (uint32_t z = pos_sym - runval; z < pos_sym; ++z) s8[z] = (uint8_t)rb;
                }
              }
              s8[pos_sym] = S.seq2unseq[v & 0xffu];
            }
          }
          const int nvalid = total - base < 32 ? total - base : 32;
          const uint32_t pa_last = __shfl_sync(FULLW, pa, 31);
          if (NR) {
            const int ql = 31 - __clz((int)NR);
            const uint32_t pa_ql = __shfl_sync(FULLW, pa, ql);
            st_nrec += (uint32_t)__popc(LR);
            st_nblock += st_v + pa_ql + (uint32_t)__popc(NR);
            st_v = pa_last - pa_ql;
            st_n = (uint32_t)(nvalid - 1 - ql);
            st_front = __shfl_sync(FULLW, v & 0xffu, ql);
          } else {
            st_v += pa_last;
            st_n += (uint32_t)nvalid;
          }
        }
        if (lastb && st_n) {  // the run that the end-of-block code closes (:306-321)
          if (st_n > 21u || st_nblock + st_v > lim) {
            lbad = true;
          } else if (st_v > BZF_INLINE_RUN) {
            if (lane == 0) {
              rv[st_nrec] = (st_v << 8) | S.seq2unseq[st_front];
              rp[st_nrec] = st_nblock;
            }
            st_nrec++;
          } else {
            if ((uint32_t)lane < st_v) s8[st_nblock + lane] = S.seq2unseq[st_front];
          }
          st_nblock += st_v;
          st_n = 0;
          st_v = 0;
        }
        if (__any_sync(FULLW, lbad) && lane == 0) S.redo = 1;
      }
    }
    __syncthreads();
    const bool redo = S.redo != 0;
    const bool cur_last = bt >= 1 && !dec_done && S.last[(bt - 1) & 1] != 0;
    __syncthreads();
    if (redo) {
      if (tid == 0) status[b] = BZ_REDO;
      return;
    }
    if (prev_last) break;  // the recorder has just finished the block's last batch
    prev_last = cur_last;
    if (cur_last) dec_done = true;
  }
  if (tid == 64) {
    const unsigned long long endp = S.end_bit;
    if (h.optr >= st_nblock || endp > total_bits) {  // (:399-402), a read past the end: the exact kernel's verdicts
      status[b] = BZ_REDO;
    } else {
      n_rec[b] = st_nrec;
      nblock_out[b] = st_nblock;
      orig_ptr[b] = h.optr;
      randomised[b] = h.rnd;
      end_bit[b] = endp;
      status[b] = BZ_OK;
      if (fast_flag) fast_flag[b] = 1;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// K7 for damaged blocks.  _getMtfVal (:732-772) returns -1 for a code that fits no table entry, for a 21-bit code and when
// the selectors run out; only its FIRST call is checked (:273-275).  Later on the -1 is used as a symbol: nn = -2 picks the
// byte two places in front of the MTF list's first block (:331-347) and decoding goes on -- until the block fills up (-1),
// the input ends (RangeError) or, often enough, an end-of-block code turns up and the block decodes to SOMETHING.  What
// that byte is depends on the reference's own list layout (4096 bytes, 16 blocks of 16 that creep downwards and are
// re-packed when the first reaches 0), so this path keeps exactly that layout.  One thread per block; damaged data only.
// ---------------------------------------------------------------------------------------------
struct BzLitSmem {
  int32_t limit[6][24];
  int32_t base[6][24];
  uint16_t perm[6][258];
  uint8_t len[6][258];
  uint8_t minlen[6];
  uint8_t selector[BZ_MAX_SEL + 2];
  uint8_t seq2unseq[256];
  uint8_t mtfa[4096];
  int32_t mtfbase[16];
};

__global__ void __launch_bounds__(32)
k_bz2_entropy_literal(const uint32_t *__restrict__ words, uint64_t n_bytes, const unsigned long long *__restrict__ blk_bit,
                      const uint32_t *__restrict__ list, uint32_t n_list, uint32_t nblock_max, uint32_t *__restrict__ rec_val,
                      uint32_t *__restrict__ rec_pos, uint32_t *__restrict__ n_rec, uint32_t *__restrict__ nblock_out,
                      unsigned long long *__restrict__ end_bit, int32_t *__restrict__ status,
                      const unsigned long long *__restrict__ blk_end, const uint32_t *__restrict__ blk_lim) {
  __shared__ BzLitSmem S;
  if (blockIdx.x >= n_list || threadIdx.x != 0) return;
  const uint32_t b = list[blockIdx.x];
  const uint64_t total_bits = blk_end ? blk_end[b] : n_bytes * 8;
  const uint32_t lim = blk_lim ? blk_lim[b] : nblock_max;  // the block's own limit; nblock_max is the stride of its arrays
  BzBits br;
  br.w = words;
  br.set_end(total_bits);
  br.seek(blk_bit[b] + 48 + 32 + 1);  // the randomised bit is K7's to report
  uint32_t optr = br.get(8);
  optr = (optr << 8) | br.get(8);
  optr = (optr << 8) | br.get(8);
  int err = 0, n_in_use = 0;
  for (int i = 0; i < 256; ++i) S.seq2unseq[i] = 0;  // Uint8List(256): entries past numInUse read 0
  {
    const uint32_t used16 = br.get(16);
    for (int i = 0; i < 16; ++i)
      if (used16 & (0x8000u >> i)) {
        const uint32_t m = br.get(16);
        for (int j = 0; j < 16; ++j)
          if (m & (0x8000u >> j)) S.seq2unseq[n_in_use++] = (uint8_t)(i * 16 + j);
      }
  }
  if (n_in_use == 0) err = BZ_DATA;
  const int alpha = n_in_use + 2;
  int n_groups = 0, n_sel = 0;
  if (!err) {
    n_groups = (int)br.get(3);
    if (n_groups < 2 || n_groups > 6) err = BZ_DATA;
  }
  if (!err) {
    n_sel = (int)br.get(15);
    if (n_sel < 1) err = BZ_DATA;
  }
  if (!err) {  // selectors (:160-186)
    uint8_t pos[6];
    for (int i = 0; i < n_groups; ++i) pos[i] = (uint8_t)i;
    for (int i = 0; i < n_sel && !err; ++i) {
      int j = 0;
      while (br.get(1)) {
        if (++j >= n_groups) {
          err = BZ_DATA;
          break;
        }
      }
      if (err) break;
      if (i >= BZ_MAX_SEL) {
        err = BZ_THROW;
        break;
      }
      const uint8_t tmp = pos[j];
      for (int v = j; v > 0; --v) pos[v] = pos[v - 1];
      pos[0] = tmp;
      S.selector[i] = tmp;
      if (br.bitpos() > total_bits) err = BZ_THROW;
    }
  }
  for (int t = 0; t < n_groups && !err; ++t) {  // code lengths (:189-212)
    int c = (int)br.get(5);
    for (int i = 0; i < alpha && !err; ++i) {
      for (;;) {
        if (c < 1 || c > 20) {
          err = BZ_DATA;
          break;
        }
        if (br.get(1) == 0) break;
        c += br.get(1) == 0 ? 1 : -1;
      }
      S.len[t][i] = (uint8_t)c;
    }
    if (!err && br.bitpos() > total_bits) err = BZ_THROW;
  }
  for (int t = 0; t < n_groups && !err; ++t) {  // _hbCreateDecodeTables (:774-813)
    int mn = 32, mx = 0;
    for (int i = 0; i < alpha; ++i) {
      const int l = S.len[t][i];
      mx = l > mx ? l : mx;
      mn = l < mn ? l : mn;
    }
    S.minlen[t] = (uint8_t)mn;
    for (int i = 0; i < 258; ++i) S.perm[t][i] = 0;
    int pp = 0;
    for (int l = mn; l <= mx; ++l)
      for (int j = 0; j < alpha; ++j)
        if (S.len[t][j] == l) S.perm[t][pp++] = (uint16_t)j;
    int32_t *base = S.base[t], *limit = S.limit[t];
    for (int i = 0; i < 24; ++i) base[i] = limit[i] = 0;
    for (int i = 0; i < alpha; ++i) base[S.len[t][i] + 1]++;
    for (int i = 1; i < 23; ++i) base[i] += base[i - 1];
    int32_t vec = 0;
    for (int l = mn; l <= mx; ++l) {
      vec += base[l + 1] - base[l];
      limit[l] = vec - 1;
      vec <<= 1;
    }
    for (int l = mn + 1; l <= mx; ++l) base[l] = ((limit[l - 1] + 1) << 1) - base[l];
  }

  uint32_t nrec = 0, nblock = 0;
  if (!err) {
    for (int i = 0; i < 4096; ++i) S.mtfa[i] = 0;  // Uint8List(4096)
    {
      int kk = 4095;
      for (int ii = 15; ii >= 0; --ii) {
        for (int jj = 15; jj >= 0; --jj) S.mtfa[kk--] = (uint8_t)(ii * 16 + jj);
        S.mtfbase[ii] = kk + 1;
      }
    }
    const int eob = n_in_use + 1;
    uint32_t *rv = rec_val + (size_t)b * nblock_max;
    uint32_t *rp = rec_pos + (size_t)b * nblock_max;
    int gpos = 0, gno = -1, gsel = 0;
    auto get_mtf_val = [&]() -> int {  // (:732-772), -1 and all
      if (gpos == 0) {
        gno++;
        if (gno >= n_sel) return -1;
        gpos = 50;
        gsel = S.selector[gno];
      }
      gpos--;
      int zn = S.minlen[gsel];
      int32_t zvec = (int32_t)br.get(zn);
      for (;;) {
        if (zn > 20) return -1;
        if (zvec <= S.limit[gsel][zn]) break;
        zn++;
        zvec = (zvec << 1) | (int32_t)br.get(1);
      }
      const int32_t idx = zvec - S.base[gsel][zn];
      if (idx < 0 || idx >= 258) return -1;
      return (int)S.perm[gsel][idx];
    };
    int next = get_mtf_val();
    if (next < 0) err = BZ_DATA;
    while (!err) {
      if (br.bitpos() > total_bits) {  // the read that produced `next` went past the end: RangeError there and then
        err = BZ_THROW;
        break;
      }
      if (next == eob) break;
      if (next == 0 || next == 1) {
        long long es = -1, n = 1;
        do {
          if (n >= 2 * 1024 * 1024) {
            err = BZ_DATA;
            break;
          }
          es += next == 0 ? n : 2 * n;
          n *= 2;
          next = get_mtf_val();
        } while ((next == 0 || next == 1) && br.bitpos() <= total_bits);
        if (err) break;
        if (br.bitpos() > total_bits) continue;  // -> BZ_THROW at the top
        es++;
        if ((long long)nblock + es > (long long)lim) {  // (:313-316): fills up to the limit, then -1
          err = BZ_DATA;
          break;
        }
        rv[nrec] = ((uint32_t)es << 8) | S.seq2unseq[S.mtfa[S.mtfbase[0]]];
        rp[nrec] = nblock;
        nrec++;
        nblock += (uint32_t)es;
        continue;
      }
      if (nblock >= lim) {
        err = BZ_DATA;
        break;
      }
      int nn = next - 1;  // next == -1: nn = -2
      uint32_t uc;
      if (nn < 16) {
        const int pp = S.mtfbase[0];
        if (pp + nn < 0) {  // _mtfa[-1]: RangeError
          err = BZ_THROW;
          break;
        }
        uc = S.mtfa[pp + nn];
        for (; nn > 0; --nn) S.mtfa[pp + nn] = S.mtfa[pp + nn - 1];
        S.mtfa[pp] = (uint8_t)uc;  // nn = -2: the stale byte simply becomes the list's front entry
      } else {
        int lno = nn >> 4;
        int pp = S.mtfbase[lno] + (nn & 15);
        uc = S.mtfa[pp];
        for (; pp > S.mtfbase[lno]; --pp) S.mtfa[pp] = S.mtfa[pp - 1];
        S.mtfbase[lno]++;
        for (; lno > 0; --lno) {
          S.mtfbase[lno]--;
          S.mtfa[S.mtfbase[lno]] = S.mtfa[S.mtfbase[lno - 1] + 15];
        }
        S.mtfbase[0]--;
        S.mtfa[S.mtfbase[0]] = (uint8_t)uc;
        if (S.mtfbase[0] == 0) {  // re-pack at the top (:364-377)
          int kk = 4095;
          for (int ii = 15; ii >= 0; --ii) {
            for (int jj = 15; jj >= 0; --jj) S.mtfa[kk--] = S.mtfa[S.mtfbase[ii] + jj];
            S.mtfbase[ii] = kk + 1;
          }
        }
      }
      rv[nrec] = (1u << 8) | S.seq2unseq[uc];
      rp[nrec] = nblock;
      nrec++;
      nblock++;
      next = get_mtf_val();
    }
    if (!err && optr >= nblock) err = BZ_DATA;
  }
  if (br.bitpos() > total_bits) err = BZ_THROW;
  n_rec[b] = nrec;
  nblock_out[b] = nblock;
  end_bit[b] = br.bitpos();
  status[b] = err;
}

// ---------------------------------------------------------------------------------------------
// records -> bytes (the low byte of tt[] in the reference, bzip2_decoder.dart:318,380)
// grid.y = block index in the chain list
// ---------------------------------------------------------------------------------------------
struct BzChain {           // one entry per block that is on the validated chain
  uint32_t cand;           // index into the K7 per-candidate arrays
  uint32_t nblock;
  uint32_t n_rec;
  uint32_t orig_ptr;
  uint32_t flags;          // bit 0: randomised block; bit 1: first block of its stream (its output starts at out_lo)
  uint32_t pad_;
  unsigned long long out_lo, out_hi;  // the stream's output slot [out_lo, out_hi) in `out` (bytes from out_hi on are dropped)
};

__global__ void __launch_bounds__(256)
k_bz2_expand(const BzChain *__restrict__ chain, const uint32_t *__restrict__ rec_val, const uint32_t *__restrict__ rec_pos,
             uint32_t nblock_max, uint8_t *__restrict__ sym8) {
  const BzChain c = chain[blockIdx.y];
  const uint32_t *rv = rec_val + (size_t)c.cand * nblock_max, *rp = rec_pos + (size_t)c.cand * nblock_max;
  uint8_t *dst = sym8 + (size_t)c.cand * nblock_max;  // (by candidate slot: k_bz2_entropy_fast writes its blocks' bytes there itself)
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < c.n_rec; r += gridDim.x * blockDim.x) {
    uint32_t v = rv[r], p = rp[r];
    uint8_t ch = (uint8_t)v;
    uint32_t n = v >> 8;
    for (uint32_t j = 0; j < n; ++j) dst[p + j] = ch;
  }
}

// per-warp-chunk (1024 positions) histograms
constexpr int BZ_CHUNK = 1024;
__global__ void __launch_bounds__(128)
k_bz2_chunk_hist(const BzChain *__restrict__ chain, const uint8_t *__restrict__ sym8, uint32_t nblock_max,
                 uint32_t chunks_max, uint32_t *__restrict__ chist) {
  __shared__ uint32_t h[4][256];
  const BzChain c = chain[blockIdx.y];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t chunk = blockIdx.x * 4 + warp;
  for (int i = lane; i < 256; i += 32) h[warp][i] = 0;
  __syncwarp();
  const uint32_t lo = chunk * BZ_CHUNK;
  const uint8_t *src = sym8 + (size_t)c.cand * nblock_max;
  if (lo < c.nblock) {
    uint32_t hi = min(lo + BZ_CHUNK, c.nblock);
    for (uint32_t i = lo + lane; i < hi; i += 32) atomicAdd(&h[warp][src[i]], 1u);
  }
  __syncwarp();
  if (chunk < chunks_max) {
    uint32_t *dst = chist + ((size_t)blockIdx.y * chunks_max + chunk) * 256;
    for (int i = lane; i < 256; i += 32) dst[i] = h[warp][i];
  }
}

// cftab (:407-432) + per-chunk start offsets: chist[chunk][c] becomes the first T index chunk `chunk` uses for byte c
__global__ void __launch_bounds__(256)
k_bz2_chunk_scan(const BzChain *__restrict__ chain, uint32_t chunks_max, uint32_t *__restrict__ chist) {
  __shared__ uint32_t tot[256];
  const BzChain c = chain[blockIdx.x];
  const uint32_t nchunks = (c.nblock + BZ_CHUNK - 1) / BZ_CHUNK;
  uint32_t *base = chist + (size_t)blockIdx.x * chunks_max * 256;
  const int v = threadIdx.x;
  uint32_t s = 0;
  for (uint32_t k = 0; k < nchunks; ++k) s += base[(size_t)k * 256 + v];
  tot[v] = s;
  __syncthreads();
  if (v == 0) {
    uint32_t run = 0;
    for (int i = 0; i < 256; ++i) {
      uint32_t t = tot[i];
      tot[i] = run;
      run += t;
    }
  }
  __syncthreads();
  uint32_t run = tot[v];
  for (uint32_t k = 0; k < nchunks; ++k) {
    uint32_t t = base[(size_t)k * 256 + v];
    base[(size_t)k * 256 + v] = run;
    run += t;
  }
}

// T^-1 (:435-439): tt[cftab[uc]++] |= i << 8 as a stable counting sort, one warp per 1024-position chunk
__global__ void __launch_bounds__(128)
k_bz2_build_tt(const BzChain *__restrict__ chain, const uint8_t *__restrict__ sym8, uint32_t nblock_max,
               uint32_t chunks_max, const uint32_t *__restrict__ chist, uint32_t *__restrict__ tt) {
  __shared__ uint32_t cnt[4][256];
  const BzChain c = chain[blockIdx.y];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t chunk = blockIdx.x * 4 + warp;
  const uint32_t lo = chunk * BZ_CHUNK;
  if (lo >= c.nblock) return;
  const uint32_t *cb = chist + ((size_t)blockIdx.y * chunks_max + chunk) * 256;
  for (int i = lane; i < 256; i += 32) cnt[warp][i] = cb[i];
  __syncwarp();
  const uint8_t *src = sym8 + (size_t)c.cand * nblock_max;
  uint32_t *T = tt + (size_t)blockIdx.y * nblock_max;
  const uint32_t hi = min(lo + BZ_CHUNK, c.nblock);
  for (uint32_t g = lo; g < hi; g += 32) {
    const uint32_t i = g + lane;
    const bool act = i < hi;
    const uint32_t ch = act ? src[i] : 0x100u + lane;  // inactive lanes never match anyone
    const unsigned m = __match_any_sync(0xffffffffu, ch);
    const uint32_t rank = __popc(m & ((1u << lane) - 1u));
    uint32_t basev = act ? cnt[warp][ch] : 0;
    __syncwarp();
    if (act) {
      // tt[j] keeps ITS OWN byte in bits 0-7 (written at :318/:380) and receives i in the upper bits (:437)
      const uint32_t j = basev + rank;
      T[j] = (i << 8) | src[j];
      if (rank == 0) cnt[warp][ch] = basev + __popc(m);
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------
// the cycle walk (:610-727 reads tPos = tt[tPos] one byte at a time): cut at splitters, walk in parallel
// ---------------------------------------------------------------------------------------------
constexpr uint32_t BZ_SPLIT = 4096;

struct BzWalkGeom {
  uint32_t stride, kb, tpos0, start_id;
};
__device__ __forceinline__ BzWalkGeom bz_geom(const BzChain &c, const uint32_t *T) {
  BzWalkGeom g;
  g.stride = (c.nblock + BZ_SPLIT - 1) / BZ_SPLIT;
  if (g.stride == 0) g.stride = 1;
  g.kb = (c.nblock + g.stride - 1) / g.stride;
  g.tpos0 = T[c.orig_ptr] >> 8;  // (:443)
  g.start_id = (g.tpos0 % g.stride == 0) ? g.tpos0 / g.stride : g.kb;
  return g;
}

// The walk is ONE pass (it was a length pass and an emit pass, both bound by the memory system: every step is a 4-byte read at a random place of a 2.1 GB table, i.e. one 32-byte sector from HBM per
// output byte).  A segment's place in the output is known only once every segment's length is, so the bytes go to a SLOT
// per segment first (BZ_SLOT bytes: segment lengths are geometric with mean nblock / 4096 ~ 220, so ~1 % overflow) and a
// second, coalesced pass moves them (k_bz2_walk_emit); a segment longer than its slot records where the walk stood at the
// slot's end and that kernel goes on from there.  Segments come off a counter (a thread whose segment ends takes the next
// one, of any block) -- measured neutral against one segment per thread.
#ifndef BZ_SLOT_BYTES
#define BZ_SLOT_BYTES 1024  // (the emulation tier builds with 64, so that most segments overflow their slot there)
#endif
constexpr uint32_t BZ_SLOT = BZ_SLOT_BYTES;
__global__ void __launch_bounds__(256)
k_bz2_walk_len(const BzChain *__restrict__ chain, uint32_t n_chain, const uint32_t *__restrict__ tt, uint32_t nblock_max,
               uint32_t *__restrict__ seg_len, uint32_t *__restrict__ seg_next, uint32_t *__restrict__ seg_resume,
               uint8_t *__restrict__ slots, uint32_t *__restrict__ ctr) {
  const uint32_t per = BZ_SPLIT + 2, total = n_chain * per;
  for (;;) {
    const uint32_t item = atomicAdd(ctr, 1u);
    if (item >= total) return;
    const uint32_t bi = item / per, j = item - bi * per;
    const BzChain c = chain[bi];
    if (c.nblock == 0) continue;
    const uint32_t *T = tt + (size_t)bi * nblock_max;
    const BzWalkGeom g = bz_geom(c, T);
    if (j > g.kb) continue;
    uint32_t *sl = seg_len + (size_t)bi * per, *sn = seg_next + (size_t)bi * per;
    if (j == g.kb && g.start_id != g.kb) {  // the start coincides with a regular splitter
      sl[j] = 0;
      sn[j] = g.start_id;
      continue;
    }
    uint32_t cur = (j == g.kb) ? g.tpos0 : j * g.stride;
    uint8_t *slot = slots + (size_t)item * BZ_SLOT;
    uint32_t n = 0;
    do {
      const uint32_t t = T[cur];
      if (n < BZ_SLOT) slot[n] = (uint8_t)t;
      else if (n == BZ_SLOT) seg_resume[item] = cur;  // (the byte of this step is still to be written)
      cur = t >> 8;
      n++;
    } while (!(cur % g.stride == 0 || cur == g.tpos0) && n < c.nblock);
    sl[j] = n;
    sn[j] = (cur == g.tpos0) ? g.start_id : cur / g.stride;
  }
}

// Order of the segments along the cycle, one CTA per block: the segment table (<= 4097 entries) is staged in shared memory,
// one thread follows it there (a chain of shared-memory reads instead of global ones), the CTA writes the offsets back.
// T (built by a stable counting sort) is always a permutation, so the walk from tPos0 returns to tPos0; for a PERIODIC
// block (e.g. "abab...", or long runs after RLE1) that happens after cycle_len < nblock steps and the reference simply
// keeps going round (bzip2_decoder.dart:648-650): raw[i] = raw[i mod cycle_len].
__global__ void __launch_bounds__(128)
k_bz2_walk_order(const BzChain *__restrict__ chain, uint32_t n_chain, const uint32_t *__restrict__ tt,
                 uint32_t nblock_max, const uint32_t *__restrict__ seg_len,
                 const uint32_t *__restrict__ seg_next, uint32_t *__restrict__ seg_off,
                 int32_t *__restrict__ irregular, uint32_t *__restrict__ cycle_len) {
  __shared__ uint32_t s_len[BZ_SPLIT + 2], s_off[BZ_SPLIT + 2];
  __shared__ uint16_t s_next[BZ_SPLIT + 2];
  const uint32_t bi = blockIdx.x;
  if (bi >= n_chain) return;
  const BzChain c = chain[bi];
  if (threadIdx.x == 0) {
    irregular[bi] = 0;
    cycle_len[bi] = c.nblock;
  }
  if (c.nblock == 0) return;
  const uint32_t *T = tt + (size_t)bi * nblock_max;
  const BzWalkGeom g = bz_geom(c, T);
  const uint32_t *sl = seg_len + (size_t)bi * (BZ_SPLIT + 2), *sn = seg_next + (size_t)bi * (BZ_SPLIT + 2);
  uint32_t *so = seg_off + (size_t)bi * (BZ_SPLIT + 2);
  for (uint32_t j = threadIdx.x; j <= g.kb; j += blockDim.x) {
    s_len[j] = sl[j];
    const uint32_t nx = sn[j];
    s_next[j] = (uint16_t)(nx > 0xffffu ? 0xffffu : nx);
    s_off[j] = 0xffffffffu;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t seg = g.start_id, off = 0, visited = 0;
    while (off < c.nblock) {
      if (seg > g.kb) {
        irregular[bi] = 1;
        break;
      }
      if (s_off[seg] != 0xffffffffu) {  // back at the start: the cycle is shorter than the block
        if (seg != g.start_id) irregular[bi] = 1;
        cycle_len[bi] = off;
        break;
      }
      if (s_len[seg] == 0 || ++visited > g.kb + 1) {
        irregular[bi] = 1;
        break;
      }
      s_off[seg] = off;
      off += s_len[seg];
      seg = s_next[seg];
    }
  }
  __syncthreads();
  for (uint32_t j = threadIdx.x; j <= g.kb; j += blockDim.x) so[j] = s_off[j];
}

// periodic blocks: repeat the cycle
__global__ void __launch_bounds__(256)
k_bz2_periodic_fill(const BzChain *__restrict__ chain, const uint32_t *__restrict__ cycle_len, uint32_t nblock_max,
                    uint8_t *__restrict__ raw) {
  const BzChain c = chain[blockIdx.y];
  const uint32_t cl = cycle_len[blockIdx.y];
  if (cl == 0 || cl >= c.nblock) return;
  uint8_t *dst = raw + (size_t)blockIdx.y * nblock_max;
  for (uint32_t i = cl + blockIdx.x * blockDim.x + threadIdx.x; i < c.nblock; i += gridDim.x * blockDim.x) dst[i] = dst[i % cl];
}

// one WARP per segment: the slot's bytes move to the segment's place in the block (coalesced); lane 0 walks on for the part
// of a segment that did not fit its slot
__global__ void __launch_bounds__(256)
k_bz2_walk_emit(const BzChain *__restrict__ chain, uint32_t n_chain, const uint32_t *__restrict__ tt, uint32_t nblock_max,
                const uint32_t *__restrict__ seg_len, const uint32_t *__restrict__ seg_off, const uint32_t *__restrict__ seg_resume,
                const uint8_t *__restrict__ slots, uint8_t *__restrict__ raw) {
  const uint32_t per = BZ_SPLIT + 2, total = n_chain * per;
  const uint32_t lane = threadIdx.x & 31u, wpb = blockDim.x >> 5;
  for (uint32_t item = blockIdx.x * wpb + (threadIdx.x >> 5); item < total; item += gridDim.x * wpb) {
    const uint32_t bi = item / per, j = item - bi * per;
    const BzChain c = chain[bi];
    if (c.nblock == 0) continue;
    const uint32_t stride0 = (c.nblock + BZ_SPLIT - 1) / BZ_SPLIT, stride = stride0 ? stride0 : 1u;
    if (j > (c.nblock + stride - 1) / stride) continue;  // (> kb)
    const uint32_t off = seg_off[item];
    if (off == 0xffffffffu) continue;
    uint32_t n = seg_len[item];
    if (off + n > c.nblock) n = c.nblock - off;
    uint8_t *dst = raw + (size_t)bi * nblock_max + off;
    const uint8_t *slot = slots + (size_t)item * BZ_SLOT;
    const uint32_t m = n < BZ_SLOT ? n : BZ_SLOT;
    // bytes up to the first 4-byte boundary of the destination, then whole words (the slot is read through two aligned
    // words and a funnel shift: its base is aligned, the offset inside it is not), then the rest
    const uint32_t headb = min(m, (uint32_t)((4u - (uint32_t)(reinterpret_cast<uintptr_t>(dst) & 3u)) & 3u));
    if (lane < headb) dst[lane] = slot[lane];
    const uint32_t nwords = (m - headb) >> 2;
    const uint32_t *s32 = reinterpret_cast<const uint32_t *>(slot);
    uint32_t *d32 = reinterpret_cast<uint32_t *>(dst + headb);
    const uint32_t sh = (headb & 3u) * 8u;
    for (uint32_t w = lane; w < nwords; w += 32u) {
      const uint32_t si = (headb >> 2) + w;  // (headb < 4: 0)
      d32[w] = sh ? __funnelshift_r(s32[si], s32[si + 1u], sh) : s32[si];  // (no read behind the slot's last word)
    }
    const uint32_t done = headb + 4u * nwords;
    if (done + lane < m) dst[done + lane] = slot[done + lane];
    if (n > BZ_SLOT && lane == 0u) {
      const uint32_t *T = tt + (size_t)bi * nblock_max;
      uint32_t cur = seg_resume[item];
      for (uint32_t i = BZ_SLOT; i < n; ++i) {
        const uint32_t t = T[cur];
        dst[i] = (uint8_t)t;
        cur = t >> 8;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// RLE1 (:610-727): 4 equal bytes are followed by a count byte.  State s = number of equal data bytes ending
// at the previous position (1..4), 0 = fresh (start, or the previous byte was a count).  Input per position:
// eq = (raw[i] == raw[i-1]).  Transition: 4 -> 0 (this byte is a COUNT); 0 -> 1; 1..3 -> eq ? s+1 : 1.
// A map over the 5 states is packed 3 bits per state; maps compose associatively, so the state in front of
// every slice comes from a scan.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t rle_step(uint32_t s, bool eq) { return s == 4 ? 0u : (s == 0 ? 1u : (eq ? s + 1u : 1u)); }
__device__ __forceinline__ uint32_t map_identity() { return 0u | (1u << 3) | (2u << 6) | (3u << 9) | (4u << 12); }
__device__ __forceinline__ uint32_t map_get(uint32_t m, uint32_t s) { return (m >> (3 * s)) & 7u; }
__device__ __forceinline__ uint32_t map_compose(uint32_t first, uint32_t then) {  // then(first(s))
  uint32_t r = 0;
#pragma unroll
  for (uint32_t s = 0; s < 5; ++s) r |= map_get(then, map_get(first, s)) << (3 * s);
  return r;
}

// bzip2 CRC helpers (MSB-first, poly 0x04c11db7).  mulmod: polynomial product mod P of two 32-bit residues.
__device__ __forceinline__ uint32_t bzcrc_mulmod(uint32_t a, uint32_t b) {
  uint32_t r = 0;
#pragma unroll 4
  for (int i = 0; i < 32; ++i) {
    if (b & 0x80000000u) r ^= a;  // processed from the top: Horner in x
    b <<= 1;
    if (i != 31) r = (r << 1) ^ ((r & 0x80000000u) ? 0x04c11db7u : 0u);
  }
  return r;
}
// x^(8n) mod P
__device__ uint32_t bzcrc_xpow8(uint64_t n) {
  uint32_t result = 1u;           // x^0
  uint32_t sq = 0x00000100u;      // x^8
  while (n) {
    if (n & 1) result = bzcrc_mulmod(result, sq);
    sq = bzcrc_mulmod(sq, sq);
    n >>= 1;
  }
  return result;
}

constexpr int BZ_RLE_THREADS = 1024;

// pass 1: per-block decoded size
__global__ void __launch_bounds__(BZ_RLE_THREADS)
k_bz2_rle_count(const BzChain *__restrict__ chain, const uint8_t *__restrict__ raw, uint32_t nblock_max,
                uint32_t *__restrict__ slice_state, uint32_t *__restrict__ slice_out, unsigned long long *__restrict__ block_out,
                const uint32_t *__restrict__ cycle_len, int32_t *__restrict__ irregular) {
  __shared__ uint32_t sm_map[BZ_RLE_THREADS];
  __shared__ uint32_t sm_cnt[BZ_RLE_THREADS];
  const BzChain c = chain[blockIdx.x];
  if (c.flags & 1u) return;  // randomised: k_bz2_rand
  const uint8_t *src = raw + (size_t)blockIdx.x * nblock_max;
  const uint32_t t = threadIdx.x;
  const uint32_t per = (c.nblock + BZ_RLE_THREADS - 1) / BZ_RLE_THREADS;
  const uint32_t lo = min(t * per, c.nblock), hi = min(lo + per, c.nblock);
  // slice map
  uint32_t m = map_identity();
  {
    uint32_t st[5] = {0, 1, 2, 3, 4};
    uint8_t prev = lo > 0 ? src[lo - 1] : 0;
    for (uint32_t i = lo; i < hi; ++i) {
      uint8_t x = src[i];
      bool eq = (i > 0) && x == prev;
#pragma unroll
      for (int k = 0; k < 5; ++k) st[k] = rle_step(st[k], eq);
      prev = x;
    }
    m = st[0] | (st[1] << 3) | (st[2] << 6) | (st[3] << 9) | (st[4] << 12);
  }
  sm_map[t] = m;
  __syncthreads();
  // exclusive scan of maps (Hillis-Steele, order preserving)
  for (int d = 1; d < BZ_RLE_THREADS; d <<= 1) {
    uint32_t mine = sm_map[t];
    uint32_t left = t >= (uint32_t)d ? sm_map[t - d] : map_identity();
    __syncthreads();
    sm_map[t] = map_compose(left, mine);
    __syncthreads();
  }
  const uint32_t incl_prev = t > 0 ? sm_map[t - 1] : map_identity();
  uint32_t s = map_get(incl_prev, 0);  // state in front of the slice, from the fresh state at the block start
  slice_state[(size_t)blockIdx.x * BZ_RLE_THREADS + t] = s;
  // slice output size
  uint32_t outn = 0;
  {
    uint8_t prev = lo > 0 ? src[lo - 1] : 0;
    for (uint32_t i = lo; i < hi; ++i) {
      uint8_t x = src[i];
      bool eq = (i > 0) && x == prev;
      outn += (s == 4) ? (uint32_t)x : 1u;
      s = rle_step(s, eq);
      prev = x;
    }
  }
  sm_cnt[t] = outn;
  __syncthreads();
  for (int d = 1; d < BZ_RLE_THREADS; d <<= 1) {
    uint32_t v = t >= (uint32_t)d ? sm_cnt[t - d] : 0;
    __syncthreads();
    sm_cnt[t] += v;
    __syncthreads();
  }
  slice_out[(size_t)blockIdx.x * BZ_RLE_THREADS + t] = sm_cnt[t] - outn;  // exclusive
  if (t == BZ_RLE_THREADS - 1) {
    // The block ends on 4 equal bytes with no count behind them (no encoder writes that; damaged data does): the reference
    // reads the count without looking at cNBlockUsed (:708-716) -- one step further round the cycle -- writes the run
    // and only then returns -1 (:628-631).  Same verdict as an overrunning randomised block: irregular = 2.
    unsigned long long total = sm_cnt[t];
    if (s == 4) {
      const uint32_t cl = cycle_len[blockIdx.x];
      total += src[cl ? c.nblock % cl : 0u];
      if (irregular[blockIdx.x] == 0) irregular[blockIdx.x] = 2;
    }
    block_out[blockIdx.x] = total;
  }
}

// exclusive scan of the block sizes (a few thousand values), started again at its slot by the first block of every stream
__global__ void k_bz2_offsets(const BzChain *__restrict__ chain, const unsigned long long *__restrict__ block_out, uint32_t n_chain,
                              unsigned long long *__restrict__ block_off, int carry) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    unsigned long long run = carry ? block_off[0] : 0;  // (a later group of the chain goes on where the one before it ended)
    for (uint32_t i = 0; i < n_chain; ++i) {
      if (chain[i].flags & 2u) run = chain[i].out_lo;
      block_off[i] = run;
      run += block_out[i];
    }
    block_off[n_chain] = run;
  }
}

// pass 2: write the decoded bytes + the block CRC
__global__ void __launch_bounds__(BZ_RLE_THREADS)
k_bz2_rle_emit(const BzChain *__restrict__ chain, const uint8_t *__restrict__ raw, uint32_t nblock_max,
               const uint32_t *__restrict__ slice_state, const uint32_t *__restrict__ slice_out,
               const unsigned long long *__restrict__ block_off, unsigned long long out_cap, uint8_t *__restrict__ out,
               uint32_t *__restrict__ block_crc, const uint32_t *__restrict__ cycle_len) {
  __shared__ uint32_t crc_tab[256];
  __shared__ uint32_t sm_crc[BZ_RLE_THREADS];
  __shared__ uint32_t sm_len[BZ_RLE_THREADS];
  const BzChain c = chain[blockIdx.x];
  if (c.flags & 1u) return;  // randomised: k_bz2_rand
  if (c.out_hi < out_cap) out_cap = c.out_hi;
  const uint32_t t = threadIdx.x;
  if (t < 256) {
    uint32_t v = t << 24;
    for (int k = 0; k < 8; ++k) v = (v & 0x80000000u) ? (v << 1) ^ 0x04c11db7u : v << 1;
    crc_tab[t] = v;
  }
  __syncthreads();
  const uint8_t *src = raw + (size_t)blockIdx.x * nblock_max;
  const uint32_t per = (c.nblock + BZ_RLE_THREADS - 1) / BZ_RLE_THREADS;
  const uint32_t lo = min(t * per, c.nblock), hi = min(lo + per, c.nblock);
  uint32_t s = slice_state[(size_t)blockIdx.x * BZ_RLE_THREADS + t];
  const unsigned long long o0 = block_off[blockIdx.x] + slice_out[(size_t)blockIdx.x * BZ_RLE_THREADS + t];
  unsigned long long o = o0;
  uint32_t crc = 0;  // register started at 0: R(0, slice)
  // output bytes are gathered eight at a time and leave as one aligned 8-byte store (a thread's slice is contiguous in the
  // output: byte stores from 1024 threads were 32 partial sectors per instruction, the larger half of this kernel's time)
  uint64_t acc = 0;
  uint32_t nacc = 0;
  auto flush = [&]() {
    const unsigned long long b0 = o - nacc;
    if (nacc == 8u && b0 + 8u <= out_cap) {
      *reinterpret_cast<uint64_t *>(out + b0) = acc;
    } else {
      for (uint32_t k = 0; k < nacc; ++k)
        if (b0 + k < out_cap) out[b0 + k] = (uint8_t)(acc >> (8u * k));
    }
    acc = 0;
    nacc = 0;
  };
  auto put = [&](uint8_t b) {
    if (nacc == 0u && (o & 7ull) != 0ull) {  // up to the first aligned address: single bytes
      if (o < out_cap) out[o] = b;
      o++;
    } else {
      acc |= (uint64_t)b << (8u * nacc);
      nacc++;
      o++;
      if (nacc == 8u) flush();
    }
    crc = (crc << 8) ^ crc_tab[(crc >> 24) ^ b];
  };
  uint8_t prev = lo > 0 ? src[lo - 1] : 0;
  for (uint32_t i = lo; i < hi; ++i) {
    uint8_t x = src[i];
    bool eq = (i > 0) && x == prev;
    if (s == 4) {
      for (uint32_t k = 0; k < x; ++k) put(prev);
    } else {
      put(x);
    }
    s = rle_step(s, eq);
    prev = x;
  }
  if (t == BZ_RLE_THREADS - 1 && s == 4) {  // a run of 4 ends the block: its count is read past the end (k_bz2_rle_count)
    const uint32_t cl = cycle_len[blockIdx.x];
    const uint32_t extra = src[cl ? c.nblock % cl : 0u];
    for (uint32_t k = 0; k < extra; ++k) put(prev);
  }
  flush();
  // combine: R(init, A||B) = R(init, A) * x^(8|B|) ^ R(0, B)
  sm_crc[t] = crc;
  sm_len[t] = (uint32_t)(o - o0);
  __syncthreads();
  for (int d = 1; d < BZ_RLE_THREADS; d <<= 1) {
    uint32_t cl = 0, ll = 0;
    const bool has = t >= (uint32_t)d;
    if (has) {
      cl = sm_crc[t - d];
      ll = sm_len[t - d];
    }
    __syncthreads();
    if (has) {
      sm_crc[t] = bzcrc_mulmod(cl, bzcrc_xpow8(sm_len[t])) ^ sm_crc[t];
      sm_len[t] += ll;
    }
    __syncthreads();
  }
  if (t == BZ_RLE_THREADS - 1) {
    // whole block with the real initial register 0xffffffff, then the final xor (bzip2.dart:9,16-18)
    uint32_t r = bzcrc_mulmod(0xffffffffu, bzcrc_xpow8(sm_len[t])) ^ sm_crc[t];
    block_crc[blockIdx.x] = r ^ 0xffffffffu;
  }
}

// ---------------------------------------------------------------------------------------------
// Randomised blocks (bzip2_decoder.dart:492-608).  The byte read from the inverse BWT is XORed with 1 whenever a countdown
// loaded from the 512-entry table stands at 1; in the reference only the FIRST read of every turn of the run-length
// state machine decrements that countdown (the 2nd-5th reads reload it at 0 but do not count down -- SURVEY Q6, unlike
// libbzip2), so the mask depends on the run structure of the already unmasked bytes: one serial walk per block.
// EMIT = false: output size of the block; EMIT = true: bytes + CRC.  A walk that overruns the block (:497-499) reports
// irregular = 2 after its bytes are written, as the reference's output stream has them by then.
// ---------------------------------------------------------------------------------------------
template <bool EMIT>
__global__ void k_bz2_rand(const BzChain *__restrict__ chain, uint32_t n_chain, const uint8_t *__restrict__ raw,
                           uint32_t nblock_max, unsigned long long *__restrict__ block_out,
                           const unsigned long long *__restrict__ block_off, unsigned long long out_cap, uint8_t *__restrict__ out,
                           uint32_t *__restrict__ block_crc, int32_t *__restrict__ irregular,
                           const uint32_t *__restrict__ cycle_len) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_chain) return;
  const BzChain c = chain[i];
  if (!(c.flags & 1u) || c.nblock == 0) return;
  if (c.out_hi < out_cap) out_cap = c.out_hi;
  const uint8_t *src = raw + (size_t)i * nblock_max;
  const uint32_t nb = c.nblock;
  const uint32_t cl = cycle_len[i] ? cycle_len[i] : nb;  // the walk goes round a cycle of cl <= nblock bytes (k_bz2_walk_order)
  unsigned long long o = EMIT ? block_off[i] : 0ull, o0 = o;
  uint32_t crc = 0xffffffffu;
  int r_n_to_go = 0, r_t_pos = 0;
  uint32_t rd = 0;  // reads so far; read number q returns byte q of the cycle: raw[q] = raw[q mod cl] below nblock, and beyond
#define BZ_READ(dst)                              \
  do {                                            \
    (dst) = src[rd < nb ? rd : rd % cl];          \
    rd++;                                         \
    if (r_n_to_go == 0) {                         \
      r_n_to_go = c_bz2_rnums[r_t_pos];           \
      r_t_pos = (r_t_pos + 1) & 511;              \
    }                                             \
  } while (0)
  int k0, k1;
  BZ_READ(k0);
  r_n_to_go--;
  k0 ^= (r_n_to_go == 1) ? 1 : 0;
  const uint32_t save = nb + 1;
  uint32_t n_used = 1;
  int out_len = 0, out_ch = 0;
  bool fail = false;
  for (;;) {
    for (; out_len > 0; --out_len) {
      if (EMIT) {
        if (o < out_cap) out[o] = (uint8_t)out_ch;
        uint32_t v = (crc >> 24) ^ (uint32_t)out_ch;
        uint32_t tv = v << 24;
        for (int b = 0; b < 8; ++b) tv = (tv & 0x80000000u) ? (tv << 1) ^ 0x04c11db7u : tv << 1;
        crc = (crc << 8) ^ tv;
      }
      o++;
    }
    if (n_used == save) break;
    if (n_used > save) {
      fail = true;
      break;
    }
    out_len = 1;
    out_ch = k0;
    BZ_READ(k1);
    r_n_to_go--;
    k1 ^= (r_n_to_go == 1) ? 1 : 0;
    n_used++;
    if (n_used == save) continue;
    if (k1 != k0) {
      k0 = k1;
      continue;
    }
    out_len = 2;
    BZ_READ(k1);
    k1 ^= (r_n_to_go == 1) ? 1 : 0;
    n_used++;
    if (n_used == save) continue;
    if (k1 != k0) {
      k0 = k1;
      continue;
    }
    out_len = 3;
    BZ_READ(k1);
    k1 ^= (r_n_to_go == 1) ? 1 : 0;
    n_used++;
    if (n_used == save) continue;
    if (k1 != k0) {
      k0 = k1;
      continue;
    }
    BZ_READ(k1);
    k1 ^= (r_n_to_go == 1) ? 1 : 0;
    n_used++;
    out_len = k1 + 4;
    BZ_READ(k0);
    k0 ^= (r_n_to_go == 1) ? 1 : 0;
    n_used++;
  }
#undef BZ_READ
  if (!EMIT) {
    block_out[i] = o - o0;
  } else {
    block_crc[i] = crc ^ 0xffffffffu;
    if (fail) irregular[i] = 2;
  }
}

// ---------------------------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------------------------
size_t bz2_entropy_smem() { return sizeof(BzSmem); }

cudaError_t bz2_launch_scan_streams(const Bz2Scan &a, uint64_t n_threads, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(a.n_cand, 0, 4, s);
  if (e != cudaSuccess) return e;
  const uint64_t blocks = (n_threads + 255) / 256;
  if (blocks == 0) return cudaSuccess;
  k_bz2_scan<<<(unsigned)blocks, 256, 0, s>>>(a);
  count_launch();
  return cudaGetLastError();
}

cudaError_t bz2_launch_scan(const uint8_t *d_in, uint64_t n_bytes, unsigned long long *d_cand, uint32_t *d_ncand, uint32_t cap,
                            cudaStream_t s) {
  Bz2Scan a;
  a.in = d_in;
  a.n_bytes = n_bytes;
  a.cand = d_cand;
  a.n_cand = d_ncand;
  a.cap = cap;
  return bz2_launch_scan_streams(a, (n_bytes + 3) / 4, s);
}

cudaError_t bz2_launch_entropy(const Bz2Entropy &a, cudaStream_t s) {
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(k_bz2_entropy, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BzSmem));
    if (e != cudaSuccess) return e;
    attr = true;
  }
  if (a.n_blocks == 0) return cudaSuccess;
  // clean blocks by the two-warp pipeline, whatever it leaves (status BZ_REDO) by the exact kernel; B200Z_BZ2_FAST=0: the
  // exact kernel only (read at every launch)
  const char *fe = getenv("B200Z_BZ2_FAST");
  const int fast = !(fe && fe[0] == '0');
  if (fast) {
    k_bz2_entropy_fast<<<a.n_blocks, BZF_NT, 0, s>>>(a.words, a.n_bytes, a.blk_bit, a.n_blocks, a.nblock_max, a.rec_val, a.rec_pos,
                                                 a.n_rec, a.nblock, a.orig_ptr, a.randomised, a.end_bit, a.status,
                                                 a.fast_flag, a.sym8, a.blk_end, a.blk_lim);
    count_launch();
  }
  k_bz2_entropy<<<a.n_blocks, 32, sizeof(BzSmem), s>>>(a.words, a.n_bytes, a.blk_bit, a.n_blocks, a.nblock_max, a.rec_val,
                                                       a.rec_pos, a.n_rec, a.nblock, a.orig_ptr, a.randomised, a.end_bit,
                                                       a.status, fast, a.blk_end, a.blk_lim);
  count_launch();
  return cudaGetLastError();
}

cudaError_t bz2_launch_entropy_literal(const Bz2Entropy &a, const uint32_t *d_list, uint32_t n_list, cudaStream_t s) {
  if (n_list == 0) return cudaSuccess;
  k_bz2_entropy_literal<<<n_list, 32, 0, s>>>(a.words, a.n_bytes, a.blk_bit, d_list, n_list, a.nblock_max, a.rec_val, a.rec_pos,
                                              a.n_rec, a.nblock, a.end_bit, a.status, a.blk_end, a.blk_lim);
  count_launch();
  return cudaGetLastError();
}

size_t bz2_slot_bytes_per_block() { return (size_t)(BZ_SPLIT + 2) * BZ_SLOT; }

cudaError_t bz2_launch_ibwt(const Bz2Ibwt &a, cudaStream_t s) {
  if (a.n_chain == 0) return cudaSuccess;
  const BzChain *chain = reinterpret_cast<const BzChain *>(a.chain);
  const uint32_t chunks_max = (a.nblock_max + BZ_CHUNK - 1) / BZ_CHUNK;
  if (a.phase != 2) {
  if (a.any_records) {  // (38 k CTAs that find nothing to do still cost 1.5 ms)
    dim3 g1(64, a.n_chain);
    k_bz2_expand<<<g1, 256, 0, s>>>(chain, a.rec_val, a.rec_pos, a.nblock_max, a.sym8);
    count_launch();
  }
  dim3 g2((chunks_max + 3) / 4, a.n_chain);
  k_bz2_chunk_hist<<<g2, 128, 0, s>>>(chain, a.sym8, a.nblock_max, chunks_max, a.chist);
  count_launch();
  k_bz2_chunk_scan<<<a.n_chain, 256, 0, s>>>(chain, chunks_max, a.chist);
  count_launch();
  k_bz2_build_tt<<<g2, 128, 0, s>>>(chain, a.sym8, a.nblock_max, chunks_max, a.chist, a.tt);
  count_launch();
  // (persistent grids: segments come off a counter)
  {
    cudaError_t e = cudaMemsetAsync(a.walk_ctr, 0, 8, s);
    if (e != cudaSuccess) return e;
  }
  const unsigned g3 = (unsigned)std::min<uint64_t>(((uint64_t)a.n_chain * (BZ_SPLIT + 2) + 255) / 256, 148u * 8u);
  k_bz2_walk_len<<<g3, 256, 0, s>>>(chain, a.n_chain, a.tt, a.nblock_max, a.seg_len, a.seg_next, a.seg_resume, a.slots, a.walk_ctr);
  count_launch();
  k_bz2_walk_order<<<a.n_chain, 128, 0, s>>>(chain, a.n_chain, a.tt, a.nblock_max, a.seg_len, a.seg_next,
                                                         a.seg_off, a.irregular, a.cycle_len);
  count_launch();
  k_bz2_walk_emit<<<g3, 256, 0, s>>>(chain, a.n_chain, a.tt, a.nblock_max, a.seg_len, a.seg_off, a.seg_resume, a.slots, a.raw);
  count_launch();
  k_bz2_periodic_fill<<<dim3(64, a.n_chain), 256, 0, s>>>(chain, a.cycle_len, a.nblock_max, a.raw);
  count_launch();
  k_bz2_rle_count<<<a.n_chain, BZ_RLE_THREADS, 0, s>>>(chain, a.raw, a.nblock_max, a.slice_state, a.slice_out, a.block_out,
                                                           a.cycle_len, a.irregular);
  count_launch();
  if (a.any_randomised) {
    k_bz2_rand<false><<<(a.n_chain + 31) / 32, 32, 0, s>>>(chain, a.n_chain, a.raw, a.nblock_max, a.block_out, a.block_off,
                                                           a.out_cap, a.out, a.block_crc, a.irregular, a.cycle_len);
    count_launch();
  }
  k_bz2_offsets<<<1, 32, 0, s>>>(chain, a.block_out, a.n_chain, a.block_off, a.carry_off ? 1 : 0);
  count_launch();
  }
  if (a.phase == 1) return cudaGetLastError();
  k_bz2_rle_emit<<<a.n_chain, BZ_RLE_THREADS, 0, s>>>(chain, a.raw, a.nblock_max, a.slice_state, a.slice_out, a.block_off,
                                                     a.out_cap, a.out, a.block_crc, a.cycle_len);
  count_launch();
  if (a.any_randomised) {
    k_bz2_rand<true><<<(a.n_chain + 31) / 32, 32, 0, s>>>(chain, a.n_chain, a.raw, a.nblock_max, a.block_out, a.block_off,
                                                          a.out_cap, a.out, a.block_crc, a.irregular, a.cycle_len);
    count_launch();
  }
  return cudaGetLastError();
}

// K8 over the blocks [lo, hi) of the chain: every per-block array of `a` is shifted to the group's first block; the group's
// output goes on where block lo - 1 ended (block_off[lo], written by the group before it).  Groups launched one after the
// other on one stream give the result of one bz2_launch_ibwt over the whole chain -- and let the caller copy a finished
// group's bytes to the host while the next group is being decoded.
cudaError_t bz2_launch_ibwt_group(const Bz2Ibwt &a, uint32_t lo, uint32_t hi, cudaStream_t s) {
  if (hi <= lo) return cudaSuccess;
  const uint32_t chunks_max = (a.nblock_max + BZ_CHUNK - 1) / BZ_CHUNK;
  Bz2Ibwt g = a;
  g.chain = reinterpret_cast<const BzChain *>(a.chain) + lo;
  g.n_chain = hi - lo;
  g.chist = a.chist + (size_t)lo * chunks_max * 256;
  g.tt = a.tt + (size_t)lo * a.nblock_max;
  g.seg_len = a.seg_len + (size_t)lo * (BZ_SPLIT + 2);
  g.seg_next = a.seg_next + (size_t)lo * (BZ_SPLIT + 2);
  g.seg_off = a.seg_off + (size_t)lo * (BZ_SPLIT + 2);
  g.seg_resume = a.seg_resume + (size_t)lo * (BZ_SPLIT + 2);
  g.slots = a.slots + (size_t)lo * (BZ_SPLIT + 2) * BZ_SLOT;
  g.irregular = a.irregular + lo;
  g.cycle_len = a.cycle_len + lo;
  g.raw = a.raw + (size_t)lo * a.nblock_max;
  g.slice_state = a.slice_state + (size_t)lo * BZ_RLE_THREADS;
  g.slice_out = a.slice_out + (size_t)lo * BZ_RLE_THREADS;
  g.block_out = a.block_out + lo;
  g.block_off = a.block_off + lo;
  g.block_crc = a.block_crc + lo;
  g.carry_off = lo > 0;
  return bz2_launch_ibwt(g, s);
}

}  // namespace b200z
