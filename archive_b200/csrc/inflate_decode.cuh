// inflate_decode.cuh -- per-stream DEFLATE decode logic shared by the sm_90a kernel
// (inflate_kernels.cu) and the host-side logic emulation used by the CPU tests.
//
// Restates (reference, paths relative to /root/reference/):
//   lib/src/codecs/zlib/inflate.dart:104-401, lib/src/codecs/zlib/_huffman_table.dart:9-46
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "../../include/b200z.h"

#ifndef B200Z_LBITS
#define B200Z_LBITS 9
#endif
#ifndef B200Z_DBITS
#define B200Z_DBITS 8
#endif

#if defined(B200Z_EMU)
// CPU emulation of the CUDA execution model (tests/host_emul/cuda_emu.h): real warp collectives, plain memory
#define B200Z_SADDR(p) (p)
#define B200Z_LDS16(base, idx) ((uint32_t)((const uint16_t *)(base))[idx])
#define B200Z_LDS32(base, idx) (((const uint32_t *)(base))[idx])
#define B200Z_PREFETCH(p) ((void)0)
typedef const void *b200z_saddr;
#define B200Z_ANY(x) __any_sync(0xffffffffu, (x))
#define B200Z_BALLOT(x) __ballot_sync(0xffffffffu, (x))
#define B200Z_SHFL(v, src) __shfl_sync(0xffffffffu, (v), (src))
#define B200Z_SYNCWARP() __syncwarp()
#define B200Z_OPAQUE(x) (x)
#define B200Z_LDG(p) (*(p))
#define B200Z_BREV(x) __brev(x)
#define B200Z_POPC(x) __popc(x)
#define B200Z_LDCG(p) (*(p))
#define B200Z_STCS(p, v) (*(p) = (v))
#define B200Z_REDOR(p, v) atomicOr((p), (v))
#elif defined(__CUDA_ARCH__)
// 32-bit shared-window addressing for the per-lane LUTs: keeps the hot loop free of 64-bit generic pointers
#define B200Z_SADDR(p) ((uint32_t)__cvta_generic_to_shared(p))
__device__ __forceinline__ uint32_t b200z_lds16(uint32_t base, uint32_t idx) {
  uint16_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(base + idx * 2u));
  return v;
}
__device__ __forceinline__ uint32_t b200z_lds32(uint32_t base, uint32_t idx) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(base + idx * 4u));
  return v;
}
#define B200Z_LDS16(base, idx) b200z_lds16(base, idx)
#define B200Z_LDS32(base, idx) b200z_lds32(base, idx)
#define B200Z_PREFETCH(p) asm volatile("prefetch.global.L1 [%0];" ::"l"(p))
typedef uint32_t b200z_saddr;
#define B200Z_ANY(x) __any_sync(0xffffffffu, (x))
#define B200Z_BALLOT(x) __ballot_sync(0xffffffffu, (x))
#define B200Z_SHFL(v, src) __shfl_sync(0xffffffffu, (v), (src))
#define B200Z_SYNCWARP() __syncwarp()
#define B200Z_POPC(x) __popc(x)
#define B200Z_LDCG(p) __ldcg(p)
#define B200Z_STCS(p, v) __stcs((p), (v))
#define B200Z_REDOR(p, v) atomicOr((p), (v))
__device__ __forceinline__ uint32_t b200z_opaque(uint32_t v) {
  uint32_t o;
  asm volatile("mov.b32 %0, %1;" : "=r"(o) : "r"(v));  // keeps a loop invariant in a register (no rematerialisation)
  return o;
}
#define B200Z_OPAQUE(x) b200z_opaque(x)
#define B200Z_LDG(p) __ldg(p)
#define B200Z_BREV(x) __brev(x)
#else
#define B200Z_SADDR(p) (p)
#define B200Z_LDS16(base, idx) ((uint32_t)((const uint16_t *)(base))[idx])
#define B200Z_LDS32(base, idx) (((const uint32_t *)(base))[idx])
#define B200Z_PREFETCH(p) ((void)0)
typedef const void *b200z_saddr;
#define B200Z_ANY(x) (x)
#define B200Z_BALLOT(x) ((x) ? 1u : 0u)
#define B200Z_SHFL(v, src) (v)
#define B200Z_SYNCWARP() ((void)0)
#define B200Z_POPC(x) __builtin_popcount(x)
#ifndef __CUDACC__
struct alignas(16) uint4 {
  uint32_t x, y, z, w;
};
#endif
#define B200Z_LDCG(p) (*(p))
#define B200Z_STCS(p, v) (*(p) = (v))
#define B200Z_REDOR(p, v) (*(p) |= (v))
#define B200Z_OPAQUE(x) (x)
#define B200Z_LDG(p) (*(p))
static inline uint32_t b200z_host_brev(uint32_t v) {
  v = ((v >> 1) & 0x55555555u) | ((v & 0x55555555u) << 1);
  v = ((v >> 2) & 0x33333333u) | ((v & 0x33333333u) << 2);
  v = ((v >> 4) & 0x0f0f0f0fu) | ((v & 0x0f0f0f0fu) << 4);
  v = ((v >> 8) & 0x00ff00ffu) | ((v & 0x00ff00ffu) << 8);
  return (v >> 16) | (v << 16);
}
#define B200Z_BREV(x) b200z_host_brev(x)
#endif
#if defined(__CUDACC__) && !defined(B200Z_EMU)
#define B200Z_HD __device__ __forceinline__
#define B200Z_CONST __constant__
#else
#define B200Z_HD inline
#define B200Z_CONST static const
#include <algorithm>
using std::max;
using std::min;
#endif

namespace b200z {

// ---------------------------------------------------------------------------------------------
// constants (inflate.dart:738-894)
// ---------------------------------------------------------------------------------------------
B200Z_CONST uint8_t c_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
// length symbol 257+i -> (base << 4) | extra_bits
B200Z_CONST uint16_t c_len_tab[32] = {
    (3 << 4) | 0,   (4 << 4) | 0,   (5 << 4) | 0,   (6 << 4) | 0,   (7 << 4) | 0,   (8 << 4) | 0,
    (9 << 4) | 0,   (10 << 4) | 0,  (11 << 4) | 1,  (13 << 4) | 1,  (15 << 4) | 1,  (17 << 4) | 1,
    (19 << 4) | 2,  (23 << 4) | 2,  (27 << 4) | 2,  (31 << 4) | 2,  (35 << 4) | 3,  (43 << 4) | 3,
    (51 << 4) | 3,  (59 << 4) | 3,  (67 << 4) | 4,  (83 << 4) | 4,  (99 << 4) | 4,  (115 << 4) | 4,
    (131 << 4) | 5, (163 << 4) | 5, (195 << 4) | 5, (227 << 4) | 5, (258 << 4) | 0, 0, 0, 0};
// distance symbol -> (base << 4) | extra_bits
B200Z_CONST uint32_t c_dist_tab[32] = {
    (1 << 4) | 0,     (2 << 4) | 0,     (3 << 4) | 0,      (4 << 4) | 0,      (5 << 4) | 1,      (7 << 4) | 1,
    (9 << 4) | 2,     (13 << 4) | 2,    (17 << 4) | 3,     (25 << 4) | 3,     (33 << 4) | 4,     (49 << 4) | 4,
    (65 << 4) | 5,    (97 << 4) | 5,    (129 << 4) | 6,    (193 << 4) | 6,    (257 << 4) | 7,    (385 << 4) | 7,
    (513 << 4) | 8,   (769 << 4) | 8,   (1025 << 4) | 9,   (1537 << 4) | 9,   (2049 << 4) | 10,  (3073 << 4) | 10,
    (4097 << 4) | 11, (6145 << 4) | 11, (8193 << 4) | 12,  (12289 << 4) | 12, (16385 << 4) | 13, (24577 << 4) | 13,
    0, 0};

// token encoding (uint32):
//   literal : 0x80000000 | byte
//   match   : (len << 16) | dist          len 1..258 (bit 31/30 clear), dist 1..32768
//   stored  : 0x40000000 | (pos >> 30) << 16 | len (3..65535), followed by ONE payload word =
//             pos & 0x3fffffff (pos = byte offset of the run in the unit's input; top bits 00 so a
//             payload never looks like a stored token); the pair never straddles a group of 32
//             tokens (a nop pads).
//   nop     : 0
#define TOK_LIT 0x80000000u
#define TOK_STORED 0x40000000u

constexpr int LBITS = B200Z_LBITS;  // primary literal/length LUT bits
constexpr int DBITS = B200Z_DBITS;  // primary distance LUT bits
constexpr int SUBN = 128;           // second-level entries shared by the codes longer than LBITS / DBITS of one block
constexpr int LUT_HALFWORDS = (1 << LBITS) + (1 << DBITS) + SUBN;
constexpr int LANE_STRIDE_WORDS = LUT_HALFWORDS / 2 + 1;  // +1 word: same index -> different bank per lane
constexpr int CONST_WORDS = 16 + 32 + 64;                  // len table (32 x u16) + dist table (32 x u32) + xtab (64 x u32)
constexpr int STAGE_WORDS = 32 * 4;                        // per warp: 4 tokens per lane, so that tokens leave as 16-byte stores

static inline size_t inflate_decode_smem_bytes(int warps_per_block, int units_per_warp) {
  return (size_t)(CONST_WORDS + warps_per_block * (units_per_warp * LANE_STRIDE_WORDS + STAGE_WORDS) + 4) * 4;
}

// Canonical-code side tables for codes longer than the LUT (rare): per lane, in local memory.
struct alignas(4) SlowTab {
  uint16_t first[16];  // first canonical code of each length
  uint16_t count[16];  // number of codes of each length
  uint16_t offs[16];   // index into perm of the first symbol of each length
  uint16_t perm[288];  // symbols sorted by (length, symbol)
  uint8_t maxlen;      // HuffmanTable.maxCodeLength (_huffman_table.dart:12-15)
};
struct alignas(4) SlowTabD {
  uint16_t first[16];
  uint16_t count[16];
  uint16_t offs[16];
  uint8_t perm[32];
  uint8_t maxlen;
};

// ---------------------------------------------------------------------------------------------
// bit reader: LSB-first (inflate.dart:159-184), refilled 32 aligned bits at a time.
//   rem_bits() is the exact number of stream bits not yet consumed; it is what the reference's
//   "isEOS while _bitBufferLen < n" tests (inflate.dart:166-168,192-195) see.
// ---------------------------------------------------------------------------------------------
struct BitReader {
  const uint32_t *w;  // 16-byte aligned word base of the unit
  uint32_t nextw;  // word `widx`, requested one refill ahead of its use (hides the L1/L2 latency)
  uint64_t buf;
  int cnt;          // bits in buf (may include `pad` invalid bits once widx >= nw)
  uint32_t widx;    // next word to load
  uint32_t nw;      // words covering the unit
  uint32_t lead;    // byte offset of the unit inside word 0
  uint32_t in_len;  // unit bytes

  B200Z_HD void seek(uint32_t byte_pos) {
    uint32_t a = lead + byte_pos;
    widx = a >> 2;
    uint32_t sh = (a & 3) * 8;
    uint32_t v = (widx < nw) ? B200Z_LDG(w + widx) : 0u;
    widx++;
    nextw = (widx < nw) ? B200Z_LDG(w + widx) : 0u;
    buf = (uint64_t)(v >> sh);
    cnt = 32 - (int)sh;
  }
  B200Z_HD void refill() {
    if (cnt < 32) {
      buf |= (uint64_t)nextw << cnt;
      cnt += 32;
      widx++;
      nextw = (widx < nw) ? B200Z_LDG(w + widx) : 0u;
    }
  }
  // all bits in buf valid and >= 32 of them after refill()
  B200Z_HD bool fast() const { return widx < nw; }
  B200Z_HD long long rem_bits() const {
    return (long long)cnt + 32ll * ((long long)nw - (long long)widx) -
           (32ll * nw - 8ll * ((long long)lead + in_len));
  }
  B200Z_HD uint32_t peek(int n) const { return (uint32_t)buf & ((1u << n) - 1u); }
  B200Z_HD void drop(int n) {
    buf >>= n;
    cnt -= n;
  }
  // _readBits: -1 when fewer than n bits remain (then nothing is consumed that matters)
  B200Z_HD int read_bits_checked(int n) {
    if (n == 0) return 0;
    refill();
    if (!fast() && rem_bits() < n) return -1;
    int v = (int)peek(n);
    drop(n);
    return v;
  }
};

// ---------------------------------------------------------------------------------------------
// Build the LUT + slow tables for one alphabet from code lengths (HuffmanTable ctor restated for a
// two-level layout).  Returns false when the set is over-subscribed (reference: later writes win in
// a flat table -- garbage; here: B200Z_U_BADCODE).
// ---------------------------------------------------------------------------------------------
// Second level (sub != nullptr): a root slot shared by codes longer than TBITS holds a LINK = (sub_base << 7) |
// (extra index bits << 4) | 0 -- the zero length nibble still reads as "miss" to code that does not know links -- and the
// entry is found at sub[sub_base + next bits].  Symbols kept out of the LUT leave zero entries there too.  When the
// pool of sub_cap entries (shared by the block's two alphabets, *sub_used so far) is exhausted the remaining long prefixes stay plain misses (the exact step decodes them).
template <int TBITS, typename PermT>
B200Z_HD bool build_table(const uint8_t *lens, int n, uint16_t *lut, uint16_t *first,
                                            uint16_t *count, uint16_t *offs, PermT *perm, uint8_t *maxlen,
                                            int lut_skip_eq = -1, int lut_skip_above = 0x7fffffff,
                                            uint16_t *sub = nullptr, int sub_cap = 0, int *sub_used = nullptr) {
  for (int l = 0; l < 16; ++l) count[l] = 0;
  int mx = 0;
  for (int i = 0; i < n; ++i) {
    int l = lens[i];
    count[l]++;
    mx = max(mx, l);
  }
  *maxlen = (uint8_t)mx;
  count[0] = 0;
  // Kraft check
  int left = 1;
  bool over = false;
  for (int l = 1; l < 16; ++l) {
    left <<= 1;
    left -= count[l];
    if (left < 0) over = true;
  }
  uint16_t next[16];
  {
    int code = 0, o = 0;
    for (int l = 1; l < 16; ++l) {
      code = (code + count[l - 1]) << 1;
      first[l] = (uint16_t)code;
      next[l] = (uint16_t)code;
      offs[l] = (uint16_t)o;
      o += count[l];
    }
    first[0] = 0;
    offs[0] = 0;
  }
  uint32_t *lut32 = reinterpret_cast<uint32_t *>(lut);
  for (int i = 0; i < (1 << TBITS) / 2; ++i) lut32[i] = 0;
  if (over) return false;
  uint16_t run[16];
  for (int l = 0; l < 16; ++l) run[l] = offs[l];
  for (int s = 0; s < n; ++s) {
    int l = lens[s];
    if (l == 0) continue;
    uint32_t c = next[l]++;
    perm[run[l]++] = (PermT)s;
    if (l <= TBITS && s != lut_skip_eq && s <= lut_skip_above) {
      uint32_t r = B200Z_BREV(c) >> (32 - l);
      uint16_t e = (uint16_t)((s << 4) | l);
      for (uint32_t j = r; j < (1u << TBITS); j += (1u << l)) lut[j] = e;
    }
  }
  if (sub != nullptr && mx > TBITS) {
    // pass 1: the longest code under every root prefix, parked in the (still empty) root slot as a bare number > TBITS
    for (int l = TBITS + 1; l < 16; ++l) next[l] = first[l];
    for (int s = 0; s < n; ++s) {
      const int l = lens[s];
      if (l <= TBITS) continue;
      const uint32_t r = B200Z_BREV((uint32_t)next[l]++) >> (32 - l);
      uint16_t &slot = lut[r & ((1u << TBITS) - 1u)];
      if (slot < (uint16_t)l) slot = (uint16_t)l;
    }
    // pass 2: allocate the prefix's block on first sight, then place the symbol
    int used = *sub_used;
    for (int l = TBITS + 1; l < 16; ++l) next[l] = first[l];
    for (int s = 0; s < n; ++s) {
      const int l = lens[s];
      if (l <= TBITS) continue;
      const uint32_t r = B200Z_BREV((uint32_t)next[l]++) >> (32 - l);
      uint16_t &slot = lut[r & ((1u << TBITS) - 1u)];
      if (slot != 0 && slot < 16) {  // still the parked length
        const int sb = (int)slot - TBITS;
        if (used + (1 << sb) <= sub_cap) {
          slot = (uint16_t)((used << 7) | (sb << 4));
          used += 1 << sb;
        } else {
          slot = 0;
        }
      }
      if (slot == 0 || (slot & 15) != 0) continue;  // pool exhausted for this prefix
      if (s == lut_skip_eq || s > lut_skip_above) continue;
      const uint32_t sb = (slot >> 4) & 7u, base = slot >> 7;
      const uint16_t e = (uint16_t)((s << 4) | l);
      for (uint32_t j = r >> TBITS; j < (1u << sb); j += (1u << (l - TBITS))) sub[base + j] = e;
    }
    *sub_used = used;
  }
  return true;
}

// canonical decode of a code longer than TBITS (or a hole).  Returns length, 0 = no code matches.
template <int TBITS, typename PermT>
B200Z_HD int slow_decode(uint32_t bits15, const uint16_t *first, const uint16_t *count,
                                           const uint16_t *offs, const PermT *perm, int maxlen, int *sym) {
  uint32_t rev = B200Z_BREV(bits15) >> 17;  // first stream bit = MSB of a 15-bit value
  for (int l = 1; l <= maxlen; ++l) {
    uint32_t code = rev >> (15 - l);
    uint32_t d = code - first[l];
    if (d < count[l]) {
      *sym = perm[offs[l] + d];
      return l;
    }
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Block header after BTYPE: the fixed tables (inflate.dart:408-735) or a dynamic header (inflate.dart:239-298, _decode
// :345-401) read from `br`, and the block's lit/len and distance tables built (LUTs + SlowTab / SlowTabD; the dynamic
// ones with the second-level pool behind lut_d).  `lens` (>= 320 entries) is left holding the code lengths.  Returns 0,
// or the status the exact step stops with: U_STOP_SHORT (a short read), B200Z_U_STOP, B200Z_U_BADCODE, B200Z_U_THROW.
// Shared by the exact step below and K12's block finder (inflate_chunked.cuh).
// ---------------------------------------------------------------------------------------------
constexpr int U_STOP_SHORT = -100;  // internal: B200Z_U_STOP because a read ran out of input (reported as B200Z_U_STOP)
B200Z_HD int parse_tables(BitReader &br, uint32_t type, uint8_t *lens, uint16_t *lut_l, uint16_t *lut_d, SlowTab &sl,
                          SlowTabD &sd) {
  if (type == 1) {
    for (int i = 0; i < 288; ++i) lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
    build_table<LBITS, uint16_t>(lens, 288, lut_l, sl.first, sl.count, sl.offs, sl.perm, &sl.maxlen, 256, 285);
    for (int i = 0; i < 30; ++i) lens[i] = 5;
    build_table<DBITS, uint8_t>(lens, 30, lut_d, sd.first, sd.count, sd.offs, sd.perm, &sd.maxlen, -1, 29);
    return 0;
  }
  int hlit = br.read_bits_checked(5);
  if (hlit < 0) return U_STOP_SHORT;
  hlit += 257;
  if (hlit > 288) return B200Z_U_STOP;
  int hdist = br.read_bits_checked(5);
  if (hdist < 0) return U_STOP_SHORT;
  hdist += 1;
  if (hdist > 32) return B200Z_U_STOP;
  int hclen = br.read_bits_checked(4);
  if (hclen < 0) return U_STOP_SHORT;
  hclen += 4;
  if (hclen > 19) return B200Z_U_STOP;
  for (int i = 0; i < 19; ++i) lens[i] = 0;
  for (int i = 0; i < hclen; ++i) {
    int l = br.read_bits_checked(3);
    if (l < 0) return U_STOP_SHORT;
    lens[c_order[i]] = (uint8_t)l;
  }
  // code-length alphabet: 7-bit LUT in the (not yet built) lit/len LUT area
  uint8_t clmax;
  {
    uint16_t f[16], c[16], o[16];
    uint8_t pm[19];
    if (!build_table<7, uint8_t>(lens, 19, lut_l, f, c, o, pm, &clmax)) return B200Z_U_BADCODE;
  }
  // _decode (inflate.dart:345-401)
  const int num = hlit + hdist;
  int i = 0, prev = 0;
  while (i < num) {
    br.refill();
    if (!br.fast() && br.rem_bits() < clmax) return U_STOP_SHORT;
    uint32_t e = lut_l[br.peek(7)];
    int l = e & 15;
    int code = e >> 4;
    // l == 0: hole in an incomplete set -- the reference's flat table yields (len 0, sym 0)
    // (_huffman_table.dart:22), i.e. a zero length for this symbol and no bits consumed.
    br.drop(l);
    int repeat;
    if (code < 16) {
      lens[i++] = (uint8_t)code;
      prev = code;
      continue;
    } else if (code == 16) {
      repeat = br.read_bits_checked(2);
      if (repeat < 0) return U_STOP_SHORT;
      repeat += 3;
    } else if (code == 17) {
      repeat = br.read_bits_checked(3);
      if (repeat < 0) return U_STOP_SHORT;
      repeat += 3;
      prev = 0;
    } else {
      repeat = br.read_bits_checked(7);
      if (repeat < 0) return U_STOP_SHORT;
      repeat += 11;
      prev = 0;
    }
    if (i + repeat > num) return B200Z_U_THROW;
    for (int k = 0; k < repeat; ++k) lens[i++] = (uint8_t)prev;
  }
  for (int k = hdist; k < 32; ++k) lens[hlit + k] = 0;
  uint16_t *sub_p = lut_d + (1 << DBITS);  // second-level pool
  int sub_used = 0;
  for (int k = 0; k < SUBN / 2; ++k) reinterpret_cast<uint32_t *>(sub_p)[k] = 0;
  bool ok = build_table<DBITS, uint8_t>(lens + hlit, hdist, lut_d, sd.first, sd.count, sd.offs, sd.perm, &sd.maxlen, -1, 29, sub_p, SUBN, &sub_used);
  ok = build_table<LBITS, uint16_t>(lens, hlit, lut_l, sl.first, sl.count, sl.offs, sl.perm, &sl.maxlen, 256, 285, sub_p, SUBN, &sub_used) && ok;
  if (!ok) return B200Z_U_BADCODE;
  return 0;
}

// ---------------------------------------------------------------------------------------------
// One stream: DEFLATE bits -> token stream.  Runs as one LANE of k_inflate_decode (and, compiled as
// plain C++, inside tests/host_emul to check the logic against the oracle without a GPU).
// ---------------------------------------------------------------------------------------------
struct UnitResult {
  uint32_t ntok, out_len, in_used;
  int32_t status;
};

// Intra-stream speculation ("helpers").  A stream's symbols form one serial chain, and 16 Ki streams cannot fill a
// GPU; so every stream owns G lanes of a warp.  Lane 0 of the group (the MASTER) is the exact decoder.  When it has
// parsed a block header it starts lanes 1..G-1 (HELPERS) at G-1 evenly spaced bit offsets of the rest of the input.
// A helper decodes from its (wrong) offset with the master's tables; Huffman streams self-synchronise, so after a few
// symbols its symbol boundaries coincide with the true ones.  Every helper marks the boundaries it passes in its first
// SPEC_W bits in a bitmap (global memory, L2); a lane that runs into its successor's window tests each of its own boundaries
// against that bitmap, and the first hit proves both parses identical from there on: helpers stop there ("linked"),
// the master instead adopts the successor's tokens (and, through the links, those of the whole chain), adds their
// output length, and resumes after the last adopted helper.  Helpers never take the exact path: anything unusual (end of
// block, invalid symbol, end of input, scratch full) just ends them, and the master continues exactly from there.  The
// tokens of a unit therefore live in PIECES (own region / helper regions); back-references of adopted tokens are range
// checked by k_inflate_expand, which knows absolute positions.
constexpr int SPEC_W = 2048;          // sync window (bits) = boundary bitmap of a helper
constexpr int SPEC_BMW = SPEC_W / 32;  // words per bitmap
constexpr int SPEC_MAX_G = 8;
constexpr int SPEC_HSHIFT = 2;         // helper token region = unit capacity >> 2
constexpr int PIECE_MAX = 30;
constexpr int PIECE_WORDS = 2 + 3 * PIECE_MAX;  // [0] = count, then (src, start, count) from word 2: src 0 = own region, k = helper k
constexpr int USCRATCH_BYTES = (SPEC_MAX_G - 1) * SPEC_BMW * 4;  // per unit: the helpers' boundary bitmaps
constexpr uint32_t SPEC_BIAS = 0x40000000u;  // helpers count output bytes from here, so "distance > produced" never fires
constexpr uint32_t SPEC_NOLINK = 0xffffffffu;

struct SpecCtx {
  int lane, sub, G;   // lane in the warp, index inside the stream's lane group (0 = master), lanes per stream
  bool spec;          // warp-uniform: helpers are in use in this launch
  bool count_only;    // warp-uniform: sizes only -- tokens are counted, not written (no expand follows)
  uint32_t *stage;    // shared memory: this lane's 4-token staging slot (16-byte aligned)
  uint32_t *hplane;   // helper k's token region = hplane + (k - 1) * hstride  [hcap words]
  size_t hstride;
  uint32_t hcap;
  uint32_t *bm;       // global: helper k's boundary bitmap = bm + (k - 1) * SPEC_BMW
  uint32_t *pieces;   // the unit's piece table (global)
  uint32_t hist = 0;  // bytes of earlier output in front of the unit that a distance may reach (InflateWs::hist)
};

B200Z_HD void piece_add(uint32_t *pieces, uint32_t &np, uint32_t src, uint32_t start, uint32_t count) {
  if (count == 0 || !pieces || np >= (uint32_t)PIECE_MAX) return;  // (the table cannot fill up: see where helpers are started)
  pieces[2 + 3 * np] = src;
  pieces[3 + 3 * np] = start;
  pieces[4 + 3 * np] = count;
  np++;
}

B200Z_HD UnitResult inflate_decode_unit(bool active, const uint8_t *in, uint32_t in_len, uint32_t cap, uint32_t *tok,
                                        uint16_t *lut_l, uint16_t *lut_d, const uint16_t *s_len_tab,
                                        const uint32_t *s_dist_tab, const uint32_t *s_xtab, const SpecCtx &sc) {
  const b200z_saddr lutl_s = B200Z_SADDR(lut_l), lutd_s = B200Z_SADDR(lut_d), xtab_s = B200Z_SADDR(s_xtab);
  uint16_t *sub_p = lut_d + (1 << DBITS);  // second-level pool (build_table)
  SlowTab sl;
  SlowTabD sd;
  uint8_t lens[320];
  const bool count_only = sc.count_only;
#define B200Z_TOK(p, v)          \
  do {                          \
    if (!count_only) B200Z_STCS((p) + nt, (v)); /* written once, read once by the expand kernel: evict first */ \
    nt++;                       \
  } while (0)
  const bool is_master = sc.sub == 0;
  const int gbase = sc.lane - sc.sub;  // the master's lane
  const bool spec_on = sc.spec;  // warp-uniform

  BitReader br;
  {
    uintptr_t a = reinterpret_cast<uintptr_t>(in);
    br.lead = (uint32_t)(a & 15);
    br.w = reinterpret_cast<const uint32_t *>(a - br.lead);
    br.in_len = in_len;
    br.nw = (uint32_t)(((uint64_t)br.lead + br.in_len + 3) >> 2);
    br.seek(0);
  }
  uint32_t nt = 0;
  uint32_t olen = 0;
  int st = B200Z_U_EOS;
  bool in_block = false;
  bool final_block = false;
  int maxl = 0, maxd = 0;
  bool mode_dist = false;  // bulk path: the next symbol is a distance code
  uint32_t mlen_pending = 0;
  uint32_t *tk = tok;      // where this lane's tokens go (master: the unit's region; helper: its own region)
  uint32_t capx = cap;     // output bound the bulk loop tests (helpers: none, their byte count is biased)
  uint32_t nt_limit = 0xffffffffu;  // token bound the bulk loop tests (helpers: end of their token region)

  // ---- speculation state (see SpecCtx) ----
  const uint32_t G = (uint32_t)sc.G;
  uint32_t hst = 0;  // helper: 0 idle, 1 running, 2 stopped with results
  bool h_fast = false;
  // Role-exclusive state shares registers: a master reads its helpers' values (and helpers the master's commands)
  // by shuffling the SAME variable from a lane of the other role.
  uint32_t v0 = 0, v1 = 0, v2 = 0, v3 = 0, v4 = 0, v5 = is_master ? 0u : SPEC_NOLINK, v6 = 0;
#define h_start_tok v0  /* helper: first token of the current run in its region      | master: cmd       */
#define h_ntok v1       /* helper: tokens of the run                                 | master: cmd_p0    */
#define h_rel_bytes v2  /* helper: bytes they produce                                | master: cmd_seg   */
#define h_end_pos v3    /* helper: bit position where it stopped                     | master: m_h       */
#define h_link_to v4    /* helper: the helper it met                                 | master: m_idx     */
#define h_link v5       /* helper: token of h_link_to where the parses met / NOLINK  | master: np        */
#define h_cur v6        /* helper: next free word of its token region                | master: piece_start */
#define cmd v0
#define cmd_p0 v1
#define cmd_seg v2
#define m_h v3
#define m_idx v4
#define np v5
#define piece_start v6
  bool m_stitch = false;  // master: adopting helper m_h from its token m_idx on
  uint32_t sp_origin = 0, sp_seg = 0;  // bit position rel_bits counts from; bits between helper starts (0: none live)
  uint32_t succ = G;                   // next helper this lane may meet
  bool sync_hit = false;
  uint32_t sync_off = 0, lb_rel = 0;

  bool done = !active || !is_master;
  // loop invariants of the bulk loop, pinned in registers
  const b200z_saddr lutl_r = B200Z_OPAQUE(lutl_s), lutd_r = B200Z_OPAQUE(lutd_s), xtab_r = B200Z_OPAQUE(xtab_s);
  const b200z_saddr sub_r = B200Z_SADDR(sub_p);
  for (;;) {  // warp-uniform: every lane reconverges here
    if (G > 1u) {  // helpers live exactly as long as their master
      const uint32_t md = B200Z_SHFL((uint32_t)done, gbase);
      if (!is_master) done = md != 0u;
    }
    if (B200Z_BALLOT(!done) == 0u) break;
    if (spec_on) {
      B200Z_SYNCWARP();
      // ---- commands of the master ----
      const uint32_t c = B200Z_SHFL(cmd, gbase), c_p0 = B200Z_SHFL(cmd_p0, gbase), c_seg = B200Z_SHFL(cmd_seg, gbase);
      if (is_master) {
        cmd = 0;
      } else if (c == 2u) {
        hst = 0;
      } else if (c == 1u && active) {
        hst = 0;
        uint32_t *bm_own = sc.bm + (sc.sub - 1) * SPEC_BMW;
        for (int i = 0; i < SPEC_BMW; ++i) bm_own[i] = 0;
        if (h_cur + 256u <= sc.hcap) {
          const uint32_t start = c_p0 + c_seg * (uint32_t)sc.sub;
          br.seek(start >> 3);
          br.drop((int)(start & 7u));
          in_block = true;
          mode_dist = false;
          mlen_pending = 0;
          tk = sc.hplane + (size_t)(sc.sub - 1) * sc.hstride;
          nt = h_cur;
          h_start_tok = h_cur;
          olen = SPEC_BIAS;
          capx = 0xffffffffu;
          nt_limit = sc.hcap - 2u;
          sp_origin = start;
          sp_seg = c_seg;
          succ = (uint32_t)sc.sub + 1u;
          sync_hit = false;
          h_link = SPEC_NOLINK;
          h_fast = true;
          hst = 1;
        }
      }
      // ---- a running helper that cannot go on in the bulk loop is finished ----
      if (!is_master && hst == 1u && (!h_fast || !(mode_dist || br.widx + 2u <= br.nw))) {
        const uint32_t pos = 32u * br.widx - (uint32_t)br.cnt - 8u * br.lead;  // bits consumed
        h_end_pos = mode_dist ? sp_origin + lb_rel : pos;  // a pending length symbol is given back
        if (!sync_hit && !h_fast && h_end_pos - sp_origin < (uint32_t)SPEC_W / 2u && br.widx + 4u <= br.nw) {
          // Stopped by an impossible symbol (typically a chance end-of-block) while still decoding from the guessed
          // offset, i.e. before it can have synchronised: nothing is lost by guessing again one bit further on.
          uint32_t *bm_own = sc.bm + (sc.sub - 1) * SPEC_BMW;
          for (int i = 0; i < SPEC_BMW; ++i) bm_own[i] = 0;
          const uint32_t again = h_end_pos + 1u;
          br.seek(again >> 3);
          br.drop((int)(again & 7u));
          mode_dist = false;
          mlen_pending = 0;
          nt = h_start_tok;
          olen = SPEC_BIAS;
          h_fast = true;
        } else {
        h_ntok = nt - h_start_tok;
        h_rel_bytes = olen - SPEC_BIAS;
        h_link = SPEC_NOLINK;
        if (sync_hit) {
          const uint32_t *bms = sc.bm + (succ - 1u) * SPEC_BMW;
          uint32_t idx = 0;
          for (uint32_t w = 0; w < (sync_off >> 5); ++w) idx += (uint32_t)B200Z_POPC(B200Z_LDCG(bms + w));
          idx += (uint32_t)B200Z_POPC(B200Z_LDCG(bms + (sync_off >> 5)) & ((1u << (sync_off & 31u)) - 1u));
          h_link = idx;
          h_link_to = succ;
        }
        h_cur = (nt + 31u) & ~31u;
        hst = 2;
        }
      }
      // ---- the master adopts the chain of helpers it met ----
      {
        const int src = (is_master && m_stitch) ? gbase + (int)m_h : sc.lane;
        const uint32_t r_hst = B200Z_SHFL(hst, src), r_start = B200Z_SHFL(h_start_tok, src), r_ntok = B200Z_SHFL(h_ntok, src);
        const uint32_t r_rel = B200Z_SHFL(h_rel_bytes, src), r_end = B200Z_SHFL(h_end_pos, src);
        const uint32_t r_link = B200Z_SHFL(h_link, src), r_to = B200Z_SHFL(h_link_to, src);
        if (is_master && m_stitch && r_hst == 2u) {
          const uint32_t *ht = sc.hplane + (size_t)(m_h - 1u) * sc.hstride + r_start;
          uint32_t r0 = 0;  // bytes the helper produced before the token the parses met at
          for (uint32_t i = 0; i < m_idx; ++i) {
            const uint32_t t = B200Z_LDCG(ht + i);
            r0 += (t & TOK_LIT) ? 1u : (t >> 16);
          }
          piece_add(sc.pieces, np, m_h, r_start + m_idx, r_ntok - m_idx);
          olen += r_rel - r0;
          if (r_link != SPEC_NOLINK) {
            m_h = r_to;
            m_idx = r_link;
          } else {  // end of the chain: go on from where that helper stopped
            br.seek(r_end >> 3);
            br.drop((int)(r_end & 7u));
            in_block = true;
            mode_dist = false;
            piece_start = nt;  // no gap: the unit's region holds at most one token per output byte
            succ = m_h + 1u;
            m_stitch = false;
            if (olen > cap) {
              st = B200Z_U_NOSPC;
              done = true;
            }
          }
        }
      }
    }
    // ---------------- bulk inner loop: warp-uniform, ONE SYMBOL per lane per turn, branch-light.  The same
    // instructions decode a literal/length symbol or a distance symbol (a lane that has just read a length
    // code reads its distance code on the next turn), so literal lanes and match lanes do not diverge.  A
    // lane speculates the symbol from two table look-ups and commits only if nothing special happened:
    // LUT miss (long code, end-of-block and invalid symbols are deliberately absent from the LUT),
    // back-reference before the start, output full, or fewer than 64 unloaded bits left.  Anything special
    // drops the warp to the exact step below for one turn.  (A token is <= 48 bits, so with >= 64 unloaded
    // bits at its start no end-of-stream test is needed in here.)
    const bool m_run = is_master && !done && !m_stitch;
    const bool can0 = ((m_run && in_block) || (!is_master && hst == 1u)) && (mode_dist || br.widx + 2u <= br.nw);
    const unsigned expect = B200Z_BALLOT(can0);
    if (B200Z_BALLOT(m_run && !can0) == 0u && expect != 0u) {
      bool fast_ok = can0;
      // position bookkeeping of the speculation (rel_bits counts from this lane's own start)
      uint32_t rel_bits = 32u * br.widx - (uint32_t)br.cnt - 8u * br.lead - sp_origin;
      uint32_t succ_rel = (sp_seg != 0u && succ < G) ? (succ - (uint32_t)sc.sub) * sp_seg : 0xffffffffu;
      bool mark = !is_master && spec_on;
      // Tokens are staged four at a time in shared memory and leave as one 16-byte store: 32 lanes writing 4 bytes each to
      // 32 different sectors per turn were almost half of this kernel's time.  q0 = first token not yet in memory.
      const bool stage_ok = !count_only && (reinterpret_cast<uintptr_t>(tk) & 15u) == 0u;
      uint32_t q0 = nt;
      for (;;) {
        const bool can = fast_ok && (mode_dist || br.widx + 2u <= br.nw);
        if (B200Z_BALLOT(can) != expect) break;
        if (!can) continue;  // lanes that are finished or waiting just keep voting
        br.refill();
        const bool dm = mode_dist;
        if (!dm) {
          lb_rel = rel_bits;
          if (rel_bits >= succ_rel) {  // inside the next helper's window: has it passed a boundary here?
            const uint32_t off = rel_bits - succ_rel;
            if (off < (uint32_t)SPEC_W) {
              if ((B200Z_LDCG(sc.bm + (succ - 1u) * SPEC_BMW + (off >> 5)) >> (off & 31u)) & 1u) {
                sync_hit = true;
                sync_off = off;
                fast_ok = false;
                continue;
              }
            } else {  // through the window without meeting it: that helper is lost, look for the next one
              succ++;
              succ_rel = succ < G ? succ_rel + sp_seg : 0xffffffffu;
            }
          }
          if (mark) {
            if (rel_bits < (uint32_t)SPEC_W) B200Z_REDOR(sc.bm + (sc.sub - 1) * SPEC_BMW + (rel_bits >> 5), 1u << (rel_bits & 31u));
            else mark = false;
          }
        }
        const uint32_t bits = (uint32_t)br.buf;
        const uint32_t e = B200Z_LDS16(dm ? lutd_r : lutl_r, bits & (dm ? ((1u << DBITS) - 1u) : ((1u << LBITS) - 1u)));
        uint32_t n = e & 15u;
        uint32_t sym = e >> 4;
        bool odd = false;
        if (n == 0u) {
          // Root miss (rare, divergent).  A link leads to the second-level entry of a code longer than the root index;
          // what is still a miss after that -- end of block, the invalid symbols, holes, an exhausted second-level
          // pool -- takes the exact step (helpers just stop there).
          if (e != 0u) {
            const uint32_t sb = (e >> 4) & 7u, sbase = e >> 7;
            const uint32_t e2 = B200Z_LDS16(sub_r, sbase + ((bits >> (dm ? DBITS : LBITS)) & ((1u << sb) - 1u)));
            n = e2 & 15u;
            sym = e2 >> 4;
          }
          odd = n == 0u;
        }
        const uint32_t xi = dm ? sym + 32u : (sym > 256u ? sym - 257u : 63u);
        const uint32_t x = B200Z_LDS32(xtab_r, xi & 63u);
        const uint32_t xb = x & 15u;
        const uint32_t val = (x >> 4) + ((bits >> n) & ~(0xffffffffu << xb));
        const bool islit = !dm && sym < 256u;
        const bool islen = !dm && sym > 256u;
        const uint32_t nolen = olen + (islit ? 1u : dm ? mlen_pending : 0u);
        const bool special = odd || (dm && val > olen + sc.hist) || nolen > capx || nt >= nt_limit;
        if (!special) {
          const uint32_t tot = n + xb;
          br.buf >>= tot;
          br.cnt -= (int)tot;
          rel_bits += tot;
          if (islit || dm) {
            const uint32_t tv = islit ? (TOK_LIT | sym) : ((mlen_pending << 16) | val);
            if (stage_ok) {
              sc.stage[nt & 3u] = tv;
              nt++;
              if ((nt & 3u) == 0u) {
                if (q0 + 4u <= nt) {
                  B200Z_STCS(reinterpret_cast<uint4 *>(tk + nt - 4u), *reinterpret_cast<const uint4 *>(sc.stage));
                } else {  // the group of four began before this bulk session
                  for (uint32_t k = q0; k < nt; ++k) B200Z_STCS(tk + k, sc.stage[k & 3u]);
                }
                q0 = nt;
              }
            } else {
              B200Z_TOK(tk, tv);
            }
          }
          olen = nolen;
          mlen_pending = islen ? val : mlen_pending;
          mode_dist = islen;
        }
        fast_ok = !special;
      }
      if (stage_ok)
        for (uint32_t k = q0; k < nt; ++k) B200Z_STCS(tk + k, sc.stage[k & 3u]);  // at most 3 left over
      if (!is_master) h_fast = fast_ok;
    }
    // ---- the master met a helper: close its own piece; the adoption runs at the top of the next turns ----
    if (spec_on && is_master && sync_hit) {
      const uint32_t *bms = sc.bm + (succ - 1u) * SPEC_BMW;
      uint32_t idx = 0;
      for (uint32_t w = 0; w < (sync_off >> 5); ++w) idx += (uint32_t)B200Z_POPC(B200Z_LDCG(bms + w));
      idx += (uint32_t)B200Z_POPC(B200Z_LDCG(bms + (sync_off >> 5)) & ((1u << (sync_off & 31u)) - 1u));
      piece_add(sc.pieces, np, 0u, piece_start, nt - piece_start);
      m_h = succ;
      m_idx = idx;
      m_stitch = true;
      sync_hit = false;
    }
    if (is_master && !done && !m_stitch) do {
    if (in_block && (mode_dist || br.widx + 2u <= br.nw)) {
      // ---------------- bulk path: ONE SYMBOL per turn, the same instructions for literal/length and
      // distance symbols (a lane that has just read a length code reads its distance code on the next
      // turn), so the lanes of a warp stay converged.  >= 64 stream bits are still unloaded when a
      // literal/length symbol starts, so no end-of-stream test is needed here (a token is <= 48 bits);
      // everything near the end of the stream goes through the exact per-token path below.
      br.refill();
      const bool dm = mode_dist;
      const uint32_t bits = (uint32_t)br.buf;
      uint32_t e = B200Z_LDS16(dm ? lutd_s : lutl_s, bits & (dm ? ((1u << DBITS) - 1u) : ((1u << LBITS) - 1u)));
      int n = (int)(e & 15u);
      int sym = (int)(e >> 4);
      if (n == 0) {
        if (dm) {
          n = slow_decode<DBITS, uint8_t>(bits & 0x7fffu, sd.first, sd.count, sd.offs, sd.perm, maxd, &sym);
          if (n == 0) sym = 0;  // hole in the flat table: (len 0, sym 0) (_huffman_table.dart:22)
        } else {
          n = slow_decode<LBITS, uint16_t>(bits & 0x7fffu, sl.first, sl.count, sl.offs, sl.perm, maxl, &sym);
          if (n == 0) {
            st = B200Z_U_BADCODE;
            done = true; break;
          }
        }
      }
      br.drop(n);
      // base + extra bits: lengths at [0,32), distances at [32,64); literals/EOB read the all-zero entry 63
      const uint32_t xi = dm ? 32u + (uint32_t)sym : (sym > 256 ? (uint32_t)(sym - 257) : 63u);
      const uint32_t x = B200Z_LDS32(xtab_s, xi & 63u);
      const int xb = (int)(x & 15u);
      const uint32_t val = (x >> 4) + ((uint32_t)br.buf & ((1u << xb) - 1u));
      br.drop(xb);
      if (!dm) {
        if (sym < 256) {
          if (olen >= cap) {
            st = B200Z_U_NOSPC;
            done = true; break;
          }
          B200Z_TOK(tok, TOK_LIT | (uint32_t)sym);
          olen++;
        } else if (sym == 256) {
          in_block = false;
        } else if (sym > 285) {
          st = B200Z_U_STOP;
          done = true; break;
        } else {
          mlen_pending = val;
          mode_dist = true;
        }
      } else {
        mode_dist = false;
        if (sym > 29) {
          st = B200Z_U_STOP;
          done = true; break;
        }
        if (val > olen + sc.hist) {  // writeBackReference before the start of the output (output_memory_stream.dart:83-86)
          st = B200Z_U_RANGE;
          done = true; break;
        }
        if (olen + mlen_pending > cap) {
          st = B200Z_U_NOSPC;
          done = true; break;
        }
        B200Z_TOK(tok, (mlen_pending << 16) | val);
        olen += mlen_pending;
      }
      break;  // next symbol
    }
    if (!in_block) {
      // ---------------- block boundary: _inflate loop + _parseBlock (inflate.dart:111-156) -------------
      if (sp_seg != 0u) {  // helpers of the block that just ended (they decode past its end-of-block symbol)
        cmd = 2;
        sp_seg = 0;
        succ = G;
      }
      if (final_block) {
        st = B200Z_U_DONE;
        done = true; break;
      }
      br.refill();
      if (br.rem_bits() < 8) {  // isEOS: every byte already pulled into the bit buffer
        st = B200Z_U_EOS;
        done = true; break;
      }
      uint32_t hdr = br.peek(3);
      br.drop(3);
      final_block = hdr & 1;
      uint32_t type = hdr >> 1;
      if (type == 0) {
        // ---- stored (inflate.dart:213-235) ----
        int k = (int)(br.rem_bits() & 7);
        br.drop(k);
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
          rem_bytes = 0;  // the short read swallowed what was left
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
        if (len != 0 && len != nlen) {
          st = B200Z_U_STOP;
          done = true; break;
        }
        if (len > rem_bytes) {
          st = B200Z_U_STOP;
          done = true; break;
        }
        if (len > 0) {
          if ((unsigned long long)olen + len > cap) {
            st = B200Z_U_NOSPC;
            done = true; break;
          }
          if (len < 3) {
            const uint8_t *src = reinterpret_cast<const uint8_t *>(br.w) + br.lead + pos;
            for (int i = 0; i < (int)len; ++i) B200Z_TOK(tok, TOK_LIT | src[i]);
          } else {
            if (((nt - piece_start) & 31u) == 31u) B200Z_TOK(tok, 0u);  // the pair must not straddle a group of 32 of its piece
            B200Z_TOK(tok, TOK_STORED | ((pos >> 30) << 16) | (uint32_t)len);
            B200Z_TOK(tok, pos & 0x3fffffffu);
          }
          olen += (uint32_t)len;
        }
        br.seek(pos + (uint32_t)len);
        break;  // next token
      } else if (type == 1 || type == 2) {
        const int pst = parse_tables(br, type, lens, lut_l, lut_d, sl, sd);
        if (pst != 0) { st = pst; done = true; break; }
      } else {
        st = B200Z_U_STOP;
        done = true; break;
      }
      maxl = sl.maxlen;
      maxd = sd.maxlen;
      in_block = true;
      // a block can add 2G pieces (own, helper 1, own, helper 2 ... when every link of the chain breaks) and one more
      // closes the unit: only start helpers while the piece table has room for that
      if (spec_on && np + 2u * G + 2u <= (uint32_t)PIECE_MAX) {  // start the helpers on the rest of the input
        br.refill();
        const uint32_t p0 = 32u * br.widx - (uint32_t)br.cnt - 8u * br.lead, eb = 8u * br.in_len;
        if (eb > p0 && (eb - p0) / G >= 2u * (uint32_t)SPEC_W) {
          cmd = 1;
          cmd_p0 = p0;
          cmd_seg = (eb - p0) / G;
          sp_origin = p0;
          sp_seg = cmd_seg;
          succ = 1;
        }
      }
    }

    // ---------------- one token: _decodeHuffman (inflate.dart:300-343) -------------------------------
    br.refill();
    const bool careful = !br.fast();
    if (careful && br.rem_bits() < maxl) {  // _readCodeByTable short read (quirk Q1)
      st = U_STOP_SHORT;
      done = true; break;
    }
    uint32_t e = lut_l[br.peek(LBITS)];
    int n = e & 15;
    int sym = e >> 4;
    if (n == 0) {
      n = slow_decode<LBITS, uint16_t>(br.peek(15), sl.first, sl.count, sl.offs, sl.perm, maxl, &sym);
      if (n == 0) {  // hole: reference would emit literal 0 for ever (or until OOM)
        st = B200Z_U_BADCODE;
        done = true; break;
      }
    }
    br.drop(n);
    if (sym < 256) {
      if (olen >= cap) {
        st = B200Z_U_NOSPC;
        done = true; break;
      }
      B200Z_TOK(tok, TOK_LIT | (uint32_t)sym);
      olen++;
      break;  // next token
    }
    if (sym == 256) {
      in_block = false;
      break;  // next token
    }
    if (sym > 285) {
      st = B200Z_U_STOP;
      done = true; break;
    }
    uint32_t le = s_len_tab[sym - 257];
    int lx = le & 15;
    int mlen = (int)(le >> 4);
    if (!careful) {
      mlen += (int)br.peek(lx);
      br.drop(lx);
    } else {
      int x = 0;
      if (lx) {
        if (br.rem_bits() < lx) x = -1;  // _readBits -> -1 is ADDED to the base (inflate.dart:323)
        else { x = (int)br.peek(lx); br.drop(lx); }
      }
      mlen += x;
    }
    br.refill();
    const bool careful2 = !br.fast();
    if (careful2 && br.rem_bits() < maxd) {
      st = U_STOP_SHORT;
      done = true; break;
    }
    uint32_t de = lut_d[br.peek(DBITS)];
    int dn = de & 15;
    int dsym = de >> 4;
    if (dn == 0) {
      dn = slow_decode<DBITS, uint8_t>(br.peek(15), sd.first, sd.count, sd.offs, sd.perm, maxd, &dsym);
      if (dn == 0) dsym = 0;  // hole in the flat table: (len 0, sym 0) (_huffman_table.dart:22)
    }
    br.drop(dn);
    if (dsym > 29) {
      st = B200Z_U_STOP;
      done = true; break;
    }
    uint32_t dd = s_dist_tab[dsym];
    int dx = dd & 15;
    int dist = (int)(dd >> 4);
    if (!careful2) {
      dist += (int)br.peek(dx);
      br.drop(dx);
    } else {
      int x = 0;
      if (dx) {
        if (br.rem_bits() < dx) x = -1;
        else { x = (int)br.peek(dx); br.drop(dx); }
      }
      dist += x;
    }
    // writeBackReference (output_memory_stream.dart:79-98)
    if (dist <= 0 || (uint32_t)dist > olen + sc.hist) {  // dist 0 only via a truncated extra-bits read
      st = B200Z_U_RANGE;
      done = true; break;
    }
    if (olen + (uint32_t)mlen > cap) {
      st = B200Z_U_NOSPC;
      done = true; break;
    }
    B200Z_TOK(tok, ((uint32_t)mlen << 16) | (uint32_t)dist);
    olen += (uint32_t)mlen;
    } while (0);
  }

  if (is_master && sc.pieces) {
    piece_add(sc.pieces, np, 0u, piece_start, nt - piece_start);
    sc.pieces[0] = np;
  }
#undef B200Z_TOK
#undef h_start_tok
#undef h_ntok
#undef h_rel_bytes
#undef h_end_pos
#undef h_link_to
#undef h_link
#undef h_cur
#undef cmd
#undef cmd_p0
#undef cmd_seg
#undef m_h
#undef m_idx
#undef np
#undef piece_start
  UnitResult r;
  r.ntok = nt;
  r.out_len = olen;
  r.status = st == U_STOP_SHORT ? B200Z_U_STOP : st;
  {
    long long rem = br.rem_bits();
    if (rem < 0) rem = 0;
    r.in_used = br.in_len - (uint32_t)(rem >> 3);  // whole unread bytes are given back (inflate.dart:337-340)
    // A read that ran out of input has pulled every byte first (_readBits / _readCodeByTable loop on isEOS,
    // inflate.dart:166-168,192-195) and nothing is given back on that path: the stream is left at its end.
    if (st == U_STOP_SHORT) r.in_used = br.in_len;
  }
  return r;
}

}  // namespace b200z
