// inflate_fast.cuh -- k_inflate_fast: one CTA decodes one DEFLATE unit entirely inside shared memory.
//
// Replaces, for units whose output fits the 64 KiB window (gzip members with size hints, flush pieces of zip members):
//   lib/src/codecs/zlib/inflate.dart:104-343          _inflate / _parseBlock / _parseDynamicHuffmanBlock / _decodeHuffman
//   lib/src/codecs/zlib/_huffman_table.dart:9-46      HuffmanTable
//   lib/src/util/output_memory_stream.dart:41-98      writeByte / writeBackReference
//
// Shape (DESIGN.md "K1f"):
//   * the compressed unit arrives by ONE bulk-async copy (cp.async.bulk + mbarrier) into shared memory; the copy of the
//     NEXT unit is issued as soon as the last block of the current one is decoded, so it hides behind the LZ77 pass;
//   * a block's symbols are one serial chain, so the CTA's 256 lanes start at 256 evenly spaced bit offsets with the
//     block's tables.  Huffman streams self-synchronise: every lane marks the token boundaries of the first K bits of its
//     segment in a bitmap, then runs on into its successor's segment until one of its own boundaries is one of the
//     successor's -- from there the two parses are identical.  Lane 0 is exact, so the chain of meeting points is the
//     true parse;
//   * each lane's share of the output is counted, prefix-summed, and the lane decodes its share again straight into the
//     64 KiB output window in shared memory: literals as bytes, a match as a 3-byte record (len-3, dist-1) at its own
//     position plus one bit in a match-start bitmap (a match is >= 3 bytes long, so the record always fits);
//   * LZ77 copies are resolved shared -> shared in 1 KiB chunks, one warp per chunk, lanes owning 32 output bytes each; a
//     match waits only while bytes it reads are still owned by an unfinished match (per-warp vote inside the chunk, one
//     counter of finished chunks across warps);
//   * the finished unit leaves with one bulk-async store (shared -> global), ragged ends by byte stores.
// Nothing but the compressed bytes is read from HBM and nothing but the output is written: no token round trip.
//
// Only CLEAN units finish here: anything the reference treats specially (a read that runs out of input, an invalid or
// missing code, a distance before the start of the output, output beyond out_cap, over-subscribed code sets ...) leaves
// the unit untouched and flagged, and the exact kernels of inflate_kernels.cu decode it (they restate every quirk).
// A clean unit's result is what those kernels produce: the same bytes, out_len, in_used and status.
#pragma once
#include <stdint.h>

namespace b200z {
namespace fp {

#ifndef FP_NT
#define FP_NT 256
#endif
constexpr int NT = FP_NT;        // decode threads (= lanes of the speculative decode) per CTA; a multiple of 32
constexpr int NW = NT / 32;
#ifndef FP_XT
#define FP_XT 0
#endif
constexpr int XT = FP_XT;        // extra threads that only take part in the LZ77 pass (latency hiding); 0 or a multiple of 32
constexpr int NTT = NT + XT;     // threads the kernel is launched with
constexpr int LB = 10;           // literal/length root bits
constexpr int DB = 8;            // distance root bits
constexpr int SUBN = 384;        // second-level entries shared by the block's two alphabets
constexpr uint32_t WIN = 65536u; // output window
constexpr uint32_t IN_CAP = 30720u;  // staged compressed bytes (incl. the <= 15 bytes in front of an unaligned unit)
constexpr uint32_t MIN_IN = 192u;    // shorter units stay with the lane-per-stream kernels (a CTA each would be waste)
constexpr uint32_t MIN_SEG = 256u;   // bits per lane at least
constexpr uint32_t END_EOB = 0xfffeu, END_BAD = 0xffffu, NONE = 0xffffffffu;
constexpr uint32_t CHUNK_SHIFT = 10;  // LZ77 resolution chunk = 1024 output bytes = one warp x 32 bytes per lane
#ifndef FP_STEP
#define FP_STEP 8
#endif
#ifndef FP_TRIES
#define FP_TRIES 1
#endif
constexpr uint32_t STEP = FP_STEP;    // bytes a lane copies per batch
#ifndef FP_DYNW
#define FP_DYNW 1   // LZ77: threads take the next bitmap word off a counter (0: thread t owns words t, t + nthr, ...)
#endif
#ifndef FP_GRAN
#define FP_GRAN 1   // LZ77 with FP_DYNW: a work item is 32 >> FP_GRAN output bytes (smaller items keep the region in flight shorter)
#endif
#ifndef FP_LOOK2
#define FP_LOOK2 0  // LZ77: a look-up examines two pending matches of the item at once
#endif
#ifndef FP_LZBLK
#define FP_LZBLK 0  // 1: LZ77 by 2 KiB blocks (far matches at once, near ones by one warp) -- measured slower; 0: per-byte readiness over the whole unit
#endif
#ifndef FP_HDRAHEAD
#define FP_HDRAHEAD 1  // thread 0 parses the NEXT unit's first block header while the other warps start the LZ77 pass
#endif

// table entry: bits 0-3 code length (0: link or hole), 4-7 extra bits, 8-9 kind, 16-31 value
constexpr uint32_t K_LIT = 0u, K_BASE = 1u, K_EOB = 2u, K_INV = 3u;
constexpr uint32_t E_PARK = 1u << 12;  // table build only: root slot holds the longest code length under it

// shared memory map (bytes)
constexpr uint32_t O_WIN = 0;
constexpr uint32_t O_FLAGS = O_WIN + WIN + 16;   // u32[2048]: match starts, one bit per output byte
constexpr uint32_t O_IN = O_FLAGS + 8192;
constexpr uint32_t O_LUTL = O_IN + IN_CAP + 16;
constexpr uint32_t O_LUTD = O_LUTL + (4u << LB);
constexpr uint32_t O_SUB = O_LUTD + (4u << DB);
constexpr uint32_t O_LENS = O_SUB + 4u * SUBN;   // u8[320]
constexpr uint32_t O_GRP = O_LENS + 320;         // u32[10][16]
constexpr uint32_t O_CNT = O_GRP + 640;          // u32 cnt_l[16], cnt_d[16], first_l[16], first_d[16]
constexpr uint32_t O_LONG = O_CNT + 256;         // u32 long_l[288], long_d[32]
// (during the LZ77 pass `nf` covers O_LUTL .. O_LONG + 356; the rest of O_LONG then holds the next unit's code lengths)
constexpr uint32_t O_LENS2 = O_LONG + 368;       // u8[320]
constexpr uint32_t O_CL2 = O_LONG + 688;         // u32[128]
static_assert((2048u + 9u) * 4u <= O_LENS2 - O_LUTL && O_CL2 + 512u <= O_LONG + 1280u, "nf / header-ahead scratch");
constexpr uint32_t O_CTL = O_LONG + 1280;
constexpr uint32_t O_MBAR = O_CTL + 384;
constexpr uint32_t SMEM_BYTES = O_MBAR + 16;
static_assert(SMEM_BYTES <= 115712, "two CTAs per SM");

struct Ctl {
  // the unit being fetched (written by fetch_next, read at the top of the loop)
  uint32_t n_unit, n_in_len, n_lead, n_cap, n_wofs, n_elig;
  // the unit being decoded
  uint32_t end_bit, pos, olen, fb, done, status, cap;
  uint32_t btype, bfinal, st_src, st_len;
  uint32_t hlit, hdist, maxl, maxd, sub_used, nlong_l, nlong_d;
  uint32_t nl, L, K, bm_stride, bm_off, p0;
  uint32_t ck_off, arr_off;  // the lanes' checkpoint counts (0: none this block) and the per-lane result arrays, in the window
  uint32_t blk_end, blk_total;
  uint32_t x_state, x_olen, x_wofs;  // for the LZ77-only warps: 0 end, 1 nothing to do for this unit, 2 LZ77 over x_olen bytes
  uint32_t lz_next;                  // LZ77: the next bitmap word nobody has taken yet
  uint32_t lz_bar;                   // LZ77 by blocks: arrivals at the pass's own barrier (emulation builds only)
  uint32_t ha_valid;                 // the unit being fetched already has its first block header parsed (lens in O_LENS2)
  uint32_t regmask[NW], validmask[NW], warp_tot[NW];
};
static_assert(sizeof(Ctl) <= 384, "Ctl");

#if defined(B200Z_EMU)
#define FP_DEV inline
#define FP_SPIN()         \
  do {                    \
    cuemu::events++;      \
    cuemu::yield();       \
  } while (0)
static inline void fp_mbar_init(uint64_t *, int) {}
static inline void fp_load_bulk(void *dst, const void *src, uint32_t bytes, uint64_t *) { memcpy(dst, src, bytes); }
static inline void fp_mbar_wait(uint64_t *, uint32_t) {}
static inline void fp_store_bulk(void *gdst, const void *ssrc, uint32_t bytes) { memcpy(gdst, ssrc, bytes); }
static inline void fp_store_wait_read() {}
static inline void fp_fence_async() {}
#define FP_VOL(x) (x)
// shared memory by 32-bit address (the hot loops): here an offset from the CTA's buffer
static uint8_t *fp_emu_base = nullptr;
#define FP_SA(ptr) ((uint32_t)(reinterpret_cast<const uint8_t *>(ptr) - fp_emu_base))
#define FP_SA_INIT(base) (fp_emu_base = (base))
#define FP_LDS32(a) (*reinterpret_cast<const uint32_t *>(fp_emu_base + (a)))
#define FP_STS32(a, v) (*reinterpret_cast<uint32_t *>(fp_emu_base + (a)) = (v))
#define FP_STS8(a, v) (*(fp_emu_base + (a)) = (uint8_t)(v))
#define FP_STS16(a, v) (*reinterpret_cast<uint16_t *>(fp_emu_base + (a)) = (uint16_t)(v))
#else
#define FP_DEV __device__ __forceinline__
#define FP_SPIN() ((void)0)
__device__ __forceinline__ uint32_t fp_saddr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void fp_mbar_init(uint64_t *mb, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(fp_saddr(mb)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// one bulk-async copy global -> shared, completion counted in bytes on the mbarrier
__device__ __forceinline__ void fp_load_bulk(void *dst, const void *src, uint32_t bytes, uint64_t *mb) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(fp_saddr(mb)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(fp_saddr(dst)),
               "l"(src), "r"(bytes), "r"(fp_saddr(mb))
               : "memory");
}
__device__ __forceinline__ void fp_mbar_wait(uint64_t *mb, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(fp_saddr(mb)), "r"(parity)
        : "memory");
  } while (!done);
}
__device__ __forceinline__ void fp_store_bulk(void *gdst, const void *ssrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(fp_saddr(ssrc)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void fp_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void fp_fence_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
#define FP_VOL(x) (*(volatile uint32_t *)&(x))
// shared memory by 32-bit address (the hot loops): no generic-address arithmetic in there
#define FP_SA(ptr) fp_saddr(ptr)
#define FP_SA_INIT(base) ((void)0)
__device__ __forceinline__ uint32_t fp_lds32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ void fp_sts32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void fp_sts8(uint32_t a, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void fp_sts16(uint32_t a, uint32_t v) {
  asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "h"((unsigned short)v) : "memory");
}
#define FP_LDS32(a) fp_lds32(a)
#define FP_STS32(a, v) fp_sts32((a), (v))
#define FP_STS8(a, v) fp_sts8((a), (v))
#define FP_STS16(a, v) fp_sts16((a), (v))
#endif

// FP_PROF builds (scripts/build_variant.sh prof -DFP_PROF): thread 0 adds the clocks between the barriers of a unit to
// g_fp_prof[phase] -- where the WALL time of a unit goes, barrier waits included (the instruction counts of the ncu source
// page do not show those).  Read and cleared by b200z_debug_fast_prof.
#ifdef FP_PROF
__device__ unsigned long long g_fp_prof[24];
#define FP_TICK(k)                                                          \
  do {                                                                      \
    if (tid == 0) {                                                         \
      const long long t_ = clock64();                                       \
      atomicAdd(&g_fp_prof[k], (unsigned long long)(t_ - tl_));             \
      tl_ = t_;                                                             \
    }                                                                       \
  } while (0)
// ... and every warp's lane 0 adds the clocks it WAITED at the barrier that ends pass A / A2 / the false-start count / C /
// LZ77 to g_fp_prof[12 + k] (sum over the CTA's warps: 8 x the phase's clocks would mean everybody waited all the time)
#define FP_ARR() ta_ = clock64()
#define FP_TICKW(k)                                                                      \
  do {                                                                                   \
    if (lane == 0) atomicAdd(&g_fp_prof[12 + (k)], (unsigned long long)(clock64() - ta_)); \
  } while (0)
#else
#define FP_TICK(k)
#define FP_ARR()
#define FP_TICKW(k)
#endif

// Two kinds of CTA barrier: FP_DSYNC among the NT decode threads (everything up to the LZ77 pass), FP_ASYNC among all NTT
// threads (around the LZ77 pass).  Without extra warps they are the same barrier.
#if defined(B200Z_EMU) || FP_XT == 0
#define FP_DSYNC() __syncthreads()
#define FP_ASYNC() __syncthreads()
#else
#define FP_STR2(x) #x
#define FP_STR(x) FP_STR2(x)
#define FP_DSYNC() asm volatile("bar.sync 1, " FP_STR(FP_NT) ";" ::: "memory")
#define FP_ASYNC() __syncthreads()
#endif

// ---- bit reader over the staged input (LSB first, inflate.dart:159-184); pos = bits consumed from word 0 ----
struct BR {
  uint64_t buf;
  int cnt;
  uint32_t wp;
};
FP_DEV void br_seek(BR &b, const uint32_t *in32, uint32_t bitpos) {
  const uint32_t w = bitpos >> 5, sh = bitpos & 31u;
  const uint64_t v = (uint64_t)in32[w] | ((uint64_t)in32[w + 1] << 32);
  b.buf = v >> sh;
  b.cnt = 64 - (int)sh;
  b.wp = w + 2;
}
FP_DEV void br_refill(BR &b, const uint32_t *in32) {
  if (b.cnt < 32) {
    b.buf |= (uint64_t)in32[b.wp] << b.cnt;
    b.cnt += 32;
    b.wp++;
  }
}
FP_DEV uint32_t br_pos(const BR &b) { return b.wp * 32u - (uint32_t)b.cnt; }
FP_DEV void br_seek_sa(BR &b, uint32_t s_in, uint32_t bitpos) {  // br_seek by shared address
  const uint32_t w = bitpos >> 5, sh = bitpos & 31u;
  const uint64_t v = (uint64_t)FP_LDS32(s_in + w * 4u) | ((uint64_t)FP_LDS32(s_in + w * 4u + 4u) << 32);
  b.buf = v >> sh;
  b.cnt = 64 - (int)sh;
  b.wp = w + 2;
}

FP_DEV uint32_t fp_lookup(uint32_t bits, bool dm, const uint32_t *lutl, const uint32_t *lutd, const uint32_t *sub) {
  uint32_t e = dm ? lutd[bits & ((1u << DB) - 1u)] : lutl[bits & ((1u << LB) - 1u)];
  if ((e & 15u) == 0u && e != 0u) {  // link to the second level
    const uint32_t sb = (e >> 4) & 15u;
    e = sub[(e >> 16) + ((bits >> (dm ? DB : LB)) & ((1u << sb) - 1u))];
  }
  return e;  // (e & 15) == 0: no code here
}


// ---- the bulk of every pass: one symbol per turn, the same instructions for literal/length and distance symbols (a lane
// that has read a length code reads its distance code next turn), tables and input by 32-bit shared address, state
// updated by selects.  It only ever COMMITS ordinary symbols; whatever needs thought -- end of
// block, an invalid code, the last 32 bits of the input, the place this lane has to stop at -- ends the loop BEFORE the
// symbol is consumed, and the careful step of the calling pass decodes that symbol again with all its checks.
//   MODE 0  pass A : count bytes, mark token boundaries in the lane's bitmap, stop at the end of the segment; the first
//                    boundary marked in a bitmap word also records the byte count there (its checkpoint)
//   MODE 1  pass A2: count bytes, stop at a boundary the successor has marked too (or beyond its window)
//   MODE 2  false-start count: count bytes, stop at `stop`
//   MODE 3  pass C : write bytes / match records into the window, stop at `stop`
#ifdef FP_DEBUG
static unsigned long fp_dbg_restarts = 0, fp_dbg_fastiters = 0;
// false starts counted: from a checkpoint that is the meeting point / from a checkpoint before it / from the guessed
// offset because the block has no checkpoints or the lane's count outgrew them
static unsigned long fp_dbg_ck_exact = 0, fp_dbg_ck_walk = 0, fp_dbg_ck_full = 0;
#endif
struct FastCtx {
  uint32_t s_in, s_lutl, s_lutd, s_sub;  // shared addresses: staged input, the two root tables, the second level
  uint32_t end_bit, stop;         // bits of the unit; where this lane stops (a token boundary >= stop), NONE = never
  uint32_t org, K, s_row;         // MODE 0: my segment start / window / my bitmap row; MODE 1: the successor's
  uint32_t s_ck;                  // MODE 0: my row of checkpoint counts (u16 per bitmap word), NONE = none this block
  uint32_t s_W;                   // MODE 3: shared address of output byte 0
  uint32_t *flags;                // MODE 3: match-start bitmap
};
template <int MODE>
FP_DEV bool fp_fast(BR &br, bool &dm_io, uint32_t &pend_io, uint32_t &acc_io, uint32_t &tokpos_io, const FastCtx &c) {
  // the bit window: w0:w1 hold the 64 bits at word `posw / 32`, nx the word behind them (asked for one crossing ahead, so
  // its latency is off the chain); sh = bits of w0 already consumed
  uint32_t pos0 = br_pos(br);
  uint32_t posw = pos0 & ~31u, sh = pos0 & 31u;
  uint32_t pa = c.s_in + (posw >> 3);
  uint32_t w0 = FP_LDS32(pa), w1 = FP_LDS32(pa + 4u), nx = FP_LDS32(pa + 8u);
  pa += 8u;
  uint32_t pend = pend_io, acc = acc_io, tokpos = tokpos_io;
  bool trouble = false;
  const uint32_t LM4 = ((1u << LB) - 1u) << 2, DM4 = ((1u << DB) - 1u) << 2;
  uint32_t tb = dm_io ? c.s_lutd : c.s_lutl, tm = dm_io ? DM4 : LM4;
  // a token that starts with 48 bits of input left needs no end-of-input test at all (15 + 5 + 15 + 13 bits at most)
  const uint32_t stop2 = c.end_bit >= 48u ? min(c.stop, c.end_bit - 47u) : 0u;
  for (;;) {
    const bool dm = tb != c.s_lutl;
    const uint32_t pos = posw + sh;
#ifdef FP_DEBUG
    fp_dbg_fastiters++;
#endif
    if (!dm) {
      tokpos = pos;
      if (pos >= stop2) break;
      if (MODE == 0) {
        const uint32_t rel = pos - c.org;
        if (rel < c.K) {
          const uint32_t a = c.s_row + ((rel >> 5) << 2), old = FP_LDS32(a);
          FP_STS32(a, old | (1u << (rel & 31u)));
          if (old == 0u && c.s_ck != NONE) FP_STS16(c.s_ck + ((rel >> 5) << 1), acc);
        }
      }
      if (MODE == 1) {
        const uint32_t off = pos - c.org;  // (the caller only comes here once pos >= org)
        if (off >= c.K) break;
        if ((FP_LDS32(c.s_row + ((off >> 5) << 2)) >> (off & 31u)) & 1u) break;
      }
    }
    const uint32_t bits = __funnelshift_r(w0, w1, sh);
    uint32_t e = FP_LDS32(tb + ((bits << 2) & tm));
    if ((e & 15u) == 0u && e != 0u)  // a code longer than the root index: its entry is in the second level
      e = FP_LDS32(c.s_sub + (((e >> 16) + ((bits >> (tm == LM4 ? LB : DB)) & ~(0xffffffffu << ((e >> 4) & 15u)))) << 2));
    if (((e & 0x20fu) - 1u) >= 15u) break;  // no code here, end of block, invalid
    const uint32_t n = e & 15u, xb = (e >> 4) & 15u;
    const uint32_t val = (e >> 16) + ((bits >> n) & ~(0xffffffffu << xb));
    const bool isbase = !dm && (e & 0x100u) != 0u;
    if (MODE == 3) {
      if (dm) {
        if (val > acc) {  // writeBackReference before the start of the output (output_memory_stream.dart:83-86)
          trouble = true;
          break;
        }
        const uint32_t a = c.s_W + acc;
        FP_STS8(a, pend - 3u);
        FP_STS8(a + 1u, val - 1u);
        FP_STS8(a + 2u, (val - 1u) >> 8);
        atomicOr(&c.flags[acc >> 5], 1u << (acc & 31u));
      } else if (!isbase) {
        FP_STS8(c.s_W + acc, val);
      }
    }
    sh += n + xb;
    if (sh >= 32u) {
      sh -= 32u;
      posw += 32u;
      w0 = w1;
      w1 = nx;
      pa += 4u;
      nx = FP_LDS32(pa);
    }
    acc += dm ? pend : (isbase ? 0u : 1u);
    pend = isbase ? val : pend;
    tb = isbase ? c.s_lutd : c.s_lutl;
    tm = isbase ? DM4 : LM4;
  }
  br_seek_sa(br, c.s_in, posw + sh);
  dm_io = tb != c.s_lutl;
  pend_io = pend;
  acc_io = acc;
  tokpos_io = tokpos;
  return trouble;
}

FP_DEV uint32_t fp_entry(uint32_t s, uint32_t l, bool dist) {
  uint32_t kind, val, xb = 0;
  if (dist) {
    if (s < 30u) {
      const uint32_t t = c_dist_tab[s];
      kind = K_BASE;
      val = t >> 4;
      xb = t & 15u;
    } else {
      kind = K_INV;
      val = 0;
    }
  } else if (s < 256u) {
    kind = K_LIT;
    val = s;
  } else if (s == 256u) {
    kind = K_EOB;
    val = 0;
  } else if (s <= 285u) {
    const uint32_t t = c_len_tab[s - 257u];
    kind = K_BASE;
    val = t >> 4;
    xb = t & 15u;
  } else {
    kind = K_INV;
    val = 0;
  }
  return (val << 16) | (kind << 8) | (xb << 4) | l;
}

// thread 0: the CTA's next unit (units are dealt round-robin); a unit that can be decoded here gets its bulk load issued
FP_DEV void fp_fetch_next(Ctl *ctl, uint8_t *s_in, uint64_t *mbar, const uint8_t *in_base, const uint64_t *in_off,
                          const uint32_t *in_len, const uint8_t *out_base, const uint64_t *out_off, const uint32_t *out_cap,
                          uint32_t n_units, uint32_t u) {
  if (u >= n_units) {
    ctl->n_unit = NONE;
    return;
  }
  const uint8_t *src = in_base + in_off[u];
  const uint32_t il = in_len[u], oc = out_cap[u];
  const uint32_t lead = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 15u);
  const uint32_t bytes = (lead + il + 15u) & ~15u;
  const bool elig = il >= MIN_IN && bytes <= IN_CAP && oc <= WIN && oc != 0u;
  ctl->n_unit = u;
  ctl->n_in_len = il;
  ctl->n_lead = lead;
  ctl->n_cap = oc;
  ctl->n_wofs = (uint32_t)(reinterpret_cast<uintptr_t>(out_base + out_off[u]) & 15u);
  ctl->n_elig = elig ? 1u : 0u;
  if (elig) fp_load_bulk(s_in, src - lead, bytes, mbar);
}

// thread 0: the unit fetch_next has announced becomes the unit being decoded
FP_DEV void fp_unit_begin(Ctl *ctl) {
  ctl->end_bit = (ctl->n_lead + ctl->n_in_len) * 8u;
  ctl->pos = ctl->n_lead * 8u;
  ctl->olen = 0;
  ctl->fb = 0;
  ctl->done = 0;
  ctl->status = B200Z_U_DONE;
  ctl->bfinal = 0;
  ctl->cap = ctl->n_cap;
}

// thread 0: _parseBlock header (inflate.dart:120-156, 213-298) -- clean cases only, anything else sets ctl->fb
FP_DEV void fp_parse_header(Ctl *ctl, const uint8_t *s_in, uint8_t *lens, uint32_t *cl_lut) {
  const uint32_t *in32 = reinterpret_cast<const uint32_t *>(s_in);
  const uint32_t end_bit = ctl->end_bit;
  uint32_t pos = ctl->pos;
  if (end_bit - pos < 8u) {  // isEOS at a block boundary (inflate.dart:111): every byte already pulled
    ctl->done = 1;
    ctl->status = B200Z_U_EOS;
    return;
  }
  BR br;
  br_seek(br, in32, pos);
#define FP_NEED(n)                       \
  if (br_pos(br) + (n) > end_bit) {      \
    ctl->fb = 1;                         \
    return;                              \
  }
#define FP_GET(var, n)                                   \
  br_refill(br, in32);                                   \
  FP_NEED(n)                                             \
  var = (uint32_t)br.buf & ((1u << (n)) - 1u);           \
  br.buf >>= (n);                                        \
  br.cnt -= (n);
  uint32_t hdr;
  FP_GET(hdr, 3)
  ctl->bfinal = hdr & 1u;
  const uint32_t type = hdr >> 1;
  ctl->btype = type;
  if (type == 0u) {
    uint32_t p = (br_pos(br) + 7u) & ~7u;
    if (p + 32u > end_bit) {  // the short reads of LEN / NLEN are the exact kernels' business
      ctl->fb = 1;
      return;
    }
    const uint32_t b = p >> 3;
    const uint32_t len = s_in[b] | ((uint32_t)s_in[b + 1] << 8), nlen = (s_in[b + 2] | ((uint32_t)s_in[b + 3] << 8)) ^ 0xffffu;
    if ((len != 0u && len != nlen) || len > ((end_bit - p) >> 3) - 4u || ctl->olen + len > ctl->cap) {
      ctl->fb = 1;
      return;
    }
    ctl->st_src = b + 4u;
    ctl->st_len = len;
    ctl->pos = p + 32u + 8u * len;
    return;
  }
  if (type == 1u) {
    ctl->hlit = 288;
    ctl->hdist = 30;
    ctl->p0 = br_pos(br);
    return;
  }
  if (type != 2u) {
    ctl->fb = 1;
    return;
  }
  uint32_t hlit, hdist, hclen;
  FP_GET(hlit, 5)
  FP_GET(hdist, 5)
  FP_GET(hclen, 4)
  hlit += 257u;
  hdist += 1u;
  hclen += 4u;
  if (hlit > 288u || hdist > 32u || hclen > 19u) {
    ctl->fb = 1;
    return;
  }
  // code-length alphabet: 7-bit table, entries (sym << 4) | len
  for (uint32_t i = 0; i < hclen; ++i) {
    uint32_t l;
    FP_GET(l, 3)
    lens[c_order[i]] = (uint8_t)l;  // scratch: the first 19 bytes of lens
  }
  for (uint32_t i = hclen; i < 19u; ++i) lens[c_order[i]] = 0;
  {
    uint32_t count[8], next[8];
    for (int l = 0; l < 8; ++l) count[l] = 0;
    for (int i = 0; i < 19; ++i) count[lens[i] & 7]++;
    count[0] = 0;
    int left = 1;
    uint32_t code = 0;
    next[0] = 0;
    for (int l = 1; l < 8; ++l) {
      left = (left << 1) - (int)count[l];
      if (left < 0) {  // over-subscribed
        ctl->fb = 1;
        return;
      }
      code = (code + count[l - 1]) << 1;
      next[l] = code;
    }
    for (int i = 0; i < 128; ++i) cl_lut[i] = 0;
    for (uint32_t s = 0; s < 19u; ++s) {
      const uint32_t l = lens[s];
      if (l == 0u) continue;
      const uint32_t c = next[l]++;
      const uint32_t r = __brev(c) >> (32 - l);
      for (uint32_t j = r; j < 128u; j += 1u << l) cl_lut[j] = (s << 4) | l;
    }
  }
  // _decode (inflate.dart:345-401)
  const uint32_t num = hlit + hdist;
  uint32_t i = 0, prev = 0;
  while (i < num) {
    br_refill(br, in32);
    const uint32_t e = cl_lut[(uint32_t)br.buf & 127u];
    const uint32_t l = e & 15u, code = e >> 4;
    if (l == 0u || br_pos(br) + 16u > end_bit) {  // hole, or close enough to the end for a short read to matter
      ctl->fb = 1;
      return;
    }
    br.buf >>= l;
    br.cnt -= (int)l;
    if (code < 16u) {
      lens[i++] = (uint8_t)code;
      prev = code;
      continue;
    }
    uint32_t rep;
    if (code == 16u) {
      rep = ((uint32_t)br.buf & 3u) + 3u;
      br.buf >>= 2;
      br.cnt -= 2;
    } else if (code == 17u) {
      rep = ((uint32_t)br.buf & 7u) + 3u;
      br.buf >>= 3;
      br.cnt -= 3;
      prev = 0;
    } else {
      rep = ((uint32_t)br.buf & 127u) + 11u;
      br.buf >>= 7;
      br.cnt -= 7;
      prev = 0;
    }
    if (i + rep > num) {  // RangeError in the reference
      ctl->fb = 1;
      return;
    }
    for (uint32_t k = 0; k < rep; ++k) lens[i++] = (uint8_t)prev;
  }
  if (br_pos(br) > end_bit) {
    ctl->fb = 1;
    return;
  }
  ctl->hlit = hlit;
  ctl->hdist = hdist;
  ctl->p0 = br_pos(br);
#undef FP_GET
#undef FP_NEED
}

// thread 0: how many lanes decode the block, their segment length, sync window and where the boundary bitmaps live
FP_DEV void fp_plan_lanes(Ctl *ctl, uint32_t wofs) {
  const uint32_t R = ctl->end_bit - ctl->p0;
  uint32_t nl = R / MIN_SEG;
  if (nl > (uint32_t)NT) nl = NT;
  const uint32_t used = wofs + ctl->olen;
  const uint32_t room = (WIN + 16u - used) & ~3u;  // the part of the window this block has not reached yet
  uint32_t L = 0, K = 0;
  for (;;) {
    if (nl < 2u) {
      nl = 1;
      break;
    }
    L = R / nl;
    K = (L < 1024u ? L : 1024u) & ~31u;  // as wide as the segment (a wider window could place a lane's start behind its end)
    while (K >= 128u && nl * (K / 32u + 1u) * 4u > room) K = (K >> 1) & ~31u;
    if (K >= 128u) break;
    nl = room / ((128u / 32u + 1u) * 4u);  // as many lanes as a 128-bit window each fits
    if (nl > (uint32_t)NT) nl = NT;
    if (nl >= 2u && R / nl < 128u) nl = R / 128u;
  }
  ctl->nl = nl;
  ctl->L = nl > 1u ? L : 0u;
  ctl->K = nl > 1u ? K : 0u;
  const uint32_t bms = nl > 1u ? K / 32u + 1u : 0u;  // (+1: one spare word, and rows that do not all start in one bank)
  ctl->bm_stride = bms;
  ctl->bm_off = nl > 1u ? ((WIN + 16u - nl * bms * 4u) & ~3u) : 0u;
  // Below the bitmaps, if the room holds them: the checkpoint counts (u16 per bitmap word) and the lanes' result arrays
  // (tgt, pos, start).  The bitmaps then stay intact until the false starts are counted.  Otherwise -- late blocks of a
  // unit whose output nearly fills the window -- the arrays take the dead bitmaps' place and every false start is decoded
  // from its guessed offset.  (K is chosen as if there were no checkpoints: it decides which lanes meet.)
  const uint32_t ckb = (nl * bms * 2u + 3u) & ~3u;
  const bool ck = nl > 1u && nl * bms * 4u + ckb + nl * 12u <= room;
  ctl->ck_off = ck ? ctl->bm_off - ckb : 0u;
  ctl->arr_off = ck ? ctl->bm_off - ckb - nl * 12u : ctl->bm_off;
}

// ---------------- LZ77: matches copy shared -> shared ----------------
// A match may copy as soon as the bytes it reads are final -- nothing else orders the copies.  (Measured on the
// benchmark text: 7.6 k matches per 64 KiB unit, longest chain of matches that feed each other 42.)  So finality is
// tracked per BYTE: `nf` holds one bit per output byte that a match still has to write (literals are final from the
// start); it lives where the block's code tables were, which are dead by now.  Every thread owns the bitmap words
// t, t + nthr, ... (32 output bytes each) and keeps trying the pending matches of its current word: a match whose source
// bits are all clear copies (up to STEP bytes per batch, loaded before they are stored) and then clears its own bits.
// The earliest pending match of the unit is always ready, so the loop ends; threads never wait for each other otherwise.
// Every thread of the CTA runs this, the decode lanes and -- when the kernel is built with some (FP_XT) -- the extra
// warps that exist for this pass only: it is bound by latency, and more warps hide more of it.
FP_DEV void fp_lz77_prep(uint8_t *smem, uint32_t tid, uint32_t nthr, uint32_t olen, uint32_t wofs) {
  uint32_t *const flags = reinterpret_cast<uint32_t *>(smem + O_FLAGS);
  uint8_t *const W = smem + O_WIN + wofs;
    uint32_t *const nf = reinterpret_cast<uint32_t *>(smem + O_LUTL);
    const uint32_t nwords = (olen + 31u) >> 5;
    for (uint32_t i = tid; i < nwords + 9u && i < 2048u + 8u; i += nthr) nf[i] = 0;
    FP_ASYNC();
    for (uint32_t w = tid; w < nwords; w += nthr) {
      uint32_t f = flags[w];
      while (f) {
        const uint32_t b = (uint32_t)(__ffs((int)f) - 1);
        f &= f - 1u;
        const uint32_t a = w * 32u + b, e = a + (uint32_t)W[a] + 3u;  // bytes [a, e) are this match's
        const uint32_t wa = a >> 5, wb = (e - 1u) >> 5;
        if (wa == wb) {
          atomicOr(&nf[wa], (0xffffffffu << (a & 31u)) & (0xffffffffu >> (31u - ((e - 1u) & 31u))));
        } else {
          atomicOr(&nf[wa], 0xffffffffu << (a & 31u));
          for (uint32_t q = wa + 1u; q < wb; ++q) atomicOr(&nf[q], 0xffffffffu);
          atomicOr(&nf[wb], 0xffffffffu >> (31u - ((e - 1u) & 31u)));
        }
      }
    }
    FP_ASYNC();
}

// (a thread may enter late: with FP_DYNW the words it would have owned are simply taken by the others)
FP_DEV void fp_lz77_run(uint8_t *smem, uint32_t tid, uint32_t nthr, uint32_t olen, uint32_t wofs) {
  const unsigned FULL = 0xffffffffu;
  uint32_t *const flags = reinterpret_cast<uint32_t *>(smem + O_FLAGS);
  uint8_t *const W = smem + O_WIN + wofs;
    uint32_t *const nf = reinterpret_cast<uint32_t *>(smem + O_LUTL);
    const uint32_t nwords = (olen + 31u) >> 5;
    const uint32_t s_Wr = FP_SA(W), s_nf = FP_SA(nf);
#if FP_DYNW
    // work items are handed out in position order off a counter: item q = output bytes [q * IB, (q + 1) * IB)
    constexpr uint32_t G = FP_GRAN, IB = 32u >> G;
    const uint32_t nitems = nwords << G;
    uint32_t *const lz_next = &reinterpret_cast<Ctl *>(smem + O_CTL)->lz_next;
#define FP_ITEM_BITS(q) ((q) < nitems ? flags[(q) >> G] & ((0xffffffffu >> (32u - IB)) << (((q) & ((1u << G) - 1u)) * IB)) : 0u)
    uint32_t w = atomicAdd(lz_next, 1u);
    uint32_t f = FP_ITEM_BITS(w), cand = f;
#else
    constexpr uint32_t G = 0;
    const uint32_t nitems = nwords;
#define FP_ITEM_BITS(q) ((q) < nitems ? flags[q] : 0u)
    uint32_t w = tid;
    uint32_t f = FP_ITEM_BITS(w), cand = f;
#endif
    bool has = false;  // a match of mine is ready and waits for the warp's next copy turn
    uint32_t rp = 0, rlen = 0, rdist = 0, rb = 0;
#ifdef FP_PROF
    // lane 0 of each warp: clocks probing (the looks before a turn) and in copy turns; turns, the sum and the maximum of
    // the ready lengths per turn; every lane: looks and failed looks.  Added to g_fp_prof[17 ..] when the pass ends.
    unsigned long long pr_probe = 0, pr_copy = 0, pr_turns = 0, pr_tsum = 0, pr_tmax = 0;
    uint32_t pr_looks = 0, pr_fail = 0;
    long long pr_t = clock64();
#define FP_LOOK(ok) (++pr_looks, pr_fail += (ok) ? 0u : 1u)
#else
#define FP_LOOK(ok)
#endif
    for (;;) {
      // ---- look for a ready match (lanes that hold one wait for the warp's next copy turn).  With FP_TRIES > 1 a warp
      // takes up to FP_TRIES looks before a turn and stops early once 20 lanes hold one; with one look per turn (the
      // default) there is nothing to stop, and the vote is not taken: it cost 4 % of bench.py config 2 ----
#pragma unroll 1
      for (int tries = 0; tries < FP_TRIES; ++tries) {
        if (!has && w < nitems) {
          if (f == 0u) {  // this item's matches are done: the next one (the kernel clears the bitmap behind the pass)
#if FP_DYNW
            w = atomicAdd(lz_next, 1u);
#else
            w += nthr;
#endif
            f = FP_ITEM_BITS(w);
            cand = f;
          }
          if (f != 0u) {
            if (cand == 0u) cand = f;  // another sweep over what is still pending here
            // is the match at bit b of my word ready?  (its 3-byte record read as one unaligned word; [src, last] must be final)
            auto probe = [&](uint32_t b, uint32_t &len, uint32_t &dist) -> bool {
              const uint32_t p = (w >> G) * 32u + b;
              const uint32_t ra = s_Wr + p;
              const uint32_t rec = __funnelshift_r(FP_LDS32(ra & ~3u), FP_LDS32((ra & ~3u) + 4u), (ra & 3u) * 8u);
              len = (rec & 0xffu) + 3u;
              dist = ((rec >> 8) & 0xffffu) + 1u;
              const uint32_t src = p - dist, last = min(src + len, p) - 1u;
              const uint32_t wa = src >> 5, wb = last >> 5;
              const uint32_t mlo = 0xffffffffu << (src & 31u), mhi = 0xffffffffu >> (31u - (last & 31u));
              // (the same instructions whether the source lies in one bitmap word or two; longer sources are rare)
              const uint32_t nfa = FP_LDS32(s_nf + wa * 4u), nfb = FP_LDS32(s_nf + wb * 4u);
              uint32_t busy = wa == wb ? (nfa & mlo & mhi) : ((nfa & mlo) | (nfb & mhi));
              if (wb > wa + 1u)
                for (uint32_t q = wa + 1u; q < wb; ++q) busy |= FP_LDS32(s_nf + q * 4u);
              return busy == 0u;
            };
            const uint32_t b0 = (uint32_t)(__ffs((int)cand) - 1);
            cand &= cand - 1u;
            uint32_t len0, dist0;
#if FP_LOOK2
            // two candidates a look: their chains of loads overlap, and a look fails less often
            const bool two = cand != 0u;
            const uint32_t b1 = two ? (uint32_t)(__ffs((int)cand) - 1) : b0;
            cand &= cand - 1u;
            uint32_t len1, dist1;
            const bool r0 = probe(b0, len0, dist0), r1 = probe(b1, len1, dist1);
            FP_LOOK(r0 || r1);
            if (r0 || r1) {
              has = true;
              rb = r0 ? b0 : b1;
              rlen = r0 ? len0 : len1;
              rdist = r0 ? dist0 : dist1;
              rp = (w >> G) * 32u + rb;
            }
#else
            const bool r0 = probe(b0, len0, dist0);
            FP_LOOK(r0);
            if (r0) {
              has = true;
              rb = b0;
              rlen = len0;
              rdist = dist0;
              rp = (w >> G) * 32u + rb;
            }
#endif
          }
        }
        if (FP_TRIES > 1 && tries == 0 && __popc(__ballot_sync(FULL, has)) >= 20) break;
      }
      if (__ballot_sync(FULL, has || w < nitems) == 0u) break;
#ifdef FP_PROF
      {
        const unsigned ready = __ballot_sync(FULL, has);
        const uint32_t tsum = __reduce_add_sync(FULL, has ? rlen : 0u), tmax = __reduce_max_sync(FULL, has ? rlen : 0u);
        const long long t = clock64();
        pr_probe += (unsigned long long)(t - pr_t);
        pr_t = t;
        if (ready) {
          ++pr_turns;
          pr_tsum += tsum;
          pr_tmax += tmax;
        }
      }
#endif
      if (has) {
        __threadfence_block();  // the bytes behind the clear bits are visible
        // overlapping run (dist < len, dist < STEP): [p - dist, p + k) is final and periodic, so any multiple of dist that
        // does not reach back beyond p - dist serves as the distance: it doubles until a batch moves STEP bytes
        uint32_t back = rdist;
        for (uint32_t k = 0; k < rlen;) {
          if (back < STEP && 2u * back <= k + rdist) back <<= 1;
          const uint32_t m = min(rlen - k, min(STEP, back));
          const uint8_t *sp = W + rp + k - back;
          uint8_t *dp = W + rp + k;
          uint8_t r[STEP];
#pragma unroll
          for (uint32_t t = 0; t < STEP; ++t) r[t] = sp[t];  // (reading past the m-th byte is harmless)
#pragma unroll
          for (uint32_t t = 0; t < STEP; ++t)
            if (t < m) dp[t] = r[t];
          k += m;
        }
        __threadfence_block();  // ... before the bits say so
        {
          const uint32_t e = rp + rlen, wa = rp >> 5, wb = (e - 1u) >> 5;
          if (wa == wb) {
            atomicAnd(&nf[wa], ~((0xffffffffu << (rp & 31u)) & (0xffffffffu >> (31u - ((e - 1u) & 31u)))));
          } else {
            atomicAnd(&nf[wa], ~(0xffffffffu << (rp & 31u)));
            for (uint32_t q = wa + 1u; q < wb; ++q) atomicAnd(&nf[q], 0u);
            atomicAnd(&nf[wb], ~(0xffffffffu >> (31u - ((e - 1u) & 31u))));
          }
        }
        f &= ~(1u << rb);
        has = false;
      }
#ifdef FP_PROF
      __syncwarp();
      {
        const long long t = clock64();
        pr_copy += (unsigned long long)(t - pr_t);
        pr_t = t;
      }
#endif
    }
#ifdef FP_PROF
    {
      const uint32_t looks = __reduce_add_sync(FULL, pr_looks), fails = __reduce_add_sync(FULL, pr_fail);
      if ((tid & 31u) == 0u) {
        atomicAdd(&g_fp_prof[17], pr_probe);
        atomicAdd(&g_fp_prof[18], pr_copy);
        atomicAdd(&g_fp_prof[19], pr_turns);
        atomicAdd(&g_fp_prof[20], pr_tsum);
        atomicAdd(&g_fp_prof[21], pr_tmax);
        atomicAdd(&g_fp_prof[22], (unsigned long long)looks);
        atomicAdd(&g_fp_prof[23], (unsigned long long)fails);
      }
    }
#endif
#undef FP_LOOK
#undef FP_ITEM_BITS
}

FP_DEV void fp_lz77(uint8_t *smem, uint32_t tid, uint32_t nthr, uint32_t olen, uint32_t wofs) {
  fp_lz77_prep(smem, tid, nthr, olen, wofs);
  fp_lz77_run(smem, tid, nthr, olen, wofs);
}

// ---------------- LZ77 by blocks (-DFP_LZBLK=1; measured and NOT the default) ----------------
// The pass above lets every thread retry the matches of its 16 bytes until their sources are final: with 4 KiB in flight
// and a median distance of 3.4 KB three looks out of four fail.  Here the output is taken in blocks of 2 KiB, in order,
// by warps 1 .. 7 (warp 0 parses the next unit's header meanwhile):
//   * a match of block b whose source ends before block b - 1 reads final bytes whatever happens -- every block before
//     b - 1 is complete -- and copies at once, no look, no retry (3 threads share a bitmap word: matches 0, 3, 6 .. of the
//     word, 1, 4, 7 .., 2, 5, 8 ..);  a source that ends inside block b - 1 is final unless it touches a byte a NEAR match
//     of that block still has to write (one look at that block's pending bitmap);
//   * what is left -- sources that reach into the match's own block, or into pending bytes of the block before -- is a
//     NEAR match: it is listed, its bytes are marked pending, and ONE warp resolves the list (per-byte readiness as above,
//     but over 2 KiB and ~60 matches) while the other six warps already take the far matches of block b + 1.
// One barrier (among the seven warps) per block.
// Measured (config 2): the pass takes about twice the clocks per unit of the per-byte pass above.  The chains of matches that feed each other (depth 42 per unit) are chains of NEAR matches, and here
// they are walked block after block by one warp -- ~10 dependent rounds in each of 32 blocks -- where the
// per-byte pass lets the chains of different regions advance side by side.  Kept as a build option (the emulation tier
// builds and checks it in tests/test_inflate_fast_emul.py::test_lz77_by_blocks_build_option).
constexpr uint32_t LZ_BL = 2048u, LZ_WB = LZ_BL / 32u;  // bytes / bitmap words per block
constexpr uint32_t LZ_NW = NW - 1u;                     // warps 1 .. NW - 1
constexpr uint32_t LZ_PW = LZ_WB + 10u;                 // pending bitmap: the block and the 258 bytes behind it
constexpr uint32_t LZ_NEAR_CAP = 704u;                  // near matches per block (a match is >= 3 bytes long: <= 683)
static_assert(LZ_NW * 32u == 3u * LZ_WB + 32u, "six warps = three threads per bitmap word of a block");
static_assert((2u * LZ_PW + 2u) * 4u + 2u * LZ_NEAR_CAP * 2u <= (O_LONG + 356u) - O_LUTL, "LZ77 scratch in the dead table space");

FP_DEV void fp_lzsync(Ctl *ctl) {
#if defined(B200Z_EMU)
  const uint32_t n = LZ_NW * 32u;
  const uint32_t t = atomicAdd(&ctl->lz_bar, 1u);
  const uint32_t target = (t / n + 1u) * n;
  while (FP_VOL(ctl->lz_bar) < target) FP_SPIN();
#else
  asm volatile("bar.sync 2, %0;" ::"n"(LZ_NW * 32) : "memory");
#endif
}

// bits [a, e] (inclusive) of a bitmap: any set / set them / clear them
FP_DEV uint32_t fp_bits_any(const uint32_t *bm, uint32_t a, uint32_t e) {
  const uint32_t wa = a >> 5, wb = e >> 5;
  const uint32_t mlo = 0xffffffffu << (a & 31u), mhi = 0xffffffffu >> (31u - (e & 31u));
  if (wa == wb) return FP_VOL(bm[wa]) & mlo & mhi;
  uint32_t busy = (FP_VOL(bm[wa]) & mlo) | (FP_VOL(bm[wb]) & mhi);
  for (uint32_t q = wa + 1u; q < wb; ++q) busy |= FP_VOL(bm[q]);
  return busy;
}
FP_DEV void fp_bits_or(uint32_t *bm, uint32_t a, uint32_t e) {
  const uint32_t wa = a >> 5, wb = e >> 5;
  const uint32_t mlo = 0xffffffffu << (a & 31u), mhi = 0xffffffffu >> (31u - (e & 31u));
  if (wa == wb) {
    atomicOr(&bm[wa], mlo & mhi);
  } else {
    atomicOr(&bm[wa], mlo);
    for (uint32_t q = wa + 1u; q < wb; ++q) atomicOr(&bm[q], 0xffffffffu);
    atomicOr(&bm[wb], mhi);
  }
}
FP_DEV void fp_bits_clear(uint32_t *bm, uint32_t a, uint32_t e) {
  const uint32_t wa = a >> 5, wb = e >> 5;
  const uint32_t mlo = 0xffffffffu << (a & 31u), mhi = 0xffffffffu >> (31u - (e & 31u));
  if (wa == wb) {
    atomicAnd(&bm[wa], ~(mlo & mhi));
  } else {
    atomicAnd(&bm[wa], ~mlo);
    for (uint32_t q = wa + 1u; q < wb; ++q) atomicAnd(&bm[q], 0u);
    atomicAnd(&bm[wb], ~mhi);
  }
}

// the copy of one match whose source is final (writeBackReference, output_memory_stream.dart:79-98): STEP bytes per batch,
// loaded before they are stored.  Overlapping run (dist < len, dist < STEP): [p - dist, p + k) is final and periodic, so any
// multiple of dist that does not reach back beyond p - dist serves as the distance: it doubles until a batch moves STEP bytes
FP_DEV void fp_lz_copy(uint8_t *W, uint32_t rp, uint32_t rlen, uint32_t rdist) {
  uint32_t back = rdist;
  for (uint32_t k = 0; k < rlen;) {
    if (back < STEP && 2u * back <= k + rdist) back <<= 1;
    const uint32_t m = min(rlen - k, min(STEP, back));
    const uint8_t *sp = W + rp + k - back;
    uint8_t *dp = W + rp + k;
    uint8_t r[STEP];
#pragma unroll
    for (uint32_t t = 0; t < STEP; ++t) r[t] = sp[t];  // (reading past the m-th byte is harmless)
#pragma unroll
    for (uint32_t t = 0; t < STEP; ++t)
      if (t < m) dp[t] = r[t];
    k += m;
  }
}

// the 3-byte record at the first bytes of a match: len - 3, dist - 1
FP_DEV void fp_lz_record(uint32_t s_Wr, uint32_t p, uint32_t &len, uint32_t &dist) {
  const uint32_t ra = s_Wr + p;
  const uint32_t rec = __funnelshift_r(FP_LDS32(ra & ~3u), FP_LDS32((ra & ~3u) + 4u), (ra & 3u) * 8u);
  len = (rec & 0xffu) + 3u;
  dist = ((rec >> 8) & 0xffffu) + 1u;
}

// warps 1 .. NW - 1 (tid >= 32)
FP_DEV void fp_lz77_blocks(uint8_t *smem, uint32_t tid, uint32_t olen, uint32_t wofs) {
  const unsigned FULL = 0xffffffffu;
  Ctl *const ctl = reinterpret_cast<Ctl *>(smem + O_CTL);
  const uint32_t *const flags = reinterpret_cast<const uint32_t *>(smem + O_FLAGS);
  uint8_t *const W = smem + O_WIN + wofs;
  uint32_t *const pend = reinterpret_cast<uint32_t *>(smem + O_LUTL);  // [2][LZ_PW]
  uint32_t *const nnear = pend + 2u * LZ_PW;                            // [2]
  uint16_t *const nearl = reinterpret_cast<uint16_t *>(nnear + 2);     // [2][LZ_NEAR_CAP]: position - start of the block
  const uint32_t lt = tid - 32u, lw = lt >> 5, lane = lt & 31u;
  const uint32_t s_Wr = FP_SA(W);
  for (uint32_t i = lt; i < 2u * LZ_PW + 2u; i += LZ_NW * 32u) pend[i] = 0u;
  fp_lzsync(ctl);
  const uint32_t nwords = (olen + 31u) >> 5, nblk = (olen + LZ_BL - 1u) / LZ_BL;
  for (uint32_t it = 0; it <= nblk; ++it) {
    const uint32_t near_w = (it + LZ_NW - 1u) % LZ_NW;  // the warp that resolves the near matches of block it - 1
    if (lw == near_w) {
      if (it > 0u) {
        // ---- the near matches of block it - 1: a lane owns entries lane, lane + 32, .. and goes round those still pending ----
        const uint32_t b = (it - 1u) & 1u, bs = (it - 1u) * LZ_BL;
        uint32_t *const pb = pend + b * LZ_PW;
        const uint16_t *const nl = nearl + b * LZ_NEAR_CAP;
        const uint32_t n = FP_VOL(nnear[b]);
        uint32_t todo = 0u;
        for (uint32_t i = lane, k = 0; i < n; i += 32u, ++k) todo |= 1u << k;
        uint32_t cand = todo;
        while (__ballot_sync(FULL, todo != 0u) != 0u) {
          if (todo != 0u) {
            if (cand == 0u) cand = todo;
            const uint32_t k = (uint32_t)(__ffs((int)cand) - 1);
            cand &= cand - 1u;
            const uint32_t rel = nl[lane + 32u * k], p = bs + rel;
            uint32_t len, dist;
            fp_lz_record(s_Wr, p, len, dist);
            const uint32_t src = p - dist, last = min(src + len, p) - 1u;
            // (everything before this block is final by now: only bytes of the block itself can be pending)
            const bool ready = last < bs || fp_bits_any(pb, (src > bs ? src : bs) - bs, last - bs) == 0u;
            if (ready) {
              __threadfence_block();  // the bytes behind the clear bits are visible
              fp_lz_copy(W, p, len, dist);
              __threadfence_block();  // ... before the bits say so
              fp_bits_clear(pb, rel, rel + len - 1u);
              todo &= ~(1u << k);
            }
          }
        }
        __syncwarp();
        if (lane == 0u) nnear[b] = 0u;
      }
    } else if (it < nblk) {
      // ---- block `it`: far matches copy at once, near ones are listed ----
      const uint32_t b = it & 1u, bs = it * LZ_BL, ps = bs - (it > 0u ? LZ_BL : 0u);
      uint32_t *const pb = pend + b * LZ_PW;
      const uint32_t *const pprev = pend + (b ^ 1u) * LZ_PW;
      uint16_t *const nl = nearl + b * LZ_NEAR_CAP;
      const uint32_t q = (lw < near_w ? lw : lw - 1u) * 32u + lane;  // 0 .. 191
      const uint32_t w = q / 3u, gw = it * LZ_WB + w;
      uint32_t c = q - 3u * w;  // my matches: set bits number c, c + 3, .. of the word
      uint32_t f = gw < nwords ? flags[gw] : 0u;
      while (f) {
        const uint32_t bit = (uint32_t)(__ffs((int)f) - 1);
        f &= f - 1u;
        if (c != 0u) {
          c--;
          continue;
        }
        c = 2u;
        const uint32_t p = gw * 32u + bit;
        uint32_t len, dist;
        fp_lz_record(s_Wr, p, len, dist);
        const uint32_t src = p - dist, last = min(src + len, p) - 1u;
        bool near = last >= bs;
        if (!near && it > 0u && last >= ps)  // ends inside the block before: final unless a near match of that block is pending there
          near = fp_bits_any(pprev, (src > ps ? src : ps) - ps, last - ps) != 0u;
        if (near) {
          const uint32_t slot = atomicAdd(&nnear[b], 1u);
          nl[slot] = (uint16_t)(p - bs);
          fp_bits_or(pb, p - bs, p - bs + len - 1u);
        } else {
          __threadfence_block();
          fp_lz_copy(W, p, len, dist);
        }
      }
    }
    __threadfence_block();
    fp_lzsync(ctl);
  }
}

}  // namespace fp

#ifdef B200Z_EMU
#define FP_DYN_SMEM(name) uint8_t *name = reinterpret_cast<uint8_t *>(cuemu_dyn_smem)
#else
#define FP_DYN_SMEM(name) extern __shared__ __align__(16) uint8_t name[]
#endif

__global__ void __launch_bounds__(fp::NTT, 2)
k_inflate_fast(const uint8_t *__restrict__ in_base, const uint64_t *__restrict__ in_off, const uint32_t *__restrict__ in_len,
               uint8_t *__restrict__ out_base, const uint64_t *__restrict__ out_off, const uint32_t *__restrict__ out_cap,
               uint32_t *__restrict__ out_len, int32_t *__restrict__ status, uint32_t *__restrict__ in_used, uint32_t n_units,
               uint32_t *__restrict__ doneflag, uint32_t flag_stride, uint32_t *__restrict__ next_unit) {
  using namespace fp;
  FP_DYN_SMEM(fsmem);
  uint8_t *const smem = fsmem;
  uint8_t *const win = smem + O_WIN;
  uint32_t *const flags = reinterpret_cast<uint32_t *>(smem + O_FLAGS);
  uint8_t *const s_in = smem + O_IN;
  const uint32_t *const in32 = reinterpret_cast<const uint32_t *>(s_in);
  uint32_t *const lutl = reinterpret_cast<uint32_t *>(smem + O_LUTL);
  uint32_t *const lutd = reinterpret_cast<uint32_t *>(smem + O_LUTD);
  uint32_t *const sub = reinterpret_cast<uint32_t *>(smem + O_SUB);
  uint8_t *const lens = smem + O_LENS;
  uint32_t *const grp = reinterpret_cast<uint32_t *>(smem + O_GRP);
  uint32_t *const cnt_l = reinterpret_cast<uint32_t *>(smem + O_CNT);
  uint32_t *const cnt_d = cnt_l + 16, *const first_l = cnt_l + 32, *const first_d = cnt_l + 48;
  uint32_t *const long_l = reinterpret_cast<uint32_t *>(smem + O_LONG);
  uint32_t *const long_d = long_l + 288;
  Ctl *const ctl = reinterpret_cast<Ctl *>(smem + O_CTL);
  uint64_t *const mbar = reinterpret_cast<uint64_t *>(smem + O_MBAR);

  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const unsigned FULL = 0xffffffffu;
  FP_SA_INIT(smem);
  FastCtx fc;
  fc.s_in = FP_SA(s_in);
  fc.s_lutl = FP_SA(lutl);
  fc.s_lutd = FP_SA(lutd);
  fc.s_sub = FP_SA(sub);
  fc.s_ck = NONE;
  fc.flags = flags;

  if (tid >= (uint32_t)NT) {  // the LZ77-only warps (FP_XT): two CTA-wide barriers per unit, the pass in between
    for (;;) {
      FP_ASYNC();  // (A) the unit's blocks are decoded, or there is nothing to do
      const uint32_t xs = ctl->x_state, xo = ctl->x_olen, xw = ctl->x_wofs;
      if (xs == 0u) return;
      if (xs == 2u) fp_lz77(smem, tid, NTT, xo, xw);
      FP_ASYNC();  // (B)
    }
  }
  for (uint32_t i = tid; i < 2048u; i += NT) flags[i] = 0;
  // units come off a counter in global memory (zeroed by the launcher): a CTA that starts late -- behind a collective's
  // kernel that holds part of an SM -- then simply takes fewer of them
  if (tid == 0) {
    fp_mbar_init(mbar, 1);
    ctl->ha_valid = 0;
    fp_fetch_next(ctl, s_in, mbar, in_base, in_off, in_len, out_base, out_off, out_cap, n_units, atomicAdd(next_unit, 1u));
  }
  uint32_t phase = 0;
#ifdef FP_PROF
  long long tl_ = clock64(), ta_ = 0;
#endif
  for (;;) {
    if (tid == 0) fp_store_wait_read();  // the previous unit's bulk store has read the window
    FP_DSYNC();
    FP_TICK(0);
    const uint32_t unit = ctl->n_unit;
    if (unit == NONE) {
      if (tid == 0) ctl->x_state = 0;
      FP_ASYNC();  // (A): releases the LZ77-only warps for good
      break;
    }
    const uint32_t u_in_len = ctl->n_in_len, lead = ctl->n_lead, cap = ctl->n_cap, wofs = ctl->n_wofs;
    const bool elig = ctl->n_elig != 0u;
    bool ahead = ctl->ha_valid != 0u;  // thread 0 has parsed the first block header already (behind the previous unit's LZ77 pass)
    uint8_t *const W = win + wofs;  // W[q] = output byte q; W is congruent to the global destination modulo 16
    FP_DSYNC();
    if (!elig) {
      if (tid == 0) {
        doneflag[(size_t)unit * flag_stride] = 0;
        ctl->x_state = 1;
        fp_fetch_next(ctl, s_in, mbar, in_base, in_off, in_len, out_base, out_off, out_cap, n_units, atomicAdd(next_unit, 1u));
      }
      FP_ASYNC();  // (A)
      FP_ASYNC();  // (B)
      continue;
    }
    fp_mbar_wait(mbar, phase);
    phase ^= 1u;
    FP_TICK(1);
    if (tid == 0) {
      if (!ahead) fp_unit_begin(ctl);
      ctl->ha_valid = 0;
    }
    FP_DSYNC();
    const uint32_t end_bit = (lead + u_in_len) * 8u;

    // ======================= blocks =======================
    for (;;) {
      if (ahead) {  // the unit's first block: its code lengths wait in O_LENS2
        for (uint32_t i = tid; i < 80u; i += NT)
          reinterpret_cast<uint32_t *>(lens)[i] = reinterpret_cast<const uint32_t *>(smem + O_LENS2)[i];
        ahead = false;
      } else if (tid == 0) {
        if (ctl->bfinal) {
          ctl->done = 1;
          ctl->status = B200Z_U_DONE;
        } else {
          fp_parse_header(ctl, s_in, lens, sub);
          if (!ctl->fb && !ctl->done && ctl->btype != 0u) fp_plan_lanes(ctl, wofs);
        }
      }
      FP_DSYNC();
      FP_TICK(2);
      if (ctl->fb || ctl->done) break;
      const uint32_t btype = ctl->btype;
      if (btype == 0u) {  // stored (inflate.dart:213-235): input bytes -> window
        const uint32_t src = ctl->st_src, n = ctl->st_len, o = ctl->olen;
        for (uint32_t i = tid; i < n; i += NT) W[o + i] = s_in[src + i];
        FP_DSYNC();
        if (tid == 0) ctl->olen = o + n;
        continue;
      }
      const uint32_t hlit = ctl->hlit, hdist = ctl->hdist;
      // ---------------- tables (HuffmanTable, _huffman_table.dart:9-46, as root + second level) ----------------
      if (btype == 1u) {
        for (uint32_t i = tid; i < 320u; i += NT) lens[i] = i < 144u ? 8 : i < 256u ? 9 : i < 280u ? 7 : i < 288u ? 8 : 5;
      }
      for (uint32_t i = tid; i < (1u << LB); i += NT) lutl[i] = 0;
      for (uint32_t i = tid; i < (1u << DB); i += NT) lutd[i] = 0;
      for (uint32_t i = tid; i < (uint32_t)fp::SUBN; i += NT) sub[i] = 0;
      for (uint32_t i = tid; i < 160u; i += NT) grp[i] = 0;
      if (tid == 0) {
        ctl->sub_used = 0;
        ctl->nlong_l = 0;
        ctl->nlong_d = 0;
      }
      FP_DSYNC();
      // a symbol's canonical code = first[l] + (symbols of the same length before it): groups of 32 symbols, ranks by match_any
      const uint32_t ngl = (hlit + 31u) >> 5;  // groups 0..ngl-1 literal/length, group 9 distance
      uint32_t my_l[2] = {0, 0}, my_rank[2] = {0, 0}, my_s[2] = {0, 0}, my_g[2] = {NONE, NONE};
#pragma unroll
      for (int k = 0; k < 2; ++k) {  // warp w: groups w and w + 8
        const uint32_t g = warp + (uint32_t)k * NW;
        if (g >= 10u || (g >= ngl && g != 9u)) continue;
        const bool dist = g == 9u;
        const uint32_t s = dist ? lane : g * 32u + lane;
        const uint32_t l = dist ? (s < hdist ? lens[hlit + s] : 0u) : (s < hlit ? lens[s] : 0u);
        const unsigned m = __match_any_sync(FULL, l);
        if (l != 0u && (m & ((1u << lane) - 1u)) == 0u) grp[g * 16u + l] = (uint32_t)__popc(m);
        my_l[k] = l;
        my_rank[k] = (uint32_t)__popc(m & ((1u << lane) - 1u));
        my_s[k] = s;
        my_g[k] = g;
      }
      FP_DSYNC();
      if (warp == 0) {
        if (lane < 16u) {
          uint32_t p = 0;
          for (uint32_t g = 0; g < ngl; ++g) {
            const uint32_t t = grp[g * 16u + lane];
            grp[g * 16u + lane] = p;
            p += t;
          }
          cnt_l[lane] = p;
        } else {
          const uint32_t l = lane - 16u;
          cnt_d[l] = grp[9u * 16u + l];
          grp[9u * 16u + l] = 0;
        }
        __syncwarp();
        if (lane < 2u) {  // lane 0: literal/length, lane 1: distance -- Kraft sum, first codes, longest code
          uint32_t *cnt = lane ? cnt_d : cnt_l, *first = lane ? first_d : first_l;
          int left = 1;
          uint32_t code = 0, mx = 0;
          bool over = false;
          first[0] = 0;
          cnt[0] = 0;
          for (uint32_t l = 1; l < 16u; ++l) {
            left = (left << 1) - (int)cnt[l];
            if (left < 0) over = true;
            code = (code + cnt[l - 1]) << 1;
            first[l] = code;
            if (cnt[l]) mx = l;
          }
          if (over) ctl->fb = 1;  // over-subscribed: the reference's flat table decodes garbage (exact kernels: BADCODE)
          if (lane) ctl->maxd = mx;
          else ctl->maxl = mx;
        }
      }
      FP_DSYNC();
      if (ctl->fb) break;
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const uint32_t l = my_l[k];
        if (my_g[k] == NONE || l == 0u) continue;
        const bool dist = my_g[k] == 9u;
        const uint32_t code = (dist ? first_d : first_l)[l] + grp[my_g[k] * 16u + l] + my_rank[k];
        const uint32_t r = __brev(code) >> (32u - l);
        const uint32_t RB = dist ? DB : LB;
        if (l <= RB) {
          const uint32_t e = fp_entry(my_s[k], l, dist);
          uint32_t *lut = dist ? lutd : lutl;
          for (uint32_t j = r; j < (1u << RB); j += 1u << l) lut[j] = e;
        } else {
          const uint32_t slot = atomicAdd(dist ? &ctl->nlong_d : &ctl->nlong_l, 1u);
          (dist ? long_d : long_l)[slot] = (r << 16) | (l << 10) | my_s[k];
        }
      }
      FP_DSYNC();
      if (tid == 0 || tid == 32) {  // codes longer than the root: one thread per alphabet places them
        const bool dist = tid != 0;
        const uint32_t RB = dist ? DB : LB, n = dist ? ctl->nlong_d : ctl->nlong_l;
        const uint32_t *list = dist ? long_d : long_l;
        uint32_t *lut = dist ? lutd : lutl;
        for (uint32_t i = 0; i < n; ++i) {  // the longest code under every root prefix
          const uint32_t it = list[i], r = it >> 16, l = (it >> 10) & 15u;
          uint32_t &slot = lut[r & ((1u << RB) - 1u)];
          if ((slot >> 16) < l) slot = (l << 16) | E_PARK;
        }
        for (uint32_t i = 0; i < n; ++i) {
          const uint32_t it = list[i], r = it >> 16, l = (it >> 10) & 15u, s = it & 1023u;
          uint32_t &slot = lut[r & ((1u << RB) - 1u)];
          if (slot & E_PARK) {
            const uint32_t sb = (slot >> 16) - RB;
            const uint32_t base = atomicAdd(&ctl->sub_used, 1u << sb);
            if (base + (1u << sb) > (uint32_t)fp::SUBN) {
              ctl->fb = 1;  // pool exhausted (pathological code sets)
              break;
            }
            slot = (base << 16) | (sb << 4) | (1u << 8);  // link: length nibble 0, not zero as a word
          }
          const uint32_t sb = (slot >> 4) & 15u, base = slot >> 16;
          const uint32_t e = fp_entry(s, l, dist);
          for (uint32_t j = r >> RB; j < (1u << sb); j += 1u << (l - RB)) sub[base + j] = e;
        }
      }
      FP_DSYNC();
      FP_TICK(3);
      if (ctl->fb) break;

      // ---------------- pass A: every lane decodes its segment, marking token boundaries ----------------
      const uint32_t nl = ctl->nl, L = ctl->L, K = ctl->K, bms = ctl->bm_stride, p0 = ctl->p0;
      const uint32_t maxl = ctl->maxl, maxd = ctl->maxd, olen0 = ctl->olen;
      uint32_t *const bm = reinterpret_cast<uint32_t *>(win + ctl->bm_off);
      uint16_t *const ck = ctl->ck_off != 0u ? reinterpret_cast<uint16_t *>(win + ctl->ck_off) : nullptr;
      // per-lane results of the block (fp_plan_lanes places them; one lane: the group counters')
      uint32_t *const tgt_arr = nl > 1u ? reinterpret_cast<uint32_t *>(win + ctl->arr_off) : grp, *const pos_arr = tgt_arr + nl,
                     *const start_arr = tgt_arr + 2u * nl;
      const bool lane_on = tid < nl;
      const uint32_t myS = p0 + tid * L;
      const uint32_t segEnd = (tid + 1u < nl) ? myS + L : NONE;
      uint32_t sprime = myS, G = 0, pend = 0, tokpos = myS;
      uint32_t tgt = END_BAD, endpos = 0;
      bool dm = false;
      int state = 2;  // 0 running, 1 at the end of the segment, 2 ended
      BR br;
      br.buf = 0;
      br.cnt = 0;
      br.wp = 0;
      fc.end_bit = end_bit;
      fc.K = K;
      if (lane_on) {
        if (nl > 1u)
          for (uint32_t w = 0; w < bms; ++w) bm[tid * bms + w] = 0;
        br_seek(br, in32, sprime);
        state = 0;
        fc.stop = segEnd;
        fc.org = myS;
        fc.s_row = FP_SA(bm + tid * bms);
        fc.s_ck = ck ? FP_SA(ck + tid * bms) : NONE;
      }
      // (the warp meets at every turn of these loops: a lane that leaves the bulk loop early must not run on by itself)
      while (__any_sync(FULL, state == 0)) {
        if (state == 0) do {  // (break / continue: end of this lane's turn)
          fp_fast<0>(br, dm, pend, G, tokpos, fc);  // the bulk; what follows is the careful step for the symbol it stopped at
          br_refill(br, in32);
          const uint32_t pos = br_pos(br);
          if (!dm) {
            tokpos = pos;
            if (pos >= segEnd) {
              state = 1;
              break;
            }
            const uint32_t rel = pos - myS;
            if (rel < K) {
              uint32_t &bw = bm[tid * bms + (rel >> 5)];
              if (bw == 0u && ck) ck[tid * bms + (rel >> 5)] = (uint16_t)G;
              bw |= 1u << (rel & 31u);
            }
          }
          const int rem = (int)(end_bit - pos);
          const uint32_t bits = (uint32_t)br.buf;
          const uint32_t e = fp_lookup(bits, dm, lutl, lutd, sub);
          const uint32_t n = e & 15u, xb = (e >> 4) & 15u, kind = (e >> 8) & 3u;
          bool bad = n == 0u || kind == K_INV;
          if (rem < 32) bad = bad || rem < (int)(dm ? maxd : maxl) || (int)(n + xb) > rem;
          if (bad || kind == K_EOB) {
            // a lane that dies while it still decodes from its guessed offset has lost nothing: guess again one bit on
            // (its checkpoint counts need no clearing: a word's count is written again with the word's first new mark)
            if (tid > 0u && tokpos + 1u - myS < K / 2u) {
              for (uint32_t w = 0; w < bms; ++w) bm[tid * bms + w] = 0;
              sprime = tokpos + 1u;
#ifdef FP_DEBUG
              fp_dbg_restarts++;
#endif
              br_seek(br, in32, sprime);
              G = 0;
              dm = false;
              continue;
            }
            if (!bad) {
              tgt = END_EOB;
              endpos = pos + n;
            } else {
              tgt = END_BAD;
              endpos = tokpos;
            }
            state = 2;
            break;
          }
          const uint32_t val = (e >> 16) + ((bits >> n) & ((1u << xb) - 1u));
          const uint32_t tot = n + xb;
          br.buf >>= tot;
          br.cnt -= (int)tot;
          if (dm) {
            G += pend;
            dm = false;
          } else if (kind == K_LIT) {
            G += 1u;
          } else {
            pend = val;
            dm = true;
          }
        } while (0);
      }
      FP_ARR();
      FP_DSYNC();
      FP_TICK(4);
      FP_TICKW(0);
      // ---------------- pass A2: run on until one of my boundaries is one of a successor's ----------------
      {
        uint32_t succ = tid + 1u, succS = myS + L;
        while (__any_sync(FULL, state == 1)) {
          if (state == 1) do {
          if (succ < nl && (dm || br_pos(br) >= succS)) {  // in (or heading for) the successor's window: test its marks
            fc.stop = NONE;
            fc.org = succS;
            fc.s_row = FP_SA(bm + succ * bms);
            fp_fast<1>(br, dm, pend, G, tokpos, fc);
          } else {  // between windows, or no lane left to meet
            fc.stop = succ < nl ? succS : NONE;
            fp_fast<2>(br, dm, pend, G, tokpos, fc);
          }
          br_refill(br, in32);
          const uint32_t pos = br_pos(br);
          if (!dm) {
            tokpos = pos;
            while (succ < nl && pos >= succS + K) {  // through that lane's window without meeting it: it is lost
              succ++;
              succS += L;
            }
            if (succ < nl && pos >= succS) {
              const uint32_t off = pos - succS;
              if ((bm[succ * bms + (off >> 5)] >> (off & 31u)) & 1u) {
                tgt = succ;
                endpos = pos;
                state = 2;
                break;
              }
            }
          }
          const int rem = (int)(end_bit - pos);
          const uint32_t bits = (uint32_t)br.buf;
          const uint32_t e = fp_lookup(bits, dm, lutl, lutd, sub);
          const uint32_t n = e & 15u, xb = (e >> 4) & 15u, kind = (e >> 8) & 3u;
          bool bad = n == 0u || kind == K_INV;
          if (rem < 32) bad = bad || rem < (int)(dm ? maxd : maxl) || (int)(n + xb) > rem;
          if (bad) {
            tgt = END_BAD;
            endpos = tokpos;
            state = 2;
            break;
          }
          if (kind == K_EOB) {
            tgt = END_EOB;
            endpos = pos + n;
            state = 2;
            break;
          }
          const uint32_t val = (e >> 16) + ((bits >> n) & ((1u << xb) - 1u));
          const uint32_t tot = n + xb;
          br.buf >>= tot;
          br.cnt -= (int)tot;
          if (dm) {
            G += pend;
            dm = false;
          } else if (kind == K_LIT) {
            G += 1u;
          } else {
            pend = val;
            dm = true;
          }
          } while (0);
        }
      }
      FP_ARR();
      FP_DSYNC();  // every lane is through with the bitmaps (they share the window with nothing live, but the lane arrays follow)
      FP_TICK(5);
      FP_TICKW(1);
      // ---------------- the chain of meeting points from lane 0 is the true parse ----------------
      if (lane_on) {
        tgt_arr[tid] = tgt;
        pos_arr[tid] = endpos;
      }
      {
        const unsigned reg = __ballot_sync(FULL, lane_on && tgt == tid + 1u);
        if (lane == 0) {
          ctl->regmask[warp] = reg;
          ctl->validmask[warp] = 0;
        }
      }
      FP_DSYNC();
      if (tid == 0) {
        uint32_t cur = 0;
        bool ok = false;
        for (int it = 0; it < NT; ++it) {
          uint32_t w = cur >> 5;
          uint32_t m = ~ctl->regmask[w] & (0xffffffffu << (cur & 31u));
          while (m == 0u && w + 1u < (uint32_t)NW) m = ~ctl->regmask[++w];
          if (m == 0u) break;
          const uint32_t E = w * 32u + (uint32_t)(__ffs((int)m) - 1);
          for (uint32_t q = cur >> 5; q <= (E >> 5); ++q) {  // lanes cur..E are on the chain
            uint32_t bits = 0xffffffffu;
            if (q == (cur >> 5)) bits &= 0xffffffffu << (cur & 31u);
            if (q == (E >> 5)) bits &= 0xffffffffu >> (31u - (E & 31u));
            ctl->validmask[q] |= bits;
          }
          const uint32_t t = tgt_arr[E];
          if (t == END_EOB) {
            ok = true;
            ctl->blk_end = pos_arr[E];
            break;
          }
          if (t == END_BAD || t <= E || t >= nl) break;
          cur = t;  // lanes in between never met the true parse: skipped
        }
        if (!ok) ctl->fb = 1;
      }
      FP_DSYNC();
      if (ctl->fb) break;
#ifdef FP_DEBUG
      if (tid == 0) { int nv = 0; for (int w = 0; w < NW; ++w) nv += __popc(ctl->validmask[w]); fprintf(stderr, "unit %u: nl %u L %u K %u valid %d restarts %lu fastiters %lu\n", unit, nl, L, K, nv, fp::fp_dbg_restarts, fp::fp_dbg_fastiters); for (uint32_t q = 0; q < nl; ++q) if (!((ctl->validmask[q >> 5] >> (q & 31)) & 1u)) fprintf(stderr, "   lane %u invalid: tgt %u endpos-rel %d ; pred tgt %u pred endrel %d\n", q, tgt_arr[q], (int)(pos_arr[q] - (p0 + q * L)), tgt_arr[q-1], (int)(pos_arr[q-1] - (p0 + q * L))); }
#endif
      const bool valid = ((ctl->validmask[warp] >> lane) & 1u) != 0u;
      if (valid && tgt < END_EOB) start_arr[tgt] = endpos;
      FP_DSYNC();
      FP_TICK(6);
      const uint32_t start = !valid ? 0u : tid == 0u ? p0 : start_arr[tid];
      // ---------------- the bytes of my false start (my guessed offset .. where the true parse met me) ----------------
      // `start` is one of my own marks, so the checkpoint of its bitmap word -- the word's first mark and my byte count
      // there -- lies at or before it on my parse: at most 31 bits are decoded again.  Without checkpoints this block, or
      // with a count too large for them, the whole false start is.
      uint32_t nbytes = 0;
      bool incons = false;
      {
        uint32_t f = 0, p3 = 0, t3 = sprime;
        bool d3 = false, go3 = valid && start != sprime;
        const bool from_ck = go3 && ck && G <= 0xffffu;  // (counts only grow: then every checkpoint count kept all its bits)
        if (from_ck) {
          const uint32_t j = (start - myS) >> 5;
          t3 = myS + j * 32u + (uint32_t)(__ffs((int)bm[tid * bms + j]) - 1);
          f = ck[tid * bms + j];
          go3 = t3 != start;
        }
#ifdef FP_DEBUG
        if (valid && start != sprime) (!from_ck ? fp_dbg_ck_full : go3 ? fp_dbg_ck_walk : fp_dbg_ck_exact)++;
#endif
        BR b3;
        b3.buf = 0;
        b3.cnt = 0;
        b3.wp = 0;
        if (go3) br_seek(b3, in32, t3);
        fc.stop = start;
        while (__any_sync(FULL, go3)) {
          if (go3) do {
            fp_fast<2>(b3, d3, p3, f, t3, fc);
            br_refill(b3, in32);
            const uint32_t pos = br_pos(b3);
            if (!d3 && pos >= start) {
              incons = pos != start;
              go3 = false;
              break;
            }
            const uint32_t bits = (uint32_t)b3.buf;
            const uint32_t e = fp_lookup(bits, d3, lutl, lutd, sub);
            const uint32_t n = e & 15u, xb = (e >> 4) & 15u, kind = (e >> 8) & 3u;
            if (n == 0u || kind >= K_EOB) {
              incons = true;
              go3 = false;
              break;
            }
            const uint32_t val = (e >> 16) + ((bits >> n) & ((1u << xb) - 1u));
            const uint32_t tot = n + xb;
            b3.buf >>= tot;
            b3.cnt -= (int)tot;
            if (d3) {
              f += p3;
              d3 = false;
            } else if (kind == K_LIT) {
              f += 1u;
            } else {
              p3 = val;
              d3 = true;
            }
          } while (0);
        }
        if (valid) nbytes = G - f;
      }
      // exclusive prefix sum of the lanes' byte counts
      uint32_t incl = nbytes;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t v = __shfl_up_sync(FULL, incl, d);
        if (lane >= (uint32_t)d) incl += v;
      }
      if (lane == 31u) ctl->warp_tot[warp] = incl;
      if (incons) ctl->fb = 1;
      FP_ARR();
      FP_DSYNC();
      FP_TICK(7);
      FP_TICKW(2);
      uint32_t wbase = 0, total = 0;
#pragma unroll
      for (int w = 0; w < NW; ++w) {
        const uint32_t t = ctl->warp_tot[w];
        if ((uint32_t)w < warp) wbase += t;
        total += t;
      }
      if (ctl->fb || olen0 + total > cap) {  // beyond out_cap: B200Z_U_NOSPC is the exact kernels' to report
        if (tid == 0) ctl->fb = 1;
        FP_DSYNC();
        FP_TICK(7);
        break;
      }
      // ---------------- pass C: my share of the block again, into the window ----------------
      {
        uint32_t o = olen0 + wbase + incl - nbytes;
        BR bc;
        bc.buf = 0;
        bc.cnt = 0;
        bc.wp = 0;
        bool dc = false, goc = valid, trouble = false;
        uint32_t pc = 0, tc = start;
        if (goc) br_seek(bc, in32, start);
        fc.stop = tgt < END_EOB ? endpos : NONE;
        fc.s_W = FP_SA(W);
        while (__any_sync(FULL, goc)) {
          if (goc) do {
            if (fp_fast<3>(bc, dc, pc, o, tc, fc)) {
              trouble = true;
              goc = false;
              break;
            }
            br_refill(bc, in32);
            const uint32_t pos = br_pos(bc);
            if (!dc && tgt < END_EOB && pos >= endpos) {
              trouble = pos != endpos;
              goc = false;
              break;
            }
            const uint32_t bits = (uint32_t)bc.buf;
            const uint32_t e = fp_lookup(bits, dc, lutl, lutd, sub);
            const uint32_t n = e & 15u, xb = (e >> 4) & 15u, kind = (e >> 8) & 3u;
            if (kind == K_EOB && n != 0u) {
              goc = false;
              break;
            }
            if (n == 0u || kind == K_INV) {
              trouble = true;
              goc = false;
              break;
            }
            const uint32_t val = (e >> 16) + ((bits >> n) & ((1u << xb) - 1u));
            const uint32_t tot = n + xb;
            bc.buf >>= tot;
            bc.cnt -= (int)tot;
            if (dc) {
              if (val > o) {  // writeBackReference before the start of the output (output_memory_stream.dart:83-86)
                trouble = true;
                goc = false;
                break;
              }
              W[o] = (uint8_t)(pc - 3u);
              W[o + 1u] = (uint8_t)(val - 1u);
              W[o + 2u] = (uint8_t)((val - 1u) >> 8);
              atomicOr(&flags[o >> 5], 1u << (o & 31u));
              o += pc;
              dc = false;
            } else if (kind == K_LIT) {
              W[o++] = (uint8_t)val;
            } else {
              pc = val;
              dc = true;
            }
          } while (0);
        }
        if (trouble) ctl->fb = 1;
      }
      FP_ARR();
      FP_DSYNC();
      FP_TICK(8);
      FP_TICKW(3);
      if (ctl->fb) break;
      if (tid == 0) {
        ctl->olen = olen0 + total;
        ctl->pos = ctl->blk_end;
      }
      // (the barrier at the top of the loop publishes olen / pos before anyone reads them)
      FP_DSYNC();
    }

    // ======================= the unit's blocks are decoded (or the unit is given up) =======================
    const bool fb = ctl->fb != 0u;
    const uint32_t olen = ctl->olen, fin_status = ctl->status, fin_pos = ctl->pos;
    FP_DSYNC();
    if (tid == 0) {
      ctl->x_state = fb ? 1u : 2u;
      ctl->x_olen = olen;
      ctl->x_wofs = wofs;
      ctl->lz_next = 0;
      ctl->lz_bar = 0;
      // the staged input is dead: fetch the next unit behind the LZ77 pass
      fp_fetch_next(ctl, s_in, mbar, in_base, in_off, in_len, out_base, out_off, out_cap, n_units, atomicAdd(next_unit, 1u));
    }
    FP_ASYNC();  // (A)
    FP_TICK(9);
    if (fb) {
      for (uint32_t i = tid; i < 2048u; i += NT) flags[i] = 0;
      if (tid == 0) doneflag[(size_t)unit * flag_stride] = 0;
      FP_ASYNC();  // (B)
      continue;
    }
#if FP_LZBLK && FP_XT == 0
    // Warp 0: the next unit's input is on its way (fetch_next above) and its first block header is a serial parse by one
    // thread (measured: a tenth of a unit's clocks with everybody else at the barrier) -- it is parsed now, behind the
    // LZ77 pass of the other seven warps.
    if (warp == 0u) {
      if (ctl->n_unit != NONE && ctl->n_elig != 0u) {
        fp_mbar_wait(mbar, phase);  // (`phase` is the next load's parity by now; the wait at the top of the loop sees the same)
        if (tid == 0) {
          fp_unit_begin(ctl);
          fp_parse_header(ctl, s_in, smem + O_LENS2, reinterpret_cast<uint32_t *>(smem + O_CL2));
          if (!ctl->fb && !ctl->done && ctl->btype != 0u) fp_plan_lanes(ctl, ctl->n_wofs);
          ctl->ha_valid = 1;
        }
        __syncwarp();
      }
    } else {
      fp_lz77_blocks(smem, tid, olen, wofs);
    }
#else
    fp_lz77_prep(smem, tid, NTT, olen, wofs);
#if FP_HDRAHEAD
    // The next unit's input is on its way (fetch_next above) and its first block header is a serial parse by one thread
    // (measured: a tenth of a unit's clocks with everybody else at the barrier).  Warp 0 does it now, the other warps
    // start on the matches, and warp 0 joins them afterwards.
    if (warp == 0u && ctl->n_unit != NONE && ctl->n_elig != 0u) {
      fp_mbar_wait(mbar, phase);  // (`phase` is the next load's parity by now; the wait at the top of the loop sees the same)
      if (tid == 0) {
        fp_unit_begin(ctl);
        fp_parse_header(ctl, s_in, smem + O_LENS2, reinterpret_cast<uint32_t *>(smem + O_CL2));
        if (!ctl->fb && !ctl->done && ctl->btype != 0u) fp_plan_lanes(ctl, ctl->n_wofs);
        ctl->ha_valid = 1;
      }
      __syncwarp();
    }
#endif
    fp_lz77_run(smem, tid, NTT, olen, wofs);
#endif
    fp_fence_async();
    FP_ARR();
    FP_ASYNC();  // (B)
    FP_TICK(10);
    FP_TICKW(4);
    for (uint32_t i = tid; i < ((olen + 31u) >> 5); i += NT) flags[i] = 0;  // (pass C of the next unit is barriers away)
    // ---------------- output: one bulk store for the 16-byte aligned body, byte stores for the ragged ends ----------------
    {
      uint8_t *g = out_base + out_off[unit];
      const uint32_t head = min((16u - wofs) & 15u, olen);
      const uint32_t body = (olen - head) & ~15u;
      if (tid < head) g[tid] = W[tid];
      const uint32_t tail0 = head + body;
      if (tail0 + tid < olen && tid < 16u) g[tail0 + tid] = W[tail0 + tid];
      if (tid == 0) {
        if (body) fp_store_bulk(g + head, W + head, body);
        out_len[unit] = olen;
        status[unit] = (int32_t)fin_status;
        in_used[unit] = fin_status == (uint32_t)B200Z_U_EOS ? u_in_len : (fin_pos - lead * 8u + 7u) >> 3;
        doneflag[(size_t)unit * flag_stride] = 1;
      }
    }
    FP_TICK(11);
  }
}

}  // namespace b200z
