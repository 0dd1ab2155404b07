// xz_kernels.cu -- XZDecoder / XZEncoder (LZMA2 in the .xz container) on the device, and CRC-64.
//
// Reference (paths relative to the reference's lib/src/):
//   codecs/xz_decoder.dart:30-458        _XZStreamDecoder: stream header, block loop, block header, LZMA2 chunk loop,
//                                        checks, index, footer
//   codecs/lzma/lzma_decoder.dart        LzmaDecoder: ONE instance for the whole stream; trimDictionary after every chunk
//   codecs/lzma/range_decoder.dart       RangeDecoder (Dart ints are 64-bit: `code` is an int64 here too)
//   codecs/xz_encoder.dart:30-283        XZEncoder: one stored chunk, 8 MiB dictionary byte, index, footer, check
//   util/_crc64_io.dart:5-11             getCrc64 (ECMA-182, reflected)
//
// Work shapes:
//   host plan     xz_plan() walks the container and every LZMA2 chunk header exactly as the reference does, without
//                 decoding: every chunk gets its input range, output offset, declared size, props in force and its
//                 dictionary position after the trims before it.  A dictionary reset (control 1, LZMA reset 3, and the
//                 end marker of every block) starts a RUN: the chunks of a run depend on each other, runs do not.
//   k_xz_copy     one CTA per stored chunk: copies its bytes into the output.  Runs first, because the LZMA chunks behind
//                 a stored chunk of the same run read those bytes as dictionary.
//   k_xz_lzma     one warp (one CTA) per run, runs taken off a counter, longest first.  Lane 0 runs the range decoder;
//                 the warp resets the probability model, which lives in shared memory when lc + lp <= 4 (and in a global
//                 slot otherwise).  The output buffer IS the dictionary: a run never reaches
//                 before its own first byte, because a reach before dictionary position 0 is an error of its own.
//                 Per chunk: XZ_OK, or XZ_OVERSHOOT / XZ_READPAST / XZ_REACH / XZ_POSSTATE, each a Dart throw (see
//                 DESIGN.md section 7 for the overshoot case).
//   k_crc64_tiles CRC-64 of 64 KiB tiles (one thread each); the host folds them with x^(8n) mod P.  CRC-32 checks go
//                 through the library's CRC-32 tile path (device_crc32_on).
//   k_xz_sha256   one thread per message (the encoder's SHA-256 check).
//
// Built by nvcc for sm_90a (product).  The CPU emulation build of the library compiles this file as part of b200z_api.cu,
// which includes it under B200Z_EMU; the launches go through XZ_LAUNCH so that both compilers take them.
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "b200z_internal.h"

#ifdef B200Z_EMU
#define XZ_LAUNCH(kern, grid, block, stream, ...) B200Z_LAUNCH(kern, grid, block, 0, stream, __VA_ARGS__)
#else
#define XZ_LAUNCH(kern, grid, block, stream, ...) kern<<<grid, block, 0, stream>>>(__VA_ARGS__)
#endif

namespace b200z {

// ---- the probability model (uint16 offsets); literal tables last: 3 x 256 x 2^(lc+lp) ----
constexpr uint32_t XP_NONLIT = 0;        // [12 states][16 posStates]: the reference's tables hold 12 (posState >= 12 throws)
constexpr uint32_t XP_REP = 192, XP_REP0 = 204, XP_REP1 = 216, XP_REP2 = 228;
constexpr uint32_t XP_LONGREP0 = 240;    // [12][16]
constexpr uint32_t XP_LEN_M = 432;       // form[2] short[32][8] medium[32][8] long[256]
constexpr uint32_t XP_LEN_R = XP_LEN_M + 770;
constexpr uint32_t XP_LEN_FORM = 0, XP_LEN_SHORT = 2, XP_LEN_MED = 258, XP_LEN_LONG = 514;
constexpr uint32_t XP_SLOT = XP_LEN_R + 770;  // [4][64]
constexpr uint32_t XP_DSHORT = XP_SLOT + 256; // [10][32] (slot 4..13: 1 << (slot / 2 - 1) entries used)
constexpr uint32_t XP_ALIGN = XP_DSHORT + 320;
constexpr uint32_t XP_LIT = (XP_ALIGN + 16 + 15) & ~15u;
constexpr uint32_t XZ_SMEM_LCLP = 4;     // models up to lc + lp = 4 stay in shared memory
constexpr uint32_t XZ_SMEM_MODEL = XP_LIT + (768u << XZ_SMEM_LCLP);
__host__ __device__ inline uint32_t xz_model_words(uint32_t lclp) { return XP_LIT + (768u << lclp); }

enum : int32_t { XZ_OK = 0, XZ_OVERSHOOT = 1, XZ_READPAST = 2, XZ_REACH = 3, XZ_POSSTATE = 4 };

struct XzChunk {
  uint64_t in_off;    // first compressed (LZMA) / stored byte in the input
  uint64_t out_off;   // where its output starts
  uint64_t dict_pos;  // the reference's dictionary write position when the chunk starts (after every trim before it)
  uint32_t in_len;    // bytes available (the declared size, clamped at the end of the input as readBytes does)
  uint32_t ulen;      // declared uncompressed size (stored: the bytes copied)
  uint32_t run;
  uint8_t lzma, reset_model, pb, lp, lc, pad_[3];
};
struct XzRun {
  uint32_t first, n;       // chunks [first, first + n)
  uint64_t bytes;          // output bytes (the ordering key)
  uint32_t global_slot;    // 0xffffffff: model in shared memory
  uint32_t lclp_max;
};

// ---- kernels ----
__global__ void __launch_bounds__(256) k_xz_copy(const uint8_t *__restrict__ in, const XzChunk *__restrict__ ch,
                                                 const uint32_t *__restrict__ list, uint8_t *__restrict__ out) {
  const XzChunk c = ch[list[blockIdx.x]];
  for (uint32_t i = threadIdx.x; i < c.in_len; i += blockDim.x) out[c.out_off + i] = in[c.in_off + i];
}

struct XzRc {
  int64_t range, code;
  const uint8_t *buf;  // the staged compressed bytes [lo, lo + XZ_STAGE) of the chunk
  uint32_t n, pos, lo;
  bool past;
};
__device__ __forceinline__ void xz_norm(XzRc &r) {
  if (r.range < 0x1000000) {
    r.range <<= 8;
    uint32_t b = 0;
    if (r.pos < r.n) b = r.buf[r.pos - r.lo];
    else r.past = true;
    r.pos++;
    r.code = (int64_t)((uint64_t)r.code << 8) | b;
  }
}
__device__ __forceinline__ uint32_t xz_bit(XzRc &r, uint16_t *p) {
  xz_norm(r);
  const int64_t pr = *p;
  const int64_t bound = (r.range >> 11) * pr;
  if (r.code < bound) {
    r.range = bound;
    *p = (uint16_t)(pr + ((2048 - pr) >> 5));
    return 0;
  }
  r.range -= bound;
  r.code -= bound;
  *p = (uint16_t)(pr - (pr >> 5));
  return 1;
}
__device__ __forceinline__ uint32_t xz_tree(XzRc &r, uint16_t *t, int count) {
  uint32_t v = 0, prefix = 1;
  for (int i = 0; i < count; ++i) {
    v = (v << 1) | xz_bit(r, t + (prefix | v));
    prefix <<= 1;
  }
  return v;
}
__device__ __forceinline__ uint32_t xz_tree_rev(XzRc &r, uint16_t *t, int count) {
  uint32_t v = 0, prefix = 1;
  for (int i = 0; i < count; ++i) {
    v |= xz_bit(r, t + (prefix | v)) << i;
    prefix <<= 1;
  }
  return v;
}
__device__ __forceinline__ uint32_t xz_len(XzRc &r, uint16_t *L, uint32_t ps) {
  if (xz_bit(r, L + XP_LEN_FORM) == 0) return 2 + xz_tree(r, L + XP_LEN_SHORT + ps * 8, 3);
  if (xz_bit(r, L + XP_LEN_FORM + 1) == 0) return 10 + xz_tree(r, L + XP_LEN_MED + ps * 8, 3);
  return 18 + xz_tree(r, L + XP_LEN_LONG, 8);
}
__device__ __forceinline__ uint32_t xz_dist(XzRc &r, uint16_t *P, uint32_t len) {
  const uint32_t ds = len - 2 < 3 ? len - 2 : 3;
  const uint32_t slot = xz_tree(r, P + XP_SLOT + ds * 64, 6);
  if (slot < 4) return slot;
  const uint32_t prefix = 2 | (slot & 1);
  const int bits = (int)(slot / 2) - 1;
  if (slot < 14) return (prefix << bits) | xz_tree_rev(r, P + XP_DSHORT + (slot - 4) * 32, bits);
  uint32_t direct = 0;
  for (int i = 0; i < bits - 4; ++i) {  // readDirect (range_decoder.dart:173-190)
    xz_norm(r);
    r.range >>= 1;
    r.code -= r.range;
    direct <<= 1;
    if (r.code & 0x80000000ll) r.code += r.range;
    else direct++;
  }
  return (prefix << bits) | (direct << 4) | xz_tree_rev(r, P + XP_ALIGN, 4);
}

struct XzState {  // what carries from chunk to chunk inside a run
  uint32_t state, d0, d1, d2, d3;
};

// k_xz_lzma's shared buffers besides the model: the chunk's compressed bytes, staged by the whole warp ahead of lane 0, and
// a ring of the most recent output, which lane 0 reads (matched literals, matches) and the warp flushes to global memory.
constexpr uint32_t XZ_STAGE = 2048;  // compressed bytes per refill
constexpr uint32_t XZ_WIN = 4096;    // output ring (a power of two)
constexpr uint32_t XZ_FLUSH = 2048;  // lane 0 hands back to the warp once this much output is unflushed
constexpr uint32_t XZ_SYM_MAX_IN = 64;  // compressed bytes one symbol can take (at most one per decoded bit, < 50)
constexpr uint32_t XZ_MATCH_MAX = 273;
static_assert(XZ_WIN >= XZ_FLUSH + 2 * XZ_MATCH_MAX, "bytes reached through the ring must not have left it unflushed");
constexpr int32_t XZ_MORE = -1;  // lane 0 needs the next stage / a flush

struct XzLane0 {  // lane 0's decoder between two hand-backs to the warp
  XzRc r;
  uint32_t pos, prev;
  XzState s;
};

// lane 0: decode chunk c from lz.pos on until it ends (XZ_OK), fails (XZ_*), or needs the warp (XZ_MORE).  `ring` holds
// output positions [g - XZ_WIN, g) (g = c.out_off + pos); older bytes are in `out`, flushed up to `flushed`.
__device__ int32_t xz_decode_step(const XzChunk &c, uint8_t *__restrict__ out, uint8_t *__restrict__ ring, uint64_t flushed,
                                  uint16_t *P, XzLane0 &lz) {
  XzRc &r = lz.r;
  XzState &s = lz.s;
  const uint64_t base = c.dict_pos;
  const uint32_t pmask = (1u << c.pb) - 1, lpmask = (1u << c.lp) - 1, lc = c.lc;
  const uint32_t end = c.ulen;
  const uint32_t hi = r.lo + min(XZ_STAGE, r.n - min(r.n, r.lo));
  uint32_t pos = lz.pos, prev = lz.prev;
  int32_t ret = XZ_OK;
  while (pos < end) {
    if ((hi < r.n && r.pos + XZ_SYM_MAX_IN > hi) || c.out_off + pos - flushed >= XZ_FLUSH) {
      ret = XZ_MORE;
      break;
    }
    const uint64_t wp = base + pos;
    const uint64_t g = c.out_off + pos;
    const uint32_t ps = (uint32_t)wp & pmask;
    if (ps >= 12) {  // _nonLiteralTables[state] holds 12 entries (lzma_decoder.dart:68-70): RangeError
      xz_norm(r);
      ret = r.past ? XZ_READPAST : XZ_POSSTATE;
      break;
    }
    const uint32_t st = s.state;
    const bool lit_prev = st < 7;
    if (xz_bit(r, P + XP_NONLIT + st * 16 + ps) == 0) {
      uint16_t *lt = P + XP_LIT + 768u * (((uint32_t)wp & lpmask) << lc | (prev >> (8 - lc)));
      uint32_t sym = 1;
      if (lit_prev) {
        for (int i = 0; i < 8; ++i) sym = (sym << 1) | xz_bit(r, lt + sym);
      } else {
        if ((uint64_t)s.d0 + 1 > wp) {
          ret = XZ_REACH;
          break;
        }
        const uint64_t q = g - s.d0 - 1;
        const uint32_t mb = s.d0 < XZ_WIN ? ring[q & (XZ_WIN - 1)] : out[q];
        bool matched = true;
        for (int i = 7; i >= 0; --i) {
          if (matched) {
            const uint32_t bit = (mb >> i) & 1;
            const uint32_t b = xz_bit(r, lt + 256 + 256 * bit + sym);
            sym = (sym << 1) | b;
            matched = b == bit;
          } else {
            sym = (sym << 1) | xz_bit(r, lt + sym);
          }
        }
      }
      if (r.past) {
        ret = XZ_READPAST;
        break;
      }
      prev = sym & 0xff;
      ring[g & (XZ_WIN - 1)] = (uint8_t)prev;
      pos++;
      s.state = st < 4 ? 0 : st < 10 ? st - 3 : st - 6;
      continue;
    }
    uint32_t dist, len;
    if (xz_bit(r, P + XP_REP + st) == 0) {
      len = xz_len(r, P + XP_LEN_M, ps);
      dist = xz_dist(r, P, len);
      s.d3 = s.d2;
      s.d2 = s.d1;
      s.d1 = s.d0;
      s.d0 = dist;
      s.state = lit_prev ? 7 : 10;
    } else {
      if (xz_bit(r, P + XP_REP0 + st) == 0) {
        if (xz_bit(r, P + XP_LONGREP0 + st * 16 + ps) == 0) {
          dist = s.d0;
          len = 1;
          s.state = lit_prev ? 9 : 11;
        } else {
          dist = s.d0;
          len = xz_len(r, P + XP_LEN_R, ps);
          s.state = lit_prev ? 8 : 11;
        }
      } else {
        if (xz_bit(r, P + XP_REP1 + st) == 0) {
          dist = s.d1;
        } else if (xz_bit(r, P + XP_REP2 + st) == 0) {
          dist = s.d2;
          s.d2 = s.d1;
        } else {
          dist = s.d3;
          s.d3 = s.d2;
          s.d2 = s.d1;
        }
        s.d1 = s.d0;
        s.d0 = dist;
        len = xz_len(r, P + XP_LEN_R, ps);
        s.state = lit_prev ? 8 : 11;
      }
    }
    if (r.past) {
      ret = XZ_READPAST;
      break;
    }
    if ((uint64_t)dist + 1 > wp) {
      ret = XZ_REACH;
      break;
    }
    if (pos + len > end) {
      ret = XZ_OVERSHOOT;
      break;
    }
    uint64_t q = g - dist - 1, d = g;
    if (dist < XZ_WIN) {  // the source is still in the ring (it may overlap what this match writes)
      for (uint32_t i = 0; i < len; ++i, ++q, ++d) ring[d & (XZ_WIN - 1)] = ring[q & (XZ_WIN - 1)];
    } else {  // flushed long ago: dist + 1 > XZ_WIN >= g - flushed + len
      for (uint32_t i = 0; i < len; ++i, ++q, ++d) ring[d & (XZ_WIN - 1)] = out[q];
    }
    prev = ring[(d - 1) & (XZ_WIN - 1)];
    pos += len;
  }
  lz.pos = pos;
  lz.prev = prev;
  return ret;
}

__global__ void __launch_bounds__(32) k_xz_lzma(const uint8_t *__restrict__ in, const XzChunk *__restrict__ ch,
                                                const XzRun *__restrict__ runs, uint32_t n_runs, uint32_t *__restrict__ next_run,
                                                uint16_t *__restrict__ global_models, uint8_t *out, int32_t *__restrict__ status) {
  __shared__ uint16_t sm_model[XZ_SMEM_MODEL];
  __shared__ uint8_t sm_stage[XZ_STAGE];
  __shared__ uint8_t sm_ring[XZ_WIN];
  const uint32_t lane = threadIdx.x;
  for (;;) {
    uint32_t ri = 0;
    if (lane == 0) ri = atomicAdd(next_run, 1u);
    ri = __shfl_sync(0xffffffffu, ri, 0);
    if (ri >= n_runs) return;
    const XzRun run = runs[ri];
    uint16_t *P = run.global_slot == 0xffffffffu ? sm_model
                                                 : global_models + (size_t)run.global_slot * xz_model_words(run.lclp_max);
    XzLane0 lz;
    lz.s = XzState{0, 0, 0, 0, 0};
    for (uint32_t k = 0; k < run.n; ++k) {
      const uint32_t ci = run.first + k;
      const XzChunk c = ch[ci];
      if (c.reset_model) {  // LzmaDecoder.reset (lzma_decoder.dart:104-160): every probability back to one half
        const uint32_t words = xz_model_words((uint32_t)c.lc + c.lp);
        for (uint32_t i = lane; i < words; i += 32) P[i] = 1024;
        lz.s = XzState{0, 0, 0, 0, 0};
      }
      if (!c.lzma) continue;  // stored: k_xz_copy has written it
      // the ring starts as the output in front of the chunk (earlier chunks of the run, stored ones included)
      const uint64_t pre = min((uint64_t)XZ_WIN, c.out_off);
      for (uint32_t i = lane; i < pre; i += 32) {
        const uint64_t q = c.out_off - pre + i;
        sm_ring[q & (XZ_WIN - 1)] = out[q];
      }
      lz.r.buf = sm_stage;
      lz.r.n = c.in_len;
      lz.r.lo = 0;
      uint64_t flushed = c.out_off;
      int32_t st = XZ_MORE;
      bool first = true;
      while (st == XZ_MORE) {
        const uint32_t lo = __shfl_sync(0xffffffffu, lz.r.pos, 0);
        const uint32_t from = first ? 0 : lo;
        const uint32_t cnt = from < c.in_len ? min(XZ_STAGE, c.in_len - from) : 0;
        for (uint32_t i = lane; i < cnt; i += 32) sm_stage[i] = in[c.in_off + from + i];
        __syncwarp();
        if (lane == 0) {
          lz.r.lo = from;
          if (first) {  // initialize() (range_decoder.dart:51-58): the first byte is skipped unchecked
            lz.r.pos = 1;
            lz.r.past = false;
            lz.r.range = 0xffffffffll;
            lz.r.code = 0;
            for (int i = 0; i < 4; ++i) {
              uint32_t b = 0;
              if (lz.r.pos < lz.r.n) b = sm_stage[lz.r.pos];
              else lz.r.past = true;
              lz.r.pos++;
              lz.r.code = (lz.r.code << 8) | b;
            }
            lz.pos = 0;
            lz.prev = c.dict_pos > 0 ? sm_ring[(c.out_off - 1) & (XZ_WIN - 1)] : 0;
          }
          st = lz.r.past ? XZ_READPAST : xz_decode_step(c, out, sm_ring, flushed, P, lz);
        }
        first = false;
        st = __shfl_sync(0xffffffffu, st, 0);
        const uint64_t upto = c.out_off + __shfl_sync(0xffffffffu, lz.pos, 0);
        __syncwarp();
        for (uint64_t q = flushed + lane; q < upto; q += 32) out[q] = sm_ring[q & (XZ_WIN - 1)];
        flushed = upto;
        __syncwarp();
      }
      if (lane == 0) status[ci] = st;
      if (st != XZ_OK) break;
    }
  }
}

__global__ void __launch_bounds__(256) k_crc64_tiles(const uint8_t *__restrict__ d, const uint64_t *__restrict__ tile_off,
                                                     const uint32_t *__restrict__ tile_len, uint32_t n_tiles,
                                                     uint64_t *__restrict__ part) {
  __shared__ uint64_t tab[256];
  {
    uint64_t c = threadIdx.x;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? 0xC96C5795D7870F42ull ^ (c >> 1) : c >> 1;
    tab[threadIdx.x] = c;
  }
  __syncthreads();
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_tiles) return;
  const uint8_t *p = d + tile_off[t];
  const uint32_t n = tile_len[t];
  uint64_t c = ~0ull;
  for (uint32_t i = 0; i < n; ++i) c = tab[(c ^ p[i]) & 0xff] ^ (c >> 8);
  part[t] = ~c;
}

__device__ __forceinline__ uint32_t xz_ror(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }
__constant__ uint32_t c_k256[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01,
    0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc,
    0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147,
    0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08,
    0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208,
    0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
__device__ void xz_sha256_block(uint32_t h[8], const uint8_t *p) {
  uint32_t w[16];
  for (int i = 0; i < 16; ++i) w[i] = (uint32_t)p[4 * i] << 24 | (uint32_t)p[4 * i + 1] << 16 | (uint32_t)p[4 * i + 2] << 8 | p[4 * i + 3];
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
  for (int i = 0; i < 64; ++i) {
    uint32_t wi;
    if (i < 16) {
      wi = w[i];
    } else {
      const uint32_t x = w[(i + 1) & 15], y = w[(i + 14) & 15];
      wi = w[i & 15] + (xz_ror(x, 7) ^ xz_ror(x, 18) ^ (x >> 3)) + w[(i + 9) & 15] + (xz_ror(y, 17) ^ xz_ror(y, 19) ^ (y >> 10));
      w[i & 15] = wi;
    }
    const uint32_t t1 = hh + (xz_ror(e, 6) ^ xz_ror(e, 11) ^ xz_ror(e, 25)) + ((e & f) ^ (~e & g)) + c_k256[i] + wi;
    const uint32_t t2 = (xz_ror(a, 2) ^ xz_ror(a, 13) ^ xz_ror(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
    hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}
__global__ void __launch_bounds__(32) k_xz_sha256(const uint8_t *__restrict__ d, uint64_t n, uint8_t *__restrict__ digest) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
  uint64_t i = 0;
  for (; i + 64 <= n; i += 64) xz_sha256_block(h, d + i);
  uint8_t last[128];
  for (int k = 0; k < 128; ++k) last[k] = 0;
  const uint32_t r = (uint32_t)(n - i);
  for (uint32_t k = 0; k < r; ++k) last[k] = d[i + k];
  last[r] = 0x80;
  const uint32_t tot = r + 9 <= 64 ? 64 : 128;
  for (int k = 0; k < 8; ++k) last[tot - 1 - k] = (uint8_t)((n * 8) >> (8 * k));
  xz_sha256_block(h, last);
  if (tot == 128) xz_sha256_block(h, last + 64);
  for (int k = 0; k < 32; ++k) digest[k] = (uint8_t)(h[k / 4] >> (24 - 8 * (k % 4)));
}

// ---- host: CRC folding (x^(8n) mod P, as zlib's crc32_combine) ----
static uint64_t crc64_mulmod(uint64_t a, uint64_t b) {
  uint64_t m = 1ull << 63, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = (b & 1) ? (b >> 1) ^ 0xC96C5795D7870F42ull : b >> 1;
  }
  return p;
}
// CRC-64 of A || B from crc(A), crc(B) and |B| (crc(A) * x^(8|B|) + crc(B), as zlib's crc32_combine does for CRC-32)
static uint64_t crc64_combine(uint64_t ca, uint64_t cb, uint64_t len_b) {
  uint64_t x = 1ull << 55;  // x^8 (bit 63 = x^0)
  uint64_t p = 1ull << 63;
  while (len_b) {
    if (len_b & 1) p = crc64_mulmod(x, p);
    len_b >>= 1;
    if (len_b) x = crc64_mulmod(x, x);
  }
  return crc64_mulmod(p, ca) ^ cb;
}

// ---- host: the container walk (xz_decoder.dart:46-458 without the LZMA decode) ----
namespace {
struct XzThrow {};
struct View {
  const uint8_t *b;
  int64_t len, pos;
  bool eos() const { return pos >= len; }
  int rb() {
    if (pos < 0 || pos >= len) throw XzThrow{};
    return b[pos++];
  }
  View read_bytes(int64_t count) {
    if (count < 0) throw XzThrow{};
    const int64_t avail = len - pos;
    View v{b + pos, count < avail ? count : avail, 0};
    pos += v.len;
    return v;
  }
  void skip(int64_t n) { pos = std::min(std::max(pos + n, (int64_t)0), len); }
  uint32_t u32() {
    uint32_t v = 0;
    for (int i = 0; i < 4; ++i) v |= (uint32_t)rb() << (8 * i);
    return v;
  }
  uint64_t u64() {
    uint64_t v = 0;
    for (int i = 0; i < 8; ++i) v |= (uint64_t)rb() << (8 * i);
    return v;
  }
  int64_t mbi() {
    uint64_t v = 0;
    int64_t shift = 0;
    for (;;) {
      const int d = rb();
      if (shift < 64) v |= (uint64_t)(d & 0x7f) << shift;
      if (!(d & 0x80)) return (int64_t)v;
      shift += 7;
    }
  }
  int64_t padding() {
    int64_t n = 0;
    while (pos % 4 != 0) {
      if (rb() != 0) return -1;
      n++;
    }
    return n;
  }
};
uint32_t host_crc32(const uint8_t *p, size_t n) {
  uint32_t c = 0xffffffffu;
  for (size_t i = 0; i < n; ++i) {
    c ^= p[i];
    for (int k = 0; k < 8; ++k) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
  }
  return ~c;
}
}  // namespace

struct XzCheck {
  uint64_t lo, hi;  // output range of the block
  uint64_t want;
  bool c64;
};
struct XzEvent {
  uint32_t check;  // 0: chunk `idx`, 1: check `idx`
  uint32_t idx;
};
struct XzPlan {
  std::vector<XzChunk> chunks;
  std::vector<XzRun> runs;
  std::vector<XzCheck> checks;
  std::vector<XzEvent> events;
  int status = B200Z_E_DATA;  // where the walk ends: B200Z_OK / B200Z_E_DATA / B200Z_E_THROW
  uint64_t out_bytes = 0;     // output at that point, if every chunk yields its declared size
};

namespace {
struct Walker {
  XzPlan &p;
  int verify;
  int flags = 0;
  // LzmaDecoder state the plan needs: props, the dictionary write position
  uint8_t pb = 2, lp = 0, lc = 3;
  uint64_t wp = 0;
  bool run_open = false, model_reset_pending = true;
  std::vector<std::pair<int64_t, int64_t>> sizes;

  void dict_reset() {
    wp = 0;
    run_open = false;
    model_reset_pending = true;
  }
  void trim(int64_t max_size) {  // trimDictionary (lzma_decoder.dart:87-101)
    const int64_t threshold = max_size + (max_size >> 2);
    if ((int64_t)wp <= threshold) return;
    const int ab = pb > lp ? pb : lp;
    wp = (uint64_t)(max_size + (int64_t)(wp & ((1ull << ab) - 1)));
  }
  void add_chunk(const View &data, uint32_t ulen, bool lzma, uint64_t out_len) {
    XzChunk c;
    memset(&c, 0, sizeof c);
    c.in_off = (uint64_t)(data.b - base);
    c.in_len = (uint32_t)data.len;
    c.out_off = p.out_bytes;
    c.dict_pos = wp;
    c.ulen = ulen;
    c.lzma = lzma;
    c.pb = pb;
    c.lp = lp;
    c.lc = lc;
    c.reset_model = model_reset_pending;
    model_reset_pending = false;
    if (!run_open) {
      XzRun r;
      memset(&r, 0, sizeof r);
      r.first = (uint32_t)p.chunks.size();
      p.runs.push_back(r);
      run_open = true;
    }
    XzRun &r = p.runs.back();
    c.run = (uint32_t)(p.runs.size() - 1);
    r.n++;
    r.bytes += out_len;
    r.lclp_max = std::max(r.lclp_max, (uint32_t)lc + lp);
    p.events.push_back({0, (uint32_t)p.chunks.size()});
    p.chunks.push_back(c);
    p.out_bytes += out_len;
    wp += ulen;
  }
  const uint8_t *base;

  bool lzma2(View &in, int64_t dict_size) {  // _readLZMA2 (xz_decoder.dart:284-351)
    while (!in.eos()) {
      const int control = in.rb();
      if (!(control & 0x80)) {
        if (control == 0) {
          dict_reset();
          return true;
        }
        if (control != 1 && control != 2) return false;
        if (control == 1) dict_reset();
        const int hi = in.rb(), lo = in.rb();
        const int64_t length = (hi << 8 | lo) + 1;
        View d = in.read_bytes(length);
        add_chunk(d, (uint32_t)length, false, (uint64_t)d.len);  // clamped bytes reach the output, wp moves by length
        trim(dict_size);
      } else {
        const int reset = (control >> 5) & 3;
        const int b1 = in.rb(), b2 = in.rb();
        const int64_t ulen = ((control & 0x1f) << 16 | b1 << 8 | b2) + 1;
        const int c1 = in.rb(), c2 = in.rb();
        const int64_t clen = (c1 << 8 | c2) + 1;
        if (reset >= 2) {
          int props = in.rb();
          pb = (uint8_t)(props / 45);
          props -= pb * 45;
          lp = (uint8_t)(props / 9);
          lc = (uint8_t)(props - lp * 9);
        }
        if (reset == 3) dict_reset();
        if (reset > 0) model_reset_pending = true;
        View d = in.read_bytes(clen);
        add_chunk(d, (uint32_t)ulen, true, (uint64_t)ulen);
        trim(dict_size);
      }
    }
    return false;
  }

  bool block(View &in, int64_t header_len) {  // _readBlock (:104-281)
    const int64_t block_start = in.pos;
    View h = in.read_bytes(header_len - 4);
    h.skip(1);
    const int bflags = h.rb();
    const int nfilters = (bflags & 3) + 1;
    const bool has_comp = bflags & 0x40, has_uncomp = bflags & 0x80;
    int64_t comp_len = 0, uncomp_len = 0;
    if (has_comp) comp_len = h.mbi();
    if (has_uncomp) uncomp_len = h.mbi();
    int64_t first_id = -1, dict_size = 0;
    for (int i = 0; i < nfilters; ++i) {
      const int64_t id = h.mbi();
      const int64_t plen = h.mbi();
      View props = h.read_bytes(plen);
      if (id == 0x03 || id == 0x21) {
        if (props.len < 1) throw XzThrow{};
        if (id == 0x21) {
          const int v = props.b[0];
          if (v > 40) return false;
          dict_size = v == 40 ? 0xffffffffll : (int64_t)(2 | (v & 1)) << ((v >> 1) + 11);
        }
      }
      if (i == 0) first_id = id;
    }
    if (h.padding() < 0) return false;
    const uint32_t crc = in.u32();
    if (host_crc32(h.b, (size_t)h.len) != crc) return false;
    if (nfilters != 1 || first_id != 0x21) return false;
    const int64_t start_pos = in.pos;
    const uint64_t start_out = p.out_bytes;
    if (!lzma2(in, dict_size)) return false;
    const int64_t actual_comp = in.pos - start_pos, actual_uncomp = (int64_t)(p.out_bytes - start_out);
    if (has_comp && comp_len != actual_comp) return false;
    if (!has_uncomp) uncomp_len = actual_uncomp;
    if (uncomp_len != actual_uncomp) return false;
    const int64_t pad = in.padding();
    if (pad < 0) return false;
    switch (flags & 0xf) {
      case 0: break;
      case 1: {
        const uint32_t want = in.u32();
        if (verify) {
          p.events.push_back({1, (uint32_t)p.checks.size()});
          p.checks.push_back({start_out, p.out_bytes, want, false});
        }
        break;
      }
      case 2: case 3: in.skip(4); break;
      case 4: {
        const uint64_t want = in.u64();
        if (verify) {
          p.events.push_back({1, (uint32_t)p.checks.size()});
          p.checks.push_back({start_out, p.out_bytes, want, true});
        }
        break;
      }
      case 5: case 6: in.skip(8); break;
      case 7: case 8: case 9: in.skip(16); break;
      case 0xa: in.read_bytes(32); break;
      case 0xb: case 0xc: in.skip(32); break;
      default: in.skip(64); break;
    }
    sizes.push_back({in.pos - block_start - pad, uncomp_len});
    return true;
  }

  int64_t index(View &in) {  // _readStreamIndex (:355-392)
    const int64_t start = in.pos;
    in.skip(1);
    const int64_t n = in.mbi();
    if (n != (int64_t)sizes.size()) return -1;
    for (int64_t i = 0; i < n; ++i) {
      const int64_t unpadded = in.mbi(), uncomp = in.mbi();
      if (sizes[i].first != unpadded || sizes[i].second != uncomp) return -1;
    }
    if (in.padding() < 0) return -1;
    const int64_t ilen = in.pos - start;
    in.skip(-ilen);
    View idx = in.read_bytes(ilen);
    const uint32_t crc = in.u32();
    if (host_crc32(idx.b, (size_t)idx.len) != crc) return -1;
    return ilen + 4;
  }

  bool footer(View &in, int64_t index_size) {  // _readStreamFooter (:396-428)
    const uint32_t crc = in.u32();
    View f = in.read_bytes(6);
    const int64_t backward = ((int64_t)f.u32() + 1) * 4;
    if (backward != index_size) return false;
    if (f.rb() != 0) return false;
    if (f.rb() != flags) return false;
    if (host_crc32(f.b, (size_t)f.len) != crc) return false;
    View m = in.read_bytes(2);
    if (m.len < 1) throw XzThrow{};
    if (m.b[0] != 89) return false;
    if (m.len < 2) throw XzThrow{};
    return m.b[1] == 90;
  }

  bool stream(View &in) {  // decode (:46-101)
    View magic = in.read_bytes(6);
    static const uint8_t mg[6] = {253, 55, 122, 88, 90, 0};
    for (int i = 0; i < 6; ++i) {
      if (i >= magic.len) throw XzThrow{};
      if (magic.b[i] != mg[i]) return false;
    }
    View h = in.read_bytes(2);
    if (h.rb() != 0) return false;
    flags = h.rb();
    const uint32_t crc = in.u32();
    if (host_crc32(h.b, (size_t)h.len) != crc) return false;
    while (!in.eos()) {
      const int bh = in.b[in.pos];
      if (bh == 0) {
        const int64_t isz = index(in);
        if (isz < 0) return false;
        return footer(in, isz);
      }
      if (!block(in, ((int64_t)bh + 1) * 4)) return false;
    }
    return false;
  }
};
}  // namespace

void xz_plan(const uint8_t *in, size_t n, int verify, XzPlan *p) {
  Walker w{*p, verify};
  w.base = in;
  View v{in, (int64_t)n, 0};
  try {
    p->status = w.stream(v) ? B200Z_OK : B200Z_E_DATA;
  } catch (const XzThrow &) {
    p->status = B200Z_E_THROW;
  }
}

// ---- host: device buffers of this file (grown, never shrunk) ----
namespace {
struct XzBuf {
  void *p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    const size_t want = n + (n >> 3) + 4096;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    else p = nullptr;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};
XzBuf x_in, x_out, x_meta, x_models;
cudaEvent_t x_ev[2] = {nullptr, nullptr};
double g_xz_lzma_ms = 0;
uint32_t g_xz_runs = 0;
}  // namespace

#define XZ_CU(x)                                                                               \
  do {                                                                                         \
    cudaError_t e__ = (x);                                                                     \
    if (e__ != cudaSuccess) {                                                                  \
      char m__[256];                                                                           \
      snprintf(m__, sizeof m__, "xz: %s failed: %s", #x, cudaGetErrorString(e__));             \
      set_error_text(m__);                                                                     \
      return B200Z_E_NODEVICE;                                                                 \
    }                                                                                          \
  } while (0)

static inline size_t xz_align(size_t v) { return (v + 255) & ~(size_t)255; }

// CRC-64 (c64) or CRC-32 of each [lo, hi) range of device bytes d.  CRC-32 is the library's tile path (device_crc32_on,
// b200z_api.cu); CRC-64 is k_crc64_tiles over 64 KiB tiles of all ranges in one launch, folded here.
static int xz_device_crcs(const uint8_t *d, const std::vector<std::pair<uint64_t, uint64_t>> &ranges, bool c64,
                          std::vector<uint64_t> *crcs, cudaStream_t s) {
  crcs->clear();
  if (!c64) {
    for (auto &r : ranges) {
      XZ_CU(x_meta.reserve(((r.second - r.first) / 8192 + 1) * 4 + 256));
      uint32_t c = 0;
      const int rc = device_crc32_on(d + r.first, (size_t)(r.second - r.first), (uint32_t *)x_meta.p, s, &c);
      if (rc) return rc;
      crcs->push_back(c);
    }
    return B200Z_OK;
  }
  const uint64_t TILE = 1u << 16;
  std::vector<uint64_t> toff;
  std::vector<uint32_t> tlen;
  for (auto &r : ranges)
    for (uint64_t o = r.first; o < r.second; o += TILE) {
      toff.push_back(o);
      tlen.push_back((uint32_t)std::min(TILE, r.second - o));
    }
  const size_t nt = toff.size();
  std::vector<uint64_t> part(nt);
  if (nt) {
    const size_t b_off = 0, b_len = xz_align(8 * nt), b_part = b_len + xz_align(4 * nt);
    XZ_CU(x_meta.reserve(b_part + 8 * nt));
    uint8_t *m = (uint8_t *)x_meta.p;
    XZ_CU(cudaMemcpyAsync(m + b_off, toff.data(), 8 * nt, cudaMemcpyHostToDevice, s));
    XZ_CU(cudaMemcpyAsync(m + b_len, tlen.data(), 4 * nt, cudaMemcpyHostToDevice, s));
    XZ_LAUNCH(k_crc64_tiles, (unsigned)((nt + 255) / 256), 256, s, d, (const uint64_t *)(m + b_off),
              (const uint32_t *)(m + b_len), (uint32_t)nt, (uint64_t *)(m + b_part));
    count_launch();
    XZ_CU(cudaGetLastError());
    XZ_CU(cudaMemcpyAsync(part.data(), m + b_part, 8 * nt, cudaMemcpyDeviceToHost, s));
    XZ_CU(cudaStreamSynchronize(s));
  }
  size_t t = 0;
  for (auto &r : ranges) {
    uint64_t c = 0;  // the CRC of nothing
    for (uint64_t o = r.first; o < r.second; o += TILE, ++t) c = crc64_combine(c, part[t], tlen[t]);
    crcs->push_back(c);
  }
  return B200Z_OK;
}

size_t xz_bound(const uint8_t *in, size_t n) {
  XzPlan p;
  xz_plan(in, n, 0, &p);
  return (size_t)p.out_bytes;
}

int xz_decode_impl(const uint8_t *in, size_t n, int verify, uint8_t *out, size_t out_cap, size_t *out_len, cudaStream_t s) {
  XzPlan p;
  xz_plan(in, n, verify, &p);
  if (p.out_bytes > out_cap) {
    *out_len = (size_t)p.out_bytes;
    set_error_text("xz_decode: out_cap is smaller than the output the stream declares (b200z_xz_bound)");
    return B200Z_E_NOSPC;
  }
  const size_t nc = p.chunks.size(), nr = p.runs.size();
  std::vector<int32_t> status(nc, XZ_OK);
  XZ_CU(x_out.reserve(p.out_bytes + 16));
  if (nc) {
    XZ_CU(x_in.reserve(n + 16));
    XZ_CU(cudaMemcpyAsync(x_in.p, in, n, cudaMemcpyHostToDevice, s));
    // runs longest first; models that do not fit shared memory get a global slot
    std::vector<uint32_t> order(nr);
    for (size_t i = 0; i < nr; ++i) order[i] = (uint32_t)i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return p.runs[a].bytes > p.runs[b].bytes; });
    std::vector<XzRun> runs(nr);
    uint32_t n_global = 0, big_lclp = 0;
    for (size_t i = 0; i < nr; ++i) {
      runs[i] = p.runs[order[i]];
      runs[i].global_slot = 0xffffffffu;
      if (runs[i].lclp_max > XZ_SMEM_LCLP) {
        big_lclp = std::max(big_lclp, runs[i].lclp_max);
        runs[i].global_slot = n_global++;
      }
    }
    for (auto &r : runs)
      if (r.global_slot != 0xffffffffu) r.lclp_max = big_lclp;  // one slot size for all of them
    std::vector<uint32_t> stored;
    for (size_t i = 0; i < nc; ++i)
      if (!p.chunks[i].lzma && p.chunks[i].in_len) stored.push_back((uint32_t)i);
    const size_t o_ch = 0, o_runs = xz_align(nc * sizeof(XzChunk)), o_st = o_runs + xz_align(nr * sizeof(XzRun)),
                 o_list = o_st + xz_align(4 * nc), o_ctr = o_list + xz_align(4 * stored.size() + 4), total = o_ctr + 256;
    XZ_CU(x_meta.reserve(total));
    uint8_t *m = (uint8_t *)x_meta.p;
    XZ_CU(cudaMemcpyAsync(m + o_ch, p.chunks.data(), nc * sizeof(XzChunk), cudaMemcpyHostToDevice, s));
    XZ_CU(cudaMemcpyAsync(m + o_runs, runs.data(), nr * sizeof(XzRun), cudaMemcpyHostToDevice, s));
    if (!stored.empty()) XZ_CU(cudaMemcpyAsync(m + o_list, stored.data(), 4 * stored.size(), cudaMemcpyHostToDevice, s));
    XZ_CU(cudaMemsetAsync(m + o_st, 0, 4 * nc, s));
    XZ_CU(cudaMemsetAsync(m + o_ctr, 0, 4, s));
    if (n_global) XZ_CU(x_models.reserve((size_t)n_global * xz_model_words(big_lclp) * 2));
    const uint8_t *d_in = (const uint8_t *)x_in.p;
    const XzChunk *d_ch = (const XzChunk *)(m + o_ch);
    if (!stored.empty()) {
      XZ_LAUNCH(k_xz_copy, (unsigned)stored.size(), 256, s, d_in, d_ch, (const uint32_t *)(m + o_list), (uint8_t *)x_out.p);
      count_launch();
    }
    if (!x_ev[0]) {  // created once, kept for the life of the library
      XZ_CU(cudaEventCreate(&x_ev[0]));
      XZ_CU(cudaEventCreate(&x_ev[1]));
    }
    cudaEvent_t e0 = x_ev[0], e1 = x_ev[1];
    XZ_CU(cudaEventRecord(e0, s));
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const unsigned grid = (unsigned)std::min<size_t>(nr, (size_t)sms * 6);  // 6 resident one-warp CTAs per SM (35 KB smem)
    XZ_LAUNCH(k_xz_lzma, grid, 32, s, d_in, d_ch, (const XzRun *)(m + o_runs), (uint32_t)nr, (uint32_t *)(m + o_ctr),
              (uint16_t *)x_models.p, (uint8_t *)x_out.p, (int32_t *)(m + o_st));
    count_launch();
    XZ_CU(cudaGetLastError());
    XZ_CU(cudaEventRecord(e1, s));
    XZ_CU(cudaMemcpyAsync(status.data(), m + o_st, 4 * nc, cudaMemcpyDeviceToHost, s));
    XZ_CU(cudaStreamSynchronize(s));
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    g_xz_lzma_ms = ms;
    g_xz_runs = (uint32_t)nr;
  }
  // the checks: one CRC pass over every verified block
  std::vector<uint64_t> crc32s, crc64s;
  {
    std::vector<std::pair<uint64_t, uint64_t>> r32, r64;
    for (auto &c : p.checks) (c.c64 ? r64 : r32).push_back({c.lo, c.hi});
    int rc = xz_device_crcs((const uint8_t *)x_out.p, r32, false, &crc32s, s);
    if (rc) return rc;
    rc = xz_device_crcs((const uint8_t *)x_out.p, r64, true, &crc64s, s);
    if (rc) return rc;
  }
  // replay the reference's order: the first chunk that throws, or the first failed check, ends the stream
  int rc = p.status;
  uint64_t got = p.out_bytes;
  size_t i32 = 0, i64 = 0;
  for (const XzEvent &e : p.events) {
    if (!e.check) {
      if (status[e.idx] != XZ_OK) {
        static const char *why[] = {"", "a match runs past the chunk's declared size", "a read past the chunk's compressed bytes",
                                    "a reach before dictionary position 0", "posState >= 12 (pb = 4 or 5)"};
        char msg[160];
        snprintf(msg, sizeof msg, "xz_decode: chunk %u: %s (Dart: RangeError)", e.idx, why[status[e.idx] & 7]);
        set_error_text(msg);
        rc = B200Z_E_THROW;
        got = p.chunks[e.idx].out_off;
        break;
      }
    } else {
      const XzCheck &c = p.checks[e.idx];
      const uint64_t have = c.c64 ? crc64s[i64++] : crc32s[i32++];
      if (have != (c.c64 ? c.want : (c.want & 0xffffffffu))) {
        set_error_text("xz_decode: block check mismatch");
        rc = B200Z_E_DATA;
        got = c.hi;
        break;
      }
    }
  }
  if (rc == p.status && rc == B200Z_E_DATA) set_error_text("xz_decode: the stream is not valid XZ (decodeStream returned false)");
  if (rc == p.status && rc == B200Z_E_THROW) set_error_text("xz_decode: the container walk reads past the input (Dart: RangeError)");
  if (got) XZ_CU(cudaMemcpyAsync(out, x_out.p, (size_t)got, cudaMemcpyDeviceToHost, s));
  XZ_CU(cudaStreamSynchronize(s));
  *out_len = (size_t)got;
  // a damaged stream can declare far more output than it yields (each 6-byte LZMA chunk header up to 2 MiB): the
  // reservation made for it is not kept for the life of the library
  if (rc != B200Z_OK && x_out.cap > ((size_t)64 << 20) && got < x_out.cap / 4) x_out.release();
  return rc;
}

int xz_crc64_impl(const uint8_t *in, size_t n, uint64_t *crc, cudaStream_t s) {
  XZ_CU(x_in.reserve(n + 16));
  if (n) XZ_CU(cudaMemcpyAsync(x_in.p, in, n, cudaMemcpyHostToDevice, s));
  std::vector<uint64_t> c;
  int rc = xz_device_crcs((const uint8_t *)x_in.p, {{0, n}}, true, &c, s);
  if (rc) return rc;
  *crc = c[0];
  return B200Z_OK;
}

size_t xz_encode_bound(size_t n) { return n + 256; }

// XZEncoder.encodeStream (xz_encoder.dart:30-62): header, ONE stored chunk (its 16-bit length field is cut for inputs
// over 64 KiB, :181-182), the check computed on the device, index, footer
int xz_encode_impl(const uint8_t *in, size_t n, int check, uint8_t *out, size_t out_cap, size_t *out_len, cudaStream_t s) {
  static const int FL[4] = {0, 1, 4, 0xa};
  if (check < 0 || check > 3) {
    set_error_text("xz_encode: check must be 0 (none), 1 (crc32), 2 (crc64) or 3 (sha256)");
    return B200Z_E_ARG;
  }
  const int flags = FL[check];
  std::vector<uint8_t> tail;  // check + index + footer
  uint8_t digest[32];
  uint64_t c = 0;
  if (n > 0 && flags) {
    XZ_CU(x_in.reserve(n + 64));
    XZ_CU(cudaMemcpyAsync(x_in.p, in, n, cudaMemcpyHostToDevice, s));
    if (flags == 0xa) {
      XZ_CU(x_meta.reserve(64));
      XZ_LAUNCH(k_xz_sha256, 1, 32, s, (const uint8_t *)x_in.p, (uint64_t)n, (uint8_t *)x_meta.p);
      count_launch();
      XZ_CU(cudaGetLastError());
      XZ_CU(cudaMemcpyAsync(digest, x_meta.p, 32, cudaMemcpyDeviceToHost, s));
      XZ_CU(cudaStreamSynchronize(s));
    } else {
      std::vector<uint64_t> cs;
      int rc = xz_device_crcs((const uint8_t *)x_in.p, {{0, n}}, flags == 4, &cs, s);
      if (rc) return rc;
      c = cs[0];
    }
  }
  std::vector<uint8_t> head = {253, 55, 122, 88, 90, 0, 0, (uint8_t)flags};
  auto put32 = [](std::vector<uint8_t> &v, uint32_t x) {
    for (int i = 0; i < 4; ++i) v.push_back((uint8_t)(x >> (8 * i)));
  };
  auto mbi = [](std::vector<uint8_t> &v, uint64_t x) {
    int shift = 0;
    while ((x >> (shift + 7)) != 0) shift += 7;
    for (; shift > 0; shift -= 7) v.push_back((uint8_t)(0x80 | ((x >> shift) & 0x7f)));
    v.push_back((uint8_t)(x & 0x7f));
  };
  put32(head, host_crc32(head.data() + 6, 2));
  size_t body = 0, pad = 0, unpadded = 0;
  if (n > 0) {
    const uint8_t bh[8] = {2, 0, 0x21, 1, 0x16, 0, 0, 0};
    head.insert(head.end(), bh, bh + 8);
    put32(head, host_crc32(bh, 8));
    head.push_back(1);
    head.push_back((uint8_t)(((n - 1) >> 8) & 0xff));
    head.push_back((uint8_t)((n - 1) & 0xff));
    body = n;
    const size_t after = head.size() + n + 1;
    pad = (4 - after % 4) % 4;
    tail.push_back(0);  // end marker
    tail.insert(tail.end(), pad, 0);
    if (flags == 1) put32(tail, (uint32_t)c);
    if (flags == 4) {
      put32(tail, (uint32_t)c);
      put32(tail, (uint32_t)(c >> 32));
    }
    if (flags == 0xa) tail.insert(tail.end(), digest, digest + 32);
    unpadded = (head.size() - 12) + n + tail.size() - pad;
  }
  std::vector<uint8_t> idx = {0};
  mbi(idx, n > 0 ? 1 : 0);
  if (n > 0) {
    mbi(idx, unpadded);
    mbi(idx, n);
  }
  while (idx.size() % 4) idx.push_back(0);
  put32(idx, host_crc32(idx.data(), idx.size()));
  std::vector<uint8_t> f;
  put32(f, (uint32_t)(idx.size() / 4 - 1));
  f.push_back(0);
  f.push_back((uint8_t)flags);
  tail.insert(tail.end(), idx.begin(), idx.end());
  put32(tail, host_crc32(f.data(), 6));
  tail.insert(tail.end(), f.begin(), f.end());
  tail.push_back(89);
  tail.push_back(90);
  const size_t total = head.size() + body + tail.size();
  *out_len = total;
  if (total > out_cap) {
    set_error_text("xz_encode: out_cap too small (b200z_xz_encode_bound)");
    return B200Z_E_NOSPC;
  }
  memcpy(out, head.data(), head.size());
  if (body) memcpy(out + head.size(), in, body);
  memcpy(out + head.size() + body, tail.data(), tail.size());
  return B200Z_OK;
}

void xz_debug(double *lzma_ms, uint32_t *n_runs) {
  *lzma_ms = g_xz_lzma_ms;
  *n_runs = g_xz_runs;
}

}  // namespace b200z
