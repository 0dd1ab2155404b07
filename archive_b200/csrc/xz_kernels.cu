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
//   k_crc_tiles   CRC-64 (64 KiB tiles) or CRC-32 (8 KiB tiles) of a tile table, one thread each; the host folds them
//                 with x^(8n) mod P.
//   k_xz_sha256   one thread per message of a table (the encoder's SHA-256 check).
//   batches       b200z_xz_decode_batch / _encode_batch: the plans of many streams in one table, each kernel launched
//                 once per device group; the single calls are batches of one.
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
  uint64_t out0;           // its first output byte: nothing in front of it belongs to the run
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
      // the ring starts as the output in front of the chunk (earlier chunks of the run, stored ones included).  Bytes
      // before the run's first byte are never read: they belong to another run, or another stream, which another CTA
      // may be writing (XZ_REACH keeps every reach inside the run, so the ring never needs them).
      const uint64_t pre = min((uint64_t)XZ_WIN, c.out_off - run.out0);
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

// CRC of each tile of a table (any offsets, any lengths), one thread each; W = uint64_t is CRC-64 (ECMA-182, the XZ
// check and getCrc64), W = uint32_t its CRC-32 twin (the XZ CRC-32 check).  Both reflected, with all-ones in and out.
constexpr uint64_t XZ_POLY64 = 0xC96C5795D7870F42ull;
constexpr uint32_t XZ_POLY32 = 0xEDB88320u;
template <class W>
__global__ void __launch_bounds__(256) k_crc_tiles(const uint8_t *__restrict__ d, const uint64_t *__restrict__ tile_off,
                                                   const uint32_t *__restrict__ tile_len, uint32_t n_tiles, W poly,
                                                   W *__restrict__ part) {
  __shared__ W tab[256];
  {
    W c = threadIdx.x;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? poly ^ (c >> 1) : c >> 1;
    tab[threadIdx.x] = c;
  }
  __syncthreads();
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_tiles) return;
  const uint8_t *p = d + tile_off[t];
  const uint32_t n = tile_len[t];
  W c = ~(W)0;
  uint32_t i = 0;
  if (((uintptr_t)p & 15) == 0) {  // 16-byte words where the tile is aligned
    for (; i + 16 <= n; i += 16) {
      const uint4 v = *(const uint4 *)(p + i);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      for (int k = 0; k < 4; ++k)
        for (int b = 0; b < 4; ++b) c = tab[(c ^ (w[k] >> (8 * b))) & 0xff] ^ (c >> 8);
    }
  }
  for (; i < n; ++i) c = tab[(c ^ p[i]) & 0xff] ^ (c >> 8);
  part[t] = ~c;
}

cudaError_t crc32_tiles_launch(const uint8_t *d, const uint64_t *tile_off, const uint32_t *tile_len, uint32_t n_tiles,
                               uint32_t *part, cudaStream_t s) {
  if (!n_tiles) return cudaSuccess;
  XZ_LAUNCH(k_crc_tiles<uint32_t>, (n_tiles + 255) / 256, 256, s, d, tile_off, tile_len, n_tiles, XZ_POLY32, part);
  count_launch();
  return cudaGetLastError();
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
#pragma unroll  // constant indices keep the message schedule w[] in registers
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
// one message of k_xz_sha256: bytes d[off, off + len), digest to digest[32 * slot, + 32)
struct XzMsg {
  uint64_t off, len;
  uint32_t slot, pad_;
};
// one thread per message (SHA-256 is a serial chain); the table is sorted longest first, so the threads of a warp get
// messages of similar lengths
__global__ void __launch_bounds__(32) k_xz_sha256(const uint8_t *__restrict__ d, const XzMsg *__restrict__ msg, uint32_t n_msg,
                                                  uint8_t *__restrict__ digest_base) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_msg) return;
  const XzMsg m = msg[t];
  const uint64_t n = m.len;
  uint8_t *digest = digest_base + 32 * (size_t)m.slot;
  d += m.off;
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

// ---- host: CRC folding (x^(8n) mod P, as zlib's crc32_combine), for CRC-64 and CRC-32 alike ----
// a * b mod P in the reflected representation (the top bit is x^0)
template <class W>
static W xz_mulmod(W a, W b, W poly) {
  W m = (W)1 << (8 * sizeof(W) - 1), p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = (b & 1) ? (b >> 1) ^ poly : b >> 1;
  }
  return p;
}
template <class W>
static W xz_xpow8(uint64_t n, W poly) {  // x^(8n) mod P
  W x = (W)1 << (8 * sizeof(W) - 9);    // x^8
  W p = (W)1 << (8 * sizeof(W) - 1);    // x^0
  while (n) {
    if (n & 1) p = xz_mulmod(x, p, poly);
    n >>= 1;
    if (n) x = xz_mulmod(x, x, poly);
  }
  return p;
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
uint32_t g_xz_max_group = 0;                    // test hook: streams per device group (0: the memory budget alone)
unsigned long long g_xz_stats[3] = {0, 0, 0};  // the last decode call's streams, device groups and runs
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

namespace {
// the host image of a device metadata area (x_meta): every table goes up in one copy; the results lie at its end and
// come back in one copy
struct XzMeta {
  std::vector<uint8_t> h;
  template <class T>
  size_t put(const T *p, size_t count) {
    const size_t o = xz_align(h.size());
    h.resize(o + count * sizeof(T));
    if (count) memcpy(h.data() + o, p, count * sizeof(T));
    return o;
  }
  size_t zeros(size_t bytes) {
    const size_t o = xz_align(h.size());
    h.resize(o + bytes);
    return o;
  }
};

// CRC-64 or CRC-32 of many [lo, hi) ranges of device bytes: their tiles (64 KiB for CRC-64, 8 KiB for CRC-32) in one
// k_crc_tiles launch, folded per range on the host
struct XzTiles {
  bool c64;
  uint64_t tile, full;  // tile bytes; x^(8 tile) mod P
  std::vector<uint64_t> off;
  std::vector<uint32_t> len;
  std::vector<size_t> first{0};  // range r is tiles [first[r], first[r + 1])
  size_t o_off = 0, o_len = 0, o_part = 0;  // where the table and the tile CRCs lie in the metadata area
  explicit XzTiles(bool c)
      : c64(c), tile(c ? 1u << 16 : 1u << 13),
        full(c ? xz_xpow8<uint64_t>(1u << 16, XZ_POLY64) : xz_xpow8<uint32_t>(1u << 13, XZ_POLY32)) {}
  size_t ranges() const { return first.size() - 1; }
  void add(uint64_t lo, uint64_t hi) {
    for (uint64_t o = lo; o < hi; o += tile) {
      off.push_back(o);
      len.push_back((uint32_t)std::min(tile, hi - o));
    }
    first.push_back(off.size());
  }
  void put_table(XzMeta &m) {
    o_off = m.put(off.data(), off.size());
    o_len = m.put(len.data(), len.size());
  }
  void put_result(XzMeta &m) { o_part = m.zeros(off.size() * (c64 ? 8 : 4)); }
  void launch(const uint8_t *d, uint8_t *m, cudaStream_t s) const {
    const uint32_t nt = (uint32_t)off.size();
    if (!nt) return;
    const unsigned grid = (nt + 255) / 256;
    if (c64)
      XZ_LAUNCH(k_crc_tiles<uint64_t>, grid, 256, s, d, (const uint64_t *)(m + o_off), (const uint32_t *)(m + o_len), nt,
                XZ_POLY64, (uint64_t *)(m + o_part));
    else
      XZ_LAUNCH(k_crc_tiles<uint32_t>, grid, 256, s, d, (const uint64_t *)(m + o_off), (const uint32_t *)(m + o_len), nt,
                XZ_POLY32, (uint32_t *)(m + o_part));
    count_launch();
  }
  // the CRC of range r; `res` is the host copy of the metadata area from byte `res0` on
  uint64_t crc(size_t r, const uint8_t *res, size_t res0) const {
    if (c64) return fold<uint64_t>(r, (const uint64_t *)(res + (o_part - res0)), XZ_POLY64);
    return fold<uint32_t>(r, (const uint32_t *)(res + (o_part - res0)), XZ_POLY32);
  }
  template <class W>
  W fold(size_t r, const W *part, W poly) const {
    W c = 0;  // the CRC of nothing
    for (size_t t = first[r]; t < first[r + 1]; ++t)
      c = xz_mulmod<W>(len[t] == tile ? (W)full : xz_xpow8<W>(len[t], poly), c, poly) ^ part[t];
    return c;
  }
};

// one copy of the inputs of streams idx[0..m) to x_in: the span of them as it is, or the inputs packed (16-byte aligned)
// when the span is mostly other bytes.  in_dev[j]: where stream idx[j] starts in x_in.
int xz_stage(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, const size_t *idx, size_t m,
             std::vector<uint64_t> *in_dev, cudaStream_t s) {
  in_dev->assign(m, 0);
  uint64_t lo = ~0ull, hi = 0, total = 0;
  for (size_t j = 0; j < m; ++j) {
    const size_t i = idx[j];
    if (!in_len[i]) continue;
    lo = std::min(lo, in_off[i]);
    hi = std::max(hi, in_off[i] + in_len[i]);
    total += (in_len[i] + 15) & ~15ull;
  }
  if (total == 0) return B200Z_OK;
  std::vector<uint8_t> packed;
  const uint8_t *src = in_base + lo;
  size_t staged = (size_t)(hi - lo);
  if (hi - lo <= 2 * total + ((uint64_t)1 << 20)) {
    for (size_t j = 0; j < m; ++j) (*in_dev)[j] = in_len[idx[j]] ? in_off[idx[j]] - lo : 0;
  } else {
    packed.resize(total);
    staged = 0;
    for (size_t j = 0; j < m; ++j) {
      const size_t i = idx[j];
      (*in_dev)[j] = staged;
      if (in_len[i]) memcpy(packed.data() + staged, in_base + in_off[i], in_len[i]);
      staged += (in_len[i] + 15) & ~15ull;
    }
    src = packed.data();
  }
  XZ_CU(x_in.reserve(staged + 16));
  XZ_CU(cudaMemcpyAsync(x_in.p, src, staged, cudaMemcpyHostToDevice, s));
  return B200Z_OK;
}

// half of what the device has free (with this file's buffers counted as free), at least 1 GiB, at most 24 GiB
int xz_budget(uint64_t *budget) {
  size_t free_b = 0, total_b = 0;
  XZ_CU(cudaMemGetInfo(&free_b, &total_b));
  const uint64_t avail = (uint64_t)free_b + x_in.cap + x_out.cap + x_meta.cap + x_models.cap;
  *budget = std::min<uint64_t>(std::max<uint64_t>(avail / 2, (uint64_t)1 << 30), (uint64_t)24 << 30);
  return B200Z_OK;
}

// one stream of a decode batch
struct XzJob {
  size_t i;  // its index in the call
  XzPlan p;
  uint64_t out_dev = 0;                // its output in x_out
  size_t chunk0 = 0, r32 = 0, r64 = 0;  // its first chunk and first CRC-32 / CRC-64 range in its group's tables
  uint32_t n_global = 0, lclp = 0;     // its runs whose model needs a global slot, and their largest lc + lp
};
}  // namespace

size_t xz_bound(const uint8_t *in, size_t n) {
  XzPlan p;
  xz_plan(in, n, 0, &p);
  return (size_t)p.out_bytes;
}

// Decode the planned streams jobs[0..m) as one device group: one copy up of the inputs and one of the tables, one
// k_xz_copy, one k_xz_lzma over the runs of all streams, one CRC launch per check kind, one copy back of the chunk
// statuses and tile CRCs.  Then each stream replays its own events, and its bytes go to its slot: one copy per stream into
// host slots, one k_copy_slots launch for the whole group into device slots (dev_out).
static int xz_decode_group(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, XzJob *jobs, size_t m,
                           uint8_t *out_base, const uint64_t *out_off, uint64_t *out_len, int32_t *rc, cudaStream_t s,
                           bool dev_out) {
  // ---- the group's tables: chunks, runs and check ranges rebased onto the staged input and the device output ----
  std::vector<size_t> idx(m);
  std::vector<uint64_t> in_dev;
  uint64_t out_total = 0;
  size_t nc = 0;
  for (size_t j = 0; j < m; ++j) {
    idx[j] = jobs[j].i;
    jobs[j].out_dev = out_total;
    out_total += xz_align(jobs[j].p.out_bytes);
    nc += jobs[j].p.chunks.size();
  }
  XZ_CU(x_out.reserve(out_total + 16));
  if (nc) {
    const int r = xz_stage(in_base, in_off, in_len, idx.data(), m, &in_dev, s);
    if (r) return r;
  }
  std::vector<XzChunk> ch;
  std::vector<XzRun> runs;
  std::vector<uint32_t> stored;
  XzTiles t32(false), t64(true);
  ch.reserve(nc);
  for (size_t j = 0; j < m; ++j) {
    XzJob &J = jobs[j];
    const XzPlan &p = J.p;
    J.chunk0 = ch.size();
    J.r32 = t32.ranges();
    J.r64 = t64.ranges();
    const uint32_t run0 = (uint32_t)runs.size();
    for (XzChunk c : p.chunks) {
      c.in_off += in_dev[j];
      c.out_off += J.out_dev;
      c.run += run0;
      if (!c.lzma && c.in_len) stored.push_back((uint32_t)ch.size());
      ch.push_back(c);
    }
    for (XzRun r : p.runs) {
      r.out0 = J.out_dev + p.chunks[r.first].out_off;
      r.first += (uint32_t)J.chunk0;
      runs.push_back(r);
    }
    for (const XzCheck &c : p.checks) (c.c64 ? t64 : t32).add(J.out_dev + c.lo, J.out_dev + c.hi);
  }
  // runs longest first across the group; models that do not fit shared memory get a global slot, all of one size
  const size_t nr = runs.size();
  std::vector<uint32_t> order(nr);
  for (size_t i = 0; i < nr; ++i) order[i] = (uint32_t)i;
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return runs[a].bytes > runs[b].bytes; });
  std::vector<XzRun> sorted(nr);
  uint32_t n_global = 0, big_lclp = 0;
  for (size_t i = 0; i < nr; ++i) {
    sorted[i] = runs[order[i]];
    sorted[i].global_slot = 0xffffffffu;
    if (sorted[i].lclp_max > XZ_SMEM_LCLP) {
      big_lclp = std::max(big_lclp, sorted[i].lclp_max);
      sorted[i].global_slot = n_global++;
    }
  }
  for (auto &r : sorted)
    if (r.global_slot != 0xffffffffu) r.lclp_max = big_lclp;
  XzMeta M;
  const size_t o_ch = M.put(ch.data(), nc), o_runs = M.put(sorted.data(), nr), o_list = M.put(stored.data(), stored.size());
  t32.put_table(M);
  t64.put_table(M);
  const size_t o_ctr = M.zeros(4), o_st = M.zeros(4 * nc);  // results from o_st on
  t32.put_result(M);
  t64.put_result(M);
  const size_t o_end = M.h.size();
  XZ_CU(x_meta.reserve(o_end));
  if (n_global) XZ_CU(x_models.reserve((size_t)n_global * xz_model_words(big_lclp) * 2));
  uint8_t *m_d = (uint8_t *)x_meta.p;
  XZ_CU(cudaMemcpyAsync(m_d, M.h.data(), o_end, cudaMemcpyHostToDevice, s));
  // ---- launches ----
  const uint8_t *d_in = (const uint8_t *)x_in.p;
  const XzChunk *d_ch = (const XzChunk *)(m_d + o_ch);
  if (!stored.empty()) {
    XZ_LAUNCH(k_xz_copy, (unsigned)stored.size(), 256, s, d_in, d_ch, (const uint32_t *)(m_d + o_list), (uint8_t *)x_out.p);
    count_launch();
  }
  if (nr) {
    if (!x_ev[0]) {  // created once, kept for the life of the library
      XZ_CU(cudaEventCreate(&x_ev[0]));
      XZ_CU(cudaEventCreate(&x_ev[1]));
    }
    XZ_CU(cudaEventRecord(x_ev[0], s));
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const unsigned grid = (unsigned)std::min<size_t>(nr, (size_t)sms * 6);  // 6 resident one-warp CTAs per SM (35 KB smem)
    XZ_LAUNCH(k_xz_lzma, grid, 32, s, d_in, d_ch, (const XzRun *)(m_d + o_runs), (uint32_t)nr, (uint32_t *)(m_d + o_ctr),
              (uint16_t *)x_models.p, (uint8_t *)x_out.p, (int32_t *)(m_d + o_st));
    count_launch();
    XZ_CU(cudaGetLastError());
    XZ_CU(cudaEventRecord(x_ev[1], s));
  }
  // the checks: one CRC pass per kind over every verified block of every stream
  t32.launch((const uint8_t *)x_out.p, m_d, s);
  t64.launch((const uint8_t *)x_out.p, m_d, s);
  XZ_CU(cudaGetLastError());
  std::vector<uint8_t> res(o_end - o_st);
  if (!res.empty()) XZ_CU(cudaMemcpyAsync(res.data(), m_d + o_st, res.size(), cudaMemcpyDeviceToHost, s));
  XZ_CU(cudaStreamSynchronize(s));
  if (nr) {
    float ms = 0;
    cudaEventElapsedTime(&ms, x_ev[0], x_ev[1]);
    g_xz_lzma_ms += ms;
  }
  g_xz_runs += (uint32_t)nr;
  g_xz_stats[2] += nr;
  // ---- each stream replays the reference's order: the first chunk that throws, or the first failed check, ends it ----
  const int32_t *status = (const int32_t *)res.data();
  uint64_t got_all = 0;
  bool failed = false;
  std::vector<SlotCopy> to_dev;
  for (size_t j = 0; j < m; ++j) {
    const XzJob &J = jobs[j];
    const XzPlan &p = J.p;
    int r = p.status;
    uint64_t got = p.out_bytes;
    size_t i32 = J.r32, i64 = J.r64;
    for (const XzEvent &e : p.events) {
      if (!e.check) {
        const int32_t st = status[J.chunk0 + e.idx];
        if (st != XZ_OK) {
          static const char *why[] = {"", "a match runs past the chunk's declared size", "a read past the chunk's compressed bytes",
                                      "a reach before dictionary position 0", "posState >= 12 (pb = 4 or 5)"};
          char msg[160];
          snprintf(msg, sizeof msg, "xz_decode: chunk %u: %s (Dart: RangeError)", e.idx, why[st & 7]);
          set_error_text(msg);
          r = B200Z_E_THROW;
          got = p.chunks[e.idx].out_off;
          break;
        }
      } else {
        const XzCheck &c = p.checks[e.idx];
        const uint64_t have = c.c64 ? t64.crc(i64++, res.data(), o_st) : t32.crc(i32++, res.data(), o_st);
        if (have != (c.c64 ? c.want : (c.want & 0xffffffffu))) {
          set_error_text("xz_decode: block check mismatch");
          r = B200Z_E_DATA;
          got = c.hi;
          break;
        }
      }
    }
    if (r == p.status && r == B200Z_E_DATA) set_error_text("xz_decode: the stream is not valid XZ (decodeStream returned false)");
    if (r == p.status && r == B200Z_E_THROW) set_error_text("xz_decode: the container walk reads past the input (Dart: RangeError)");
    if (got && dev_out)
      to_dev.push_back(SlotCopy{J.out_dev, out_off[J.i], got});
    else if (got)
      XZ_CU(cudaMemcpyAsync(out_base + out_off[J.i], (const uint8_t *)x_out.p + J.out_dev, (size_t)got, cudaMemcpyDeviceToHost, s));
    rc[J.i] = r;
    out_len[J.i] = got;
    got_all += got;
    failed |= r != B200Z_OK;
  }
  if (dev_out) XZ_CU(copy_slots((const uint8_t *)x_out.p, out_base, to_dev.data(), to_dev.size(), s));
  XZ_CU(cudaStreamSynchronize(s));
  // a damaged stream can declare far more output than it yields (each 6-byte LZMA chunk header up to 2 MiB): the
  // reservation made for it is not kept for the life of the library
  if (failed && x_out.cap > ((size_t)64 << 20) && got_all < x_out.cap / 4) x_out.release();
  return B200Z_OK;
}

int xz_decode_streams(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                      uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len, int32_t *rc,
                      cudaStream_t s, bool dev_out) {
  g_xz_lzma_ms = 0;
  g_xz_runs = 0;
  g_xz_stats[0] = n;
  g_xz_stats[1] = g_xz_stats[2] = 0;
  // every stream's own walk, clamps, events and checks
  std::vector<XzJob> jobs;
  jobs.reserve(n);
  for (size_t i = 0; i < n; ++i) {
    out_len[i] = 0;
    rc[i] = B200Z_OK;
    XzJob J;
    J.i = i;
    xz_plan(in_len[i] ? in_base + in_off[i] : in_base, (size_t)in_len[i], verify, &J.p);
    if (J.p.out_bytes > out_cap[i]) {
      out_len[i] = J.p.out_bytes;
      rc[i] = B200Z_E_NOSPC;
      set_error_text("xz_decode: out_cap is smaller than the output the stream declares (b200z_xz_bound)");
      continue;
    }
    for (const XzRun &r : J.p.runs)
      if (r.lclp_max > XZ_SMEM_LCLP) {
        J.n_global++;
        J.lclp = std::max(J.lclp, r.lclp_max);
      }
    jobs.push_back(std::move(J));
  }
  if (jobs.empty()) return B200Z_OK;
  uint64_t budget = ~0ull;
  if (jobs.size() > 1) {
    const int r = xz_budget(&budget);
    if (r) return r;
  }
  // consecutive streams in device groups whose input, output, tables and model slots fit the budget; the first stream
  // of a group always goes in, so a stream too large for any group is decoded on its own as the single call does
  for (size_t k = 0; k < jobs.size();) {
    uint64_t bytes = 0, n_global = 0;
    uint32_t lclp = 0;
    size_t e = k;
    for (; e < jobs.size(); ++e) {
      const XzPlan &p = jobs[e].p;
      uint64_t b2 = bytes + xz_align(in_len[jobs[e].i]) + xz_align(p.out_bytes) + p.chunks.size() * (sizeof(XzChunk) + 8) +
                    p.runs.size() * sizeof(XzRun);
      for (const XzCheck &c : p.checks) b2 += ((c.hi - c.lo) / 8192 + 1) * 20;
      const uint64_t g2 = n_global + jobs[e].n_global;
      const uint32_t l2 = std::max(lclp, jobs[e].lclp);
      const uint64_t need = b2 + (g2 ? g2 * xz_model_words(l2) * 2 : 0);
      if (e > k && ((g_xz_max_group && e - k >= g_xz_max_group) || need > budget)) break;
      bytes = b2;
      n_global = g2;
      lclp = l2;
    }
    g_xz_stats[1]++;
    const int r = xz_decode_group(in_base, in_off, in_len, jobs.data() + k, e - k, out_base, out_off, out_len, rc, s, dev_out);
    if (r) return r;
    k = e;
  }
  return B200Z_OK;
}

int xz_decode_impl(const uint8_t *in, size_t n, int verify, uint8_t *out, size_t out_cap, size_t *out_len, cudaStream_t s) {
  const uint64_t off = 0, len = n, cap = out_cap;
  uint64_t got = 0;
  int32_t r1 = B200Z_OK;
  const int rc = xz_decode_streams(in, &off, &len, 1, verify, out, &off, &cap, &got, &r1, s);
  *out_len = (size_t)got;
  return rc ? rc : r1;
}

// CRC tiles over device bytes d, blocking: the table up, one launch, the tile CRCs back into *res (the metadata area
// from byte *res0 on)
static int xz_tiles_run(XzTiles &t, const uint8_t *d, std::vector<uint8_t> *res, size_t *res0, cudaStream_t s) {
  if (t.off.empty()) return B200Z_OK;
  XzMeta M;
  t.put_table(M);
  t.put_result(M);
  *res0 = t.o_part;
  XZ_CU(x_meta.reserve(M.h.size()));
  uint8_t *m_d = (uint8_t *)x_meta.p;
  XZ_CU(cudaMemcpyAsync(m_d, M.h.data(), t.o_part, cudaMemcpyHostToDevice, s));
  t.launch(d, m_d, s);
  XZ_CU(cudaGetLastError());
  res->resize(M.h.size() - t.o_part);
  XZ_CU(cudaMemcpyAsync(res->data(), m_d + t.o_part, res->size(), cudaMemcpyDeviceToHost, s));
  XZ_CU(cudaStreamSynchronize(s));
  return B200Z_OK;
}

int xz_crc64_impl(const uint8_t *in, size_t n, uint64_t *crc, cudaStream_t s) {
  XZ_CU(x_in.reserve(n + 16));
  if (n) XZ_CU(cudaMemcpyAsync(x_in.p, in, n, cudaMemcpyHostToDevice, s));
  XzTiles t(true);
  t.add(0, n);
  std::vector<uint8_t> res;
  size_t res0 = 0;
  const int rc = xz_tiles_run(t, (const uint8_t *)x_in.p, &res, &res0, s);
  if (rc) return rc;
  *crc = t.crc(0, res.data(), res0);
  return B200Z_OK;
}

size_t xz_encode_bound(size_t n) { return n + 256; }

// XZEncoder.encodeStream (xz_encoder.dart:30-62) around the check field `chk` (4, 8 or 32 bytes by flags): header, ONE
// stored chunk (its 16-bit length field is cut for inputs over 64 KiB, :181-182), check, index, footer.  The input's
// bytes go between head and tail.
static void xz_container(size_t n, int flags, const uint8_t *chk, std::vector<uint8_t> *head_p, std::vector<uint8_t> *tail_p) {
  std::vector<uint8_t> &head = *head_p, &tail = *tail_p;
  head = {253, 55, 122, 88, 90, 0, 0, (uint8_t)flags};
  tail.clear();
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
  size_t pad = 0, unpadded = 0;
  if (n > 0) {
    const uint8_t bh[8] = {2, 0, 0x21, 1, 0x16, 0, 0, 0};
    head.insert(head.end(), bh, bh + 8);
    put32(head, host_crc32(bh, 8));
    head.push_back(1);
    head.push_back((uint8_t)(((n - 1) >> 8) & 0xff));
    head.push_back((uint8_t)((n - 1) & 0xff));
    const size_t after = head.size() + n + 1;
    pad = (4 - after % 4) % 4;
    tail.push_back(0);  // end marker
    tail.insert(tail.end(), pad, 0);
    const size_t ck = flags == 1 ? 4 : flags == 4 ? 8 : flags == 0xa ? 32 : 0;
    tail.insert(tail.end(), chk, chk + ck);
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
}

// n XZEncoder().encodeBytes(data, check:) calls.  The checks are the device's: the inputs of a device group go up in one
// copy, then one k_crc_tiles launch (CRC-32 / CRC-64, folded per stream here) or one k_xz_sha256 launch over a table of
// all messages; the containers are written on the host.
int xz_encode_streams(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int check,
                      uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len, int32_t *rc,
                      cudaStream_t s) {
  static const int FL[4] = {0, 1, 4, 0xa};
  if (check < 0 || check > 3) {
    set_error_text("xz_encode: check must be 0 (none), 1 (crc32), 2 (crc64) or 3 (sha256)");
    return B200Z_E_ARG;
  }
  const int flags = FL[check];
  const size_t ck = flags == 1 ? 4 : flags == 4 ? 8 : flags == 0xa ? 32 : 0;
  std::vector<uint8_t> chk(n * ck), head, tail;
  std::vector<size_t> dev;  // the streams whose check the device computes
  for (size_t i = 0; i < n; ++i) {
    xz_container((size_t)in_len[i], flags, chk.data(), &head, &tail);
    out_len[i] = head.size() + in_len[i] + tail.size();
    rc[i] = B200Z_OK;
    if (out_len[i] > out_cap[i]) {
      set_error_text("xz_encode: out_cap too small (b200z_xz_encode_bound)");
      rc[i] = B200Z_E_NOSPC;
    } else if (in_len[i] && flags) {
      dev.push_back(i);
    }
  }
  uint64_t budget = ~0ull;
  if (dev.size() > 1) {
    const int r = xz_budget(&budget);
    if (r) return r;
  }
  for (size_t k = 0; k < dev.size();) {
    size_t e = k;
    for (uint64_t bytes = 0; e < dev.size(); ++e) {
      const uint64_t b2 = bytes + xz_align(in_len[dev[e]]) + (in_len[dev[e]] / 8192 + 1) * 20 + 64;
      if (e > k && b2 > budget) break;
      bytes = b2;
    }
    const size_t m = e - k;
    std::vector<uint64_t> in_dev;
    int r = xz_stage(in_base, in_off, in_len, dev.data() + k, m, &in_dev, s);
    if (r) return r;
    const uint8_t *d_in = (const uint8_t *)x_in.p;
    if (flags == 0xa) {
      // SHA-256: one thread per message, longest first
      std::vector<XzMsg> msg(m);
      for (size_t j = 0; j < m; ++j) msg[j] = XzMsg{in_dev[j], in_len[dev[k + j]], (uint32_t)j, 0};
      std::stable_sort(msg.begin(), msg.end(), [](const XzMsg &a, const XzMsg &b) { return a.len > b.len; });
      XzMeta M;
      const size_t o_msg = M.put(msg.data(), m), o_dig = M.zeros(32 * m);
      XZ_CU(x_meta.reserve(M.h.size()));
      uint8_t *m_d = (uint8_t *)x_meta.p;
      XZ_CU(cudaMemcpyAsync(m_d, M.h.data(), o_dig, cudaMemcpyHostToDevice, s));
      XZ_LAUNCH(k_xz_sha256, (unsigned)((m + 31) / 32), 32, s, d_in, (const XzMsg *)(m_d + o_msg), (uint32_t)m, m_d + o_dig);
      count_launch();
      XZ_CU(cudaGetLastError());
      std::vector<uint8_t> dig(32 * m);
      XZ_CU(cudaMemcpyAsync(dig.data(), m_d + o_dig, 32 * m, cudaMemcpyDeviceToHost, s));
      XZ_CU(cudaStreamSynchronize(s));
      for (size_t j = 0; j < m; ++j) memcpy(chk.data() + 32 * dev[k + j], dig.data() + 32 * j, 32);
    } else {
      XzTiles t(flags == 4);
      for (size_t j = 0; j < m; ++j) t.add(in_dev[j], in_dev[j] + in_len[dev[k + j]]);
      std::vector<uint8_t> res;
      size_t res0 = 0;
      r = xz_tiles_run(t, d_in, &res, &res0, s);
      if (r) return r;
      for (size_t j = 0; j < m; ++j) {
        const uint64_t c = t.crc(j, res.data(), res0);
        for (size_t b = 0; b < ck; ++b) chk[ck * dev[k + j] + b] = (uint8_t)(c >> (8 * b));
      }
    }
    k = e;
  }
  for (size_t i = 0; i < n; ++i) {
    if (rc[i] != B200Z_OK) continue;
    xz_container((size_t)in_len[i], flags, chk.data() + ck * i, &head, &tail);
    uint8_t *out = out_base + out_off[i];
    memcpy(out, head.data(), head.size());
    if (in_len[i]) memcpy(out + head.size(), in_base + in_off[i], (size_t)in_len[i]);
    memcpy(out + head.size() + in_len[i], tail.data(), tail.size());
  }
  return B200Z_OK;
}

int xz_encode_impl(const uint8_t *in, size_t n, int check, uint8_t *out, size_t out_cap, size_t *out_len, cudaStream_t s) {
  const uint64_t off = 0, len = n, cap = out_cap;
  uint64_t got = 0;
  int32_t r1 = B200Z_OK;
  const int rc = xz_encode_streams(in, &off, &len, 1, check, out, &off, &cap, &got, &r1, s);
  if (rc) return rc;
  *out_len = (size_t)got;
  return r1;
}

void xz_debug(double *lzma_ms, uint32_t *n_runs) {
  *lzma_ms = g_xz_lzma_ms;
  *n_runs = g_xz_runs;
}
void xz_batch_set(uint32_t max_streams) { g_xz_max_group = max_streams; }
void xz_batch_stats(unsigned long long out[3]) {
  for (int k = 0; k < 3; ++k) out[k] = g_xz_stats[k];
}

}  // namespace b200z
