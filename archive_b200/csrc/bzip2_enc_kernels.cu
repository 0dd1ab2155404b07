// bzip2_enc_kernels.cu -- BZip2 block encoder on the device (SURVEY.md 8a rows a16-a17).
//
// Reproduces, bit for bit, the stream BZip2Encoder.encodeBytes writes (/root/reference/lib/src/codecs/bzip2_encoder.dart):
//   front end   _writeBlock :83-110, _addCharToBlock/_addPairToBlock :2013-2071   (RLE1, block cut, block CRC)
//   block sort  _blockSort :880-928 (+ _mainSort / _fallbackSort)                  (order of all rotations)
//   MTF         _generateMTFValues :139-265                                         (move-to-front, RUNA/RUNB)
//   entropy     _sendMTFValues :267-745, _hbMakeCodeLengths :747-864, _hbAssignCodes :866-878, bz2_bit_writer.dart
//
// The reference is a serial program; the device formulation is not a translation of it:
//   * the front end is three scans over 4 KiB input tiles (run carry, emitted-byte prefix) and a one-warp walk that
//     places the block cuts by binary search in the prefix (the reference's cut is "first closed run that reaches
//     899 981 bytes, plus the byte that closed it");
//   * the rotation order of a block is unique unless the block is periodic, so it is computed by prefix doubling:
//     a 5-byte radix key first, then (group, rank[i+h]) keys with h = 5, 10, 20 ..., each round one batched LSD radix
//     sort (8-bit digits, 40-bit keys) over the still-unresolved rotations of ALL blocks of the batch, followed by
//     regrouping and compaction.  Periodic blocks (ties that never resolve) take the serial restatement in
//     k_bz2e_serial_sort, because the reference's order among identical rotations is an artefact of its sort;
//   * MTF runs per 2048-symbol chunk from a start list recovered from last-occurrence positions (a max-scan),
//     RUNA/RUNB and the code emission are prefix-sum compactions; the table refinement is one CTA per block.
//
// Built twice: by nvcc for sm_90a (product) and by g++ with -DB200Z_EMU against tests/host_emul/cuda_emu.h (tests).
#ifdef B200Z_EMU
#include "cuda_emu.h"
#define BZ2E_COUNT()
#else
#include <cuda_runtime.h>

#include "b200z_internal.h"
#define BZ2E_COUNT() b200z::count_launch()
#define B200Z_LAUNCH(kern, grid, block, smem, stream, ...) \
  do {                                                     \
    kern<<<grid, block, smem, stream>>>(__VA_ARGS__);      \
    BZ2E_COUNT();                                          \
  } while (0)
#endif
#include <stddef.h>
#include <stdint.h>

#include <vector>

#include "bzip2_enc.h"

namespace b200z {
namespace bz2e {

constexpr uint32_t TI = 4096;              // input tile (bytes)
constexpr uint32_t SUB = 128;              // input sub-tile
constexpr uint32_t SUBS = TI / SUB;        // 32
constexpr uint32_t NBLOCK_MAX = 900000 - 19;  // bzip2_encoder.dart:43 (_nblockMax = 100000 * 9 - 19)
constexpr uint32_t TS = 2048;              // sort / MTF tile (elements)
constexpr uint32_t NT = BZ2E_BSTRIDE / TS;  // 440 tiles per block
static_assert(NT * TS == BZ2E_BSTRIDE, "stride");
constexpr uint32_t ET = 2000;              // emission tile: 40 groups of 50 symbols
constexpr uint32_t NET = 451;              // ceil(900 000 / 2000) + 1

__device__ __forceinline__ uint32_t emit_of(uint32_t cl) { return cl < 4 ? cl : 5u; }

// ---------------------------------------------------------------------------------------------
// A1: per input tile, the end of its stream and the length of its leading and trailing run.  Every stream starts on a
// tile, so no tile holds bytes of two streams.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_e_tile_info(const uint8_t *__restrict__ in, const StreamDesc *__restrict__ sd, uint32_t n_streams,
              uint32_t *__restrict__ t_end, uint32_t *__restrict__ t_head, uint32_t *__restrict__ t_tail) {
  __shared__ uint32_t s_min, s_max, s_n;
  const uint32_t tile = blockIdx.x, t = threadIdx.x;
  const uint32_t base = tile * TI;
  if (t == 0) {
    // the last stream whose first tile is at or before this one: an empty stream has no tile, so it is never the answer
    uint32_t lo = 0, hi = n_streams;
    while (hi - lo > 1) {
      uint32_t mid = (lo + hi) >> 1;
      if (sd[mid].tile0 <= tile) lo = mid;
      else hi = mid;
    }
    s_n = sd[lo].in0 + sd[lo].n;
    t_end[tile] = s_n;
  }
  __syncthreads();
  const uint32_t n = s_n;
  const uint32_t len = umin(TI, n - base);
  if (t == 0) {
    s_min = len;
    s_max = 0;
  }
  __syncthreads();
  const uint8_t f = in[base], l = in[base + len - 1];
  uint32_t mn = len, mx = 0;
  for (uint32_t j = 0; j < 16; ++j) {
    uint32_t i = t * 16 + j;
    if (i >= len) break;
    uint8_t b = in[base + i];
    if (b != f) mn = umin(mn, i);
    if (b != l) mx = umax(mx, i + 1);
  }
  if (mn < len) atomicMin(&s_min, mn);
  if (mx > 0) atomicMax(&s_max, mx);
  __syncthreads();
  if (t == 0) {
    t_head[tile] = s_min;
    t_tail[tile] = len - s_max;
  }
}

// A2: pre[t] = number of bytes immediately before tile t, in its stream, that equal its first byte (a segmented sum over
// tiles that restarts at every stream's first tile)
__global__ void __launch_bounds__(1024)
k_e_tile_pre(const uint8_t *__restrict__ in, uint32_t nt, const uint32_t *__restrict__ t_head,
             const uint32_t *__restrict__ t_tail, const uint32_t *__restrict__ t_end, uint32_t *__restrict__ pre) {
  __shared__ uint32_t s_p[1024], s_v[1024];
  const uint32_t t = threadIdx.x;
  const uint32_t per = (nt + 1023) / 1024;
  const uint32_t lo = umin(nt, umax(1u, t * per)), hi = umin(nt, (t + 1) * per);
  // element k (1 <= k < nt): pre[k] = p ? pre[k-1] + v : v
  uint32_t P = 1, V = 0;
  for (uint32_t k = lo; k < hi; ++k) {
    bool conn = t_end[k - 1] == t_end[k] && in[(size_t)k * TI - 1] == in[(size_t)k * TI];
    bool uni = t_head[k - 1] == TI;
    uint32_t p = conn && uni, v = conn ? (uni ? TI : t_tail[k - 1]) : 0u;
    if (p) V += v;
    else {
      P = 0;
      V = v;
    }
  }
  s_p[t] = P;
  s_v[t] = V;
  __syncthreads();
  if (t == 0) {
    uint32_t run = 0;  // pre[] value in front of each thread's range
    for (uint32_t k = 0; k < 1024; ++k) {
      uint32_t p = s_p[k], v = s_v[k];
      s_v[k] = run;
      run = p ? run + v : v;
    }
  }
  __syncthreads();
  uint32_t run = s_v[t];
  if (t == 0) pre[0] = 0;
  for (uint32_t k = lo; k < hi; ++k) {
    bool conn = t_end[k - 1] == t_end[k] && in[(size_t)k * TI - 1] == in[(size_t)k * TI];
    bool uni = t_head[k - 1] == TI;
    run = conn ? (uni ? run + TI : t_tail[k - 1]) : 0u;
    pre[k] = run;
  }
}

// ---------------------------------------------------------------------------------------------
// A3 / A6: walk the closed runs ("chunks": a run chopped every 255 bytes counted from the start of the run)
// of one tile.  FILL = false: per-tile and per-sub-tile emitted-byte counts.  FILL = true: write the RLE1 bytes of
// every chunk that lies in the scanned region of its block (BlkInfo.e0 <= last byte < BlkInfo.c).
// ---------------------------------------------------------------------------------------------
template <bool FILL>
__global__ void __launch_bounds__(256)
k_e_tile_emit(const uint8_t *__restrict__ in, const uint32_t *__restrict__ t_end, uint32_t tile0, const uint32_t *__restrict__ pre,
              uint32_t *__restrict__ t_sum, uint16_t *__restrict__ sub_sum, uint32_t *__restrict__ sub_pre,
              const unsigned long long *__restrict__ G, const BlkInfo *__restrict__ blk, uint32_t blk_lo, uint32_t blk_hi,
              uint8_t *__restrict__ blockbuf, uint32_t *__restrict__ inuse) {
  __shared__ int s_ls[256];
  __shared__ uint32_t s_sum[256];
  __shared__ uint32_t s_b0;
  __shared__ uint32_t s_use[2][8];
  const uint32_t tile = tile0 + blockIdx.x, t = threadIdx.x;
  const uint32_t base = tile * TI;
  const uint32_t n = t_end[tile];  // end of the tile's stream: no run reaches past it
  const uint32_t len = umin(TI, n - base);
  const uint32_t i0 = t * 16;
  uint8_t by[18];  // by[0] = byte before the range, by[1..16] = the range, by[17] = byte after
  for (uint32_t j = 0; j < 18; ++j) {
    long long g = (long long)base + i0 + j - 1;
    by[j] = (g >= 0 && g < (long long)n && i0 + j - 1 < len + 1) ? in[g] : 0;
  }
  // last run start at or before each position
  int ls = -1;
  for (uint32_t j = 0; j < 16; ++j) {
    uint32_t i = i0 + j;
    if (i >= len) break;
    if (i == 0 || by[j + 1] != by[j]) ls = (int)i;
  }
  s_ls[t] = ls;
  if (FILL) {
    if (t < 16) s_use[t >> 3][t & 7] = 0;
    if (t == 0) {
      // block holding the first byte of the tile
      uint32_t lo = blk_lo, hi = blk_hi;  // blk[lo].start <= base is not guaranteed for the first tile
      while (hi - lo > 1) {
        uint32_t mid = (lo + hi) >> 1;
        if (blk[mid].start <= base) lo = mid;
        else hi = mid;
      }
      s_b0 = lo;
    }
  }
  __syncthreads();
  for (int d = 1; d < 256; d <<= 1) {
    int o = (t >= (uint32_t)d) ? s_ls[t - d] : -1;
    __syncthreads();
    if (o > s_ls[t]) s_ls[t] = o;
    __syncthreads();
  }
  int cur_start = (t > 0) ? s_ls[t - 1] : -1;
  const uint32_t pre_t = pre[tile];
  // pass 1: emitted bytes of the chunks that end in this thread's range
  uint32_t sum = 0;
  {
    int cs = cur_start;
    for (uint32_t j = 0; j < 16; ++j) {
      uint32_t i = i0 + j;
      if (i >= len) break;
      if (i == 0 || by[j + 1] != by[j]) cs = (int)i;
      uint32_t o = i - (uint32_t)cs + (cs == 0 ? pre_t : 0u);
      bool last = (base + i + 1 >= n) || by[j + 2] != by[j + 1];
      if (last || (o + 1) % 255 == 0) sum += emit_of(o % 255 + 1);
      if (!FILL && j == 0 && (t & 7) == 0) sub_pre[tile * SUBS + (t >> 3)] = o;
    }
  }
  if (!FILL) {
    uint32_t v = sum;
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    if ((t & 7) == 0) sub_sum[tile * SUBS + (t >> 3)] = (uint16_t)v;
  }
  s_sum[t] = sum;
  __syncthreads();
  for (int d = 1; d < 256; d <<= 1) {
    uint32_t o = (t >= (uint32_t)d) ? s_sum[t - d] : 0;
    __syncthreads();
    s_sum[t] += o;
    __syncthreads();
  }
  if (!FILL) {
    if (t == 255) t_sum[tile] = s_sum[255];
    return;
  }
  // pass 2 (FILL): place the chunks
  unsigned long long E = G[tile] + (s_sum[t] - sum);
  const uint32_t b0 = s_b0;
  int cs = cur_start;
  for (uint32_t j = 0; j < 16; ++j) {
    uint32_t i = i0 + j;
    if (i >= len) break;
    if (i == 0 || by[j + 1] != by[j]) cs = (int)i;
    uint32_t o = i - (uint32_t)cs + (cs == 0 ? pre_t : 0u);
    bool last = (base + i + 1 >= n) || by[j + 2] != by[j + 1];
    if (!(last || (o + 1) % 255 == 0)) continue;
    uint32_t cl = o % 255 + 1, em = emit_of(cl);
    unsigned long long e_start = E;
    E += em;
    uint32_t gi = base + i;
    uint32_t b = b0, w = 0;
    if (gi >= blk[b].end) {
      b++;
      w = 1;
    }
    if (b < blk_lo || b >= blk_hi) continue;
    const BlkInfo bi = blk[b];
    if (gi < bi.e0 || gi >= bi.c) continue;
    uint8_t ch = by[j + 1];
    uint8_t *dst = blockbuf + (size_t)(b - blk_lo) * BZ2E_BLKBYTES + bi.A + (uint32_t)(e_start - bi.gx0);
    atomicOr(&s_use[w][ch >> 5], 1u << (ch & 31));
    if (cl < 4) {
      for (uint32_t k = 0; k < cl; ++k) dst[k] = ch;
    } else {
      dst[0] = dst[1] = dst[2] = dst[3] = ch;
      dst[4] = (uint8_t)(cl - 4);
      atomicOr(&s_use[w][(cl - 4) >> 5], 1u << ((cl - 4) & 31));
    }
  }
  __syncthreads();
  if (t < 16) {
    uint32_t v = s_use[t >> 3][t & 7];
    uint32_t b = b0 + (t >> 3);
    if (v && b >= blk_lo && b < blk_hi) atomicOr(&inuse[(size_t)(b - blk_lo) * 8 + (t & 7)], v);
  }
}

// exclusive scan u32 -> u64 (one CTA), out[n] = total
__global__ void __launch_bounds__(1024)
k_scan_u32_u64(const uint32_t *__restrict__ in, uint32_t n, unsigned long long *__restrict__ out) {
  __shared__ unsigned long long s[1024];
  const uint32_t t = threadIdx.x;
  const uint32_t per = (n + 1023) / 1024;
  const uint32_t lo = umin(n, t * per), hi = umin(n, lo + per);
  unsigned long long a = 0;
  for (uint32_t k = lo; k < hi; ++k) a += in[k];
  s[t] = a;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {
    unsigned long long o = (t >= (uint32_t)d) ? s[t - d] : 0;
    __syncthreads();
    s[t] += o;
    __syncthreads();
  }
  unsigned long long run = s[t] - a;
  for (uint32_t k = lo; k < hi; ++k) {
    out[k] = run;
    run += in[k];
  }
  if (t == 1023) out[n] = s[1023];
}

// ---------------------------------------------------------------------------------------------
// A5: the block cuts (one warp per stream; every lane runs the same scalar code, only the two searches are lane-parallel).
// The context is the stream alone: positions from its first byte, its tiles, so no search reads past its last byte.
// ---------------------------------------------------------------------------------------------
struct CutCtx {
  const uint8_t *in;
  uint32_t n, nt;
  const uint16_t *sub_sum;
  const uint32_t *sub_pre;
  const unsigned long long *G;
};

// emitted bytes of all chunks (global chopping) whose last byte is < p;  p < n
__device__ unsigned long long gx_at(const CutCtx &c, uint32_t p) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t tile = p / TI, sub = (p % TI) / SUB;
  uint32_t v = (lane < sub) ? c.sub_sum[tile * SUBS + lane] : 0u;
  for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  unsigned long long acc = c.G[tile] + v;
  uint32_t i = tile * TI + sub * SUB;
  uint32_t o = c.sub_pre[tile * SUBS + sub];
  for (; i < p; ++i) {
    bool same = c.in[i + 1] == c.in[i];  // i + 1 <= p < n
    if (!same || (o + 1) % 255 == 0) acc += emit_of(o % 255 + 1);
    o = same ? o + 1 : 0;
  }
  return acc;
}

// end of the run that contains position s
__device__ uint32_t run_end(const CutCtx &c, uint32_t s) {
  const uint32_t lane = threadIdx.x & 31;
  const uint8_t ch = c.in[s];
  uint32_t i = s + 1;
  for (;;) {
    if (i >= c.n) return c.n;
    if ((i % SUB) == 0) {
      // whole sub-tiles of ch: sub-tile k is uniform ch iff sub_pre[k+1] >= SUB and in[(k+1)*SUB] == ch
      uint32_t k = i / SUB + lane;
      unsigned long long nxt = (unsigned long long)(k + 1) * SUB;
      bool ok = nxt < c.n && c.sub_pre[k + 1] >= SUB && c.in[nxt] == ch;
      uint32_t bal = __ballot_sync(0xffffffffu, ok);
      uint32_t cnt = (bal == 0xffffffffu) ? 32u : (uint32_t)(__ffs((int)~bal) - 1);
      i += cnt * SUB;
      if (cnt == 32) continue;
    }
    uint32_t j = i + lane;
    bool diff = j < c.n && c.in[j] != ch;
    bool stop = diff || j >= c.n;
    uint32_t bal = __ballot_sync(0xffffffffu, stop);
    if (bal) {
      uint32_t first = (uint32_t)(__ffs((int)bal) - 1);
      return umin(c.n, i + first);
    }
    uint32_t adv = umin(32u, SUB - (i % SUB));
    i += adv;
  }
}

__global__ void __launch_bounds__(32)
k_e_cut(const uint8_t *__restrict__ in_all, const StreamDesc *__restrict__ sd, const uint16_t *__restrict__ sub_sum_all,
        const uint32_t *__restrict__ sub_pre_all, const unsigned long long *__restrict__ G_all, BlkInfo *__restrict__ blk_all,
        uint32_t *__restrict__ n_blocks_all) {
  const uint32_t si = blockIdx.x;
  const StreamDesc d = sd[si];
  const uint8_t *in = in_all + d.in0;
  const uint32_t n = d.n, nt = d.n_tiles, max_blocks = d.max_blocks;
  const uint16_t *sub_sum = sub_sum_all + (size_t)d.tile0 * SUBS;
  const uint32_t *sub_pre = sub_pre_all + (size_t)d.tile0 * SUBS;
  const unsigned long long *G = G_all + d.tile0;
  BlkInfo *blk = blk_all + d.blk0;
  uint32_t *n_blocks = n_blocks_all + 2 * si;
  CutCtx c{in, n, nt, sub_sum, sub_pre, G};
  const uint32_t lane = threadIdx.x & 31;
  const unsigned long long gtot = n ? G[nt] : 0;
  uint32_t b = 0, s = 0;
  while (s < n && b < max_blocks) {
    const uint32_t e0 = run_end(c, s);
    const uint32_t L0 = e0 - s, full = L0 / 255, rem = L0 % 255;
    uint32_t cpos, F, A, e0u;
    unsigned long long gx0 = 0;
    if ((unsigned long long)5 * full >= NBLOCK_MAX) {
      uint32_t k = (NBLOCK_MAX + 4) / 5;
      cpos = s + 255 * k;
      F = 5 * k;
      A = F;
      e0u = cpos;
    } else {
      A = 5 * full + emit_of(rem);
      e0u = e0;
      if (A >= NBLOCK_MAX || e0 >= n) {
        cpos = e0;
        F = A;
      } else {
        gx0 = gx_at(c, e0);
        const unsigned long long T = gx0 + (NBLOCK_MAX - A);
        if (gtot < T) {
          cpos = n;
          F = A + (uint32_t)(gtot - gx0);
        } else {
          uint32_t lo = e0 / TI, hi = nt;  // largest tile with G[tile] < T
          while (hi - lo > 1) {
            uint32_t mid = (lo + hi) >> 1;
            if (G[mid] < T) lo = mid;
            else hi = mid;
          }
          const uint32_t tile = lo;
          uint32_t v = sub_sum[tile * SUBS + lane], inc = v;
          for (int d = 1; d < 32; d <<= 1) {
            uint32_t o = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= (uint32_t)d) inc += o;
          }
          unsigned long long before = G[tile] + (inc - v);
          uint32_t bal = __ballot_sync(0xffffffffu, before + v >= T);
          uint32_t sub = (uint32_t)(__ffs((int)bal) - 1);  // bal != 0 because G[tile + 1] >= T
          unsigned long long acc = __shfl_sync(0xffffffffu, before, sub);
          uint32_t i = tile * TI + sub * SUB;
          uint32_t o = sub_pre[tile * SUBS + sub];
          cpos = n;
          for (;; ++i) {
            bool same = (i + 1 < n) && in[i + 1] == in[i];
            if (!same || (o + 1) % 255 == 0) {
              acc += emit_of(o % 255 + 1);
              if (acc >= T) {
                cpos = i + 1;
                break;
              }
            }
            o = same ? o + 1 : 0;
          }
          F = A + (uint32_t)(acc - gx0);
        }
      }
    }
    const uint32_t end = cpos < n ? cpos + 1 : n;
    if (lane == 0) {
      BlkInfo bi;
      bi.start = d.in0 + s;
      bi.end = d.in0 + end;
      bi.e0 = d.in0 + e0u;
      bi.c = d.in0 + cpos;
      bi.A = A;
      bi.nblock = F + (cpos < n ? 1u : 0u);
      bi.gx0 = gx0;
      bi.stream = si;
      bi.send = d.in0 + n;
      blk[b] = bi;
    }
    s = end;
    b++;
  }
  if (lane == 0) {
    n_blocks[0] = b;
    n_blocks[1] = (s < n) ? 1u : 0u;  // overflow of the block table
  }
}

// A7: the first run of every block (chopped from the block start, not from the start of the run) + the closing byte
__global__ void __launch_bounds__(256)
k_e_fill_head(const uint8_t *__restrict__ in, const BlkInfo *__restrict__ blk, uint32_t blk_lo,
              uint8_t *__restrict__ blockbuf, uint32_t *__restrict__ inuse) {
  const uint32_t bl = blockIdx.y;
  const BlkInfo bi = blk[blk_lo + bl];
  uint8_t *dst = blockbuf + (size_t)bl * BZ2E_BLKBYTES;
  const uint8_t ch = in[bi.start];
  const uint32_t L = bi.e0 - bi.start, full = L / 255, rem = L % 255;
  for (uint32_t j = blockIdx.x * 256 + threadIdx.x; j < bi.A; j += gridDim.x * 256) {
    uint32_t q = j / 5, r = j % 5;
    uint8_t v;
    if (q < full) v = r < 4 ? ch : (uint8_t)251;
    else {
      uint32_t jj = j - 5 * full;
      v = (rem < 4 || jj < 4) ? ch : (uint8_t)(rem - 4);
    }
    dst[j] = v;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    uint32_t *u = inuse + (size_t)bl * 8;
    atomicOr(&u[ch >> 5], 1u << (ch & 31));
    if (full > 0) atomicOr(&u[251 >> 5], 1u << (251 & 31));
    if (rem >= 4) atomicOr(&u[(rem - 4) >> 5], 1u << ((rem - 4) & 31));
    if (bi.c < bi.send) {
      uint8_t p = in[bi.c];
      dst[bi.nblock - 1] = p;
      atomicOr(&u[p >> 5], 1u << (p & 31));
    }
  }
}

// ---------------------------------------------------------------------------------------------
// A8: block CRCs (bzip2.dart:7-18: MSB-first, 0x04c11db7) over the input bytes of each block
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t bzcrc_mulmod(uint32_t a, uint32_t b) {
  uint32_t r = 0;
  for (int i = 0; i < 32; ++i) {
    if (b & 0x80000000u) r ^= a;
    b <<= 1;
    if (i != 31) r = (r << 1) ^ ((r & 0x80000000u) ? 0x04c11db7u : 0u);
  }
  return r;
}
__device__ uint32_t bzcrc_xpow8(unsigned long long n) {
  uint32_t result = 1u, sq = 0x00000100u;
  while (n) {
    if (n & 1) result = bzcrc_mulmod(result, sq);
    sq = bzcrc_mulmod(sq, sq);
    n >>= 1;
  }
  return result;
}
constexpr uint32_t CRC_PARTS = 32;
__global__ void __launch_bounds__(256)
k_e_crc_part(const uint8_t *__restrict__ in, const BlkInfo *__restrict__ blk, uint32_t blk_lo, uint32_t *__restrict__ part_crc,
             uint32_t *__restrict__ part_len) {
  __shared__ uint32_t crc_tab[256];
  __shared__ uint32_t sm_crc[256], sm_len[256];
  const uint32_t t = threadIdx.x, bl = blockIdx.y, part = blockIdx.x;
  {
    uint32_t v = t << 24;
    for (int k = 0; k < 8; ++k) v = (v & 0x80000000u) ? (v << 1) ^ 0x04c11db7u : v << 1;
    crc_tab[t] = v;
  }
  __syncthreads();
  const BlkInfo bi = blk[blk_lo + bl];
  const uint32_t total = bi.end - bi.start;
  const uint32_t per = (total + CRC_PARTS * 256 - 1) / (CRC_PARTS * 256);
  const uint32_t slice = part * 256 + t;
  const uint32_t lo = (uint32_t)ullmin((unsigned long long)slice * per, total), hi = umin(total, lo + per);
  uint32_t crc = 0;
  for (uint32_t i = lo; i < hi; ++i) crc = (crc << 8) ^ crc_tab[(crc >> 24) ^ in[bi.start + i]];
  sm_crc[t] = crc;
  sm_len[t] = hi - lo;
  __syncthreads();
  for (int d = 1; d < 256; d <<= 1) {
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
  if (t == 255) {
    part_crc[bl * CRC_PARTS + part] = sm_crc[255];
    part_len[bl * CRC_PARTS + part] = sm_len[255];
  }
}
__global__ void k_e_crc_final(const uint32_t *__restrict__ part_crc, const uint32_t *__restrict__ part_len, uint32_t nb,
                              uint32_t *__restrict__ block_crc) {
  const uint32_t bl = blockIdx.x * blockDim.x + threadIdx.x;
  if (bl >= nb) return;
  uint32_t crc = 0;
  unsigned long long len = 0;
  for (uint32_t p = 0; p < CRC_PARTS; ++p) {
    uint32_t l = part_len[bl * CRC_PARTS + p];
    crc = bzcrc_mulmod(crc, bzcrc_xpow8(l)) ^ part_crc[bl * CRC_PARTS + p];
    len += l;
  }
  uint32_t r = bzcrc_mulmod(0xffffffffu, bzcrc_xpow8(len)) ^ crc;
  block_crc[bl] = r ^ 0xffffffffu;
}

// A9: CRC-32 (reflected 0xEDB88320, as zlib's crc32) of every input tile, one thread each; crc32_fold joins a stream's
__global__ void __launch_bounds__(256)
k_e_crc32_tiles(const uint8_t *__restrict__ in, const uint32_t *__restrict__ t_end, uint32_t nt, uint32_t *__restrict__ tile_crc) {
  __shared__ uint32_t tab[256];
  {
    uint32_t c = threadIdx.x;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
    tab[threadIdx.x] = c;
  }
  __syncthreads();
  const uint32_t tile = blockIdx.x * 256 + threadIdx.x;
  if (tile >= nt) return;
  const uint32_t base = tile * TI, len = umin(TI, t_end[tile] - base);
  uint32_t c = 0xffffffffu;
  uint32_t i = 0;
  if (len == TI) {  // tiles start at 4 KiB offsets of the staged input, so whole tiles read as 16-byte words
    const uint4 *w4 = (const uint4 *)(in + base);
    for (; i < TI; i += 16) {
      const uint4 v = w4[i / 16];
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      for (int k = 0; k < 4; ++k)
        for (int b = 0; b < 4; ++b) c = tab[(c ^ (w[k] >> (8 * b))) & 0xffu] ^ (c >> 8);
    }
  }
  for (; i < len; ++i) c = tab[(c ^ in[base + i]) & 0xffu] ^ (c >> 8);
  tile_crc[tile] = c ^ 0xffffffffu;
}

#include "bzip2_enc_sort.inl"
#include "bzip2_enc_entropy.inl"
#include "bzip2_enc_serial.inl"
#include "bzip2_enc_driver.inl"

}  // namespace bz2e
}  // namespace b200z
