// b200z_api.cu -- the C ABI (include/b200z.h): context, staging, and the host-side framing logic
// that sits between the reference's codec classes and the kernels.
//
// Host logic restated here (reference, paths relative to /root/reference/):
//   lib/src/codecs/zlib/_gzip_decoder_web.dart:27-138   member loop + header skip
//   lib/src/codecs/zlib/_zlib_decoder_web.dart:31-107   stream loop + FCHECK/FDICT + Adler verify
// The byte-level work (Huffman decode, LZ77, Adler-32) runs on the GPU; nothing here decodes.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "b200z_internal.h"
#include "bzip2_enc.h"
#ifdef B200Z_EMU
// The CPU emulation build of the library compiles the generated copies of the .cu files it lists; the encrypted-member
// and XZ kernels come in here (zip_crypt_kernels.cu and xz_kernels.cu launch through macros both compilers take).  The
// emulated runtime's pointer attributes come from the test tree (tests/host_emul/cuda_emu_pointer.h).
#include "cuda_emu_pointer.h"
#include "zip_crypt_kernels.cu"
#include "xz_kernels.cu"
#endif

namespace b200z {

static thread_local char t_err[512] = "";
static void set_err(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(t_err, sizeof t_err, fmt, ap);
  va_end(ap);
}

static std::atomic<uint64_t> g_launches{0};
static std::atomic<unsigned long long> g_bz2_fast_blocks{0}, g_bz2_exact_blocks{0};  // K7: blocks by the fast / the exact kernel
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

struct DevBuf {
  void *p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = n + (n >> 3) + 4096;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) {
      p = nullptr;
      return e;
    }
    cap = want;
    return cudaSuccess;
  }
  // grow but keep the first `keep` bytes (decoded members already sitting in the buffer)
  cudaError_t reserve_keep(size_t n, size_t keep, cudaStream_t s) {
    if (n <= cap) return cudaSuccess;
    size_t want = n + (n >> 2) + 4096;
    void *np = nullptr;
    cudaError_t e = cudaMalloc(&np, want);
    if (e != cudaSuccess) return e;
    if (p && keep) {
      e = cudaMemcpyAsync(np, p, keep < cap ? keep : cap, cudaMemcpyDeviceToDevice, s);
      if (e == cudaSuccess) e = cudaStreamSynchronize(s);
      if (e != cudaSuccess) {
        cudaFree(np);
        return e;
      }
    }
    if (p) cudaFree(p);
    p = np;
    cap = want;
    return cudaSuccess;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};
struct PinBuf {
  void *p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
    size_t want = n + (n >> 2) + 4096;
    cudaError_t e = cudaHostAlloc(&p, want, cudaHostAllocDefault);
    if (e != cudaSuccess) {
      p = nullptr;
      return e;
    }
    cap = want;
    return cudaSuccess;
  }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
  }
};

struct Ctx {
  std::mutex mu;
  bool inited = false;
  int device = -1;
  cudaStream_t stream = nullptr, s_h2d = nullptr, s_d2h = nullptr;
  static const int kCompStreams = 8;
  cudaStream_t s_comp[kCompStreams] = {};
  DevBuf d_in, d_out, d_ws, d_meta, d_small, d_bz, d_tok, d_crypt;
  DevBuf d_slots;  // the piece table of k_copy_slots (copy_slots)
  PinBuf h_meta, h_stage;  // h_stage: the outputs of a gzip / zlib decode batch on their way to the caller's slots (GZ_STAGE)
};
static Ctx g;

#define CU(x)                                                                       \
  do {                                                                              \
    cudaError_t e__ = (x);                                                          \
    if (e__ != cudaSuccess) {                                                       \
      set_err("%s failed: %s (%s:%d)", #x, cudaGetErrorString(e__), __FILE__, __LINE__); \
      return B200Z_E_NODEVICE;                                                      \
    }                                                                               \
  } while (0)

static int require_init() {
  if (!g.inited) {
    set_err("b200z_init has not been called (or no CUDA device): there is no CPU fallback");
    return B200Z_E_NODEVICE;
  }
  return B200Z_OK;
}

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ---------------------------------------------------------------------------------------------
// Adler-32 on the device (adler32.dart:29-52).  s1 = 1 + sum b_i ; s2 = n + sum (n - i) b_i  (mod 65521)
// Each block reduces one tile of at most 64 KiB to (sum, weighted sum); a launch takes the tiles of many messages.  The
// host folds each message's per-tile pairs (a few integers per 64 KiB -- framing arithmetic, not a pass over the data).
// ---------------------------------------------------------------------------------------------
constexpr uint32_t ADLER_TILE = 1u << 16;
struct AdlerTile {
  uint64_t off;  // first byte, from the launch's base pointer
  uint32_t len, pad_;
};
__global__ void __launch_bounds__(256) k_adler_tiles(const uint8_t *__restrict__ base, const AdlerTile *__restrict__ tiles,
                                                     uint64_t *__restrict__ part) {
  const uint8_t *p = base + tiles[blockIdx.x].off;
  const uint32_t len = tiles[blockIdx.x].len;
  uint64_t s = 0, ws = 0;  // ws = sum (len - i) * b_i  within the tile
  for (uint32_t i = threadIdx.x; i < len; i += blockDim.x) {
    uint32_t b = p[i];
    s += b;
    ws += (uint64_t)(len - i) * b;
  }
  __shared__ uint64_t sh[2][8];
  for (int d = 16; d >= 1; d >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, d);
    ws += __shfl_xor_sync(0xffffffffu, ws, d);
  }
  if ((threadIdx.x & 31) == 0) {
    sh[0][threadIdx.x >> 5] = s;
    sh[1][threadIdx.x >> 5] = ws;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint64_t a = 0, b = 0;
    for (int i = 0; i < 8; ++i) {
      a += sh[0][i];
      b += sh[1][i];
    }
    part[2 * blockIdx.x] = a;
    part[2 * blockIdx.x + 1] = b;
  }
}

// Adler-32 of the n device messages base[off[m], off[m] + len[m]) with one launch and one synchronise (blocking)
static int device_adler32_many(const uint8_t *base, const uint64_t *off, const uint64_t *len, size_t n, uint32_t *out) {
  const uint32_t MOD = 65521;
  std::vector<AdlerTile> tiles;
  for (size_t m = 0; m < n; ++m)
    for (uint64_t t = 0; t < len[m]; t += ADLER_TILE)
      tiles.push_back({off[m] + t, (uint32_t)std::min<uint64_t>(ADLER_TILE, len[m] - t), 0});
  std::vector<uint64_t> part(tiles.size() * 2);
  if (!tiles.empty()) {
    const size_t nt = tiles.size(), tab = align_up(nt * 16, 256);
    CU(g.d_small.reserve(tab + nt * 16));
    CU(cudaMemcpyAsync(g.d_small.p, tiles.data(), nt * sizeof(AdlerTile), cudaMemcpyHostToDevice, g.stream));
    uint64_t *d_part = (uint64_t *)((uint8_t *)g.d_small.p + tab);
    k_adler_tiles<<<(unsigned)nt, 256, 0, g.stream>>>(base, (const AdlerTile *)g.d_small.p, d_part);
    count_launch();
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(part.data(), d_part, nt * 16, cudaMemcpyDeviceToHost, g.stream));
    CU(cudaStreamSynchronize(g.stream));
  }
  size_t t = 0;
  for (size_t m = 0; m < n; ++m) {
    uint64_t s1 = 1, s2 = 0;
    for (uint64_t at = 0; at < len[m]; at += ADLER_TILE, ++t) {
      const uint64_t tl = std::min<uint64_t>(ADLER_TILE, len[m] - at);
      uint64_t ts = part[2 * t] % MOD, tw = part[2 * t + 1] % MOD;
      // appending a tile: s2' = s2 + len * s1 + tw ; s1' = s1 + ts
      s2 = (s2 + (tl % MOD) * s1 + tw) % MOD;
      s1 = (s1 + ts) % MOD;
    }
    out[m] = (uint32_t)((s2 << 16) | s1);
  }
  return B200Z_OK;
}

// device buffer -> adler32 (blocking)
static int device_adler32(const uint8_t *d, size_t n, uint32_t *out) {
  const uint64_t off = 0, len = n;
  return device_adler32_many(d, &off, &len, 1, out);
}

// ---------------------------------------------------------------------------------------------
// k_copy_slots: the device sink of the decode batches.  The host cuts every SlotCopy into pieces of at most COPY_PIECE bytes
// and each warp takes one piece at a time, so a large slot spreads over many CTAs and small slots share one.  Stores are
// 16-byte vectors from the destination's first 16-byte boundary on, with byte heads and tails.  When source and destination
// disagree modulo 16, each stored vector is cut from the two aligned source vectors it straddles (both hold bytes of the
// piece, so nothing outside the source's aligned 16-byte blocks is read).  Nothing outside [dst, dst + len) is written.
// ---------------------------------------------------------------------------------------------
constexpr uint64_t COPY_PIECE = 64u << 10;
constexpr unsigned COPY_THREADS = 256;

// bytes [4q + r/8, +16) of the 32 bytes a || b (q in 0..3, r in {0, 8, 16, 24}); q is the same for the whole warp
__device__ __forceinline__ uint4 copy_shift16(const uint4 a, const uint4 b, uint32_t q, uint32_t r) {
  switch (q) {
    case 0: return make_uint4(__funnelshift_r(a.x, a.y, r), __funnelshift_r(a.y, a.z, r), __funnelshift_r(a.z, a.w, r), __funnelshift_r(a.w, b.x, r));
    case 1: return make_uint4(__funnelshift_r(a.y, a.z, r), __funnelshift_r(a.z, a.w, r), __funnelshift_r(a.w, b.x, r), __funnelshift_r(b.x, b.y, r));
    case 2: return make_uint4(__funnelshift_r(a.z, a.w, r), __funnelshift_r(a.w, b.x, r), __funnelshift_r(b.x, b.y, r), __funnelshift_r(b.y, b.z, r));
    default: return make_uint4(__funnelshift_r(a.w, b.x, r), __funnelshift_r(b.x, b.y, r), __funnelshift_r(b.y, b.z, r), __funnelshift_r(b.z, b.w, r));
  }
}

__global__ void __launch_bounds__(COPY_THREADS) k_copy_slots(const uint8_t *__restrict__ src, uint8_t *__restrict__ dst,
                                                            const SlotCopy *__restrict__ pieces, uint32_t n) {
  const uint32_t lane = threadIdx.x & 31, n_warps = gridDim.x * (COPY_THREADS / 32);
  for (uint32_t w = blockIdx.x * (COPY_THREADS / 32) + (threadIdx.x >> 5); w < n; w += n_warps) {
    const SlotCopy c = pieces[w];
    const uint8_t *s = src + c.src;
    uint8_t *d = dst + c.dst;
    const uint32_t to16 = (uint32_t)(-(uintptr_t)d & 15);
    const uint32_t head = c.len < to16 ? (uint32_t)c.len : to16;
    if (lane < head) d[lane] = s[lane];
    const uint64_t nv = (c.len - head) >> 4;
    uint4 *dv = (uint4 *)(d + head);
    const uint8_t *sh = s + head;
    const uint32_t k = (uint32_t)((uintptr_t)sh & 15);
    const uint4 *sv = (const uint4 *)(sh - k);
    if (k == 0) {
      for (uint64_t i = lane; i < nv; i += 32) dv[i] = sv[i];
    } else {
      for (uint64_t i = lane; i < nv; i += 32) dv[i] = copy_shift16(sv[i], sv[i + 1], k >> 2, 8 * (k & 3));
    }
    for (uint64_t i = head + (nv << 4) + lane; i < c.len; i += 32) d[i] = s[i];
  }
}

cudaError_t copy_slots(const uint8_t *src, uint8_t *dst, const SlotCopy *copies, size_t n, cudaStream_t s) {
  std::vector<SlotCopy> pieces;
  for (size_t i = 0; i < n; ++i)
    for (uint64_t at = 0; at < copies[i].len; at += COPY_PIECE)
      pieces.push_back(SlotCopy{copies[i].src + at, copies[i].dst + at, std::min(COPY_PIECE, copies[i].len - at)});
  if (pieces.empty()) return cudaSuccess;
  cudaError_t e = g.d_slots.reserve(pieces.size() * sizeof(SlotCopy));
  if (e == cudaSuccess) e = cudaMemcpyAsync(g.d_slots.p, pieces.data(), pieces.size() * sizeof(SlotCopy), cudaMemcpyHostToDevice, s);
  if (e != cudaSuccess) return e;
  const size_t per_cta = COPY_THREADS / 32;
  const unsigned grid = (unsigned)std::min<size_t>((pieces.size() + per_cta - 1) / per_cta, 1u << 16);
  k_copy_slots<<<grid, COPY_THREADS, 0, s>>>(src, dst, (const SlotCopy *)g.d_slots.p, (uint32_t)pieces.size());
  count_launch();
  return cudaGetLastError();
}

// A *_to_device decode batch: d_out_base is device memory of the library's device whenever a slot has room (with no room
// at all nothing is ever written, and the host batches' rules already let such a base be anything)
static int device_out_arg(const char *name, const uint8_t *d_out_base, size_t n, const uint64_t *out_cap) {
  bool room = false;
  for (size_t i = 0; i < n && !room; ++i) room = out_cap[i] != 0;
  if (!room) return B200Z_OK;
  cudaPointerAttributes a;
  if (!d_out_base || cudaPointerGetAttributes(&a, d_out_base) != cudaSuccess) {
    cudaGetLastError();
    set_err("%s: d_out_base is not a CUDA pointer", name);
    return B200Z_E_ARG;
  }
  if (a.type != cudaMemoryTypeDevice || a.device != g.device) {
    set_err("%s: d_out_base is not device memory of device %d", name, g.device);
    return B200Z_E_ARG;
  }
  return B200Z_OK;
}

// the library's stream waits for what the caller enqueued on cuda_stream before the call (NULL: the library's own stream)
static int wait_for_caller(void *cuda_stream) {
  if (!cuda_stream) return B200Z_OK;
  cudaEvent_t ev;
  CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  const cudaError_t e1 = cudaEventRecord(ev, (cudaStream_t)cuda_stream);
  const cudaError_t e2 = e1 == cudaSuccess ? cudaStreamWaitEvent(g.stream, ev, 0) : e1;
  cudaEventDestroy(ev);  // (released once it has completed)
  CU(e2);
  return B200Z_OK;
}

// ---------------------------------------------------------------------------------------------
// batch plumbing
// ---------------------------------------------------------------------------------------------
struct MetaLayout {
  size_t n;
  size_t off_in_off, off_out_off, off_in_len, off_out_cap, off_out_len, off_status, off_in_used, off_hist, bytes;
  explicit MetaLayout(size_t n_) : n(n_) {
    size_t o = 0;
    off_in_off = o;
    o += 8 * n;
    off_out_off = o;
    o += 8 * n;
    off_in_len = o;
    o += 4 * n;
    off_out_cap = o;
    o += 4 * n;
    off_out_len = o;
    o += 4 * n;
    off_status = o;
    o += 4 * n;
    off_in_used = o;
    o += 4 * n;
    off_hist = o;  // (per-unit history, when a batch has one: InflateWs::unit_hist)
    o += 4 * n;
    bytes = align_up(o, 256);
  }
  size_t inputs_bytes() const { return off_out_len; }
};

static size_t workspace_bytes(size_t n_units, size_t total_out_cap) { return inflate_ws_bytes(n_units, total_out_cap); }

// Runs one batch whose compressed bytes are ALREADY in g.d_in (at offset 0 = in_base) and whose
// output goes to g.d_out.  Meta arrays are host arrays; results are copied back into them.  `unit_hist`: each unit's own
// history (InflateWs::unit_hist), or null.
static int run_batch_on_staged(const uint64_t *in_off, const uint32_t *in_len, const uint64_t *out_off,
                               const uint32_t *out_cap, uint32_t *out_len, int32_t *status, uint32_t *in_used,
                               size_t n, size_t out_extent, bool count_only = false, uint32_t hist = 0,
                               const uint32_t *unit_hist = nullptr) {
  MetaLayout ml(n);
  CU(g.h_meta.reserve(ml.bytes));
  CU(g.d_meta.reserve(ml.bytes));
  uint8_t *hm = (uint8_t *)g.h_meta.p;
  memcpy(hm + ml.off_in_off, in_off, 8 * n);
  memcpy(hm + ml.off_out_off, out_off, 8 * n);
  memcpy(hm + ml.off_in_len, in_len, 4 * n);
  memcpy(hm + ml.off_out_cap, out_cap, 4 * n);
  CU(cudaMemcpyAsync(g.d_meta.p, hm, ml.inputs_bytes(), cudaMemcpyHostToDevice, g.stream));
  if (unit_hist) {
    memcpy(hm + ml.off_hist, unit_hist, 4 * n);
    CU(cudaMemcpyAsync((uint8_t *)g.d_meta.p + ml.off_hist, hm + ml.off_hist, 4 * n, cudaMemcpyHostToDevice, g.stream));
  }
  const size_t ws = workspace_bytes(n, out_extent);
  CU(g.d_ws.reserve(ws));
  uint8_t *dm = (uint8_t *)g.d_meta.p;
  InflateBatch b;
  b.in_base = (const uint8_t *)g.d_in.p;
  b.in_off = (const uint64_t *)(dm + ml.off_in_off);
  b.in_len = (const uint32_t *)(dm + ml.off_in_len);
  b.out_base = (uint8_t *)g.d_out.p;
  b.out_off = (const uint64_t *)(dm + ml.off_out_off);
  b.out_cap = (const uint32_t *)(dm + ml.off_out_cap);
  b.out_len = (uint32_t *)(dm + ml.off_out_len);
  b.status = (int32_t *)(dm + ml.off_status);
  b.in_used = (uint32_t *)(dm + ml.off_in_used);
  b.n_units = n;
  b.ws = inflate_ws_carve(g.d_ws.p, n, out_extent);
  b.ws.hist = hist;
  if (unit_hist) b.ws.unit_hist = (const uint32_t *)(dm + ml.off_hist);
  b.count_only = count_only;
  CU(launch_inflate(b, g.stream));
  CU(cudaMemcpyAsync(hm + ml.off_out_len, dm + ml.off_out_len, ml.off_hist - ml.off_out_len, cudaMemcpyDeviceToHost,
                     g.stream));
  CU(cudaStreamSynchronize(g.stream));
  memcpy(out_len, hm + ml.off_out_len, 4 * n);
  memcpy(status, hm + ml.off_status, 4 * n);
  memcpy(in_used, hm + ml.off_in_used, 4 * n);
  return B200Z_OK;
}

static int stage_input(const uint8_t *in, size_t n) {
  CU(g.d_in.reserve(n + 64));
  if (n) CU(cudaMemcpyAsync(g.d_in.p, in, n, cudaMemcpyHostToDevice, g.stream));
  return B200Z_OK;
}

// largest possible DEFLATE expansion: a 258-byte match costs at least 2 bits
static size_t max_inflate_out(size_t in_len) {
  const size_t lim = (size_t)0xffffffffu;
  if (in_len > lim / 1040) return lim;
  return in_len * 1040 + 1024;
}

// one stream from staged input at [pos, in_total): returns unit results
struct OneResult {
  uint32_t out_len, in_used;
  int32_t status;
};
// `shared_output`: the stream is a gzip member -- everything already in g.d_out[0, out_pos) belongs to the same OutputStream
// and is within reach of its back-references (InflateWs::hist)
// ---------------------------------------------------------------------------------------------
// K12: large streams, each decoded by many chunks (inflate_chunked.cuh, DESIGN.md "K12").  A stream's compressed input is
// worked through in regions that double from g_ck.thresh bytes: per region the block finder guesses a block start in
// every chunk, all chunks decode at once, the chain is proven on the host from the region's exact start and the chunks
// that started at a wrong guess are redone from their predecessor's end; then the windows are resolved and the region
// is written to its final place.  The result is accepted only when the chain reaches a final block with every chunk
// on it clean, no back-reference reaches before the allowed history and the output fits the cap; anything else leaves
// the stream to the exact path, which gives every other result exactly.  A batch of streams (large ZIP members) moves
// through these phases in lockstep, one launch per phase for all of them; a single stream is the batch of one.
// ---------------------------------------------------------------------------------------------
// Compressed bytes from which a stream takes K12, and the chunk size (0: a region's bytes over CK_TARGET, at least
// CK_MIN_CHUNK).  Both are set by the benchmark's measurements (DESIGN.md "K12"); b200z_debug_inflate_chunked_set moves them
// for tests.
constexpr size_t CK_THRESH = 16u << 20;
constexpr size_t CK_MIN_CHUNK = 32u << 10;
constexpr size_t CK_TARGET = 2048;
constexpr int CK_MAX_ROUNDS = 16;  // redo rounds per region before the stream goes to the exact path
struct CkConfig {
  size_t thresh = CK_THRESH, chunk = 0;
};
static CkConfig g_ck;
static unsigned long long g_ck_stats[6];  // last call: regions, chunks, redo rounds, chunks merged, fell back, chunked path ran
static double g_ck_ms[3];  // last call's kernel times (CUDA events): block finder, chunk decodes (all rounds), windows + emit
// Times the kernels of one phase of run_chunked on g.stream; the phase's own synchronisation makes the reading cheap.
struct CkTimer {
  cudaEvent_t a = nullptr, b = nullptr;
  CkTimer() {
    cudaEventCreate(&a);
    cudaEventCreate(&b);
  }
  ~CkTimer() {
    cudaEventDestroy(a);
    cudaEventDestroy(b);
  }
  void start() { cudaEventRecord(a, g.stream); }
  void stop(double *acc) {
    cudaEventRecord(b, g.stream);
    float ms = 0.f;
    if (cudaEventSynchronize(b) == cudaSuccess && cudaEventElapsedTime(&ms, a, b) == cudaSuccess) *acc += ms;
  }
};

static size_t ck_carve(size_t &o, size_t bytes) {
  const size_t at = o;
  o = align_up(o + bytes, 256);
  return at;
}

// One stream of a K12 batch, as the host sees it.
struct CkIn {
  const uint8_t *h_in;  // host copy of its compressed bytes (the stored-block checks below read a few of them)
  size_t pos;           // its first compressed byte in g.d_in
  uint32_t il;          // its compressed bytes
  size_t out_pos;       // its first output byte in g.d_out
  uint32_t oc;          // its output room
  uint32_t hist;        // bytes in front of out_pos its back-references may reach
  uint32_t n_pages;     // its share of the pool (ck_pages_for, not 0)
};
struct CkOut {
  bool accepted = false;
  OneResult r{};
  unsigned long long stats[5] = {};  // regions, chunks, redo rounds, chunks merged, fell back
};

// g.d_ws for a batch of ns streams: the per-chunk records, the stream table and counters, then n_pages pages
struct CkLayout {
  size_t finds, cand, jobs, res, chain, chain_lo, streams, ctr, fixed, pinfo, flat, pool, bytes;
  CkLayout(size_t ns, size_t n_pages) {
    const size_t mc = ns * (CK_TARGET + 8);
    size_t o = 0;
    finds = ck_carve(o, mc * sizeof(CkFind));
    cand = ck_carve(o, mc * 8);
    jobs = ck_carve(o, mc * sizeof(CkJob));
    res = ck_carve(o, mc * sizeof(CkRes));
    chain = ck_carve(o, mc * sizeof(CkChain));
    chain_lo = ck_carve(o, (ns + 1) * 4);
    streams = ck_carve(o, ns * sizeof(CkStream));
    ctr = ck_carve(o, ns * 8);  // page counters, then "reached too far" flags
    fixed = o;
    pinfo = ck_carve(o, n_pages * sizeof(CkPage));
    flat = ck_carve(o, n_pages * 8);  // the flat page list, then the chain entry of each
    pool = ck_carve(o, n_pages * (size_t)CK_PAGE * 2);
    bytes = o;
  }
};
// a page: its symbols, its record and its two flat-list entries
constexpr size_t CK_PER_PAGE = (size_t)CK_PAGE * 2 + sizeof(CkPage) + 8;

// The pages of one stream's pool when it may use `ws` bytes -- the exact path's workspace for the same output, so that K12
// never takes more device memory than the exact path would -- or 0 when that is too small to be worth carving.
// (Checked before the subtraction: a small output room gives a small workspace.  The 1024 bytes cover the alignment of
// the three page arrays.)
static uint32_t ck_pages_for(size_t ws) {
  const size_t fixed = CkLayout(1, 0).fixed;
  if (ws < fixed + 1024 + 8 * CK_PER_PAGE) return 0;
  return (uint32_t)std::min<size_t>((ws - fixed - 1024) / CK_PER_PAGE, 0xffffffu);
}

// Moves every stream of `in` through K12 in lockstep: per phase one launch for all the streams still live (the block
// finder, the chunk decodes, each redo round, windows + emit).  Every acceptance and fallback rule is the single stream's,
// applied per stream: a stream that falls back drops out and leaves the others running.  out[s].accepted: K12 produced
// stream s's result (out[s].r); otherwise it is the exact path's to decode.  An error code only for CUDA failures.
static int run_chunked(const std::vector<CkIn> &in, std::vector<CkOut> &out, double ms[3]) {
  const size_t ns = in.size();
  out.assign(ns, CkOut());
  CkTimer tm;
  size_t total_pages = 0;
  for (const CkIn &c : in) total_pages += c.n_pages;
  const CkLayout ly(ns, total_pages);
  CU(g.d_ws.reserve(ly.bytes));
  uint8_t *w = (uint8_t *)g.d_ws.p;
  auto *d_finds = (CkFind *)(w + ly.finds);
  auto *d_cand = (unsigned long long *)(w + ly.cand);
  auto *d_jobs = (CkJob *)(w + ly.jobs);
  auto *d_res = (CkRes *)(w + ly.res);
  auto *d_chain = (CkChain *)(w + ly.chain);
  auto *d_chain_lo = (uint32_t *)(w + ly.chain_lo);
  auto *d_streams = (CkStream *)(w + ly.streams);
  auto *d_ctr = (uint32_t *)(w + ly.ctr), *d_bad = d_ctr + ns;
  auto *d_pinfo = (CkPage *)(w + ly.pinfo);
  auto *d_flat = (uint32_t *)(w + ly.flat);
  auto *d_pool = (uint16_t *)(w + ly.pool);
  const uint8_t *d_in = (const uint8_t *)g.d_in.p;
  uint8_t *d_out = (uint8_t *)g.d_out.p;

  struct St {  // a stream's progress
    bool live = true, final_seen = false, proving = false;
    unsigned long long bit0 = 0, end_bits = 0, pos_b = 0;  // the region's exact start; the input's end; the proven end
    size_t emitted = 0, R = 0, rend = 0, span = 0, n = 0, find0 = 0, job0 = 0, total = 0;
    std::vector<unsigned long long> S, cand;
    std::vector<CkJob> jobs;
    std::vector<CkRes> res;
    std::vector<uint32_t> on_chain;
  };
  std::vector<St> st(ns);
  std::vector<CkStream> tab(ns);
  for (size_t s = 0, page0 = 0; s < ns; ++s) {
    tab[s] = CkStream{(unsigned long long)in[s].pos, (unsigned long long)(in[s].out_pos - in[s].hist), in[s].il, (uint32_t)page0,
                      in[s].n_pages, 0};
    page0 += in[s].n_pages;
    st[s].end_bits = 8ull * in[s].il;
    st[s].R = g_ck.thresh;
  }
  CU(cudaMemcpyAsync(d_streams, tab.data(), ns * sizeof(CkStream), cudaMemcpyHostToDevice, g.stream));
  auto fall = [&](size_t s) {
    out[s].stats[4] = 1;
    st[s].live = false;
  };
  // A block that is not final starts at `e` with a stored header that reads the same LEN / NLEN as the one found at `c`:
  // bits e .. e + 2 are 000 and both reach the same byte boundary.
  auto bit_at = [&](size_t s, unsigned long long b) {
    return b < st[s].end_bits ? (in[s].h_in[b >> 3] >> (b & 7)) & 1u : 1u;
  };
  auto stored_alike = [&](size_t s, unsigned long long e, unsigned long long c) {
    return ((e + 10) >> 3) == ((c + 10) >> 3) && bit_at(s, e) == 0 && bit_at(s, e + 1) == 0 && bit_at(s, e + 2) == 0;
  };
  for (size_t s = 0; s < ns; ++s)  // a stream that opens with a stored block: incompressible data, see below
    if (bit_at(s, 1) == 0 && bit_at(s, 2) == 0) fall(s);

  std::vector<CkFind> finds;
  std::vector<unsigned long long> cand_all;
  std::vector<CkJob> jobs_all;
  std::vector<CkRes> res_all;
  std::vector<std::pair<uint32_t, uint32_t>> redo_at;  // (stream, job) of each redone chunk
  std::vector<CkPage> pinfo(total_pages);
  std::vector<CkChain> chain;
  std::vector<uint32_t> flat, flat_chunk, chain_lo, walks, ctr(ns), bad(ns), slot_to_chain;
  for (;;) {
    // ---- per live stream: its region, nominal chunk starts (chunk 0 starts at the proven bit0), and a block start guessed
    // in every other chunk ----
    finds.clear();
    bool any = false;
    for (size_t s = 0; s < ns; ++s) {
      St &t = st[s];
      if (!t.live) continue;
      any = true;
      out[s].stats[0]++;
      const size_t il = in[s].il, b0 = (size_t)(t.bit0 >> 3);
      t.rend = std::min<size_t>(il, b0 + t.R);
      t.span = t.rend - b0;
      size_t C = g_ck.chunk ? g_ck.chunk : std::max<size_t>(CK_MIN_CHUNK, (t.span + CK_TARGET - 1) / CK_TARGET);
      size_t n = std::max<size_t>(1, (t.span + C - 1) / C);
      if (n > CK_TARGET) {
        C = (t.span + CK_TARGET - 1) / CK_TARGET;
        n = (t.span + C - 1) / C;
      }
      t.n = n;
      t.S.assign(n + 1, 0);
      t.S[0] = t.bit0;
      for (size_t k = 1; k < n; ++k) t.S[k] = 8ull * (b0 + k * C);
      t.S[n] = t.rend == il ? ~0ull : 8ull * t.rend;
      t.cand.assign(n, CK_NOCAND);
      t.cand[0] = t.bit0;
      t.find0 = finds.size();
      for (size_t k = 1; k < n; ++k) finds.push_back(CkFind{t.S[k], std::min(t.S[k + 1], t.end_bits), (uint32_t)s, 0});
    }
    if (!any) break;
    if (!finds.empty()) {
      cand_all.resize(finds.size());
      CU(cudaMemcpyAsync(d_finds, finds.data(), finds.size() * sizeof(CkFind), cudaMemcpyHostToDevice, g.stream));
      tm.start();
      CU(ck_launch_find(d_in, d_streams, d_finds, d_cand, (uint32_t)finds.size(), g.stream));
      tm.stop(&ms[0]);
      CU(cudaMemcpyAsync(cand_all.data(), d_cand, finds.size() * 8, cudaMemcpyDeviceToHost, g.stream));
      CU(cudaStreamSynchronize(g.stream));
      for (size_t s = 0; s < ns; ++s)
        if (st[s].live) std::copy(cand_all.begin() + st[s].find0, cand_all.begin() + st[s].find0 + st[s].n - 1, st[s].cand.begin() + 1);
    }
    // ---- a chunk without a candidate is merged into its predecessor: jobs[i] covers up to the next kept start ----
    jobs_all.clear();
    for (size_t s = 0; s < ns; ++s) {
      St &t = st[s];
      if (!t.live) continue;
      const size_t n = t.n;
      t.jobs.clear();
      for (size_t k = 0; k < n; ++k)
        if (t.cand[k] != CK_NOCAND) t.jobs.push_back(CkJob{t.cand[k], 0, (uint32_t)t.jobs.size(), 0, (uint16_t)s});
      const size_t nj = t.jobs.size();
      for (size_t k = 0, i = 0; k < n; ++k) {
        if (t.cand[k] == CK_NOCAND) continue;
        size_t k2 = k + 1;
        while (k2 < n && t.cand[k2] == CK_NOCAND) ++k2;
        t.jobs[i++].stop_bit = t.S[k2];
      }
      out[s].stats[1] += nj;
      out[s].stats[3] += n - nj;
      // No block start found in a whole MiB (fixed-Huffman streams look like noise to the finder; stored blocks hold at
      // most 64 KiB and zlib's dynamic ones far less): one lane would walk all of it, slower than the exact path's warp.
      if (nj == 1 && t.span >= (1u << 20)) {
        fall(s);
        continue;
      }
      // Mostly stored blocks (incompressible data): the exact path moves a stored block as one run of bytes, where a chunk
      // lane copies it symbol by symbol; measured slower here (DESIGN.md "K12"), so such a stream stays on the exact path.
      size_t n_stored = 0;
      for (const CkJob &jb : t.jobs) {
        const size_t at = (size_t)((jb.start_bit + 10) >> 3);  // LEN of a stored block starting there
        n_stored += bit_at(s, jb.start_bit + 1) == 0 && bit_at(s, jb.start_bit + 2) == 0 && at + 2 <= in[s].il &&
                    (in[s].h_in[at] | (in[s].h_in[at + 1] << 8)) >= 1024;  // (flush markers are empty stored blocks)
      }
      if (nj >= 8 && 2 * n_stored > nj) {
        fall(s);
        continue;
      }
      t.job0 = jobs_all.size();
      jobs_all.insert(jobs_all.end(), t.jobs.begin(), t.jobs.end());
    }
    if (jobs_all.empty()) continue;
    CU(cudaMemsetAsync(d_ctr, 0, ns * 4, g.stream));
    CU(cudaMemcpyAsync(d_jobs, jobs_all.data(), jobs_all.size() * sizeof(CkJob), cudaMemcpyHostToDevice, g.stream));
    tm.start();
    CU(ck_launch_chunks(d_in, d_streams, d_jobs, (uint32_t)jobs_all.size(), d_res, d_pool, d_pinfo, d_ctr, g.stream));
    tm.stop(&ms[1]);
    res_all.resize(jobs_all.size());
    CU(cudaMemcpyAsync(res_all.data(), d_res, res_all.size() * sizeof(CkRes), cudaMemcpyDeviceToHost, g.stream));
    CU(cudaStreamSynchronize(g.stream));
    for (size_t s = 0; s < ns; ++s)
      if (st[s].live) {
        st[s].res.assign(res_all.begin() + st[s].job0, res_all.begin() + st[s].job0 + st[s].jobs.size());
        st[s].proving = true;
      }
    // ---- prove every chain from its bit0; redo what started at a wrong guess (all streams' redos in one launch) ----
    for (int round = 0;; ++round) {
      jobs_all.clear();
      redo_at.clear();
      for (size_t s = 0; s < ns; ++s) {
        St &t = st[s];
        if (!t.live || !t.proving) continue;
        const size_t nj = t.jobs.size();
        std::vector<CkJob> &jobs = t.jobs;
        std::vector<CkRes> &res = t.res;
        t.pos_b = t.bit0;
        t.on_chain.clear();
        t.final_seen = false;
        size_t bad_at = nj;
        bool failed = false;
        for (size_t i = 0; i < nj; ++i) {
          if (i > 0 && t.pos_b >= jobs[i].stop_bit) continue;  // its whole slice lies inside its predecessor's last block
          if (jobs[i].start_bit != t.pos_b && res[i].first_stored && stored_alike(s, t.pos_b, jobs[i].start_bit))
            jobs[i].start_bit = t.pos_b;  // the same stored block read from its true header: the same result
          if (jobs[i].start_bit != t.pos_b) {
            bad_at = i;
            break;
          }
          const int cs = res[i].status;
          if (cs != CK_BOUNDARY && cs != CK_FINAL) {  // the exact step fails here too (or the stream's pages ran out)
            failed = true;
            break;
          }
          t.on_chain.push_back((uint32_t)i);
          t.pos_b = res[i].end_bit;
          if (cs == CK_FINAL) {
            t.final_seen = true;
            break;
          }
        }
        if (failed || (bad_at != nj && round >= CK_MAX_ROUNDS)) {
          fall(s);
          continue;
        }
        if (bad_at == nj) {
          t.proving = false;
          continue;
        }
        // Redo the first unproven chunk from the proven end and, together with it, every later chunk that does not start
        // where its predecessor's last attempt ended (from that end: usually right, and proven or redone next round).
        unsigned long long prev_end = t.pos_b;
        for (size_t i = bad_at; i < nj; ++i) {
          if (prev_end >= jobs[i].stop_bit) continue;  // empty: the end carries over
          const bool mism = jobs[i].start_bit != prev_end && !(res[i].first_stored && stored_alike(s, prev_end, jobs[i].start_bit));
          if (mism) {
            jobs[i].start_bit = prev_end;
            jobs[i].gen++;
            jobs_all.push_back(jobs[i]);
            redo_at.emplace_back((uint32_t)s, (uint32_t)i);
          }
          if (res[i].status != CK_BOUNDARY) break;
          prev_end = res[i].end_bit;
        }
        out[s].stats[2]++;
      }
      if (jobs_all.empty()) break;
      CU(cudaMemcpyAsync(d_jobs, jobs_all.data(), jobs_all.size() * sizeof(CkJob), cudaMemcpyHostToDevice, g.stream));
      tm.start();
      CU(ck_launch_chunks(d_in, d_streams, d_jobs, (uint32_t)jobs_all.size(), d_res, d_pool, d_pinfo, d_ctr, g.stream));
      tm.stop(&ms[1]);
      res_all.resize(jobs_all.size());
      CU(cudaMemcpyAsync(res_all.data(), d_res, res_all.size() * sizeof(CkRes), cudaMemcpyDeviceToHost, g.stream));
      CU(cudaStreamSynchronize(g.stream));
      for (size_t q = 0; q < redo_at.size(); ++q) st[redo_at[q].first].res[redo_at[q].second] = res_all[q];
    }
    for (size_t s = 0; s < ns; ++s)  // the input ends without a final block: the exact step's EOS / STOP
      if (st[s].live && !st[s].final_seen && st[s].rend == in[s].il) fall(s);
    // ---- per stream: output offsets and its chain's pages in order; then windows and bytes for all of them ----
    CU(cudaMemcpyAsync(ctr.data(), d_ctr, ns * 4, cudaMemcpyDeviceToHost, g.stream));
    CU(cudaStreamSynchronize(g.stream));
    for (size_t s = 0; s < ns; ++s) {
      ctr[s] = std::min(ctr[s], in[s].n_pages);
      if (st[s].live && ctr[s])
        CU(cudaMemcpyAsync(pinfo.data() + tab[s].page0, d_pinfo + tab[s].page0, ctr[s] * sizeof(CkPage), cudaMemcpyDeviceToHost,
                           g.stream));
    }
    CU(cudaStreamSynchronize(g.stream));
    chain.clear();
    flat.clear();
    flat_chunk.clear();
    chain_lo.clear();
    walks.clear();
    for (size_t s = 0; s < ns; ++s) {
      St &t = st[s];
      if (!t.live) continue;
      const size_t nj = t.jobs.size(), chain0 = chain.size(), flat0 = flat.size();
      slot_to_chain.assign(nj, 0xffffffffu);
      size_t total = 0, nflat = flat0;
      for (uint32_t i : t.on_chain) {
        slot_to_chain[i] = (uint32_t)chain.size();
        chain.push_back(CkChain{(unsigned long long)(in[s].out_pos + t.emitted + total), t.res[i].nsym, (uint32_t)nflat, (uint32_t)s, 0});
        total += t.res[i].nsym;
        nflat += (t.res[i].nsym + CK_PAGE - 1) / CK_PAGE;
      }
      bool ok = t.emitted + total <= in[s].oc;  // else the exact path's NOSPC
      if (ok) {
        flat.resize(nflat, 0xffffffffu);
        flat_chunk.resize(nflat, 0);
        for (uint32_t p = 0; p < ctr[s]; ++p) {
          const CkPage &pi = pinfo[tab[s].page0 + p];
          if (pi.slot >= nj || slot_to_chain[pi.slot] == 0xffffffffu || pi.gen != t.jobs[pi.slot].gen) continue;
          const CkChain &c = chain[slot_to_chain[pi.slot]];
          if ((size_t)pi.seq * CK_PAGE >= c.nsym) continue;
          flat[c.page0 + pi.seq] = tab[s].page0 + p;
          flat_chunk[c.page0 + pi.seq] = slot_to_chain[pi.slot];
        }
        for (size_t f = flat0; f < nflat && ok; ++f) ok = flat[f] != 0xffffffffu;  // (cannot fail: every symbol of a clean chunk is on a page)
      }
      if (!ok) {
        chain.resize(chain0);
        flat.resize(flat0);
        flat_chunk.resize(flat0);
        fall(s);
        continue;
      }
      t.total = total;
      if (chain.size() > chain0) {
        chain_lo.push_back((uint32_t)chain0);
        walks.push_back((uint32_t)s);
      }
    }
    chain_lo.push_back((uint32_t)chain.size());
    std::fill(bad.begin(), bad.end(), 0u);
    if (!walks.empty()) {
      const size_t nflat = flat.size();
      CU(cudaMemcpyAsync(d_chain, chain.data(), chain.size() * sizeof(CkChain), cudaMemcpyHostToDevice, g.stream));
      CU(cudaMemcpyAsync(d_chain_lo, chain_lo.data(), chain_lo.size() * 4, cudaMemcpyHostToDevice, g.stream));
      CU(cudaMemcpyAsync(d_flat, flat.data(), nflat * 4, cudaMemcpyHostToDevice, g.stream));
      CU(cudaMemcpyAsync(d_flat + nflat, flat_chunk.data(), nflat * 4, cudaMemcpyHostToDevice, g.stream));
      CU(cudaMemsetAsync(d_bad, 0, ns * 4, g.stream));
      tm.start();
      CU(ck_launch_resolve(d_chain, d_chain_lo, (uint32_t)walks.size(), d_flat, d_flat + nflat, (uint32_t)nflat, d_pool, d_out,
                           d_streams, d_bad, g.stream));
      tm.stop(&ms[2]);
      CU(cudaMemcpyAsync(bad.data(), d_bad, ns * 4, cudaMemcpyDeviceToHost, g.stream));
      CU(cudaStreamSynchronize(g.stream));
    }
    for (size_t s = 0; s < ns; ++s) {
      St &t = st[s];
      if (!t.live) continue;
      if (bad[s]) {  // a back-reference before the allowed history: the exact path's RANGE
        fall(s);
        continue;
      }
      t.emitted += t.total;
      if (t.final_seen) {
        out[s].r.out_len = (uint32_t)t.emitted;
        out[s].r.in_used = (uint32_t)((t.pos_b + 7) >> 3);
        out[s].r.status = B200Z_U_DONE;
        out[s].accepted = true;
        t.live = false;
        continue;
      }
      t.bit0 = t.pos_b;
      t.R *= 2;
    }
  }
  return B200Z_OK;
}

// `try_chunked`: K12 may take the stream (the caller knows nothing that makes it pointless)
static int run_one_staged(const uint8_t *h_in, size_t pos, size_t in_total, size_t out_pos, size_t out_cap_total, OneResult *r,
                          bool shared_output = false, bool try_chunked = true) {
  uint64_t io = pos, oo = out_pos;
  size_t avail_in = in_total - pos;
  uint32_t il = (uint32_t)(avail_in > 0xfffffff0u ? 0xfffffff0u : avail_in);
  size_t room = out_cap_total - out_pos;
  size_t mx = max_inflate_out(il);
  if (room > mx) room = mx;
  uint32_t oc = (uint32_t)(room > 0xfffffff0u ? 0xfffffff0u : room);
  CU(g.d_out.reserve_keep(out_pos + oc + 64, out_pos, g.stream));
  const uint32_t hist = shared_output ? (uint32_t)(out_pos > 65535 ? 65535 : out_pos) : 0u;  // distances end at 32768
  for (auto &v : g_ck_stats) v = 0;
  for (auto &v : g_ck_ms) v = 0;
  if (try_chunked && il >= g_ck.thresh) {
    // the exact path's workspace for the same call: the pool is carved from it
    const size_t ws = workspace_bytes(1, out_pos + oc);
    CU(g.d_ws.reserve(ws));
    const uint32_t n_pages = ck_pages_for(ws);
    g_ck_stats[4] = g_ck_stats[5] = 1;
    if (n_pages) {
      const std::vector<CkIn> one{CkIn{h_in + pos, pos, il, out_pos, oc, hist, n_pages}};
      std::vector<CkOut> res;
      const int rc = run_chunked(one, res, g_ck_ms);
      if (rc) return rc;
      for (int k = 0; k < 5; ++k) g_ck_stats[k] = res[0].stats[k];
      if (res[0].accepted) {
        *r = res[0].r;
        return B200Z_OK;
      }
    }
  }
  return run_batch_on_staged(&io, &il, &oo, &oc, &r->out_len, &r->status, &r->in_used, 1, out_pos + oc, false, hist);
}

static inline uint32_t le32(const uint8_t *p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }
static inline uint32_t le16(const uint8_t *p) { return p[0] | (p[1] << 8); }

// _readHeader (_gzip_decoder_web.dart:60-138).  Returns 1 ok, 0 "not gzip" (-> zlib fallback), -1 = the
// Dart code would have thrown (readByte past the end).  *bsize = BGZF 'BC' member size hint or 0.
static int gzip_header(const uint8_t *in, size_t n, size_t pos, size_t *hdr_end, size_t *bsize) {
  *bsize = 0;
  if (pos + 2 > n) return -1;
  if (le16(in + pos) != 0x8b1f) return 0;
  if (pos + 3 > n) return -1;
  if (in[pos + 2] != 8) return 0;
  if (pos + 10 > n) return -1;
  uint8_t flags = in[pos + 3];
  size_t p = pos + 10;
  if (flags & 0x04) {
    if (p + 2 > n) return -1;
    size_t xlen = le16(in + p);
    p += 2;
    size_t xend = p + xlen;
    if (xend > n) xend = n;  // readBytes clamps (input_stream.dart:132-136)
    // look for the BGZF subfield  'B' 'C' SLEN=2  BSIZE(u16) = member size - 1
    size_t q = p;
    while (q + 4 <= xend) {
      size_t slen = le16(in + q + 2);
      if (in[q] == 'B' && in[q + 1] == 'C' && slen == 2 && q + 6 <= xend) *bsize = (size_t)le16(in + q + 4) + 1;
      q += 4 + slen;
    }
    p = xend;
  }
  if (flags & 0x08) {
    while (p < n && in[p] != 0) ++p;
    if (p < n) ++p;
  }
  if (flags & 0x10) {
    while (p < n && in[p] != 0) ++p;
    if (p < n) ++p;
  }
  if (flags & 0x02) {
    if (p + 2 > n) return -1;
    p += 2;
  }
  *hdr_end = p;
  return 1;
}

static int zlib_decode_staged(const uint8_t *in, size_t in_len, size_t pos, int verify, int raw, int big_endian,
                              size_t out_pos, size_t out_cap, size_t *out_len_total);

// An ISIZE that DEFLATE cannot reach from `comp` bytes (1032:1 at most: a 258-byte match costs two bits) is no size hint:
// such a member is decoded the hint-free way instead of being believed (it would size buffers).
static inline bool isize_possible(uint32_t isize, size_t comp) { return (uint64_t)isize <= (uint64_t)comp * 1040u + 1024u; }

// THE definition of a hinted run: whole members from `pos` on that carry the BGZF 'BC' size and a believable ISIZE.
// Returns the position behind the run; appends the members to `ms` when given; *out_bytes = what their ISIZE fields promise.
// (struct HintedMember: b200z_internal.h)
static size_t hinted_run(const uint8_t *in, size_t n, size_t pos, std::vector<HintedMember> *ms, size_t *out_bytes) {
  size_t p = pos, o = 0;
  while (p < n) {
    size_t hdr_end, bsize;
    if (gzip_header(in, n, p, &hdr_end, &bsize) != 1 || bsize == 0) break;
    const size_t next = p + bsize;
    if (next > n || next < hdr_end + 8) break;
    const uint32_t isize = le32(in + next - 4);
    if (!isize_possible(isize, next - hdr_end)) break;
    if (ms) ms->push_back({hdr_end, next, isize});
    o += isize;
    p = next;
  }
  if (out_bytes) *out_bytes = o;
  return p;
}

// Is there a gzip member header (1f 8b 08, no reserved flag bits, a known XFL and OS byte) in in[from, from + span)?  Only
// a hint of where the member that starts before `from` ends: chance hits in compressed data are about 2^-38 per byte.
static bool gzip_member_header_within(const uint8_t *in, size_t n, size_t from, size_t span) {
  const size_t end = std::min(n, from + span);
  for (size_t p = from; p + 10 <= end;) {
    const void *q = memchr(in + p, 0x1f, end - 9 - p);
    if (!q) return false;
    p = (size_t)((const uint8_t *)q - in);
    const uint8_t *h = in + p;
    if (h[1] == 0x8b && h[2] == 8 && (h[3] & 0xe0) == 0 && (h[8] == 0 || h[8] == 2 || h[8] == 4) && (h[9] <= 13 || h[9] == 255))
      return true;
    ++p;
  }
  return false;
}

// ---------------------------------------------------------------------------------------------
// The rules that turn one unit's result into the next step of a gzip member loop or a zlib stream loop.  The single calls
// (gzip_decode_staged, gzip_fast_path, zlib_decode_staged) and the batch driver (gzip_zlib_decode_streams) apply these.
// ---------------------------------------------------------------------------------------------
// The members of a hinted run whose hints were exact, from the front: the prefix that is accepted.
static size_t hinted_exact_prefix(const std::vector<HintedMember> &ms, const uint32_t *len, const int32_t *st, const uint32_t *used) {
  size_t k = 0;
  while (k < ms.size() && st[k] == B200Z_U_DONE && len[k] == ms[k].isize && ms[k].hdr_end + used[k] + 8 == ms[k].next) ++k;
  return k;
}

// A hinted run whose ISIZE fields bring the output to `o` bytes: B200Z_OK, or B200Z_E_NOSPC when out_cap is short of it.
static int gzip_hinted_room_rule(size_t o, size_t out_cap) {
  if (o <= out_cap) return B200Z_OK;
  set_err("gzip_decode: output needs at least %zu bytes, out_cap %zu", o, out_cap);
  return B200Z_E_NOSPC;
}

// The header of a member at `pos` that is decoded without a hint: 1 with *hdr_end = its DEFLATE stream, 0 when there is
// no gzip header (the zlib loop goes on from `pos` on the same little-endian stream, :31-37), or B200Z_E_THROW.
static int gzip_member_header_rule(const uint8_t *in, size_t in_len, size_t pos, size_t *hdr_end) {
  size_t bsize;
  const int h = gzip_header(in, in_len, pos, hdr_end, &bsize);
  if (h >= 0) return h;
  set_err("gzip_decode: truncated header (Dart: RangeError)");
  return B200Z_E_THROW;
}

// The member at `pos` without a (valid) hint, its DEFLATE stream from hdr_end, came back as r: B200Z_OK with *next = where
// the next member starts, or the call's result code.
static int gzip_member_rule(const OneResult &r, size_t pos, size_t hdr_end, size_t in_len, size_t out_cap, size_t *next) {
  if (r.status == B200Z_U_NOSPC) {
    set_err("gzip_decode: out_cap %zu too small", out_cap);
    return B200Z_E_NOSPC;
  }
  if (r.status == B200Z_U_RANGE || r.status == B200Z_U_THROW) {
    set_err("gzip_decode: member at %zu: Dart would throw RangeError (status %d)", pos, r.status);
    return B200Z_E_THROW;
  }
  const size_t after = hdr_end + r.in_used;
  if (r.status == B200Z_U_STOP && after + 8 > in_len) {
    // Inflate gave up because the input ran out inside a block (inflate.dart:166-168, 192-195): the byte-wise bit reader
    // has pulled every byte by then, so the two readUint32 of the trailer (:40-41) start past the end -- RangeError.
    // This is what a truncated file does.
    set_err("gzip_decode: member at %zu: input ends inside the stream (Dart: RangeError)", pos);
    return B200Z_E_THROW;
  }
  if (r.status != B200Z_U_DONE && r.status != B200Z_U_EOS) {
    set_err("gzip_decode: member at %zu stopped with status %d", pos, r.status);
    return B200Z_E_DATA;  // DESIGN.md "Divergences": reference keeps parsing from an unspecified position
  }
  if (after + 8 > in_len) {  // readUint32 x2 past the end (:40-41)
    set_err("gzip_decode: truncated trailer (Dart: RangeError)");
    return B200Z_E_THROW;
  }
  *next = after + 8;
  return B200Z_OK;
}

// The zlib stream header at *pos (_zlib_decoder_web.dart:50-80): B200Z_OK with *pos behind it, or the call's result code.
static int zlib_header_rule(const uint8_t *in, size_t in_len, size_t *pos) {
  size_t p = *pos;
  if (p + 2 > in_len) {
    set_err("zlib_decode: truncated header (Dart: RangeError)");
    return B200Z_E_THROW;
  }
  uint32_t cmf = in[p], flg = in[p + 1];
  p += 2;
  if ((cmf & 8) != 8) {  // :57 (sic)
    set_err("zlib_decode: method != deflate");
    return B200Z_E_DATA;
  }
  if (((cmf * 256) + flg) % 31 != 0) {
    set_err("zlib_decode: bad FCHECK");
    return B200Z_E_DATA;
  }
  if ((flg & 32) != 0) {
    if (p + 4 > in_len) {
      set_err("zlib_decode: truncated DICTID (Dart: RangeError)");
      return B200Z_E_THROW;
    }
    set_err("zlib_decode: FDICT not supported");
    return B200Z_E_DATA;
  }
  *pos = p;
  return B200Z_OK;
}

// The zlib stream decoded from *pos came back as r, behind `committed` bytes of output: B200Z_OK with *pos behind the
// stream and its Adler-32 field in *stored (not raw), or the call's result code with *out_len_total where it ends.
static int zlib_stream_rule(const OneResult &r, const uint8_t *in, size_t in_len, int raw, int big_endian, size_t committed,
                            size_t out_cap, size_t *pos, uint32_t *stored, size_t *out_len_total) {
  if (r.status == B200Z_U_NOSPC) {
    *out_len_total = committed + r.out_len;
    set_err("zlib_decode: out_cap %zu too small", out_cap);
    return B200Z_E_NOSPC;
  }
  if (r.status == B200Z_U_RANGE || r.status == B200Z_U_THROW) {
    set_err("zlib_decode: Dart would throw RangeError (status %d)", r.status);
    return B200Z_E_THROW;
  }
  if (r.status == B200Z_U_BADCODE) {
    *out_len_total = committed + r.out_len;
    set_err("zlib_decode: unusable Huffman code set");
    return B200Z_E_DATA;
  }
  size_t p = *pos + r.in_used;
  if (r.status == B200Z_U_STOP && p < in_len) {
    // Inflate gave up with input left: the reference's stream position is then wherever its byte-wise bit buffer had
    // got to (not rewound) -- unspecified; stop here with the partial output (DESIGN.md "Divergences").
    *out_len_total = committed + r.out_len;
    set_err("zlib_decode: inflate stopped early");
    return B200Z_E_DATA;
  }
  // (B200Z_U_STOP with the input used up == the stream ends inside a block: Inflate simply returns what it has, :85)
  if (!raw) {
    if (p + 4 > in_len) {  // readUint32 past the end (:88); the stream's bytes were not handed over yet
      set_err("zlib_decode: truncated Adler-32 (Dart: RangeError)");
      return B200Z_E_THROW;
    }
    *stored = big_endian ? ((uint32_t)in[p] << 24 | in[p + 1] << 16 | in[p + 2] << 8 | in[p + 3]) : le32(in + p);
    p += 4;
  }
  *pos = p;
  return B200Z_OK;
}

static int zlib_adler_rule(uint32_t computed, uint32_t stored) {
  if (computed == stored) return B200Z_OK;
  set_err("zlib_decode: Adler-32 mismatch");
  return B200Z_E_DATA;  // this stream's bytes are dropped (:91-94)
}

// GZip member loop on staged input.
static int gzip_decode_staged(const uint8_t *in, size_t in_len, int verify, size_t out_cap, size_t *out_len_total,
                              size_t pos = 0, size_t out_pos = 0) {
  std::vector<uint64_t> v_in_off, v_out_off;
  std::vector<uint32_t> v_in_len, v_out_cap, v_out_len, v_in_used;
  std::vector<int32_t> v_status;
  std::vector<size_t> v_next;
  while (pos < in_len) {
    // -------- gather a run of members that carry a size hint (BGZF 'BC' + ISIZE) --------
    v_in_off.clear(); v_out_off.clear(); v_in_len.clear(); v_out_cap.clear(); v_next.clear();
    size_t o = out_pos;
    std::vector<HintedMember> run;
    hinted_run(in, in_len, pos, &run, nullptr);
    for (const HintedMember &m : run) {
      v_in_off.push_back(m.hdr_end);
      v_in_len.push_back((uint32_t)(m.next - m.hdr_end));
      v_out_off.push_back(o);
      v_out_cap.push_back(m.isize);
      v_next.push_back(m.next);
      o += m.isize;
    }
    size_t nb = v_in_off.size();
    if (nb > 0) {
      if (gzip_hinted_room_rule(o, out_cap)) {
        *out_len_total = o;  // best knowledge of what is needed so far
        return B200Z_E_NOSPC;
      }
      CU(g.d_out.reserve_keep(o + 64, out_pos, g.stream));
      v_out_len.resize(nb); v_status.resize(nb); v_in_used.resize(nb);
      int rc = run_batch_on_staged(v_in_off.data(), v_in_len.data(), v_out_off.data(), v_out_cap.data(),
                                   v_out_len.data(), v_status.data(), v_in_used.data(), nb, o);
      if (rc) return rc;
      // accept the prefix whose hints were exact; anything else is redone the slow, hint-free way
      const size_t k = hinted_exact_prefix(run, v_out_len.data(), v_status.data(), v_in_used.data());
      if (k > 0) {
        pos = v_next[k - 1];
        out_pos = v_out_off[k - 1] + v_out_len[k - 1];
      }
      if (k == nb) continue;
    }
    if (pos >= in_len) break;
    // -------- one member without (valid) hints: decode it alone to learn where it ends --------
    size_t hdr_end;
    const int h = gzip_member_header_rule(in, in_len, pos, &hdr_end);
    if (h < 0) {
      *out_len_total = out_pos;
      return h;
    }
    if (h == 0)  // no gzip header: fall back to zlib on the same little-endian stream (:31-37)
      return zlib_decode_staged(in, in_len, pos, verify & B200Z_GZIP_VERIFY, (verify & B200Z_GZIP_RAW) != 0, /*big_endian=*/0, out_pos,
                                out_cap, out_len_total);  // decodeStream(input, output, verify: verify, raw: raw)
    OneResult r;
    // A member's input runs to the end of the file, so K12 would work through a whole region of g_ck.thresh bytes for a
    // small member.  A member whose successor's header shows up closer than that is small: it takes the exact path.
    int rc = run_one_staged(in, hdr_end, in_len, out_pos, out_cap, &r, /*shared_output=*/true,
                            !gzip_member_header_within(in, in_len, hdr_end, g_ck.thresh));
    if (rc) return rc;
    out_pos += r.out_len;
    *out_len_total = out_pos;
    rc = gzip_member_rule(r, pos, hdr_end, in_len, out_cap, &pos);
    if (rc) return rc;
  }
  *out_len_total = out_pos;
  return B200Z_OK;
}


// ---------------------------------------------------------------------------------------------
// End-to-end fast path for the common shape: a run of members that all carry size hints.  The run is cut
// into chunks; chunk c's host->device copy, its two kernels and chunk c-1's device->host copy run on
// three streams, so the PCIe transfers hide behind each other and behind the decode.  Every hint is
// verified afterwards; the first member whose hint was not exact ends the accepted prefix and the
// caller continues from there on the slow, hint-free path (same bytes out either way).
// ---------------------------------------------------------------------------------------------
static int gzip_fast_path_piped_fwd(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, size_t *pos_io, size_t *out_pos_io,
                                    size_t *needed);
static int gzip_fast_path(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, size_t *pos_io,
                          size_t *out_pos_io, size_t *needed) {
  // B200Z_GZIP_PIPED_WALK=1: the walk inside the pipeline (below).  Off by default: it was measured slower than
  // walk-first (config 2, pinned buffers) -- see the comment on gzip_fast_path_piped.
  {
    const char *pe = getenv("B200Z_GZIP_PIPED_WALK");
    const bool piped = pe && atoi(pe) != 0;
    const size_t span = in_len - *pos_io, room = out_cap >= *out_pos_io ? out_cap - *out_pos_io : 0;
    if (piped && *pos_io < in_len && room <= 32 * span + (64u << 20)) return gzip_fast_path_piped_fwd(in, in_len, out, out_cap, pos_io, out_pos_io, needed);
  }
  std::vector<HintedMember> ms;
  size_t promised = 0;
  const size_t p = hinted_run(in, in_len, *pos_io, &ms, &promised);
  const size_t o = *out_pos_io + promised;
  const size_t nb = ms.size();
  if (nb == 0) return B200Z_OK;
  if (gzip_hinted_room_rule(o, out_cap)) {
    *needed = o;
    return B200Z_E_NOSPC;
  }
  const size_t in_lo = *pos_io, in_hi = p, out_lo = *out_pos_io;
  // chunks: ~8 per call (one compute stream each, so their kernels overlap: a stream's decode time is set by
  // its token count, not by how many streams run beside it), at least 4 MiB of compressed bytes each
  size_t min_chunk = 4u << 20;  // (B200Z_GZIP_CHUNK_KB: smaller chunks for tests of the pipeline itself)
  if (const char *e = getenv("B200Z_GZIP_CHUNK_KB")) min_chunk = std::max<size_t>(1, (size_t)atoll(e)) << 10;
  size_t target = (in_hi - in_lo) / Ctx::kCompStreams;
  if (target < min_chunk) target = min_chunk;
  // The device->host copy of the output bounds this path (it moves ~2.5x the bytes of the input copy over the same link),
  // and it cannot start before the first chunk has been copied in and decoded: the first two chunks are a quarter and a
  // half of a regular one, so that it starts early and is fed without a gap from then on.  (B200Z_GZIP_RAMP=0: equal chunks.)
  const char *ramp_env = getenv("B200Z_GZIP_RAMP");
  const bool ramp = !ramp_env || atoi(ramp_env) != 0;
  std::vector<size_t> cut{0};
  {
    size_t acc_start = in_lo;
    for (size_t i = 0; i < nb; ++i) {
      size_t want = target;
      if (ramp && cut.size() <= 2) want = std::max<size_t>(target >> (3 - cut.size()), min_chunk);  // chunk 0: /4, chunk 1: /2
      if (ms[i].next - acc_start >= want && i + 1 < nb) {
        cut.push_back(i + 1);
        acc_start = ms[i].next;
      }
    }
    cut.push_back(nb);
  }
  const size_t nchunks = cut.size() - 1;
  MetaLayout ml(nb);
  CU(g.h_meta.reserve(ml.bytes));
  CU(g.d_meta.reserve(ml.bytes));
  CU(g.d_in.reserve(in_len + 64));
  CU(g.d_out.reserve_keep(o + 64, out_lo, g.stream));
  uint8_t *hm = (uint8_t *)g.h_meta.p, *dm = (uint8_t *)g.d_meta.p;
  uint64_t *h_in_off = (uint64_t *)(hm + ml.off_in_off), *h_out_off = (uint64_t *)(hm + ml.off_out_off);
  uint32_t *h_in_len = (uint32_t *)(hm + ml.off_in_len), *h_out_cap = (uint32_t *)(hm + ml.off_out_cap);
  size_t max_chunk_out = 0;
  std::vector<size_t> chunk_out_lo(nchunks + 1);
  {
    size_t oo = out_lo;
    for (size_t c = 0; c < nchunks; ++c) {
      chunk_out_lo[c] = oo;
      size_t rel = 0;
      for (size_t i = cut[c]; i < cut[c + 1]; ++i) {
        h_in_off[i] = ms[i].hdr_end;
        h_in_len[i] = (uint32_t)(ms[i].next - ms[i].hdr_end);
        h_out_off[i] = rel;  // relative to the chunk's slice of d_out
        h_out_cap[i] = ms[i].isize;
        rel += ms[i].isize;
      }
      oo += rel;
      if (rel > max_chunk_out) max_chunk_out = rel;
    }
    chunk_out_lo[nchunks] = oo;
  }
  size_t max_units = 0;
  for (size_t c = 0; c < nchunks; ++c) max_units = cut[c + 1] - cut[c] > max_units ? cut[c + 1] - cut[c] : max_units;
  (void)max_units;
  (void)max_chunk_out;
  CU(g.d_ws.reserve(inflate_ws_bytes(nb, o - out_lo)));  // token layout mirrors the output layout
  const InflateWs ws_all = inflate_ws_carve(g.d_ws.p, nb, o - out_lo);
  std::vector<cudaEvent_t> ev_in(nchunks), ev_k(nchunks);
  for (size_t c = 0; c < nchunks; ++c) {
    CU(cudaEventCreateWithFlags(&ev_in[c], cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&ev_k[c], cudaEventDisableTiming));
  }
  CU(cudaMemcpyAsync(dm, hm, ml.inputs_bytes(), cudaMemcpyHostToDevice, g.s_h2d));
  int rc = B200Z_OK;
  for (size_t c = 0; c < nchunks && rc == B200Z_OK; ++c) {
    const size_t a = cut[c], b = cut[c + 1];
    const size_t lo = c == 0 ? in_lo : ms[a - 1].next, hi = ms[b - 1].next;
    CU(cudaMemcpyAsync((uint8_t *)g.d_in.p + lo, in + lo, hi - lo, cudaMemcpyHostToDevice, g.s_h2d));
    CU(cudaEventRecord(ev_in[c], g.s_h2d));
    cudaStream_t cs = g.s_comp[c % Ctx::kCompStreams];
    CU(cudaStreamWaitEvent(cs, ev_in[c], 0));
    InflateBatch bt;
    bt.in_base = (const uint8_t *)g.d_in.p;
    bt.in_off = (const uint64_t *)(dm + ml.off_in_off) + a;
    bt.in_len = (const uint32_t *)(dm + ml.off_in_len) + a;
    bt.out_base = (uint8_t *)g.d_out.p + chunk_out_lo[c];
    bt.out_off = (const uint64_t *)(dm + ml.off_out_off) + a;
    bt.out_cap = (const uint32_t *)(dm + ml.off_out_cap) + a;
    bt.out_len = (uint32_t *)(dm + ml.off_out_len) + a;
    bt.status = (int32_t *)(dm + ml.off_status) + a;
    bt.in_used = (uint32_t *)(dm + ml.off_in_used) + a;
    bt.n_units = b - a;
    bt.share = (int)(nchunks < (size_t)Ctx::kCompStreams ? nchunks : (size_t)Ctx::kCompStreams);
    bt.ws = inflate_ws_slice(ws_all, a, chunk_out_lo[c] - out_lo);
    CU(launch_inflate(bt, cs));
    CU(cudaEventRecord(ev_k[c], cs));
    CU(cudaStreamWaitEvent(g.s_d2h, ev_k[c], 0));
    const size_t ob = chunk_out_lo[c + 1] - chunk_out_lo[c];
    if (ob) CU(cudaMemcpyAsync(out + chunk_out_lo[c], (uint8_t *)g.d_out.p + chunk_out_lo[c], ob, cudaMemcpyDeviceToHost, g.s_d2h));
  }
  CU(cudaMemcpyAsync(hm + ml.off_out_len, dm + ml.off_out_len, ml.off_hist - ml.off_out_len, cudaMemcpyDeviceToHost, g.s_d2h));
  CU(cudaStreamSynchronize(g.s_d2h));
  for (size_t c = 0; c < nchunks; ++c) {
    cudaEventDestroy(ev_in[c]);
    cudaEventDestroy(ev_k[c]);
  }
  const uint32_t *r_len = (const uint32_t *)(hm + ml.off_out_len), *r_used = (const uint32_t *)(hm + ml.off_in_used);
  const int32_t *r_st = (const int32_t *)(hm + ml.off_status);
  const size_t k = hinted_exact_prefix(ms, r_len, r_st, r_used);
  if (k > 0) {
    *pos_io = ms[k - 1].next;
    size_t oo = out_lo;
    for (size_t i = 0; i < k; ++i) oo += ms[i].isize;
    *out_pos_io = oo;
  }
  return B200Z_OK;
}

// ---------------------------------------------------------------------------------------------
// The same path with the HOST walk inside the pipeline.  Finding the members is a pointer chase through the compressed
// bytes (a member's size is in its own header), a sizeable share of the whole call when it runs before anything else
// starts.  Here every chunk is sent and launched as soon as the walk
// has covered its members, and the walk of the next chunk runs while the device works on this one.  Buffers are sized
// from what the caller offers (out_cap) instead of from the walk's totals, so this form is taken when that is a sane
// bound; anything unexpected (a hint that overflows out_cap, more members than the tables were sized for) ends the run
// early and the caller goes on from the returned position exactly as before.
// Measured (config 2) slower than the walk in front -- in both forms tried (whole input sent ahead in 16 MiB pieces;
// one copy per chunk as here).  The walk is a chain of dependent cache misses into the caller's buffer, and it now runs
// while the copy engines move data through the same host memory; the chunks reach the device later than the device
// could take them.  Kept as an option (B200Z_GZIP_PIPED_WALK=1) with its
// tests; the default is walk-first.
// ---------------------------------------------------------------------------------------------
static int gzip_fast_path_piped(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, size_t *pos_io, size_t *out_pos_io,
                                size_t *needed) {
  const size_t in_lo = *pos_io, out_lo = *out_pos_io;
  size_t hdr0, bsize0;
  if (in_lo >= in_len || gzip_header(in, in_len, in_lo, &hdr0, &bsize0) != 1 || bsize0 == 0) return B200Z_OK;
  const size_t room = out_cap - out_lo;
  const size_t span = in_len - in_lo;
  // members expected: from the first one's size, with slack; the tables are sized once
  size_t nb_cap = span / bsize0;
  nb_cap = nb_cap + nb_cap / 4 + 4096;
  size_t min_chunk = 4u << 20;
  if (const char *e = getenv("B200Z_GZIP_CHUNK_KB")) min_chunk = std::max<size_t>(1, (size_t)atoll(e)) << 10;
  size_t target = span / Ctx::kCompStreams;
  if (target < min_chunk) target = min_chunk;
  const char *ramp_env = getenv("B200Z_GZIP_RAMP");
  const bool ramp = !ramp_env || atoi(ramp_env) != 0;

  MetaLayout ml(nb_cap);
  CU(g.h_meta.reserve(ml.bytes));
  CU(g.d_meta.reserve(ml.bytes));
  CU(g.d_in.reserve(in_len + 64));
  CU(g.d_out.reserve_keep(out_lo + room + 64, out_lo, g.stream));
  CU(g.d_ws.reserve(inflate_ws_bytes(nb_cap, room)));
  const InflateWs ws_all = inflate_ws_carve(g.d_ws.p, nb_cap, room);
  uint8_t *hm = (uint8_t *)g.h_meta.p, *dm = (uint8_t *)g.d_meta.p;
  uint64_t *h_in_off = (uint64_t *)(hm + ml.off_in_off), *h_out_off = (uint64_t *)(hm + ml.off_out_off);
  uint32_t *h_in_len = (uint32_t *)(hm + ml.off_in_len), *h_out_cap = (uint32_t *)(hm + ml.off_out_cap);

  std::vector<cudaEvent_t> ev_k, ev_piece;
  std::vector<HintedMember> ms;
  ms.reserve(nb_cap);
  size_t p = in_lo, o = out_lo;          // walk position, output position
  size_t chunk_a = 0, chunk_in_lo = in_lo, chunk_out_lo = out_lo, n_chunks = 0;
  bool nospc = false;
  auto launch_chunk = [&](size_t a, size_t b) -> int {  // members [a, b): bytes [chunk_in_lo, ms[b-1].next) -> [chunk_out_lo, o)
    const size_t hi = ms[b - 1].next;
    cudaStream_t cs = g.s_comp[n_chunks % Ctx::kCompStreams];
    // the chunk's bytes, then (on the chunk's stream, behind them on the copy engine) its slices of the four input arrays.
    // (Sending the whole input ahead in one go was tried: the small copies below then queue behind ALL of it on the
    // host-to-device engine and the first decode starts late.)
    cudaEvent_t ei;
    CU(cudaEventCreateWithFlags(&ei, cudaEventDisableTiming));
    ev_piece.push_back(ei);
    CU(cudaMemcpyAsync((uint8_t *)g.d_in.p + chunk_in_lo, in + chunk_in_lo, hi - chunk_in_lo, cudaMemcpyHostToDevice, g.s_h2d));
    CU(cudaEventRecord(ei, g.s_h2d));
    CU(cudaStreamWaitEvent(cs, ei, 0));
    CU(cudaMemcpyAsync(dm + ml.off_in_off + 8 * a, hm + ml.off_in_off + 8 * a, 8 * (b - a), cudaMemcpyHostToDevice, cs));
    CU(cudaMemcpyAsync(dm + ml.off_out_off + 8 * a, hm + ml.off_out_off + 8 * a, 8 * (b - a), cudaMemcpyHostToDevice, cs));
    CU(cudaMemcpyAsync(dm + ml.off_in_len + 4 * a, hm + ml.off_in_len + 4 * a, 4 * (b - a), cudaMemcpyHostToDevice, cs));
    CU(cudaMemcpyAsync(dm + ml.off_out_cap + 4 * a, hm + ml.off_out_cap + 4 * a, 4 * (b - a), cudaMemcpyHostToDevice, cs));
    InflateBatch bt;
    bt.in_base = (const uint8_t *)g.d_in.p;
    bt.in_off = (const uint64_t *)(dm + ml.off_in_off) + a;
    bt.in_len = (const uint32_t *)(dm + ml.off_in_len) + a;
    bt.out_base = (uint8_t *)g.d_out.p + chunk_out_lo;
    bt.out_off = (const uint64_t *)(dm + ml.off_out_off) + a;
    bt.out_cap = (const uint32_t *)(dm + ml.off_out_cap) + a;
    bt.out_len = (uint32_t *)(dm + ml.off_out_len) + a;
    bt.status = (int32_t *)(dm + ml.off_status) + a;
    bt.in_used = (uint32_t *)(dm + ml.off_in_used) + a;
    bt.n_units = b - a;
    bt.share = Ctx::kCompStreams;
    bt.ws = inflate_ws_slice(ws_all, a, chunk_out_lo - out_lo);
    CU(launch_inflate(bt, cs));
    cudaEvent_t ek;
    CU(cudaEventCreateWithFlags(&ek, cudaEventDisableTiming));
    ev_k.push_back(ek);
    CU(cudaEventRecord(ek, cs));
    CU(cudaStreamWaitEvent(g.s_d2h, ek, 0));
    const size_t ob = o - chunk_out_lo;
    if (ob) CU(cudaMemcpyAsync(out + chunk_out_lo, (uint8_t *)g.d_out.p + chunk_out_lo, ob, cudaMemcpyDeviceToHost, g.s_d2h));
    n_chunks++;
    chunk_a = b;
    chunk_in_lo = hi;
    chunk_out_lo = o;
    return B200Z_OK;
  };
  int rc = B200Z_OK;
  size_t promised = out_lo;  // what the hints ask for, also beyond out_cap (reported with B200Z_E_NOSPC)
  while (p < in_len && ms.size() < nb_cap) {
    size_t hdr_end, bsize;
    if (gzip_header(in, in_len, p, &hdr_end, &bsize) != 1 || bsize == 0) break;
    const size_t next = p + bsize;
    if (next > in_len || next < hdr_end + 8) break;
    const uint32_t isize = le32(in + next - 4);
    if (!isize_possible(isize, next - hdr_end)) break;
    promised += isize;
    if (promised > out_cap) nospc = true;
    if (!nospc) {
      const size_t i = ms.size();
      ms.push_back({hdr_end, next, isize});
      h_in_off[i] = hdr_end;
      h_in_len[i] = (uint32_t)(next - hdr_end);
      h_out_off[i] = o - chunk_out_lo;  // relative to the chunk's slice of d_out
      h_out_cap[i] = isize;
      o += isize;
      size_t want = target;
      if (ramp && n_chunks < 2) want = std::max<size_t>(target >> (2 - n_chunks), min_chunk);  // chunk 0: /4, chunk 1: /2
      if (next - chunk_in_lo >= want) {
        rc = launch_chunk(chunk_a, ms.size());
        if (rc) break;
      }
    }
    p = next;
  }
  if (rc == B200Z_OK && !nospc && chunk_a < ms.size()) rc = launch_chunk(chunk_a, ms.size());
  const size_t nb = ms.size();
  if (rc == B200Z_OK && nb) {
    CU(cudaMemcpyAsync(hm + ml.off_out_len, dm + ml.off_out_len, 4 * nb, cudaMemcpyDeviceToHost, g.s_d2h));
    CU(cudaMemcpyAsync(hm + ml.off_status, dm + ml.off_status, 4 * nb, cudaMemcpyDeviceToHost, g.s_d2h));
    CU(cudaMemcpyAsync(hm + ml.off_in_used, dm + ml.off_in_used, 4 * nb, cudaMemcpyDeviceToHost, g.s_d2h));
  }
  CU(cudaStreamSynchronize(g.s_h2d));
  CU(cudaStreamSynchronize(g.s_d2h));
  for (cudaEvent_t e : ev_piece) cudaEventDestroy(e);
  for (cudaEvent_t e : ev_k) cudaEventDestroy(e);
  if (rc) return rc;
  if (nospc) {
    *needed = promised;
    return gzip_hinted_room_rule(promised, out_cap);
  }
  const uint32_t *r_len = (const uint32_t *)(hm + ml.off_out_len), *r_used = (const uint32_t *)(hm + ml.off_in_used);
  const int32_t *r_st = (const int32_t *)(hm + ml.off_status);
  const size_t k = hinted_exact_prefix(ms, r_len, r_st, r_used);
  size_t oo = out_lo;
  for (size_t i = 0; i < k; ++i) oo += ms[i].isize;
  if (k > 0) {
    *pos_io = ms[k - 1].next;
    *out_pos_io = oo;
  }
  return B200Z_OK;
}

static int gzip_fast_path_piped_fwd(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, size_t *pos_io, size_t *out_pos_io,
                                    size_t *needed) {
  return gzip_fast_path_piped(in, in_len, out, out_cap, pos_io, out_pos_io, needed);
}

// ---- hooks for the file-stream layer (b200z_file.cu) ----
void set_error_text(const char *msg) { set_err("%s", msg); }

// Bytes of `in` covered by whole members that carry a size hint, from offset 0 (the run gzip_fast_path would take), and the
// output bytes their ISIZE fields promise.
size_t gzip_hinted_prefix(const uint8_t *in, size_t n, size_t *out_bytes) { return hinted_run(in, n, 0, nullptr, out_bytes); }
size_t gzip_hinted_members(const uint8_t *in, size_t n, size_t pos, std::vector<HintedMember> *ms, size_t *out_bytes) {
  return hinted_run(in, n, pos, ms, out_bytes);
}

// The hinted run at the front of `in`, decoded through the chunk pipeline: *in_used = end of the last member whose hint
// was exact (== the whole run unless a hint lied), *out_len = the bytes those members produced.
int gzip_decode_hinted(const uint8_t *in, size_t n, uint8_t *out, size_t out_cap, size_t *in_used, size_t *out_len) {
  int rc = require_init();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  size_t pos = 0, out_pos = 0, needed = 0;
  rc = gzip_fast_path(in, n, out, out_cap, &pos, &out_pos, &needed);
  *in_used = pos;
  *out_len = rc == B200Z_E_NOSPC ? needed : out_pos;
  return rc;
}

// The member loop over `in`, continuing a decodeStream call that has already produced output: its last `hist_len` bytes
// (<= 65535; distances end at 32768) are placed in front, because the members share one OutputStream and may copy from it
// (InflateWs::hist).  *out_len counts the new bytes only.
int gzip_decode_after(const uint8_t *in, size_t n, int verify, const uint8_t *hist, size_t hist_len, uint8_t *out, size_t out_cap,
                      size_t *out_len) {
  int rc = require_init();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  rc = stage_input(in, n);
  if (rc) return rc;
  CU(g.d_out.reserve(hist_len + 64));
  if (hist_len) CU(cudaMemcpyAsync(g.d_out.p, hist, hist_len, cudaMemcpyHostToDevice, g.stream));
  size_t total = hist_len;
  rc = gzip_decode_staged(in, n, verify, out_cap + hist_len, &total, 0, hist_len);
  const size_t produced = total > hist_len ? total - hist_len : 0;
  *out_len = produced;
  if (rc == B200Z_E_NOSPC || rc == B200Z_E_NODEVICE) return rc;
  const size_t hi = produced > out_cap ? out_cap : produced;
  if (hi) CU(cudaMemcpyAsync(out, (const uint8_t *)g.d_out.p + hist_len, hi, cudaMemcpyDeviceToHost, g.stream));
  CU(cudaStreamSynchronize(g.stream));
  return rc;
}

// _zlib_decoder_web.dart:31-107 on staged input.
static int zlib_decode_staged(const uint8_t *in, size_t in_len, size_t pos, int verify, int raw, int big_endian,
                              size_t out_pos, size_t out_cap, size_t *out_len_total) {
  // The reference inflates every stream into a buffer of its own and hands it to `output` only when the NEXT stream's
  // header has been accepted, or at the end of the loop (:82-84, :101-103).  A stream whose successor's header is bad, or
  // whose Adler-32 is wrong or missing, therefore never reaches the output.  Here the streams are decoded straight into
  // their final position; `committed` is what `output` holds, `pending` the bytes of the stream that waits.
  size_t committed = out_pos, pending = 0;
  *out_len_total = committed;
  while (pos < in_len) {
    if (!raw) {
      const int rc = zlib_header_rule(in, in_len, &pos);
      if (rc) return rc;
    }
    committed += pending;  // output.writeBytes(buffer) (:82-84)
    pending = 0;
    *out_len_total = committed;
    OneResult r;
    int rc = run_one_staged(in, pos, in_len, committed, out_cap, &r);
    if (rc) return rc;
    uint32_t stored = 0;
    rc = zlib_stream_rule(r, in, in_len, raw, big_endian, committed, out_cap, &pos, &stored, out_len_total);
    if (rc) return rc;
    if (!raw && verify) {
      uint32_t a;
      rc = device_adler32((const uint8_t *)g.d_out.p + committed, r.out_len, &a);
      if (rc) return rc;
      rc = zlib_adler_rule(a, stored);
      if (rc) return rc;
    }
    pending = r.out_len;
  }
  *out_len_total = committed + pending;  // (:101-103)
  return B200Z_OK;
}

// ---------------------------------------------------------------------------------------------
// Many gzip / zlib streams in one call (b200z_gzip_decode_batch / b200z_zlib_decode_batch).  Every stream keeps the state of
// its own member loop (gzip_decode_staged) or stream loop (zlib_decode_staged) and takes its steps by the same rules; what
// changes is that the steps of all streams of a device group are decoded together.  Per round each live stream offers its
// hinted run, or else its next member / zlib stream, whose input view runs to the end of its own stream; the units of all of
// them are one inflate batch, after the large ones have been offered to one K12 batch.  A batch of single-member files is
// one round; a stream of k unhinted members takes k rounds, as it takes k steps alone.  The single calls keep their own
// paths (the hinted run of a single gzip call is pipelined through gzip_fast_path).
// ---------------------------------------------------------------------------------------------
constexpr size_t GZ_STAGE = 64u << 20;        // the pinned staging buffer of the decode batch's outputs (Ctx::h_stage)
static uint32_t g_gzb_max_group = 0;          // test hook: streams per device group (0: the memory budget alone)
static unsigned long long g_gzb_stats[6];     // last call: streams, groups, rounds, units, offered to K12, accepted by K12

struct GzStream {
  const uint8_t *h = nullptr;  // the caller's bytes of the stream
  size_t len = 0, cap = 0;     // its length and out_cap
  size_t din = 0, dout = 0;    // its first byte in g.d_in / its output slot in g.d_out
  size_t slot = 0;             // the slot's bytes: min(cap, max_inflate_out(len))
  bool zlib = false, raw = false, verify = false, big_endian = false, skip_hint = false;
  bool live = true;
  int rc = B200Z_OK;
  size_t pos = 0, out_pos = 0;  // gzip: position and output so far; zlib: out_pos = committed
  size_t pending = 0, out_len = 0;
  // this round
  int kind = 0;  // 1: hinted run, 2: unhinted member, 3: zlib stream
  size_t u0 = 0, hdr_end = 0;
  std::vector<HintedMember> ms;
  void finish(int r, size_t n) {
    rc = r;
    out_len = n;
    live = false;
    kind = 0;  // (a finished stream has no unit in this or any later round)
  }
};

// The room of a unit that starts at out_pos of a stream's slot with `il` compressed bytes (run_one_staged's)
static uint32_t gz_unit_room(const GzStream &s, size_t out_pos, uint32_t il) {
  size_t room = s.slot > out_pos ? s.slot - out_pos : 0;
  room = std::min(room, max_inflate_out(il));
  return (uint32_t)std::min<size_t>(room, 0xfffffff0u);
}

// Puts the next step of a stream that is in its zlib stream loop into the unit table, or finishes it.
struct GzUnits {
  std::vector<uint64_t> in_off, out_off;
  std::vector<uint32_t> in_len, cap, hist;
  void add(uint64_t io, uint32_t il, uint64_t oo, uint32_t oc, uint32_t h) {
    in_off.push_back(io);
    in_len.push_back(il);
    out_off.push_back(oo);
    cap.push_back(oc);
    hist.push_back(h);
  }
  size_t size() const { return in_off.size(); }
};
static void gz_zlib_step(GzStream &s, GzUnits &u) {
  if (s.pos >= s.len) return s.finish(B200Z_OK, s.out_pos + s.pending);  // (:101-103)
  if (!s.raw) {
    const int r = zlib_header_rule(s.h, s.len, &s.pos);
    if (r) return s.finish(r, s.out_pos);
  }
  s.out_pos += s.pending;  // output.writeBytes(buffer) (:82-84)
  s.pending = 0;
  const size_t avail = s.len - s.pos;
  const uint32_t il = (uint32_t)std::min<size_t>(avail, 0xfffffff0u);
  s.kind = 3;
  s.u0 = u.size();
  u.add(s.din + s.pos, il, s.dout + s.out_pos, gz_unit_room(s, s.out_pos, il), 0);
}
static void gz_gzip_step(GzStream &s, GzUnits &u) {
  if (s.pos >= s.len) return s.finish(B200Z_OK, s.out_pos);
  if (!s.skip_hint) {
    s.ms.clear();
    size_t promised = 0;
    hinted_run(s.h, s.len, s.pos, &s.ms, &promised);
    if (!s.ms.empty()) {
      const size_t o = s.out_pos + promised;
      if (gzip_hinted_room_rule(o, s.cap)) return s.finish(B200Z_E_NOSPC, o);
      s.kind = 1;
      s.u0 = u.size();
      size_t op = s.out_pos;
      for (const HintedMember &m : s.ms) {
        // a hint that lies can promise more than the slot holds (slot < cap): the member then gets what is left, fails
        // its hint and is redone hint-free, as a lying hint is anyway
        const uint32_t room = (uint32_t)std::min<size_t>(m.isize, s.slot > op ? s.slot - op : 0);
        u.add(s.din + m.hdr_end, (uint32_t)(m.next - m.hdr_end), s.dout + op, room, 0);
        op += m.isize;
      }
      return;
    }
  }
  s.skip_hint = false;
  const int h = gzip_member_header_rule(s.h, s.len, s.pos, &s.hdr_end);
  if (h < 0) return s.finish(h, s.out_pos);
  if (h == 0) {  // no gzip header: the zlib loop on the same little-endian stream (:31-37), from here on
    s.zlib = true;
    s.big_endian = false;
    s.pending = 0;
    return gz_zlib_step(s, u);
  }
  const uint32_t il = (uint32_t)std::min<size_t>(s.len - s.hdr_end, 0xfffffff0u);
  s.kind = 2;
  s.u0 = u.size();
  u.add(s.din + s.hdr_end, il, s.dout + s.out_pos, gz_unit_room(s, s.out_pos, il),
        (uint32_t)std::min<size_t>(s.out_pos, 65535));  // distances end at 32768
}

// One device group: streams [a, b) of `st`, whose inputs and slots are laid out from 0 in g.d_in / g.d_out.
static int gz_decode_group(std::vector<GzStream> &st, size_t a, size_t b, size_t in_bytes, size_t out_bytes,
                           const std::vector<uint8_t> &packed_in) {
  CU(g.d_in.reserve(in_bytes + 64));
  CU(g.d_out.reserve(out_bytes + 64));
  if (in_bytes) CU(cudaMemcpyAsync(g.d_in.p, packed_in.data(), in_bytes, cudaMemcpyHostToDevice, g.stream));
  g_gzb_stats[1]++;
  GzUnits u;
  std::vector<uint32_t> r_len, r_used;
  std::vector<int32_t> r_st;
  for (;;) {
    u = GzUnits();
    for (size_t i = a; i < b; ++i) {
      GzStream &s = st[i];
      if (!s.live) continue;
      s.kind = 0;
      if (s.zlib)
        gz_zlib_step(s, u);
      else
        gz_gzip_step(s, u);
    }
    const size_t nu = u.size();
    if (nu == 0) break;
    g_gzb_stats[2]++;
    g_gzb_stats[3] += nu;
    r_len.assign(nu, 0);
    r_used.assign(nu, 0);
    r_st.assign(nu, 0);
    std::vector<bool> done(nu, false);
    // K12 first for the large units (run_one_staged's rule; a gzip member only when no successor header is near)
    std::vector<CkIn> ck;
    std::vector<size_t> ck_unit;
    for (size_t i = a; i < b; ++i) {
      const GzStream &s = st[i];
      if (!s.live || (s.kind != 2 && s.kind != 3)) continue;
      const size_t k = s.u0;
      if (u.in_len[k] < g_ck.thresh) continue;
      if (s.kind == 2 && gzip_member_header_within(s.h, s.len, s.hdr_end, g_ck.thresh)) continue;
      const uint32_t n_pages = ck_pages_for(workspace_bytes(1, s.out_pos + u.cap[k]));
      if (!n_pages) continue;
      const size_t at = s.kind == 2 ? s.hdr_end : s.pos;
      ck.push_back(CkIn{s.h + at, u.in_off[k], u.in_len[k], u.out_off[k], u.cap[k], u.hist[k], n_pages});
      ck_unit.push_back(k);
    }
    if (!ck.empty()) {
      std::vector<CkOut> res;
      double ms[3] = {0, 0, 0};
      const int rc = run_chunked(ck, res, ms);
      if (rc) return rc;
      g_gzb_stats[4] += ck.size();
      for (size_t c = 0; c < ck.size(); ++c)
        if (res[c].accepted) {
          const size_t k = ck_unit[c];
          r_len[k] = res[c].r.out_len;
          r_used[k] = res[c].r.in_used;
          r_st[k] = res[c].r.status;
          done[k] = true;
          g_gzb_stats[5]++;
        }
    }
    // everything else: one inflate batch (k_inflate_fast first when no unit has a history)
    {
      GzUnits v;
      std::vector<size_t> back;
      bool any_hist = false;
      for (size_t k = 0; k < nu; ++k)
        if (!done[k]) {
          v.add(u.in_off[k], u.in_len[k], u.out_off[k], u.cap[k], u.hist[k]);
          back.push_back(k);
          any_hist |= u.hist[k] != 0;
        }
      if (!back.empty()) {
        const size_t m = back.size();
        size_t extent = 0;
        for (size_t k = 0; k < m; ++k) extent = std::max<size_t>(extent, v.out_off[k] + v.cap[k]);
        std::vector<uint32_t> l(m), us(m);
        std::vector<int32_t> sv(m);
        const int rc = run_batch_on_staged(v.in_off.data(), v.in_len.data(), v.out_off.data(), v.cap.data(), l.data(), sv.data(),
                                           us.data(), m, extent, false, 0, any_hist ? v.hist.data() : nullptr);
        if (rc) return rc;
        for (size_t k = 0; k < m; ++k) {
          r_len[back[k]] = l[k];
          r_used[back[k]] = us[k];
          r_st[back[k]] = sv[k];
        }
      }
    }
    // each stream's next step, by the rules of the single calls
    std::vector<size_t> ad_stream;
    std::vector<uint64_t> ad_off, ad_len;
    std::vector<uint32_t> ad_stored;
    for (size_t i = a; i < b; ++i) {
      GzStream &s = st[i];
      if (!s.live || s.kind == 0) continue;
      const size_t k = s.u0;
      if (s.kind == 1) {
        const size_t acc = hinted_exact_prefix(s.ms, &r_len[k], &r_st[k], &r_used[k]);
        size_t op = s.out_pos;
        for (size_t j = 0; j < acc; ++j) op += s.ms[j].isize;
        if (acc > 0) s.pos = s.ms[acc - 1].next;
        s.out_pos = op;
        s.skip_hint = acc < s.ms.size();
        continue;
      }
      const OneResult r{r_len[k], r_used[k], r_st[k]};
      if (s.kind == 2) {
        s.out_pos += r.out_len;
        const int rc = gzip_member_rule(r, s.pos, s.hdr_end, s.len, s.cap, &s.pos);
        if (rc) s.finish(rc, s.out_pos);
        continue;
      }
      uint32_t stored = 0;
      size_t n = s.out_pos;
      const int rc = zlib_stream_rule(r, s.h, s.len, s.raw, s.big_endian, s.out_pos, s.cap, &s.pos, &stored, &n);
      if (rc) {
        s.finish(rc, n);
        continue;
      }
      s.pending = r.out_len;
      if (!s.raw && s.verify) {
        ad_stream.push_back(i);
        ad_off.push_back(s.dout + s.out_pos);
        ad_len.push_back(r.out_len);
        ad_stored.push_back(stored);
      }
    }
    if (!ad_stream.empty()) {  // one Adler-32 launch for every stream of the round that finished a zlib stream
      std::vector<uint32_t> ad(ad_stream.size());
      const int rc = device_adler32_many((const uint8_t *)g.d_out.p, ad_off.data(), ad_len.data(), ad_stream.size(), ad.data());
      if (rc) return rc;
      for (size_t j = 0; j < ad_stream.size(); ++j) {
        GzStream &s = st[ad_stream[j]];
        if (zlib_adler_rule(ad[j], ad_stored[j])) s.finish(B200Z_E_DATA, s.out_pos);
      }
    }
  }
  return B200Z_OK;
}

// n streams (arguments checked): rc[i] / out_len[i] / the slot's bytes as b200z_gzip_decode (gzip) or b200z_zlib_decode
// give for stream i alone; `verify` takes B200Z_GZIP_VERIFY / B200Z_GZIP_RAW for gzip, a bool for zlib.  dev_out: out_base
// is device memory on the library's device
static int gzip_zlib_decode_streams(bool gzip, const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n,
                                    int verify, int raw, uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                    uint64_t *out_len, int32_t *rc, bool dev_out = false) {
  for (auto &v : g_gzb_stats) v = 0;
  g_gzb_stats[0] = n;
  std::vector<GzStream> st(n);
  for (size_t i = 0; i < n; ++i) {
    GzStream &s = st[i];
    s.h = in_len[i] ? in_base + in_off[i] : nullptr;
    s.len = (size_t)in_len[i];
    s.cap = (size_t)out_cap[i];
    s.slot = std::min<size_t>(s.cap, max_inflate_out(s.len));
    if (gzip) {
      s.verify = (verify & B200Z_GZIP_VERIFY) != 0;
      s.raw = (verify & B200Z_GZIP_RAW) != 0;
    } else {
      s.zlib = true;
      s.verify = verify != 0;
      s.raw = raw != 0;
      s.big_endian = true;
    }
  }
  // device groups: consecutive streams whose inputs, slots and inflate workspace fit half the free device memory
  size_t budget = (size_t)32 << 30;
  {
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess && free_b)
      budget = std::min(budget, (free_b + g.d_in.cap + g.d_out.cap + g.d_ws.cap) / 2);
  }
  std::vector<uint8_t> packed;
  size_t a = 0;
  while (a < n) {
    size_t b = a, in_bytes = 0, out_bytes = 0;
    while (b < n) {
      const size_t ib = align_up(st[b].len + 64, 256), ob = align_up(st[b].slot + 64, 256);
      const size_t need = in_bytes + ib + out_bytes + ob + workspace_bytes(b - a + 1, out_bytes + ob);
      if (b > a && (need > budget || (g_gzb_max_group && b - a >= g_gzb_max_group))) break;
      st[b].din = in_bytes;
      st[b].dout = out_bytes;
      in_bytes += ib;
      out_bytes += ob;
      ++b;
    }
    // the group's inputs, each followed by zeros up to the next, go up in one copy
    packed.assign(in_bytes, 0);
    for (size_t i = a; i < b; ++i)
      if (st[i].len) memcpy(packed.data() + st[i].din, st[i].h, st[i].len);
    int r = gz_decode_group(st, a, b, in_bytes, out_bytes, packed);
    if (r) return r;
    if (dev_out) {  // device slots: the bytes of every stream that did not run out of room, in one k_copy_slots launch
      std::vector<SlotCopy> cp;
      for (size_t i = a; i < b; ++i) {
        const size_t k = st[i].rc == B200Z_E_NOSPC ? 0 : std::min(st[i].out_len, st[i].cap);
        if (k) cp.push_back(SlotCopy{st[i].dout, out_off[i], k});
      }
      CU(copy_slots((const uint8_t *)g.d_out.p, out_base, cp.data(), cp.size(), g.stream));
      CU(cudaStreamSynchronize(g.stream));
    } else {
      // results, and the bytes of every stream that did not run out of room (the single calls copy nothing then).  The
      // bytes come back through a pinned staging buffer of at most GZ_STAGE bytes, one asynchronous copy per stream and one
      // synchronise per fill; a stream larger than the buffer is copied straight into its slot.
      size_t i0 = a, o = 0;
      auto drain = [&](size_t i1) -> int {  // streams [i0, i1) are in the staging buffer, back to back
        CU(cudaStreamSynchronize(g.stream));
        for (size_t p = 0; i0 < i1; ++i0) {
          const size_t k = st[i0].rc == B200Z_E_NOSPC ? 0 : std::min(st[i0].out_len, st[i0].cap);
          if (k && k <= GZ_STAGE) {
            memcpy(out_base + out_off[i0], (const uint8_t *)g.h_stage.p + p, k);
            p += k;
          }
        }
        o = 0;
        return B200Z_OK;
      };
      for (size_t i = a; i < b; ++i) {
        const size_t k = st[i].rc == B200Z_E_NOSPC ? 0 : std::min(st[i].out_len, st[i].cap);
        const uint8_t *src = (const uint8_t *)g.d_out.p + st[i].dout;
        if (k > GZ_STAGE) {
          CU(cudaMemcpyAsync(out_base + out_off[i], src, k, cudaMemcpyDeviceToHost, g.stream));
        } else if (k) {
          if (o + k > GZ_STAGE && (r = drain(i)) != B200Z_OK) return r;
          CU(g.h_stage.reserve(GZ_STAGE));
          CU(cudaMemcpyAsync((uint8_t *)g.h_stage.p + o, src, k, cudaMemcpyDeviceToHost, g.stream));
          o += k;
        }
      }
      if ((r = drain(b)) != B200Z_OK) return r;
    }
    for (size_t i = a; i < b; ++i) {
      out_len[i] = st[i].out_len;
      rc[i] = st[i].rc;
    }
    a = b;
  }
  return B200Z_OK;
}

}  // namespace b200z


// =============================================================================================
// BZip2Decoder.decodeBytes / decodeStream  (bzip2_decoder.dart:13-88)
// Host side: stream header, ordering + chain validation of the block candidates the scan kernel finds,
// stored-CRC comparison.  All bit/byte work is in bzip2_kernels.cu.
// =============================================================================================
namespace b200z {

struct Carver {  // carve typed arrays out of one device allocation
  uint8_t *p;
  size_t off = 0;
  explicit Carver(void *base) : p((uint8_t *)base) {}
  template <typename T>
  T *take(size_t n) {
    off = align_up(off, 256);
    T *r = p ? (T *)(p + off) : nullptr;
    off += n * sizeof(T);
    return r;
  }
};

// shard != nullptr: decode only this rank's share of the block candidates and report every block instead of walking the
// chain (the ranks' reports are merged and validated by the caller, archive_b200/shard.py).
struct Bz2Shard {
  uint32_t rank, world;
  b200z_bz2_block *blocks;
  size_t blocks_cap, n_blocks;
};

// One stream of a batch: its bytes d_base[in_off, +in_len) on the device, its output slot on the host, and what
// decodeStream makes of it (rc, out_len: what b200z_bzip2_decode returns and reports for the stream alone).
struct Bz2Job {
  uint64_t in_off, in_len;
  uint8_t *out;
  size_t out_cap;
  size_t out_len;
  int rc;
};

// (test hooks) cap on the blocks of one device group (0: the memory budget alone); the last call's streams, device groups
// and blocks
static uint32_t g_bz2_max_group_blocks = 0;
static unsigned long long g_bz2_stats[3];
// Device memory a group of streams may take for K7/K8 workspace and output slots, unless the buffers already hold more.
// One stream that needs more runs as a group of its own.
constexpr size_t BZ2_GROUP_BUDGET = (size_t)8 << 30;

struct Bz2Arrays {
  unsigned long long *blk_bit, *blk_end, *end_bit, *block_out, *block_off;
  uint32_t *blk_lim, *rec_val, *rec_pos, *n_rec, *nblock, *orig_ptr, *rnd, *chist, *tt, *seg_len, *seg_next, *seg_off, *seg_resume,
      *slice_state, *slice_out, *block_crc, *cycle_len, *fast, *walk_ctr;
  int32_t *status, *irregular;
  uint8_t *sym8, *raw, *slots;
  BzChainHost *chain;
  size_t bytes;
};
// nb_all candidate blocks, the big per-block arrays for nbk of them at a stride of `stride` (the largest level x 100000 of
// the group's streams)
static Bz2Arrays bz2_carve(void *base, uint32_t nb_all, uint32_t nbk, uint32_t stride) {
  Carver c(base);
  const uint32_t chunks_max = (stride + 1023) / 1024;
  Bz2Arrays a;
  a.blk_bit = c.take<unsigned long long>(nb_all);
  a.blk_end = c.take<unsigned long long>(nb_all);
  a.blk_lim = c.take<uint32_t>(nb_all);
  a.end_bit = c.take<unsigned long long>(nbk);
  a.block_out = c.take<unsigned long long>(nbk);
  a.block_off = c.take<unsigned long long>(nbk + 1);
  a.n_rec = c.take<uint32_t>(nbk);
  a.nblock = c.take<uint32_t>(nbk);
  a.orig_ptr = c.take<uint32_t>(nbk);
  a.rnd = c.take<uint32_t>(nbk);
  a.status = c.take<int32_t>(nbk);
  a.irregular = c.take<int32_t>(nbk);
  a.block_crc = c.take<uint32_t>(nbk);
  a.cycle_len = c.take<uint32_t>(nbk);
  a.fast = c.take<uint32_t>(nbk);
  a.walk_ctr = c.take<uint32_t>(4);
  a.chain = c.take<BzChainHost>(nbk);
  a.seg_len = c.take<uint32_t>((size_t)nbk * 4098);
  a.seg_next = c.take<uint32_t>((size_t)nbk * 4098);
  a.seg_off = c.take<uint32_t>((size_t)nbk * 4098);
  a.seg_resume = c.take<uint32_t>((size_t)nbk * 4098);
  a.slice_state = c.take<uint32_t>((size_t)nbk * 1024);
  a.slice_out = c.take<uint32_t>((size_t)nbk * 1024);
  a.chist = c.take<uint32_t>((size_t)nbk * chunks_max * 256);
  a.rec_val = c.take<uint32_t>((size_t)nbk * stride);
  a.rec_pos = c.take<uint32_t>((size_t)nbk * stride);
  a.tt = c.take<uint32_t>((size_t)nbk * stride);
  a.sym8 = c.take<uint8_t>((size_t)nbk * stride);
  a.raw = c.take<uint8_t>((size_t)nbk * stride);
  a.slots = c.take<uint8_t>((size_t)nbk * bz2_slot_bytes_per_block());
  a.bytes = align_up(c.off, 256);
  return a;
}

// the 32 bits from `bit` on (big-endian; bytes past the end read 0) of a stream of `len` bytes, for a bit among its last 48:
// they lie in its last 8 bytes, which are all the host has of it
static inline uint32_t be32_in_tail(const uint8_t *tail8, uint64_t len, uint64_t bit) {
  uint64_t v = 0;
  const uint64_t b0 = bit >> 3;
  for (int i = 0; i < 5; ++i) {
    const uint64_t j = b0 + i;
    v = (v << 8) | (j < len && j + 8 >= len ? tail8[j + 8 - len] : 0u);
  }
  return (uint32_t)(v >> (8 - (bit & 7)));
}

// BZip2Decoder.decodeStream for n streams whose bytes are on the device already.  K6 scans all of them in one launch; the
// streams are then cut into consecutive device groups that fit the memory budget, and each group takes one K7 and one K8
// over the blocks of all its streams, each stream's output going to a slot of its own.  Returns B200Z_OK unless the device
// fails; each stream's result is in its job.  dev_out != nullptr: the jobs' slots are device memory from dev_out on, and each
// delivery is one k_copy_slots launch for the streams it serves instead of one copy to the host per stream.
static int bzip2_decode_device(const uint8_t *d_base, Bz2Job *jobs, size_t n, int verify, Bz2Shard *shard = nullptr,
                               uint8_t *dev_out = nullptr) {
  g_bz2_stats[0] = n;
  g_bz2_stats[1] = g_bz2_stats[2] = 0;
  if (n == 0) return B200Z_OK;

  // ---- K6: candidates of every stream, with their stream, their stored CRC and the streams' first and last bytes ----
  std::vector<Bz2ScanStream> h_str(n);
  std::vector<unsigned long long> h_thr(n + 1, 0);
  for (size_t i = 0; i < n; ++i) {
    jobs[i].out_len = 0;
    jobs[i].rc = B200Z_OK;
    h_str[i] = {jobs[i].in_off, jobs[i].in_len};
    h_thr[i + 1] = h_thr[i] + std::max<uint64_t>(1, (jobs[i].in_len + 3) / 4);
  }
  auto scan_layout = [&](void *base, uint32_t cap, size_t *bytes) {
    Carver c(base);
    Bz2Scan a;
    a.in = d_base;
    a.n_streams = (uint32_t)n;
    a.cap = cap;
    a.n_cand = c.take<uint32_t>(1);
    a.streams = c.take<Bz2ScanStream>(n);
    a.first_thr = c.take<unsigned long long>(n + 1);
    a.ends = c.take<uint8_t>(n * 12);
    a.cand = c.take<unsigned long long>(cap);
    a.cand_stream = c.take<uint32_t>(cap);
    a.cand_crc = c.take<uint32_t>(cap);
    *bytes = align_up(c.off, 256);
    return a;
  };
  const uint32_t cand_cap = 1u << 20;  // per stream
  uint32_t cap = cand_cap, ncand = 0;
  Bz2Scan sc;
  for (;;) {
    size_t bytes = 0;
    scan_layout(nullptr, cap, &bytes);
    CU(g.d_small.reserve(bytes));
    sc = scan_layout(g.d_small.p, cap, &bytes);
    CU(cudaMemcpyAsync((void *)sc.streams, h_str.data(), n * sizeof(Bz2ScanStream), cudaMemcpyHostToDevice, g.stream));
    CU(cudaMemcpyAsync((void *)sc.first_thr, h_thr.data(), (n + 1) * 8, cudaMemcpyHostToDevice, g.stream));
    CU(bz2_launch_scan_streams(sc, h_thr[n], g.stream));
    CU(cudaMemcpyAsync(&ncand, sc.n_cand, 4, cudaMemcpyDeviceToHost, g.stream));
    CU(cudaStreamSynchronize(g.stream));
    if (ncand <= cap) break;
    cap = ncand;  // (more candidates than the buffer holds: once more with room for all of them)
  }
  std::vector<unsigned long long> h_cand(ncand);
  std::vector<uint32_t> h_cstr(ncand), h_ccrc(ncand);
  std::vector<uint8_t> ends(n * 12);
  if (ncand) {
    CU(cudaMemcpyAsync(h_cand.data(), sc.cand, (size_t)ncand * 8, cudaMemcpyDeviceToHost, g.stream));
    CU(cudaMemcpyAsync(h_cstr.data(), sc.cand_stream, (size_t)ncand * 4, cudaMemcpyDeviceToHost, g.stream));
    CU(cudaMemcpyAsync(h_ccrc.data(), sc.cand_crc, (size_t)ncand * 4, cudaMemcpyDeviceToHost, g.stream));
  }
  CU(cudaMemcpyAsync(ends.data(), sc.ends, n * 12, cudaMemcpyDeviceToHost, g.stream));
  CU(cudaStreamSynchronize(g.stream));
  // candidates by stream, then by bit; positions from here on are bits of their stream (| end-of-stream << 63)
  std::vector<uint32_t> order(ncand);
  for (uint32_t i = 0; i < ncand; ++i) order[i] = i;
  const unsigned long long POS = ~(1ull << 63);
  std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
    return h_cstr[a] != h_cstr[b] ? h_cstr[a] < h_cstr[b] : (h_cand[a] & POS) < (h_cand[b] & POS);
  });
  std::vector<unsigned long long> cand(ncand);
  std::vector<uint32_t> ccrc(ncand);
  std::vector<uint32_t> c_lo(n + 1, 0);
  for (uint32_t i = 0; i < ncand; ++i) {
    const uint32_t o = order[i], s = h_cstr[o];
    cand[i] = h_cand[o] - jobs[s].in_off * 8;
    ccrc[i] = h_ccrc[o];
    c_lo[s + 1]++;
  }
  for (size_t s = 0; s < n; ++s) c_lo[s + 1] += c_lo[s];

  // ---- stream headers: 'B' 'Z' 'h' level, each a readByte() that throws at EOS (bz2_bit_reader.dart:17-20) ----
  std::vector<uint32_t> lim(n, 0), nblk(n, 0);
  std::vector<char> live(n, 0);
  static const uint8_t sig[3] = {0x42, 0x5a, 0x68};
  for (size_t s = 0; s < n; ++s) {
    const uint8_t *hd = ends.data() + s * 12;
    const uint64_t len = jobs[s].in_len;
    int r = B200Z_OK;
    for (int i = 0; i < 3 && r == B200Z_OK; ++i) {
      if ((uint64_t)i >= len) {
        set_err("bzip2: truncated signature (Dart: RangeError)");
        r = B200Z_E_THROW;
      } else if (hd[i] != sig[i]) {
        set_err("bzip2: bad signature");
        r = B200Z_E_DATA;
      }
    }
    if (r == B200Z_OK && len < 4) {
      set_err("bzip2: truncated header (Dart: RangeError)");
      r = B200Z_E_THROW;
    }
    const int level = (int)hd[3] - 0x30;
    if (r == B200Z_OK && (level < 0 || level > 9)) {
      set_err("bzip2: bad block size");
      r = B200Z_E_DATA;
    }
    if (r == B200Z_OK && c_lo[s + 1] - c_lo[s] > cand_cap) {
      set_err("bzip2: more than %u magic candidates", cand_cap);
      r = B200Z_E_INTERNAL;
    }
    jobs[s].rc = r;
    if (r != B200Z_OK || len == 4) continue;  // (len 4: while (!input.isEOS) never runs)
    live[s] = 1;
    lim[s] = (uint32_t)level * 100000u;
    for (uint32_t c = c_lo[s]; c < c_lo[s + 1]; ++c) nblk[s] += (cand[c] >> 63) ? 0u : 1u;
  }

  size_t budget = g.d_bz.cap + g.d_out.cap, free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess) budget = std::max(budget, std::min(free_b / 2, BZ2_GROUP_BUDGET));
  std::vector<size_t> grp;
  for (size_t s0 = 0; s0 < n;) {
    // ---- the next device group: consecutive streams whose workspace and output slots fit the budget ----
    grp.clear();
    uint32_t nb = 0, stride = 0;
    size_t room = 0;
    for (; s0 < n; ++s0) {
      if (!live[s0]) continue;
      const uint32_t nb2 = nb + nblk[s0], stride2 = std::max(stride, lim[s0]);
      const size_t room2 = room + jobs[s0].out_cap;
      if (!grp.empty() && ((g_bz2_max_group_blocks && nb2 > g_bz2_max_group_blocks) ||
                           bz2_carve(nullptr, std::max(nb2, 1u), std::max(nb2, 1u), stride2).bytes + room2 > budget))
        break;
      grp.push_back(s0);
      nb = nb2;
      stride = stride2;
      room = room2;
    }
    if (grp.empty()) break;
    const size_t G = grp.size();
    g_bz2_stats[1]++;
    g_bz2_stats[2] += nb;

    // blocks of the group, stream after stream; blk_of[c] = the block a candidate is (for block candidates)
    std::vector<unsigned long long> blk_bits, blk_end;
    std::vector<uint32_t> blk_lim, blk_crc, blk_of(ncand, 0xffffffffu);
    for (size_t s : grp)
      for (uint32_t c = c_lo[s]; c < c_lo[s + 1]; ++c)
        if (!(cand[c] >> 63)) {
          blk_of[c] = (uint32_t)blk_bits.size();
          blk_bits.push_back(jobs[s].in_off * 8 + cand[c]);
          blk_end.push_back((jobs[s].in_off + jobs[s].in_len) * 8);
          blk_lim.push_back(lim[s]);
          blk_crc.push_back(cand[c] + 80 <= jobs[s].in_len * 8 ? ccrc[c] : 0u);
        }
    const uint32_t nb_all = nb ? nb : 1;
    uint32_t k_lo = 0, k_hi = nb;  // candidates this call decodes
    if (shard) {
      k_lo = (uint32_t)((uint64_t)nb * shard->rank / shard->world);
      k_hi = (uint32_t)((uint64_t)nb * (shard->rank + 1) / shard->world);
    }
    const uint32_t nbk = k_hi > k_lo ? k_hi - k_lo : 1;  // (a shard needs the big per-block arrays for its share only)
    CU(g.d_bz.reserve(bz2_carve(nullptr, nb_all, nbk, stride).bytes));
    const Bz2Arrays A = bz2_carve(g.d_bz.p, nb_all, nbk, stride);

    // ---- K7 on every candidate (speculative: a magic-looking bit pattern inside a block just decodes to junk) ----
    std::vector<uint32_t> h_nrec(nb), h_nblock(nb), h_optr(nb), h_rnd(nb);
    std::vector<unsigned long long> h_end(nb);
    std::vector<int32_t> h_st(nb);
    if (k_hi > k_lo) {
      CU(cudaMemcpyAsync(A.blk_bit, blk_bits.data(), (size_t)nb * 8, cudaMemcpyHostToDevice, g.stream));
      CU(cudaMemcpyAsync(A.blk_end, blk_end.data(), (size_t)nb * 8, cudaMemcpyHostToDevice, g.stream));
      CU(cudaMemcpyAsync(A.blk_lim, blk_lim.data(), (size_t)nb * 4, cudaMemcpyHostToDevice, g.stream));
      Bz2Entropy e;
      e.words = (const uint32_t *)d_base;
      e.n_bytes = 0;  // (every block has its stream's end in blk_end)
      e.blk_bit = A.blk_bit + k_lo;
      e.blk_end = A.blk_end + k_lo;
      e.blk_lim = A.blk_lim + k_lo;
      e.n_blocks = k_hi - k_lo;
      e.nblock_max = stride;
      // block k of this call uses slot k - k_lo of every per-block array
      e.rec_val = A.rec_val; e.rec_pos = A.rec_pos; e.n_rec = A.n_rec; e.nblock = A.nblock; e.orig_ptr = A.orig_ptr;
      e.randomised = A.rnd; e.end_bit = A.end_bit; e.status = A.status; e.fast_flag = A.fast; e.sym8 = A.sym8;
      CU(bz2_launch_entropy(e, g.stream));
      const uint32_t m = k_hi - k_lo;
      auto fetch = [&]() -> int {
        CU(cudaMemcpyAsync(h_nrec.data() + k_lo, A.n_rec, m * 4, cudaMemcpyDeviceToHost, g.stream));
        CU(cudaMemcpyAsync(h_nblock.data() + k_lo, A.nblock, m * 4, cudaMemcpyDeviceToHost, g.stream));
        CU(cudaMemcpyAsync(h_optr.data() + k_lo, A.orig_ptr, m * 4, cudaMemcpyDeviceToHost, g.stream));
        CU(cudaMemcpyAsync(h_rnd.data() + k_lo, A.rnd, m * 4, cudaMemcpyDeviceToHost, g.stream));
        CU(cudaMemcpyAsync(h_end.data() + k_lo, A.end_bit, (size_t)m * 8, cudaMemcpyDeviceToHost, g.stream));
        CU(cudaMemcpyAsync(h_st.data() + k_lo, A.status, m * 4, cudaMemcpyDeviceToHost, g.stream));
        CU(cudaStreamSynchronize(g.stream));
        return B200Z_OK;
      };
      int rc = fetch();
      if (rc) return rc;
      {
        std::vector<uint32_t> h_fast(m);
        CU(cudaMemcpy(h_fast.data(), A.fast, (size_t)m * 4, cudaMemcpyDeviceToHost));
        unsigned long long nf = 0;
        for (uint32_t v : h_fast) nf += v;
        g_bz2_fast_blocks += nf;
        g_bz2_exact_blocks += m - nf;
      }
      // damaged blocks that the reference keeps decoding past a bad Huffman code (K7 status -3): decoded again the reference's
      // way, one thread each (bzip2_kernels.cu: k_bz2_entropy_literal); intact streams have none
      std::vector<uint32_t> quirk;
      for (uint32_t k = k_lo; k < k_hi; ++k)
        if (h_st[k] == -3) quirk.push_back(k - k_lo);
      if (!quirk.empty()) {
        uint32_t *d_list = (uint32_t *)((uint8_t *)g.d_small.p + 256);  // the scan's arrays are on the host by now
        CU(cudaMemcpyAsync(d_list, quirk.data(), quirk.size() * 4, cudaMemcpyHostToDevice, g.stream));
        CU(bz2_launch_entropy_literal(e, d_list, (uint32_t)quirk.size(), g.stream));
        rc = fetch();
        if (rc) return rc;
      }
    }

    // ---- walk each stream's chain exactly as decodeStream's loop does (:46-87) ----
    std::vector<BzChainHost> chain;
    std::vector<uint32_t> stored_crc, ch_lo(G + 1, 0), eos_crc(G, 0);
    std::vector<char> have_eos(G, 0);
    std::vector<int> s_rc(G, B200Z_OK);
    std::vector<unsigned long long> s_lo(G), s_hi(G);  // each stream's output slot in g.d_out
    std::vector<uint32_t> chain_of(nb, 0xffffffffu);
    size_t dev_room = 0;
    for (size_t q = 0; q < G; ++q) {
      const size_t s = grp[q];
      s_lo[q] = dev_room;
      dev_room += jobs[s].out_cap;
      s_hi[q] = dev_room;
      ch_lo[q] = (uint32_t)chain.size();
      const uint64_t in_len = jobs[s].in_len, total_bits = in_len * 8, base_bit = jobs[s].in_off * 8;
      auto push_block = [&](uint32_t k, uint32_t crc) {
        chain_of[k] = (uint32_t)chain.size();
        BzChainHost ce{k - k_lo, h_nblock[k], h_nrec[k], h_optr[k], h_rnd[k] ? 1u : 0u};  // randomised: serial walk in K8
        if (chain.size() == ch_lo[q]) ce.flags |= 2u;
        ce.out_lo = s_lo[q];
        ce.out_hi = s_hi[q];
        chain.push_back(ce);
        stored_crc.push_back(crc);
      };
      if (shard) {
        for (uint32_t k = k_lo; k < k_hi; ++k)
          if (h_st[k] == 0) push_block(k, blk_crc[k]);
        continue;
      }
      const uint8_t *tail = ends.data() + s * 12 + 4;
      int final_rc = B200Z_OK;
      uint64_t pos = 32;
      uint32_t ci = c_lo[s];
      const uint32_t c_end = c_lo[s + 1];
      for (;;) {
        if ((pos + 7) / 8 >= in_len) break;  // input.isEOS: every byte has been pulled into the bit reader
        if (pos + 48 > total_bits) {
          // _readBlockType (:90-111) reads its 6 bytes one at a time: the first one that fits neither magic returns -1 before
          // the missing bytes are asked for (RangeError)
          static const uint8_t blk_magic[6] = {0x31, 0x41, 0x59, 0x26, 0x53, 0x59}, eos_magic[6] = {0x17, 0x72, 0x45, 0x38, 0x50, 0x90};
          bool blk = true, eos = true, mismatch = false;
          for (int i = 0; i < 6 && pos + 8 * (uint64_t)(i + 1) <= total_bits; ++i) {
            const uint8_t b = (uint8_t)(be32_in_tail(tail, in_len, pos + 8 * (uint64_t)i) >> 24);
            blk = blk && b == blk_magic[i];
            eos = eos && b == eos_magic[i];
            if (!blk && !eos) {
              mismatch = true;
              break;
            }
          }
          if (mismatch) {
            set_err("bzip2: no block signature at bit %llu", (unsigned long long)pos);
            final_rc = B200Z_E_DATA;
          } else {
            set_err("bzip2: truncated block header (Dart: RangeError)");
            final_rc = B200Z_E_THROW;
          }
          break;
        }
        while (ci < c_end && (cand[ci] & POS) < pos) ++ci;
        if (ci >= c_end || (cand[ci] & POS) != pos) {
          set_err("bzip2: no block signature at bit %llu", (unsigned long long)pos);
          final_rc = B200Z_E_DATA;  // _readBlockType -> -1 -> false
          break;
        }
        if (pos + 80 > total_bits) {  // 4 CRC bytes follow either magic
          set_err("bzip2: truncated CRC (Dart: RangeError)");
          final_rc = B200Z_E_THROW;
          break;
        }
        if (cand[ci] >> 63) {
          have_eos[q] = 1;
          eos_crc[q] = ccrc[ci];
          break;  // end of stream: whatever follows is ignored (:83-84)
        }
        const uint32_t k = blk_of[ci];
        if (h_st[k] == -2) {
          set_err("bzip2: block at bit %llu reads past the end (Dart: RangeError)", (unsigned long long)pos);
          final_rc = B200Z_E_THROW;
          break;
        }
        if (h_st[k] != 0) {
          set_err("bzip2: data error in the block at bit %llu", (unsigned long long)pos);
          final_rc = B200Z_E_DATA;
          break;
        }
        push_block(k, ccrc[ci]);
        pos = h_end[k] - base_bit;
      }
      s_rc[q] = final_rc;
      if (getenv("B200Z_DEBUG"))
        fprintf(stderr, "[b200z] bzip2: stream %zu: %u candidates, chain %zu, rc so far %d, eos %d\n", s, c_end - c_lo[s],
                chain.size() - ch_lo[q], final_rc, (int)have_eos[q]);
    }
    ch_lo[G] = (uint32_t)chain.size();

    // ---- K8 on the chains of the group ----
    const uint32_t nc = (uint32_t)chain.size();
    std::vector<unsigned long long> h_off(nc + 1, 0), h_out(nc, 0);
    std::vector<unsigned long long> early(s_lo);  // output bytes [s_lo, early) of each stream are on their way to the host (s_d2h)
    bool any_early = false;
    std::vector<uint32_t> h_crc(nc);
    std::vector<int32_t> h_irr(nc);
    // the bytes of the chain entries below `hi` are written: those in the streams' slots go to the host on the copy stream
    auto copy_early = [&](uint32_t hi) -> int {
      std::vector<SlotCopy> cp;
      for (size_t q = 0; q < G; ++q) {
        if (ch_lo[q] >= hi || ch_lo[q] == ch_lo[q + 1]) continue;
        const uint32_t last = std::min(hi, ch_lo[q + 1]) - 1;
        const unsigned long long end = std::min(h_off[last] + h_out[last], s_hi[q]);
        if (end > early[q]) {
          if (dev_out)
            cp.push_back(SlotCopy{early[q], (uint64_t)(jobs[grp[q]].out - dev_out) + (early[q] - s_lo[q]), end - early[q]});
          else
            CU(cudaMemcpyAsync(jobs[grp[q]].out + (early[q] - s_lo[q]), (uint8_t *)g.d_out.p + early[q], end - early[q],
                               cudaMemcpyDeviceToHost, g.s_d2h));
          early[q] = end;
          any_early = true;
        }
      }
      if (dev_out) CU(copy_slots((const uint8_t *)g.d_out.p, dev_out, cp.data(), cp.size(), g.s_d2h));
      return B200Z_OK;
    };
    if (nc) {
      CU(g.d_out.reserve(dev_room + 64));
      CU(cudaMemcpyAsync(A.chain, chain.data(), (size_t)nc * sizeof(BzChainHost), cudaMemcpyHostToDevice, g.stream));
      Bz2Ibwt w;
      w.chain = A.chain; w.n_chain = nc; w.nblock_max = stride;
      w.rec_val = A.rec_val; w.rec_pos = A.rec_pos; w.sym8 = A.sym8; w.chist = A.chist; w.tt = A.tt;
      w.seg_len = A.seg_len; w.seg_next = A.seg_next; w.seg_off = A.seg_off; w.seg_resume = A.seg_resume; w.slots = A.slots; w.walk_ctr = A.walk_ctr; w.irregular = A.irregular; w.cycle_len = A.cycle_len; w.raw = A.raw;
      w.slice_state = A.slice_state; w.slice_out = A.slice_out; w.block_out = A.block_out; w.block_off = A.block_off;
      w.block_crc = A.block_crc; w.out = (uint8_t *)g.d_out.p; w.out_cap = ~0ull;  // (each entry is clipped at its slot)
      for (const BzChainHost &ce : chain) w.any_randomised = w.any_randomised || (ce.flags & 1u);
      w.any_records = false;
      for (const BzChainHost &ce : chain) w.any_records = w.any_records || ce.n_rec != 0;
      // B200Z_BZ2_GROUPS=n decodes a long chain of one stream in n groups, the bytes of a finished group on their way to the
      // host (copy stream) while the next group is decoded.  Measured slower than one piece (512 MiB, 597 blocks), and
      // slower the more groups -- the pointer-chasing kernels of K8 are bound by latency, not by the number of blocks, so a
      // group costs nearly what the whole chain costs.  Off by default.
      uint32_t groups = 1u;
      if (const char *ge = getenv("B200Z_BZ2_GROUPS")) groups = (uint32_t)std::max(1, atoi(ge));
      if (shard || groups > nc || G > 1) groups = 1;
      // The RLE1 output pass (per block) runs in 4 groups and a finished group's bytes go to the host on
      // the copy stream while the next group is written: the blocks' offsets are known before it, so nothing waits
      // (B200Z_BZ2_EMIT_GROUPS, 1: one pass, one copy at the end).
      uint32_t emit_groups = (!shard && nc >= 64) ? 4u : 1u;
      if (const char *ge = getenv("B200Z_BZ2_EMIT_GROUPS")) emit_groups = (uint32_t)std::max(1, atoi(ge));
      if (shard || emit_groups > nc || groups > 1) emit_groups = 1;
      if (groups <= 1 && emit_groups > 1) {
        w.phase = 1;
        CU(bz2_launch_ibwt(w, g.stream));
        CU(cudaMemcpyAsync(h_off.data(), A.block_off, (size_t)(nc + 1) * 8, cudaMemcpyDeviceToHost, g.stream));
        CU(cudaMemcpyAsync(h_out.data(), A.block_out, (size_t)nc * 8, cudaMemcpyDeviceToHost, g.stream));
        CU(cudaStreamSynchronize(g.stream));
        w.phase = 2;
        for (uint32_t gi = 0; gi < emit_groups; ++gi) {
          const uint32_t lo = (uint32_t)((uint64_t)nc * gi / emit_groups), hi = (uint32_t)((uint64_t)nc * (gi + 1) / emit_groups);
          CU(bz2_launch_ibwt_group(w, lo, hi, g.stream));
          cudaEvent_t ev;
          CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
          CU(cudaEventRecord(ev, g.stream));
          CU(cudaStreamWaitEvent(g.s_d2h, ev, 0));
          cudaEventDestroy(ev);  // (released once it has completed)
          const int rc = copy_early(hi);
          if (rc) return rc;
        }
        w.phase = 0;
      } else if (groups <= 1) {
        CU(bz2_launch_ibwt(w, g.stream));
      } else {  // (one stream: its slot starts at 0)
        CU(g.h_meta.reserve((size_t)groups * 8));
        volatile unsigned long long *h_end_off = (volatile unsigned long long *)g.h_meta.p;
        std::vector<cudaEvent_t> ev(groups);
        for (uint32_t gi = 0; gi < groups; ++gi) {
          const uint32_t lo = (uint32_t)((uint64_t)nc * gi / groups), hi = (uint32_t)((uint64_t)nc * (gi + 1) / groups);
          CU(bz2_launch_ibwt_group(w, lo, hi, g.stream));
          CU(cudaMemcpyAsync((void *)(h_end_off + gi), A.block_off + hi, 8, cudaMemcpyDeviceToHost, g.stream));
          CU(cudaEventCreateWithFlags(&ev[gi], cudaEventDisableTiming));
          CU(cudaEventRecord(ev[gi], g.stream));
        }
        for (uint32_t gi = 0; gi < groups; ++gi) {
          CU(cudaEventSynchronize(ev[gi]));
          cudaEventDestroy(ev[gi]);
          const unsigned long long end = std::min((unsigned long long)h_end_off[gi], s_hi[0]);
          if (end > early[0]) {
            const SlotCopy c{early[0], dev_out ? (uint64_t)(jobs[grp[0]].out - dev_out) + early[0] : 0, end - early[0]};
            if (dev_out)
              CU(copy_slots((const uint8_t *)g.d_out.p, dev_out, &c, 1, g.s_d2h));
            else
              CU(cudaMemcpyAsync(jobs[grp[0]].out + early[0], (uint8_t *)g.d_out.p + early[0], end - early[0], cudaMemcpyDeviceToHost,
                                 g.s_d2h));
            early[0] = end;
            any_early = true;
          }
        }
      }
      CU(cudaMemcpyAsync(h_off.data(), A.block_off, (size_t)(nc + 1) * 8, cudaMemcpyDeviceToHost, g.stream));
      CU(cudaMemcpyAsync(h_out.data(), A.block_out, (size_t)nc * 8, cudaMemcpyDeviceToHost, g.stream));
      CU(cudaMemcpyAsync(h_crc.data(), A.block_crc, (size_t)nc * 4, cudaMemcpyDeviceToHost, g.stream));
      CU(cudaMemcpyAsync(h_irr.data(), A.irregular, (size_t)nc * 4, cudaMemcpyDeviceToHost, g.stream));
      CU(cudaStreamSynchronize(g.stream));
      if (any_early) CU(cudaStreamSynchronize(g.s_d2h));  // (no copy into the caller's buffer outlives this call)
    }
    if (shard) {
      // one report per candidate of the range + one per end-of-stream candidate (every rank reports those)
      Bz2Job &j = jobs[grp[0]];
      const uint64_t total_bits = j.in_len * 8, base_bit = j.in_off * 8;
      shard->n_blocks = 0;
      auto push = [&](const b200z_bz2_block &b) {
        if (shard->n_blocks < shard->blocks_cap) shard->blocks[shard->n_blocks] = b;
        shard->n_blocks++;
      };
      for (uint32_t k = k_lo; k < k_hi; ++k) {
        b200z_bz2_block b{};
        b.start_bit = blk_bits[k] - base_bit;
        b.end_bit = h_end[k] - base_bit;
        b.status = h_st[k];
        b.flags = 0u;  // randomised blocks are decoded like the others (serial walk)
        b.crc_stored = blk_crc[k];
        const uint32_t c = chain_of[k];
        if (c != 0xffffffffu) {
          b.out_bytes = h_out[c];
          b.crc_calc = h_crc[c];
          if (h_irr[c] == 2) b.flags |= B200Z_BZ2_OVERRUN;
          else if (h_irr[c]) b.flags |= B200Z_BZ2_CORRUPT_CYCLE;
        }
        push(b);
      }
      for (uint32_t i = c_lo[grp[0]]; i < c_lo[grp[0] + 1]; ++i)
        if (cand[i] >> 63) {
          b200z_bz2_block b{};
          b.start_bit = cand[i] & POS;
          b.end_bit = b.start_bit + 80;
          b.flags = B200Z_BZ2_EOS;
          b.crc_stored = b.start_bit + 80 <= total_bits ? ccrc[i] : 0u;
          push(b);
        }
      const size_t n_local = nc ? (size_t)(h_off[nc - 1] + h_out[nc - 1]) : 0;
      j.out_len = n_local;
      if (shard->n_blocks > shard->blocks_cap) {
        set_err("bzip2 shard: %zu block reports, capacity %zu", shard->n_blocks, shard->blocks_cap);
        j.rc = B200Z_E_NOSPC;
      } else if (n_local > j.out_cap) {
        set_err("bzip2 shard: output needs %zu bytes, out_cap %zu", n_local, j.out_cap);
        j.rc = B200Z_E_NOSPC;
      } else if (n_local) {
        CU(cudaMemcpyAsync(j.out, g.d_out.p, n_local, cudaMemcpyDeviceToHost, g.stream));
      }
      CU(cudaStreamSynchronize(g.stream));
      continue;
    }
    // blocks are committed in order; the first bad one ends the stream (its bytes are already written when the
    // reference compares the CRC, :58-66)
    std::vector<SlotCopy> cp;
    for (size_t q = 0; q < G; ++q) {
      Bz2Job &j = jobs[grp[q]];
      int final_rc = s_rc[q];
      bool eos = have_eos[q] != 0;
      size_t n_out = 0;
      uint32_t combined = 0;
      for (uint32_t i = ch_lo[q]; i < ch_lo[q + 1]; ++i) {
        const uint32_t bi = i - ch_lo[q];
        if (h_irr[i] == 1) {
          set_err("bzip2: block %u: corrupt BWT cycle", bi);
          final_rc = B200Z_E_DATA;
          break;
        }
        n_out = (size_t)(h_off[i] + h_out[i] - s_lo[q]);
        if (h_irr[i] == 2) {  // the run-length walk overran the block (:497-499, :628-631): false, its bytes are already written
          set_err("bzip2: block %u: run overruns the block", bi);
          final_rc = B200Z_E_DATA;
          eos = false;
          break;
        }
        if (verify && h_crc[i] != stored_crc[i]) {
          set_err("bzip2: block %u CRC mismatch", bi);
          final_rc = B200Z_E_DATA;
          eos = false;
          break;
        }
        combined = ((combined << 1) | (combined >> 31)) ^ h_crc[i];
      }
      if (final_rc == B200Z_OK && eos && verify && eos_crc[q] != combined) {
        set_err("bzip2: combined CRC mismatch");
        final_rc = B200Z_E_DATA;
      }
      j.out_len = n_out;
      if (n_out > j.out_cap) {
        set_err("bzip2: output needs %zu bytes, out_cap %zu", n_out, j.out_cap);
        j.rc = B200Z_E_NOSPC;
        continue;
      }
      j.rc = final_rc;
      const size_t from = (size_t)(early[q] - s_lo[q]);
      if (n_out > from && dev_out)
        cp.push_back(SlotCopy{s_lo[q] + from, (uint64_t)(j.out - dev_out) + from, n_out - from});
      else if (n_out > from)
        CU(cudaMemcpyAsync(j.out + from, (uint8_t *)g.d_out.p + s_lo[q] + from, n_out - from, cudaMemcpyDeviceToHost, g.stream));
    }
    if (dev_out) CU(copy_slots((const uint8_t *)g.d_out.p, dev_out, cp.data(), cp.size(), g.stream));
    CU(cudaStreamSynchronize(g.stream));
  }
  return B200Z_OK;
}

}  // namespace b200z

// =============================================================================================
// Deflate(bytes, level:, windowBits:).getBytes() + crc32  (deflate.dart:25-100), and the encoder framing of
// _zlib_encoder_web.dart:27-73 / _gzip_encoder_web.dart:27-100
// =============================================================================================
namespace b200z {

// CRC-32 (reflected 0xEDB88320) combination, as in zlib's crc32_combine: crc(A||B) = crc(A) * x^(8|B|) + crc(B)
static uint32_t crc_multmodp(uint32_t a, uint32_t b) {
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = (b & 1) ? (b >> 1) ^ 0xEDB88320u : b >> 1;
  }
  return p;
}
static uint32_t crc_xpow8(uint64_t nbytes) {
  uint32_t p = 1u << 31;      // x^0
  uint32_t sq = 1u << 23;     // x^8 in the reflected representation (bit 31 = x^0)
  while (nbytes) {
    if (nbytes & 1) p = crc_multmodp(sq, p);
    sq = crc_multmodp(sq, sq);
    nbytes >>= 1;
  }
  return p;
}
static const uint32_t kCrcTile = 1u << 13;
// CRC-32 of d[0, n) on stream s: tile CRCs into d_part ((n / kCrcTile + 1) words of device memory), folded on the host
int device_crc32_on(const uint8_t *d, size_t n, uint32_t *d_part, cudaStream_t s, uint32_t *out) {
  const uint32_t TILE = kCrcTile;
  if (n == 0) {
    *out = 0;
    return B200Z_OK;
  }
  size_t tiles = (n + TILE - 1) / TILE;
  CU(crc32_tiles_device(d, n, TILE, d_part, s));
  std::vector<uint32_t> part(tiles);
  CU(cudaMemcpyAsync(part.data(), d_part, tiles * 4, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  uint32_t crc = part[0];
  const uint32_t xfull = crc_xpow8(TILE);
  for (size_t t = 1; t < tiles; ++t) {
    size_t len = (t + 1 == tiles) ? n - t * TILE : TILE;
    crc = crc_multmodp(len == TILE ? xfull : crc_xpow8(len), crc) ^ part[t];
  }
  *out = crc;
  return B200Z_OK;
}
static int device_crc32(const uint8_t *d, size_t n, uint32_t *out) {
  CU(g.d_small.reserve((n / kCrcTile + 1) * 4 + 256));
  return device_crc32_on(d, n, (uint32_t *)g.d_small.p, g.stream, out);
}

// the old deflate_stored (deflate.dart:691-737) touches no data: its block list follows from the length alone
// windowBits sets the window (deflate.dart:132-134) and with it where the blocks are cut: 2^windowBits - 262 bytes at most
static void stored_block_list(size_t n, int window_bits, std::vector<DeflStoredBlock> &out) {
  const long long w_size = 1ll << window_bits, window_size = 2 * w_size, min_lookahead = 262;
  const long long max_block_size = 65536 - 5 < 0xffff ? 65536 - 5 : 0xffff;
  long long strstart = 0, block_start = 0, lookahead = 0, base = 0;  // base: absolute position of window index 0
  long long in_pos = 0;
  auto flush = [&](bool eof) {
    // (block_start is never negative here: a block is flushed once it is w_size - min_lookahead long, and the window
    // slides only when strstart has reached 2 * w_size - min_lookahead, so the data is always still there to be stored)
    out.push_back({(uint32_t)(base + block_start), (uint32_t)(strstart - block_start), eof ? 1u : 0u});
    block_start = strstart;
  };
  auto fill_window = [&]() {
    do {
      long long more = window_size - lookahead - strstart;
      if (more == 0 && strstart == 0 && lookahead == 0) {
        more = w_size;
      } else if (strstart >= w_size + w_size - min_lookahead) {
        strstart -= w_size;
        block_start -= w_size;
        base += w_size;
        more += w_size;
      }
      if (in_pos >= (long long)n) return;
      long long len = (long long)n - in_pos;
      if (len > more) len = more;
      in_pos += len;
      lookahead += len;
    } while (lookahead < min_lookahead && in_pos < (long long)n);
  };
  for (;;) {
    if (lookahead <= 1) {
      fill_window();
      if (lookahead == 0) break;
    }
    strstart += lookahead;
    lookahead = 0;
    const long long max_start = block_start + max_block_size;
    if (strstart >= max_start) {
      lookahead = strstart - max_start;
      strstart = max_start;
      flush(false);
    }
    if (strstart - block_start >= w_size - min_lookahead) flush(false);
  }
  flush(true);
}

// compresses d_in[0, n) (already staged in g.d_in) into g.d_out; returns the compressed size
static int deflate_staged(size_t n, int level, int window_bits, size_t *out_len) {
  if (window_bits < 9 || window_bits > 15 || level < 0 || level > 9) {
    set_err("deflate: invalid level %d / windowBits %d (Dart: LateInitializationError)", level, window_bits);
    return B200Z_E_ARG;
  }
  if (n >= 0xffff0000ull) {
    set_err("deflate: inputs of 4 GiB and more are not supported");
    return B200Z_E_ARG;
  }
  const size_t cap = align_up(deflate_bound(n) + 16, 256);
  CU(g.d_out.reserve(cap));
  if (level == 0) {
    std::vector<DeflStoredBlock> bl;
    stored_block_list(n, window_bits, bl);
    const size_t ws = bl.size() * 64 + 1024;
    CU(g.d_ws.reserve(ws));
    CU(deflate_stored_device((const uint8_t *)g.d_in.p, bl.data(), (uint32_t)bl.size(), (uint8_t *)g.d_out.p, cap, g.d_ws.p,
                             g.d_ws.cap, out_len, g.stream));
    return B200Z_OK;
  }
  const size_t ws = deflate_workspace_bytes(n);
  CU(g.d_ws.reserve(ws));
  uint32_t stats[3];
  CU(deflate_slow_device((const uint8_t *)g.d_in.p, n, level, window_bits, (uint8_t *)g.d_out.p, cap, g.d_ws.p, g.d_ws.cap, out_len, stats,
                         g.stream));
  return B200Z_OK;
}

// ---------------------------------------------------------------------------------------------
// Many independent streams at once (ZipEncoder's members, zip_encoder.dart:185-259).  One stream's kernels are a chain
// with three host round trips (token count, block count, bit count) and, at levels 1-3, a single serial thread: a lone
// member leaves the device almost idle.  All inputs are staged with one burst of copies; `lanes` host threads then take
// members off a counter, each with its own CUDA stream, workspace and output slot, so the chains of different members
// overlap on the device.  Every member is compressed exactly as b200z_deflate_raw compresses it.
// ---------------------------------------------------------------------------------------------
static int deflate_member_on(const uint8_t *d_in, size_t n, int level, int window_bits, uint8_t *d_out, size_t cap, void *ws,
                             size_t ws_bytes, cudaStream_t s, size_t *out_len, uint32_t *crc, const DeflFastMember *pre = nullptr) {
  if (level == 0) {
    std::vector<DeflStoredBlock> bl;
    stored_block_list(n, window_bits, bl);
    CU(deflate_stored_device(d_in, bl.data(), (uint32_t)bl.size(), d_out, cap, ws, ws_bytes, out_len, s));
  } else {
    uint32_t stats[3];
    CU(deflate_slow_device(d_in, n, level, window_bits, d_out, cap, ws, ws_bytes, out_len, stats, s, pre));
  }
  // the tile CRCs go to the front of the workspace: the encoder is done with it (both paths end synchronised)
  return device_crc32_on(d_in, n, (uint32_t *)ws, s, crc);
}

// adler32, when given: every input's Adler-32 as well, from one launch over the staged inputs
static int deflate_batch_impl(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n_units, int level,
                              int window_bits, uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                              uint64_t *out_len, uint32_t *crc32, int32_t *status, uint32_t *adler32 = nullptr) {
  std::vector<size_t> din(n_units + 1), dout(n_units + 1);
  size_t ws_lane = 4096, acc_in = 0, acc_out = 0;
  for (size_t i = 0; i < n_units; ++i) {
    const size_t n = (size_t)in_len[i];
    if (n >= 0xffff0000ull) {
      set_err("deflate_batch: unit %zu: inputs of 4 GiB and more are not supported", i);
      return B200Z_E_ARG;
    }
    din[i] = acc_in;
    dout[i] = acc_out;
    acc_in += align_up(n + 64, 256);
    acc_out += align_up(deflate_bound(n) + 16, 256);
    size_t ws = (n / kCrcTile + 1) * 4 + 256;
    if (level == 0) {
      std::vector<DeflStoredBlock> bl;
      stored_block_list(n, window_bits, bl);
      ws = std::max(ws, bl.size() * 64 + 1024);
    } else {
      ws = std::max(ws, deflate_workspace_bytes(n));
    }
    ws_lane = std::max(ws_lane, align_up(ws, 256));
  }
  din[n_units] = acc_in;
  dout[n_units] = acc_out;
  size_t lanes = Ctx::kCompStreams;
  if (const char *e = getenv("B200Z_DEFLATE_LANES")) lanes = (size_t)atoi(e);
  lanes = std::max<size_t>(1, std::min<size_t>(std::min<size_t>(lanes, Ctx::kCompStreams), n_units));
  CU(g.d_in.reserve(acc_in + 64));
  CU(g.d_out.reserve(acc_out + 64));
  CU(g.d_ws.reserve(lanes * ws_lane));
  cudaEvent_t staged;
  CU(cudaEventCreateWithFlags(&staged, cudaEventDisableTiming));
  CU(cudaMemsetAsync(g.d_in.p, 0, acc_in, g.s_h2d));  // the bytes behind every member read as zeros (as in deflate_raw)
  for (size_t i = 0; i < n_units; ++i)
    if (in_len[i])
      CU(cudaMemcpyAsync((uint8_t *)g.d_in.p + din[i], in_base + in_off[i], (size_t)in_len[i], cudaMemcpyHostToDevice, g.s_h2d));
  CU(cudaEventRecord(staged, g.s_h2d));
  std::atomic<size_t> next{0};
  size_t next_end = n_units;  // the lanes take members [next, next_end)
  std::vector<int> lane_rc(lanes, B200Z_OK);
  std::vector<std::string> lane_err(lanes);
  std::vector<DeflFastMember> pre;  // levels 1-3: where the batch kernel has put every member's tokens
  const int device = g.device;
  auto lane = [&](size_t l) {
    auto fail = [&](int rc) {
      lane_rc[l] = rc;
      lane_err[l] = t_err;
      next.store(n_units);  // the other lanes stop taking members
    };
    if (cudaSetDevice(device) != cudaSuccess) return fail(B200Z_E_NODEVICE);  // a new thread starts on device 0
    cudaStream_t s = g.s_comp[l];
    if (cudaStreamWaitEvent(s, staged, 0) != cudaSuccess) return fail(B200Z_E_NODEVICE);
    void *ws = (uint8_t *)g.d_ws.p + l * ws_lane;
    for (;;) {
      const size_t i = next.fetch_add(1);
      if (i >= next_end) break;
      size_t olen = 0;
      uint32_t crc = 0;
      const int rc = deflate_member_on((const uint8_t *)g.d_in.p + din[i], (size_t)in_len[i], level, window_bits,
                                       (uint8_t *)g.d_out.p + dout[i], dout[i + 1] - dout[i], ws, ws_lane, s, &olen, &crc,
                                       pre.empty() || in_len[i] == 0 ? nullptr : &pre[i]);
      if (rc) return fail(rc);
      out_len[i] = olen;
      if (crc32) crc32[i] = crc;
      if (olen > out_cap[i]) {
        status[i] = B200Z_U_NOSPC;
        continue;
      }
      status[i] = B200Z_OK;
      if (olen && cudaMemcpyAsync(out_base + out_off[i], (uint8_t *)g.d_out.p + dout[i], olen, cudaMemcpyDeviceToHost, s) !=
                      cudaSuccess)
        return fail(B200Z_E_NODEVICE);
    }
    if (cudaStreamSynchronize(s) != cudaSuccess) fail(B200Z_E_NODEVICE);
  };
  auto run_lanes = [&]() {
    if (lanes == 1) {
      lane(0);
    } else {
      std::vector<std::thread> th;
      for (size_t l = 1; l < lanes; ++l) th.emplace_back(lane, l);
      lane(0);
      for (auto &t : th) t.join();
    }
  };
  if (level >= 1 && level <= 3) {
    // _deflateFast is one serial chain per member; the batch is the parallel axis: ONE launch makes the tokens of a whole
    // group of members (a warp per member, deflate_kernels.cu: k_defl_fast_batch), then the lanes cut the blocks, build
    // the trees and emit the bits of each.  A group is as many members as the token store holds (12 bytes per input
    // byte; B200Z_DEFLATE_TOK_MB, default 49152).
    size_t budget = (size_t)48 << 30;
    {
      size_t free_b = 0, total_b = 0;  // (never more than 60 % of what the device has free right now)
      if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess && free_b) budget = std::min(budget, free_b / 10 * 6 + g.d_tok.cap);
    }
    if (const char *e = getenv("B200Z_DEFLATE_TOK_MB")) budget = std::max<size_t>(1, (size_t)atoll(e)) << 20;
    pre.assign(n_units, DeflFastMember());
    size_t lo = 0;
    auto failed = [&]() {
      for (size_t l = 0; l < lanes; ++l)
        if (lane_rc[l]) return true;
      return false;
    };
    while (lo < n_units && !failed()) {
      size_t hi = lo, bytes = 256;
      std::vector<size_t> off;
      while (hi < n_units) {
        const size_t need = align_up(((size_t)in_len[hi] + 2) * 4, 256) * 3 + 256;
        if (hi > lo && bytes + need > budget) break;
        off.push_back(bytes);
        bytes += need;
        hi++;
      }
      const size_t list_off = align_up(bytes, 256);
      bytes = list_off + (hi - lo) * sizeof(DeflFastMember);
      CU(g.d_tok.reserve(bytes));
      std::vector<DeflFastMember> order;
      for (size_t i = lo; i < hi; ++i) {
        const size_t n = (size_t)in_len[i], a = align_up((n + 2) * 4, 256);
        uint8_t *base = (uint8_t *)g.d_tok.p + off[i - lo];
        DeflFastMember m;
        m.d = (const uint8_t *)g.d_in.p + din[i];
        m.n = (uint32_t)n;
        m.tok = (uint32_t *)base;
        m.tally_ss = (uint32_t *)(base + a);
        m.next_ss = (uint32_t *)(base + 2 * a);
        m.ntok = (uint32_t *)(base + 3 * a);
        pre[i] = m;
        if (n) order.push_back(m);
      }
      std::stable_sort(order.begin(), order.end(), [](const DeflFastMember &x, const DeflFastMember &y) { return x.n > y.n; });
      if (!order.empty()) {
        CU(cudaStreamWaitEvent(g.stream, staged, 0));
        CU(cudaMemcpyAsync((uint8_t *)g.d_tok.p + list_off, order.data(), order.size() * sizeof(DeflFastMember),
                           cudaMemcpyHostToDevice, g.stream));
        CU(deflate_fast_tokens_batch((const DeflFastMember *)((uint8_t *)g.d_tok.p + list_off), (uint32_t)order.size(), level,
                                     window_bits, (uint32_t *)g.d_tok.p, g.stream));
        CU(cudaStreamSynchronize(g.stream));
      }
      next.store(lo);
      next_end = hi;
      run_lanes();
      lo = hi;
    }
  } else {
    run_lanes();
  }
  cudaEventDestroy(staged);
  for (size_t l = 0; l < lanes; ++l)
    if (lane_rc[l]) {
      set_err("deflate_batch: %s", lane_err[l].empty() ? "a lane failed" : lane_err[l].c_str());
      return lane_rc[l];
    }
  if (adler32) {
    const std::vector<uint64_t> off(din.begin(), din.end() - 1);
    return device_adler32_many((const uint8_t *)g.d_in.p, off.data(), in_len, n_units, adler32);
  }
  return B200Z_OK;
}

// The framing GZipEncoder / ZLibEncoder write around the DEFLATE bytes.  Header (_gzip_encoder_web.dart:77-90): magic,
// deflate, flags 0, MTIME, XFL 0, OS 255; trailer: CRC-32 and ISIZE, little-endian.
static void gzip_put_header(uint8_t *o, uint32_t mtime) {
  o[0] = 0x1f; o[1] = 0x8b; o[2] = 8; o[3] = 0;
  for (int i = 0; i < 4; ++i) o[4 + i] = (uint8_t)(mtime >> (8 * i));
  o[8] = 0; o[9] = 255;
}
static void gzip_put_trailer(uint8_t *o, uint32_t crc, size_t n) {
  for (int i = 0; i < 4; ++i) o[i] = (uint8_t)(crc >> (8 * i));
  for (int i = 0; i < 4; ++i) o[4 + i] = (uint8_t)((uint32_t)n >> (8 * i));
}
// CMF / FLG with FLEVEL 0 for every level (_zlib_encoder_web.dart:44-60, quirk Q4); the Adler-32 behind is big-endian
static void zlib_put_header(uint8_t *o, int window_bits) {
  int wb = window_bits < 0 ? 0 : window_bits > 15 ? 15 : window_bits;
  int cmf = ((wb - 8) << 4) | 8, flag = 0, fcheck = 0;
  while ((cmf * 256 + (flag | fcheck)) % 31 != 0) fcheck++;
  o[0] = (uint8_t)cmf;
  o[1] = (uint8_t)(flag | fcheck);
}
static void zlib_put_adler(uint8_t *o, uint32_t ad) {
  o[0] = (uint8_t)(ad >> 24); o[1] = (uint8_t)(ad >> 16); o[2] = (uint8_t)(ad >> 8); o[3] = (uint8_t)ad;
}

// n inputs (arguments, level and windowBits checked) encoded as b200z_gzip_encode (gzip) or b200z_zlib_encode give each
// alone: one deflate batch whose raw DEFLATE goes behind the header inside each slot; CRC-32 from the batch, Adler-32 from
// one launch; the host writes the headers and trailers.
static int gzip_zlib_encode_streams(bool gzip, const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n,
                                    int level, int window_bits, int raw, uint32_t mtime, uint8_t *out_base,
                                    const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len, int32_t *rc) {
  const size_t hdr = gzip ? 10 : raw ? 0 : 2, trl = gzip ? 8 : raw ? 0 : 4;
  std::vector<size_t> idx;
  for (size_t i = 0; i < n; ++i) {
    if (in_len[i] >= 0xffff0000ull) {  // deflate_staged's limit
      rc[i] = B200Z_E_ARG;
      out_len[i] = 0;
    } else {
      idx.push_back(i);
    }
  }
  const size_t m = idx.size();
  if (m == 0) return B200Z_OK;
  std::vector<uint64_t> io(m), il(m), oo(m), oc(m), ol(m);
  std::vector<uint32_t> crc(m), ad(m);
  std::vector<int32_t> st(m);
  for (size_t k = 0; k < m; ++k) {
    const size_t i = idx[k];
    io[k] = in_off[i];
    il[k] = in_len[i];
    oo[k] = out_off[i] + hdr;
    oc[k] = out_cap[i] >= hdr + trl ? out_cap[i] - hdr - trl : 0;
  }
  const int r = deflate_batch_impl(in_base, io.data(), il.data(), m, level, window_bits, out_base, oo.data(), oc.data(), ol.data(),
                                   crc.data(), st.data(), !gzip && !raw ? ad.data() : nullptr);
  if (r) return r;
  for (size_t k = 0; k < m; ++k) {
    const size_t i = idx[k];
    out_len[i] = ol[k] + hdr + trl;
    if (st[k] != B200Z_OK) {
      rc[i] = B200Z_E_NOSPC;
      continue;
    }
    uint8_t *o = out_base + out_off[i];
    if (gzip) {
      gzip_put_header(o, mtime);
      gzip_put_trailer(o + hdr + ol[k], crc[k], (size_t)il[k]);
    } else if (!raw) {
      zlib_put_header(o, window_bits);
      zlib_put_adler(o + hdr + ol[k], ad[k]);
    }
    rc[i] = B200Z_OK;
  }
  return B200Z_OK;
}

}  // namespace b200z

using namespace b200z;

// =============================================================================================
// C ABI
// =============================================================================================

// ---------------------------------------------------------------------------------------------
// ZIP container (SURVEY.md 8f2): directory parse on the host, members as ONE inflate batch
// ---------------------------------------------------------------------------------------------
static inline uint64_t le64(const uint8_t *p) { return (uint64_t)le32(p) | ((uint64_t)le32(p + 4) << 32); }

// ZipDirectory._findSignature (zip_directory.dart:139-182): 1024-byte chunks from the end, each scanned backwards; a
// signature that straddles two chunks, or lies in the last 4 bytes, is not seen.
static long long zip_find_eocd(const uint8_t *z, size_t len) {
  if (len <= 4) return -1;
  const long long length = (long long)len - 4;
  const long long chunk = length < 1024 ? length : 1024;
  long long start = length - chunk;
  while (start >= 0) {
    for (long long cp = chunk - 4; cp >= 0; --cp)
      if (le32(z + start + cp) == 0x06054b50u) return start + cp;
    if (start > 0 && start < chunk) start = 0;
    else start -= chunk;
  }
  return -1;
}

extern "C" int b200z_zip_list(const uint8_t *z, size_t len, b200z_zip_entry *entries, size_t cap, size_t *n_entries) {
  if (n_entries) *n_entries = 0;
  if (!z && len) return B200Z_E_ARG;
  const long long fp = zip_find_eocd(z, len);
  if (fp < 0) return B200Z_OK;  // ZipDirectory.read returns with no headers (zip_directory.dart:26-29)
  // (overflow-safe: positions and sizes come from the archive as full 64-bit values)
#define ZNEED_IN(pos, k, lim)                                                       \
  if ((unsigned long long)(pos) > (unsigned long long)(lim) ||                      \
      (unsigned long long)(k) > (unsigned long long)(lim) - (unsigned long long)(pos)) { \
    set_err("zip: read past the end at %llu (Dart: RangeError)", (unsigned long long)(pos)); \
    return B200Z_E_THROW;                                                          \
  }
#define ZNEED(pos, k) ZNEED_IN(pos, k, len)
  ZNEED(fp, 22);
  uint64_t cd_size = le32(z + fp + 12), cd_off = le32(z + fp + 16);
  {
    const size_t clen = le16(z + fp + 20);
    ZNEED(fp + 22, clen);  // the comment is read (readString) before the zip64 records are looked at
  }
  // _readZip64Data :65-137
  if (fp >= 20 && le32(z + fp - 20) == 0x07064b50u) {
    const uint64_t z64 = le64(z + fp - 20 + 8);
    if (z64 <= len && len - z64 >= 4 && le32(z + z64) == 0x06064b50u) {
      ZNEED(z64, 56);
      cd_size = le64(z + z64 + 40);
      cd_off = le64(z + z64 + 48);
    } else if (z64 > len || len - z64 < 4) {
      ZNEED(z64, 4);
    }
  }
  // central directory :50-63
  size_t n = 0;
  uint64_t p = cd_off;
  // dirContent = input.subset(position: offset, length: size) (input_memory_stream.dart:15-27,111-119): a length that
  // reaches beyond the archive is cut to what is there; an offset beyond it, or a negative (>= 2^63) offset or size, makes
  // Uint8List.view throw.  The headers are then read from that sub-stream: running over ITS end throws.
  if (cd_off > len || (cd_size >> 63) != 0) {
    set_err("zip: central directory at %llu (+%llu) lies outside the archive (Dart: RangeError)", (unsigned long long)cd_off,
            (unsigned long long)cd_size);
    return B200Z_E_THROW;
  }
  const uint64_t cd_end = cd_size > len - cd_off ? (uint64_t)len : cd_off + cd_size;
#define DNEED(pos, k) ZNEED_IN(pos, k, cd_end)
  while (p < cd_end) {
    DNEED(p, 4);
    if (le32(z + p) != 0x02014b50u) break;
    DNEED(p, 46);
    // ZipFileHeader.read (zip_file_header.dart:28-111)
    const uint8_t *h = z + p;
    b200z_zip_entry e;
    memset(&e, 0, sizeof e);
    e.version_made_by = le16(h + 4);
    uint64_t comp = le32(h + 20), uncomp = le32(h + 24), lho = le32(h + 42);
    const size_t fn_len = le16(h + 28), ex_len = le16(h + 30), cm_len = le16(h + 32);
    uint32_t disk = le16(h + 34);
    e.ext_attr = le32(h + 38);
    DNEED(p + 46, fn_len + ex_len + cm_len);
    e.cd_name_off = p + 46;
    e.cd_name_len = (uint32_t)fn_len;
    if (ex_len >= 4) {  // :48-98 -- shorter extra fields are ignored
      const uint8_t *x = h + 46 + fn_len;
      size_t xo = 0;
      while (ex_len - xo >= 4) {
        const uint32_t id = le16(x + xo);
        size_t size = le16(x + xo + 2);
        xo += 4;
        if (xo + size > ex_len) {
          set_err("zip: extra field overruns its record (Dart: RangeError)");
          return B200Z_E_THROW;
        }
        if (id == 1) {
          size_t q = xo;
          if (size >= 8 && uncomp == 0xffffffffu) { uncomp = le64(x + q); q += 8; size -= 8; }
          if (size >= 8 && comp == 0xffffffffu) { comp = le64(x + q); q += 8; size -= 8; }
          if (size >= 8 && lho == 0xffffffffu) { lho = le64(x + q); q += 8; size -= 8; }
          if (size >= 4 && disk == 0xffffu) { disk = le32(x + q); q += 4; size -= 4; }
          xo = q + size;
        } else {
          xo += size;
        }
      }
    }
    (void)disk;
    p += 46 + fn_len + ex_len + cm_len;
    // ZipFile.read at the local header (zip_file.dart:73-149)
    e.local_header_off = lho;
    e.comp_size = comp;
    e.uncomp_size = uncomp;
    e.hint_uncomp_size = uncomp;
    ZNEED(lho, 4);
    if (le32(z + lho) == 0x04034b50u) {
      ZNEED(lho, 30);
      const uint8_t *l = z + lho;
      e.flags = le16(l + 6);
      e.method = le16(l + 8);
      e.mod_time = le16(l + 10);
      e.mod_date = le16(l + 12);
      e.crc32 = le32(l + 14);
      const size_t lfn = le16(l + 26), lex = le16(l + 28);
      ZNEED(lho + 30, lfn + lex);
      e.name_off = lho + 30;
      e.name_len = (uint32_t)lfn;
      e.data_off = lho + 30 + lfn + lex;
      e.has_data = 1;
      if ((comp >> 63) != 0) {  // readBytes(negative count): Uint8List.view throws
        set_err("zip: compressed size %llu (Dart: RangeError)", (unsigned long long)comp);
        return B200Z_E_THROW;
      }
      if (comp > len - e.data_off) {  // readBytes hands out what is there (data_off <= len: checked above)
        e.comp_size = len - e.data_off;
      }
      if (e.flags & 0x08) {  // data descriptor :137-148: CRC and the 32-bit sizes are replaced by what follows the data
        uint64_t q = e.data_off + e.comp_size;
        ZNEED(q, 4);
        const uint32_t sig_or_crc = le32(z + q);
        q += 4;
        if (sig_or_crc == 0x08074b50u) {
          ZNEED(q, 4);
          e.crc32 = le32(z + q);
          q += 4;
        } else {
          e.crc32 = sig_or_crc;
        }
        ZNEED(q, 8);
        e.uncomp_size = le32(z + q + 4);
      }
    }
    if (n < cap && entries) entries[n] = e;
    n++;
  }
#undef DNEED
#undef ZNEED
#undef ZNEED_IN
  if (n_entries) *n_entries = n;
  if (n > cap && entries) {
    set_err("zip: %zu entries, capacity %zu", n, cap);
    return B200Z_E_NOSPC;
  }
  return B200Z_OK;
}

// ZipDirectory.zipFileComment (zip_directory.dart:41-44): byte range of the archive comment, or length 0
extern "C" int b200z_zip_comment(const uint8_t *z, size_t len, uint64_t *off, uint32_t *clen) {
  if (off) *off = 0;
  if (clen) *clen = 0;
  const long long fp = zip_find_eocd(z, len);
  if (fp < 0) return B200Z_OK;
  if ((unsigned long long)fp + 22 > len) {
    set_err("zip: read past the end at %lld (Dart: RangeError)", fp);
    return B200Z_E_THROW;
  }
  const uint32_t n = le16(z + fp + 20);
  if ((unsigned long long)fp + 22 + n > len) {
    set_err("zip: comment overruns the archive (Dart: RangeError)");
    return B200Z_E_THROW;
  }
  if (off) *off = (uint64_t)fp + 22;
  if (clen) *clen = n;
  return B200Z_OK;
}

// Encrypted members after decryption (b200z_zip_extract_password): their plaintext sits in g.d_in behind the archive, and
// the entries handed to zip_extract_core point there.
struct ZipPlain {
  size_t staged;       // bytes of g.d_in in use: the archive, then the plaintext area
  size_t archive_len;  // of which the archive (the bytes the host holds)
};

// (test hooks) last b200z_zip_extract call's K12 batch: members offered, accepted, fell back, redo rounds, batches; kernel
// times as g_ck_ms.  Caps on the streams of one batch and on each stream's pool pages (0: none, the built-in share).
static unsigned long long g_zck_stats[5];
static double g_zck_ms[3];
static uint32_t g_zck_max_streams = 0, g_zck_max_pages = 0;

// K12 for the large ZIP members (zip_extract_core): every unit that is a whole deflate member of g_ck.thresh compressed
// bytes or more is decoded by K12 from exactly the input view its unit has, straight to its place in the output.  All
// of them go through one K12 batch, or several when their pools do not fit: each member's pool is what its exact-path
// workspace would be (ck_pages_for), and a batch takes at most the buffer K12 already has plus half the free device
// memory.  Accepted members leave the unit list (their out_len is set here, their status stays B200Z_U_DONE); a member
// K12 declines stays in the list at its place and the exact path decodes it as if K12 had never run.
static int zip_chunked(const uint8_t *z, size_t len, const b200z_zip_entry *entries, const ZipPlain *pl,
                       std::vector<uint64_t> &u_in_off, std::vector<uint32_t> &u_in_len, std::vector<uint64_t> &u_out_off,
                       std::vector<uint32_t> &u_cap, std::vector<uint32_t> &u_idx, uint64_t *out_len) {
  const size_t host_len = pl ? pl->archive_len : len;
  std::vector<size_t> big;
  for (size_t k = 0; k < u_idx.size(); ++k)  // (a split member's pieces carry the 0x80000000 mark or start behind data_off)
    if (!(u_idx[k] & 0x80000000u) && u_in_off[k] == entries[u_idx[k]].data_off && u_in_len[k] >= g_ck.thresh) big.push_back(k);
  if (big.empty()) return B200Z_OK;
  size_t budget = g.d_ws.cap, free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess) budget += free_b / 2;
  std::vector<char> taken(u_idx.size(), 0);
  std::vector<std::vector<uint8_t>> h_plain;  // host copies of decrypted members (their bytes live on the device only)
  std::vector<CkIn> batch;
  std::vector<size_t> at;
  std::vector<CkOut> res;
  for (size_t b = 0; b < big.size();) {
    batch.clear();
    at.clear();
    h_plain.clear();
    size_t pages = 0;
    for (; b < big.size(); ++b) {
      const size_t k = big[b];
      uint32_t np = ck_pages_for(workspace_bytes(1, u_cap[k]));
      if (g_zck_max_pages) np = std::min(np, g_zck_max_pages);
      if (!batch.empty() && ((g_zck_max_streams && batch.size() >= g_zck_max_streams) ||
                             CkLayout(batch.size() + 1, pages + np).bytes > budget))
        break;
      if (np == 0 || CkLayout(1, np).bytes > budget) {  // no pool, or not even on its own: left to the exact path
        g_zck_stats[0]++;
        g_zck_stats[2]++;
        continue;
      }
      const uint8_t *h = z + u_in_off[k];
      if (u_in_off[k] + u_in_len[k] > host_len) {
        h_plain.emplace_back(u_in_len[k]);
        CU(cudaMemcpyAsync(h_plain.back().data(), (const uint8_t *)g.d_in.p + u_in_off[k], u_in_len[k], cudaMemcpyDeviceToHost,
                           g.stream));
        h = h_plain.back().data();
      }
      batch.push_back(CkIn{h, (size_t)u_in_off[k], u_in_len[k], (size_t)u_out_off[k], u_cap[k], 0, np});
      at.push_back(k);
      pages += np;
    }
    if (batch.empty()) continue;
    CU(cudaStreamSynchronize(g.stream));
    const int rc = run_chunked(batch, res, g_zck_ms);
    if (rc) return rc;
    g_zck_stats[4]++;
    for (size_t q = 0; q < batch.size(); ++q) {
      g_zck_stats[0]++;
      g_zck_stats[3] += res[q].stats[2];
      if (!res[q].accepted) {
        g_zck_stats[2]++;
        continue;
      }
      g_zck_stats[1]++;
      out_len[u_idx[at[q]]] = res[q].r.out_len;
      taken[at[q]] = 1;
    }
  }
  size_t m = 0;
  for (size_t k = 0; k < u_idx.size(); ++k) {
    if (taken[k]) continue;
    u_in_off[m] = u_in_off[k];
    u_in_len[m] = u_in_len[k];
    u_out_off[m] = u_out_off[k];
    u_cap[m] = u_cap[k];
    u_idx[m] = u_idx[k];
    m++;
  }
  u_in_off.resize(m);
  u_in_len.resize(m);
  u_out_off.resize(m);
  u_cap.resize(m);
  u_idx.resize(m);
  return B200Z_OK;
}

static uint64_t g_zip_out_bytes = 0;  // (test hook) g.d_out bytes the last ZIP extract asked for

// ZipFile.getStream for all members (g.mu held).  pl == nullptr: the archive is not staged yet and `len` is its size;
// otherwise `len` = pl->staged and everything is in g.d_in already.  Deflate, stored and K12 members decode into g.d_out,
// which holds the slots' span [lo, hi) only (offset out_off[i] - lo); dev_out: `out` is device memory, and the bytes go
// from g.d_out into the slots with one k_copy_slots launch instead of the copies of [lo, hi) to the host.
static int zip_extract_core(const uint8_t *z, size_t len, const b200z_zip_entry *entries, size_t n, uint8_t *out,
                            size_t out_cap, const uint64_t *out_off, const uint64_t *out_room, uint64_t *out_len,
                            int32_t *status, uint32_t flags, const ZipPlain *pl, bool dev_out) {
  int rc = B200Z_OK;
  // members: deflate -> one inflate batch; stored (and unknown methods, which the reference treats as stored,
  // zip_file.dart:83) -> device copies; bzip2 -> one BZip2 batch, afterwards
  std::vector<uint64_t> u_in_off, u_out_off;
  std::vector<uint32_t> u_in_len, u_cap, u_idx;
  std::vector<size_t> bz_idx;
  uint64_t lo = ~0ull, hi = 0;
  for (size_t i = 0; i < n; ++i) {
    const b200z_zip_entry &e = entries[i];
    out_len[i] = 0;
    status[i] = B200Z_U_DONE;
    if (!e.has_data) continue;
    if (e.flags & 1u) {
      status[i] = B200Z_ZIP_ENCRYPTED;
      continue;
    }
    if (out_off[i] > out_cap || out_room[i] > out_cap - out_off[i] || e.data_off > len || e.comp_size > len - e.data_off) {
      set_err("zip_extract: entry %zu lies outside the buffers", i);
      return B200Z_E_ARG;
    }
    if (e.method == 8 || e.method == 12) {
      if (e.comp_size > 0xfffffff0ull || out_room[i] > 0xfffffff0ull) {
        status[i] = B200Z_ZIP_TOO_LARGE;
        continue;
      }
    }
    if (e.method == 12) {
      bz_idx.push_back(i);
      continue;
    }
    if (out_room[i]) {
      lo = out_off[i] < lo ? out_off[i] : lo;
      hi = out_off[i] + out_room[i] > hi ? out_off[i] + out_room[i] : hi;
    }
    if (e.method == 8) {
      // ZipFile.getStream: ZLibDecoder().decodeBytes(compressed, raw: true) on exactly the member's bytes.  On the Dart
      // VM that is dart:io's zlib; the pure-Dart Inflate wants maxCodeLength bits after the last code (SURVEY Q1) and
      // so can drop the last symbols of such a stream.  Default: what the VM gives -- a few bytes that follow the
      // member are made readable so the lookahead is satisfied; B200Z_ZIP_WEB_EOS: the pure-Dart behaviour.
      uint64_t pad = 0;
      if (!(flags & B200Z_ZIP_WEB_EOS)) {
        pad = len - (e.data_off + e.comp_size);
        if (pad > 8) pad = 8;
      }
      u_in_off.push_back(e.data_off);
      u_in_len.push_back((uint32_t)(e.comp_size + pad));
      u_out_off.push_back(out_off[i]);
      u_cap.push_back((uint32_t)out_room[i]);
      u_idx.push_back((uint32_t)i);
    }
  }
  const bool any_dev = hi > lo;
  if (!any_dev) lo = hi = 0;
  // units live at out_off - lo in g.d_out; a unit without room may name any offset, and keeps its order among the others
  for (auto &o : u_out_off) o = std::min(std::max(o, lo), hi) - lo;
  g_zip_out_bytes = 0;
  if (any_dev || !u_idx.empty() || !bz_idx.empty()) {
    if (!pl) {
      rc = stage_input(z, len);
      if (rc) return rc;
    }
    CU(cudaMemsetAsync((uint8_t *)g.d_in.p + len, 0, 64, g.stream));
    g_zip_out_bytes = std::max<uint64_t>(hi - lo, 1) + 64;
    CU(g.d_out.reserve(g_zip_out_bytes));
  }
  for (size_t i = 0; i < n; ++i) {
    const b200z_zip_entry &e = entries[i];
    if (!e.has_data || (e.flags & 1u) || e.method == 8 || e.method == 12) continue;
    uint64_t k = e.comp_size < out_room[i] ? e.comp_size : out_room[i];
    if (k) CU(cudaMemcpyAsync((uint8_t *)g.d_out.p + (out_off[i] - lo), (const uint8_t *)g.d_in.p + e.data_off, k, cudaMemcpyDeviceToDevice, g.stream));
    out_len[i] = e.comp_size;
    if (e.comp_size > out_room[i]) status[i] = B200Z_U_NOSPC;
  }
  // ---- flush points: a member that was written with Z_FULL_FLUSH every so often is many independent raw DEFLATE
  // streams back to back (each ends with the byte-aligned empty stored block 00 00 FF FF and restarts the window).
  // Candidates are found by a byte scan and PROVEN by a sizing pass (count-only decode of every piece: a piece must end
  // exactly on its marker at a block boundary and must not reach back before its own start -- which also rejects
  // Z_SYNC_FLUSH points, whose window continues); a member with any doubtful piece is decoded whole.
  if (!u_idx.empty() && !(flags & B200Z_ZIP_NO_SPLIT)) {
    bool worth = false;
    for (size_t k = 0; k < u_idx.size(); ++k) worth = worth || u_in_len[k] >= (256u << 10);
    if (worth) {
      const uint32_t ccap = 1u << 22;
      CU(g.d_small.reserve((size_t)ccap * 8 + 256));
      unsigned long long *d_list = (unsigned long long *)((uint8_t *)g.d_small.p + 256);
      uint32_t *d_cnt = (uint32_t *)g.d_small.p;
      CU(launch_find_markers((const uint8_t *)g.d_in.p, len, d_list, d_cnt, ccap, g.stream));
      uint32_t ncand = 0;
      CU(cudaMemcpyAsync(&ncand, d_cnt, 4, cudaMemcpyDeviceToHost, g.stream));
      CU(cudaStreamSynchronize(g.stream));
      if (ncand > 0 && ncand <= ccap) {
        std::vector<unsigned long long> cand(ncand);
        CU(cudaMemcpy(cand.data(), d_list, (size_t)ncand * 8, cudaMemcpyDeviceToHost));
        std::sort(cand.begin(), cand.end());
        // pieces of every big member
        std::vector<uint64_t> s_in_off, s_out_off;
        std::vector<uint32_t> s_in_len, s_cap, s_member, first_seg(u_idx.size() + 1, 0);
        for (size_t k = 0; k < u_idx.size(); ++k) {
          first_seg[k] = (uint32_t)s_in_off.size();
          if (u_in_len[k] < (256u << 10)) continue;
          const uint64_t a0 = u_in_off[k], a1 = a0 + entries[u_idx[k]].comp_size, aend = a0 + u_in_len[k];
          auto it = std::upper_bound(cand.begin(), cand.end(), a0);
          uint64_t start = a0;
          size_t pieces = 0;
          for (; it != cand.end() && *it < a1; ++it) {
            if (*it - start < 4096) continue;  // not worth a unit of its own
            s_in_off.push_back(start);
            s_in_len.push_back((uint32_t)(*it - start));
            s_member.push_back((uint32_t)k);
            start = *it;
            pieces++;
          }
          if (pieces == 0) continue;
          s_in_off.push_back(start);
          s_in_len.push_back((uint32_t)(aend - start));
          s_member.push_back((uint32_t)k);
        }
        first_seg[u_idx.size()] = (uint32_t)s_in_off.size();
        const size_t ns = s_in_off.size();
        if (ns) {
          s_out_off.assign(ns, 0);
          s_cap.assign(ns, 0xfffffff0u);
          std::vector<uint32_t> a_len(ns), a_used(ns);
          std::vector<int32_t> a_st(ns);
          rc = run_batch_on_staged(s_in_off.data(), s_in_len.data(), s_out_off.data(), s_cap.data(), a_len.data(), a_st.data(),
                                   a_used.data(), ns, 0, true);
          if (rc) return rc;
          // rebuild the unit list: proven members contribute their pieces, the others stay whole
          std::vector<uint64_t> n_in_off, n_out_off;
          std::vector<uint32_t> n_in_len, n_cap, n_idx;
          for (size_t k = 0; k < u_idx.size(); ++k) {
            const uint32_t f = first_seg[k], l = first_seg[k + 1];
            bool ok = l > f;
            uint64_t total = 0;
            for (uint32_t q = f; q < l && ok; ++q) {
              const bool last = q + 1 == l;
              ok = last ? (a_st[q] == B200Z_U_DONE) : (a_st[q] == B200Z_U_EOS && a_used[q] == s_in_len[q]);
              total += a_len[q];
            }
            ok = ok && total <= u_cap[k];
            if (!ok) {
              n_in_off.push_back(u_in_off[k]); n_in_len.push_back(u_in_len[k]); n_out_off.push_back(u_out_off[k]);
              n_cap.push_back(u_cap[k]); n_idx.push_back(u_idx[k]);
              continue;
            }
            uint64_t o = u_out_off[k];
            for (uint32_t q = f; q < l; ++q) {
              n_in_off.push_back(s_in_off[q]); n_in_len.push_back(s_in_len[q]); n_out_off.push_back(o);
              n_cap.push_back(a_len[q]); n_idx.push_back(u_idx[k] | (q + 1 == l ? 0u : 0x80000000u));
              o += a_len[q];
            }
          }
          u_in_off.swap(n_in_off); u_in_len.swap(n_in_len); u_out_off.swap(n_out_off); u_cap.swap(n_cap); u_idx.swap(n_idx);
        }
      }
    }
  }
  for (auto &v : g_zck_stats) v = 0;
  for (auto &v : g_zck_ms) v = 0;
  if (!u_idx.empty()) {
    rc = zip_chunked(z, len, entries, pl, u_in_off, u_in_len, u_out_off, u_cap, u_idx, out_len);
    if (rc) return rc;
  }
  size_t early_to = (size_t)lo;  // output bytes [lo, early_to) are on their way to the host already (copy stream)
  if (!u_idx.empty()) {
    const size_t m = u_idx.size();
    std::vector<uint32_t> r_len(m), r_used(m);
    std::vector<int32_t> r_st(m);
    // A large archive is decoded in chunks of units (in output order), and the bytes of a finished chunk -- with the stored
    // members that lie between its units -- go to the host on the copy stream while the next chunk is decoded
    // (B200Z_ZIP_CHUNKS, default 8 from 512 MiB of output on; 1: one batch, one copy at the end).  Device slots have no
    // PCIe copy to hide: one batch by default, and chunks (when asked for) deliver nothing early.
    size_t nchunks = !dev_out && (hi - lo) >= ((size_t)512 << 20) ? 8 : 1;
    if (const char *ce = getenv("B200Z_ZIP_CHUNKS")) nchunks = (size_t)std::max(1, atoi(ce));
    for (size_t k = 1; k < m && nchunks > 1; ++k)
      if (u_out_off[k] < u_out_off[k - 1]) nchunks = 1;  // (units are made in output order; if ever not, no early copies)
    if (nchunks > m) nchunks = m;
    for (size_t c = 0, k0 = 0; c < nchunks; ++c) {
      const size_t k1 = m * (c + 1) / nchunks;
      if (k1 == k0) continue;
      rc = run_batch_on_staged(u_in_off.data() + k0, u_in_len.data() + k0, u_out_off.data() + k0, u_cap.data() + k0, r_len.data() + k0,
                               r_st.data() + k0, r_used.data() + k0, k1 - k0, (size_t)(hi - lo));
      if (rc) {
        if (early_to > lo) cudaStreamSynchronize(g.s_d2h);
        return rc;
      }
      const size_t end = k1 < m ? (size_t)(lo + u_out_off[k1]) : (size_t)hi;
      if (nchunks > 1 && !dev_out && end > early_to && end <= hi) {
        CU(cudaMemcpyAsync(out + early_to, (const uint8_t *)g.d_out.p + (early_to - lo), end - early_to, cudaMemcpyDeviceToHost,
                           g.s_d2h));
        early_to = end;
      }
      k0 = k1;
    }
    for (size_t k = 0; k < m; ++k) {
      const uint32_t i = u_idx[k] & 0x7fffffffu;
      const bool inner = (u_idx[k] & 0x80000000u) != 0;  // a piece that is not the member's last
      out_len[i] += r_len[k];
      if (!inner) {
        if (status[i] == B200Z_U_DONE) status[i] = r_st[k];
      } else if (!(r_st[k] == B200Z_U_EOS && r_len[k] == u_cap[k])) {
        status[i] = r_st[k] == B200Z_U_EOS || r_st[k] == B200Z_U_DONE ? B200Z_U_STOP : r_st[k];  // cannot happen after the sizing pass
      }
    }
  }
  if (any_dev && dev_out) {  // each member's bytes into its slot, one k_copy_slots launch for all of them
    std::vector<SlotCopy> cp;
    for (size_t i = 0; i < n; ++i) {
      const b200z_zip_entry &e = entries[i];
      const uint64_t k = std::min(out_len[i], out_room[i]);
      if (e.has_data && !(e.flags & 1u) && e.method != 12 && k) cp.push_back(SlotCopy{out_off[i] - lo, out_off[i], k});
    }
    CU(copy_slots((const uint8_t *)g.d_out.p, out, cp.data(), cp.size(), g.stream));
    CU(cudaStreamSynchronize(g.stream));
  } else if (any_dev) {
    if (hi > early_to)
      CU(cudaMemcpyAsync(out + early_to, (const uint8_t *)g.d_out.p + (early_to - lo), hi - early_to, cudaMemcpyDeviceToHost,
                         g.stream));
    CU(cudaStreamSynchronize(g.stream));
    if (early_to > lo) CU(cudaStreamSynchronize(g.s_d2h));
  }
  if (!bz_idx.empty()) {  // BZip2Decoder().decodeStream(_rawContent, output) (zip_file.dart:189-192,239-245), all members at once
    std::vector<Bz2Job> jobs(bz_idx.size());
    for (size_t k = 0; k < bz_idx.size(); ++k) {
      const size_t i = bz_idx[k];
      jobs[k] = Bz2Job{entries[i].data_off, entries[i].comp_size, out + out_off[i], (size_t)out_room[i], 0, B200Z_OK};
    }
    rc = bzip2_decode_device((const uint8_t *)g.d_in.p, jobs.data(), jobs.size(), 0, nullptr, dev_out ? out : nullptr);
    if (rc) return rc;
    for (size_t k = 0; k < bz_idx.size(); ++k) {
      const size_t i = bz_idx[k];
      const int r = jobs[k].rc;
      out_len[i] = jobs[k].out_len;
      status[i] = r == B200Z_OK ? B200Z_U_DONE : r == B200Z_E_NOSPC ? B200Z_U_NOSPC : r == B200Z_E_THROW ? B200Z_U_THROW : B200Z_U_STOP;
    }
  }
  return B200Z_OK;
}

// ---------------------------------------------------------------------------------------------
// Encrypted ZIP members (zip_file.dart:98-130 read, :164-216 getStream, :260-359 ZipCrypto / AES)
// ---------------------------------------------------------------------------------------------
// ZipFile.read :98-130: flag bit 0 means ZipCrypto, unless the LOCAL extra field is longer than 2 bytes and holds id 0x9901.
// The scan reads 16-bit ids at 2-byte steps and never skips the payload of another id (the reference's loop, kept as is);
// a read past the end of the extra field throws there.
static int zip_crypt_info_impl(const uint8_t *z, size_t len, const b200z_zip_entry *e, uint32_t *mode, uint32_t *strength,
                               uint32_t *method) {
  *mode = B200Z_ZIP_CRYPT_NONE;
  *strength = 0;
  *method = e->method;
  if (!e->has_data || !(e->flags & 1u)) return B200Z_OK;
  *mode = B200Z_ZIP_CRYPT_ZIPCRYPTO;
  const uint64_t x0 = e->name_off + e->name_len;
  if (x0 > e->data_off || e->data_off > len) {
    set_err("zip_crypt_info: entry does not lie inside the archive");
    return B200Z_E_ARG;
  }
  const uint64_t xl = e->data_off - x0;
  if (xl <= 2) return B200Z_OK;
  const uint8_t *x = z + x0;
  uint64_t q = 0;
  bool past = false;  // a read ran over the end of the extra field
  while (q < xl && !past) {
    if (xl - q < 2) {
      past = true;
      break;
    }
    const uint32_t id = le16(x + q);
    q += 2;
    if (id != 0x9901u) continue;
    q += 4;                             // dataSize, vendorVersion
    q = q + 2 > xl ? (q > xl ? q : xl) : q + 2;  // readString(size: 2): readBytes hands out what is there
    if (q > xl || xl - q < 3) {        // strength (1 byte) and compression method (2 bytes)
      past = true;
      break;
    }
    *mode = B200Z_ZIP_CRYPT_AES;
    *strength = x[q];
    *method = le16(x + q + 1);
    q += 3;
  }
  if (past) {
    set_err("zip: the scan of the AES extra field reads past its end (Dart: RangeError)");
    return B200Z_E_THROW;
  }
  return B200Z_OK;
}

static double g_crypt_ms[4];  // last call: PBKDF2, CTR, MAC, ZipCrypto kernel times (b200z_debug_zip_crypt_ms)

struct CryptEvents {  // CUDA events around the kernels: PBKDF2 [0,1], CTR [2,3], MAC [2,5] (it may start at 2), ZipCrypto [6,7]
  cudaEvent_t ev[8] = {};
  bool used[4] = {};
  CryptEvents() {
    for (auto &e : ev) cudaEventCreate(&e);
  }
  ~CryptEvents() {
    for (auto &e : ev)
      if (e) cudaEventDestroy(e);
  }
};

static inline uint32_t aes_salt_len(uint32_t strength) { return strength == 1 ? 8 : strength == 2 ? 12 : 16; }

// tiles of k_zip_aes_ctr over the members with len > 0
static void ctr_tiles(const std::vector<ZipAesMember> &m, std::vector<ZipCtrTile> &t) {
  const uint64_t tb = zip_ctr_tile_blocks();
  t.clear();
  for (size_t k = 0; k < m.size(); ++k) {
    const uint64_t blocks = (m[k].len + 15) / 16;
    for (uint64_t b = 0; b < blocks; b += tb) t.push_back(ZipCtrTile{b, (uint32_t)k, 0});
  }
}

// device layout of the crypt metadata in g.d_crypt
struct CryptLayout {
  size_t members, dk, rk, ver, mac, tiles, zc, bytes;
  CryptLayout(size_t na, size_t nt, size_t nz) {
    size_t o = 0;
    members = o; o = align_up(o + na * sizeof(ZipAesMember), 256);
    dk = o;      o = align_up(o + na * 80, 256);
    rk = o;      o = align_up(o + na * 240, 256);
    ver = o;     o = align_up(o + na * 2, 256);
    mac = o;     o = align_up(o + na * 10, 256);
    tiles = o;   o = align_up(o + nt * sizeof(ZipCtrTile), 256);
    zc = o;      o = align_up(o + nz * sizeof(ZipCryptoMember), 256);
    bytes = o + 256;
  }
};

static int zip_extract_crypt(const uint8_t *z, size_t len, const b200z_zip_entry *entries, size_t n, uint8_t *out,
                             size_t out_cap, const uint64_t *out_off, const uint64_t *out_room, uint64_t *out_len,
                             int32_t *status, uint32_t flags, const uint8_t *pw, size_t pw_len, bool dev_out) {
  // 1. which members are encrypted how, and where their plaintext goes: the plaintext area starts behind the archive in
  //    g.d_in, every member is followed by >= 64 zero bytes (the inflate look-ahead reads zeros, as the oracle's does)
  std::vector<b200z_zip_entry> ve(entries, entries + n);
  std::vector<int32_t> forced(n, 1);  // 1: none; otherwise the member's final status (out_len 0)
  std::vector<ZipAesMember> aes;
  std::vector<uint32_t> aes_idx;
  std::vector<ZipCryptoMember> zc;
  size_t p = align_up(len + 64, 256);
  for (size_t i = 0; i < n; ++i) {
    const b200z_zip_entry &e = entries[i];
    if (!e.has_data || !(e.flags & 1u)) continue;
    if (e.data_off > len || e.comp_size > len - e.data_off) {
      set_err("zip_extract: entry %zu lies outside the buffers", i);
      return B200Z_E_ARG;
    }
    uint32_t mode, strength, method;
    const int ci = zip_crypt_info_impl(z, len, &e, &mode, &strength, &method);
    if (ci == B200Z_E_ARG) return ci;
    ve[i].flags &= ~1u;
    ve[i].method = method;
    if (ci != B200Z_OK) {  // ZipFile.read throws for this member
      forced[i] = B200Z_U_THROW;
      ve[i].has_data = 0;
      continue;
    }
    if (e.comp_size == 0) continue;  // :170-171: an empty member is not decrypted; it is an empty member of its method
    uint64_t plen;
    if (mode == B200Z_ZIP_CRYPT_ZIPCRYPTO) {
      if (e.comp_size < 12) {  // _decodeZipCrypto: readByte past the end
        forced[i] = B200Z_U_THROW;
        ve[i].has_data = 0;
        continue;
      }
      plen = e.comp_size - 12;
      zc.push_back(ZipCryptoMember{e.data_off, p, e.comp_size});
    } else {
      const uint32_t sl = aes_salt_len(strength);
      if (e.comp_size < sl + 12 || pw_len == 0) {  // readBytes(input.length - 10) < 0; deriveKey('') -> sublist throws
        forced[i] = B200Z_U_THROW;
        ve[i].has_data = 0;
        continue;
      }
      plen = e.comp_size - sl - 12;
      ZipAesMember m;
      memset(&m, 0, sizeof m);
      m.src_off = e.data_off + sl + 2;
      m.dst_off = p;
      m.len = plen;
      m.salt_len = sl;
      m.key_len = 2 * sl;
      memcpy(m.salt, z + e.data_off, sl);
      aes.push_back(m);
      aes_idx.push_back((uint32_t)i);
    }
    ve[i].data_off = p;
    ve[i].comp_size = plen;
    p = align_up(p + plen + 64, 256);
  }
  if (aes.empty() && zc.empty()) {
    int rc = zip_extract_core(z, len, ve.data(), n, out, out_cap, out_off, out_room, out_len, status, flags, nullptr, dev_out);
    for (size_t i = 0; i < n && rc == B200Z_OK; ++i)
      if (forced[i] != 1) {
        status[i] = forced[i];
        out_len[i] = 0;
      }
    return rc;
  }
  // 2. stage the archive once; the plaintext area is zeroed
  const size_t staged = p;
  CU(g.d_in.reserve(staged + 64));
  uint8_t *d_base = (uint8_t *)g.d_in.p;
  CU(cudaMemcpyAsync(d_base, z, len, cudaMemcpyHostToDevice, g.stream));
  CU(cudaMemsetAsync(d_base + len, 0, staged + 64 - len, g.stream));
  std::vector<ZipCtrTile> tiles;
  const uint32_t na = (uint32_t)aes.size(), nz = (uint32_t)zc.size();
  // tiles are counted for every member: the verifier check below can only shrink the list
  ctr_tiles(aes, tiles);
  const CryptLayout cl(na, tiles.size(), nz);
  CU(g.d_crypt.reserve(cl.bytes));
  uint8_t *dc = (uint8_t *)g.d_crypt.p;
  CryptEvents ev;
  std::vector<uint8_t> macs(na * 10);
  cudaStream_t s_mac = g.s_comp[0];
  // 3. AES: key derivation, verifier check on the host, then the MAC (second stream) and the CTR pass
  if (na) {
    ZipHmacPads pads;
    zip_hmac_pads(pw, pw_len, &pads);
    CU(cudaMemcpyAsync(dc + cl.members, aes.data(), na * sizeof(ZipAesMember), cudaMemcpyHostToDevice, g.stream));
    CU(cudaEventRecord(ev.ev[0], g.stream));
    CU(zip_launch_pbkdf2((const ZipAesMember *)(dc + cl.members), na, pads, dc + cl.dk, (uint32_t *)(dc + cl.rk), dc + cl.ver,
                         g.stream));
    CU(cudaEventRecord(ev.ev[1], g.stream));
    ev.used[0] = true;
    std::vector<uint8_t> ver(na * 2);
    CU(cudaMemcpyAsync(ver.data(), dc + cl.ver, na * 2, cudaMemcpyDeviceToHost, g.stream));
    CU(cudaStreamSynchronize(g.stream));
    bool any_bad = false;
    for (uint32_t k = 0; k < na; ++k) {
      const b200z_zip_entry &e = entries[aes_idx[k]];
      if (memcmp(ver.data() + 2 * k, z + e.data_off + aes[k].salt_len, 2) != 0) {  // Exception('password error')
        forced[aes_idx[k]] = B200Z_ZIP_BAD_PASSWORD;
        ve[aes_idx[k]].has_data = 0;
        aes[k].len = 0;
        any_bad = true;
      }
    }
    if (any_bad) {
      ctr_tiles(aes, tiles);
      CU(cudaMemcpyAsync(dc + cl.members, aes.data(), na * sizeof(ZipAesMember), cudaMemcpyHostToDevice, g.stream));
    }
    CU(cudaMemcpyAsync(dc + cl.tiles, tiles.data(), tiles.size() * sizeof(ZipCtrTile), cudaMemcpyHostToDevice, g.stream));
    CU(cudaEventRecord(ev.ev[2], g.stream));  // the MAC stream starts once the key material and the member list are there
    CU(cudaStreamWaitEvent(s_mac, ev.ev[2], 0));
    CU(zip_launch_hmac((const ZipAesMember *)(dc + cl.members), na, dc + cl.dk, d_base, false, dc + cl.mac, s_mac));
    CU(cudaEventRecord(ev.ev[5], s_mac));
    ev.used[2] = true;
    CU(zip_launch_aes_ctr((const ZipAesMember *)(dc + cl.members), (const uint32_t *)(dc + cl.rk), (const ZipCtrTile *)(dc + cl.tiles),
                          (uint32_t)tiles.size(), d_base, g.stream));
    CU(cudaEventRecord(ev.ev[3], g.stream));
    ev.used[1] = true;
  }
  // 4. ZipCrypto
  if (nz) {
    uint32_t keys[3];
    zipcrypto_keys(pw, pw_len, keys);
    CU(cudaMemcpyAsync(dc + cl.zc, zc.data(), nz * sizeof(ZipCryptoMember), cudaMemcpyHostToDevice, g.stream));
    CU(cudaEventRecord(ev.ev[6], g.stream));
    CU(zip_launch_zipcrypto((const ZipCryptoMember *)(dc + cl.zc), nz, keys, d_base, g.stream));
    CU(cudaEventRecord(ev.ev[7], g.stream));
    ev.used[3] = true;
  }
  // 5. every member kind sees the decrypted members as ranges of the staged buffer
  const ZipPlain pl{staged, len};
  int rc = zip_extract_core(z, staged, ve.data(), n, out, out_cap, out_off, out_room, out_len, status, flags, &pl, dev_out);
  if (rc) {
    cudaStreamSynchronize(s_mac);
    return rc;
  }
  // 6. the MACs: HMAC-SHA1 of the ciphertext, first 10 bytes, against the 10 bytes that end the member
  if (na) {
    CU(cudaStreamSynchronize(s_mac));
    CU(cudaMemcpy(macs.data(), dc + cl.mac, na * 10, cudaMemcpyDeviceToHost));
    for (uint32_t k = 0; k < na; ++k) {
      const uint32_t i = aes_idx[k];
      if (forced[i] != 1) continue;
      const b200z_zip_entry &e = entries[i];
      if (memcmp(macs.data() + 10 * k, z + e.data_off + e.comp_size - 10, 10) != 0) forced[i] = B200Z_ZIP_BAD_MAC;
    }
  }
  CU(cudaStreamSynchronize(g.stream));
  {
    float ms = 0;
    g_crypt_ms[0] = ev.used[0] && cudaEventElapsedTime(&ms, ev.ev[0], ev.ev[1]) == cudaSuccess ? ms : 0.0;
    g_crypt_ms[1] = ev.used[1] && cudaEventElapsedTime(&ms, ev.ev[2], ev.ev[3]) == cudaSuccess ? ms : 0.0;
    g_crypt_ms[2] = ev.used[2] && cudaEventElapsedTime(&ms, ev.ev[2], ev.ev[5]) == cudaSuccess ? ms : 0.0;
    g_crypt_ms[3] = ev.used[3] && cudaEventElapsedTime(&ms, ev.ev[6], ev.ev[7]) == cudaSuccess ? ms : 0.0;
  }
  for (size_t i = 0; i < n; ++i)
    if (forced[i] != 1) {
      status[i] = forced[i];
      out_len[i] = 0;
    }
  return B200Z_OK;
}

extern "C" int b200z_zip_crypt_info(const uint8_t *zip, size_t zip_len, const b200z_zip_entry *entry, uint32_t *mode,
                                    uint32_t *aes_strength, uint32_t *method) {
  if (!entry || !mode || !aes_strength || !method || (!zip && zip_len)) return B200Z_E_ARG;
  return zip_crypt_info_impl(zip, zip_len, entry, mode, aes_strength, method);
}

extern "C" int b200z_zip_extract_password(const uint8_t *z, size_t len, const b200z_zip_entry *entries, size_t n, uint8_t *out,
                                          size_t out_cap, const uint64_t *out_off, const uint64_t *out_room, uint64_t *out_len,
                                          int32_t *status, uint32_t flags, const uint8_t *password, size_t password_len) {
  int rc = require_init();
  if (rc) return rc;
  if (n == 0) return B200Z_OK;
  if (!entries || !out_off || !out_room || !out_len || !status) return B200Z_E_ARG;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  if (!password)
    return zip_extract_core(z, len, entries, n, out, out_cap, out_off, out_room, out_len, status, flags, nullptr, false);
  return zip_extract_crypt(z, len, entries, n, out, out_cap, out_off, out_room, out_len, status, flags, password, password_len,
                           false);
}

// crc32[i] = getCrc32 of the bytes member i delivered, d_out[out_off[i], + min(out_len[i], out_room[i])) (0 for a
// B200Z_U_NOSPC member): the 8 KiB tiles of all members in one k_crc_tiles launch, folded per member on the host
static int zip_slot_crc32(const uint8_t *d_out, const uint64_t *out_off, const uint64_t *out_room, const uint64_t *out_len,
                          const int32_t *status, size_t n, uint32_t *crc32) {
  const uint64_t TILE = kCrcTile;
  std::vector<uint64_t> t_off;
  std::vector<uint32_t> t_len;
  std::vector<size_t> first(n + 1, 0);
  for (size_t i = 0; i < n; ++i) {
    first[i] = t_off.size();
    const uint64_t k = status[i] == B200Z_U_NOSPC ? 0 : std::min(out_len[i], out_room[i]);
    for (uint64_t o = 0; o < k; o += TILE) {
      t_off.push_back(out_off[i] + o);
      t_len.push_back((uint32_t)std::min(TILE, k - o));
    }
  }
  first[n] = t_off.size();
  const size_t nt = t_off.size();
  std::vector<uint32_t> part(nt);
  if (nt) {
    const size_t o_len = align_up(nt * 8, 256), o_part = align_up(o_len + nt * 4, 256);
    CU(g.d_small.reserve(o_part + nt * 4));
    uint8_t *m = (uint8_t *)g.d_small.p;
    CU(cudaMemcpyAsync(m, t_off.data(), nt * 8, cudaMemcpyHostToDevice, g.stream));
    CU(cudaMemcpyAsync(m + o_len, t_len.data(), nt * 4, cudaMemcpyHostToDevice, g.stream));
    CU(crc32_tiles_launch(d_out, (const uint64_t *)m, (const uint32_t *)(m + o_len), (uint32_t)nt, (uint32_t *)(m + o_part),
                          g.stream));
    CU(cudaMemcpyAsync(part.data(), m + o_part, nt * 4, cudaMemcpyDeviceToHost, g.stream));
    CU(cudaStreamSynchronize(g.stream));
  }
  const uint32_t xfull = crc_xpow8(TILE);
  for (size_t i = 0; i < n; ++i) {
    uint32_t c = 0;  // the CRC of nothing
    for (size_t t = first[i]; t < first[i + 1]; ++t) c = crc_multmodp(t_len[t] == TILE ? xfull : crc_xpow8(t_len[t]), c) ^ part[t];
    crc32[i] = c;
  }
  return B200Z_OK;
}

extern "C" int b200z_zip_extract_to_device(const uint8_t *z, size_t len, const b200z_zip_entry *entries, size_t n,
                                           uint8_t *d_out, size_t out_cap, const uint64_t *out_off, const uint64_t *out_room,
                                           uint64_t *out_len, int32_t *status, uint32_t *crc32, uint32_t flags,
                                           const uint8_t *password, size_t password_len, void *cuda_stream) {
  int rc = require_init();
  if (rc) return rc;
  if (n == 0) return B200Z_OK;
  if (!entries || !out_off || !out_room || !out_len || !status) return B200Z_E_ARG;
  if ((rc = device_out_arg("zip_extract_to_device", d_out, n, out_room)) != B200Z_OK) return rc;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  if ((rc = wait_for_caller(cuda_stream)) != B200Z_OK) return rc;
  // results go to the caller's arrays only once the call has succeeded, so that an argument error writes nothing
  std::vector<uint64_t> r_len(n);
  std::vector<int32_t> r_st(n);
  std::vector<uint32_t> r_crc(crc32 ? n : 0);
  rc = password ? zip_extract_crypt(z, len, entries, n, d_out, out_cap, out_off, out_room, r_len.data(), r_st.data(), flags,
                                    password, password_len, true)
                : zip_extract_core(z, len, entries, n, d_out, out_cap, out_off, out_room, r_len.data(), r_st.data(), flags,
                                   nullptr, true);
  if (rc == B200Z_OK && crc32) rc = zip_slot_crc32(d_out, out_off, out_room, r_len.data(), r_st.data(), n, r_crc.data());
  if (rc) return rc;
  memcpy(out_len, r_len.data(), n * 8);
  memcpy(status, r_st.data(), n * 4);
  if (crc32) memcpy(crc32, r_crc.data(), n * 4);
  return B200Z_OK;
}

// (test hook) the g.d_out bytes the last b200z_zip_extract* call asked for: the slots' span, not their end
extern "C" uint64_t b200z_debug_zip_out_bytes(void) { return g_zip_out_bytes; }

// ---------------------------------------------------------------------------------------------
// TAR member walk (b200z_tar_walk_device): TarDecoder._decode's loop with storeData (tar_decoder.dart:28-38) and the
// position arithmetic of TarFile.read (tar_file.dart:74-118, input_memory_stream.dart:96-119).  A header's size field
// says where the next header is, so the walk is a dependent chain of loads, one per member.  One warp per archive: the
// bytes a member's step needs (the first two, the size field and the type byte) are one load per lane, then every lane
// parses the field the same way and lane 0 writes the record.
// ---------------------------------------------------------------------------------------------
constexpr unsigned TAR_THREADS = 128;
static cudaEvent_t g_tar_ev[2] = {nullptr, nullptr};  // created once, kept for the life of the library
static double g_tar_walk_ms = 0;  // k_tar_walk of the last call, by CUDA events (b200z_debug_tar_walk)
struct TarArchive {
  uint64_t off, len;  // the archive, from the call's d_base
  uint64_t rec;       // its first record slot in the workspace (the prefix sum of the bounds len / 512 + 1)
};
struct TarCount {
  uint64_t count, first;  // members, and where they start in the gathered area
  int32_t rc, pad_;
};

__device__ __forceinline__ uint32_t tar_fb(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t i) {
  return ((i < 4 ? w0 : i < 8 ? w1 : w2) >> (8 * (i & 3))) & 0xffu;
}
// a three-byte UTF-8 form of a character Dart's trim removes: U+1680, U+2000-200A, U+2028/9, U+202F, U+205F, U+3000, U+FEFF
__device__ __forceinline__ bool tar_ws3(uint32_t a, uint32_t b, uint32_t c) {
  return (a == 0xE1 && b == 0x9A && c == 0x80) ||
         (a == 0xE2 && b == 0x80 && ((c >= 0x80 && c <= 0x8A) || c == 0xA8 || c == 0xA9 || c == 0xAF)) ||
         (a == 0xE2 && b == 0x81 && c == 0x9F) || (a == 0xE3 && b == 0x80 && c == 0x80) || (a == 0xEF && b == 0xBB && c == 0xBF);
}
__device__ __forceinline__ bool tar_ascii_ws(uint32_t c) { return c == 0x20 || (c >= 0x09 && c <= 0x0D); }

// _parseInt (tar_file.dart:211-225) of the field's first n bytes (already cut at the first NUL): decoded as UTF-8 when the
// bytes are valid UTF-8 (Python's strict decoder: no overlong forms, surrogates or code points past U+10FFFF), else as
// Latin-1; Dart's trim at both ends; then int.parse(radix: 8), which takes [+-]?[0-7]+ and nothing else (0 otherwise)
__device__ int64_t tar_parse_size(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t n) {
  bool utf8 = true;
  for (uint32_t i = 0; i < n && utf8;) {
    const uint32_t c = tar_fb(w0, w1, w2, i);
    if (c < 0x80) {
      ++i;
      continue;
    }
    const uint32_t need = c < 0xC2 ? 0 : c < 0xE0 ? 1 : c < 0xF0 ? 2 : c < 0xF5 ? 3 : 0;
    if (need == 0 || i + need >= n) {  // not a lead byte, or the sequence is cut short
      utf8 = false;
      break;
    }
    const uint32_t lo = c == 0xE0 ? 0xA0 : c == 0xF0 ? 0x90 : 0x80, hi = c == 0xED ? 0x9F : c == 0xF4 ? 0x8F : 0xBF;
    const uint32_t c1 = tar_fb(w0, w1, w2, i + 1);
    utf8 = c1 >= lo && c1 <= hi;
    for (uint32_t k = 2; k <= need && utf8; ++k) {
      const uint32_t ck = tar_fb(w0, w1, w2, i + k);
      utf8 = ck >= 0x80 && ck <= 0xBF;
    }
    i += need + 1;
  }
  uint32_t l = 0, r = n;
  while (l < r) {  // the left end
    const uint32_t c = tar_fb(w0, w1, w2, l);
    uint32_t k = 0;
    if (tar_ascii_ws(c)) k = 1;
    else if (!utf8) k = c == 0x85 || c == 0xA0 ? 1 : 0;
    else if (c == 0xC2 && l + 1 < r) k = tar_fb(w0, w1, w2, l + 1) == 0x85 || tar_fb(w0, w1, w2, l + 1) == 0xA0 ? 2 : 0;
    else if (l + 2 < r && tar_ws3(c, tar_fb(w0, w1, w2, l + 1), tar_fb(w0, w1, w2, l + 2))) k = 3;
    if (k == 0) break;
    l += k;
  }
  while (r > l) {  // the right end (valid UTF-8: a lead byte at r - 2 or r - 3 starts the last character)
    const uint32_t c = tar_fb(w0, w1, w2, r - 1);
    uint32_t k = 0;
    if (tar_ascii_ws(c)) k = 1;
    else if (!utf8) k = c == 0x85 || c == 0xA0 ? 1 : 0;
    else if (r - l >= 2 && tar_fb(w0, w1, w2, r - 2) == 0xC2 && (c == 0x85 || c == 0xA0)) k = 2;
    else if (r - l >= 3 && tar_ws3(tar_fb(w0, w1, w2, r - 3), tar_fb(w0, w1, w2, r - 2), c)) k = 3;
    if (k == 0) break;
    r -= k;
  }
  bool neg = false;
  if (l < r) {
    const uint32_t c = tar_fb(w0, w1, w2, l);
    if (c == '+' || c == '-') {
      neg = c == '-';
      ++l;
    }
  }
  if (l >= r) return 0;  // nothing, or a sign alone
  int64_t v = 0;
  for (uint32_t i = l; i < r; ++i) {
    const uint32_t c = tar_fb(w0, w1, w2, i);
    if (c < '0' || c > '7') return 0;
    v = v * 8 + (c - '0');  // at most 12 digits: below 2^36
  }
  return neg ? -v : v;
}

// rec: the records at each archive's bound slots.  When its walk ends, the warp takes the next count slots of the gathered
// area (one atomicAdd on *next) and writes a k_copy_slots piece for each header there: from d_from + off + header_off
// (d_from: d_base from the launch's source base) to slot * 512.
__global__ void __launch_bounds__(TAR_THREADS) k_tar_walk(const uint8_t *__restrict__ base, const TarArchive *__restrict__ ar,
                                                          uint32_t n, b200z_tar_member *__restrict__ rec, TarCount *__restrict__ res,
                                                          SlotCopy *__restrict__ pieces, unsigned long long *__restrict__ next,
                                                          uint64_t d_from) {
  const uint32_t lane = threadIdx.x & 31, w = blockIdx.x * (TAR_THREADS / 32) + (threadIdx.x >> 5);
  if (w >= n) return;  // (the whole warp)
  const TarArchive a = ar[w];
  const uint8_t *D = base + a.off;
  const uint64_t L = a.len, bound = L / 512 + 1;
  b200z_tar_member *R = rec + a.rec;
  // lanes 0-11: the size field (header bytes 124-135); lane 12: the type byte (156); lanes 13, 14: the first two bytes
  const uint32_t at = lane < 12 ? 124 + lane : lane == 12 ? 156 : lane - 13;
  uint64_t pos = 0, k = 0;
  int32_t st = B200Z_OK;
  while (pos < L) {
    const uint64_t left = L - pos;
    const int b = lane < 15 && at < left ? (int)D[pos + at] : -1;  // -1: past the archive's end
    const int b0 = __shfl_sync(0xffffffffu, b, 13), b1 = __shfl_sync(0xffffffffu, b, 14);
    if (b1 < 0 || (b0 == 0 && b1 == 0)) break;  // one byte left, or two zero bytes: the end (tar_decoder.dart:35-38)
    if (k == bound) {  // (cannot happen: every member but the last takes 512 bytes or more)
      st = B200Z_E_INTERNAL;
      break;
    }
    const uint32_t hl = left < 512 ? (uint32_t)left : 512;
    // the field: the bytes present, cut at the first NUL
    const uint32_t present = __ballot_sync(0xffffffffu, lane < 12 && b >= 0), nul = __ballot_sync(0xffffffffu, lane < 12 && b == 0);
    uint32_t fl = __popc(present);
    if (nul) fl = min(fl, (uint32_t)(__ffs(nul) - 1));
    const uint32_t v = b > 0 ? (uint32_t)b : 0;
    uint32_t wd[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      uint32_t x = 0;
#pragma unroll
      for (int q = 0; q < 4; ++q) x |= __shfl_sync(0xffffffffu, v, 4 * j + q) << (8 * q);
      wd[j] = x;
    }
    const int64_t size = tar_parse_size(wd[0], wd[1], wd[2], fl);
    if (size < 0) {  // readBytes of a negative count: RangeError
      st = B200Z_E_THROW;
      break;
    }
    const uint64_t content_off = pos + hl, clen = min((uint64_t)size, L - content_off);
    if (lane == 0) {
      b200z_tar_member m;
      m.header_off = pos;
      m.content_off = content_off;
      m.content_len = clen;
      m.size = size;
      m.header_len = hl;
      m.pad_ = 0;
      R[k] = m;
    }
    ++k;
    pos = content_off + clen;
    const int type = __shfl_sync(0xffffffffu, b, 12);
    if (type != '5' && size % 512 != 0) pos = min(pos + 512 - (uint64_t)(size % 512), L);  // (size 0: no padding)
  }
  unsigned long long first = 0;
  if (lane == 0) first = atomicAdd(next, (unsigned long long)k);
  first = __shfl_sync(0xffffffffu, first, 0);
  __syncwarp();  // (lane 0's records, read back by every lane)
  for (uint64_t j = lane; j < k; j += 32)
    pieces[first + j] = SlotCopy{d_from + a.off + R[j].header_off, (first + j) * 512, R[j].header_len};
  if (lane == 0) {
    res[w].count = k;
    res[w].first = first;
    res[w].rc = st;
    res[w].pad_ = 0;
  }
}

extern "C" int b200z_tar_walk_device(const uint8_t *d_base, const uint64_t *off, const uint64_t *len, size_t n,
                                     b200z_tar_member *members, uint8_t *headers, size_t cap, uint64_t *first, uint64_t *count,
                                     int32_t *rc, size_t *n_total, void *cuda_stream) {
  int r = require_init();
  if (r) return r;
  if (n == 0) {
    if (n_total) *n_total = 0;
    return B200Z_OK;
  }
  if (!off || !len || !first || !count || !rc || !n_total || (cap && (!members || !headers))) {
    set_err("tar_walk_device: null array");
    return B200Z_E_ARG;
  }
  uint64_t n_rec = 0;  // the record bound of the call
  for (size_t i = 0; i < n; ++i) {
    if (off[i] + len[i] < off[i] || (len[i] && !d_base)) {
      set_err("tar_walk_device: archive %zu: bad range", i);
      return B200Z_E_ARG;
    }
    for (int end = 0; end < 2 && len[i]; ++end) {  // the archive's first and last byte
      cudaPointerAttributes pa;
      if (cudaPointerGetAttributes(&pa, d_base + off[i] + (end ? len[i] - 1 : 0)) != cudaSuccess ||
          pa.type != cudaMemoryTypeDevice || pa.device != g.device) {
        cudaGetLastError();
        set_err("tar_walk_device: archive %zu is not in device memory of device %d", i, g.device);
        return B200Z_E_ARG;
      }
    }
    n_rec += len[i] / 512 + 1;
  }
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  if ((r = wait_for_caller(cuda_stream))) return r;
  // g.d_ws: the archive table and the gathered-slot counter (one upload), the per-archive counts, the records at their
  // bound slots, and the k_copy_slots pieces: one per member's header, then the records' pieces (one per archive and per
  // COPY_PIECE bytes of records: at most n + n_rec * 40 / COPY_PIECE of them)
  const size_t o_next = n * sizeof(TarArchive), o_cnt = align_up(o_next + 8, 256);
  const size_t o_rec = o_cnt + align_up(n * sizeof(TarCount), 256);
  const size_t o_pc = o_rec + align_up(n_rec * sizeof(b200z_tar_member), 256);
  const size_t ws_bytes = o_pc + (n_rec + n + n_rec * sizeof(b200z_tar_member) / COPY_PIECE + 1) * sizeof(SlotCopy);
  std::vector<uint8_t> up(o_next + 8, 0);
  TarArchive *tab = (TarArchive *)up.data();
  for (size_t i = 0, at = 0; i < n; at += len[i] / 512 + 1, ++i) tab[i] = TarArchive{off[i], len[i], at};
  CU(g.d_ws.reserve(ws_bytes));
  uint8_t *ws = (uint8_t *)g.d_ws.p;
  // one source base for k_copy_slots: the lower of d_base and the workspace (headers come from the one, records from the other)
  const uint8_t *src = d_base && d_base < ws ? d_base : ws;
  CU(cudaMemcpyAsync(ws, up.data(), up.size(), cudaMemcpyHostToDevice, g.stream));
  const unsigned per_cta = TAR_THREADS / 32;
  if (!g_tar_ev[0]) {
    CU(cudaEventCreate(&g_tar_ev[0]));
    CU(cudaEventCreate(&g_tar_ev[1]));
  }
  CU(cudaEventRecord(g_tar_ev[0], g.stream));
  k_tar_walk<<<(unsigned)((n + per_cta - 1) / per_cta), TAR_THREADS, 0, g.stream>>>(
      d_base, (const TarArchive *)ws, (uint32_t)n, (b200z_tar_member *)(ws + o_rec), (TarCount *)(ws + o_cnt),
      (SlotCopy *)(ws + o_pc), (unsigned long long *)(ws + o_next), d_base ? (uint64_t)(d_base - src) : 0);
  count_launch();
  CU(cudaGetLastError());
  CU(cudaEventRecord(g_tar_ev[1], g.stream));
  std::vector<TarCount> cnt(n);
  CU(cudaMemcpyAsync(cnt.data(), ws + o_cnt, n * sizeof(TarCount), cudaMemcpyDeviceToHost, g.stream));
  CU(cudaStreamSynchronize(g.stream));
  float walk_ms = 0;
  CU(cudaEventElapsedTime(&walk_ms, g_tar_ev[0], g_tar_ev[1]));
  g_tar_walk_ms = walk_ms;
  uint64_t total = 0;
  std::vector<uint64_t> at_first(n);  // archive i's members start at the exclusive prefix sum of the counts
  for (size_t i = 0; i < n; ++i) {
    if (cnt[i].rc == B200Z_E_INTERNAL) {
      set_err("tar_walk_device: archive %zu has more members than its bound", i);
      return B200Z_E_INTERNAL;
    }
    at_first[i] = total;
    total += cnt[i].count;
  }
  if (total > cap) {
    set_err("tar_walk_device: %llu members, cap %zu", (unsigned long long)total, cap);
    *n_total = (size_t)total;
    return B200Z_E_NOSPC;
  }
  if (total) {
    // g.d_out: the gathered area, every header (512 bytes each, in the slots the warps took) and then the records (in
    // archive order); one k_copy_slots takes the header pieces the walk wrote and the records' pieces, and the area comes
    // back in one copy through the pinned staging buffer.  The host puts each archive's headers in archive order.
    const size_t o_recs = total * 512, out_bytes = o_recs + total * sizeof(b200z_tar_member);
    std::vector<SlotCopy> rp;
    for (size_t i = 0; i < n; ++i) {
      const uint64_t from = (uint64_t)(ws - src) + o_rec + tab[i].rec * sizeof(b200z_tar_member);
      const uint64_t to = o_recs + at_first[i] * sizeof(b200z_tar_member), bytes = cnt[i].count * sizeof(b200z_tar_member);
      for (uint64_t at = 0; at < bytes; at += COPY_PIECE) rp.push_back(SlotCopy{from + at, to + at, std::min(COPY_PIECE, bytes - at)});
    }
    const size_t n_pc = total + rp.size();
    CU(cudaMemcpyAsync(ws + o_pc + total * sizeof(SlotCopy), rp.data(), rp.size() * sizeof(SlotCopy), cudaMemcpyHostToDevice,
                       g.stream));
    CU(g.d_out.reserve(out_bytes));
    const unsigned grid = (unsigned)std::min<size_t>((n_pc + COPY_THREADS / 32 - 1) / (COPY_THREADS / 32), 1u << 16);
    k_copy_slots<<<grid, COPY_THREADS, 0, g.stream>>>(src, (uint8_t *)g.d_out.p, (const SlotCopy *)(ws + o_pc), (uint32_t)n_pc);
    count_launch();
    CU(cudaGetLastError());
    CU(g.h_stage.reserve(out_bytes));
    CU(cudaMemcpyAsync(g.h_stage.p, g.d_out.p, out_bytes, cudaMemcpyDeviceToHost, g.stream));
    CU(cudaStreamSynchronize(g.stream));
    const uint8_t *h = (const uint8_t *)g.h_stage.p;
    memcpy(members, h + o_recs, total * sizeof(b200z_tar_member));
    for (size_t i = 0; i < n; ++i) memcpy(headers + 512 * at_first[i], h + 512 * cnt[i].first, 512 * cnt[i].count);
    for (uint64_t k = 0; k < total; ++k)  // zero past a short header (only an archive's last member can have one)
      if (members[k].header_len < 512) memset(headers + 512 * k + members[k].header_len, 0, 512 - members[k].header_len);
  }
  for (size_t i = 0; i < n; ++i) {
    first[i] = at_first[i];
    count[i] = cnt[i].count;
    rc[i] = cnt[i].rc;
  }
  *n_total = (size_t)total;
  return B200Z_OK;
}

// (test hook, not part of the ABI) the device time of the last b200z_tar_walk_device call's k_tar_walk, by CUDA events
extern "C" void b200z_debug_tar_walk(double *walk_ms) { *walk_ms = g_tar_walk_ms; }

extern "C" int b200z_zip_extract(const uint8_t *z, size_t len, const b200z_zip_entry *entries, size_t n, uint8_t *out,
                                 size_t out_cap, const uint64_t *out_off, const uint64_t *out_room, uint64_t *out_len,
                                 int32_t *status, uint32_t flags) {
  return b200z_zip_extract_password(z, len, entries, n, out, out_cap, out_off, out_room, out_len, status, flags, nullptr, 0);
}

// ZipEncoder._encryptCompressedData (zip_encoder.dart:166-183) for n members at once: AES-256, CTR in place, then the MAC
// of the ciphertext.  One copy of data[0, max(off + len)) to the device and one back.
extern "C" int b200z_zip_aes_encrypt(uint8_t *data, const uint64_t *off, const uint64_t *len, size_t n, const uint8_t *salts,
                                     const uint8_t *password, size_t password_len, uint8_t *pwd_verify, uint8_t *mac) {
  int rc = require_init();
  if (rc) return rc;
  if (n == 0) return B200Z_OK;
  if (!data || !off || !len || !salts || !password || !pwd_verify || !mac) return B200Z_E_ARG;
  if (password_len == 0) {
    set_err("zip_aes_encrypt: empty password (Dart: ZipFile.deriveKey returns an empty list, sublist throws)");
    return B200Z_E_THROW;
  }
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  std::vector<ZipAesMember> aes(n);
  size_t extent = 0;
  for (size_t k = 0; k < n; ++k) {
    if (off[k] + len[k] < off[k]) return B200Z_E_ARG;
    ZipAesMember &m = aes[k];
    memset(&m, 0, sizeof m);
    m.src_off = m.dst_off = off[k];
    m.len = len[k];
    m.salt_len = 16;
    m.key_len = 32;
    memcpy(m.salt, salts + 16 * k, 16);
    extent = std::max(extent, (size_t)(off[k] + len[k]));
  }
  std::vector<ZipCtrTile> tiles;
  ctr_tiles(aes, tiles);
  const CryptLayout cl(n, tiles.size(), 0);
  CU(g.d_crypt.reserve(cl.bytes));
  CU(g.d_in.reserve(extent + 64));
  uint8_t *dc = (uint8_t *)g.d_crypt.p, *d_base = (uint8_t *)g.d_in.p;
  ZipHmacPads pads;
  zip_hmac_pads(password, password_len, &pads);
  if (extent) CU(cudaMemcpyAsync(d_base, data, extent, cudaMemcpyHostToDevice, g.stream));
  CU(cudaMemsetAsync(d_base + extent, 0, 64, g.stream));
  CU(cudaMemcpyAsync(dc + cl.members, aes.data(), n * sizeof(ZipAesMember), cudaMemcpyHostToDevice, g.stream));
  CU(cudaMemcpyAsync(dc + cl.tiles, tiles.data(), tiles.size() * sizeof(ZipCtrTile), cudaMemcpyHostToDevice, g.stream));
  const ZipAesMember *dm = (const ZipAesMember *)(dc + cl.members);
  CU(zip_launch_pbkdf2(dm, (uint32_t)n, pads, dc + cl.dk, (uint32_t *)(dc + cl.rk), dc + cl.ver, g.stream));
  CU(zip_launch_aes_ctr(dm, (const uint32_t *)(dc + cl.rk), (const ZipCtrTile *)(dc + cl.tiles), (uint32_t)tiles.size(), d_base,
                        g.stream));
  CU(zip_launch_hmac(dm, (uint32_t)n, dc + cl.dk, d_base, true, dc + cl.mac, g.stream));
  if (extent) CU(cudaMemcpyAsync(data, d_base, extent, cudaMemcpyDeviceToHost, g.stream));
  CU(cudaMemcpyAsync(pwd_verify, dc + cl.ver, 2 * n, cudaMemcpyDeviceToHost, g.stream));
  CU(cudaMemcpyAsync(mac, dc + cl.mac, 10 * n, cudaMemcpyDeviceToHost, g.stream));
  CU(cudaStreamSynchronize(g.stream));
  return B200Z_OK;
}

// kernel times of the last b200z_zip_extract_password call (ms): PBKDF2, CTR, MAC (from the moment it may start), ZipCrypto
extern "C" void b200z_debug_zip_crypt_ms(double out[4]) {
  for (int k = 0; k < 4; ++k) out[k] = g_crypt_ms[k];
}

// (test hooks, not part of the ABI) K12's threshold and chunk size in compressed bytes (0 each: the built-in values), and
// the last single-stream call's statistics: regions, chunks, redo rounds, chunks merged, fell back to the exact path,
// chunked path ran
extern "C" void b200z_debug_inflate_chunked_set(unsigned long long thresh, unsigned long long chunk) {
  g_ck.thresh = thresh ? (size_t)thresh : CK_THRESH;
  g_ck.chunk = (size_t)chunk;
}
extern "C" void b200z_debug_inflate_chunked_stats(unsigned long long out[6]) {
  for (int k = 0; k < 6; ++k) out[k] = g_ck_stats[k];
}
// (test hook) the last single-stream call's K12 kernel times in ms (CUDA events): finder, chunk decodes, windows + emit
extern "C" void b200z_debug_inflate_chunked_ms(double out[3]) {
  for (int k = 0; k < 3; ++k) out[k] = g_ck_ms[k];
}
// (test hooks) K12 for ZIP members (zip_chunked): caps on the members of one K12 batch and on each member's pool pages
// (0 each: none, the built-in share), and the last b200z_zip_extract call's statistics -- members offered, accepted,
// fell back, redo rounds, batches -- and kernel times in ms (finder, chunk decodes, windows + emit).  The threshold and
// the chunk size are b200z_debug_inflate_chunked_set's.
extern "C" void b200z_debug_zip_chunked_set(unsigned max_streams, unsigned max_pages) {
  g_zck_max_streams = max_streams;
  g_zck_max_pages = max_pages;
}
extern "C" void b200z_debug_zip_chunked_stats(unsigned long long out[5], double ms[3]) {
  for (int k = 0; k < 5; ++k) out[k] = g_zck_stats[k];
  for (int k = 0; k < 3; ++k) ms[k] = g_zck_ms[k];
}
// (test hooks) cap on the blocks b200z_bzip2_encode / _encode_batch sort and code in one batch (0: the built-in plan), so
// that inputs of a few blocks run through several batches; cap on the streams of one device group (0: the memory budget
// alone); the last encode call's streams, device groups, block batches, blocks and serially sorted blocks
static uint32_t g_bz2e_max_batch = 0, g_bz2e_max_group = 0;
static unsigned long long g_bz2e_stats[5] = {0, 0, 0, 0, 0};
extern "C" void b200z_debug_bzip2_encode_batch_set(unsigned max_batch) { g_bz2e_max_batch = max_batch; }
extern "C" void b200z_debug_bzip2_encode_group_set(unsigned max_streams) { g_bz2e_max_group = max_streams; }
extern "C" void b200z_debug_bzip2_encode_batch_stats(unsigned long long out[5]) {
  for (int k = 0; k < 5; ++k) out[k] = g_bz2e_stats[k];
}

// n BZip2 encodes (arguments checked, g.mu held).  Consecutive streams form device groups that fit the memory budget
// and keep staged positions below 4 GiB; each group is one multi-stream pass of the encoder (bz2e::encode_streams).
static int bzip2_encode_streams(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n,
                                uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len,
                                uint32_t *crc32, int32_t *rc) {
  const uint64_t kTile = 4096, kMaxIn = 0xfff00000ull;
  for (int k = 0; k < 5; ++k) g_bz2e_stats[k] = 0;
  g_bz2e_stats[0] = n;
  std::vector<size_t> todo;
  for (size_t i = 0; i < n; ++i) {
    out_len[i] = 0;
    if (crc32) crc32[i] = 0;
    if (in_len[i] >= kMaxIn) {
      set_err("bzip2 encode: inputs of 4 GiB and more are not supported");
      rc[i] = B200Z_E_ARG;
    } else {
      todo.push_back(i);
    }
  }
  if (todo.empty()) return B200Z_OK;
  CU(cudaSetDevice(g.device));
  size_t free_b = 0, total_b = 0;
  CU(cudaMemGetInfo(&free_b, &total_b));
  size_t budget = free_b + g.d_ws.cap > ((size_t)2 << 30) ? (free_b + g.d_ws.cap) / 2 : ((size_t)1 << 30);
  if (budget > ((size_t)24 << 30)) budget = (size_t)24 << 30;
  auto slot_of = [](uint64_t len) { return (uint64_t)align_up(bz2e::bound(len) + 64, 256); };
  for (size_t k = 0; k < todo.size();) {
    // the group [k, e): the first stream always, then while input, slots and workspace fit
    bz2e::PlanSums sums;
    bz2e::Plan plan{};
    uint64_t staged = 0, slots = 0;
    size_t e = k;
    for (; e < todo.size(); ++e) {
      const uint64_t len = in_len[todo[e]];
      bz2e::PlanSums t = sums;
      bz2e::plan_add(t, len);
      const uint64_t st2 = staged + align_up(len, kTile), sl2 = slots + slot_of(len);
      const bz2e::Plan p2 = bz2e::plan_of(t, budget);
      if (e > k && (st2 > kMaxIn || (g_bz2e_max_group && e - k >= g_bz2e_max_group) || st2 + sl2 + p2.ws_bytes > budget))
        break;
      sums = t;
      staged = st2;
      slots = sl2;
      plan = p2;
    }
    if (g_bz2e_max_batch && g_bz2e_max_batch < plan.batch) plan.batch = g_bz2e_max_batch;
    const size_t m = e - k;
    // layout: every stream starts on a 4 KiB tile, in stream order
    std::vector<bz2e::StreamDesc> sd(m);
    uint64_t in0 = 0, out0 = 0, in_end = 0, out_end = 0;
    uint32_t blk0 = 0;
    bool as_is = true;  // the inputs already lie so in the caller's buffer: stage the span as it is
    uint64_t lo = ~0ull;
    for (size_t j = 0; j < m; ++j) {
      const size_t i = todo[k + j];
      const uint64_t len = in_len[i];
      sd[j] = bz2e::StreamDesc{(uint32_t)in0, (uint32_t)len, (uint32_t)(in0 / kTile), bz2e::tiles_of(len), blk0,
                               bz2e::max_blocks_of(len), out0, slot_of(len)};
      if (len) {
        if (lo == ~0ull) lo = in_off[i];
        if (in_off[i] != lo + in0) as_is = false;
        in_end = in0 + len;
      }
      in0 += align_up(len, kTile);
      blk0 += sd[j].max_blocks;
      out0 += sd[j].out_cap;
    }
    out_end = out0;
    std::unique_ptr<uint8_t[]> packed;
    const uint8_t *src = nullptr;
    if (in_end && as_is) {
      src = in_base + lo;
    } else if (in_end) {
      packed.reset(new uint8_t[in_end]);
      for (size_t j = 0; j < m; ++j)
        if (sd[j].n) memcpy(packed.get() + sd[j].in0, in_base + in_off[todo[k + j]], sd[j].n);
      src = packed.get();
    }
    int r = stage_input(src, in_end);
    if (r) return r;
    CU(g.d_out.reserve(out_end));
    CU(g.d_ws.reserve(plan.ws_bytes));
    std::vector<unsigned long long> lens(m);
    std::vector<uint32_t> tile_crc(crc32 ? plan.n_tiles : 0);
    bz2e::Stats st{0, 0, 0, 0, 0};
    r = bz2e::encode_streams((const uint8_t *)g.d_in.p, sd.data(), (uint8_t *)g.d_out.p, g.d_ws.p, plan, lens.data(),
                             crc32 ? tile_crc.data() : nullptr, &st, (void *)g.stream);
    if (r == -3) {
      set_err("bzip2 encode: internal output bound too small");
      return B200Z_E_INTERNAL;
    }
    if (r != 0) {
      cudaError_t ce = cudaGetLastError();
      set_err("bzip2 encode: device failure (%s)", cudaGetErrorString(ce));
      return B200Z_E_INTERNAL;
    }
    g_bz2e_stats[1]++;
    g_bz2e_stats[2] += st.n_batches;
    g_bz2e_stats[3] += st.n_blocks;
    g_bz2e_stats[4] += st.n_serial_blocks;
    // the outputs: one copy back, then each stream to its slot
    const uint64_t used = sd[m - 1].out0 + lens[m - 1];
    for (size_t j = 0; j < m; ++j) {
      const size_t i = todo[k + j];
      out_len[i] = lens[j];
      if (crc32) crc32[i] = bz2e::crc32_fold(tile_crc.data() + sd[j].tile0, sd[j].n);
      rc[i] = lens[j] > out_cap[i] ? B200Z_E_NOSPC : B200Z_OK;
      if (rc[i] == B200Z_E_NOSPC)
        set_err("bzip2 encode: output needs %llu bytes, out_cap %llu", (unsigned long long)lens[j],
                (unsigned long long)out_cap[i]);
    }
    if (m == 1) {
      if (rc[todo[k]] == B200Z_OK)
        CU(cudaMemcpyAsync(out_base + out_off[todo[k]], g.d_out.p, lens[0], cudaMemcpyDeviceToHost, g.stream));
      CU(cudaStreamSynchronize(g.stream));
    } else {
      std::unique_ptr<uint8_t[]> h_out(new uint8_t[used]);
      CU(cudaMemcpyAsync(h_out.get(), g.d_out.p, used, cudaMemcpyDeviceToHost, g.stream));
      CU(cudaStreamSynchronize(g.stream));
      for (size_t j = 0; j < m; ++j) {
        const size_t i = todo[k + j];
        if (rc[i] == B200Z_OK && lens[j]) memcpy(out_base + out_off[i], h_out.get() + sd[j].out0, lens[j]);
      }
    }
    k = e;
  }
  return B200Z_OK;
}

extern "C" {

const char *b200z_version(void) { return "b200z 0.1 (sm_90a)"; }
const char *b200z_last_error(void) { return t_err; }
uint64_t b200z_launch_count(void) { return g_launches.load(); }
// (debug, not part of the ABI) BZip2 candidate blocks decoded by k_bz2_entropy_fast / left to the exact kernel so far
void b200z_debug_bz2_blocks(unsigned long long out[2]) {
  out[0] = g_bz2_fast_blocks.load();
  out[1] = g_bz2_exact_blocks.load();
}

int b200z_bzip2_decode(const uint8_t *in, size_t in_len, int verify, uint8_t *out, size_t out_cap, size_t *out_len) {
  int rc = require_init();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  rc = stage_input(in, in_len);
  if (rc) return rc;
  CU(cudaMemsetAsync((uint8_t *)g.d_in.p + in_len, 0, 64, g.stream));
  Bz2Job j{0, in_len, out, out_cap, 0, B200Z_OK};
  rc = bzip2_decode_device((const uint8_t *)g.d_in.p, &j, 1, verify);
  if (out_len) *out_len = j.out_len;
  return rc ? rc : j.rc;
}

}  // extern "C"
// b200z_bzip2_decode_batch, or b200z_bzip2_decode_batch_to_device with a stream (dev_out)
static int bzip2_decode_batch_impl(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                                   uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len,
                                   int32_t *rc, bool dev_out, void *cuda_stream) {
  int r = require_init();
  if (r) return r;
  if (n && (!in_off || !in_len || !out_off || !out_cap || !out_len || !rc)) {
    set_err("bzip2_decode_batch: null array");
    return B200Z_E_ARG;
  }
  uint64_t lo = ~0ull, hi = 0, total = 0;
  std::vector<size_t> by_out;
  for (size_t i = 0; i < n; ++i) {
    if (in_off[i] + in_len[i] < in_off[i] || out_off[i] + out_cap[i] < out_off[i] || (in_len[i] && !in_base) ||
        (out_cap[i] && !out_base)) {
      set_err("bzip2_decode_batch: stream %zu: bad range", i);
      return B200Z_E_ARG;
    }
    if (in_len[i]) {
      lo = std::min(lo, in_off[i]);
      hi = std::max(hi, in_off[i] + in_len[i]);
      total += in_len[i];
    }
    if (out_cap[i]) by_out.push_back(i);
  }
  std::sort(by_out.begin(), by_out.end(), [&](size_t a, size_t b) { return out_off[a] < out_off[b]; });
  for (size_t k = 1; k < by_out.size(); ++k)
    if (out_off[by_out[k - 1]] + out_cap[by_out[k - 1]] > out_off[by_out[k]]) {
      set_err("bzip2_decode_batch: output slots %zu and %zu overlap", by_out[k - 1], by_out[k]);
      return B200Z_E_ARG;
    }
  if (dev_out && (r = device_out_arg("bzip2_decode_batch_to_device", out_base, n, out_cap)) != B200Z_OK) return r;
  std::lock_guard<std::mutex> lk(g.mu);
  if (n == 0) return bzip2_decode_device(nullptr, nullptr, 0, verify);
  CU(cudaSetDevice(g.device));
  if (dev_out && (r = wait_for_caller(cuda_stream)) != B200Z_OK) return r;
  // one copy to the device: the span of all inputs as it is, or the inputs packed when the span is mostly other bytes
  std::vector<Bz2Job> jobs(n);
  std::vector<uint8_t> packed;
  const uint8_t *src = nullptr;
  size_t staged = 0;
  if (total == 0) {
    for (size_t i = 0; i < n; ++i) jobs[i].in_off = 0;
  } else if (hi - lo <= 2 * total + ((size_t)1 << 20)) {
    src = in_base + lo;
    staged = (size_t)(hi - lo);
    for (size_t i = 0; i < n; ++i) jobs[i].in_off = in_len[i] ? in_off[i] - lo : 0;
  } else {
    packed.resize(total);
    for (size_t i = 0; i < n; ++i) {
      jobs[i].in_off = staged;
      if (in_len[i]) memcpy(packed.data() + staged, in_base + in_off[i], in_len[i]);
      staged += in_len[i];
    }
    src = packed.data();
  }
  r = stage_input(src, staged);
  if (r) return r;
  CU(cudaMemsetAsync((uint8_t *)g.d_in.p + staged, 0, 64, g.stream));
  for (size_t i = 0; i < n; ++i) {
    jobs[i].in_len = in_len[i];
    jobs[i].out = out_base + out_off[i];
    jobs[i].out_cap = out_cap[i];
  }
  r = bzip2_decode_device((const uint8_t *)g.d_in.p, jobs.data(), n, verify, nullptr, dev_out ? out_base : nullptr);
  for (size_t i = 0; i < n; ++i) {
    out_len[i] = jobs[i].out_len;
    rc[i] = jobs[i].rc;
  }
  return r;
}
extern "C" {
int b200z_bzip2_decode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                             uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len, int32_t *rc) {
  return bzip2_decode_batch_impl(in_base, in_off, in_len, n, verify, out_base, out_off, out_cap, out_len, rc, false, nullptr);
}
int b200z_bzip2_decode_batch_to_device(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n,
                                       int verify, uint8_t *d_out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                       uint64_t *out_len, int32_t *rc, void *cuda_stream) {
  return bzip2_decode_batch_impl(in_base, in_off, in_len, n, verify, d_out_base, out_off, out_cap, out_len, rc, true, cuda_stream);
}
// (test hooks, not part of the ABI) cap on the blocks of one BZip2 device group (0: the memory budget alone); the last
// b200z_bzip2_decode* or ZIP call's bzip2 streams, device groups and blocks
void b200z_debug_bz2_batch_set(unsigned max_blocks) { g_bz2_max_group_blocks = max_blocks; }
void b200z_debug_bz2_batch_stats(unsigned long long out[3]) {
  for (int k = 0; k < 3; ++k) out[k] = g_bz2_stats[k];
}
void b200z_profile_enable(int on) { profile_enable(on != 0); }
int b200z_crc32(const uint8_t *in, size_t in_len, uint32_t *crc) {
  int rc = require_init();
  if (rc) return rc;
  if (!crc) return B200Z_E_ARG;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  rc = stage_input(in, in_len);
  if (rc) return rc;
  return device_crc32((const uint8_t *)g.d_in.p, in_len, crc);
}

int b200z_xz_decode(const uint8_t *in, size_t in_len, int verify, uint8_t *out, size_t out_cap, size_t *out_len) {
  int rc = require_init();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  size_t n = 0;
  rc = xz_decode_impl(in, in_len, verify, out, out_cap, &n, g.stream);
  if (out_len) *out_len = n;
  return rc;
}
size_t b200z_xz_bound(const uint8_t *in, size_t in_len) { return xz_bound(in, in_len); }
int b200z_xz_encode(const uint8_t *in, size_t in_len, int check, uint8_t *out, size_t out_cap, size_t *out_len) {
  int rc = require_init();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  size_t n = 0;
  rc = xz_encode_impl(in, in_len, check, out, out_cap, &n, g.stream);
  if (out_len) *out_len = n;
  return rc;
}
size_t b200z_xz_encode_bound(size_t in_len) { return xz_encode_bound(in_len); }
int b200z_crc64(const uint8_t *in, size_t in_len, uint64_t *crc) {
  int rc = require_init();
  if (rc) return rc;
  if (!crc) return B200Z_E_ARG;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  return xz_crc64_impl(in, in_len, crc, g.stream);
}
// (debug, not part of the ABI) k_xz_lzma time in ms and the run count of the last b200z_xz_decode*
void b200z_debug_xz(double *lzma_ms, uint32_t *n_runs) { xz_debug(lzma_ms, n_runs); }

// the argument rules of the XZ batch entries (those of the BZip2 ones): no null array, no range that wraps, no output
// slots that overlap; nothing is written when one is broken
static int xz_batch_args(const char *name, const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n,
                         uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len, int32_t *rc) {
  if (n && (!in_off || !in_len || !out_off || !out_cap || !out_len || !rc)) {
    set_err("%s: null array", name);
    return B200Z_E_ARG;
  }
  std::vector<size_t> by_out;
  for (size_t i = 0; i < n; ++i) {
    if (in_off[i] + in_len[i] < in_off[i] || out_off[i] + out_cap[i] < out_off[i] || (in_len[i] && !in_base) ||
        (out_cap[i] && !out_base)) {
      set_err("%s: stream %zu: bad range", name, i);
      return B200Z_E_ARG;
    }
    if (out_cap[i]) by_out.push_back(i);
  }
  std::sort(by_out.begin(), by_out.end(), [&](size_t a, size_t b) { return out_off[a] < out_off[b]; });
  for (size_t k = 1; k < by_out.size(); ++k)
    if (out_off[by_out[k - 1]] + out_cap[by_out[k - 1]] > out_off[by_out[k]]) {
      set_err("%s: output slots %zu and %zu overlap", name, by_out[k - 1], by_out[k]);
      return B200Z_E_ARG;
    }
  return B200Z_OK;
}
int b200z_xz_decode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                          uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len, int32_t *rc) {
  int r = require_init();
  if (r) return r;
  r = xz_batch_args("xz_decode_batch", in_base, in_off, in_len, n, out_base, out_off, out_cap, out_len, rc);
  if (r) return r;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  return xz_decode_streams(in_base, in_off, in_len, n, verify, out_base, out_off, out_cap, out_len, rc, g.stream);
}
int b200z_xz_decode_batch_to_device(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                                    uint8_t *d_out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len,
                                    int32_t *rc, void *cuda_stream) {
  int r = require_init();
  if (r) return r;
  r = xz_batch_args("xz_decode_batch_to_device", in_base, in_off, in_len, n, d_out_base, out_off, out_cap, out_len, rc);
  if (r || (r = device_out_arg("xz_decode_batch_to_device", d_out_base, n, out_cap))) return r;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  if ((r = wait_for_caller(cuda_stream))) return r;
  return xz_decode_streams(in_base, in_off, in_len, n, verify, d_out_base, out_off, out_cap, out_len, rc, g.stream, true);
}
int b200z_xz_encode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int check,
                          uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len, int32_t *rc) {
  int r = require_init();
  if (r) return r;
  if (check < 0 || check > 3) {
    set_err("xz_encode_batch: check must be 0 (none), 1 (crc32), 2 (crc64) or 3 (sha256)");
    return B200Z_E_ARG;
  }
  r = xz_batch_args("xz_encode_batch", in_base, in_off, in_len, n, out_base, out_off, out_cap, out_len, rc);
  if (r || n == 0) return r;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  return xz_encode_streams(in_base, in_off, in_len, n, check, out_base, out_off, out_cap, out_len, rc, g.stream);
}
// (test hooks, not part of the ABI) cap on the streams of one XZ decode device group (0: the memory budget alone); the
// last b200z_xz_decode* call's streams, device groups and runs
void b200z_debug_xz_batch_set(unsigned max_streams) { xz_batch_set(max_streams); }
void b200z_debug_xz_batch_stats(unsigned long long out[3]) { xz_batch_stats(out); }

int b200z_bzip2_decode_shard(const uint8_t *in, size_t in_len, uint32_t rank, uint32_t world, uint8_t *out, size_t out_cap,
                             size_t *out_len, b200z_bz2_block *blocks, size_t blocks_cap, size_t *n_blocks) {
  int rc = require_init();
  if (rc) return rc;
  if (world == 0 || rank >= world || !blocks) {
    set_err("bzip2_decode_shard: bad rank/world");
    return B200Z_E_ARG;
  }
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  Bz2Shard sh{rank, world, blocks, blocks_cap, 0};
  rc = stage_input(in, in_len);
  if (rc) return rc;
  CU(cudaMemsetAsync((uint8_t *)g.d_in.p + in_len, 0, 64, g.stream));
  Bz2Job j{0, in_len, out, out_cap, 0, B200Z_OK};
  rc = bzip2_decode_device((const uint8_t *)g.d_in.p, &j, 1, 0, &sh);
  if (out_len) *out_len = j.out_len;
  if (n_blocks) *n_blocks = sh.n_blocks;
  return rc ? rc : j.rc;
}

int b200z_bzip2_encode(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, size_t *out_len) {
  int rc = require_init();
  if (rc) return rc;
  if (in_len >= 0xfff00000ull) {
    set_err("bzip2 encode: inputs of 4 GiB and more are not supported");
    return B200Z_E_ARG;
  }
  std::lock_guard<std::mutex> lk(g.mu);
  const uint64_t off = 0, len = in_len, cap = out_cap;
  uint64_t n = 0;
  int32_t r1 = B200Z_OK;
  rc = bzip2_encode_streams(in, &off, &len, 1, out, &off, &cap, &n, nullptr, &r1);
  if (rc) return rc;
  if (out_len) *out_len = (size_t)n;
  return r1;
}

int b200z_bzip2_encode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n,
                             uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len,
                             uint32_t *crc32, int32_t *rc) {
  int r = require_init();
  if (r) return r;
  if (n && (!in_off || !in_len || !out_off || !out_cap || !out_len || !rc)) {
    set_err("bzip2_encode_batch: null array");
    return B200Z_E_ARG;
  }
  std::vector<size_t> by_out;
  for (size_t i = 0; i < n; ++i) {
    if (in_off[i] + in_len[i] < in_off[i] || out_off[i] + out_cap[i] < out_off[i] || (in_len[i] && !in_base) ||
        (out_cap[i] && !out_base)) {
      set_err("bzip2_encode_batch: stream %zu: bad range", i);
      return B200Z_E_ARG;
    }
    if (out_cap[i]) by_out.push_back(i);
  }
  std::sort(by_out.begin(), by_out.end(), [&](size_t a, size_t b) { return out_off[a] < out_off[b]; });
  for (size_t k = 1; k < by_out.size(); ++k)
    if (out_off[by_out[k - 1]] + out_cap[by_out[k - 1]] > out_off[by_out[k]]) {
      set_err("bzip2_encode_batch: output slots %zu and %zu overlap", by_out[k - 1], by_out[k]);
      return B200Z_E_ARG;
    }
  std::lock_guard<std::mutex> lk(g.mu);
  return bzip2_encode_streams(in_base, in_off, in_len, n, out_base, out_off, out_cap, out_len, crc32, rc);
}
size_t b200z_bzip2_bound(size_t in_len) { return bz2e::bound(in_len); }

int b200z_profile_read(double *fast_ms, double *decode_ms, double *expand_ms, uint64_t *n_batches) {
  return profile_read(fast_ms, decode_ms, expand_ms, n_batches) ? B200Z_E_NODEVICE : B200Z_OK;
}

int b200z_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

int b200z_init(int device, uint32_t flags) {
  (void)flags;
  std::lock_guard<std::mutex> lk(g.mu);
  if (g.inited && g.device == device) return B200Z_OK;
  int n = b200z_device_count();
  if (n <= 0 || device < 0 || device >= n) {
    set_err("b200z_init: CUDA device %d not available (%d visible): there is no CPU fallback", device, n);
    return B200Z_E_NODEVICE;
  }
  CU(cudaSetDevice(device));
  if (!g.stream) {
    CU(cudaStreamCreateWithFlags(&g.stream, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&g.s_h2d, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&g.s_d2h, cudaStreamNonBlocking));
    for (int i = 0; i < Ctx::kCompStreams; ++i) CU(cudaStreamCreateWithFlags(&g.s_comp[i], cudaStreamNonBlocking));
  }
  g.device = device;
  g.inited = true;
  return B200Z_OK;
}

void b200z_shutdown(void) {
  file_release();  // before g.mu: a file call holds its own lock while it takes g.mu, never the other way round
  std::lock_guard<std::mutex> lk(g.mu);
  if (!g.inited) return;
  cudaSetDevice(g.device);
  cudaStreamSynchronize(g.stream);
  g.d_in.release(); g.d_out.release(); g.d_ws.release(); g.d_meta.release(); g.d_small.release(); g.d_bz.release(); g.d_tok.release(); g.d_crypt.release();
  g.d_slots.release();
  g.h_meta.release(); g.h_stage.release();
  cudaStreamDestroy(g.stream);
  cudaStreamDestroy(g.s_h2d);
  cudaStreamDestroy(g.s_d2h);
  for (int i = 0; i < Ctx::kCompStreams; ++i) cudaStreamDestroy(g.s_comp[i]);
  g.stream = g.s_h2d = g.s_d2h = nullptr;
  g.inited = false;
}

void *b200z_host_alloc(size_t bytes) {
  void *p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    set_err("b200z_host_alloc(%zu) failed", bytes);
    return nullptr;
  }
  return p;
}
void b200z_host_free(void *p) {
  if (p) cudaFreeHost(p);
}

size_t b200z_inflate_workspace_bytes(size_t n_units, size_t total_in_bytes, size_t total_out_cap) {
  (void)total_in_bytes;
  return workspace_bytes(n_units, total_out_cap);
}

int b200z_inflate_batch_device(const uint8_t *d_in_base, const uint64_t *d_in_off, const uint32_t *d_in_len,
                               uint8_t *d_out_base, const uint64_t *d_out_off, const uint32_t *d_out_cap,
                               uint32_t *d_out_len, int32_t *d_status, uint32_t *d_in_used, size_t n_units,
                               void *d_workspace, size_t workspace_bytes_, void *cuda_stream) {
  int rc = require_init();
  if (rc) return rc;
  if (n_units == 0) return B200Z_OK;
  const size_t extent = inflate_ws_extent_for(n_units, workspace_bytes_);
  if (extent == INFLATE_WS_TOO_SMALL) {
    set_err("inflate_batch_device: workspace too small (size it with b200z_inflate_workspace_bytes)");
    return B200Z_E_ARG;
  }
  InflateBatch b;
  b.in_base = d_in_base; b.in_off = d_in_off; b.in_len = d_in_len;
  b.out_base = d_out_base; b.out_off = d_out_off; b.out_cap = d_out_cap;
  b.out_len = d_out_len; b.status = d_status; b.in_used = d_in_used;
  b.n_units = n_units;
  b.ws = inflate_ws_carve(d_workspace, n_units, extent);
  cudaStream_t s = cuda_stream ? (cudaStream_t)cuda_stream : g.stream;
  CU(launch_inflate(b, s));
  return B200Z_OK;
}

int b200z_inflate_batch(const uint8_t *in_base, size_t in_bytes, const uint64_t *in_off, const uint32_t *in_len,
                        uint8_t *out_base, size_t out_bytes, const uint64_t *out_off, const uint32_t *out_cap,
                        uint32_t *out_len, int32_t *status, uint32_t *in_used, size_t n_units) {
  int rc = require_init();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  for (size_t u = 0; u < n_units; ++u) {
    if (in_off[u] + in_len[u] > in_bytes || out_off[u] + out_cap[u] > out_bytes) {
      set_err("inflate_batch: unit %zu exceeds the buffers", u);
      return B200Z_E_ARG;
    }
  }
  rc = stage_input(in_base, in_bytes);
  if (rc) return rc;
  CU(g.d_out.reserve(out_bytes + 64));
  rc = run_batch_on_staged(in_off, in_len, out_off, out_cap, out_len, status, in_used, n_units, out_bytes);
  if (rc) return rc;
  if (out_bytes) CU(cudaMemcpyAsync(out_base, g.d_out.p, out_bytes, cudaMemcpyDeviceToHost, g.stream));
  CU(cudaStreamSynchronize(g.stream));
  return B200Z_OK;
}

int b200z_inflate_raw(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, size_t *out_len,
                      size_t *in_consumed, int32_t *unit_status) {
  int rc = require_init();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  if (in_len > 0xfffffff0u) {
    set_err("inflate_raw: streams above 4 GiB are not supported");
    return B200Z_E_ARG;
  }
  rc = stage_input(in, in_len);
  if (rc) return rc;
  OneResult r{0, 0, B200Z_U_EOS};
  if (in_len > 0) {
    rc = run_one_staged(in, 0, in_len, 0, out_cap, &r);
    if (rc) return rc;
    if (r.out_len) CU(cudaMemcpyAsync(out, g.d_out.p, r.out_len, cudaMemcpyDeviceToHost, g.stream));
    CU(cudaStreamSynchronize(g.stream));
  }
  if (out_len) *out_len = r.out_len;
  if (in_consumed) *in_consumed = r.in_used;
  if (unit_status) *unit_status = r.status;
  if (r.status == B200Z_U_NOSPC) {
    set_err("inflate_raw: out_cap %zu too small", out_cap);
    return B200Z_E_NOSPC;
  }
  if (r.status == B200Z_U_RANGE || r.status == B200Z_U_THROW) {
    set_err("inflate_raw: Dart would throw RangeError (unit status %d)", r.status);
    return B200Z_E_THROW;
  }
  return B200Z_OK;  // STOP / BADCODE: reference keeps the partial output silently
}

int b200z_deflate_raw(const uint8_t *in, size_t in_len, int level, int window_bits, uint8_t *out, size_t out_cap,
                      size_t *out_len, uint32_t *crc32_of_input) {
  int rc = require_init();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  rc = stage_input(in, in_len);
  if (rc) return rc;
  CU(cudaMemsetAsync((uint8_t *)g.d_in.p + in_len, 0, 64, g.stream));
  size_t n = 0;
  rc = deflate_staged(in_len, level, window_bits, &n);
  if (rc) return rc;
  if (out_len) *out_len = n;
  if (n > out_cap) {
    set_err("deflate: output needs %zu bytes, out_cap %zu", n, out_cap);
    return B200Z_E_NOSPC;
  }
  if (n) CU(cudaMemcpyAsync(out, g.d_out.p, n, cudaMemcpyDeviceToHost, g.stream));
  if (crc32_of_input) {
    rc = device_crc32((const uint8_t *)g.d_in.p, in_len, crc32_of_input);
    if (rc) return rc;
  }
  CU(cudaStreamSynchronize(g.stream));
  return B200Z_OK;
}

size_t b200z_deflate_bound(size_t in_len) { return deflate_bound(in_len) + 32; }

int b200z_deflate_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n_units, int level,
                        int window_bits, uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len,
                        uint32_t *crc32, int32_t *status) {
  int rc = require_init();
  if (rc) return rc;
  if (window_bits < 9 || window_bits > 15 || level < 0 || level > 9) {
    set_err("deflate: invalid level %d / windowBits %d (Dart: LateInitializationError)", level, window_bits);
    return B200Z_E_ARG;
  }
  if (n_units == 0) return B200Z_OK;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  return deflate_batch_impl(in_base, in_off, in_len, n_units, level, window_bits, out_base, out_off, out_cap, out_len, crc32,
                            status);
}

int b200z_zlib_encode(const uint8_t *in, size_t in_len, int level, int window_bits, int raw, uint8_t *out, size_t out_cap,
                      size_t *out_len) {
  int rc = require_init();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  rc = stage_input(in, in_len);
  if (rc) return rc;
  CU(cudaMemsetAsync((uint8_t *)g.d_in.p + in_len, 0, 64, g.stream));
  size_t n = 0;
  rc = deflate_staged(in_len, level, window_bits, &n);
  if (rc) return rc;
  const size_t total = raw ? n : n + 6;
  if (out_len) *out_len = total;
  if (total > out_cap) {
    set_err("zlib_encode: output needs %zu bytes, out_cap %zu", total, out_cap);
    return B200Z_E_NOSPC;
  }
  size_t o = 0;
  if (!raw) {
    zlib_put_header(out, window_bits);
    o = 2;
  }
  if (n) CU(cudaMemcpyAsync(out + o, g.d_out.p, n, cudaMemcpyDeviceToHost, g.stream));
  o += n;
  if (!raw) {
    uint32_t ad;
    rc = device_adler32((const uint8_t *)g.d_in.p, in_len, &ad);
    if (rc) return rc;
    zlib_put_adler(out + o, ad);
  }
  CU(cudaStreamSynchronize(g.stream));
  return B200Z_OK;
}

int b200z_gzip_encode(const uint8_t *in, size_t in_len, int level, uint32_t mtime, uint8_t *out, size_t out_cap,
                      size_t *out_len) {
  int rc = require_init();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  rc = stage_input(in, in_len);
  if (rc) return rc;
  CU(cudaMemsetAsync((uint8_t *)g.d_in.p + in_len, 0, 64, g.stream));
  size_t n = 0;
  rc = deflate_staged(in_len, level, 15, &n);
  if (rc) return rc;
  const size_t total = n + 18;
  if (out_len) *out_len = total;
  if (total > out_cap) {
    set_err("gzip_encode: output needs %zu bytes, out_cap %zu", total, out_cap);
    return B200Z_E_NOSPC;
  }
  gzip_put_header(out, mtime);
  if (n) CU(cudaMemcpyAsync(out + 10, g.d_out.p, n, cudaMemcpyDeviceToHost, g.stream));
  uint32_t crc;
  rc = device_crc32((const uint8_t *)g.d_in.p, in_len, &crc);
  if (rc) return rc;
  gzip_put_trailer(out + 10 + n, crc, in_len);
  CU(cudaStreamSynchronize(g.stream));
  return B200Z_OK;
}

size_t b200z_gzip_bound(const uint8_t *in, size_t in_len) {
  size_t total = 0;
  return hinted_run(in, in_len, 0, nullptr, &total) == in_len ? total : 0;  // every member hinted, or unknown
}

int b200z_gzip_decode(const uint8_t *in, size_t in_len, int verify, uint8_t *out, size_t out_cap, size_t *out_len) {
  int rc = require_init();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  size_t pos = 0, out_pos = 0, needed = 0;
  rc = gzip_fast_path(in, in_len, out, out_cap, &pos, &out_pos, &needed);
  if (rc) {
    if (out_len) *out_len = needed;
    return rc;
  }
  size_t n = out_pos;
  if (pos < in_len) {
    // whatever the hinted run did not cover (no hints, a lying hint, the zlib fall-back): generic path
    const size_t done_out = out_pos;
    rc = stage_input(in, in_len);
    if (rc) return rc;
    rc = gzip_decode_staged(in, in_len, verify, out_cap, &n, pos, out_pos);
    if (out_len) *out_len = n;
    if (rc == B200Z_E_NOSPC || rc == B200Z_E_NODEVICE) return rc;
    size_t hi = n > out_cap ? out_cap : n;
    if (hi > done_out)
      CU(cudaMemcpyAsync(out + done_out, (uint8_t *)g.d_out.p + done_out, hi - done_out, cudaMemcpyDeviceToHost, g.stream));
    CU(cudaStreamSynchronize(g.stream));
    return rc;
  }
  if (out_len) *out_len = n;
  return B200Z_OK;
}

int b200z_zlib_decode(const uint8_t *in, size_t in_len, int verify, int raw, uint8_t *out, size_t out_cap,
                      size_t *out_len) {
  int rc = require_init();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  rc = stage_input(in, in_len);
  if (rc) return rc;
  size_t n = 0;
  rc = zlib_decode_staged(in, in_len, 0, verify, raw, /*big_endian=*/1, 0, out_cap, &n);
  if (out_len) *out_len = n;
  if (rc == B200Z_E_NOSPC || rc == B200Z_E_NODEVICE) return rc;
  if (n > out_cap) n = out_cap;
  if (n) CU(cudaMemcpyAsync(out, g.d_out.p, n, cudaMemcpyDeviceToHost, g.stream));
  CU(cudaStreamSynchronize(g.stream));
  return rc;
}

int b200z_gzip_decode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                            uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len, int32_t *rc) {
  int r = require_init();
  if (r) return r;
  r = xz_batch_args("gzip_decode_batch", in_base, in_off, in_len, n, out_base, out_off, out_cap, out_len, rc);
  if (r) return r;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  return gzip_zlib_decode_streams(true, in_base, in_off, in_len, n, verify, 0, out_base, out_off, out_cap, out_len, rc);
}
int b200z_zlib_decode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify, int raw,
                            uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len, int32_t *rc) {
  int r = require_init();
  if (r) return r;
  r = xz_batch_args("zlib_decode_batch", in_base, in_off, in_len, n, out_base, out_off, out_cap, out_len, rc);
  if (r) return r;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  return gzip_zlib_decode_streams(false, in_base, in_off, in_len, n, verify, raw, out_base, out_off, out_cap, out_len, rc);
}
int b200z_gzip_decode_batch_to_device(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                                      uint8_t *d_out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len,
                                      int32_t *rc, void *cuda_stream) {
  int r = require_init();
  if (r) return r;
  r = xz_batch_args("gzip_decode_batch_to_device", in_base, in_off, in_len, n, d_out_base, out_off, out_cap, out_len, rc);
  if (r || (r = device_out_arg("gzip_decode_batch_to_device", d_out_base, n, out_cap))) return r;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  if ((r = wait_for_caller(cuda_stream))) return r;
  return gzip_zlib_decode_streams(true, in_base, in_off, in_len, n, verify, 0, d_out_base, out_off, out_cap, out_len, rc, true);
}
int b200z_zlib_decode_batch_to_device(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                                      int raw, uint8_t *d_out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                      uint64_t *out_len, int32_t *rc, void *cuda_stream) {
  int r = require_init();
  if (r) return r;
  r = xz_batch_args("zlib_decode_batch_to_device", in_base, in_off, in_len, n, d_out_base, out_off, out_cap, out_len, rc);
  if (r || (r = device_out_arg("zlib_decode_batch_to_device", d_out_base, n, out_cap))) return r;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  if ((r = wait_for_caller(cuda_stream))) return r;
  return gzip_zlib_decode_streams(false, in_base, in_off, in_len, n, verify, raw, d_out_base, out_off, out_cap, out_len, rc, true);
}
int b200z_gzip_encode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int level,
                            uint32_t mtime, uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len,
                            int32_t *rc) {
  int r = require_init();
  if (r) return r;
  if (level < 0 || level > 9) {
    set_err("gzip_encode_batch: invalid level %d (Dart: LateInitializationError)", level);
    return B200Z_E_ARG;
  }
  r = xz_batch_args("gzip_encode_batch", in_base, in_off, in_len, n, out_base, out_off, out_cap, out_len, rc);
  if (r || n == 0) return r;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  return gzip_zlib_encode_streams(true, in_base, in_off, in_len, n, level, 15, 0, mtime, out_base, out_off, out_cap, out_len, rc);
}
int b200z_zlib_encode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int level,
                            int window_bits, int raw, uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                            uint64_t *out_len, int32_t *rc) {
  int r = require_init();
  if (r) return r;
  if (window_bits < 9 || window_bits > 15 || level < 0 || level > 9) {
    set_err("zlib_encode_batch: invalid level %d / windowBits %d (Dart: LateInitializationError)", level, window_bits);
    return B200Z_E_ARG;
  }
  r = xz_batch_args("zlib_encode_batch", in_base, in_off, in_len, n, out_base, out_off, out_cap, out_len, rc);
  if (r || n == 0) return r;
  std::lock_guard<std::mutex> lk(g.mu);
  CU(cudaSetDevice(g.device));
  return gzip_zlib_encode_streams(false, in_base, in_off, in_len, n, level, window_bits, raw, 0, out_base, out_off, out_cap, out_len,
                                  rc);
}
// (test hooks, not part of the ABI) cap on the streams of one gzip / zlib decode device group (0: the memory budget
// alone); the last b200z_gzip_decode_batch / b200z_zlib_decode_batch call's streams, device groups, rounds, inflate units,
// and units offered to / accepted by K12
void b200z_debug_gzip_batch_set(unsigned max_streams) { g_gzb_max_group = max_streams; }
void b200z_debug_gzip_batch_stats(unsigned long long out[6]) {
  for (int k = 0; k < 6; ++k) out[k] = g_gzb_stats[k];
}

}  // extern "C"
