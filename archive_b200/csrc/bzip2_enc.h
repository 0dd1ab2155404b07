// bzip2_enc.h -- plan / entry point of the device BZip2 encoder (bzip2_enc_kernels.cu).  Not installed.
#pragma once
#include <stddef.h>
#include <stdint.h>

#define BZ2E_BSTRIDE 901120u          // element stride of one block in every per-block array (440 tiles of 2048)
#define BZ2E_BLKBYTES (BZ2E_BSTRIDE)  // byte stride of the RLE1 block buffer

namespace b200z {
namespace bz2e {

struct BlkInfo {
  uint32_t start, end;  // input range [start, end) consumed by the block
  uint32_t e0;          // end of the block's first run (chopped from `start`)
  uint32_t c;           // end of the last closed run; in[c] (if c < n) is the byte that closed it
  uint32_t A;           // RLE1 bytes produced by [start, e0)
  uint32_t nblock;      // RLE1 bytes of the whole block
  unsigned long long gx0;  // global emitted-byte prefix at e0
  uint32_t stream;      // the stream the block belongs to
  uint32_t send;        // end of that stream's input
};

// one stream of a multi-stream encode: where its input, tiles, cut-table rows and output slot lie
struct StreamDesc {
  uint32_t in0, n;                   // staged input [in0, in0 + n); in0 is a multiple of the 4 KiB input tile
  uint32_t tile0, n_tiles;           // its input tiles
  uint32_t blk0, max_blocks;         // its rows of the cut table
  unsigned long long out0, out_cap;  // its output slot in the device output (bytes; out0 a multiple of 4)
};

struct Plan {
  size_t ws_bytes;      // device workspace
  uint32_t n_tiles;     // input tiles
  uint32_t max_blocks;  // capacity of the block table
  uint32_t batch;       // blocks sorted / coded together
  uint32_t n_streams;   // streams encoded together
};
Plan plan(size_t n, size_t mem_budget);
// the plan of streams whose input tiles, cut-table rows and wanted batch add up to the given sums (plan_add per stream)
struct PlanSums {
  unsigned long long n_tiles = 0, max_blocks = 0, want = 1;
  uint32_t n_streams = 0;
};
void plan_add(PlanSums &s, size_t n);
Plan plan_of(const PlanSums &s, size_t mem_budget);
uint32_t tiles_of(size_t n);
uint32_t max_blocks_of(size_t n);
size_t bound(size_t n);

struct Stats {
  uint32_t n_blocks, n_serial_blocks, rounds, reserved, n_batches;
};

// status: 0 ok, -3 out_cap too small (*out_len = bytes needed), -6 internal
int encode_device(const uint8_t *d_in, size_t n, uint8_t *d_out, size_t out_cap, void *ws, const Plan &p, size_t *out_len,
                  Stats *stats, void *stream);

// n_streams independent streams in one pass (sd[]: host copy, streams in input order, tiles and cut rows as laid out by
// tiles_of / max_blocks_of).  out_len[i]: bytes of stream i's slot.  tile_crc (may be null): the CRC-32 (reflected, as
// zlib's) of every input tile, nt = p.n_tiles words, for crc32_fold.  status: 0 ok, -3 a slot too small, -6 internal
int encode_streams(const uint8_t *d_in, const StreamDesc *sd, uint8_t *d_out, void *ws, const Plan &p,
                   unsigned long long *out_len, uint32_t *tile_crc, Stats *stats, void *stream);
// CRC-32 of a stream of n bytes from the CRCs of its input tiles
uint32_t crc32_fold(const uint32_t *tile_crc, size_t n);

}  // namespace bz2e
}  // namespace b200z
