// inflate_chunked.h -- what the host and K12's kernels (inflate_chunked.cuh) exchange.  DESIGN.md "K12".
#pragma once
#include <stdint.h>

namespace b200z {

constexpr uint32_t CK_PAGE = 32768;  // symbols per page of the pool (64 KiB)
constexpr unsigned long long CK_NOCAND = ~0ull;
// chunk status: stopped at a block boundary at or past its stop bit / decoded a final block / the pool ran out;
// anything else is the B200Z_U_* (or U_STOP_SHORT) status the exact step stops with
constexpr int CK_BOUNDARY = 100, CK_FINAL = 101, CK_POOL = 102;

// One stream of a K12 batch.  Its pages are [page0, page0 + n_pages) of the pool, counted by its own page counter, so
// that one stream's runaway output (a false start, highly compressible data) cannot starve another's chunks.
struct CkStream {
  unsigned long long in_off;    // its first compressed byte, from the batch's input base
  unsigned long long lo_valid;  // the first output byte its back-references may reach
  uint32_t in_len, page0, n_pages, pad;
};
struct CkFind {  // a block start is looked for at bits [lo, hi) of stream `stream`
  unsigned long long lo, hi;
  uint32_t stream, pad;
};
struct CkJob {
  unsigned long long start_bit, stop_bit;  // bits from the stream's first byte
  uint32_t slot;                           // chunk slot in its stream's region (pages carry it)
  uint16_t gen, stream;                    // attempt number (pages carry it too); the stream it belongs to
};
struct CkRes {
  unsigned long long end_bit;
  uint32_t nsym;
  int32_t status;
  uint32_t first_stored, pad;  // the first block decoded was a stored block
};
struct CkPage {
  uint32_t slot, seq, gen, pad;  // page `seq` of attempt `gen` of chunk `slot`
};
struct CkChain {  // a proven chunk, in chain order (the streams' chains one after another)
  unsigned long long out_off;  // absolute offset of its first byte in the output buffer
  uint32_t nsym, page0;        // symbols; its first page in the flat page list
  uint32_t stream, pad;
};

}  // namespace b200z
