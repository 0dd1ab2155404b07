// inflate_chunked.h -- what the host and K12's kernels (inflate_chunked.cuh) exchange.  DESIGN.md "K12".
#pragma once
#include <stdint.h>

namespace b200z {

constexpr uint32_t CK_PAGE = 32768;  // symbols per page of the pool (64 KiB)
constexpr unsigned long long CK_NOCAND = ~0ull;
// chunk status: stopped at a block boundary at or past its stop bit / decoded a final block / the pool ran out;
// anything else is the B200Z_U_* (or U_STOP_SHORT) status the exact step stops with
constexpr int CK_BOUNDARY = 100, CK_FINAL = 101, CK_POOL = 102;

struct CkJob {
  unsigned long long start_bit, stop_bit;  // bits from the stream's first byte
  uint32_t slot, gen;                      // chunk slot in the region, attempt number (pages carry both)
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
struct CkChain {  // a proven chunk, in chain order
  unsigned long long out_off;  // absolute offset of its first byte in the output buffer
  uint32_t nsym, page0;        // symbols; its first page in the chain's flat page list
};

}  // namespace b200z
