// b200z_internal.h -- shared declarations between the kernels and the C-ABI layer (not installed).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <vector>

#include "../../include/b200z.h"
#include "inflate_chunked.h"

#ifndef B200Z_LBITS
#define B200Z_LBITS 9  // literal/length primary LUT bits (2^9 x u16 per stream)
#endif
#ifndef B200Z_DBITS
#define B200Z_DBITS 8  // distance primary LUT bits
#endif
#define B200Z_DECODE_THREADS 32   // one warp per block: finest block-scheduler granularity
#define B200Z_EXPAND_THREADS 256

namespace b200z {

// Device workspace of one inflate batch (inflate_kernels.cu).  `extent` = size of the output layout in bytes.
struct InflateWs {
  uint32_t *tokens = nullptr;   // [extent] u32: unit u's own tokens start at word out_off[u] (<= 1 token per output byte)
  uint32_t *htokens = nullptr;  // 7 helper planes of hstride words: helper k of unit u writes from plane k-1, word out_off[u] >> 2
  size_t hstride = 0;
  uint32_t *pieces = nullptr;   // [n_units][PIECE_WORDS]: which token runs make up the unit, in order
  uint8_t *uscratch = nullptr;  // [n_units][USCRATCH_BYTES]: slow tables + helper boundary bitmaps
  // Bytes of EARLIER output that lie directly in front of a unit's output slot and that its back-references may reach.
  // 0 for independent streams (Inflate(bytes), zip members, zlib streams: each has an output stream of its own).  GZip
  // members share ONE OutputStream in the reference (_gzip_decoder_web.dart:38: Inflate.stream(input, output: output)), so
  // a member's distance may reach into the members before it (output_memory_stream.dart:79-98 checks against the whole
  // stream): the member-by-member path sets this for its single-unit batches.
  uint32_t hist = 0;
  // The same per unit ([n_units], device memory) when the units of one batch have different histories (members of many
  // gzip streams decoded together); it takes the place of `hist` when set.
  const uint32_t *unit_hist = nullptr;
};
size_t inflate_ws_bytes(size_t n_units, size_t extent);
// largest extent a workspace of `bytes` serves (extent 0 is valid); INFLATE_WS_TOO_SMALL when it serves none
constexpr size_t INFLATE_WS_TOO_SMALL = ~(size_t)0;
size_t inflate_ws_extent_for(size_t n_units, size_t bytes);
InflateWs inflate_ws_carve(void *ws, size_t n_units, size_t extent);
InflateWs inflate_ws_slice(const InflateWs &w, size_t first_unit, size_t first_out_byte);

struct InflateBatch {
  const uint8_t *in_base;
  const uint64_t *in_off;
  const uint32_t *in_len;
  uint8_t *out_base;
  const uint64_t *out_off;
  const uint32_t *out_cap;
  uint32_t *out_len;
  int32_t *status;
  uint32_t *in_used;
  size_t n_units;
  InflateWs ws;
  int share = 1;     // how many batches run concurrently on the device (sizes the streams-per-warp choice)
  bool count_only = false;  // sizes only: out_len / status / in_used, no tokens, no output bytes
};

cudaError_t launch_inflate(const InflateBatch &b, cudaStream_t stream);
// K12 (inflate_chunked.cuh) over a batch of streams; `streams` is the device copy of the batch's stream table
cudaError_t ck_launch_find(const uint8_t *in_base, const CkStream *streams, const CkFind *finds, unsigned long long *cand,
                           uint32_t n, cudaStream_t s);
cudaError_t ck_launch_chunks(const uint8_t *in_base, const CkStream *streams, const CkJob *jobs, uint32_t n, CkRes *res,
                             uint16_t *pool, CkPage *pinfo, uint32_t *page_ctr, cudaStream_t s);
// windows: one CTA per chain walk chain[chain_lo[w] .. chain_lo[w + 1]); then emit over the n_flat pages of all of them
cudaError_t ck_launch_resolve(const CkChain *chain, const uint32_t *chain_lo, uint32_t n_walks, const uint32_t *flat,
                              const uint32_t *flat_chunk, uint32_t n_flat, const uint16_t *pool, uint8_t *out,
                              const CkStream *streams, uint32_t *bad, cudaStream_t s);
cudaError_t launch_find_markers(const uint8_t *d_in, size_t n, unsigned long long *d_list, uint32_t *d_count, uint32_t cap,
                                cudaStream_t stream);

// ---- BZip2 (bzip2_kernels.cu) ----
struct Bz2Entropy {  // K7, one warp per candidate block
  const uint32_t *words;
  uint64_t n_bytes;
  const unsigned long long *blk_bit;  // bit position of each candidate's 48-bit magic
  uint32_t n_blocks, nblock_max;
  uint32_t *rec_val, *rec_pos;  // [n_blocks][nblock_max]
  uint32_t *n_rec, *nblock, *orig_ptr, *randomised;
  unsigned long long *end_bit;
  int32_t *status;
  uint32_t *fast_flag = nullptr;  // [n_blocks], may be null: 1 = the block was decoded by k_bz2_entropy_fast
  uint8_t *sym8 = nullptr;        // [n_blocks][nblock_max]: K8's byte array, by candidate slot (the fast kernel writes it)
  // [n_blocks], both may be null (every block then ends at n_bytes and has the limit nblock_max): the bit where the block's
  // stream ends in `words` (reads from there on see zeros and are past the end) and its stream's level x 100000.  nblock_max
  // stays the stride of the per-block arrays.
  const unsigned long long *blk_end = nullptr;
  const uint32_t *blk_lim = nullptr;
};
struct Bz2Ibwt {  // K8 over the validated chain
  const void *chain;  // BzChain[n_chain] (device)
  uint32_t n_chain, nblock_max;
  const uint32_t *rec_val, *rec_pos;
  uint8_t *sym8;    // [n_chain][nblock_max]
  uint32_t *chist;  // [n_chain][chunks_max][256]
  uint32_t *tt;     // [n_chain][nblock_max]
  uint32_t *seg_len, *seg_next, *seg_off;  // [n_chain][4098]
  uint32_t *seg_resume;                    // [n_chain][4098]: where the walk of a segment stood when its slot was full
  uint8_t *slots;                          // [n_chain][4098][bz2_slot_bytes_per_block() / 4098]: a segment's bytes before they are placed
  uint32_t *walk_ctr;                      // [2]: the work counters of k_bz2_walk_len / k_bz2_walk_emit
  int32_t *irregular;                      // [n_chain]
  uint32_t *cycle_len;                     // [n_chain]
  uint8_t *raw;                            // [n_chain][nblock_max]
  uint32_t *slice_state, *slice_out;       // [n_chain][1024]
  unsigned long long *block_out, *block_off;  // [n_chain], [n_chain + 1]
  uint32_t *block_crc;                         // [n_chain]
  uint8_t *out;
  unsigned long long out_cap;
  bool any_randomised = false;
  bool carry_off = false;  // block_off[0] already holds the first block's offset (bz2_launch_ibwt_group)
  bool any_records = true; // some block of the chain comes with records (the exact kernels'; long runs of the fast one)
  int phase = 0;           // 0: all of K8; 1: everything up to the blocks' output offsets; 2: the RLE1 output pass only
};
struct BzChainHost {
  uint32_t cand, nblock, n_rec, orig_ptr;
  uint32_t flags;  // bit 0: randomised block (serial path in K8); bit 1: first block of its stream (output starts at out_lo)
  uint32_t pad_ = 0;
  unsigned long long out_lo = 0, out_hi = ~0ull;  // the stream's output slot in Bz2Ibwt::out (clipped at out_cap as well)
};
struct Bz2ScanStream {
  unsigned long long off, len;  // bytes of Bz2Scan::in
};
struct Bz2Scan {  // K6
  const uint8_t *in = nullptr;
  uint64_t n_bytes = 0;                            // without a stream table: one stream, in[0, n_bytes)
  const Bz2ScanStream *streams = nullptr;          // [n_streams] (device), or null
  const unsigned long long *first_thr = nullptr;   // [n_streams + 1]: first thread of each stream (4 bytes each, at least one)
  uint32_t n_streams = 0;
  unsigned long long *cand = nullptr;              // [cap]: bit in `in` | end-of-stream << 63
  uint32_t *n_cand = nullptr, cap = 0;
  uint32_t *cand_stream = nullptr, *cand_crc = nullptr;  // [cap], with a stream table: its stream, the 32 bits behind the magic
  uint8_t *ends = nullptr;                         // [n_streams][12], with a stream table: first 4 and last 8 bytes (0 where none)
};
size_t bz2_entropy_smem();
cudaError_t bz2_launch_scan(const uint8_t *d_in, uint64_t n_bytes, unsigned long long *d_cand, uint32_t *d_ncand,
                            uint32_t cap, cudaStream_t s);
cudaError_t bz2_launch_scan_streams(const Bz2Scan &a, uint64_t n_threads, cudaStream_t s);
cudaError_t bz2_launch_entropy(const Bz2Entropy &a, cudaStream_t s);
// blocks K7 left with status -3 (a damaged block that the reference keeps decoding): d_list = their indices into a's arrays
cudaError_t bz2_launch_entropy_literal(const Bz2Entropy &a, const uint32_t *d_list, uint32_t n_list, cudaStream_t s);
size_t bz2_slot_bytes_per_block();
cudaError_t bz2_launch_ibwt(const Bz2Ibwt &a, cudaStream_t s);
cudaError_t bz2_launch_ibwt_group(const Bz2Ibwt &a, uint32_t lo, uint32_t hi, cudaStream_t s);
void count_launch();
// The device sink of the decode batches (b200z_*_decode_batch_to_device): one copy of `len` bytes from the library's group
// buffer (src + src) into a slot of the caller's device buffer (dst + dst).
struct SlotCopy {
  uint64_t src, dst, len;
};
// every copy of `copies` as one k_copy_slots launch on stream s, not synchronised (nothing when there is no byte to copy);
// the table goes up on s, so launches on one stream may follow each other freely
cudaError_t copy_slots(const uint8_t *src, uint8_t *dst, const SlotCopy *copies, size_t n, cudaStream_t s);
void profile_enable(bool on);
int profile_read(double *fast_ms, double *decode_ms, double *expand_ms, uint64_t *n);

// ---- file streams (b200z_file.cu) and the hooks it uses (b200z_api.cu) ----
void set_error_text(const char *msg);  // b200z_last_error() text of the calling thread
size_t gzip_hinted_prefix(const uint8_t *in, size_t n, size_t *out_bytes);
struct HintedMember {
  size_t hdr_end, next;  // first byte of the DEFLATE stream; first byte behind the member
  uint32_t isize;
};
// the run of members from `pos` on that carry the BGZF 'BC' size and a believable ISIZE (b200z_api.cu: hinted_run)
size_t gzip_hinted_members(const uint8_t *in, size_t n, size_t pos, std::vector<HintedMember> *ms, size_t *out_bytes);
int gzip_decode_hinted(const uint8_t *in, size_t n, uint8_t *out, size_t out_cap, size_t *in_used, size_t *out_len);
int gzip_decode_after(const uint8_t *in, size_t n, int verify, const uint8_t *hist, size_t hist_len, uint8_t *out, size_t out_cap,
                      size_t *out_len);
void file_release();  // frees the pinned segment buffers (b200z_shutdown)

// ---- Deflate (deflate_kernels.cu) ----
struct DeflStoredBlock {
  uint32_t start, len, eof;
};
size_t deflate_bound(size_t n);
// levels 1-3 over a batch (k_defl_fast_batch): where one member's bytes are and where its tokens go (device pointers;
// tok / tally_ss / next_ss hold n + 2 words each)
struct DeflFastMember {
  const uint8_t *d = nullptr;
  uint32_t n = 0, pad_ = 0;
  uint32_t *tok = nullptr, *tally_ss = nullptr, *next_ss = nullptr, *ntok = nullptr;
};
cudaError_t deflate_fast_tokens_batch(const DeflFastMember *d_list, uint32_t n_mem, int level, int window_bits, uint32_t *d_counter,
                                      cudaStream_t s);
size_t deflate_workspace_bytes(size_t n);
cudaError_t deflate_slow_device(const uint8_t *d_in, size_t n, int level, int window_bits, uint8_t *d_out, size_t out_cap,
                                void *ws, size_t ws_bytes, size_t *out_len, uint32_t *stats, cudaStream_t s, const DeflFastMember *pre = nullptr);
cudaError_t deflate_stored_device(const uint8_t *d_in, const DeflStoredBlock *h_blocks, uint32_t n_blocks, uint8_t *d_out,
                                  size_t out_cap, void *ws, size_t ws_bytes, size_t *out_len, cudaStream_t s);
cudaError_t crc32_tiles_device(const uint8_t *d_in, size_t n, uint32_t tile, uint32_t *d_part, cudaStream_t s);
// CRC-32 of device bytes d[0, n) on stream s (blocking): tiles of 8 KiB into d_part ((n / 8192 + 1) words), folded on the host
int device_crc32_on(const uint8_t *d, size_t n, uint32_t *d_part, cudaStream_t s, uint32_t *out);

// ---- encrypted ZIP members (zip_crypt_kernels.cu) ----
struct ZipAesMember {   // one WinZip AES member; offsets are bytes from the device base pointer of the call
  uint64_t src_off;     // ciphertext (decrypt) / plaintext (encrypt)
  uint64_t dst_off;     // where the CTR pass writes (may equal src_off)
  uint64_t len;         // bytes of ciphertext
  uint32_t salt_len;    // 8 / 12 / 16
  uint32_t key_len;     // 16 / 24 / 32
  uint8_t salt[16];
};
struct ZipCryptoMember {  // one ZipCrypto member: len bytes at src_off (12-byte header included) -> len - 12 at dst_off
  uint64_t src_off, dst_off, len;
};
struct ZipCtrTile {  // one CTA of k_zip_aes_ctr: zip_ctr_tile_blocks() 16-byte blocks of one member from first_block on
  uint64_t first_block;
  uint32_t member, pad_;
};
struct ZipHmacPads {  // SHA-1 states after the HMAC inner / outer pad block of the password
  uint32_t ipad[5], opad[5];
};
void zip_hmac_pads(const uint8_t *key, size_t klen, ZipHmacPads *p);
void zipcrypto_keys(const uint8_t *pw, size_t len, uint32_t k[3]);  // the three keys after the password (host)
uint64_t zip_ctr_tile_blocks();
// d_dk: 80 bytes per member (derived key), d_rk: 60 words per member (AES round keys), d_ver: 2 bytes per member
cudaError_t zip_launch_pbkdf2(const ZipAesMember *d_m, uint32_t n, const ZipHmacPads &pads, uint8_t *d_dk, uint32_t *d_rk,
                              uint8_t *d_ver, cudaStream_t s);
cudaError_t zip_launch_aes_ctr(const ZipAesMember *d_m, const uint32_t *d_rk, const ZipCtrTile *d_tiles, uint32_t n_tiles,
                               uint8_t *d_base, cudaStream_t s);
// 10 bytes of MAC per member over the bytes at src_off, or at dst_off when after_ctr (encryption: MAC of the ciphertext)
cudaError_t zip_launch_hmac(const ZipAesMember *d_m, uint32_t n, const uint8_t *d_dk, const uint8_t *d_base, bool after_ctr,
                            uint8_t *d_mac, cudaStream_t s);
cudaError_t zip_launch_zipcrypto(const ZipCryptoMember *d_m, uint32_t n, const uint32_t keys[3], uint8_t *d_base, cudaStream_t s);

// ---- XZ (xz_kernels.cu): host buffers in, host buffers out, blocking on `s` ----
size_t xz_bound(const uint8_t *in, size_t n);  // the output the container declares, up to where its walk stops
// n streams (arguments checked): rc[i] / out_len[i] / bytes as xz_decode_impl / xz_encode_impl give for stream i alone;
// the return value is B200Z_OK, B200Z_E_ARG (encode: a bad check kind) or a device failure.  dev_out: out_base is device
// memory (the decode's bytes go to the slots through k_copy_slots, one launch per device group)
int xz_decode_streams(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                      uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len, int32_t *rc,
                      cudaStream_t s, bool dev_out = false);
// CRC-32 (getCrc32) of each tile d[tile_off[t], + tile_len[t]) into part[t]: one k_crc_tiles<uint32_t> launch on s, not
// synchronised (nothing when n_tiles == 0); the caller folds the tiles of a range with the x^(8n) mod P combine
cudaError_t crc32_tiles_launch(const uint8_t *d, const uint64_t *tile_off, const uint32_t *tile_len, uint32_t n_tiles,
                               uint32_t *part, cudaStream_t s);
int xz_encode_streams(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int check,
                      uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len, int32_t *rc,
                      cudaStream_t s);
// the batch of one
int xz_decode_impl(const uint8_t *in, size_t n, int verify, uint8_t *out, size_t out_cap, size_t *out_len, cudaStream_t s);
int xz_crc64_impl(const uint8_t *in, size_t n, uint64_t *crc, cudaStream_t s);
size_t xz_encode_bound(size_t n);
int xz_encode_impl(const uint8_t *in, size_t n, int check, uint8_t *out, size_t out_cap, size_t *out_len, cudaStream_t s);
void xz_debug(double *lzma_ms, uint32_t *n_runs);  // k_xz_lzma time (CUDA events) and run count of the last decode call
void xz_batch_set(uint32_t max_streams);           // test hook: streams per device group (0: the memory budget alone)
void xz_batch_stats(unsigned long long out[3]);    // the last decode call's streams, device groups and runs

}  // namespace b200z
