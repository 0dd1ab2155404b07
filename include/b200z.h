/*
 * b200z.h -- C ABI of libb200z.so: H100 (sm_90a) DEFLATE / BZip2 block codecs behind the
 * Dart `archive` package's codec classes.
 *
 * The reference (brendan-duncan/archive 4.2.0) is pure Dart and has no FFI of its own; the
 * entry points below are what a `dart:ffi` binding for its codec hot path binds (see
 * INTEGRATION.md and dart/lib/src/b200z_ffi.dart).  Each entry point cites the reference
 * interface it replaces (paths relative to /root/reference/).
 *
 * Conventions
 *   - plain pointers + sizes, no C++ / torch types; every call is blocking.
 *   - one process drives ONE GPU (b200z_init(device)); multi-GPU = one process per GPU,
 *     units sharded by the caller (bench.py / torchrun), see DESIGN.md "Multi-GPU".
 *   - return value: 0 (B200Z_OK) or a negative B200Z_E_* code.  The reference's error
 *     convention on this path is "stop, keep partial output, never throw"
 *     (inflate.dart:150-151,166-168; bzip2_decoder.dart:32-78): data errors therefore still
 *     produce the partial output the reference would have produced, and the per-stream
 *     status says why decoding stopped.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails with
 *     B200Z_E_NODEVICE.
 */
#ifndef B200Z_H
#define B200Z_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes -------------------------------------------------------------------- */
#define B200Z_OK 0
#define B200Z_E_NODEVICE (-1) /* no CUDA device / b200z_init not called / CUDA runtime error   */
#define B200Z_E_ARG (-2)      /* invalid argument (Deflate._init returning false, deflate.dart:107-118) */
#define B200Z_E_NOSPC (-3)    /* out_cap too small; *out_len = bytes needed when known          */
#define B200Z_E_DATA (-4)     /* decodeStream() returned false (bad header / adler / crc)       */
#define B200Z_E_THROW (-5)    /* the Dart code would have thrown (RangeError: distance > output,
                                 output_memory_stream.dart:83-86; code-length overrun inflate.dart:359) */
#define B200Z_E_INTERNAL (-6)

/* per-unit status written by the batch decoders (int32) */
#define B200Z_U_DONE 0       /* BFINAL block decoded (inflate.dart:155)                          */
#define B200Z_U_EOS 1        /* input exhausted before a final block (inflate.dart:111 loop end)  */
#define B200Z_U_STOP (-1)    /* _parseBlock returned false: bad block type / code / short read    */
#define B200Z_U_NOSPC (-2)   /* unit output would exceed out_cap                                  */
#define B200Z_U_RANGE (-3)   /* back-reference before start of output (Dart RangeError)           */
#define B200Z_U_BADCODE (-4) /* over-subscribed or unusable Huffman code set (reference would
                                decode garbage / never terminate; see DESIGN.md "Divergences")    */
#define B200Z_U_THROW (-5)   /* code-length run overruns HLIT+HDIST (Dart RangeError)             */
#define B200Z_U_TOKCAP (-6)  /* internal token buffer too small (library retries)                 */

/* ---- lifetime ------------------------------------------------------------------------ */
int b200z_init(int device, uint32_t flags); /* selects the GPU for this process; idempotent  */
void b200z_shutdown(void);
const char *b200z_last_error(void); /* thread-local, never NULL                      */
int b200z_device_count(void);       /* 0 when no CUDA device is visible              */
const char *b200z_version(void);

/* pinned host memory for callers that want full-speed PCIe copies (Dart: Pointer<Uint8>) */
void *b200z_host_alloc(size_t bytes);
void b200z_host_free(void *p);

/* ---- single stream, reference class semantics ---------------------------------------- */
/* Inflate(bytes).getBytes()  -- inflate.dart:23-28,102.  Raw DEFLATE.  *in_consumed is where
 * the reference leaves the input stream (inflate.dart:337-340).  *unit_status = B200Z_U_*.  */
int b200z_inflate_raw(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap,
                      size_t *out_len, size_t *in_consumed, int32_t *unit_status);

/* GZipDecoderWeb().decodeBytes -- _gzip_decoder_web.dart:19-58 (member loop, header skip,
 * CRC/ISIZE read and ignored, zlib fallback when there is no gzip header).  The members share
 * one output stream, as in the reference (:38): a member's back-references may reach into the
 * members decoded before it.  A stream that ends inside a block: B200Z_E_THROW (the reference's
 * trailer read runs past the end), with the bytes decoded so far in `out`.                  */
#define B200Z_GZIP_VERIFY 1 /* bits of `verify`: verify, and the `raw` the reference hands on to the zlib decoder when */
#define B200Z_GZIP_RAW 2    /* the input has no gzip header (_gzip_decoder_web.dart:31-37)                            */
int b200z_gzip_decode(const uint8_t *in, size_t in_len, int verify, uint8_t *out, size_t out_cap,
                      size_t *out_len);
/* ZLibDecoderWeb().decodeBytes -- _zlib_decoder_web.dart:21-107 (stream loop, Adler-32 when
 * verify, raw = no wrapper).  Every stream has an output of its own and reaches `out` only once
 * the next stream's header has been accepted, or at the end (:82-84, :101-103).            */
int b200z_zlib_decode(const uint8_t *in, size_t in_len, int verify, int raw, uint8_t *out,
                      size_t out_cap, size_t *out_len);
/* Upper bound for the output of b200z_gzip_decode / b200z_zlib_decode, from the framing's own
 * size fields where present (ISIZE), else 0 = unknown (call with a guess, retry on E_NOSPC). */
size_t b200z_gzip_bound(const uint8_t *in, size_t in_len);

/* Deflate(bytes, level:, windowBits:).getBytes() and .crc32 -- deflate.dart:39-48,72-75,31.  Raw DEFLATE, byte-identical
 * to the reference at the same level and windowBits (9..15).  Levels 4-9 are data parallel inside a stream; 1-3
 * (deflate_fast, whose hash chains depend on the parse) are one warp per stream with all state in shared memory -- their
 * parallel axis is the batch (b200z_deflate_batch); 0 is stored.  Invalid level / windowBits
 * (Deflate._init returning false, :107-118) -> B200Z_E_ARG.                                                          */
int b200z_deflate_raw(const uint8_t *in, size_t in_len, int level, int window_bits, uint8_t *out, size_t out_cap,
                      size_t *out_len, uint32_t *crc32_of_input);
size_t b200z_deflate_bound(size_t in_len); /* output capacity that always suffices (+18 for gzip, +6 for zlib) */
/* n_units independent Deflate(bytes, level:, windowBits:) streams in one call -- what ZipEncoder does member by member
 * (zip_encoder.dart:185-259, platformZLibEncoder.encodeStream(raw: true) :244-249).  Unit u reads
 * in_base[in_off[u] .. +in_len[u]) and writes out_base[out_off[u] .. +out_cap[u]); out_len[u] = its compressed size,
 * crc32[u] (may be NULL) = CRC-32 of its input, status[u] = B200Z_OK or B200Z_U_NOSPC (out_len[u] = bytes needed).  All
 * inputs are staged at once and up to 8 members (B200Z_DEFLATE_LANES) are in flight on separate CUDA streams; at levels
 * 1-3 the match finding of ALL members runs first, as one launch with a warp per member.  Every stream is byte-identical
 * to b200z_deflate_raw of the same input.                                                                            */
int b200z_deflate_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n_units, int level,
                        int window_bits, uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                        uint64_t *out_len, uint32_t *crc32, int32_t *status);
/* ZLibEncoderWeb().encodeBytes -- _zlib_encoder_web.dart:17-73 (header 78 01 at every level, Adler-32 trailer)      */
int b200z_zlib_encode(const uint8_t *in, size_t in_len, int level, int window_bits, int raw, uint8_t *out,
                      size_t out_cap, size_t *out_len);
/* GZipEncoderWeb().encodeBytes -- _gzip_encoder_web.dart:17-100 (MTIME is "now" in the reference: a parameter here) */
int b200z_gzip_encode(const uint8_t *in, size_t in_len, int level, uint32_t mtime, uint8_t *out, size_t out_cap,
                      size_t *out_len);
/* n independent b200z_gzip_decode / b200z_zlib_decode calls in one.  Stream i reads in_base[in_off[i] .. +in_len[i]) and
 * writes out_base[out_off[i] .. +out_cap[i]); rc[i], out_len[i] and the bytes in its slot (up to out_len[i]) are exactly
 * what the single call gives for that stream alone with out_cap[i]: B200Z_OK, B200Z_E_DATA and B200Z_E_THROW with their
 * partial output, B200Z_E_NOSPC with the same out_len (the slot's contents unspecified).  `verify` of the gzip batch takes
 * the B200Z_GZIP_VERIFY / B200Z_GZIP_RAW bits, as b200z_gzip_decode.  Input ranges may overlap or repeat; n == 0 is OK.
 * Returns B200Z_OK unless an argument is wrong (null arrays, wrapping ranges, overlapping output slots: B200Z_E_ARG and
 * nothing is written) or the device fails.  All inputs of a device group go up in one copy; per round, the hinted runs and
 * the next member / zlib stream of every stream are one inflate batch, so a batch of single-member files is one launch
 * chain where one call per file keeps one CTA busy.                                                                  */
int b200z_gzip_decode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                            uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len, int32_t *rc);
int b200z_zlib_decode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                            int raw, uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len,
                            int32_t *rc);
/* n independent b200z_gzip_encode / b200z_zlib_encode calls in one: rc[i], out_len[i] and the slot's bytes as the single
 * call gives them (B200Z_E_NOSPC: out_len[i] = the size needed, b200z_deflate_bound + 18 always suffices; an input of
 * 4 GiB or more: B200Z_E_ARG, the others are still encoded).  An invalid level or windowBits is B200Z_E_ARG for the
 * whole call; otherwise the argument rules of b200z_gzip_decode_batch.  One deflate batch (b200z_deflate_batch) for all
 * inputs; the Adler-32 of all zlib inputs is one launch.                                                            */
int b200z_gzip_encode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int level,
                            uint32_t mtime, uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                            uint64_t *out_len, int32_t *rc);
int b200z_zlib_encode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int level,
                            int window_bits, int raw, uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                            uint64_t *out_len, int32_t *rc);

/* BZip2Decoder().decodeBytes(data, verify:) -- bzip2_decoder.dart:13-88.  Stops after the first end-of-stream
 * block; CRCs are compared only when verify; B200Z_E_DATA == decodeStream returning false (the blocks decoded
 * before the failure are kept, as in the reference).                                                    */
int b200z_bzip2_decode(const uint8_t *in, size_t in_len, int verify, uint8_t *out, size_t out_cap,
                       size_t *out_len);
/* n independent BZip2Decoder().decodeBytes(data, verify:) calls in one.  Stream i reads in_base[in_off[i] .. +in_len[i])
 * and writes out_base[out_off[i] .. +out_cap[i]); rc[i] and out_len[i] are exactly what b200z_bzip2_decode returns and
 * reports for that stream alone (B200Z_OK / _E_DATA / _E_THROW / _E_NOSPC), and so are the bytes in its slot (up to
 * out_len[i]; after B200Z_E_NOSPC the slot's contents are unspecified, as after a single call).  The call
 * returns B200Z_OK unless an argument is wrong or the device fails; n == 0 is OK.  Input ranges may overlap or repeat;
 * output slots must not overlap.  All inputs go to the device in one copy, one scan finds the blocks of all streams, and
 * the streams share the entropy and inverse-BWT launches (in groups that fit the device memory).                     */
int b200z_bzip2_decode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                             uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len,
                             int32_t *rc);
/* One rank's share of a BZip2 stream (SURVEY.md 8e: blocks are independent once the bit-level magic scan has found
 * them; only the combined CRC and the output offsets chain across blocks).  Rank `rank` of `world` decodes the block
 * candidates [n*rank/world, n*(rank+1)/world) into `out`, back to back, and reports EVERY candidate of its share plus
 * the end-of-stream candidates: the caller merges the reports of all ranks, walks the chain as decodeStream does
 * (bzip2_decoder.dart:46-87: a block must start where the previous one ended), checks the CRCs and derives the output
 * offsets (archive_b200/shard.py: bzip2_decode_sharded).                                                         */
typedef struct {
  uint64_t start_bit, end_bit; /* position of the 48-bit magic; first bit after the block's last symbol */
  uint64_t out_bytes;          /* decoded size (0 when the block could not be decoded)                  */
  uint32_t crc_calc, crc_stored;
  int32_t status;              /* 0 ok, -1 data error, -2 read past the end of the input               */
  uint32_t flags;              /* B200Z_BZ2_*                                                           */
} b200z_bz2_block;
#define B200Z_BZ2_EOS 1u            /* an end-of-stream magic (crc_stored = the combined CRC) */
#define B200Z_BZ2_RANDOMISED 2u     /* (unused: randomised blocks are decoded)                */
#define B200Z_BZ2_CORRUPT_CYCLE 4u  /* inverse BWT is not one cycle: not decoded              */
#define B200Z_BZ2_OVERRUN 8u        /* the run-length walk overran the block (bzip2_decoder.dart:497-499, 628-631):
                                     * its bytes ARE written, then decodeStream returns false */
int b200z_bzip2_decode_shard(const uint8_t *in, size_t in_len, uint32_t rank, uint32_t world, uint8_t *out,
                             size_t out_cap, size_t *out_len, b200z_bz2_block *blocks, size_t blocks_cap,
                             size_t *n_blocks);
/* BZip2Encoder().encodeBytes(data) -- bzip2_encoder.dart:15-81: always "BZh9", never randomised, the pending RLE1
 * run is closed at every block end (which is where the bytes differ from libbzip2 on multi-block inputs).
 * Inputs of 4 GiB and more: B200Z_E_ARG.                                                                       */
int b200z_bzip2_encode(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, size_t *out_len);
size_t b200z_bzip2_bound(size_t in_len); /* output capacity that always suffices */
/* n independent BZip2Encoder().encodeBytes(data) calls in one.  Stream i reads in_base[in_off[i] .. +in_len[i]) and
 * writes out_base[out_off[i] .. +out_cap[i]); rc[i], out_len[i] and the bytes in its slot are exactly what
 * b200z_bzip2_encode gives for that stream alone: B200Z_OK, B200Z_E_NOSPC (out_len[i] = the size needed, the slot's
 * contents unspecified) or B200Z_E_ARG for a stream of 4 GiB or more (the others are still encoded).  crc32 may be
 * NULL; otherwise crc32[i] = getCrc32 of stream i's input (crc32.dart, as b200z_crc32), computed on the device.  The
 * call returns B200Z_OK unless an argument is wrong (null arrays, wrapping ranges, overlapping output slots: nothing
 * is written) or the device fails; n == 0 is OK.  Input ranges may overlap or repeat.  All inputs go to the device in
 * one copy, and blocks of different streams share the sort, MTF and entropy launches (in groups that fit the device
 * memory).                                                                                                        */
int b200z_bzip2_encode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n,
                             uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len,
                             uint32_t *crc32, int32_t *rc);

/* getCrc32(bytes) -- crc32.dart:6-27 (CRC-32, reflected 0xEDB88320) of a host buffer, computed on the device (tile CRCs
 * folded with x^(8n) mod P): what ZipEncoder stores for members it does not deflate (zip_encoder.dart:113-134).   */
int b200z_crc32(const uint8_t *in, size_t in_len, uint32_t *crc);

/* ---- XZ: XZDecoder / XZEncoder (codecs/xz_decoder.dart, codecs/xz_encoder.dart, codecs/lzma/) ------------------------
 * b200z_xz_decode = XZDecoder().decodeBytes(data, verify:): ONE stream (bytes after its footer are ignored).  The host walks
 * the container and every LZMA2 chunk header; the runs between dictionary resets are decoded on the device in parallel
 * (one warp each), stored chunks are copies.  B200Z_OK: decodeStream returned true.  B200Z_E_DATA: it returned false, and
 * `out` holds the bytes the reference would have written.  B200Z_E_THROW: the reference throws (a read past the input or
 * a chunk's compressed bytes, a reach before the dictionary, posState >= 12 with pb = 4 or 5, or a match that runs past
 * its chunk's declared size -- DESIGN.md section 7).  B200Z_E_NOSPC: out_cap is below b200z_xz_bound, *out_len = that.
 * With `verify`, CRC-32 / CRC-64 block checks are compared (on the device); SHA-256 is read and never compared.
 * b200z_xz_bound (host only): the output the container declares up to where its walk stops; 0 when it declares none.
 * b200z_xz_encode = XZEncoder().encodeBytes(data, check:) with check 0 none, 1 crc32, 2 crc64, 3 sha256 (XZCheck.index):
 * one stored chunk whose 16-bit length field is cut for inputs over 64 KiB, as in the reference.
 * b200z_crc64 = getCrc64(bytes) (util/_crc64_io.dart: ECMA-182, reflected), tile CRCs on the device folded on the host. */
int b200z_xz_decode(const uint8_t *in, size_t in_len, int verify, uint8_t *out, size_t out_cap, size_t *out_len);
size_t b200z_xz_bound(const uint8_t *in, size_t in_len);
int b200z_xz_encode(const uint8_t *in, size_t in_len, int check, uint8_t *out, size_t out_cap, size_t *out_len);
size_t b200z_xz_encode_bound(size_t in_len);
int b200z_crc64(const uint8_t *in, size_t in_len, uint64_t *crc);
/* b200z_xz_decode_batch = n independent XZDecoder().decodeBytes(data, verify:) calls in one.  Stream i reads
 * in_base[in_off[i] .. +in_len[i]) and writes out_base[out_off[i] .. +out_cap[i]); rc[i], out_len[i] and the bytes in its
 * slot are exactly what b200z_xz_decode gives for that stream alone (OK / E_DATA / E_THROW / E_NOSPC with out_len[i] =
 * b200z_xz_bound, which is the room that always suffices).  Input ranges may overlap or repeat; n == 0 returns OK.  Returns
 * OK unless an argument is wrong (null arrays, wrapping ranges, overlapping output slots: B200Z_E_ARG and nothing is
 * written) or the device fails.  The runs of all streams share one k_xz_lzma launch, so many single-block streams (one
 * warp each) fill the GPU where one call per stream keeps one warp busy; streams are cut into consecutive device groups
 * that fit the device memory.
 * b200z_xz_encode_batch = n independent XZEncoder().encodeBytes(data, check:) calls in one, one check kind for all (0..3
 * as b200z_xz_encode, anything else is B200Z_E_ARG); rc[i] / out_len[i] / bytes as b200z_xz_encode for that stream alone
 * (E_NOSPC: out_len[i] = the size needed, b200z_xz_encode_bound always suffices).  The checks of all streams are one
 * launch: CRC tiles, or SHA-256 with one thread per message.  The same argument rules as b200z_xz_decode_batch.      */
int b200z_xz_decode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                          uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len, int32_t *rc);
int b200z_xz_encode_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int check,
                          uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len, int32_t *rc);

/* ---- decode batches into device memory ------------------------------------------------------------------------------
 * b200z_gzip_decode_batch_to_device / _zlib_ / _bzip2_ / _xz_ = the host batch of the same name with the output slots in
 * device memory, so that decoded bytes never make the round trip through the host.
 *   Memory: the inputs and every array (in_off, in_len, out_off, out_cap, out_len, rc) are host memory, as in the host
 *     batch (the framing rules read the compressed bytes on the host).  d_out_base is device memory on the b200z_init device.
 *   Results: for every stream, rc[i], out_len[i] and the bytes in the slot d_out_base[out_off[i] .. +out_cap[i]) are exactly
 *     what the host batch gives for the same arguments; after B200Z_E_NOSPC the slot's contents are unspecified.  Nothing is
 *     written outside the slots; slots may come in any order, leave gaps and start at any byte alignment.
 *   Argument errors: the host batch's rules (null arrays, wrapping ranges, overlapping slots), and d_out_base must be device
 *     memory of the library's device (cudaPointerGetAttributes) whenever a slot has room: B200Z_E_ARG, nothing is written.
 *     n == 0 is OK.  No device (b200z_init not called or failed): B200Z_E_NODEVICE.
 *   Ordering: the library's stream waits on an event recorded on cuda_stream (a cudaStream_t; NULL = the library's own
 *     stream, cudaStreamLegacy for the legacy default stream) when the call starts, so work enqueued there before the call
 *     comes before any write to the slots.  The call returns once the bytes are in place, like the host batches: the output
 *     may be used on any stream from then on.
 * Each device group's results go from the library's buffer into the slots with one k_copy_slots launch (one per delivery
 * point for BZip2), whatever the number of streams.                                                                     */
int b200z_gzip_decode_batch_to_device(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                                      uint8_t *d_out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len,
                                      int32_t *rc, void *cuda_stream);
int b200z_zlib_decode_batch_to_device(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                                      int raw, uint8_t *d_out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                      uint64_t *out_len, int32_t *rc, void *cuda_stream);
int b200z_bzip2_decode_batch_to_device(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n,
                                       int verify, uint8_t *d_out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                       uint64_t *out_len, int32_t *rc, void *cuda_stream);
int b200z_xz_decode_batch_to_device(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n, int verify,
                                    uint8_t *d_out_base, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len,
                                    int32_t *rc, void *cuda_stream);

/* ---- ZIP container: ZipDecoder / ZipDirectory / ZipFileHeader / ZipFile ------------------------------------
 * b200z_zip_list   = ZipDirectory.read (zip_directory.dart:25-183) + ZipFileHeader.read (zip_file_header.dart:28-111)
 *                    + ZipFile.read (zip_file.dart:73-149), host only: no device is needed.
 * b200z_zip_extract = ZipFile.getStream / decompress (zip_file.dart:164-249) for ALL listed members at once: the deflate
 *                    members are one batch of the inflate kernels, stored members are copies, the bzip2 members
 *                    are one BZip2 batch (b200z_bzip2_decode_batch) on the staged archive.  Names are byte ranges of
 *                    the archive (decoding them is the host language's business).  Encrypted members (ZipCrypto / AES) are reported, not decoded, unless a
 *                    password is given (b200z_zip_extract_password).                                                    */
typedef struct {
  uint64_t local_header_off; /* ZipFileHeader.localHeaderOffset (zip64 applied)                               */
  uint64_t data_off;         /* first byte of the member's data; valid when has_data                          */
  uint64_t comp_size;        /* bytes of member data (central directory value, clipped to the archive)        */
  uint64_t uncomp_size;      /* ZipFile.uncompressedSize: central directory value, or the data descriptor's   */
  uint64_t hint_uncomp_size; /* the central directory value (a size hint only: the data decide)               */
  uint64_t name_off, cd_name_off; /* file name in the local header (what ZipFile.filename is) / in the directory */
  uint32_t name_len, cd_name_len;
  uint32_t crc32, method, flags; /* from the local header (CRC from the data descriptor when flag bit 3 is set) */
  uint32_t mod_time, mod_date, ext_attr, version_made_by;
  uint32_t has_data;         /* 0: no local header signature at local_header_off -> empty content              */
} b200z_zip_entry;
int b200z_zip_list(const uint8_t *zip, size_t zip_len, b200z_zip_entry *entries, size_t cap, size_t *n_entries);
/* ZipDirectory.zipFileComment: byte range of the archive comment inside `zip` (host only). */
int b200z_zip_comment(const uint8_t *zip, size_t zip_len, uint64_t *off, uint32_t *len);
#define B200Z_ZIP_WEB_EOS 1u      /* flags: pure-Dart Inflate end-of-stream behaviour (SURVEY Q1) instead of dart:io's  */
#define B200Z_ZIP_NO_SPLIT 2u     /* flags: do not look for full-flush points inside members                        */
#define B200Z_ZIP_ENCRYPTED (-20)  /* status: encrypted member, not decoded                                      */
#define B200Z_ZIP_TOO_LARGE (-21)  /* status: member of 4 GiB or more                                            */
/* Member i is written to out[out_off[i] .. +out_room[i]); out_len[i] = bytes it produced (may exceed the room:
 * status B200Z_U_NOSPC), status[i] = B200Z_U_* / B200Z_ZIP_*.  All members are decoded in one call: deflate members
 * as units of one inflate batch, except that a member of 16 MiB compressed or more without full-flush points is decoded
 * across the whole GPU by many chunks at once (several such members together).  Which path decodes a member never
 * changes its bytes, out_len or status.                                                                           */
int b200z_zip_extract(const uint8_t *zip, size_t zip_len, const b200z_zip_entry *entries, size_t n, uint8_t *out,
                      size_t out_cap, const uint64_t *out_off, const uint64_t *out_room, uint64_t *out_len,
                      int32_t *status, uint32_t flags);
/* Encrypted members -- ZipDecoder().decodeBytes(bytes, password:) (zip_file.dart:98-134, 164-216, 260-359).
 * b200z_zip_crypt_info (host only): how member `e` is encrypted, as ZipFile.read decides it: flag bit 0 is ZipCrypto unless
 * the LOCAL extra field (longer than 2 bytes) holds an AES record (id 0x9901); `method` is the method the content is stored
 * with (the AES record's for AES members), `aes_strength` the record's strength byte (1: 128, 2: 192, else 256 bits).  The
 * reference's scan walks the extra field in 2-byte steps without skipping other records' payloads; when that walk reads
 * past the end (ZipFile.read throws): B200Z_E_THROW.
 * b200z_zip_extract_password: b200z_zip_extract with a password (`password_len` bytes: the low byte of each UTF-16 code
 * unit, as the reference's codeUnits; length 0 is the empty password).  password == NULL is exactly b200z_zip_extract.
 * Per member, beyond the B200Z_U_* statuses: B200Z_ZIP_BAD_PASSWORD (AES verifier mismatch), B200Z_ZIP_BAD_MAC (the
 * HMAC-SHA1 of the ciphertext does not match; the member was decoded, its bytes are withheld), B200Z_U_THROW (the member
 * is too short for its ZipCrypto header / AES salt + verifier + MAC, an empty password on an AES member, or the extra field
 * scan throws); out_len = 0 for all three.  ZipCrypto has no check: a wrong password decodes to garbage, as in the
 * reference.  The reference decrypts inside the caller's archive buffer; `zip` is const here and stays as it was.     */
#define B200Z_ZIP_CRYPT_NONE 0u
#define B200Z_ZIP_CRYPT_ZIPCRYPTO 1u
#define B200Z_ZIP_CRYPT_AES 2u
#define B200Z_ZIP_BAD_PASSWORD (-22) /* status: AES password verifier mismatch (Exception('password error'))       */
#define B200Z_ZIP_BAD_MAC (-23)      /* status: AES authentication code mismatch                                 */
int b200z_zip_crypt_info(const uint8_t *zip, size_t zip_len, const b200z_zip_entry *e, uint32_t *mode,
                         uint32_t *aes_strength, uint32_t *method);
int b200z_zip_extract_password(const uint8_t *zip, size_t zip_len, const b200z_zip_entry *entries, size_t n, uint8_t *out,
                               size_t out_cap, const uint64_t *out_off, const uint64_t *out_room, uint64_t *out_len,
                               int32_t *status, uint32_t flags, const uint8_t *password, size_t password_len);
/* b200z_zip_extract_to_device = b200z_zip_extract_password (password == NULL: b200z_zip_extract) with the member slots in
 * device memory, so that decoded members never make the round trip through the host.
 *   Memory: `zip`, `entries` and every array are host memory; d_out is device memory on the b200z_init device.
 *   Results: for every member, status[i], out_len[i] and the bytes d_out[out_off[i] .. + min(out_len[i], out_room[i])) are
 *     exactly what the host call gives for the same arguments; slot contents beyond that, and the whole slot of a
 *     B200Z_U_NOSPC member, are unspecified, as on the host.
 *     Nothing is written outside the slots; slots may come in any order, leave gaps and start at any byte alignment.
 *   crc32 (may be NULL): crc32[i] = getCrc32 of member i's delivered bytes, computed on the device over the slot after
 *     delivery (0 for members without data and for B200Z_U_NOSPC members) -- what ZipFile.verifyCrc32 compares.
 *   Argument errors: the host call's rules, and d_out must be device memory of the library's device
 *     (cudaPointerGetAttributes) whenever a member has room: B200Z_E_ARG.  No device: B200Z_E_NODEVICE.  On any error
 *     nothing is written, neither to d_out nor to out_len / status / crc32.
 *   Ordering: the library's stream waits on an event recorded on cuda_stream (a cudaStream_t; NULL = the library's own
 *     stream, cudaStreamLegacy for the legacy default stream) when the call starts, and the call returns once the bytes are
 *     in place, as the *_decode_batch_to_device calls do.
 * Members decode into the library's buffer as in the host call (sized by the slots' span, not their end), and reach their
 * slots with one k_copy_slots launch for all deflate / stored members plus the BZip2 batch's own deliveries; the CRCs take
 * one launch more.  The launch count does not grow with the member count.                                          */
int b200z_zip_extract_to_device(const uint8_t *zip, size_t zip_len, const b200z_zip_entry *entries, size_t n, uint8_t *d_out,
                                size_t out_cap, const uint64_t *out_off, const uint64_t *out_room, uint64_t *out_len,
                                int32_t *status, uint32_t *crc32, uint32_t flags, const uint8_t *password,
                                size_t password_len, void *cuda_stream);

/* ---- TAR member walk on the device -----------------------------------------------------------------------------------
 * b200z_tar_walk_device = the member walk of TarDecoder.decodeBytes(storeData: true) (tar_decoder.dart:28-38,
 * tar_file.dart:74-118) over n archives already in device memory, d_base[off[i] .. +len[i]).  Each header's size field says
 * where the next header is, so the walk runs on the device (k_tar_walk, one warp per archive) and only the members' records
 * and headers come back.  From pos = 0, while pos < len: one byte left, or two zero bytes at pos, end the walk
 * (OK); the header is the next min(512, len - pos) bytes; `size` is its field at 124..136 as _parseInt reads it (cut at the
 * first NUL, UTF-8 or else Latin-1, Dart's trim, then [+-]?[0-7]+ or 0); a negative size ends the walk with B200Z_E_THROW
 * (readBytes' RangeError); the content is the next min(size, what is left) bytes; unless the type byte (156) is '5', a size
 * that is not a multiple of 512 is padded up to one, clamped to the archive.  Names, links, LongLink and PAX entries do not
 * move the walk: they are the caller's, read from the headers.
 *   Memory: d_base is device memory on the b200z_init device; every other array is host memory.
 *   Results: archive i's members are members[first[i] .. +count[i]), in order, with offsets from the archive's first byte;
 *     headers[512 k .. +512) is member k's header (zero-filled past header_len); rc[i] is B200Z_OK or B200Z_E_THROW (count[i]
 *     is then the members before the negative size field); *n_total = the members of all archives.  first[] is the
 *     exclusive prefix sum of count[]: the layout is archive order, the same on every call.  An archive has at most floor(len[i] / 512) + 1 members, so cap >= sum(floor(len[i] / 512) + 1) always
 *     suffices.  cap < *n_total: B200Z_E_NOSPC, with *n_total set and nothing else written.
 *   Argument errors: null arrays (members / headers may be null when cap == 0), wrapping ranges, or an archive whose first or
 *     last byte is not device memory of the library's device (cudaPointerGetAttributes; archives in separate allocations may
 *     share d_base through pointer differences, so every archive's range is checked, not d_base alone): B200Z_E_ARG, and
 *     nothing is written.  n == 0 is OK.  No device: B200Z_E_NODEVICE, nothing is written.
 *   Ordering: the library's stream waits on an event recorded on cuda_stream (as in the *_decode_batch_to_device calls), and
 *     the call returns once the results are in place.
 * One call is two launches whatever n and the member count: k_tar_walk, then one k_copy_slots that gathers the records and
 * headers into one area, which comes back in one copy.                                                                   */
typedef struct {
  uint64_t header_off, content_off, content_len; /* from the archive's first byte; content_len is the clipped read */
  int64_t size;                                  /* the size field as _parseInt reads it                            */
  uint32_t header_len, pad_;                     /* 512, fewer when the archive ends inside the header              */
} b200z_tar_member;
int b200z_tar_walk_device(const uint8_t *d_base, const uint64_t *off, const uint64_t *len, size_t n, b200z_tar_member *members,
                          uint8_t *headers, size_t cap, uint64_t *first, uint64_t *count, int32_t *rc, size_t *n_total,
                          void *cuda_stream);
/* ZipEncoder(password:) member payloads (zip_encoder.dart:166-183): AES-256 in place on host buffers.  Member i is
 * data[off[i] .. +len[i]) (already compressed), salts[16 i ..] its salt; on return it is the ciphertext,
 * pwd_verify[2 i ..] its password verifier and mac[10 i ..] the first 10 bytes of the HMAC-SHA1 of the ciphertext.  An
 * empty password: B200Z_E_THROW (the reference's deriveKey returns an empty list and sublist throws).               */
int b200z_zip_aes_encrypt(uint8_t *data, const uint64_t *off, const uint64_t *len, size_t n, const uint8_t *salts,
                          const uint8_t *password, size_t password_len, uint8_t *pwd_verify, uint8_t *mac);

/* ---- file streams: InputFileStream -> codec -> OutputFileStream -------------------------------------------------
 * decodeStream / encodeStream with an InputFileStream and an OutputFileStream (input_file_stream.dart:11-221,
 * output_file_stream.dart:11-235; callers: extractFileToDisk, io/extract_archive_to_disk.dart:160-267, and the *_test.dart
 * stream tests).  The reference pulls the file through a FileBuffer cache (file_buffer.dart:10, 1 KiB by default) one
 * readByte() at a time; here the binding passes the PATHS and byte ranges and the library moves the data itself: page-locked
 * segment buffers kept for the life of the library, filled and drained by threads with large pread()/pwrite() calls, so
 * that reading segment k+1, decoding segment k and writing segment k-1 overlap.  GZip members with size hints are cut into
 * segments at member boundaries (B200Z_FILE_SEG_KB, default 256 MiB of compressed bytes); every other case is one segment.
 *
 * Reads in_path[in_off .. in_off+in_len) (clamped to the file, as readBytes does) and writes the result to out_path from
 * byte out_off on (the file is created if needed and NOT truncated: OutputFileStream has done that when it opened it).
 * *in_used = bytes consumed (the streams are read to their end), *out_len = bytes written.  Return codes as for the memory
 * entry points; on B200Z_E_DATA / B200Z_E_THROW the bytes produced before the error are in the file, as in the reference.
 *   op                        a0       a1           a2
 *   B200Z_FILE_GZIP_DECODE    verify   -            -        GZipDecoderWeb.decodeStream  (_gzip_decoder_web.dart:27-58)
 *   B200Z_FILE_ZLIB_DECODE    verify   raw          -        ZLibDecoderWeb.decodeStream  (_zlib_decoder_web.dart:31-107)
 *   B200Z_FILE_BZIP2_DECODE   verify   -            -        BZip2Decoder.decodeStream    (bzip2_decoder.dart:21-88)
 *   B200Z_FILE_ZLIB_ENCODE    level    window_bits  raw      ZLibEncoderWeb.encodeStream  (_zlib_encoder_web.dart:30-73)
 *   B200Z_FILE_GZIP_ENCODE    level    -            mtime    GZipEncoderWeb.encodeStream  (_gzip_encoder_web.dart:30-100)
 *   B200Z_FILE_BZIP2_ENCODE   -        -            -        BZip2Encoder.encodeStream    (bzip2_encoder.dart:25-81)
 *   B200Z_FILE_XZ_DECODE      verify   -            -        XZDecoder.decodeStream       (xz_decoder.dart:22-26)
 *   B200Z_FILE_XZ_ENCODE      check    -            -        XZEncoder.encodeStream       (xz_encoder.dart:30-62)       */
#define B200Z_FILE_GZIP_DECODE 1
#define B200Z_FILE_ZLIB_DECODE 2
#define B200Z_FILE_BZIP2_DECODE 3
#define B200Z_FILE_ZLIB_ENCODE 4
#define B200Z_FILE_GZIP_ENCODE 5
#define B200Z_FILE_BZIP2_ENCODE 6
#define B200Z_FILE_XZ_DECODE 7
#define B200Z_FILE_XZ_ENCODE 8
int b200z_file_codec(int op, const char *in_path, uint64_t in_off, uint64_t in_len, const char *out_path, uint64_t out_off,
                     int32_t a0, int32_t a1, uint32_t a2, uint64_t *in_used, uint64_t *out_len);
/* How the last b200z_file_codec call of this process went: segments decoded through the member-boundary pipeline, and
 * ranges handed to a memory entry point in one piece (tests, tuning of B200Z_FILE_SEG_KB).                          */
void b200z_file_last_stats(uint32_t *n_segments, uint32_t *n_whole);

/* ---- batched independent units (what the kernels run) --------------------------------- */
/* n_units raw DEFLATE streams: unit u reads in_base[in_off[u] .. +in_len[u]) and writes
 * out_base[out_off[u] .. +out_cap[u]).  Per unit: out_len, status (B200Z_U_*), in_used.
 * Host-pointer variant: copies in, runs, copies out (the end-to-end path).                  */
int b200z_inflate_batch(const uint8_t *in_base, size_t in_bytes, const uint64_t *in_off,
                        const uint32_t *in_len, uint8_t *out_base, size_t out_bytes,
                        const uint64_t *out_off, const uint32_t *out_cap, uint32_t *out_len,
                        int32_t *status, uint32_t *in_used, size_t n_units);
/* Device-pointer variant: every pointer is device memory on the b200z_init device; work is
 * enqueued on `cuda_stream` (a cudaStream_t, NULL = the library's stream) and NOT synchronised:
 * read the results after that stream has been synchronised.
 * Input: d_in_base is 16-byte aligned, and the kernels read whole aligned 16-byte blocks, so
 * the buffer must be readable through round_up(max(in_off[u] + in_len[u]), 16) bytes from
 * d_in_base (what lies past a unit's in_len is read but never decoded).
 * Output: unit u writes d_out_base[out_off[u] .. +out_cap[u]); slots may come in any order and
 * leave gaps, which are not written.
 * Workspace: `workspace` must hold b200z_inflate_workspace_bytes(n_units, total_in_bytes,
 * total_out_cap) bytes, where total_out_cap is the layout's EXTENT, max(out_off[u] + out_cap[u])
 * (not the sum of the caps: the workspace is indexed by out_off).  total_in_bytes is not used.
 * The workspace needs no initialisation, may be reused by the next call on the same stream,
 * and must not be shared by batches in flight at the same time.  A workspace smaller than
 * b200z_inflate_workspace_bytes(n_units, 0, 0) gives B200Z_E_ARG with nothing enqueued.     */
size_t b200z_inflate_workspace_bytes(size_t n_units, size_t total_in_bytes, size_t total_out_cap);
int b200z_inflate_batch_device(const uint8_t *d_in_base, const uint64_t *d_in_off,
                               const uint32_t *d_in_len, uint8_t *d_out_base,
                               const uint64_t *d_out_off, const uint32_t *d_out_cap,
                               uint32_t *d_out_len, int32_t *d_status, uint32_t *d_in_used,
                               size_t n_units, void *d_workspace, size_t workspace_bytes,
                               void *cuda_stream);

/* ---- several GPUs of one box driven by ONE process (SURVEY.md 8b: device_mask / n_gpus; 8e) ----------------
 * The reference decodes the members of a gzip stream in one loop and returns one buffer
 * (_gzip_decoder_web.dart:27-38).  Here the members -- or the units of a batch -- are cut into one contiguous range
 * per GPU (balanced by compressed bytes); every GPU receives its range over its own link, decodes it, and its part of
 * the output stream goes straight to its place in the caller's buffer.  B200Z_MULTI_GATHER: the shards are also
 * exchanged over NVLink (NCCL, communicators owned by the library, looked up at run time) so that EVERY device then
 * holds the whole stream in block order (b200z_multi_device_output) -- BASELINE north_star's all-gather.
 * b200z_multi_init(mask): bit d = CUDA device d; also runs b200z_init on the first device of the mask, which serves
 * whatever cannot be dealt (members without size hints, hints that lie, the zlib fall-back).                       */
#define B200Z_MULTI_GATHER 1u
int b200z_multi_init(uint32_t device_mask, uint32_t flags);
void b200z_multi_shutdown(void);
int b200z_multi_device_count(void);
int b200z_gzip_decode_multi(const uint8_t *in, size_t in_len, int verify, uint8_t *out, size_t out_cap,
                            size_t *out_len, uint32_t flags);
int b200z_inflate_batch_multi(const uint8_t *in_base, size_t in_bytes, const uint64_t *in_off,
                              const uint32_t *in_len, uint8_t *out_base, size_t out_bytes,
                              const uint64_t *out_off, const uint32_t *out_cap, uint32_t *out_len,
                              int32_t *status, uint32_t *in_used, size_t n_units, uint32_t flags);
/* after a B200Z_MULTI_GATHER call: device `slot` (0 .. b200z_multi_device_count()-1) holds *bytes of output at the
 * returned device pointer; NULL when the last call did not gather.                                             */
const void *b200z_multi_device_output(int slot, size_t *bytes);

/* Number of kernel launches issued by this library since b200z_init (bench.py gpu_launches). */
uint64_t b200z_launch_count(void);
/* Optional per-kernel timing with CUDA events on the launching stream: enable, run batches, then read
 * the summed durations (ms) of the three inflate kernels (k_inflate_fast, then the exact pair k_inflate_decode /
 * k_inflate_expand over the units the first one left) and the number of batches timed.                        */
void b200z_profile_enable(int on);
int b200z_profile_read(double *fast_ms, double *decode_ms, double *expand_ms, uint64_t *n_batches);

#ifdef __cplusplus
}
#endif
#endif /* B200Z_H */
