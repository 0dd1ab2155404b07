/*
 * oracle/orc_xz.h -- CPU ORACLE (test infrastructure only; see orc.h): the XZ codec.
 *   xz.c   _XZStreamDecoder, LzmaDecoder, RangeDecoder (codecs/xz_decoder.dart, codecs/lzma/), XZEncoder
 *          (codecs/xz_encoder.dart), CRC-64 (util/_crc64_io.dart) and SHA-256 (PcSHA256Digest, util/encryption.dart)
 */
#ifndef ORC_XZ_H
#define ORC_XZ_H
#include "orc.h"

/* XZDecoder().decodeBytes(data, verify:) -- ORC_OK / ORC_FALSE / ORC_THROW, and in *out the bytes the reference's
 * OutputMemoryStream holds at that point (free with orc_free) */
int orc_xz_decode(const uint8_t *in, size_t n, int verify, uint8_t **out, size_t *out_len);
/* XZEncoder().encodeBytes(data, check:) with check 0 none, 1 crc32, 2 crc64, 3 sha256 (XZCheck.index) */
int orc_xz_encode(const uint8_t *in, size_t n, int check, uint8_t **out, size_t *out_len);
uint64_t orc_crc64(const uint8_t *p, size_t n, uint64_t crc); /* getCrc64(array, crc) */
void orc_sha256(const uint8_t *p, size_t n, uint8_t digest[32]);

#endif
