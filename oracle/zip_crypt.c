/*
 * oracle/zip_crypt.c -- CPU ORACLE (test infrastructure only; see orc.h).
 *
 * Restates the encrypted branches of the reference's ZIP reader (the ciphers are in aes.c):
 *   lib/src/codecs/zip/zip_file.dart:98-130   ZipFile.read: ZipCrypto vs AES (the local extra field scan)
 *   lib/src/codecs/zip/zip_file.dart:164-216  getStream / decompress: decrypt first, then as an unencrypted member
 *   lib/src/codecs/zip/zip_file.dart:260-359  _decodeZipCrypto, _decodeAes, deriveKey
 * written as the Dart reads it: a cursor over the bytes whose reads throw past the end (input_memory_stream.dart:121-124).
 * Pinned by the reference's encrypted fixtures (tests/golden/zip_crypt/) and CPython's zipfile.
 */
#include <stdlib.h>
#include <string.h>

#include "orc_crypt.h"

typedef struct {
  const uint8_t *b;
  int64_t len, pos;
  int threw;
} cur;

static uint32_t rd(cur *c, int n) { /* little-endian readByte / readUint16 */
  uint32_t v = 0;
  for (int i = 0; i < n; i++) {
    if (c->pos >= c->len || c->pos < 0) {
      c->threw = 1;
      return 0;
    }
    v |= (uint32_t)c->b[c->pos++] << (8 * i);
  }
  return v;
}

/* ZipFile.read :98-130.  Flag bit 0 is ZipCrypto unless the LOCAL extra field (longer than 2 bytes) holds id 0x9901.  The
 * scan reads 16-bit ids at 2-byte steps and does not skip the payload of other ids, as the reference does. */
int orc_zip_crypt_info(const uint8_t *b, size_t blen, const orc_zip_entry *e, uint32_t *mode, uint32_t *strength,
                       uint32_t *method) {
  *mode = ORC_ZIP_NONE;
  *strength = 0;
  *method = e->method;
  if (!e->has_data || !(e->flags & 1)) return ORC_OK;
  *mode = ORC_ZIP_ZIPCRYPTO;
  const int64_t x0 = (int64_t)(e->name_off + e->name_len), xl = (int64_t)e->data_off - x0;
  if (xl <= 2) return ORC_OK;
  cur x = {b, x0 + xl, x0, 0};
  while (x.pos < x.len) {
    const uint32_t id = rd(&x, 2);
    if (x.threw) return ORC_THROW;
    if (id != 0x9901) continue;
    rd(&x, 2); /* dataSize */
    rd(&x, 2); /* vendorVersion */
    x.pos = x.pos + 2 < x.len ? x.pos + 2 : x.len; /* readString(size: 2): readBytes hands out what is there */
    const uint32_t st = rd(&x, 1), cm = rd(&x, 2);
    if (x.threw) return ORC_THROW;
    *mode = ORC_ZIP_AES;
    *strength = st;
    *method = cm;
  }
  return ORC_OK;
}

/* decompress the plaintext of a decrypted member: the reference decodes exactly these bytes.  web_eos == 0 (dart:io's
 * zlib, all symbols): Inflate may look at 8 zero bytes behind them, which only satisfies its look-ahead. */
static int decode_plain(const uint8_t *p, size_t n, uint32_t method, int web_eos, uint8_t **out, size_t *out_len) {
  if (method == 8) {
    const size_t pad = web_eos ? 0 : 8;
    uint8_t *buf = (uint8_t *)calloc(n + pad + 1, 1);
    memcpy(buf, p, n);
    size_t consumed;
    const int st = orc_inflate_bytes(buf, n + pad, out, out_len, &consumed);
    free(buf);
    return st;
  }
  if (method == 12) return orc_bzip2_decode_bytes(p, n, 0, out, out_len);
  *out = (uint8_t *)malloc(n ? n : 1);
  memcpy(*out, p, n);
  *out_len = n;
  return ORC_OK;
}

/* getStream (:201-248) with _decodeZipCrypto (:288-303) / _decodeAes (:305-343).  Statuses: ORC_THROW for the reads that
 * throw (ZipCrypto member shorter than its 12-byte header; AES member shorter than salt + verifier + MAC) and for the
 * empty password (deriveKey returns an empty list, sublist throws); ORC_BAD_PASSWORD; ORC_BAD_MAC. */
int orc_zip_member_password(const uint8_t *b, size_t blen, const orc_zip_entry *e, int web_eos, const uint8_t *pw,
                            size_t pwlen, uint8_t **out, size_t *out_len) {
  *out = NULL;
  *out_len = 0;
  if (!pw || !e->has_data || !(e->flags & 1)) return orc_zip_member(b, blen, e, web_eos, out, out_len);
  uint32_t mode, strength, method;
  if (orc_zip_crypt_info(b, blen, e, &mode, &strength, &method) != ORC_OK) return ORC_THROW;
  if (e->comp_size == 0) { /* :170-171: an empty member is not decrypted */
    orc_zip_entry plain = *e;
    plain.flags &= ~1u;
    plain.method = method;
    return orc_zip_member(b, blen, &plain, web_eos, out, out_len);
  }
  const uint8_t *d = b + e->data_off;
  const size_t n = (size_t)e->comp_size;
  if (mode == ORC_ZIP_ZIPCRYPTO) {
    if (n < 12) return ORC_THROW; /* readByte past the end */
    uint8_t *pt = (uint8_t *)malloc(n);
    orc_zipcrypto_decrypt(pw, pwlen, d, n, pt);
    const int st = decode_plain(pt + 12, n - 12, method, web_eos, out, out_len);
    free(pt);
    return st;
  }
  const size_t sl = strength == 1 ? 8 : strength == 2 ? 12 : 16, ks = sl * 2;
  if (n < sl + 12) return ORC_THROW; /* readBytes(input.length - 10) with a negative count */
  if (pwlen == 0) return ORC_THROW;
  uint8_t dk[66], mac[20];
  orc_pbkdf2_sha1(pw, pwlen, d, sl, 1000, dk, 2 * ks + 2);
  if (memcmp(dk + 2 * ks, d + sl, 2) != 0) return ORC_BAD_PASSWORD;
  const uint8_t *ct = d + sl + 2;
  const size_t cl = n - sl - 12;
  orc_hmac_sha1(dk + ks, ks, ct, cl, mac);
  if (memcmp(mac, ct + cl, 10) != 0) return ORC_BAD_MAC;
  uint8_t *pt = (uint8_t *)malloc(cl ? cl : 1);
  memcpy(pt, ct, cl);
  orc_winzip_ctr(dk, (int)ks, pt, cl);
  const int st = decode_plain(pt, cl, method, web_eos, out, out_len);
  free(pt);
  return st;
}
