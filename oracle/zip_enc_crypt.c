/*
 * oracle/zip_enc_crypt.c -- CPU ORACLE (test infrastructure only; see orc.h).
 *
 * ZipEncoder(password:) of lib/src/codecs/zip_encoder.dart: the container of zip_enc.c with the AES parts of add /
 * _writeFile / _writeCentralDirectory (:270-310, 347-437) and _encryptCompressedData :166-183 (aes.c), quirks included --
 * every entry (directories too) gets method 99, flag bit 0 and the AE-1 record; the verifier and MAC of the last encrypted
 * member live on in the encoder, so a directory after a file has compressedSize 12 and that file's MAC (10 bytes) behind
 * its local header.  The salts are passed in (the reference draws them from Random.secure).
 * PARITY UNPINNED by the reference's own tests (round trip only, test/zip_test.dart:625-648).
 */
#include <stdlib.h>
#include <string.h>

#include "orc_crypt.h"

static void w16(orc_oms *o, uint32_t v) {
  orc_oms_write_byte(o, v & 0xff);
  orc_oms_write_byte(o, (v >> 8) & 0xff);
}
static void w32(orc_oms *o, uint32_t v) {
  w16(o, v & 0xffff);
  w16(o, v >> 16);
}
static void w64(orc_oms *o, uint64_t v) {
  w32(o, (uint32_t)v);
  w32(o, (uint32_t)(v >> 32));
}

typedef struct {
  uint64_t csize, usize, pos;
  uint32_t crc, method_id;
} fdata;

/* _getAexExtraData :347-363 */
static void aes_extra(orc_oms *o, uint32_t method_id) {
  w16(o, 0x9901);
  w16(o, 7);
  w16(o, 1);
  orc_oms_write_byte(o, 'A');
  orc_oms_write_byte(o, 'E');
  orc_oms_write_byte(o, 3);
  w16(o, method_id);
}

int orc_zip_encode_password(const orc_zip_member_in *m, size_t n, int level, const char *comment, const uint8_t *pw,
                            size_t pwlen, const uint8_t *salts, uint8_t **out, size_t *out_len) {
  if (!pw) return orc_zip_encode(m, n, level, comment, out, out_len);
  orc_oms o;
  if (pwlen == 0) { /* ZipFile.deriveKey returns an empty list: sublist throws */
    *out = NULL;
    *out_len = 0;
    return ORC_THROW;
  }
  uint8_t mac[10], ver[2];
  int have_mac = 0;
  orc_oms_init(&o, 0x8000);
  fdata *fd = (fdata *)calloc(n ? n : 1, sizeof(fdata));
  int rc = ORC_OK;
  for (size_t i = 0; i < n && rc == ORC_OK; ++i) {
    uint8_t *payload = NULL;
    size_t plen = 0;
    uint32_t crc = 0;
    if (m[i].is_file) {
      crc = orc_crc32(m[i].content, m[i].content_len, 0);
      if (m[i].method == 1) {
        uint32_t c2;
        rc = orc_deflate_bytes(m[i].content, m[i].content_len, level, 15, &payload, &plen, &c2);
      } else if (m[i].method == 2) {
        rc = orc_bzip2_encode_bytes(m[i].content, m[i].content_len, &payload, &plen);
      } else {
        payload = (uint8_t *)malloc(m[i].content_len ? m[i].content_len : 1);
        memcpy(payload, m[i].content, m[i].content_len);
        plen = m[i].content_len;
      }
      if (rc != ORC_OK) break;
    }
    if (m[i].is_file) {
      orc_zip_aes_encrypt(payload, plen, salts + 16 * i, pw, pwlen, ver, mac);
      have_mac = 1;
    }
    fd[i].crc = crc;
    fd[i].csize = plen + (m[i].is_file ? 16 : 0) + (have_mac ? 12 : 0);
    fd[i].usize = m[i].is_file ? m[i].content_len : 0;
    fd[i].pos = (uint64_t)o.len;
    fd[i].method_id = m[i].method == 1 ? 8 : m[i].method == 2 ? 12 : 0;
    /* _writeFile */
    const int z64 = fd[i].csize > 0xFFFFFFFFull || fd[i].usize > 0xFFFFFFFFull;
    const size_t nl = strlen(m[i].name);
    w32(&o, 0x04034b50u);
    w16(&o, 20);
    w16(&o, 2048 | 1); /* languageEncodingBitUtf8 | fileEncryptionBit (:375-382) */
    w16(&o, 99);
    w16(&o, m[i].dos_time);
    w16(&o, m[i].dos_date);
    w32(&o, crc);
    w32(&o, z64 ? 0xFFFFFFFFu : (uint32_t)fd[i].csize);
    w32(&o, z64 ? 0xFFFFFFFFu : (uint32_t)fd[i].usize);
    w16(&o, (uint32_t)nl);
    w16(&o, (z64 ? 20 : 0) + 11);
    orc_oms_write_bytes(&o, (const uint8_t *)m[i].name, (int64_t)nl);
    if (z64) {
      orc_oms_write_byte(&o, 1); orc_oms_write_byte(&o, 0); orc_oms_write_byte(&o, 0x10); orc_oms_write_byte(&o, 0);
      w64(&o, fd[i].usize);
      w64(&o, fd[i].csize);
    }
    aes_extra(&o, fd[i].method_id);
    if (m[i].is_file) {
      orc_oms_write_bytes(&o, salts + 16 * i, 16);
      orc_oms_write_bytes(&o, ver, 2);
    }
    if (payload) orc_oms_write_bytes(&o, payload, (int64_t)plen);
    if (have_mac) orc_oms_write_bytes(&o, mac, 10);
    free(payload);
  }
  if (rc != ORC_OK) {
    free(fd);
    *out = o.buf;
    *out_len = (size_t)o.len;
    return rc;
  }
  /* _writeCentralDirectory */
  const uint64_t cd_pos = (uint64_t)o.len;
  int any64 = 0;
  for (size_t i = 0; i < n; ++i) {
    const int z64 = fd[i].csize > 0xFFFFFFFFull || fd[i].usize > 0xFFFFFFFFull || fd[i].pos > 0xFFFFFFFFull;
    any64 |= z64;
    const size_t nl = strlen(m[i].name), cl = m[i].comment ? strlen(m[i].comment) : 0;
    w32(&o, 0x02014b50u);
    w16(&o, (0 << 8) | 20);
    w16(&o, 20);
    w16(&o, 2048 | 1);
    w16(&o, 99);
    w16(&o, m[i].dos_time);
    w16(&o, m[i].dos_date);
    w32(&o, fd[i].crc);
    w32(&o, z64 ? 0xFFFFFFFFu : (uint32_t)fd[i].csize);
    w32(&o, z64 ? 0xFFFFFFFFu : (uint32_t)fd[i].usize);
    w16(&o, (uint32_t)nl);
    w16(&o, (z64 ? 28 : 0) + 11);
    w16(&o, (uint32_t)cl);
    w16(&o, 0);
    w16(&o, 0);
    w32(&o, (uint32_t)((uint64_t)m[i].mode << 16));
    w32(&o, z64 ? 0xFFFFFFFFu : (uint32_t)fd[i].pos);
    orc_oms_write_bytes(&o, (const uint8_t *)m[i].name, (int64_t)nl);
    if (z64) {
      orc_oms_write_byte(&o, 1); orc_oms_write_byte(&o, 0); orc_oms_write_byte(&o, 0x18); orc_oms_write_byte(&o, 0);
      w64(&o, fd[i].usize);
      w64(&o, fd[i].csize);
      w64(&o, fd[i].pos);
    }
    aes_extra(&o, fd[i].method_id);
    if (cl) orc_oms_write_bytes(&o, (const uint8_t *)m[i].comment, (int64_t)cl);
  }
  const uint64_t cd_size = (uint64_t)o.len - cd_pos;
  const int need64 = any64 || n > 0xffff || cd_size > 0xffffffffull || cd_pos > 0xffffffffull;
  if (need64) {
    const uint64_t eocd_off = (uint64_t)o.len;
    w32(&o, 0x06064b50u);
    w64(&o, 0x2c);
    w16(&o, 0x2d);
    w16(&o, 0x2d);
    w32(&o, 0);
    w32(&o, 0);
    w64(&o, n);
    w64(&o, n);
    w64(&o, cd_size);
    w64(&o, cd_pos);
    w32(&o, 0x07064b50u);
    w32(&o, 0);
    w64(&o, eocd_off);
    w32(&o, 1);
  }
  const size_t zl = comment ? strlen(comment) : 0;
  w32(&o, 0x06054b50u);
  w16(&o, 0);
  w16(&o, need64 ? 0xffff : 0);
  w16(&o, need64 ? 0xffff : (uint32_t)n);
  w16(&o, need64 ? 0xffff : (uint32_t)n);
  w32(&o, need64 ? 0xffffffffu : (uint32_t)cd_size);
  w32(&o, need64 ? 0xffffffffu : (uint32_t)cd_pos);
  w16(&o, (uint32_t)zl);
  if (zl) orc_oms_write_bytes(&o, (const uint8_t *)comment, (int64_t)zl);
  free(fd);
  *out = o.buf;
  *out_len = (size_t)o.len;
  return ORC_OK;
}
