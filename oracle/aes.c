/*
 * oracle/aes.c -- CPU ORACLE (test infrastructure only; see orc.h).
 *
 * Restates what the reference's ZIP encryption uses:
 *   lib/src/util/encryption.dart  PcAESEngine (forward cipher, 128/192/256-bit keys), PcSHA1Digest, PcHMac,
 *                                 PcPBKDF2KeyDerivator (:60-132)
 *   lib/src/util/aes.dart:17-81   the WinZip CTR mode: counter block = little-endian block number (from 1) in bytes
 *                                 0-3, zeros in 4-15; the HMAC-SHA1 over the ciphertext, cut to 10 bytes
 *   lib/src/codecs/zip/zip_file.dart:260-303  ZipCrypto (the three keys, one CRC-32 step per byte)
 * The AES tables are derived from GF(2^8) arithmetic at first use rather than written out.
 * Pinned by FIPS-197 Appendix C, RFC 2202, RFC 6070 and the reference's encrypted fixtures (tests/golden/zip_crypt/).
 */
#include <pthread.h>
#include <stdlib.h>
#include <string.h>

#include "orc_crypt.h"

/* ---- AES forward cipher ------------------------------------------------------------------------------------------ */
static uint8_t S[256];
static uint32_t Te[4][256];
static pthread_once_t aes_once = PTHREAD_ONCE_INIT;

static uint8_t xt(uint8_t a) { return (uint8_t)((a << 1) ^ ((a & 0x80) ? 0x1b : 0)); }
static uint8_t gmul(uint8_t a, uint8_t b) {
  uint8_t r = 0;
  while (b) {
    if (b & 1) r ^= a;
    a = xt(a);
    b >>= 1;
  }
  return r;
}
static uint32_t ror32(uint32_t v, int s) { return (v >> s) | (v << (32 - s)); }

static void aes_tables(void) {
  for (int x = 0; x < 256; ++x) {
    uint8_t inv = 0;
    if (x) { /* x^254 = x^-1 in GF(2^8) */
      uint8_t p = (uint8_t)x, r = 1;
      for (int e = 254; e; e >>= 1) {
        if (e & 1) r = gmul(r, p);
        p = gmul(p, p);
      }
      inv = r;
    }
    uint8_t s = inv;
    for (int k = 1; k <= 4; ++k) s ^= (uint8_t)((inv << k) | (inv >> (8 - k)));
    S[x] = s ^ 0x63;
  }
  for (int x = 0; x < 256; ++x) {
    const uint8_t s = S[x];
    const uint32_t t = ((uint32_t)xt(s) << 24) | ((uint32_t)s << 16) | ((uint32_t)s << 8) | (uint32_t)(xt(s) ^ s);
    Te[0][x] = t;
    Te[1][x] = ror32(t, 8);
    Te[2][x] = ror32(t, 16);
    Te[3][x] = ror32(t, 24);
  }
}

static uint32_t be32(const uint8_t *p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
static void put_be32(uint8_t *p, uint32_t v) {
  p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v;
}
static uint32_t sub_word(uint32_t w) {
  return ((uint32_t)S[w >> 24] << 24) | ((uint32_t)S[(w >> 16) & 255] << 16) | ((uint32_t)S[(w >> 8) & 255] << 8) | S[w & 255];
}

int orc_aes_expand(const uint8_t *key, int key_len, uint32_t *rk) {
  pthread_once(&aes_once, aes_tables);
  const int nk = key_len / 4, nr = nk + 6;
  uint8_t rcon = 1;
  for (int i = 0; i < nk; ++i) rk[i] = be32(key + 4 * i);
  for (int i = nk; i < 4 * (nr + 1); ++i) {
    uint32_t t = rk[i - 1];
    if (i % nk == 0) {
      t = sub_word((t << 8) | (t >> 24)) ^ ((uint32_t)rcon << 24);
      rcon = xt(rcon);
    } else if (nk > 6 && i % nk == 4) {
      t = sub_word(t);
    }
    rk[i] = rk[i - nk] ^ t;
  }
  return nr;
}

void orc_aes_encrypt_block(const uint32_t *rk, int nr, const uint8_t in[16], uint8_t out[16]) {
  uint32_t s0 = be32(in) ^ rk[0], s1 = be32(in + 4) ^ rk[1], s2 = be32(in + 8) ^ rk[2], s3 = be32(in + 12) ^ rk[3];
  for (int r = 1; r < nr; ++r) {
    const uint32_t *k = rk + 4 * r;
    const uint32_t t0 = Te[0][s0 >> 24] ^ Te[1][(s1 >> 16) & 255] ^ Te[2][(s2 >> 8) & 255] ^ Te[3][s3 & 255] ^ k[0];
    const uint32_t t1 = Te[0][s1 >> 24] ^ Te[1][(s2 >> 16) & 255] ^ Te[2][(s3 >> 8) & 255] ^ Te[3][s0 & 255] ^ k[1];
    const uint32_t t2 = Te[0][s2 >> 24] ^ Te[1][(s3 >> 16) & 255] ^ Te[2][(s0 >> 8) & 255] ^ Te[3][s1 & 255] ^ k[2];
    const uint32_t t3 = Te[0][s3 >> 24] ^ Te[1][(s0 >> 16) & 255] ^ Te[2][(s1 >> 8) & 255] ^ Te[3][s2 & 255] ^ k[3];
    s0 = t0; s1 = t1; s2 = t2; s3 = t3;
  }
  const uint32_t *k = rk + 4 * nr;
#define FIN(a, b, c, d) \
  (((uint32_t)S[a >> 24] << 24) | ((uint32_t)S[(b >> 16) & 255] << 16) | ((uint32_t)S[(c >> 8) & 255] << 8) | S[d & 255])
  put_be32(out, FIN(s0, s1, s2, s3) ^ k[0]);
  put_be32(out + 4, FIN(s1, s2, s3, s0) ^ k[1]);
  put_be32(out + 8, FIN(s2, s3, s0, s1) ^ k[2]);
  put_be32(out + 12, FIN(s3, s0, s1, s2) ^ k[3]);
#undef FIN
}

/* Aes.processData (aes.dart:48-73), the cipher half: data ^= E(counter) block by block, counter from 1 */
void orc_winzip_ctr(const uint8_t *key, int key_len, uint8_t *data, size_t n) {
  uint32_t rk[60];
  const int nr = orc_aes_expand(key, key_len, rk);
  uint8_t iv[16], ks[16];
  uint32_t nonce = 1;
  for (size_t j = 0; j < n; j += 16, ++nonce) {
    memset(iv, 0, 16);
    iv[0] = (uint8_t)nonce; iv[1] = (uint8_t)(nonce >> 8); iv[2] = (uint8_t)(nonce >> 16); iv[3] = (uint8_t)(nonce >> 24);
    orc_aes_encrypt_block(rk, nr, iv, ks);
    const size_t m = n - j < 16 ? n - j : 16;
    for (size_t k = 0; k < m; ++k) data[j + k] ^= ks[k];
  }
}

/* ---- SHA-1, HMAC-SHA1, PBKDF2 ------------------------------------------------------------------------------------ */
typedef struct {
  uint32_t h[5];
  uint64_t len;
  uint8_t buf[64];
  size_t fill;
} sha1_ctx;

static uint32_t rol(uint32_t v, int s) { return (v << s) | (v >> (32 - s)); }
static void sha1_block(uint32_t h[5], const uint8_t *p) {
  uint32_t w[80];
  for (int i = 0; i < 16; ++i) w[i] = be32(p + 4 * i);
  for (int i = 16; i < 80; ++i) w[i] = rol(w[i - 3] ^ w[i - 8] ^ w[i - 14] ^ w[i - 16], 1);
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4];
  for (int i = 0; i < 80; ++i) {
    uint32_t f, k;
    if (i < 20) { f = (b & c) | (~b & d); k = 0x5A827999u; }
    else if (i < 40) { f = b ^ c ^ d; k = 0x6ED9EBA1u; }
    else if (i < 60) { f = (b & c) | (b & d) | (c & d); k = 0x8F1BBCDCu; }
    else { f = b ^ c ^ d; k = 0xCA62C1D6u; }
    const uint32_t t = rol(a, 5) + f + e + k + w[i];
    e = d; d = c; c = rol(b, 30); b = a; a = t;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e;
}
static void sha1_init(sha1_ctx *c) {
  static const uint32_t iv[5] = {0x67452301u, 0xEFCDAB89u, 0x98BADCFEu, 0x10325476u, 0xC3D2E1F0u};
  memcpy(c->h, iv, sizeof iv);
  c->len = 0;
  c->fill = 0;
}
static void sha1_update(sha1_ctx *c, const uint8_t *p, size_t n) {
  c->len += n;
  if (c->fill) {
    while (n && c->fill < 64) { c->buf[c->fill++] = *p++; n--; }
    if (c->fill < 64) return;
    sha1_block(c->h, c->buf);
    c->fill = 0;
  }
  for (; n >= 64; n -= 64, p += 64) sha1_block(c->h, p);
  memcpy(c->buf, p, n);
  c->fill = n;
}
static void sha1_final(sha1_ctx *c, uint8_t out[20]) {
  const uint64_t bits = c->len * 8;
  uint8_t pad = 0x80;
  sha1_update(c, &pad, 1);
  pad = 0;
  while (c->fill != 56) sha1_update(c, &pad, 1);
  uint8_t l[8];
  for (int i = 0; i < 8; ++i) l[i] = (uint8_t)(bits >> (56 - 8 * i));
  sha1_update(c, l, 8);
  for (int i = 0; i < 5; ++i) put_be32(out + 4 * i, c->h[i]);
}

void orc_sha1(const uint8_t *p, size_t n, uint8_t out[20]) {
  sha1_ctx c;
  sha1_init(&c);
  sha1_update(&c, p, n);
  sha1_final(&c, out);
}

/* PcHMac with PcSHA1Digest, block 64: a key longer than the block is hashed first */
typedef struct {
  sha1_ctx in, out;
} hmac_ctx;
static void hmac_init(hmac_ctx *m, const uint8_t *key, size_t klen) {
  uint8_t k[64] = {0}, pad[64];
  if (klen > 64) orc_sha1(key, klen, k);
  else memcpy(k, key, klen);
  for (int i = 0; i < 64; ++i) pad[i] = k[i] ^ 0x36;
  sha1_init(&m->in);
  sha1_update(&m->in, pad, 64);
  for (int i = 0; i < 64; ++i) pad[i] = k[i] ^ 0x5c;
  sha1_init(&m->out);
  sha1_update(&m->out, pad, 64);
}
static void hmac_final(const hmac_ctx *base, hmac_ctx *m, uint8_t out[20]) {
  uint8_t ih[20];
  sha1_final(&m->in, ih);
  m->out = base->out;
  sha1_update(&m->out, ih, 20);
  sha1_final(&m->out, out);
}

void orc_hmac_sha1(const uint8_t *key, size_t klen, const uint8_t *msg, size_t n, uint8_t out[20]) {
  hmac_ctx base, m;
  hmac_init(&base, key, klen);
  m = base;
  sha1_update(&m.in, msg, n);
  hmac_final(&base, &m, out);
}

/* PcPBKDF2KeyDerivator.deriveKey / _f (encryption.dart:83-131) */
void orc_pbkdf2_sha1(const uint8_t *pw, size_t pwlen, const uint8_t *salt, size_t slen, int iters, uint8_t *out, size_t dklen) {
  hmac_ctx base, m;
  hmac_init(&base, pw, pwlen);
  for (uint32_t blk = 1; (size_t)(blk - 1) * 20 < dklen; ++blk) {
    uint8_t ib[4] = {(uint8_t)(blk >> 24), (uint8_t)(blk >> 16), (uint8_t)(blk >> 8), (uint8_t)blk}, u[20], t[20];
    m = base;
    sha1_update(&m.in, salt, slen);
    sha1_update(&m.in, ib, 4);
    hmac_final(&base, &m, u);
    memcpy(t, u, 20);
    for (int c = 1; c < iters; ++c) {
      m = base;
      sha1_update(&m.in, u, 20);
      hmac_final(&base, &m, u);
      for (int j = 0; j < 20; ++j) t[j] ^= u[j];
    }
    const size_t at = (size_t)(blk - 1) * 20, k = dklen - at < 20 ? dklen - at : 20;
    memcpy(out + at, t, k);
  }
}

/* ---- ZipCrypto (zip_file.dart:260-303) --------------------------------------------------------------------------- */
typedef struct {
  uint32_t k0, k1, k2;
} zc_keys;
static uint32_t crc_tab[256];
static pthread_once_t crc_once = PTHREAD_ONCE_INIT;
static void crc_init(void) {
  for (uint32_t i = 0; i < 256; ++i) {
    uint32_t c = i;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
    crc_tab[i] = c;
  }
}
/* getCrc32Byte (crc32.dart:2) */
static uint32_t crc_byte(uint32_t crc, uint32_t b) { return crc_tab[(crc ^ b) & 0xff] ^ (crc >> 8); }
static void zc_update(zc_keys *k, uint32_t c) {
  k->k0 = crc_byte(k->k0, c);
  k->k1 = (k->k1 + (k->k0 & 0xff)) * 134775813u + 1u;
  k->k2 = crc_byte(k->k2, k->k1 >> 24);
}
static uint8_t zc_byte(const zc_keys *k) {
  const uint32_t t = (k->k2 & 0xffff) | 2;
  return (uint8_t)((t * (t ^ 1)) >> 8);
}
static void zc_init(zc_keys *k, const uint8_t *pw, size_t pwlen) {
  pthread_once(&crc_once, crc_init);
  k->k0 = 305419896u; k->k1 = 591751049u; k->k2 = 878082192u;
  for (size_t i = 0; i < pwlen; ++i) zc_update(k, pw[i]);
}

/* in[0..n) -> out[0..n): all n bytes, the 12 header bytes included (the caller drops them) */
void orc_zipcrypto_decrypt(const uint8_t *pw, size_t pwlen, const uint8_t *in, size_t n, uint8_t *out) {
  zc_keys k;
  zc_init(&k, pw, pwlen);
  for (size_t i = 0; i < n; ++i) {
    const uint8_t p = in[i] ^ zc_byte(&k);
    zc_update(&k, p);
    out[i] = p;
  }
}
/* the inverse, for tests that build ZipCrypto archives (the reference writes none) */
void orc_zipcrypto_encrypt(const uint8_t *pw, size_t pwlen, const uint8_t *in, size_t n, uint8_t *out) {
  zc_keys k;
  zc_init(&k, pw, pwlen);
  for (size_t i = 0; i < n; ++i) {
    const uint8_t c = in[i] ^ zc_byte(&k);
    zc_update(&k, in[i]);
    out[i] = c;
  }
}

/* ZipEncoder._encryptCompressedData (zip_encoder.dart:166-183): AES-256, the MAC taken after the cipher pass */
void orc_zip_aes_encrypt(uint8_t *data, size_t n, const uint8_t salt[16], const uint8_t *pw, size_t pwlen, uint8_t ver[2],
                         uint8_t mac[10]) {
  uint8_t dk[66], h[20];
  orc_pbkdf2_sha1(pw, pwlen, salt, 16, 1000, dk, sizeof dk);
  orc_winzip_ctr(dk, 32, data, n);
  orc_hmac_sha1(dk + 32, 32, data, n, h);
  memcpy(ver, dk + 64, 2);
  memcpy(mac, h, 10);
}
