/*
 * oracle/orc_crypt.h -- CPU ORACLE (test infrastructure only; see orc.h): encrypted ZIP members.
 *   aes.c          AES forward cipher, SHA-1, HMAC-SHA1, PBKDF2, WinZip CTR, ZipCrypto
 *   zip_crypt.c    the ZipCrypto / AES branches of ZipFile.read / getStream (zip_file.dart:98-134, 164-216, 260-359)
 *   zip_enc_crypt.c  ZipEncoder(password:) (zip_encoder.dart:166-183, 270-310, 347-437)
 */
#ifndef ORC_CRYPT_H
#define ORC_CRYPT_H
#include "orc.h"

/* extra statuses of orc_zip_member_password */
#define ORC_BAD_PASSWORD 4 /* AES password verifier mismatch: Exception('password error') (zip_file.dart:333-335) */
#define ORC_BAD_MAC 5      /* AES authentication code mismatch: Exception("macs don't match") (:339-341)          */
#define ORC_ZIP_NONE 0
#define ORC_ZIP_ZIPCRYPTO 1
#define ORC_ZIP_AES 2
/* ZipFile.read :98-130: which mode the member uses, the AES strength byte and the method its content is stored with;
 * ORC_THROW when the scan of the local extra field reads past its end */
int orc_zip_crypt_info(const uint8_t *b, size_t blen, const orc_zip_entry *e, uint32_t *mode, uint32_t *strength,
                       uint32_t *method);
/* getStream with a password (pw == NULL: no password, exactly orc_zip_member) */
int orc_zip_member_password(const uint8_t *b, size_t blen, const orc_zip_entry *e, int web_eos, const uint8_t *pw,
                            size_t pwlen, uint8_t **out, size_t *out_len);
int orc_aes_expand(const uint8_t *key, int key_len, uint32_t *rk); /* -> rounds; rk holds 4 * (rounds + 1) words */
void orc_aes_encrypt_block(const uint32_t *rk, int nr, const uint8_t in[16], uint8_t out[16]);
void orc_winzip_ctr(const uint8_t *key, int key_len, uint8_t *data, size_t n);
void orc_sha1(const uint8_t *p, size_t n, uint8_t out[20]);
void orc_hmac_sha1(const uint8_t *key, size_t klen, const uint8_t *msg, size_t n, uint8_t out[20]);
void orc_pbkdf2_sha1(const uint8_t *pw, size_t pwlen, const uint8_t *salt, size_t slen, int iters, uint8_t *out, size_t dklen);
void orc_zipcrypto_decrypt(const uint8_t *pw, size_t pwlen, const uint8_t *in, size_t n, uint8_t *out);
void orc_zipcrypto_encrypt(const uint8_t *pw, size_t pwlen, const uint8_t *in, size_t n, uint8_t *out);
/* ZipEncoder(password:): AES-256 members; salts[16 * i] is member i's salt (only files use theirs).
 * pw == NULL: exactly orc_zip_encode. */
int orc_zip_encode_password(const orc_zip_member_in *m, size_t n, int level, const char *comment, const uint8_t *pw,
                            size_t pwlen, const uint8_t *salts, uint8_t **out, size_t *out_len);
/* the bytes of one AES-256 member as ZipEncoder._encryptCompressedData makes them, in place: CTR over data, then the
 * verifier (2 bytes) and the MAC (10 bytes) */
void orc_zip_aes_encrypt(uint8_t *data, size_t n, const uint8_t salt[16], const uint8_t *pw, size_t pwlen, uint8_t ver[2],
                         uint8_t mac[10]);

#endif
