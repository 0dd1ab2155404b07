// zip_crypt_kernels.cu -- encrypted ZIP members on the device: WinZip AES (PBKDF2-HMAC-SHA1 key derivation, AES-CTR,
// HMAC-SHA1 authentication) and the traditional ZipCrypto stream cipher.
//
// Reference (paths relative to the reference's lib/src/):
//   util/aes.dart:17-81                 Aes.processData: counter block = little-endian block number from 1 in bytes 0-3,
//                                       zeros in 4-15; HMAC-SHA1 over the ciphertext, cut to 10 bytes
//   util/encryption.dart:60-132         PcPBKDF2KeyDerivator (1000 iterations of HMAC-SHA1), PcAESEngine (forward cipher)
//   codecs/zip/zip_file.dart:260-359    _initKeys / _updateKeys / _decodeZipCrypto, _decodeAes, deriveKey
//
// Work shapes:
//   k_zip_pbkdf2     one thread per (member, 20-byte block of the derived key); the password's HMAC pad states are hashed
//                    once on the host, so each of the 1000 iterations is two SHA-1 compressions.  The tail expands each
//                    member's AES key schedule and writes its 2-byte password verifier.
//   k_zip_aes_ctr    a grid over the 16-byte blocks of all members: every CTA takes one tile (zip_ctr_tile_blocks() blocks) of
//                    one member; S-box, T-tables and round keys live in shared memory.  src and dst may be equal.
//   k_zip_hmac_sha1  one thread per member over its ciphertext (a serial chain: one large member runs at one thread's rate).
//   k_zipcrypto      one thread per member (serial by construction: every key update depends on the previous byte).
// The AES S-box is derived from GF(2^8) inversion in shared memory at the start of each CTA rather than written out.
//
// Built by nvcc for sm_90a (product).  The CPU emulation build of the library (tests/host_emul, -DB200Z_EMU against
// cuda_emu.h) compiles this file as part of b200z_api.cu, which includes it under B200Z_EMU; the launches go through
// ZC_LAUNCH so that both compilers take them.
#include "b200z_internal.h"

#ifdef B200Z_EMU
#define ZC_LAUNCH(kern, grid, block, stream, ...) B200Z_LAUNCH(kern, grid, block, 0, stream, __VA_ARGS__)
#else
#define ZC_LAUNCH(kern, grid, block, stream, ...) kern<<<grid, block, 0, stream>>>(__VA_ARGS__)
#endif

namespace b200z {

#ifdef __CUDA_ARCH__
#define ZC_UNROLL _Pragma("unroll")
#else
#define ZC_UNROLL  // (the host pass of __host__ __device__ code)
#endif

__host__ __device__ __forceinline__ uint32_t zc_rol(uint32_t v, int s) { return (v << s) | (v >> (32 - s)); }

// SHA-1 compression of one 64-byte block given as 16 big-endian words (w is clobbered)
__host__ __device__ __forceinline__ void sha1_compress(uint32_t h[5], uint32_t w[16]) {
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4];
ZC_UNROLL
  for (int i = 0; i < 80; ++i) {
    uint32_t wi;
    if (i < 16) {
      wi = w[i];
    } else {
      wi = zc_rol(w[(i + 13) & 15] ^ w[(i + 8) & 15] ^ w[(i + 2) & 15] ^ w[i & 15], 1);
      w[i & 15] = wi;
    }
    uint32_t f, k;
    if (i < 20) {
      f = (b & c) | (~b & d);
      k = 0x5A827999u;
    } else if (i < 40) {
      f = b ^ c ^ d;
      k = 0x6ED9EBA1u;
    } else if (i < 60) {
      f = (b & c) | (b & d) | (c & d);
      k = 0x8F1BBCDCu;
    } else {
      f = b ^ c ^ d;
      k = 0xCA62C1D6u;
    }
    const uint32_t t = zc_rol(a, 5) + f + e + k + wi;
    e = d;
    d = c;
    c = zc_rol(b, 30);
    b = a;
    a = t;
  }
  h[0] += a;
  h[1] += b;
  h[2] += c;
  h[3] += d;
  h[4] += e;
}

__host__ __device__ __forceinline__ void sha1_iv(uint32_t h[5]) {
  h[0] = 0x67452301u;
  h[1] = 0xEFCDAB89u;
  h[2] = 0x98BADCFEu;
  h[3] = 0x10325476u;
  h[4] = 0xC3D2E1F0u;
}

// SHA-1 states after the HMAC inner / outer pad block of a key of at most 64 bytes
__host__ __device__ __forceinline__ void hmac_pad_states(const uint8_t *key, uint32_t klen, uint32_t ipad[5], uint32_t opad[5]) {
  uint32_t kw[16], w[16];
ZC_UNROLL
  for (int i = 0; i < 16; ++i) kw[i] = 0;
  for (uint32_t i = 0; i < klen; ++i) kw[i >> 2] |= (uint32_t)key[i] << (24 - 8 * (i & 3));
  sha1_iv(ipad);
ZC_UNROLL
  for (int i = 0; i < 16; ++i) w[i] = kw[i] ^ 0x36363636u;
  sha1_compress(ipad, w);
  sha1_iv(opad);
ZC_UNROLL
  for (int i = 0; i < 16; ++i) w[i] = kw[i] ^ 0x5c5c5c5cu;
  sha1_compress(opad, w);
}

// PcHMac, block 64: a key longer than the block is replaced by its SHA-1 (a password may be that long)
void zip_hmac_pads(const uint8_t *key, size_t klen, ZipHmacPads *p) {
  if (klen <= 64) {
    hmac_pad_states(key, (uint32_t)klen, p->ipad, p->opad);
    return;
  }
  std::vector<uint8_t> msg(key, key + klen);
  msg.push_back(0x80);
  while (msg.size() % 64 != 56) msg.push_back(0);
  const uint64_t bits = (uint64_t)klen * 8;
  for (int i = 7; i >= 0; --i) msg.push_back((uint8_t)(bits >> (8 * i)));
  uint32_t h[5], w[16];
  sha1_iv(h);
  for (size_t q = 0; q < msg.size(); q += 64) {
    for (int i = 0; i < 16; ++i)
      w[i] = ((uint32_t)msg[q + 4 * i] << 24) | ((uint32_t)msg[q + 4 * i + 1] << 16) | ((uint32_t)msg[q + 4 * i + 2] << 8) |
             msg[q + 4 * i + 3];
    sha1_compress(h, w);
  }
  uint8_t d[20];
  for (int i = 0; i < 20; ++i) d[i] = (uint8_t)(h[i >> 2] >> (24 - 8 * (i & 3)));
  hmac_pad_states(d, 20, p->ipad, p->opad);
}

// ---- ZipCrypto keys (zip_file.dart:260-286) ----
__host__ __device__ __forceinline__ uint32_t crc_entry(uint32_t i) {
  uint32_t c = i;
  for (int k = 0; k < 8; ++k) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
  return c;
}
void zipcrypto_keys(const uint8_t *pw, size_t len, uint32_t k[3]) {
  k[0] = 305419896u;
  k[1] = 591751049u;
  k[2] = 878082192u;
  for (size_t i = 0; i < len; ++i) {  // _updateKeys with the low byte of each code unit (getCrc32Byte masks it)
    k[0] = crc_entry((k[0] ^ pw[i]) & 0xff) ^ (k[0] >> 8);
    k[1] = (k[1] + (k[0] & 0xff)) * 134775813u + 1u;
    k[2] = crc_entry((k[2] ^ (k[1] >> 24)) & 0xff) ^ (k[2] >> 8);
  }
}

// ---- AES tables in shared memory ----
__device__ __forceinline__ uint32_t gf_xt(uint32_t a) { return ((a << 1) ^ ((a & 0x80) ? 0x1b : 0)) & 0xff; }
__device__ __forceinline__ uint32_t gf_mul(uint32_t a, uint32_t b) {
  uint32_t r = 0;
  for (int i = 0; i < 8; ++i) {
    if (b & 1) r ^= a;
    a = gf_xt(a);
    b >>= 1;
  }
  return r;
}
// S-box entry x: the affine map of x^-1 (x^254) in GF(2^8)
__device__ inline uint32_t aes_sbox_entry(uint32_t x) {
  uint32_t inv = 0;
  if (x) {
    uint32_t p = x, r = 1;
    for (int e = 254; e; e >>= 1) {
      if (e & 1) r = gf_mul(r, p);
      p = gf_mul(p, p);
    }
    inv = r;
  }
  uint32_t s = inv;
  for (int k = 1; k <= 4; ++k) s ^= ((inv << k) | (inv >> (8 - k))) & 0xff;
  return s ^ 0x63;
}

__device__ __forceinline__ uint32_t be_load_salt(const uint8_t *p) {
  return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
}

// ---------------------------------------------------------------------------------------------
// k_zip_pbkdf2: 4 threads per member (lane & 3 = output block); 32 members per CTA of 128 threads
// ---------------------------------------------------------------------------------------------
constexpr int kPbkdfThreads = 128;
__global__ void __launch_bounds__(kPbkdfThreads) k_zip_pbkdf2(const ZipAesMember *__restrict__ m, uint32_t n, ZipHmacPads pads,
                                                              uint8_t *__restrict__ dk_out, uint32_t *__restrict__ rk_out,
                                                              uint8_t *__restrict__ ver_out) {
  __shared__ uint8_t sbox[256];
  __shared__ uint32_t dk[kPbkdfThreads / 4][20];  // 80 bytes of derived key per member, as big-endian words
  for (uint32_t x = threadIdx.x; x < 256; x += blockDim.x) sbox[x] = (uint8_t)aes_sbox_entry(x);
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x, mi = g >> 2, blk = g & 3, lm = threadIdx.x >> 2;
  uint32_t ks = 0;
  if (mi < n) {
    ks = m[mi].key_len;
    const uint32_t sl = m[mi].salt_len;
    if (blk * 20 < 2 * ks + 2) {
      uint32_t w[16], u[5], t[5], h[5];
      // U1 = HMAC(salt || INT(blk + 1))
      for (int i = 0; i < 16; ++i) w[i] = 0;
      for (uint32_t i = 0; i < sl / 4; ++i) w[i] = be_load_salt(m[mi].salt + 4 * i);
      w[sl / 4] = blk + 1;
      w[sl / 4 + 1] = 0x80000000u;
      w[15] = (64 + sl + 4) * 8;
      for (int i = 0; i < 5; ++i) h[i] = pads.ipad[i];
      sha1_compress(h, w);
      for (int i = 0; i < 5; ++i) u[i] = h[i];
      for (int i = 0; i < 5; ++i) h[i] = pads.opad[i];
      for (int i = 0; i < 5; ++i) w[i] = u[i];
      w[5] = 0x80000000u;
      for (int i = 6; i < 15; ++i) w[i] = 0;
      w[15] = (64 + 20) * 8;
      sha1_compress(h, w);
      for (int i = 0; i < 5; ++i) t[i] = u[i] = h[i];
      for (int c = 1; c < 1000; ++c) {
        for (int i = 0; i < 5; ++i) h[i] = pads.ipad[i];
        for (int i = 0; i < 5; ++i) w[i] = u[i];
        w[5] = 0x80000000u;
        for (int i = 6; i < 15; ++i) w[i] = 0;
        w[15] = (64 + 20) * 8;
        sha1_compress(h, w);
        for (int i = 0; i < 5; ++i) w[i] = h[i];
        for (int i = 0; i < 5; ++i) h[i] = pads.opad[i];
        w[5] = 0x80000000u;
        for (int i = 6; i < 15; ++i) w[i] = 0;
        w[15] = (64 + 20) * 8;
        sha1_compress(h, w);
        for (int i = 0; i < 5; ++i) {
          u[i] = h[i];
          t[i] ^= h[i];
        }
      }
      for (int i = 0; i < 5; ++i) dk[lm][blk * 5 + i] = t[i];
    }
  }
  __syncthreads();
  if (mi >= n || blk != 0) return;
  // the derived key: ks bytes of AES key, ks bytes of HMAC key, 2 bytes of password verifier
  uint8_t *dko = dk_out + (size_t)mi * 80;
  for (uint32_t i = 0; i < 2 * ks + 2; ++i) dko[i] = (uint8_t)(dk[lm][i >> 2] >> (24 - 8 * (i & 3)));
  ver_out[2 * mi] = dko[2 * ks];
  ver_out[2 * mi + 1] = dko[2 * ks + 1];
  // AES key schedule (FIPS-197 5.2)
  uint32_t *rk = rk_out + (size_t)mi * 60;
  const uint32_t nk = ks / 4, nr = nk + 6;
  for (uint32_t i = 0; i < nk; ++i) rk[i] = dk[lm][i];
  uint32_t rcon = 1;
  for (uint32_t i = nk; i < 4 * (nr + 1); ++i) {
    uint32_t t = rk[i - 1];
    if (i % nk == 0) {
      t = (t << 8) | (t >> 24);
      t = ((uint32_t)sbox[t >> 24] << 24) | ((uint32_t)sbox[(t >> 16) & 255] << 16) | ((uint32_t)sbox[(t >> 8) & 255] << 8) |
          sbox[t & 255];
      t ^= rcon << 24;
      rcon = gf_xt(rcon);
    } else if (nk > 6 && i % nk == 4) {
      t = ((uint32_t)sbox[t >> 24] << 24) | ((uint32_t)sbox[(t >> 16) & 255] << 16) | ((uint32_t)sbox[(t >> 8) & 255] << 8) |
          sbox[t & 255];
    }
    rk[i] = rk[i - nk] ^ t;
  }
}

// ---------------------------------------------------------------------------------------------
// k_zip_aes_ctr: tile = (member, first 16-byte block); each thread takes kCtrPerThread blocks of the tile
// ---------------------------------------------------------------------------------------------
constexpr int kCtrThreads = 256;
constexpr int kCtrPerThread = 4;
__global__ void __launch_bounds__(kCtrThreads) k_zip_aes_ctr(const ZipAesMember *__restrict__ m, const uint32_t *__restrict__ rk_all,
                                                             const ZipCtrTile *__restrict__ tiles, uint8_t *base) {
  __shared__ uint32_t te[4][256];
  __shared__ uint8_t sbox[256];
  __shared__ uint32_t rk[60];
  const ZipCtrTile tile = tiles[blockIdx.x];
  const uint32_t x = threadIdx.x;
  {
    const uint32_t s = aes_sbox_entry(x);
    sbox[x] = (uint8_t)s;
    const uint32_t t = (gf_xt(s) << 24) | (s << 16) | (s << 8) | (gf_xt(s) ^ s);
    te[0][x] = t;
    te[1][x] = (t >> 8) | (t << 24);
    te[2][x] = (t >> 16) | (t << 16);
    te[3][x] = (t >> 24) | (t << 8);
  }
  if (x < 60) rk[x] = rk_all[(size_t)tile.member * 60 + x];
  __syncthreads();
  const ZipAesMember &mm = m[tile.member];
  const uint32_t nr = mm.key_len / 4 + 6;
  const uint64_t len = mm.len;
  const uint8_t *src = base + mm.src_off;
  uint8_t *dst = base + mm.dst_off;
  for (int q = 0; q < kCtrPerThread; ++q) {
    const uint64_t b = tile.first_block + (uint64_t)q * kCtrThreads + x;
    if (b * 16 >= len) break;
    const uint32_t ctr = (uint32_t)(b + 1);  // nonce, little-endian in bytes 0-3
    uint32_t s0 = ((ctr & 0xff) << 24 | ((ctr >> 8) & 0xff) << 16 | ((ctr >> 16) & 0xff) << 8 | (ctr >> 24)) ^ rk[0];
    uint32_t s1 = rk[1], s2 = rk[2], s3 = rk[3];
    for (uint32_t r = 1; r < nr; ++r) {
      const uint32_t *k = rk + 4 * r;
      const uint32_t t0 = te[0][s0 >> 24] ^ te[1][(s1 >> 16) & 255] ^ te[2][(s2 >> 8) & 255] ^ te[3][s3 & 255] ^ k[0];
      const uint32_t t1 = te[0][s1 >> 24] ^ te[1][(s2 >> 16) & 255] ^ te[2][(s3 >> 8) & 255] ^ te[3][s0 & 255] ^ k[1];
      const uint32_t t2 = te[0][s2 >> 24] ^ te[1][(s3 >> 16) & 255] ^ te[2][(s0 >> 8) & 255] ^ te[3][s1 & 255] ^ k[2];
      const uint32_t t3 = te[0][s3 >> 24] ^ te[1][(s0 >> 16) & 255] ^ te[2][(s1 >> 8) & 255] ^ te[3][s2 & 255] ^ k[3];
      s0 = t0;
      s1 = t1;
      s2 = t2;
      s3 = t3;
    }
    const uint32_t *k = rk + 4 * nr;
    uint32_t o[4];
    o[0] = (((uint32_t)sbox[s0 >> 24] << 24) | ((uint32_t)sbox[(s1 >> 16) & 255] << 16) | ((uint32_t)sbox[(s2 >> 8) & 255] << 8) |
            sbox[s3 & 255]) ^ k[0];
    o[1] = (((uint32_t)sbox[s1 >> 24] << 24) | ((uint32_t)sbox[(s2 >> 16) & 255] << 16) | ((uint32_t)sbox[(s3 >> 8) & 255] << 8) |
            sbox[s0 & 255]) ^ k[1];
    o[2] = (((uint32_t)sbox[s2 >> 24] << 24) | ((uint32_t)sbox[(s3 >> 16) & 255] << 16) | ((uint32_t)sbox[(s0 >> 8) & 255] << 8) |
            sbox[s1 & 255]) ^ k[2];
    o[3] = (((uint32_t)sbox[s3 >> 24] << 24) | ((uint32_t)sbox[(s0 >> 16) & 255] << 16) | ((uint32_t)sbox[(s1 >> 8) & 255] << 8) |
            sbox[s2 & 255]) ^ k[3];
    const uint64_t at = b * 16;
    const uint32_t cnt = len - at < 16 ? (uint32_t)(len - at) : 16u;
#pragma unroll
    for (uint32_t i = 0; i < 16; ++i)
      if (i < cnt) dst[at + i] = src[at + i] ^ (uint8_t)(o[i >> 2] >> (24 - 8 * (i & 3)));
  }
}

// ---------------------------------------------------------------------------------------------
// k_zip_hmac_sha1: one thread per member, HMAC-SHA1 over the ciphertext at src_off (or dst_off when `after_ctr`)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t bswap32(uint32_t v) { return __byte_perm(v, 0, 0x0123); }
__global__ void __launch_bounds__(64) k_zip_hmac_sha1(const ZipAesMember *__restrict__ m, uint32_t n, const uint8_t *__restrict__ dk_all,
                                                      const uint8_t *base, int after_ctr, uint8_t *__restrict__ mac_out) {
  const uint32_t mi = blockIdx.x * blockDim.x + threadIdx.x;
  if (mi >= n) return;
  const ZipAesMember &mm = m[mi];
  const uint32_t ks = mm.key_len;
  uint32_t ipad[5], opad[5], h[5], w[16];
  hmac_pad_states(dk_all + (size_t)mi * 80 + ks, ks, ipad, opad);
  const uint8_t *p = base + (after_ctr ? mm.dst_off : mm.src_off);
  const uint64_t len = mm.len;
  for (int i = 0; i < 5; ++i) h[i] = ipad[i];
  // whole blocks: aligned 32-bit loads, shifted into place (the buffers carry >= 4 readable bytes past every member)
  const uint32_t mis = (uint32_t)((uintptr_t)p & 3);
  const uint32_t *aw = (const uint32_t *)(p - mis);
  uint64_t done = 0;
  for (; done + 64 <= len; done += 64, aw += 16) {
    uint32_t cur = aw[0];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const uint32_t nxt = aw[i + 1];
      const uint32_t le = mis ? __funnelshift_r(cur, nxt, 8 * mis) : cur;
      w[i] = bswap32(le);
      cur = nxt;
    }
    sha1_compress(h, w);
  }
  // tail + padding: the message length includes the 64-byte ipad block
  const uint32_t r = (uint32_t)(len - done);
  const uint64_t bits = (len + 64) * 8;
  for (int i = 0; i < 16; ++i) w[i] = 0;
  for (uint32_t i = 0; i < r; ++i) w[i >> 2] |= (uint32_t)p[done + i] << (24 - 8 * (i & 3));
  w[r >> 2] |= 0x80u << (24 - 8 * (r & 3));
  if (r >= 56) {
    sha1_compress(h, w);
    for (int i = 0; i < 16; ++i) w[i] = 0;
  }
  w[14] = (uint32_t)(bits >> 32);
  w[15] = (uint32_t)bits;
  sha1_compress(h, w);
  for (int i = 0; i < 5; ++i) w[i] = h[i];
  for (int i = 0; i < 5; ++i) h[i] = opad[i];
  w[5] = 0x80000000u;
  for (int i = 6; i < 15; ++i) w[i] = 0;
  w[15] = (64 + 20) * 8;
  sha1_compress(h, w);
  for (int i = 0; i < 10; ++i) mac_out[(size_t)mi * 10 + i] = (uint8_t)(h[i >> 2] >> (24 - 8 * (i & 3)));
}

// ---------------------------------------------------------------------------------------------
// k_zipcrypto: one thread per member; the 12 header bytes are decrypted and dropped
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_zipcrypto(const ZipCryptoMember *__restrict__ m, uint32_t n, uint32_t k0, uint32_t k1,
                                                   uint32_t k2, uint8_t *base) {
  __shared__ uint32_t crc[256];
  for (uint32_t x = threadIdx.x; x < 256; x += blockDim.x) crc[x] = crc_entry(x);
  __syncthreads();
  const uint32_t mi = blockIdx.x * blockDim.x + threadIdx.x;
  if (mi >= n) return;
  const ZipCryptoMember mm = m[mi];
  const uint8_t *src = base + mm.src_off;
  uint8_t *dst = base + mm.dst_off;
  for (uint64_t i = 0; i < mm.len; ++i) {
    const uint32_t t = (k2 & 0xffff) | 2;
    const uint32_t pl = (src[i] ^ ((t * (t ^ 1)) >> 8)) & 0xff;
    k0 = crc[(k0 ^ pl) & 0xff] ^ (k0 >> 8);
    k1 = (k1 + (k0 & 0xff)) * 134775813u + 1u;
    k2 = crc[(k2 ^ (k1 >> 24)) & 0xff] ^ (k2 >> 8);
    if (i >= 12) dst[i - 12] = (uint8_t)pl;
  }
}

// ---------------------------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------------------------
cudaError_t zip_launch_pbkdf2(const ZipAesMember *d_m, uint32_t n, const ZipHmacPads &pads, uint8_t *d_dk, uint32_t *d_rk,
                              uint8_t *d_ver, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  const uint32_t grid = (uint32_t)(((uint64_t)n * 4 + kPbkdfThreads - 1) / kPbkdfThreads);
  ZC_LAUNCH(k_zip_pbkdf2, grid, kPbkdfThreads, s, d_m, n, pads, d_dk, d_rk, d_ver);
  count_launch();
  return cudaGetLastError();
}

cudaError_t zip_launch_aes_ctr(const ZipAesMember *d_m, const uint32_t *d_rk, const ZipCtrTile *d_tiles, uint32_t n_tiles,
                               uint8_t *d_base, cudaStream_t s) {
  if (n_tiles == 0) return cudaSuccess;
  ZC_LAUNCH(k_zip_aes_ctr, n_tiles, kCtrThreads, s, d_m, d_rk, d_tiles, d_base);
  count_launch();
  return cudaGetLastError();
}

uint64_t zip_ctr_tile_blocks() { return (uint64_t)kCtrThreads * kCtrPerThread; }

cudaError_t zip_launch_hmac(const ZipAesMember *d_m, uint32_t n, const uint8_t *d_dk, const uint8_t *d_base, bool after_ctr,
                            uint8_t *d_mac, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  ZC_LAUNCH(k_zip_hmac_sha1, (n + 63) / 64, 64, s, d_m, n, d_dk, d_base, after_ctr ? 1 : 0, d_mac);
  count_launch();
  return cudaGetLastError();
}

cudaError_t zip_launch_zipcrypto(const ZipCryptoMember *d_m, uint32_t n, const uint32_t keys[3], uint8_t *d_base, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  ZC_LAUNCH(k_zipcrypto, (n + 127) / 128, 128, s, d_m, n, keys[0], keys[1], keys[2], d_base);
  count_launch();
  return cudaGetLastError();
}

}  // namespace b200z
