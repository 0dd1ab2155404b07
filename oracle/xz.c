/*
 * oracle/xz.c -- CPU ORACLE (test infrastructure only; see orc.h, orc_xz.h): the reference's XZ codec restated in C.
 *
 *   codecs/xz_decoder.dart        _XZStreamDecoder: container walk, LZMA2 chunk loop, checks, index, footer
 *   codecs/lzma/lzma_decoder.dart LzmaDecoder: one instance for the whole stream, trimDictionary, buffer growth
 *   codecs/lzma/range_decoder.dart RangeDecoder / RangeDecoderTable
 *   codecs/xz_encoder.dart        XZEncoder: one stored chunk, 8 MiB dictionary byte, index, footer, checks
 *   util/_crc64_io.dart           getCrc64 (ECMA-182, reflected)
 *
 * Dart ints are 64-bit: the range coder's `code` is an int64 here (it only leaves 32 bits on damaged input, where the
 * reference keeps going with the wider value).  Every Dart RangeError (an index outside a typed list, a read past the
 * end of an InputMemoryStream) is a longjmp to ORC_THROW.
 */
#include <setjmp.h>
#include <stdlib.h>
#include <string.h>

#include "orc_xz.h"

typedef struct {
  jmp_buf jb;
} xz_ctx;

static void xz_throw(xz_ctx *c) { longjmp(c->jb, 1); }

/* ---- InputMemoryStream views (input_memory_stream.dart:15-27, 58-62, 90-134; input_stream.dart:48-136) ---- */
typedef struct {
  const uint8_t *b;
  int64_t len, pos;
} view;

static int eos(const view *s) { return s->pos >= s->len; }
static int rb(xz_ctx *c, view *s) {
  if (s->pos < 0 || s->pos >= s->len) xz_throw(c);
  return s->b[s->pos++];
}
/* readBytes: subset(position, count) clamped to the end (input_memory_stream.dart:19-22); a negative count makes
 * Uint8List.view throw */
static view read_bytes(xz_ctx *c, view *s, int64_t count) {
  if (count < 0) xz_throw(c);
  view v;
  int64_t avail = s->len - s->pos;
  v.b = s->b + s->pos;
  v.len = count < avail ? count : avail;
  v.pos = 0;
  s->pos += v.len;
  return v;
}
static void skip(view *s, int64_t n) {
  s->pos += n;
  if (s->pos < 0) s->pos = 0;
  if (s->pos > s->len) s->pos = s->len;
}
static uint32_t read_u32(xz_ctx *c, view *s) {
  uint32_t b1 = rb(c, s), b2 = rb(c, s), b3 = rb(c, s), b4 = rb(c, s);
  return b4 << 24 | b3 << 16 | b2 << 8 | b1;
}
static uint64_t read_u64(xz_ctx *c, view *s) {
  uint64_t v = 0;
  for (int i = 0; i < 8; ++i) v |= (uint64_t)rb(c, s) << (8 * i);
  return v;
}
/* _readMultibyteInteger (xz_decoder.dart:431-442): Dart's << past 63 bits gives 0 */
static int64_t read_mbi(xz_ctx *c, view *s) {
  uint64_t value = 0;
  int64_t shift = 0;
  for (;;) {
    int d = rb(c, s);
    if (shift < 64) value |= (uint64_t)(d & 0x7f) << shift;
    if (!(d & 0x80)) return (int64_t)value;
    shift += 7;
  }
}
/* _readPadding (:447-457) */
static int64_t read_padding(xz_ctx *c, view *s) {
  int64_t n = 0;
  while (s->pos % 4 != 0) {
    if (rb(c, s) != 0) return -1;
    n++;
  }
  return n;
}

/* ---- CRC-64 (_crc64_io.dart:5-11) ---- */
static uint64_t crc64_tab[256];
static void crc64_init(void) {
  if (crc64_tab[1]) return;
  for (int i = 0; i < 256; ++i) {
    uint64_t r = (uint64_t)i;
    for (int k = 0; k < 8; ++k) r = (r & 1) ? (r >> 1) ^ 0xC96C5795D7870F42ull : r >> 1;
    crc64_tab[i] = r;
  }
}
uint64_t orc_crc64(const uint8_t *p, size_t n, uint64_t crc) {
  crc64_init();
  crc = ~crc;
  for (size_t i = 0; i < n; ++i) crc = crc64_tab[(crc & 0xff) ^ p[i]] ^ (crc >> 8);
  return ~crc;
}

/* ---- RangeDecoder (range_decoder.dart) ---- */
#define NPOS_MAX 32 /* pb <= 5: props ~/ 45 of a byte */
typedef struct {
  uint16_t form[2], shrt[NPOS_MAX][8], med[NPOS_MAX][8], lng[256];
} lendec;

typedef struct {
  int64_t range, code;
  const uint8_t *buf;
  int64_t blen, bpos;
  int pb, lp, lc;
  uint16_t nonlit[12][12], rep[12], rep0[12], longrep0[12][12], rep1[12], rep2[12];
  uint16_t *lit, *mlit0, *mlit1; /* [nlit][256] each */
  int64_t nlit;
  lendec mlen, rlen;
  uint16_t slot[4][64], dshort[10][32], dalign[16];
  int64_t d0, d1, d2, d3;
  int state;
  uint8_t *dict;
  int64_t dlen, wp, cap;
} lzma;

static int next_byte(xz_ctx *c, lzma *z) {
  if (z->bpos < 0 || z->bpos >= z->blen) xz_throw(c);
  return z->buf[z->bpos++];
}
static inline void norm(xz_ctx *c, lzma *z) {
  if (z->range < 0x1000000) {
    z->range <<= 8;
    z->code = (int64_t)((uint64_t)z->code << 8) | next_byte(c, z);
  }
}
/* readBit (:62-79); `size` is the table's length: an index past it is a RangeError */
static int read_bit(xz_ctx *c, lzma *z, uint16_t *t, int64_t size, int64_t index) {
  norm(c, z);
  if (index >= size) xz_throw(c);
  const int64_t p = t[index];
  const int64_t bound = (z->range >> 11) * p;
  if (z->code < bound) {
    z->range = bound;
    t[index] += (2048 - p) >> 5;
    return 0;
  }
  z->range -= bound;
  z->code -= bound;
  t[index] -= p >> 5;
  return 1;
}
static int decode_byte(xz_ctx *c, lzma *z, uint16_t *probs) { /* :81-101 */
  int symbol = 1;
  for (int i = 0; i < 8; ++i) symbol = (symbol << 1) | read_bit(c, z, probs, 256, symbol);
  return symbol & 0xff;
}
static int decode_matched_byte(xz_ctx *c, lzma *z, uint16_t *probs, uint16_t *m0, uint16_t *m1, int match_byte) { /* :103-144 */
  int symbol = 1, matched = 1;
  for (int i = 7; i >= 0; --i) {
    if (matched) {
      const int mb = (match_byte >> i) & 1;
      const int b = read_bit(c, z, mb ? m1 : m0, 256, symbol);
      symbol = (symbol << 1) | b;
      matched = b == mb;
    } else {
      symbol = (symbol << 1) | read_bit(c, z, probs, 256, symbol);
    }
  }
  return symbol & 0xff;
}
static int64_t bittree(xz_ctx *c, lzma *z, uint16_t *t, int64_t size, int count) { /* :147-157 */
  int64_t value = 0, prefix = 1;
  for (int i = 0; i < count; ++i) {
    value = ((value << 1) | read_bit(c, z, t, size, prefix | value)) & 0xffffffff;
    prefix = (prefix << 1) & 0xffffffff;
  }
  return value;
}
static int64_t bittree_rev(xz_ctx *c, lzma *z, uint16_t *t, int64_t size, int count) { /* :160-170 */
  int64_t value = 0, prefix = 1;
  for (int i = 0; i < count; ++i) {
    value = (value | (int64_t)read_bit(c, z, t, size, prefix | value) << i) & 0xffffffff;
    prefix = (prefix << 1) & 0xffffffff;
  }
  return value;
}
static int64_t read_direct(xz_ctx *c, lzma *z, int count) { /* :173-190 */
  int64_t value = 0;
  for (int i = 0; i < count; ++i) {
    norm(c, z);
    z->range >>= 1;
    z->code -= z->range;
    value <<= 1;
    if (z->code & 0x80000000) z->code += z->range;
    else value++;
  }
  return value;
}

/* ---- LzmaDecoder (lzma_decoder.dart) ---- */
static void fill_half(uint16_t *t, size_t n) {
  for (size_t i = 0; i < n; ++i) t[i] = 1024;
}
static void lz_reset(lzma *z, int pb, int lp, int lc, int reset_dict) { /* :104-160; -1 = keep */
  if (pb >= 0) z->pb = pb;
  if (lp >= 0) z->lp = lp;
  if (lc >= 0) z->lc = lc;
  z->state = 0;
  z->d0 = z->d1 = z->d2 = z->d3 = 0;
  const int64_t nl = (int64_t)1 << (z->lp + z->lc);
  if (nl > z->nlit) { /* the literal tables only ever grow (:122-129) */
    z->lit = realloc(z->lit, nl * 512);
    z->mlit0 = realloc(z->mlit0, nl * 512);
    z->mlit1 = realloc(z->mlit1, nl * 512);
    z->nlit = nl;
  }
  fill_half(&z->nonlit[0][0], 144);
  fill_half(z->rep, 12);
  fill_half(z->rep0, 12);
  fill_half(&z->longrep0[0][0], 144);
  fill_half(z->rep1, 12);
  fill_half(z->rep2, 12);
  fill_half(z->lit, z->nlit * 256);
  fill_half(z->mlit0, z->nlit * 256);
  fill_half(z->mlit1, z->nlit * 256);
  fill_half((uint16_t *)&z->mlen, sizeof(lendec) / 2);
  fill_half((uint16_t *)&z->rlen, sizeof(lendec) / 2);
  fill_half(&z->slot[0][0], 256);
  fill_half(&z->dshort[0][0], 320);
  fill_half(z->dalign, 16);
  if (reset_dict) {
    free(z->dict);
    z->dict = NULL;
    z->dlen = 0;
    z->wp = 0;
  }
}
static void lz_trim(lzma *z, int64_t max_size) { /* :87-101 */
  const int64_t threshold = max_size + (max_size >> 2);
  if (z->wp <= threshold) return;
  const int align_bits = z->pb > z->lp ? z->pb : z->lp;
  const int64_t keep = max_size + (z->wp & (((int64_t)1 << align_bits) - 1));
  memmove(z->dict, z->dict + (z->wp - keep), (size_t)keep);
  z->wp = keep;
}
static void lz_grow(lzma *z, int64_t final_size) { /* :165-184, :199-219: a new zeroed list holding [0, wp) */
  if (final_size <= z->dlen) return;
  int64_t n = z->dlen == 0 ? final_size : z->dlen;
  while (n < final_size) n *= 2;
  if (z->cap > 0 && n > z->cap && z->cap >= final_size) n = z->cap;
  uint8_t *d = calloc((size_t)n, 1);
  if (z->wp > 0) memcpy(d, z->dict, (size_t)z->wp);
  free(z->dict);
  z->dict = d;
  z->dlen = n;
}
/* decodeUncompressed (:162-191): the clamped bytes go to the output, the write position moves by the full length */
static view lz_stored(xz_ctx *c, lzma *z, view *in, int64_t length) {
  view d = read_bytes(c, in, length);
  lz_grow(z, z->wp + length);
  memcpy(z->dict + z->wp, d.b, (size_t)d.len);
  z->wp += length;
  return d;
}
static void repeat_data(xz_ctx *c, lzma *z, int64_t distance, int64_t length) { /* :371-386 */
  const int64_t src = z->wp - distance - 1;
  if (distance >= length) {
    if (src < 0 || z->wp + length > z->dlen) xz_throw(c); /* setRange's range checks */
    memcpy(z->dict + z->wp, z->dict + src, (size_t)length);
    z->wp += length;
  } else {
    const int64_t end = z->wp + length;
    int64_t s = src, d = z->wp;
    while (d < end) {
      if (s < 0 || d >= z->dlen) xz_throw(c);
      z->dict[d++] = z->dict[s++];
    }
    z->wp = end;
  }
}
static int64_t read_length(xz_ctx *c, lzma *z, lendec *L, int64_t pos_state) { /* :453-464 */
  if (read_bit(c, z, L->form, 2, 0) == 0) return 2 + bittree(c, z, L->shrt[pos_state], 8, 3);
  if (read_bit(c, z, L->form, 2, 1) == 0) return 10 + bittree(c, z, L->med[pos_state], 8, 3);
  return 18 + bittree(c, z, L->lng, 256, 8);
}
static int64_t read_distance(xz_ctx *c, lzma *z, int64_t length) { /* :515-549 */
  int64_t ds = length - 2;
  if (ds >= 4) ds = 3;
  const int64_t slot = bittree(c, z, z->slot[ds], 64, 6);
  if (slot < 4) return slot;
  const int64_t prefix = 2 | (slot & 1);
  const int bit_count = (int)(slot / 2) - 1;
  if (slot < 14) return (prefix << bit_count) | bittree_rev(c, z, z->dshort[slot - 4], (int64_t)1 << bit_count, bit_count);
  const int64_t direct = read_direct(c, z, bit_count - 4);
  const int64_t align = bittree_rev(c, z, z->dalign, 16, 4);
  return ((prefix << bit_count) & 0xffffffff) | ((direct << 4) & 0xffffffff) | align;
}
/* decode (:195-237): returns the bytes added, [initial, wp) -- a match may overshoot the declared size */
static void lz_decode(xz_ctx *c, lzma *z, view data, int64_t ulen, orc_oms *out) {
  z->buf = data.b;
  z->blen = data.len;
  z->bpos = 0;
  z->code = 0; /* initialize (:51-58): the first byte is skipped unchecked */
  z->range = 0xffffffff;
  z->bpos++;
  for (int i = 0; i < 4; ++i) z->code = (z->code << 8) | next_byte(c, z);
  const int64_t initial = z->wp, final_size = initial + ulen;
  lz_grow(z, final_size);
  const int64_t pmask = ((int64_t)1 << z->pb) - 1;
  while (z->wp < final_size) {
    const int64_t ps = z->wp & pmask;
    const int lit_prev = z->state < 7;
    if (read_bit(c, z, z->nonlit[z->state], 12, ps) == 0) { /* _decodeLiteral (:260-313) */
      const int prev = z->wp > 0 ? z->dict[z->wp - 1] : 0;
      const int64_t hash = (prev >> (8 - z->lc)) + ((z->wp & (((int64_t)1 << z->lp) - 1)) << z->lc);
      int v;
      if (lit_prev) {
        v = decode_byte(c, z, z->lit + hash * 256);
      } else {
        const int64_t mi = z->wp - z->d0 - 1;
        if (mi < 0) xz_throw(c);
        v = decode_matched_byte(c, z, z->lit + hash * 256, z->mlit0 + hash * 256, z->mlit1 + hash * 256, z->dict[mi]);
      }
      z->dict[z->wp++] = (uint8_t)v;
      static const int nxt[12] = {0, 0, 0, 0, 1, 2, 3, 4, 5, 6, 4, 5};
      z->state = nxt[z->state];
    } else if (read_bit(c, z, z->rep, 12, z->state) == 0) { /* _decodeMatch (:316-329) */
      const int64_t len = read_length(c, z, &z->mlen, ps);
      const int64_t dist = read_distance(c, z, len);
      repeat_data(c, z, dist, len);
      z->d3 = z->d2;
      z->d2 = z->d1;
      z->d1 = z->d0;
      z->d0 = dist;
      z->state = lit_prev ? 7 : 10;
    } else { /* _decodeRepeat (:332-367) */
      int64_t dist;
      if (read_bit(c, z, z->rep0, 12, z->state) == 0) {
        if (read_bit(c, z, z->longrep0[z->state], 12, ps) == 0) {
          repeat_data(c, z, z->d0, 1);
          z->state = lit_prev ? 9 : 11;
          continue;
        }
        dist = z->d0;
      } else if (read_bit(c, z, z->rep1, 12, z->state) == 0) {
        dist = z->d1;
        z->d1 = z->d0;
        z->d0 = dist;
      } else if (read_bit(c, z, z->rep2, 12, z->state) == 0) {
        dist = z->d2;
        z->d2 = z->d1;
        z->d1 = z->d0;
        z->d0 = dist;
      } else {
        dist = z->d3;
        z->d3 = z->d2;
        z->d2 = z->d1;
        z->d1 = z->d0;
        z->d0 = dist;
      }
      const int64_t len = read_length(c, z, &z->rlen, ps);
      repeat_data(c, z, dist, len);
      z->state = lit_prev ? 8 : 11;
    }
  }
  orc_oms_write_bytes(out, z->dict + initial, z->wp - initial);
}

/* ---- _XZStreamDecoder (xz_decoder.dart:30-458) ---- */
typedef struct {
  int64_t unpadded, uncompressed;
} block_size;

typedef struct {
  xz_ctx c;
  lzma z;
  int verify, flags;
  block_size *bs;
  int64_t nbs;
} xz_dec;

static int read_lzma2(xz_dec *x, view *in, orc_oms *out, int64_t dict_size) { /* :284-351 */
  xz_ctx *c = &x->c;
  lzma *z = &x->z;
  while (!eos(in)) {
    const int control = rb(c, in);
    if (!(control & 0x80)) {
      if (control == 0) {
        lz_reset(z, -1, -1, -1, 1);
        return 1;
      } else if (control == 1 || control == 2) {
        if (control == 1) lz_reset(z, -1, -1, -1, 1);
        const int hi = rb(c, in), lo = rb(c, in);
        const int64_t length = (hi << 8 | lo) + 1;
        view chunk = read_bytes(c, in, length);
        view d = lz_stored(c, z, &chunk, length);
        orc_oms_write_bytes(out, d.b, d.len);
        lz_trim(z, dict_size);
      } else {
        return 0;
      }
    } else {
      const int reset = (control >> 5) & 3;
      const int b1 = rb(c, in), b2 = rb(c, in);
      const int64_t ulen = ((control & 0x1f) << 16 | b1 << 8 | b2) + 1;
      const int c1 = rb(c, in), c2 = rb(c, in);
      const int64_t clen = (c1 << 8 | c2) + 1;
      int lc = -1, lp = -1, pb = -1;
      if (reset >= 2) {
        int props = rb(c, in);
        pb = props / 45;
        props -= pb * 45;
        lp = props / 9;
        lc = props - lp * 9;
      }
      if (reset > 0) lz_reset(z, pb, lp, lc, reset == 3);
      view data = read_bytes(c, in, clen);
      lz_decode(c, z, data, ulen, out);
      lz_trim(z, dict_size);
    }
  }
  return 0;
}

static int read_block(xz_dec *x, view *in, orc_oms *out, int64_t header_len) { /* :104-281 */
  xz_ctx *c = &x->c;
  const int64_t block_start = in->pos;
  view header = read_bytes(c, in, header_len - 4);
  skip(&header, 1);
  const int bflags = rb(c, &header);
  const int nfilters = (bflags & 3) + 1;
  int64_t comp_len = -1, uncomp_len = -1;
  int has_comp = (bflags & 0x40) != 0, has_uncomp = (bflags & 0x80) != 0;
  if (has_comp) comp_len = read_mbi(c, &header);
  if (has_uncomp) uncomp_len = read_mbi(c, &header);
  int nf = 0;
  int64_t first_id = -1;
  int64_t dict_size = 0;
  for (int i = 0; i < nfilters; ++i) {
    const int64_t id = read_mbi(c, &header);
    const int64_t plen = read_mbi(c, &header);
    view props = read_bytes(c, &header, plen);
    if (id == 0x03) {
      if (props.len < 1) xz_throw(c);
    } else if (id == 0x21) {
      if (props.len < 1) xz_throw(c);
      const int v = props.b[0];
      if (v > 40) return 0;
      dict_size = v == 40 ? 0xffffffffll : (int64_t)(2 | (v & 1)) << ((v >> 1) + 11);
    }
    if (nf == 0) first_id = id;
    nf++;
  }
  if (dict_size > 0 && dict_size < 0x40000000) x->z.cap = dict_size + (dict_size >> 2) + (2 << 20) + 16;
  if (read_padding(c, &header) < 0) return 0;
  const uint32_t crc = read_u32(c, in);
  if (orc_crc32(header.b, (size_t)header.len, 0) != crc) return 0;
  if (nf != 1 || first_id != 0x21) return 0;
  const int64_t start_pos = in->pos, start_out = out->len;
  if (!read_lzma2(x, in, out, dict_size)) return 0;
  const int64_t actual_comp = in->pos - start_pos, actual_uncomp = out->len - start_out;
  if (has_comp && comp_len != actual_comp) return 0;
  if (!has_uncomp) uncomp_len = actual_uncomp;
  if (uncomp_len != actual_uncomp) return 0;
  const int64_t padding = read_padding(c, in);
  if (padding < 0) return 0;
  switch (x->flags & 0xf) {
    case 0: break;
    case 1: {
      const uint32_t want = read_u32(c, in);
      if (x->verify && orc_crc32(out->buf + start_out, (size_t)actual_uncomp, 0) != want) return 0;
      break;
    }
    case 2: case 3: skip(in, 4); break;
    case 4: {
      const uint64_t want = read_u64(c, in);
      if (x->verify && orc_crc64(out->buf + start_out, (size_t)actual_uncomp, 0) != want) return 0;
      break;
    }
    case 5: case 6: skip(in, 8); break;
    case 7: case 8: case 9: skip(in, 16); break;
    case 0xa: read_bytes(c, in, 32); break; /* read, never compared */
    case 0xb: case 0xc: skip(in, 32); break;
    default: skip(in, 64); break;
  }
  x->bs = realloc(x->bs, (size_t)(x->nbs + 1) * sizeof(block_size));
  x->bs[x->nbs].unpadded = in->pos - block_start - padding;
  x->bs[x->nbs].uncompressed = uncomp_len;
  x->nbs++;
  return 1;
}

static int64_t read_index(xz_dec *x, view *in) { /* :355-392 */
  xz_ctx *c = &x->c;
  const int64_t start = in->pos;
  skip(in, 1);
  const int64_t n = read_mbi(c, in);
  if (n != x->nbs) return -1;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t unpadded = read_mbi(c, in), uncomp = read_mbi(c, in);
    if (x->bs[i].unpadded != unpadded) return -1;
    if (x->bs[i].uncompressed != uncomp) return -1;
  }
  if (read_padding(c, in) < 0) return -1;
  const int64_t ilen = in->pos - start;
  skip(in, -ilen);
  view idx = read_bytes(c, in, ilen);
  const uint32_t crc = read_u32(c, in);
  if (orc_crc32(idx.b, (size_t)idx.len, 0) != crc) return -1;
  return ilen + 4;
}

static int read_footer(xz_dec *x, view *in, int64_t index_size) { /* :396-428 */
  xz_ctx *c = &x->c;
  const uint32_t crc = read_u32(c, in);
  view f = read_bytes(c, in, 6);
  const int64_t backward = ((int64_t)read_u32(c, &f) + 1) * 4;
  if (backward != index_size) return 0;
  if (rb(c, &f) != 0) return 0;
  if (rb(c, &f) != x->flags) return 0;
  if (orc_crc32(f.b, (size_t)f.len, 0) != crc) return 0;
  view m = read_bytes(c, in, 2);
  if (m.len < 1) xz_throw(c);
  if (m.b[0] != 89) return 0;
  if (m.len < 2) xz_throw(c);
  return m.b[1] == 90;
}

static int xz_decode_stream(xz_dec *x, view *in, orc_oms *out) { /* :46-101 */
  xz_ctx *c = &x->c;
  view magic = read_bytes(c, in, 6);
  static const uint8_t mg[6] = {253, 55, 122, 88, 90, 0};
  for (int i = 0; i < 6; ++i) { /* `&&` stops at the first mismatch; a short list throws where it is indexed */
    if (i >= magic.len) xz_throw(c);
    if (magic.b[i] != mg[i]) return 0;
  }
  view h = read_bytes(c, in, 2);
  if (rb(c, &h) != 0) return 0;
  x->flags = rb(c, &h);
  const uint32_t crc = read_u32(c, in);
  if (orc_crc32(h.b, (size_t)h.len, 0) != crc) return 0;
  while (!eos(in)) {
    const int bh = in->b[in->pos];
    if (bh == 0) {
      const int64_t isz = read_index(x, in);
      if (isz < 0) return 0;
      return read_footer(x, in, isz);
    }
    if (!read_block(x, in, out, ((int64_t)bh + 1) * 4)) return 0;
  }
  return 0;
}

int orc_xz_decode(const uint8_t *in, size_t n, int verify, uint8_t **out, size_t *out_len) {
  xz_dec *x = calloc(1, sizeof *x);
  x->verify = verify;
  x->z.pb = 2; /* LzmaDecoder() (:17-24, :67-85) */
  x->z.lp = 0;
  x->z.lc = 3;
  lz_reset(&x->z, -1, -1, -1, 1);
  orc_oms o;
  orc_oms_init(&o, 1 << 16);
  view v = {in, (int64_t)n, 0};
  int st;
  if (setjmp(x->c.jb) == 0) st = xz_decode_stream(x, &v, &o) ? ORC_OK : ORC_FALSE;
  else st = ORC_THROW;
  *out = malloc(o.len ? (size_t)o.len : 1);
  memcpy(*out, o.buf, (size_t)o.len);
  *out_len = (size_t)o.len;
  orc_oms_free(&o);
  free(x->z.lit);
  free(x->z.mlit0);
  free(x->z.mlit1);
  free(x->z.dict);
  free(x->bs);
  free(x);
  return st;
}

/* ---- SHA-256 (FIPS 180-4; what PcSHA256Digest computes) ---- */
static const uint32_t K256[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01,
    0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc,
    0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147,
    0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08,
    0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208,
    0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
#define ROR(x, n) (((x) >> (n)) | ((x) << (32 - (n))))
static void sha256_block(uint32_t h[8], const uint8_t *p) {
  uint32_t w[64];
  for (int i = 0; i < 16; ++i) w[i] = (uint32_t)p[4 * i] << 24 | p[4 * i + 1] << 16 | p[4 * i + 2] << 8 | p[4 * i + 3];
  for (int i = 16; i < 64; ++i) {
    uint32_t s0 = ROR(w[i - 15], 7) ^ ROR(w[i - 15], 18) ^ (w[i - 15] >> 3);
    uint32_t s1 = ROR(w[i - 2], 17) ^ ROR(w[i - 2], 19) ^ (w[i - 2] >> 10);
    w[i] = w[i - 16] + s0 + w[i - 7] + s1;
  }
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
  for (int i = 0; i < 64; ++i) {
    uint32_t t1 = hh + (ROR(e, 6) ^ ROR(e, 11) ^ ROR(e, 25)) + ((e & f) ^ (~e & g)) + K256[i] + w[i];
    uint32_t t2 = (ROR(a, 2) ^ ROR(a, 13) ^ ROR(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
    hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}
void orc_sha256(const uint8_t *p, size_t n, uint8_t digest[32]) {
  uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
  size_t i = 0;
  for (; i + 64 <= n; i += 64) sha256_block(h, p + i);
  uint8_t last[128] = {0};
  const size_t r = n - i;
  memcpy(last, p + i, r);
  last[r] = 0x80;
  const size_t tot = r + 9 <= 64 ? 64 : 128;
  const uint64_t bits = (uint64_t)n * 8;
  for (int k = 0; k < 8; ++k) last[tot - 1 - k] = (uint8_t)(bits >> (8 * k));
  sha256_block(h, last);
  if (tot == 128) sha256_block(h, last + 64);
  for (int k = 0; k < 8; ++k)
    for (int j = 0; j < 4; ++j) digest[4 * k + j] = (uint8_t)(h[k] >> (24 - 8 * j));
}

/* ---- XZEncoder (xz_encoder.dart) ---- */
/* one byte through writeBytes: orc_oms_write_byte carries the inflate oracle's runaway guard, which a large input trips */
static void put1(orc_oms *o, int v) {
  const uint8_t b = (uint8_t)v;
  orc_oms_write_bytes(o, &b, 1);
}
static void w_u32(orc_oms *o, uint32_t v) {
  for (int i = 0; i < 4; ++i) put1(o, (v >> (8 * i)) & 0xff);
}
static void w_mbi(orc_oms *o, int64_t value) { /* _writeMultibyteInteger (:229-239) */
  int shift = 0;
  while ((value >> (shift + 7)) != 0) shift += 7;
  while (shift > 0) {
    put1(o, 0x80 | ((value >> shift) & 0x7f));
    shift -= 7;
  }
  put1(o, value & 0x7f);
}
static int64_t w_pad(orc_oms *o) {
  int64_t n = 0;
  while (o->len % 4 != 0) {
    put1(o, 0);
    n++;
  }
  return n;
}
int orc_xz_encode(const uint8_t *in, size_t n, int check, uint8_t **out, size_t *out_len) {
  static const int FL[4] = {0, 1, 4, 0xa}; /* encodeStream (:30-62) */
  if (check < 0 || check > 3) return ORC_THROW;
  const int flags = FL[check];
  orc_oms o;
  orc_oms_init(&o, (int64_t)n + 128);
  static const uint8_t magic[6] = {253, 55, 122, 88, 90, 0}; /* _writeStreamHeader (:64-74) */
  orc_oms_write_bytes(&o, magic, 6);
  const uint8_t sh[2] = {0, (uint8_t)flags};
  orc_oms_write_bytes(&o, sh, 2);
  w_u32(&o, orc_crc32(sh, 2, 0));
  int64_t unpadded = 0;
  if (n > 0) { /* _writeBlock (:76-162): header 02 00 21 01 16 + padding, one stored chunk (control 1), end marker */
    const uint8_t bh[8] = {2, 0, 0x21, 1, 0x16, 0, 0, 0};
    const int64_t block_start = o.len;
    orc_oms_write_bytes(&o, bh, 8);
    w_u32(&o, orc_crc32(bh, 8, 0));
    put1(&o, 1);
    put1(&o, (int)(((n - 1) >> 8) & 0xff)); /* a 16-bit field: inputs over 64 KiB are cut (:181-182) */
    put1(&o, (int)((n - 1) & 0xff));
    orc_oms_write_bytes(&o, in, (int64_t)n);
    put1(&o, 0);
    const int64_t pad = w_pad(&o);
    if (flags == 1) {
      w_u32(&o, orc_crc32(in, n, 0));
    } else if (flags == 4) {
      const uint64_t c = orc_crc64(in, n, 0);
      w_u32(&o, (uint32_t)c);
      w_u32(&o, (uint32_t)(c >> 32));
    } else if (flags == 0xa) {
      uint8_t d[32];
      orc_sha256(in, n, d);
      orc_oms_write_bytes(&o, d, 32);
    }
    unpadded = o.len - block_start - pad;
  }
  orc_oms idx; /* _writeStreamIndex (:198-211) */
  orc_oms_init(&idx, 64);
  put1(&idx, 0);
  w_mbi(&idx, n > 0 ? 1 : 0);
  if (n > 0) {
    w_mbi(&idx, unpadded);
    w_mbi(&idx, (int64_t)n);
  }
  w_pad(&idx);
  const int64_t index_start = o.len;
  orc_oms_write_bytes(&o, idx.buf, idx.len);
  w_u32(&o, orc_crc32(idx.buf, (size_t)idx.len, 0));
  const int64_t index_size = o.len - index_start;
  orc_oms_free(&idx);
  uint8_t f[6]; /* _writeStreamFooter (:213-225) */
  const uint32_t bw = (uint32_t)(index_size / 4 - 1);
  for (int i = 0; i < 4; ++i) f[i] = (uint8_t)(bw >> (8 * i));
  f[4] = 0;
  f[5] = (uint8_t)flags;
  w_u32(&o, orc_crc32(f, 6, 0));
  orc_oms_write_bytes(&o, f, 6);
  put1(&o, 89);
  put1(&o, 90);
  *out = malloc(o.len ? (size_t)o.len : 1);
  memcpy(*out, o.buf, (size_t)o.len);
  *out_len = (size_t)o.len;
  orc_oms_free(&o);
  return ORC_OK;
}
