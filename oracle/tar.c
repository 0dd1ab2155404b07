/*
 * oracle/tar.c -- CPU ORACLE (test infrastructure only; see orc.h).
 *
 * Restates the TAR container of the reference:
 *   TarFile.read   lib/src/codecs/tar/tar_file.dart:74-118 (_parseInt :211-225, _parseString :227-239)
 *   TarFile.write  lib/src/codecs/tar/tar_file.dart:144-209 (_writeString :241-248, _writeInt :250-256)
 *   TarDecoder.decodeStream  lib/src/codecs/tar_decoder.dart:24-128 over an InputMemoryStream
 *     (readBytes / subset / skip: lib/src/util/input_stream.dart:132-136, input_memory_stream.dart:15-28, 96-119;
 *      readString: input_stream.dart:140-164)
 *   TarEncoder.add / finish  lib/src/codecs/tar_encoder.dart:39-88
 * Dart strings are handled as code points: a field decodes as strict UTF-8 or, failing that, one code point per byte,
 * and is trimmed with String.trim()'s set; every string handed back is UTF-8.
 */
#include <stdlib.h>
#include <string.h>

#include "orc.h"

/* One TarFile of TarDecoder.files, with what TarDecoder made of it.  Strings are (offset, length) into the string block. */
typedef struct {
  int64_t mode, uid, gid, size, mtime, checksum, devmajor, devminor;
  uint64_t name_off, name_len, link_off, link_len, type_off, type_len;
  uint64_t magic_off, magic_len, uname_off, uname_len, gname_off, gname_len;
  int64_t content_off, content_len; /* range of the input read as content; content_len -1: none was read */
  int32_t is_file;                  /* typeFlag != '5' */
  int32_t archive_index;            /* the Archive slot it holds at the end; -1 when a later member of its name took it */
} orc_tar_member;

/* One ArchiveFile handed to TarEncoder.add. */
typedef struct {
  const char *name;        /* UTF-8, zero terminated */
  const char *symlink;     /* NULL when symbolicLink is null */
  const uint8_t *content;  /* what getContent() gives; NULL when it gives null */
  size_t content_len;
  int64_t size, mode, uid, gid, mtime;
  int is_file;
} orc_tar_entry_in;

/* ---- strings ---------------------------------------------------------------------------------------------------- */

/* Strict UTF-8 (what utf8.decode accepts): no overlongs, no surrogates, nothing above U+10FFFF.  Returns the number of
 * code points written to cp, or -1. */
static int64_t utf8_decode(const uint8_t *p, int64_t n, uint32_t *cp) {
  int64_t i = 0, k = 0;
  while (i < n) {
    uint32_t c = p[i];
    int more;
    uint8_t lo = 0x80, hi = 0xbf;
    if (c < 0x80) { cp[k++] = c; i++; continue; }
    if (c >= 0xc2 && c <= 0xdf) { more = 1; c &= 0x1f; }
    else if (c >= 0xe0 && c <= 0xef) { more = 2; c &= 0x0f; if (p[i] == 0xe0) lo = 0xa0; if (p[i] == 0xed) hi = 0x9f; }
    else if (c >= 0xf0 && c <= 0xf4) { more = 3; c &= 0x07; if (p[i] == 0xf0) lo = 0x90; if (p[i] == 0xf4) hi = 0x8f; }
    else return -1;
    if (i + more >= n) return -1;
    for (int j = 1; j <= more; ++j) {
      uint8_t b = p[i + j];
      if (j == 1 ? (b < lo || b > hi) : (b < 0x80 || b > 0xbf)) return -1;
      c = (c << 6) | (b & 0x3f);
    }
    cp[k++] = c;
    i += more + 1;
  }
  return k;
}

/* utf8.decode with the fallback to String.fromCharCodes (tar_file.dart:231-237, input_stream.dart:141-149). */
static int64_t dart_decode(const uint8_t *p, int64_t n, uint32_t *cp) {
  int64_t k = utf8_decode(p, n, cp);
  if (k >= 0) return k;
  for (int64_t i = 0; i < n; ++i) cp[i] = p[i];
  return n;
}

/* String.trim()'s whitespace: Unicode White_Space and U+FEFF. */
static int dart_ws(uint32_t c) {
  return (c >= 0x09 && c <= 0x0d) || c == 0x20 || c == 0x85 || c == 0xa0 || c == 0x1680 || (c >= 0x2000 && c <= 0x200a) ||
         c == 0x2028 || c == 0x2029 || c == 0x202f || c == 0x205f || c == 0x3000 || c == 0xfeff;
}

static void put_utf8(orc_oms *o, uint32_t c) {
  if (c < 0x80) {
    orc_oms_write_byte(o, c);
  } else if (c < 0x800) {
    orc_oms_write_byte(o, 0xc0 | (c >> 6));
    orc_oms_write_byte(o, 0x80 | (c & 0x3f));
  } else if (c < 0x10000) {
    orc_oms_write_byte(o, 0xe0 | (c >> 12));
    orc_oms_write_byte(o, 0x80 | ((c >> 6) & 0x3f));
    orc_oms_write_byte(o, 0x80 | (c & 0x3f));
  } else {
    orc_oms_write_byte(o, 0xf0 | (c >> 18));
    orc_oms_write_byte(o, 0x80 | ((c >> 12) & 0x3f));
    orc_oms_write_byte(o, 0x80 | ((c >> 6) & 0x3f));
    orc_oms_write_byte(o, 0x80 | (c & 0x3f));
  }
}

typedef struct {
  uint64_t off, len;
} str_ref;

/* Decode p[0, n) (optionally trimmed) into the string block. */
static str_ref put_string(orc_oms *strs, const uint8_t *p, int64_t n, int trim) {
  uint32_t *cp = (uint32_t *)malloc(sizeof(uint32_t) * (n ? n : 1));
  int64_t k = dart_decode(p, n, cp), a = 0, b = k;
  if (trim) {
    while (a < b && dart_ws(cp[a])) a++;
    while (b > a && dart_ws(cp[b - 1])) b--;
  }
  str_ref r = {(uint64_t)strs->len, 0};
  for (int64_t i = a; i < b; ++i) put_utf8(strs, cp[i]);
  r.len = (uint64_t)strs->len - r.off;
  free(cp);
  return r;
}

/* _parseString (tar_file.dart:227-239) of header field [off, off + width), the header being hl bytes long (a short read
 * leaves later fields short or empty, as readBytes clips them). */
static str_ref parse_string(orc_oms *strs, const uint8_t *h, int64_t hl, int64_t off, int64_t width) {
  int64_t n = off >= hl ? 0 : (off + width > hl ? hl - off : width);
  const uint8_t *p = h + (off < hl ? off : hl);
  const uint8_t *z = (const uint8_t *)memchr(p, 0, (size_t)n);
  return put_string(strs, p, z ? z - p : n, 1);
}

static int str_eq(const orc_oms *strs, str_ref r, const char *s) {
  size_t n = strlen(s);
  return r.len == n && memcmp(strs->buf + r.off, s, n) == 0;
}

/* _parseInt (tar_file.dart:211-225): int.parse(s, radix: 8) -- an optional sign, then ASCII octal digits -- or 0. */
static int64_t parse_int(orc_oms *strs, const uint8_t *h, int64_t hl, int64_t off, int64_t width) {
  str_ref r = parse_string(strs, h, hl, off, width);
  const uint8_t *s = strs->buf + r.off;
  uint64_t i = 0, neg = 0;
  int64_t v = 0;
  if (i < r.len && (s[i] == '+' || s[i] == '-')) neg = s[i++] == '-';
  if (i == r.len) return 0;
  for (; i < r.len; ++i) {
    if (s[i] < '0' || s[i] > '7') return 0;
    v = v * 8 + (s[i] - '0');
  }
  return neg ? -v : v;
}

/* ---- decoder ---------------------------------------------------------------------------------------------------- */

static int64_t clamp(int64_t v, int64_t lo, int64_t hi) { return v < lo ? lo : v > hi ? hi : v; }

/* TarDecoder().decodeBytes(in, storeData:) -> status (ORC_OK / ORC_THROW), the TarFiles of decoder.files (at most cap are
 * written; *n_out is how many there are) and the string block (*strings, malloc'ed). */
int orc_tar_decode(const uint8_t *in, size_t n, int store_data, orc_tar_member *out, size_t cap, size_t *n_out,
                   uint8_t **strings, size_t *strings_len) {
  orc_oms strs;
  orc_oms_init(&strs, 4096);
  orc_oms_write_byte(&strs, 0); /* keeps the block non-empty */
  int64_t len = (int64_t)n, pos = 0;
  int rc = ORC_OK;
  size_t count = 0, nslots = 0, slot_cap = 64;
  size_t *slots = (size_t *)malloc(sizeof(size_t) * slot_cap);
  orc_tar_member *all = NULL;
  size_t all_cap = 0;
  int has_next_name = 0, has_next_link = 0;
  str_ref next_name = {0, 0}, next_link = {0, 0};
  while (pos < len) { /* !input.isEOS */
    if (len - pos < 2 || (in[pos] == 0 && in[pos + 1] == 0)) break; /* peekBytes(2) (:35-38) */
    /* TarFile.read (tar_file.dart:74-118) */
    orc_tar_member m;
    memset(&m, 0, sizeof m);
    int64_t hl = len - pos < 512 ? len - pos : 512;
    const uint8_t *h = in + pos;
    pos += hl;
    str_ref name = parse_string(&strs, h, hl, 0, 100);
    m.mode = parse_int(&strs, h, hl, 100, 8);
    m.uid = parse_int(&strs, h, hl, 108, 8);
    m.gid = parse_int(&strs, h, hl, 116, 8);
    m.size = parse_int(&strs, h, hl, 124, 12);
    m.mtime = parse_int(&strs, h, hl, 136, 12);
    m.checksum = parse_int(&strs, h, hl, 148, 8);
    str_ref type = parse_string(&strs, h, hl, 156, 1);
    str_ref link = parse_string(&strs, h, hl, 157, 100);
    str_ref magic = parse_string(&strs, h, hl, 257, 6), uname = {0, 0}, gname = {0, 0};
    if (str_eq(&strs, magic, "ustar")) {
      parse_string(&strs, h, hl, 263, 2);
      uname = parse_string(&strs, h, hl, 265, 32);
      gname = parse_string(&strs, h, hl, 297, 32);
      m.devmajor = parse_int(&strs, h, hl, 329, 8);
      m.devminor = parse_int(&strs, h, hl, 337, 8);
      str_ref prefix = parse_string(&strs, h, hl, 345, 155);
      if (prefix.len) { /* '$filenamePrefix/$filename' */
        uint8_t *j = (uint8_t *)malloc(prefix.len + 1 + name.len);
        memcpy(j, strs.buf + prefix.off, prefix.len);
        j[prefix.len] = '/';
        memcpy(j + prefix.len + 1, strs.buf + name.off, name.len);
        name.off = (uint64_t)strs.len;
        name.len = prefix.len + 1 + name.len;
        orc_oms_write_bytes(&strs, j, (int64_t)name.len);
        free(j);
      }
    }
    int is_long_link = str_eq(&strs, name, "././@LongLink");
    m.content_len = -1;
    if (store_data || is_long_link) {
      if (m.size < 0) { rc = ORC_THROW; break; } /* a negative Uint8List.view length: RangeError */
      m.content_off = pos;
      m.content_len = m.size < len - pos ? m.size : len - pos;
      pos += m.content_len;
    } else {
      pos = clamp(pos + m.size, 0, len);
    }
    m.is_file = !str_eq(&strs, type, "5");
    if (m.is_file && m.size > 0 && m.size % 512) pos = clamp(pos + 512 - m.size % 512, 0, len);

    /* TarDecoder.decodeStream (tar_decoder.dart:43-124) */
    if (is_long_link) { /* readString(): to the first NUL, no trim */
      const uint8_t *c = in + m.content_off;
      const uint8_t *z = (const uint8_t *)memchr(c, 0, (size_t)m.content_len);
      next_name = put_string(&strs, c, z ? z - c : m.content_len, 0);
      has_next_name = 1;
      continue;
    }
    if (str_eq(&strs, type, "g") || str_eq(&strs, type, "G")) continue;
    if (str_eq(&strs, type, "x") || str_eq(&strs, type, "X")) {
      if (m.content_len < 0) { rc = ORC_THROW; break; } /* rawContent! with storeData false */
      const uint8_t *c = in + m.content_off;
      int64_t cl = m.content_len;
      uint32_t *tmp = (uint32_t *)malloc(sizeof(uint32_t) * (cl ? cl : 1));
      int64_t ok = utf8_decode(c, cl, tmp);
      free(tmp);
      if (ok < 0) { rc = ORC_THROW; break; } /* utf8.decode: FormatException */
      for (int64_t a = 0; a <= cl;) { /* split('\n') */
        const uint8_t *nl = (const uint8_t *)memchr(c + a, '\n', (size_t)(cl - a));
        int64_t b = nl ? nl - c : cl;
        /* firstMatch of (\d+) (\w+)=(.*): the leftmost digit run followed by ' ', a word run and '='.  Neither greedy run
         * can give back a character that would let the next one match, so the first start that matches is found by
         * scanning maximal runs; `.` stops at \r, U+2028 and U+2029. */
        for (int64_t i = a; i < b; ++i) {
          if (c[i] < '0' || c[i] > '9') continue;
          int64_t j = i;
          while (j < b && c[j] >= '0' && c[j] <= '9') j++;
          if (j >= b || c[j] != ' ') continue;
          int64_t k0 = j + 1, k = k0;
          while (k < b && ((c[k] >= '0' && c[k] <= '9') || (c[k] >= 'a' && c[k] <= 'z') || (c[k] >= 'A' && c[k] <= 'Z') || c[k] == '_'))
            k++;
          if (k == k0 || k >= b || c[k] != '=') continue;
          int64_t v0 = k + 1, v = v0;
          while (v < b && c[v] != '\r' && !(v + 2 < b && c[v] == 0xe2 && c[v + 1] == 0x80 && (c[v + 2] == 0xa8 || c[v + 2] == 0xa9)))
            v++;
          if (k - k0 == 4 && memcmp(c + k0, "path", 4) == 0) {
            next_name = put_string(&strs, c + v0, v - v0, 0);
            has_next_name = 1;
          } else if (k - k0 == 8 && memcmp(c + k0, "linkpath", 8) == 0) {
            next_link = put_string(&strs, c + v0, v - v0, 0);
            has_next_link = 1;
          }
          break;
        }
        a = b + 1;
      }
      continue;
    }
    if (has_next_name) name = next_name, has_next_name = 0;
    if (has_next_link) link = next_link, has_next_link = 0;
    m.name_off = name.off, m.name_len = name.len, m.link_off = link.off, m.link_len = link.len;
    m.type_off = type.off, m.type_len = type.len, m.magic_off = magic.off, m.magic_len = magic.len;
    m.uname_off = uname.off, m.uname_len = uname.len, m.gname_off = gname.off, m.gname_len = gname.len;
    m.archive_index = -1;
    if (count == all_cap) {
      all_cap = all_cap ? 2 * all_cap : 64;
      all = (orc_tar_member *)realloc(all, sizeof(orc_tar_member) * all_cap);
    }
    all[count] = m;
    /* Archive.add (archive.dart:19-31): a name already present keeps its slot and takes the new entry */
    size_t s = 0;
    for (; s < nslots; ++s) {
      const orc_tar_member *o = &all[slots[s]];
      if (o->name_len == name.len && memcmp(strs.buf + o->name_off, strs.buf + name.off, name.len) == 0) break;
    }
    if (s == nslots) {
      if (nslots == slot_cap) slots = (size_t *)realloc(slots, sizeof(size_t) * (slot_cap *= 2));
      nslots++;
    }
    slots[s] = count++;
  }
  for (size_t s = 0; s < nslots; ++s) all[slots[s]].archive_index = (int32_t)s;
  for (size_t i = 0; i < count && i < cap; ++i) out[i] = all[i];
  *n_out = count;
  *strings = strs.buf;
  *strings_len = (size_t)strs.len;
  free(all);
  free(slots);
  return rc;
}

/* ---- encoder ---------------------------------------------------------------------------------------------------- */

/* _writeString (tar_file.dart:241-248) */
static void write_string(orc_oms *o, const uint8_t *s, size_t n, size_t width) {
  for (size_t i = 0; i < width; ++i) orc_oms_write_byte(o, i < n ? s[i] : 0);
}

/* _writeInt (tar_file.dart:250-256): toRadixString(8), '0's in front to width-1 characters, cut to the field. */
static void write_int(orc_oms *o, int64_t v, size_t width) {
  char digits[32], s[48];
  int nd = 0;
  uint64_t u = v < 0 ? (uint64_t)(-(v + 1)) + 1 : (uint64_t)v;
  do { digits[nd++] = (char)('0' + (u & 7)); u >>= 3; } while (u);
  size_t k = 0;
  if (v < 0) s[k++] = '-';
  while (nd) s[k++] = digits[--nd];
  size_t pad = k < width - 1 ? width - 1 - k : 0;
  char t[64];
  memset(t, '0', pad);
  memcpy(t + pad, s, k);
  write_string(o, (const uint8_t *)t, pad + k, width);
}

typedef struct {
  const uint8_t *name;
  size_t name_len;
  int64_t mode, uid, gid, size, mtime;
  char type;
  const uint8_t *link;
  size_t link_len;
  const uint8_t *content; /* NULL: no content */
  size_t content_len;
} tar_header;

/* TarFile.write (tar_file.dart:144-209) */
static void tar_write(orc_oms *o, const tar_header *t) {
  int64_t start = o->len;
  write_string(o, t->name, t->name_len, 100);
  write_int(o, t->mode, 8);
  write_int(o, t->uid, 8);
  write_int(o, t->gid, 8);
  write_int(o, t->size, 12);
  write_int(o, t->mtime, 12);
  write_string(o, (const uint8_t *)"        ", 8, 8);
  write_string(o, (const uint8_t *)&t->type, 1, 1);
  write_string(o, t->link, t->link_len, 100);
  while (o->len - start < 512) orc_oms_write_byte(o, 0);
  uint32_t sum = 0;
  for (int i = 0; i < 512; ++i) sum += o->buf[start + i];
  char cs[16];
  int nd = 0;
  do { cs[nd++] = (char)('0' + (sum & 7)); sum >>= 3; } while (sum);
  while (nd < 6) cs[nd++] = '0';
  for (int i = 0; i < 6; ++i) o->buf[start + 148 + i] = (uint8_t)cs[nd - 1 - i];
  o->buf[start + 154] = 0;
  o->buf[start + 155] = 32;
  if (t->content) orc_oms_write_bytes(o, t->content, (int64_t)t->content_len);
  if (t->type != '5' && t->size > 0 && t->size % 512)
    for (int64_t i = 0; i < 512 - t->size % 512; ++i) orc_oms_write_byte(o, 0);
}

/* UTF-16 code units of a UTF-8 string (Dart's String.length). */
static int64_t utf16_units(const uint8_t *s, size_t n) {
  int64_t u = 0;
  for (size_t i = 0; i < n; ++i) {
    if ((s[i] & 0xc0) != 0x80) u++;
    if (s[i] >= 0xf0) u++;
  }
  return u;
}

/* TarEncoder().encodeBytes over the entries, in order (tar_encoder.dart:17-88). */
int orc_tar_encode(const orc_tar_entry_in *e, size_t n, uint8_t **out, size_t *out_len) {
  orc_oms o;
  orc_oms_init(&o, 0x8000);
  for (size_t i = 0; i < n; ++i) {
    const uint8_t *name = (const uint8_t *)e[i].name;
    size_t nl = strlen(e[i].name);
    int64_t units = utf16_units(name, nl);
    if (units > 100) { /* ././@LongLink: size is the UTF-16 length, content the UTF-8 bytes, type '0' */
      tar_header l = {(const uint8_t *)"././@LongLink", 13, 0, 0, 0, units, 0, '0', (const uint8_t *)"", 0, name, nl};
      tar_write(&o, &l);
    }
    tar_header t = {name, nl, e[i].mode, e[i].uid, e[i].gid, 0, e[i].mtime, '0', (const uint8_t *)"", 0, NULL, 0};
    if (!e[i].is_file) {
      t.type = '5';
    } else if (e[i].symlink) {
      t.type = '2';
      t.link = (const uint8_t *)e[i].symlink;
      t.link_len = strlen(e[i].symlink);
    } else {
      t.size = e[i].size;
      t.content = e[i].content;
      t.content_len = e[i].content_len;
    }
    tar_write(&o, &t);
  }
  for (int i = 0; i < 1024; ++i) orc_oms_write_byte(&o, 0);
  *out = o.buf;
  *out_len = (size_t)o.len;
  return ORC_OK;
}
