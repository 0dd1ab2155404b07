// b200z_file.cu -- file streams either side of the codecs (SURVEY.md 8f4).
//
// In the reference an InputFileStream feeds a codec through a FileBuffer cache (input_file_stream.dart:11,
// file_buffer.dart:10 -- 1 KiB by default, :21) one readByte() at a time, and OutputFileStream collects the result in a
// 1 MiB buffer (output_file_stream.dart:11,22).  Here the file meets the device in segments: page-locked segment buffers
// that live as long as the library does, filled and drained by a few threads with large pread()/pwrite() calls, so that
// reading segment k+1, decoding segment k (host->device copy, kernels and device->host copy already overlap inside the
// codec call) and writing segment k-1 run at the same time.
//
// GZip streams whose members carry size hints (the BGZF 'BC' subfield + ISIZE) are cut into segments at member boundaries;
// the member loop of _gzip_decoder_web.dart:27-58 does not carry state from one member to the next, so the bytes are those
// of one call over the whole file.  Everything else (members without hints, zlib, BZip2, the encoders: one stream whose
// blocks depend on each other or whose cuts depend on the data) is one segment.
//
// Pure host code: no kernel lives here; the codecs are called through the same entry points a caller with memory buffers
// uses (include/b200z.h), and there is no CPU fallback behind them.
#include <errno.h>
#include <fcntl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <mutex>
#include <thread>
#include <vector>

#include "b200z_internal.h"

namespace b200z {
namespace {

struct PinnedSlot {
  uint8_t *p = nullptr;
  size_t cap = 0;
  bool reserve(size_t n) {
    if (n <= cap) return true;
    b200z_host_free(p);
    p = nullptr;
    cap = 0;
    const size_t want = ((n + (n >> 3)) | ((2u << 20) - 1)) + 1;  // 12% slack, whole 2 MiB pages
    p = (uint8_t *)b200z_host_alloc(want);
    if (!p) return false;
    cap = want;
    return true;
  }
  void release() {
    b200z_host_free(p);
    p = nullptr;
    cap = 0;
  }
};

struct FileCtx {
  std::mutex mu;  // one file call at a time per process (the device is serialised behind it anyway)
  PinnedSlot in[2], out[2];
  uint32_t n_segments = 0, n_whole = 0;  // of the last call (b200z_file_last_stats)
};
FileCtx F;

void errf(const char *fmt, const char *path, int err) {
  char buf[400];
  snprintf(buf, sizeof buf, fmt, path ? path : "", strerror(err));
  set_error_text(buf);
}

size_t env_size(const char *name, size_t dflt, size_t lo, size_t hi) {
  const char *v = getenv(name);
  if (!v || !*v) return dflt;
  const unsigned long long x = strtoull(v, nullptr, 10);
  return x < lo ? lo : (x > hi ? hi : (size_t)x);
}

bool rw_full(bool write, int fd, uint8_t *buf, size_t n, uint64_t off) {
  while (n) {
    const ssize_t k = write ? pwrite(fd, buf, n, (off_t)off) : pread(fd, buf, n, (off_t)off);
    if (k < 0 && errno == EINTR) continue;
    if (k <= 0) return false;  // a short file counts as an error: the length came from fstat
    buf += k;
    n -= (size_t)k;
    off += (uint64_t)k;
  }
  return true;
}

// n bytes between a file and a (pinned) buffer, in 8 MiB slices handed out to a few threads
bool par_io(bool write, int fd, uint8_t *buf, size_t n, uint64_t off) {
  const size_t slice = 8u << 20;
  const size_t want = env_size("B200Z_FILE_THREADS", 8, 1, 64);
  const size_t nthreads = std::min(want, (n + slice - 1) / slice);
  if (nthreads <= 1) return n == 0 || rw_full(write, fd, buf, n, off);
  std::atomic<size_t> next{0};
  std::atomic<bool> ok{true};
  auto work = [&]() {
    for (;;) {
      const size_t i = next.fetch_add(slice);
      if (i >= n || !ok.load()) return;
      if (!rw_full(write, fd, buf + i, std::min(slice, n - i), off + i)) ok.store(false);
    }
  };
  std::vector<std::thread> th;
  for (size_t t = 1; t < nthreads; ++t) th.emplace_back(work);
  work();
  for (auto &t : th) t.join();
  return ok.load();
}

// an IO request running on its own thread (one read-ahead and one write-behind are in flight at most)
struct AsyncIo {
  std::thread th;
  bool ok = true;
  void start(bool write, int fd, uint8_t *buf, size_t n, uint64_t off) {
    ok = true;
    th = std::thread([=]() { ok = par_io(write, fd, buf, n, off); });
  }
  bool wait() {
    if (th.joinable()) th.join();
    return ok;
  }
  ~AsyncIo() { wait(); }
};

struct Args {
  int op;
  int32_t a0, a1;
  uint32_t a2;
};

// DEFLATE cannot expand by more than 1032:1 (a 258-byte match costs at least two bits): ISIZE fields that promise more are
// lying, and are not allowed to size a page-locked buffer
const size_t kMaxExpansion = 1040;

size_t first_cap(const Args &a, const uint8_t *in, size_t n) {
  switch (a.op) {
    case B200Z_FILE_GZIP_DECODE: {
      const size_t b = b200z_gzip_bound(in, n);
      return b && b <= kMaxExpansion * n + 1024 ? b + 64 : 4 * n + 4096;  // size fields that cannot be true are no bound
    }
    case B200Z_FILE_ZLIB_DECODE: return 4 * n + 4096;
    case B200Z_FILE_BZIP2_DECODE: return 6 * n + (1u << 20);
    case B200Z_FILE_ZLIB_ENCODE:
    case B200Z_FILE_GZIP_ENCODE: return b200z_deflate_bound(n);
    case B200Z_FILE_BZIP2_ENCODE: return b200z_bzip2_bound(n);
    case B200Z_FILE_XZ_DECODE: return b200z_xz_bound(in, n) + 64;
    case B200Z_FILE_XZ_ENCODE: return b200z_xz_encode_bound(n);
  }
  return 0;
}

// `hist`: the tail of what this decodeStream call has already written (gzip only: the members share one OutputStream and a
// member may copy from the ones before it -- b200z_internal.h InflateWs::hist)
int call_codec(const Args &a, const uint8_t *in, size_t n, uint8_t *out, size_t cap, size_t *got,
               const std::vector<uint8_t> *hist = nullptr) {
  switch (a.op) {
    case B200Z_FILE_GZIP_DECODE:
      if (hist && !hist->empty()) return gzip_decode_after(in, n, a.a0, hist->data(), hist->size(), out, cap, got);
      return b200z_gzip_decode(in, n, a.a0, out, cap, got);
    case B200Z_FILE_ZLIB_DECODE: return b200z_zlib_decode(in, n, a.a0, a.a1, out, cap, got);
    case B200Z_FILE_BZIP2_DECODE: return b200z_bzip2_decode(in, n, a.a0, out, cap, got);
    case B200Z_FILE_ZLIB_ENCODE: return b200z_zlib_encode(in, n, a.a0, a.a1, (int)a.a2, out, cap, got);
    case B200Z_FILE_GZIP_ENCODE: return b200z_gzip_encode(in, n, a.a0, a.a2, out, cap, got);
    case B200Z_FILE_BZIP2_ENCODE: return b200z_bzip2_encode(in, n, out, cap, got);
    case B200Z_FILE_XZ_DECODE: return b200z_xz_decode(in, n, a.a0, out, cap, got);
    case B200Z_FILE_XZ_ENCODE: return b200z_xz_encode(in, n, a.a0, out, cap, got);
  }
  return B200Z_E_ARG;
}

// One segment = the whole range [off, off + n): read, one codec call (grown on B200Z_E_NOSPC), write.  What a data error
// leaves behind is written too -- the reference's streams have it by then (bzip2_decoder.dart:32-78, inflate.dart:150-151).
int whole_range(const Args &a, int ifd, uint64_t off, size_t n, int ofd, uint64_t out_off, uint64_t *written,
                const std::vector<uint8_t> *hist = nullptr) {
  *written = 0;
  F.n_whole++;
  if (!F.in[0].reserve(n + 8)) return B200Z_E_NODEVICE;
  if (!par_io(false, ifd, F.in[0].p, n, off)) {
    set_error_text("b200z_file_codec: read failed (I/O error, or the file shrank)");
    return B200Z_E_ARG;
  }
  size_t cap = first_cap(a, F.in[0].p, n), got = 0;
  int rc;
  for (;;) {
    if (!F.out[0].reserve(cap)) return B200Z_E_NODEVICE;
    got = 0;
    rc = call_codec(a, F.in[0].p, n, F.out[0].p, cap, &got, hist);
    if (rc != B200Z_E_NOSPC || cap >= ((size_t)1 << 40)) break;
    cap = std::max(cap * 2, got + (got >> 3) + 64);
  }
  if (rc != B200Z_OK && rc != B200Z_E_DATA && rc != B200Z_E_THROW) return rc;
  const size_t nw = std::min(got, cap);
  if (nw && !par_io(true, ofd, F.out[0].p, nw, out_off)) {
    set_error_text("b200z_file_codec: write failed");
    return B200Z_E_ARG;
  }
  *written = nw;
  return rc;
}

// GZip members with size hints, segment by segment.  Falls back to whole_range for whatever is left as soon as the front
// of a segment is not a hinted member (no hints at all, a member larger than a segment) or a hint turns out wrong.
int gzip_segments(const Args &a, int ifd, uint64_t off, uint64_t end, int ofd, uint64_t out_off, uint64_t *written) {
  const size_t seg = env_size("B200Z_FILE_SEG_KB", 256u << 10, 64, 1u << 26) << 10;
  *written = 0;
  if (end - off <= seg) return whole_range(a, ifd, off, (size_t)(end - off), ofd, out_off, written);
  AsyncIo rd, wr;
  int s = 0;
  size_t have = (size_t)std::min<uint64_t>(seg, end - off);
  if (!F.in[0].reserve(seg + 8) || !F.in[1].reserve(seg + 8)) return B200Z_E_NODEVICE;
  rd.start(false, ifd, F.in[0].p, have, off);
  uint64_t wpos = out_off;
  int rc = B200Z_OK;
  bool rest = false;  // hand [off, end) to whole_range
  std::vector<uint8_t> hist;  // the last 32 KiB written so far: within reach of the next member's back-references
  const size_t kHist = 32768;
  while (off < end) {
    if (!rd.wait()) {
      set_error_text("b200z_file_codec: read failed (I/O error, or the file shrank)");
      rc = B200Z_E_ARG;
      break;
    }
    size_t promised = 0;
    const size_t e = gzip_hinted_prefix(F.in[s].p, have, &promised);
    if (e == 0 || promised > kMaxExpansion * e + 1024) {  // (hints that cannot be true: the hint-free path decides)
      rest = true;
      break;
    }
    const uint64_t next_off = off + e;
    size_t next_have = 0;
    if (next_off < end) {  // read ahead while this segment is on the device
      next_have = (size_t)std::min<uint64_t>(seg, end - next_off);
      rd.start(false, ifd, F.in[s ^ 1].p, next_have, next_off);
    }
    if (!F.out[s].reserve(promised + 64)) {
      rc = B200Z_E_NODEVICE;
      break;
    }
    size_t used = 0, got = 0;
    rc = gzip_decode_hinted(F.in[s].p, e, F.out[s].p, promised + 64, &used, &got);
    if (rc) break;
    F.n_segments++;
    if (!wr.wait()) {  // the write of the segment before this one
      set_error_text("b200z_file_codec: write failed");
      rc = B200Z_E_ARG;
      break;
    }
    if (got) wr.start(true, ofd, F.out[s].p, got, wpos);
    wpos += got;
    if (got >= kHist) {
      hist.assign(F.out[s].p + got - kHist, F.out[s].p + got);
    } else if (got) {
      hist.insert(hist.end(), F.out[s].p, F.out[s].p + got);
      if (hist.size() > kHist) hist.erase(hist.begin(), hist.end() - kHist);
    }
    off += used;
    if (used < e) {  // a hint lied: the member at `off` is decoded the hint-free way, with the rest of the file behind it
      rest = true;
      break;
    }
    have = next_have;
    s ^= 1;
  }
  rd.wait();
  if (!wr.wait() && rc == B200Z_OK) {
    set_error_text("b200z_file_codec: write failed");
    rc = B200Z_E_ARG;
  }
  *written = wpos - out_off;
  if (rc == B200Z_OK && rest && off < end) {
    uint64_t w2 = 0;
    rc = whole_range(a, ifd, off, (size_t)(end - off), ofd, wpos, &w2, &hist);
    *written += w2;
  }
  return rc;
}

}  // namespace

void file_release() {
  std::lock_guard<std::mutex> lk(F.mu);
  for (int i = 0; i < 2; ++i) {
    F.in[i].release();
    F.out[i].release();
  }
}

}  // namespace b200z

using namespace b200z;

extern "C" int b200z_file_codec(int op, const char *in_path, uint64_t in_off, uint64_t in_len, const char *out_path,
                                uint64_t out_off, int32_t a0, int32_t a1, uint32_t a2, uint64_t *in_used,
                                uint64_t *out_len) {
  if (in_used) *in_used = 0;
  if (out_len) *out_len = 0;
  if (op < B200Z_FILE_GZIP_DECODE || op > B200Z_FILE_XZ_ENCODE || !in_path || !out_path) {
    set_error_text("b200z_file_codec: invalid argument");
    return B200Z_E_ARG;
  }
  if (b200z_device_count() <= 0) {  // before any file is touched: there is no CPU fallback
    set_error_text("b200z_file_codec: no CUDA device (there is no CPU fallback)");
    return B200Z_E_NODEVICE;
  }
  std::lock_guard<std::mutex> lk(F.mu);
  F.n_segments = F.n_whole = 0;
  const int ifd = open(in_path, O_RDONLY | O_CLOEXEC);
  if (ifd < 0) {
    errf("b200z_file_codec: cannot open %s: %s", in_path, errno);
    return B200Z_E_ARG;
  }
  struct stat st;
  if (fstat(ifd, &st) != 0) {
    errf("b200z_file_codec: cannot stat %s: %s", in_path, errno);
    close(ifd);
    return B200Z_E_ARG;
  }
  const uint64_t size = (uint64_t)st.st_size;
  if (in_off > size) in_off = size;
  if (in_len > size - in_off) in_len = size - in_off;  // readBytes clamps to what is there (input_file_stream.dart:196-207)
  const int ofd = open(out_path, O_WRONLY | O_CREAT | O_CLOEXEC, 0644);  // not truncated: the stream has written before us
  if (ofd < 0) {
    errf("b200z_file_codec: cannot open %s for writing: %s", out_path, errno);
    close(ifd);
    return B200Z_E_ARG;
  }
  const Args a{op, a0, a1, a2};
  uint64_t written = 0;
  int rc;
  if (in_len >= ((uint64_t)1 << 40)) {
    set_error_text("b200z_file_codec: range of 1 TiB or more");
    rc = B200Z_E_ARG;
  } else if (op == B200Z_FILE_GZIP_DECODE) {
    rc = gzip_segments(a, ifd, in_off, in_off + in_len, ofd, out_off, &written);
  } else {
    rc = whole_range(a, ifd, in_off, (size_t)in_len, ofd, out_off, &written);
  }
  close(ifd);
  if (close(ofd) != 0 && rc == B200Z_OK) {
    errf("b200z_file_codec: close of %s failed: %s", out_path, errno);
    rc = B200Z_E_ARG;
  }
  if (in_used) *in_used = in_len;  // decodeStream / encodeStream consume the input stream to its end
  if (out_len) *out_len = written;
  return rc;
}

extern "C" void b200z_file_last_stats(uint32_t *n_segments, uint32_t *n_whole) {
  std::lock_guard<std::mutex> lk(F.mu);
  if (n_segments) *n_segments = F.n_segments;
  if (n_whole) *n_whole = F.n_whole;
}
