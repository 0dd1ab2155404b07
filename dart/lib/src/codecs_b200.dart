// The plug point of the reference is the conditional-export seam that binds
// `platformZLibDecoder` / `platformGZipDecoder` (lib/src/codecs/zlib/_zlib_decoder.dart:1,
// _gzip_decoder.dart:1) to an object implementing ZLibDecoderBase
// (lib/src/codecs/zlib/_zlib_decoder_base.dart:5-13).  These classes implement that interface on top
// of libb200z.so; `Inflate` mirrors lib/src/codecs/zlib/inflate.dart:12-116 and BZip2Decoder mirrors
// lib/src/codecs/bzip2_decoder.dart:12-21.
import 'dart:ffi';
import 'dart:typed_data';

import 'package:archive/archive.dart' as ar;
import 'package:ffi/ffi.dart';

import 'b200z_ffi.dart';

Uint8List _drain(ar.InputStream input) =>
    input is ar.InputMemoryStream ? input.toUint8List() : input.toUint8List();

/// Same surface as the reference's `Inflate`: all work in the constructor, never throws on bad data.
class Inflate {
  final ar.OutputStream _output;
  int status = 1;

  Inflate(List<int> bytes, {ar.OutputStream? output, int? uncompressedSize})
      : _output = output ?? ar.OutputMemoryStream(size: uncompressedSize) {
    _run(ar.InputMemoryStream(bytes), uncompressedSize);
  }

  Inflate.stream(ar.InputStream? input, {ar.OutputStream? output, int? uncompressedSize})
      : _output = output ?? ar.OutputMemoryStream(size: uncompressedSize) {
    if (input != null) _run(input, uncompressedSize);
  }

  void _run(ar.InputStream input, int? sizeHint) {
    final z = B200Z.instance;
    final data = _drain(input);
    if (data.isEmpty) return;
    final inp = z.toNative(data);
    final consumed = calloc<Size>();
    final ust = calloc<Int32>();
    try {
      final (out, _) = z.grow(sizeHint ?? data.length * 4 + 1024,
          (o, cap, outLen) => z.inflateRaw(inp, data.length, o, cap, outLen, consumed, ust));
      status = ust.value;
      _output.writeBytes(out);
      input.skip(consumed.value); // inflate.dart:337-340: stream left on the first unread byte
    } finally {
      calloc.free(consumed);
      calloc.free(ust);
      z.hostFree(inp);
    }
  }

  Uint8List getBytes() => _output.getBytes();
}

/// decodeStream / encodeStream with an InputFileStream and an OutputFileStream: hand the library the two files.
/// InputFileStream exposes its FileBuffer (`file`, input_file_stream.dart:218) but neither its path nor its offset
/// into the file; the one-line getters INTEGRATION.md lists (`InputFileStream.path` / `.fileOffset`,
/// `OutputFileStream.path` / `.advanced(n)`) are the only change to the reference's own classes this path needs.
/// Returns null when the pair is not file/file (the caller then takes the in-memory route).
bool? _fileToFile(int op, ar.InputStream input, ar.OutputStream output, {int a0 = 0, int a1 = 0, int a2 = 0}) {
  if (input is! ar.InputFileStream || output is! ar.OutputFileStream) return null;
  final inPath = (input as dynamic).path as String?;
  final outPath = (output as dynamic).path as String?;
  if (inPath == null || outPath == null) return null; // RAM file handles have no path: in-memory route
  output.flush();
  final start = ((input as dynamic).fileOffset as int) + input.position;
  final n = input.length;
  final (written, ok) =
      B200Z.instance.fileCodecCall(op, inPath, start, n, outPath, output.length, a0: a0, a1: a1, a2: a2);
  (output as dynamic).advanced(written); // _length += written; _fileHandle.position += written
  input.skip(n);
  return ok;
}

class _B200ZLibDecoder extends ar.ZLibDecoderBase {
  const _B200ZLibDecoder();

  @override
  Uint8List decodeBytes(List<int> data, {bool verify = false, bool raw = false}) {
    final z = B200Z.instance;
    final inp = z.toNative(data);
    try {
      final (out, _) = z.grow(data.length * 4 + 1024,
          (o, cap, outLen) => z.zlibDecode(inp, data.length, verify ? 1 : 0, raw ? 1 : 0, o, cap, outLen));
      return out;
    } finally {
      z.hostFree(inp);
    }
  }

  @override
  bool decodeStream(ar.InputStream input, ar.OutputStream output, {bool verify = false, bool raw = false}) {
    final viaFiles = _fileToFile(b200zFileZlibDecode, input, output, a0: verify ? 1 : 0, a1: raw ? 1 : 0);
    if (viaFiles != null) return viaFiles;
    final z = B200Z.instance;
    final data = _drain(input);
    final inp = z.toNative(data);
    try {
      final (out, ok) = z.grow(data.length * 4 + 1024,
          (o, cap, outLen) => z.zlibDecode(inp, data.length, verify ? 1 : 0, raw ? 1 : 0, o, cap, outLen));
      output.writeBytes(out);
      input.skip(data.length);
      return ok;
    } finally {
      z.hostFree(inp);
    }
  }
}

class _B200GZipDecoder extends ar.ZLibDecoderBase {
  const _B200GZipDecoder();

  @override
  Uint8List decodeBytes(List<int> data, {bool verify = false, bool raw = false}) {
    final output = ar.OutputMemoryStream();
    decodeStream(ar.InputMemoryStream(data), output, verify: verify, raw: raw);
    return output.getBytes();
  }

  @override
  bool decodeStream(ar.InputStream input, ar.OutputStream output, {bool verify = false, bool raw = false}) {
    // `verify` carries two bits for the library: 1 = verify, 2 = raw (B200Z_GZIP_RAW: handed on to the zlib decoder when the
    // input has no gzip header, _gzip_decoder_web.dart:31-37)
    final vr = (verify ? 1 : 0) | (raw ? 2 : 0);
    final viaFiles = _fileToFile(b200zFileGzipDecode, input, output, a0: vr);
    if (viaFiles != null) return viaFiles;
    final z = B200Z.instance;
    final data = _drain(input);
    final inp = z.toNative(data);
    try {
      final bound = z.gzipBound(inp, data.length);
      final (out, ok) = z.grow(bound > 0 ? bound : data.length * 4 + 1024,
          // several devices initialised (B200Z.multiInit): the members are dealt to them -- the same bytes come back
          (o, cap, outLen) => z.multiDeviceCount() > 1
              ? z.gzipDecodeMulti(inp, data.length, vr, o, cap, outLen, 0)
              : z.gzipDecode(inp, data.length, vr, o, cap, outLen));
      output.writeBytes(out);
      input.skip(data.length);
      return ok;
    } finally {
      z.hostFree(inp);
    }
  }
}

/// Drop these four names into a `_zlib_decoder_b200.dart` / `_gzip_decoder_b200.dart` selected by the
/// reference's conditional export (INTEGRATION.md).
const platformZLibDecoder = _B200ZLibDecoder();
const platformGZipDecoder = _B200GZipDecoder();

class BZip2Decoder {
  Uint8List decodeBytes(List<int> data, {bool verify = false}) {
    final z = B200Z.instance;
    final inp = z.toNative(data);
    try {
      final (out, _) = z.grow(data.length * 6 + 1024,
          (o, cap, outLen) => z.bzip2Decode(inp, data.length, verify ? 1 : 0, o, cap, outLen));
      return out;
    } finally {
      z.hostFree(inp);
    }
  }

  bool decodeStream(ar.InputStream input, ar.OutputStream output, {bool verify = false}) {
    final viaFiles = _fileToFile(b200zFileBzip2Decode, input, output, a0: verify ? 1 : 0);
    if (viaFiles != null) return viaFiles;
    final z = B200Z.instance;
    final data = _drain(input);
    final inp = z.toNative(data);
    try {
      final (out, ok) = z.grow(data.length * 6 + 1024,
          (o, cap, outLen) => z.bzip2Decode(inp, data.length, verify ? 1 : 0, o, cap, outLen));
      output.writeBytes(out);
      input.skip(data.length);
      return ok;
    } finally {
      z.hostFree(inp);
    }
  }
}

/// `XZDecoder` (xz_decoder.dart:15-27): one stream; the LZMA2 runs between dictionary resets decode on the device.
class XZDecoder {
  Uint8List decodeBytes(List<int> data, {bool verify = false}) {
    final out = ar.OutputMemoryStream();
    decodeStream(ar.InputMemoryStream(data), out, verify: verify);
    return out.getBytes();
  }

  bool decodeStream(ar.InputStream input, ar.OutputStream output, {bool verify = false}) {
    final viaFiles = _fileToFile(b200zFileXzDecode, input, output, a0: verify ? 1 : 0);
    if (viaFiles != null) return viaFiles;
    final z = B200Z.instance;
    final data = _drain(input);
    final inp = z.toNative(data);
    try {
      final (out, ok) = z.grow(z.xzBound(inp, data.length) + 64,
          (o, cap, outLen) => z.xzDecode(inp, data.length, verify ? 1 : 0, o, cap, outLen));
      output.writeBytes(out);
      input.skip(data.length);
      return ok;
    } finally {
      z.hostFree(inp);
    }
  }
}

/// `XZEncoder` (xz_encoder.dart:18-62): one stored LZMA2 chunk and the check, computed on the device.
class XZEncoder {
  Uint8List encodeBytes(List<int> data, {ar.XZCheck check = ar.XZCheck.crc64}) {
    final z = B200Z.instance;
    final inp = z.toNative(data);
    try {
      final (out, _) = z.grow(z.xzEncodeBound(data.length),
          (o, cap, outLen) => z.xzEncode(inp, data.length, check.index, o, cap, outLen));
      return out;
    } finally {
      z.hostFree(inp);
    }
  }

  List<int> encode(List<int> data, {ar.XZCheck check = ar.XZCheck.crc64}) => encodeBytes(data, check: check);

  void encodeStream(ar.InputStream input, ar.OutputStream output, {ar.XZCheck check = ar.XZCheck.crc64}) {
    if (_fileToFile(b200zFileXzEncode, input, output, a0: check.index) != null) return;
    output.writeBytes(encodeBytes(_drain(input), check: check));
  }
}

// ---- encoders: the `platformZLibEncoder` / `platformGZipEncoder` seam (_zlib_encoder.dart:1, _gzip_encoder.dart:1),
// `Deflate` (deflate.dart:25-100) and `BZip2Encoder` (bzip2_encoder.dart:15-81) ----

/// Same surface as the reference's `Deflate`: the stream is produced in the constructor.
class Deflate {
  final ar.OutputStream _output;
  int crc32 = 0;

  Deflate(List<int> bytes, {int level = 6, int windowBits = 15, ar.OutputStream? output})
      : _output = output ?? ar.OutputMemoryStream() {
    final z = B200Z.instance;
    final inp = z.toNative(bytes);
    final crc = calloc<Uint32>();
    try {
      final (out, _) = z.grow(z.deflateBound(bytes.length),
          (o, cap, outLen) => z.deflateRaw(inp, bytes.length, level, windowBits, o, cap, outLen, crc));
      crc32 = crc.value;
      _output.writeBytes(out);
    } finally {
      calloc.free(crc);
      z.hostFree(inp);
    }
  }

  Uint8List getBytes() => _output.getBytes();
}

class _B200ZLibEncoder extends ar.ZLibEncoderBase {
  const _B200ZLibEncoder();

  @override
  Uint8List encodeBytes(List<int> bytes, {int? level, int? windowBits, bool raw = false}) {
    final z = B200Z.instance;
    final inp = z.toNative(bytes);
    try {
      final (out, _) = z.grow(z.deflateBound(bytes.length) + 16,
          (o, cap, outLen) => z.zlibEncode(inp, bytes.length, level ?? 6, windowBits ?? 15, raw ? 1 : 0, o, cap, outLen));
      return out;
    } finally {
      z.hostFree(inp);
    }
  }

  @override
  void encodeStream(ar.InputStream input, ar.OutputStream output, {int? level, int? windowBits, bool raw = false}) {
    if (_fileToFile(b200zFileZlibEncode, input, output, a0: level ?? 6, a1: windowBits ?? 15, a2: raw ? 1 : 0) != null) return;
    output.writeBytes(encodeBytes(_drain(input), level: level, windowBits: windowBits, raw: raw));
  }
}

class _B200GZipEncoder extends ar.ZLibEncoderBase {
  const _B200GZipEncoder();

  @override
  Uint8List encodeBytes(List<int> bytes, {int? level, int? windowBits, bool raw = false}) {
    final z = B200Z.instance;
    final inp = z.toNative(bytes);
    final mtime = DateTime.now().millisecondsSinceEpoch ~/ 1000; // _gzip_encoder_web.dart:82-90 writes "now"
    try {
      final (out, _) = z.grow(z.deflateBound(bytes.length) + 32,
          (o, cap, outLen) => z.gzipEncode(inp, bytes.length, level ?? 6, mtime, o, cap, outLen));
      return out;
    } finally {
      z.hostFree(inp);
    }
  }

  @override
  void encodeStream(ar.InputStream input, ar.OutputStream output, {int? level, int? windowBits, bool raw = false}) {
    final now = DateTime.now().millisecondsSinceEpoch ~/ 1000; // _gzip_encoder_web.dart:82
    if (_fileToFile(b200zFileGzipEncode, input, output, a0: level ?? 6, a2: now) != null) return;
    output.writeBytes(encodeBytes(_drain(input), level: level));
  }
}

const platformZLibEncoder = _B200ZLibEncoder();
const platformGZipEncoder = _B200GZipEncoder();

class BZip2Encoder {
  Uint8List encodeBytes(List<int> data) {
    final z = B200Z.instance;
    final inp = z.toNative(data);
    try {
      final (out, _) =
          z.grow(z.bzip2Bound(data.length), (o, cap, outLen) => z.bzip2Encode(inp, data.length, o, cap, outLen));
      return out;
    } finally {
      z.hostFree(inp);
    }
  }

  Uint8List encode(List<int> data) => encodeBytes(data);

  bool encodeStream(ar.InputStream input, ar.OutputStream output) {
    if (_fileToFile(b200zFileBzip2Encode, input, output) != null) return true;
    output.writeBytes(encodeBytes(_drain(input)));
    return true;
  }
}

/// ZipDecoder (zip_decoder.dart:18-81) with all members decompressed by ONE b200z_zip_extract_password call; the password
/// (if any) goes to the library as the low bytes of its code units, as ZipFile.deriveKey / _initKeys use it.
class ZipDecoder {
  ar.Archive decodeBytes(List<int> bytes, {bool verify = false, String? password}) {
    final z = B200Z.instance;
    final inp = z.toNative(bytes);
    final n = calloc<Size>();
    try {
      var rc = z.zipList(inp, bytes.length, nullptr, 0, n);
      if (rc == b200zEThrow) throw RangeError(z.lastError);
      final count = n.value;
      final archive = ar.Archive();
      if (count == 0) return archive;
      final ents = calloc<ZipEntry>(count);
      final off = calloc<Uint64>(count), room = calloc<Uint64>(count), len = calloc<Uint64>(count);
      final st = calloc<Int32>(count);
      try {
        rc = z.zipList(inp, bytes.length, ents, count, n);
        if (rc != b200zOk) throw B200ZException(rc, z.lastError);
        var total = 0;
        for (var i = 0; i < count; i++) {
          final e = ents[i];
          final r = e.hasData != 0 ? (e.hintUncompSize > e.uncompSize ? e.hintUncompSize : e.uncompSize) : 0;
          off[i] = total;
          room[i] = r;
          total += (r + 63) & ~63;
        }
        final out = z.hostAlloc(total == 0 ? 64 : total);
        final pw = password == null ? nullptr : calloc<Uint8>(password.length + 1);
        for (var i = 0; password != null && i < password.length; i++) {
          pw[i] = password.codeUnitAt(i) & 0xff;
        }
        try {
          rc = z.zipExtractPassword(inp, bytes.length, ents, count, out, total, off, room, len, st, 0, pw, password?.length ?? 0);
          if (rc != b200zOk) throw B200ZException(rc, z.lastError);
          // (members whose size fields lied report B200Z_U_NOSPC: retry those with more room, as archive_b200/zip.py does)
          final all = out.asTypedList(total == 0 ? 0 : total);
          for (var i = 0; i < count; i++) {
            final e = ents[i];
            final name = e.hasData != 0 ? String.fromCharCodes(bytes.sublist(e.nameOff, e.nameOff + e.nameLen)) : '';
            if (archive.find(name) != null) continue;
            final isDir = name.endsWith('/') || name.endsWith('\\');
            // the reference throws when such a member is read (zip_file.dart:333-341); this shim reads every member here
            if (st[i] == -22) throw Exception('password error');
            if (st[i] == -23) throw Exception('macs don\'t match');
            if (st[i] == -5) throw RangeError('$name: encrypted member too short, or an empty password');
            final content = Uint8List.fromList(all.sublist(off[i], off[i] + (len[i] < room[i] ? len[i] : room[i])));
            final f = isDir ? ar.ArchiveFile.directory(name) : ar.ArchiveFile.bytes(name, content);
            f.mode = e.extAttr >> 16;
            f.crc32 = e.crc32;
            f.lastModTime = e.modDate << 16 | e.modTime;
            archive.add(f);
          }
        } finally {
          z.hostFree(out);
          if (pw != nullptr) calloc.free(pw);
        }
        return archive;
      } finally {
        calloc.free(ents);
        calloc.free(off);
        calloc.free(room);
        calloc.free(len);
        calloc.free(st);
      }
    } finally {
      calloc.free(n);
      z.hostFree(inp);
    }
  }
}
