// dart:ffi binding of include/b200z.h.  NOT compiled or run in the build image (no Dart SDK there):
// it is the reference-side stub INTEGRATION.md describes, written to the letter of the C ABI.
// The Python ctypes mirror (archive_b200/_ffi.py) binds the same symbols and IS exercised by the tests.
import 'dart:ffi';
import 'dart:io' show Platform;
import 'dart:typed_data';

import 'package:ffi/ffi.dart';

const b200zOk = 0;
const b200zENoDevice = -1;
const b200zEArg = -2;
const b200zENoSpc = -3;
const b200zEData = -4;
const b200zEThrow = -5;

typedef _InitC = Int32 Function(Int32 device, Uint32 flags);
typedef _InitD = int Function(int device, int flags);
typedef _ErrC = Pointer<Utf8> Function();
typedef _HostAllocC = Pointer<Uint8> Function(Size bytes);
typedef _HostAllocD = Pointer<Uint8> Function(int bytes);
typedef _HostFreeC = Void Function(Pointer<Uint8> p);
typedef _HostFreeD = void Function(Pointer<Uint8> p);
typedef _InflateRawC = Int32 Function(Pointer<Uint8> inp, Size inLen, Pointer<Uint8> out, Size outCap,
    Pointer<Size> outLen, Pointer<Size> inConsumed, Pointer<Int32> unitStatus);
typedef _InflateRawD = int Function(Pointer<Uint8> inp, int inLen, Pointer<Uint8> out, int outCap,
    Pointer<Size> outLen, Pointer<Size> inConsumed, Pointer<Int32> unitStatus);
typedef _GzipDecodeC = Int32 Function(
    Pointer<Uint8> inp, Size inLen, Int32 verify, Pointer<Uint8> out, Size outCap, Pointer<Size> outLen);
typedef _GzipDecodeD = int Function(
    Pointer<Uint8> inp, int inLen, int verify, Pointer<Uint8> out, int outCap, Pointer<Size> outLen);
typedef _ZlibDecodeC = Int32 Function(Pointer<Uint8> inp, Size inLen, Int32 verify, Int32 raw,
    Pointer<Uint8> out, Size outCap, Pointer<Size> outLen);
typedef _ZlibDecodeD = int Function(Pointer<Uint8> inp, int inLen, int verify, int raw,
    Pointer<Uint8> out, int outCap, Pointer<Size> outLen);
typedef _BoundC = Size Function(Pointer<Uint8> inp, Size inLen);
typedef _BoundD = int Function(Pointer<Uint8> inp, int inLen);
typedef _Bz2DecodeC = Int32 Function(
    Pointer<Uint8> inp, Size inLen, Int32 verify, Pointer<Uint8> out, Size outCap, Pointer<Size> outLen);
typedef _Bz2DecodeD = int Function(
    Pointer<Uint8> inp, int inLen, int verify, Pointer<Uint8> out, int outCap, Pointer<Size> outLen);
typedef _Bz2DecodeBatchC = Int32 Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, Size n,
    Int32 verify, Pointer<Uint8> outBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap, Pointer<Uint64> outLen, Pointer<Int32> rc);
typedef _Bz2DecodeBatchD = int Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, int n,
    int verify, Pointer<Uint8> outBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap, Pointer<Uint64> outLen, Pointer<Int32> rc);
// b200z_zlib_decode_batch: (inBase, inOff, inLen, n, verify, raw, outBase, outOff, outCap, outLen, rc)
typedef _ZlibDecodeBatchC = Int32 Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, Size n,
    Int32 verify, Int32 raw, Pointer<Uint8> outBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap, Pointer<Uint64> outLen,
    Pointer<Int32> rc);
typedef _ZlibDecodeBatchD = int Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, int n,
    int verify, int raw, Pointer<Uint8> outBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap, Pointer<Uint64> outLen,
    Pointer<Int32> rc);
// b200z_{gzip,bzip2,xz}_decode_batch_to_device: the host batch's arguments, then the cudaStream_t (dOutBase is device memory)
typedef _DecodeBatchToDeviceC = Int32 Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, Size n,
    Int32 verify, Pointer<Uint8> dOutBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap, Pointer<Uint64> outLen,
    Pointer<Int32> rc, Pointer<Void> cudaStream);
typedef _DecodeBatchToDeviceD = int Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, int n,
    int verify, Pointer<Uint8> dOutBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap, Pointer<Uint64> outLen,
    Pointer<Int32> rc, Pointer<Void> cudaStream);
// b200z_zlib_decode_batch_to_device: (inBase, inOff, inLen, n, verify, raw, dOutBase, outOff, outCap, outLen, rc, cudaStream)
typedef _ZlibDecodeBatchToDeviceC = Int32 Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, Size n,
    Int32 verify, Int32 raw, Pointer<Uint8> dOutBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap, Pointer<Uint64> outLen,
    Pointer<Int32> rc, Pointer<Void> cudaStream);
typedef _ZlibDecodeBatchToDeviceD = int Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, int n,
    int verify, int raw, Pointer<Uint8> dOutBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap, Pointer<Uint64> outLen,
    Pointer<Int32> rc, Pointer<Void> cudaStream);
// b200z_gzip_encode_batch: (inBase, inOff, inLen, n, level, mtime, outBase, outOff, outCap, outLen, rc)
typedef _GzipEncodeBatchC = Int32 Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, Size n,
    Int32 level, Uint32 mtime, Pointer<Uint8> outBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap,
    Pointer<Uint64> outLen, Pointer<Int32> rc);
typedef _GzipEncodeBatchD = int Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, int n,
    int level, int mtime, Pointer<Uint8> outBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap, Pointer<Uint64> outLen,
    Pointer<Int32> rc);
// b200z_zlib_encode_batch: (inBase, inOff, inLen, n, level, windowBits, raw, outBase, outOff, outCap, outLen, rc)
typedef _ZlibEncodeBatchC = Int32 Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, Size n,
    Int32 level, Int32 windowBits, Int32 raw, Pointer<Uint8> outBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap,
    Pointer<Uint64> outLen, Pointer<Int32> rc);
typedef _ZlibEncodeBatchD = int Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, int n,
    int level, int windowBits, int raw, Pointer<Uint8> outBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap,
    Pointer<Uint64> outLen, Pointer<Int32> rc);
typedef _Bz2EncodeBatchC = Int32 Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, Size n,
    Pointer<Uint8> outBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap, Pointer<Uint64> outLen, Pointer<Uint32> crc32,
    Pointer<Int32> rc);
typedef _Bz2EncodeBatchD = int Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, int n,
    Pointer<Uint8> outBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap, Pointer<Uint64> outLen, Pointer<Uint32> crc32,
    Pointer<Int32> rc);

typedef _DeflateRawC = Int32 Function(Pointer<Uint8> inp, Size inLen, Int32 level, Int32 windowBits, Pointer<Uint8> out,
    Size outCap, Pointer<Size> outLen, Pointer<Uint32> crc32OfInput);
typedef _DeflateRawD = int Function(Pointer<Uint8> inp, int inLen, int level, int windowBits, Pointer<Uint8> out,
    int outCap, Pointer<Size> outLen, Pointer<Uint32> crc32OfInput);
typedef _SizeOfC = Size Function(Size inLen);
typedef _SizeOfD = int Function(int inLen);
typedef _ZlibEncodeC = Int32 Function(Pointer<Uint8> inp, Size inLen, Int32 level, Int32 windowBits, Int32 raw,
    Pointer<Uint8> out, Size outCap, Pointer<Size> outLen);
typedef _ZlibEncodeD = int Function(Pointer<Uint8> inp, int inLen, int level, int windowBits, int raw,
    Pointer<Uint8> out, int outCap, Pointer<Size> outLen);
typedef _GzipEncodeC = Int32 Function(
    Pointer<Uint8> inp, Size inLen, Int32 level, Uint32 mtime, Pointer<Uint8> out, Size outCap, Pointer<Size> outLen);
typedef _GzipEncodeD = int Function(
    Pointer<Uint8> inp, int inLen, int level, int mtime, Pointer<Uint8> out, int outCap, Pointer<Size> outLen);
typedef _Bz2EncodeC = Int32 Function(Pointer<Uint8> inp, Size inLen, Pointer<Uint8> out, Size outCap, Pointer<Size> outLen);
typedef _Bz2EncodeD = int Function(Pointer<Uint8> inp, int inLen, Pointer<Uint8> out, int outCap, Pointer<Size> outLen);

// b200z_file_codec (include/b200z.h): paths and byte ranges instead of bytes
const b200zFileGzipDecode = 1;
const b200zFileZlibDecode = 2;
const b200zFileBzip2Decode = 3;
const b200zFileZlibEncode = 4;
const b200zFileGzipEncode = 5;
const b200zFileBzip2Encode = 6;
const b200zFileXzDecode = 7;
const b200zFileXzEncode = 8;
typedef _FileCodecC = Int32 Function(Int32 op, Pointer<Utf8> inPath, Uint64 inOff, Uint64 inLen, Pointer<Utf8> outPath,
    Uint64 outOff, Int32 a0, Int32 a1, Uint32 a2, Pointer<Uint64> inUsed, Pointer<Uint64> outLen);
typedef _FileCodecD = int Function(int op, Pointer<Utf8> inPath, int inOff, int inLen, Pointer<Utf8> outPath, int outOff,
    int a0, int a1, int a2, Pointer<Uint64> inUsed, Pointer<Uint64> outLen);

/// b200z_zip_entry (include/b200z.h)
final class ZipEntry extends Struct {
  @Uint64()
  external int localHeaderOff;
  @Uint64()
  external int dataOff;
  @Uint64()
  external int compSize;
  @Uint64()
  external int uncompSize;
  @Uint64()
  external int hintUncompSize;
  @Uint64()
  external int nameOff;
  @Uint64()
  external int cdNameOff;
  @Uint32()
  external int nameLen;
  @Uint32()
  external int cdNameLen;
  @Uint32()
  external int crc32;
  @Uint32()
  external int method;
  @Uint32()
  external int flags;
  @Uint32()
  external int modTime;
  @Uint32()
  external int modDate;
  @Uint32()
  external int extAttr;
  @Uint32()
  external int versionMadeBy;
  @Uint32()
  external int hasData;
}

typedef _ZipListC = Int32 Function(
    Pointer<Uint8> zip, Size zipLen, Pointer<ZipEntry> entries, Size cap, Pointer<Size> nEntries);
typedef _ZipListD = int Function(Pointer<Uint8> zip, int zipLen, Pointer<ZipEntry> entries, int cap, Pointer<Size> nEntries);
typedef _ZipExtractC = Int32 Function(Pointer<Uint8> zip, Size zipLen, Pointer<ZipEntry> entries, Size n, Pointer<Uint8> out,
    Size outCap, Pointer<Uint64> outOff, Pointer<Uint64> outRoom, Pointer<Uint64> outLen, Pointer<Int32> status, Uint32 flags);
typedef _ZipExtractD = int Function(Pointer<Uint8> zip, int zipLen, Pointer<ZipEntry> entries, int n, Pointer<Uint8> out,
    int outCap, Pointer<Uint64> outOff, Pointer<Uint64> outRoom, Pointer<Uint64> outLen, Pointer<Int32> status, int flags);
typedef _ZipCryptInfoC = Int32 Function(Pointer<Uint8> zip, Size zipLen, Pointer<ZipEntry> entry, Pointer<Uint32> mode,
    Pointer<Uint32> aesStrength, Pointer<Uint32> method);
typedef _ZipCryptInfoD = int Function(Pointer<Uint8> zip, int zipLen, Pointer<ZipEntry> entry, Pointer<Uint32> mode,
    Pointer<Uint32> aesStrength, Pointer<Uint32> method);
typedef _ZipExtractPasswordC = Int32 Function(Pointer<Uint8> zip, Size zipLen, Pointer<ZipEntry> entries, Size n,
    Pointer<Uint8> out, Size outCap, Pointer<Uint64> outOff, Pointer<Uint64> outRoom, Pointer<Uint64> outLen,
    Pointer<Int32> status, Uint32 flags, Pointer<Uint8> password, Size passwordLen);
typedef _ZipExtractPasswordD = int Function(Pointer<Uint8> zip, int zipLen, Pointer<ZipEntry> entries, int n,
    Pointer<Uint8> out, int outCap, Pointer<Uint64> outOff, Pointer<Uint64> outRoom, Pointer<Uint64> outLen,
    Pointer<Int32> status, int flags, Pointer<Uint8> password, int passwordLen);
typedef _ZipExtractToDeviceC = Int32 Function(Pointer<Uint8> zip, Size zipLen, Pointer<ZipEntry> entries, Size n,
    Pointer<Uint8> dOut, Size outCap, Pointer<Uint64> outOff, Pointer<Uint64> outRoom, Pointer<Uint64> outLen,
    Pointer<Int32> status, Pointer<Uint32> crc32, Uint32 flags, Pointer<Uint8> password, Size passwordLen,
    Pointer<Void> cudaStream);
typedef _ZipExtractToDeviceD = int Function(Pointer<Uint8> zip, int zipLen, Pointer<ZipEntry> entries, int n,
    Pointer<Uint8> dOut, int outCap, Pointer<Uint64> outOff, Pointer<Uint64> outRoom, Pointer<Uint64> outLen,
    Pointer<Int32> status, Pointer<Uint32> crc32, int flags, Pointer<Uint8> password, int passwordLen,
    Pointer<Void> cudaStream);
/// b200z_tar_member (include/b200z.h): one member found by b200z_tar_walk_device.
final class TarMember extends Struct {
  @Uint64()
  external int headerOff;
  @Uint64()
  external int contentOff;
  @Uint64()
  external int contentLen;
  @Int64()
  external int size;
  @Uint32()
  external int headerLen;
  @Uint32()
  external int pad_;
}

typedef _TarWalkDeviceC = Int32 Function(Pointer<Uint8> dBase, Pointer<Uint64> off, Pointer<Uint64> len, Size n,
    Pointer<TarMember> members, Pointer<Uint8> headers, Size cap, Pointer<Uint64> first, Pointer<Uint64> count,
    Pointer<Int32> rc, Pointer<Size> nTotal, Pointer<Void> cudaStream);
typedef _TarWalkDeviceD = int Function(Pointer<Uint8> dBase, Pointer<Uint64> off, Pointer<Uint64> len, int n,
    Pointer<TarMember> members, Pointer<Uint8> headers, int cap, Pointer<Uint64> first, Pointer<Uint64> count,
    Pointer<Int32> rc, Pointer<Size> nTotal, Pointer<Void> cudaStream);
typedef _ZipAesEncryptC = Int32 Function(Pointer<Uint8> data, Pointer<Uint64> off, Pointer<Uint64> len, Size n,
    Pointer<Uint8> salts, Pointer<Uint8> password, Size passwordLen, Pointer<Uint8> pwdVerify, Pointer<Uint8> mac);
typedef _ZipAesEncryptD = int Function(Pointer<Uint8> data, Pointer<Uint64> off, Pointer<Uint64> len, int n,
    Pointer<Uint8> salts, Pointer<Uint8> password, int passwordLen, Pointer<Uint8> pwdVerify, Pointer<Uint8> mac);


// ---- the rest of include/b200z.h: batches, sharding, checksums, diagnostics ----
/// b200z_bz2_block (include/b200z.h)
final class Bz2Block extends Struct {
  @Uint64()
  external int startBit;
  @Uint64()
  external int endBit;
  @Uint64()
  external int outBytes;
  @Uint32()
  external int crcCalc;
  @Uint32()
  external int crcStored;
  @Int32()
  external int status;
  @Uint32()
  external int flags;
}

typedef _Bz2ShardC = Int32 Function(Pointer<Uint8> inp, Size inLen, Uint32 rank, Uint32 world, Pointer<Uint8> out, Size outCap,
    Pointer<Size> outLen, Pointer<Bz2Block> blocks, Size blocksCap, Pointer<Size> nBlocks);
typedef _Bz2ShardD = int Function(Pointer<Uint8> inp, int inLen, int rank, int world, Pointer<Uint8> out, int outCap,
    Pointer<Size> outLen, Pointer<Bz2Block> blocks, int blocksCap, Pointer<Size> nBlocks);
typedef _Crc32C = Int32 Function(Pointer<Uint8> inp, Size inLen, Pointer<Uint32> crc);
typedef _Crc32D = int Function(Pointer<Uint8> inp, int inLen, Pointer<Uint32> crc);
typedef _Crc64C = Int32 Function(Pointer<Uint8> inp, Size inLen, Pointer<Uint64> crc);
typedef _Crc64D = int Function(Pointer<Uint8> inp, int inLen, Pointer<Uint64> crc);
typedef _DeflateBatchC = Int32 Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, Size nUnits,
    Int32 level, Int32 windowBits, Pointer<Uint8> outBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap, Pointer<Uint64> outLen,
    Pointer<Uint32> crc32, Pointer<Int32> status);
typedef _DeflateBatchD = int Function(Pointer<Uint8> inBase, Pointer<Uint64> inOff, Pointer<Uint64> inLen, int nUnits, int level,
    int windowBits, Pointer<Uint8> outBase, Pointer<Uint64> outOff, Pointer<Uint64> outCap, Pointer<Uint64> outLen,
    Pointer<Uint32> crc32, Pointer<Int32> status);
typedef _InflateBatchC = Int32 Function(Pointer<Uint8> inBase, Size inBytes, Pointer<Uint64> inOff, Pointer<Uint32> inLen,
    Pointer<Uint8> outBase, Size outBytes, Pointer<Uint64> outOff, Pointer<Uint32> outCap, Pointer<Uint32> outLen,
    Pointer<Int32> status, Pointer<Uint32> inUsed, Size nUnits);
typedef _InflateBatchD = int Function(Pointer<Uint8> inBase, int inBytes, Pointer<Uint64> inOff, Pointer<Uint32> inLen,
    Pointer<Uint8> outBase, int outBytes, Pointer<Uint64> outOff, Pointer<Uint32> outCap, Pointer<Uint32> outLen,
    Pointer<Int32> status, Pointer<Uint32> inUsed, int nUnits);
typedef _InflateBatchDeviceC = Int32 Function(Pointer<Uint8> dInBase, Pointer<Uint64> dInOff, Pointer<Uint32> dInLen,
    Pointer<Uint8> dOutBase, Pointer<Uint64> dOutOff, Pointer<Uint32> dOutCap, Pointer<Uint32> dOutLen, Pointer<Int32> dStatus,
    Pointer<Uint32> dInUsed, Size nUnits, Pointer<Void> dWorkspace, Size workspaceBytes, Pointer<Void> cudaStream);
typedef _InflateBatchDeviceD = int Function(Pointer<Uint8> dInBase, Pointer<Uint64> dInOff, Pointer<Uint32> dInLen,
    Pointer<Uint8> dOutBase, Pointer<Uint64> dOutOff, Pointer<Uint32> dOutCap, Pointer<Uint32> dOutLen, Pointer<Int32> dStatus,
    Pointer<Uint32> dInUsed, int nUnits, Pointer<Void> dWorkspace, int workspaceBytes, Pointer<Void> cudaStream);
// several GPUs driven by this one isolate (include/b200z.h "several GPUs of one box")
typedef _MultiInitC = Int32 Function(Uint32 deviceMask, Uint32 flags);
typedef _MultiInitD = int Function(int deviceMask, int flags);
typedef _GzipDecodeMultiC = Int32 Function(Pointer<Uint8> inp, Size inLen, Int32 verify, Pointer<Uint8> out, Size outCap,
    Pointer<Size> outLen, Uint32 flags);
typedef _GzipDecodeMultiD = int Function(Pointer<Uint8> inp, int inLen, int verify, Pointer<Uint8> out, int outCap,
    Pointer<Size> outLen, int flags);
typedef _InflateBatchMultiC = Int32 Function(Pointer<Uint8> inBase, Size inBytes, Pointer<Uint64> inOff, Pointer<Uint32> inLen,
    Pointer<Uint8> outBase, Size outBytes, Pointer<Uint64> outOff, Pointer<Uint32> outCap, Pointer<Uint32> outLen,
    Pointer<Int32> status, Pointer<Uint32> inUsed, Size nUnits, Uint32 flags);
typedef _InflateBatchMultiD = int Function(Pointer<Uint8> inBase, int inBytes, Pointer<Uint64> inOff, Pointer<Uint32> inLen,
    Pointer<Uint8> outBase, int outBytes, Pointer<Uint64> outOff, Pointer<Uint32> outCap, Pointer<Uint32> outLen,
    Pointer<Int32> status, Pointer<Uint32> inUsed, int nUnits, int flags);
typedef _MultiOutputC = Pointer<Void> Function(Int32 slot, Pointer<Size> bytes);
typedef _MultiOutputD = Pointer<Void> Function(int slot, Pointer<Size> bytes);
typedef _WorkspaceBytesC = Size Function(Size nUnits, Size totalInBytes, Size totalOutCap);
typedef _WorkspaceBytesD = int Function(int nUnits, int totalInBytes, int totalOutCap);
typedef _FileStatsC = Void Function(Pointer<Uint32> nSegments, Pointer<Uint32> nWhole);
typedef _FileStatsD = void Function(Pointer<Uint32> nSegments, Pointer<Uint32> nWhole);
typedef _ZipCommentC = Int32 Function(Pointer<Uint8> zip, Size zipLen, Pointer<Uint64> off, Pointer<Uint32> len);
typedef _ZipCommentD = int Function(Pointer<Uint8> zip, int zipLen, Pointer<Uint64> off, Pointer<Uint32> len);
typedef _VoidC = Void Function();
typedef _VoidD = void Function();
typedef _IntC = Int32 Function();
typedef _IntD = int Function();
typedef _U64C = Uint64 Function();
typedef _ProfileEnableC = Void Function(Int32 on);
typedef _ProfileEnableD = void Function(int on);
typedef _ProfileReadC = Int32 Function(Pointer<Double> fastMs, Pointer<Double> decodeMs, Pointer<Double> expandMs, Pointer<Uint64> nBatches);
typedef _ProfileReadD = int Function(Pointer<Double> fastMs, Pointer<Double> decodeMs, Pointer<Double> expandMs, Pointer<Uint64> nBatches);

class B200ZException implements Exception {
  final int code;
  final String message;
  B200ZException(this.code, this.message);
  @override
  String toString() => 'B200ZException($code): $message';
}

/// One process drives one GPU (b200z_init(device)); every call blocks.
class B200Z {
  static B200Z? _instance;
  final DynamicLibrary _lib;
  late final _InitD _init = _lib.lookupFunction<_InitC, _InitD>('b200z_init');
  late final _ErrC _lastError = _lib.lookupFunction<_ErrC, _ErrC>('b200z_last_error');
  late final _HostAllocD hostAlloc = _lib.lookupFunction<_HostAllocC, _HostAllocD>('b200z_host_alloc');
  late final _HostFreeD hostFree = _lib.lookupFunction<_HostFreeC, _HostFreeD>('b200z_host_free');
  late final _InflateRawD inflateRaw = _lib.lookupFunction<_InflateRawC, _InflateRawD>('b200z_inflate_raw');
  late final _GzipDecodeD gzipDecode = _lib.lookupFunction<_GzipDecodeC, _GzipDecodeD>('b200z_gzip_decode');
  late final _ZlibDecodeD zlibDecode = _lib.lookupFunction<_ZlibDecodeC, _ZlibDecodeD>('b200z_zlib_decode');
  late final _BoundD gzipBound = _lib.lookupFunction<_BoundC, _BoundD>('b200z_gzip_bound');
  late final _Bz2DecodeD bzip2Decode = _lib.lookupFunction<_Bz2DecodeC, _Bz2DecodeD>('b200z_bzip2_decode');
  late final _Bz2DecodeBatchD bzip2DecodeBatch =
      _lib.lookupFunction<_Bz2DecodeBatchC, _Bz2DecodeBatchD>('b200z_bzip2_decode_batch');
  late final _DeflateRawD deflateRaw = _lib.lookupFunction<_DeflateRawC, _DeflateRawD>('b200z_deflate_raw');
  late final _SizeOfD deflateBound = _lib.lookupFunction<_SizeOfC, _SizeOfD>('b200z_deflate_bound');
  late final _ZlibEncodeD zlibEncode = _lib.lookupFunction<_ZlibEncodeC, _ZlibEncodeD>('b200z_zlib_encode');
  late final _GzipEncodeD gzipEncode = _lib.lookupFunction<_GzipEncodeC, _GzipEncodeD>('b200z_gzip_encode');
  late final _Bz2EncodeD bzip2Encode = _lib.lookupFunction<_Bz2EncodeC, _Bz2EncodeD>('b200z_bzip2_encode');
  late final _Bz2EncodeBatchD bzip2EncodeBatch =
      _lib.lookupFunction<_Bz2EncodeBatchC, _Bz2EncodeBatchD>('b200z_bzip2_encode_batch');
  late final _SizeOfD bzip2Bound = _lib.lookupFunction<_SizeOfC, _SizeOfD>('b200z_bzip2_bound');
  late final _FileCodecD fileCodec = _lib.lookupFunction<_FileCodecC, _FileCodecD>('b200z_file_codec');
  late final _ZipListD zipList = _lib.lookupFunction<_ZipListC, _ZipListD>('b200z_zip_list');
  late final _ZipExtractD zipExtract = _lib.lookupFunction<_ZipExtractC, _ZipExtractD>('b200z_zip_extract');
  late final _ZipCommentD zipComment = _lib.lookupFunction<_ZipCommentC, _ZipCommentD>('b200z_zip_comment');
  late final _ZipCryptInfoD zipCryptInfo = _lib.lookupFunction<_ZipCryptInfoC, _ZipCryptInfoD>('b200z_zip_crypt_info');
  late final _ZipExtractPasswordD zipExtractPassword =
      _lib.lookupFunction<_ZipExtractPasswordC, _ZipExtractPasswordD>('b200z_zip_extract_password');
  // dOut: device memory of the library's device; crc32 may be nullptr
  late final _ZipExtractToDeviceD zipExtractToDevice =
      _lib.lookupFunction<_ZipExtractToDeviceC, _ZipExtractToDeviceD>('b200z_zip_extract_to_device');
  // the TAR member walk over archives in device memory: records and headers come back to the host
  late final _TarWalkDeviceD tarWalkDevice =
      _lib.lookupFunction<_TarWalkDeviceC, _TarWalkDeviceD>('b200z_tar_walk_device');
  late final _ZipAesEncryptD zipAesEncrypt = _lib.lookupFunction<_ZipAesEncryptC, _ZipAesEncryptD>('b200z_zip_aes_encrypt');
  late final _Bz2ShardD bzip2DecodeShard = _lib.lookupFunction<_Bz2ShardC, _Bz2ShardD>('b200z_bzip2_decode_shard');
  late final _Crc32D crc32 = _lib.lookupFunction<_Crc32C, _Crc32D>('b200z_crc32');
  // XZ: (in, inLen, verify | check, out, cap, outLen) -- the same shape as b200z_bzip2_decode
  late final _Bz2DecodeD xzDecode = _lib.lookupFunction<_Bz2DecodeC, _Bz2DecodeD>('b200z_xz_decode');
  late final _BoundD xzBound = _lib.lookupFunction<_BoundC, _BoundD>('b200z_xz_bound');
  late final _Bz2DecodeD xzEncode = _lib.lookupFunction<_Bz2DecodeC, _Bz2DecodeD>('b200z_xz_encode');
  late final _SizeOfD xzEncodeBound = _lib.lookupFunction<_SizeOfC, _SizeOfD>('b200z_xz_encode_bound');
  late final _Crc64D crc64 = _lib.lookupFunction<_Crc64C, _Crc64D>('b200z_crc64');
  // XZ batches: (inBase, inOff, inLen, n, verify | check, outBase, outOff, outCap, outLen, rc) -- the shape of
  // b200z_bzip2_decode_batch
  late final _Bz2DecodeBatchD xzDecodeBatch =
      _lib.lookupFunction<_Bz2DecodeBatchC, _Bz2DecodeBatchD>('b200z_xz_decode_batch');
  late final _Bz2DecodeBatchD xzEncodeBatch =
      _lib.lookupFunction<_Bz2DecodeBatchC, _Bz2DecodeBatchD>('b200z_xz_encode_batch');
  // gzip / zlib batches: gzip decode has the shape of b200z_bzip2_decode_batch (verify = B200Z_GZIP_VERIFY | _RAW bits)
  late final _Bz2DecodeBatchD gzipDecodeBatch =
      _lib.lookupFunction<_Bz2DecodeBatchC, _Bz2DecodeBatchD>('b200z_gzip_decode_batch');
  late final _ZlibDecodeBatchD zlibDecodeBatch =
      _lib.lookupFunction<_ZlibDecodeBatchC, _ZlibDecodeBatchD>('b200z_zlib_decode_batch');
  late final _DecodeBatchToDeviceD gzipDecodeBatchToDevice =
      _lib.lookupFunction<_DecodeBatchToDeviceC, _DecodeBatchToDeviceD>('b200z_gzip_decode_batch_to_device');
  late final _ZlibDecodeBatchToDeviceD zlibDecodeBatchToDevice =
      _lib.lookupFunction<_ZlibDecodeBatchToDeviceC, _ZlibDecodeBatchToDeviceD>('b200z_zlib_decode_batch_to_device');
  late final _DecodeBatchToDeviceD bzip2DecodeBatchToDevice =
      _lib.lookupFunction<_DecodeBatchToDeviceC, _DecodeBatchToDeviceD>('b200z_bzip2_decode_batch_to_device');
  late final _DecodeBatchToDeviceD xzDecodeBatchToDevice =
      _lib.lookupFunction<_DecodeBatchToDeviceC, _DecodeBatchToDeviceD>('b200z_xz_decode_batch_to_device');
  late final _GzipEncodeBatchD gzipEncodeBatch =
      _lib.lookupFunction<_GzipEncodeBatchC, _GzipEncodeBatchD>('b200z_gzip_encode_batch');
  late final _ZlibEncodeBatchD zlibEncodeBatch =
      _lib.lookupFunction<_ZlibEncodeBatchC, _ZlibEncodeBatchD>('b200z_zlib_encode_batch');
  late final _DeflateBatchD deflateBatch = _lib.lookupFunction<_DeflateBatchC, _DeflateBatchD>('b200z_deflate_batch');
  late final _InflateBatchD inflateBatch = _lib.lookupFunction<_InflateBatchC, _InflateBatchD>('b200z_inflate_batch');
  late final _InflateBatchDeviceD inflateBatchDevice =
      _lib.lookupFunction<_InflateBatchDeviceC, _InflateBatchDeviceD>('b200z_inflate_batch_device');
  late final _WorkspaceBytesD inflateWorkspaceBytes =
      _lib.lookupFunction<_WorkspaceBytesC, _WorkspaceBytesD>('b200z_inflate_workspace_bytes');
  late final _FileStatsD fileLastStats = _lib.lookupFunction<_FileStatsC, _FileStatsD>('b200z_file_last_stats');
  late final _MultiInitD multiInit = _lib.lookupFunction<_MultiInitC, _MultiInitD>('b200z_multi_init');
  late final _VoidD multiShutdown = _lib.lookupFunction<_VoidC, _VoidD>('b200z_multi_shutdown');
  late final _IntD multiDeviceCount = _lib.lookupFunction<_IntC, _IntD>('b200z_multi_device_count');
  late final _GzipDecodeMultiD gzipDecodeMulti =
      _lib.lookupFunction<_GzipDecodeMultiC, _GzipDecodeMultiD>('b200z_gzip_decode_multi');
  late final _InflateBatchMultiD inflateBatchMulti =
      _lib.lookupFunction<_InflateBatchMultiC, _InflateBatchMultiD>('b200z_inflate_batch_multi');
  late final _MultiOutputD multiDeviceOutput = _lib.lookupFunction<_MultiOutputC, _MultiOutputD>('b200z_multi_device_output');
  late final _VoidD shutdown = _lib.lookupFunction<_VoidC, _VoidD>('b200z_shutdown');
  late final _IntD deviceCount = _lib.lookupFunction<_IntC, _IntD>('b200z_device_count');
  late final _ErrC _version = _lib.lookupFunction<_ErrC, _ErrC>('b200z_version');
  late final _IntD launchCount = _lib.lookupFunction<_U64C, _IntD>('b200z_launch_count');
  late final _ProfileEnableD profileEnable = _lib.lookupFunction<_ProfileEnableC, _ProfileEnableD>('b200z_profile_enable');
  late final _ProfileReadD profileRead = _lib.lookupFunction<_ProfileReadC, _ProfileReadD>('b200z_profile_read');

  B200Z._(this._lib);

  static B200Z get instance {
    if (_instance == null) {
      final path = Platform.environment['B200Z_LIB'] ?? 'libb200z.so';
      final z = B200Z._(DynamicLibrary.open(path));
      final device = int.parse(Platform.environment['LOCAL_RANK'] ?? '0');
      final rc = z._init(device, 0);
      if (rc != b200zOk) {
        throw B200ZException(rc, z.lastError); // no CPU fallback: fail loudly
      }
      _instance = z;
    }
    return _instance!;
  }

  String get lastError => _lastError().toDartString();
  String get version => _version().toDartString();

  /// Copies [bytes] into pinned native memory (full-speed PCIe); caller frees with [hostFree].
  Pointer<Uint8> toNative(List<int> bytes) {
    final p = hostAlloc(bytes.isEmpty ? 1 : bytes.length);
    if (p == nullptr) throw B200ZException(b200zENoDevice, lastError);
    p.asTypedList(bytes.length).setAll(0, bytes);
    return p;
  }

  /// InputFileStream -> codec -> OutputFileStream without the bytes entering the Dart heap: the library reads
  /// [inPath] from [inOff] for [inLen] bytes and writes the result into [outPath] from [outOff] on (pinned segment
  /// buffers, threaded pread/pwrite; csrc/b200z_file.cu).  Returns (bytes written, ok); ok == false is the
  /// reference's `decodeStream` returning false -- what was produced before the error is in the file.
  (int, bool) fileCodecCall(int op, String inPath, int inOff, int inLen, String outPath, int outOff,
      {int a0 = 0, int a1 = 0, int a2 = 0}) {
    final ip = inPath.toNativeUtf8(), op_ = outPath.toNativeUtf8();
    final used = calloc<Uint64>(), got = calloc<Uint64>();
    try {
      final rc = fileCodec(op, ip, inOff, inLen, op_, outOff, a0, a1, a2, used, got);
      if (rc == b200zEThrow) throw RangeError(lastError);
      if (rc != b200zOk && rc != b200zEData) throw B200ZException(rc, lastError);
      return (got.value, rc == b200zOk);
    } finally {
      calloc.free(ip);
      calloc.free(op_);
      calloc.free(used);
      calloc.free(got);
    }
  }

  /// Runs [call](out, cap, outLen) growing the output buffer on B200Z_E_NOSPC; returns a Dart-owned copy.
  /// A B200Z_E_DATA result still yields the partial output (the reference keeps it too) with ok == false.
  (Uint8List, bool) grow(int firstCap, int Function(Pointer<Uint8>, int, Pointer<Size>) call) {
    var cap = firstCap < 4096 ? 4096 : firstCap;
    final outLen = calloc<Size>();
    try {
      while (true) {
        final out = hostAlloc(cap);
        try {
          final rc = call(out, cap, outLen);
          if (rc == b200zENoSpc) {
            cap = cap * 2 > outLen.value ? cap * 2 : outLen.value + (outLen.value >> 3);
            continue;
          }
          if (rc == b200zEThrow) throw RangeError(lastError);
          if (rc != b200zOk && rc != b200zEData) throw B200ZException(rc, lastError);
          return (Uint8List.fromList(out.asTypedList(outLen.value)), rc == b200zOk);
        } finally {
          hostFree(out);
        }
      }
    } finally {
      calloc.free(outLen);
    }
  }
}
