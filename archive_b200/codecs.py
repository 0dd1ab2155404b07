"""Host-side mirror of the reference's codec classes (same names, argument meaning and error
behaviour), calling the sm_90a kernels through the C ABI.

Mirrors (paths relative to /root/reference/):
  Inflate            lib/src/codecs/zlib/inflate.dart:12-116
  ZLibDecoder(Web)   lib/src/codecs/zlib_decoder.dart:14-35, codecs/zlib/_zlib_decoder_web.dart:14-107
  GZipDecoder(Web)   lib/src/codecs/gzip_decoder.dart:14-30, codecs/zlib/_gzip_decoder_web.dart:14-58
  inflateBuffer      lib/src/codecs/zlib/inflate_buffer.dart:7
  XZDecoder / XZEncoder  lib/src/codecs/xz_decoder.dart, xz_encoder.dart; getCrc64 lib/src/util/crc64.dart

In the Dart package these classes stay Dart and bind libb200z.so with dart:ffi (dart/, INTEGRATION.md);
no Dart SDK exists in the build image, so the parity tests drive this Python mirror instead.
"""
from __future__ import annotations

import ctypes as C
import os

from . import _ffi
from .streams import BIG_ENDIAN, InputFileStream, InputMemoryStream, OutputFileStream, OutputMemoryStream


def _rest(input):
    """The rest of an input stream as one bytes-like object (InputStream.toUint8List)."""
    if isinstance(input, InputFileStream):
        return input.to_uint8_list()
    return input.buffer[input.position:]


def _consume(input):
    """decodeStream / encodeStream read their input to its end."""
    if isinstance(input, InputFileStream):
        input.skip(max(0, input.length))
    else:
        input.position = len(input.buffer)


def _both_files(input, output) -> bool:
    return isinstance(input, InputFileStream) and isinstance(output, OutputFileStream)


def _file_codec(op: int, input: InputFileStream, output: OutputFileStream, a0: int = 0, a1: int = 0, a2: int = 0) -> int:
    """InputFileStream -> codec -> OutputFileStream without the bytes passing through the host language: the library gets
    the two paths and byte ranges (b200z_file_codec, include/b200z.h; csrc/b200z_file.cu)."""
    L = _ffi.ensure_init()
    path, off, n = input.file_range()
    opath, ooff = output.file_tail()
    used, got = C.c_uint64(0), C.c_uint64(0)
    rc = L.b200z_file_codec(op, os.fsencode(path), off, n, os.fsencode(opath), ooff, a0, a1, a2 & 0xFFFFFFFF,
                            C.byref(used), C.byref(got))
    output.advanced(got.value)
    input.skip(n)
    return rc


def _stream_result(rc: int) -> bool:
    if rc == _ffi.E_DATA:
        return False
    _ffi.check(rc)
    return True


def _grow_call(fn, in_addr, in_len, first_cap):
    """Call fn(out_addr, cap) -> (rc, out_len); retry with a larger buffer on E_NOSPC."""
    cap = max(first_cap, 1 << 12)
    while True:
        out = (C.c_uint8 * cap)()
        rc, n = fn(C.addressof(out), cap)
        if rc == _ffi.E_NOSPC and cap < (1 << 40):
            cap = max(cap * 2, n + (n >> 3))
            continue
        return rc, out, n


class Inflate:
    """`Inflate(bytes)` / `Inflate.stream(input, output:)`: all work happens in the constructor
    (inflate.dart:23-40); bad data never raises -- decoding stops and the partial output is kept
    (inflate.dart:150-151); `RangeError` cases raise DartRangeError."""

    def __init__(self, data=None, output: OutputMemoryStream | None = None, uncompressed_size: int | None = None,
                 _input: InputMemoryStream | None = None):
        self._input = _input if _input is not None else InputMemoryStream(data if data is not None else b"")
        self._output = output if output is not None else OutputMemoryStream(size=uncompressed_size)
        self.status = _ffi.U_EOS
        self._inflate(uncompressed_size)

    @classmethod
    def stream(cls, input: InputMemoryStream | None, output: OutputMemoryStream | None = None,
               uncompressed_size: int | None = None) -> "Inflate":
        return cls(None, output=output, uncompressed_size=uncompressed_size,
                   _input=input if input is not None else InputMemoryStream(b""))

    def _inflate(self, size_hint):
        L = _ffi.ensure_init()
        view = _rest(self._input)
        if len(view) == 0:
            return
        addr, n, keep = _ffi.as_buffer(view)
        out_len, used, ust = C.c_size_t(0), C.c_size_t(0), C.c_int32(0)

        def call(out_addr, cap):
            rc = L.b200z_inflate_raw(addr, n, out_addr, cap, C.byref(out_len), C.byref(used), C.byref(ust))
            return rc, out_len.value

        rc, out, got = _grow_call(call, addr, n, size_hint or 4 * n + 1024)
        self.status = ust.value
        if got:
            self._output.write_bytes(C.string_at(out, got))
        self._input.position += used.value  # (a file stream's setter skips forward)
        _ffi.check(rc)

    def get_bytes(self) -> bytes:
        return self._output.get_bytes()


def inflate_buffer(data) -> bytes:  # inflate_buffer.dart:7 (web variant: Inflate(data).getBytes())
    return Inflate(data).get_bytes()


class _FramedDecoder:
    _fn = None
    _has_raw = True

    def decode_bytes(self, data, verify: bool = False, raw: bool = False) -> bytes:
        """decodeBytes ignores decodeStream's bool and returns whatever was written
        (_gzip_decoder_web.dart:19-24, _zlib_decoder_web.dart:21-28)."""
        out = OutputMemoryStream()
        self.decode_stream(InputMemoryStream(data), out, verify=verify, raw=raw)
        return out.get_bytes()

    def decode_stream(self, input: InputMemoryStream, output: OutputMemoryStream, verify: bool = False,
                      raw: bool = False) -> bool:
        if _both_files(input, output):
            a0 = int(bool(verify)) | (2 if raw and self._file_op == _ffi.FILE_GZIP_DECODE else 0)  # B200Z_GZIP_RAW
            return _stream_result(_file_codec(self._file_op, input, output, a0, int(raw)))
        L = _ffi.ensure_init()
        view = _rest(input)
        addr, n, keep = _ffi.as_buffer(view)
        out_len = C.c_size_t(0)
        rc, out, got = _grow_call(lambda oa, cap: self._call(L, addr, n, verify, raw, oa, cap, out_len),
                                  addr, n, self._first_cap(L, addr, n))
        if got:
            output.write_bytes(C.string_at(out, got))
        _consume(input)
        return _stream_result(rc)


class ZLibDecoderWeb(_FramedDecoder):
    _file_op = _ffi.FILE_ZLIB_DECODE

    def _first_cap(self, L, addr, n):
        return 4 * n + 1024

    def _call(self, L, addr, n, verify, raw, oa, cap, out_len):
        rc = L.b200z_zlib_decode(addr, n, int(verify), int(raw), oa, cap, C.byref(out_len))
        return rc, out_len.value


class GZipDecoderWeb(_FramedDecoder):
    _file_op = _ffi.FILE_GZIP_DECODE

    def _first_cap(self, L, addr, n):
        return L.b200z_gzip_bound(addr, n) or 4 * n + 1024

    def _call(self, L, addr, n, verify, raw, oa, cap, out_len):
        rc = L.b200z_gzip_decode(addr, n, int(bool(verify)) | (2 if raw else 0), oa, cap, C.byref(out_len))  # B200Z_GZIP_RAW
        return rc, out_len.value


# The platform-dispatched names (zlib_decoder.dart:14, gzip_decoder.dart:14) bind the same backend:
# this is the `platformZLibDecoder` / `platformGZipDecoder` seam (_zlib_decoder.dart:1, _gzip_decoder.dart:1).
ZLibDecoder = ZLibDecoderWeb
GZipDecoder = GZipDecoderWeb


class BZip2Decoder:
    """BZip2Decoder().decodeBytes / decodeStream (lib/src/codecs/bzip2_decoder.dart:12-88): CRCs are compared only
    when `verify`; decodeStream returns False on any data error and keeps the blocks decoded before it."""

    def decode_bytes(self, data, verify: bool = False) -> bytes:
        out = OutputMemoryStream()
        self.decode_stream(InputMemoryStream(data), out, verify=verify)
        return out.get_bytes()

    def decode_stream(self, input: InputMemoryStream, output: OutputMemoryStream, verify: bool = False) -> bool:
        if _both_files(input, output):
            return _stream_result(_file_codec(_ffi.FILE_BZIP2_DECODE, input, output, int(verify)))
        L = _ffi.ensure_init()
        view = _rest(input)
        addr, n, keep = _ffi.as_buffer(view)
        out_len = C.c_size_t(0)

        def call(oa, cap):
            rc = L.b200z_bzip2_decode(addr, n, int(verify), oa, cap, C.byref(out_len))
            return rc, out_len.value

        rc, out, got = _grow_call(call, addr, n, 6 * n + 4096)
        if got:
            output.write_bytes(C.string_at(out, got))
        _consume(input)
        return _stream_result(rc)


def bzip2_decode_batch(streams, verify: bool = False, device=None) -> list:
    """BZip2Decoder().decodeBytes(stream, verify:) for every stream of `streams` in one b200z_bzip2_decode_batch call:
    a list of (rc, bytes) in the same order.  rc is what b200z_bzip2_decode gives for that stream alone: OK, E_DATA
    (decodeStream returned false; bytes = the blocks decoded before the failure) or E_THROW (the reference throws a
    RangeError).  Each output room starts at BZip2Decoder's first guess; only the streams that did not fit are decoded
    again, in larger rooms.  device: see gzip_decode_batch."""
    L = _ffi.ensure_init()
    sink = _Sink(device)
    views = [memoryview(s).cast("B") for s in streams]
    n = len(views)
    if n == 0:
        return []
    in_off = (C.c_uint64 * n)()
    in_len = (C.c_uint64 * n)()
    pos = 0
    for i, v in enumerate(views):
        in_off[i], in_len[i] = pos, len(v)
        pos += len(v)
    in_buf = (C.c_uint8 * max(pos, 1))()
    for i, v in enumerate(views):
        C.memmove(C.addressof(in_buf) + in_off[i], bytes(v), len(v))
    rooms = [max(6 * len(v) + 4096, 1 << 12) for v in views]
    result = [None] * n
    todo = list(range(n))
    while todo:
        m = len(todo)
        a_in_off = (C.c_uint64 * m)(*[in_off[i] for i in todo])
        a_in_len = (C.c_uint64 * m)(*[in_len[i] for i in todo])
        a_out_off = (C.c_uint64 * m)()
        a_cap = (C.c_uint64 * m)(*[rooms[i] for i in todo])
        total = 0
        for k in range(m):
            a_out_off[k] = total
            total += sink.room(a_cap[k])
        out, out_addr = sink.alloc(total)
        a_len = (C.c_uint64 * m)()
        a_rc = (C.c_int32 * m)()
        _ffi.check(sink.call(L, "b200z_bzip2_decode_batch", C.addressof(in_buf), a_in_off, a_in_len, m, int(verify), out_addr,
                             a_out_off, a_cap, a_len, a_rc))
        again = []
        for k, i in enumerate(todo):
            rc, got = a_rc[k], a_len[k]
            if rc == _ffi.E_NOSPC and rooms[i] < (1 << 40):
                rooms[i] = max(rooms[i] * 2, got + (got >> 3))
                again.append(i)
                continue
            if rc not in (_ffi.OK, _ffi.E_DATA, _ffi.E_THROW):
                _ffi.check(rc)
            result[i] = (rc, sink.take(out, a_out_off[k], got))
        todo = again
    return result


class BZip2Encoder:
    """BZip2Encoder().encodeBytes / encode / encodeStream (lib/src/codecs/bzip2_encoder.dart:15-81): one "BZh9"
    stream; encodeStream returns True."""

    def encode_bytes(self, data) -> bytes:
        out = OutputMemoryStream()
        self.encode_stream(InputMemoryStream(data), out)
        return out.get_bytes()

    encode = encode_bytes

    def encode_stream(self, input: InputMemoryStream, output: OutputMemoryStream) -> bool:
        if _both_files(input, output):
            _ffi.check(_file_codec(_ffi.FILE_BZIP2_ENCODE, input, output))
            return True
        L = _ffi.ensure_init()
        view = _rest(input)
        addr, n, keep = _ffi.as_buffer(view)
        cap = L.b200z_bzip2_bound(n)
        out = (C.c_uint8 * cap)()
        out_len = C.c_size_t(0)
        _ffi.check(L.b200z_bzip2_encode(addr, n, C.addressof(out), cap, C.byref(out_len)))
        output.write_bytes(C.string_at(out, out_len.value))
        _consume(input)
        return True


class XZCheck:
    """XZCheck (lib/src/codecs/xz_encoder.dart:11): the values are the enum's indices."""
    none, crc32, crc64, sha256 = 0, 1, 2, 3


class XZDecoder:
    """XZDecoder().decodeBytes / decodeStream (lib/src/codecs/xz_decoder.dart:15-27): one stream; block CRC-32 / CRC-64
    checks are compared only when `verify`; decodeStream returns False on a container or check error and keeps what was
    written before it; a Dart throw raises DartRangeError."""

    def decode_bytes(self, data, verify: bool = False) -> bytes:
        out = OutputMemoryStream()
        self.decode_stream(InputMemoryStream(data), out, verify=verify)
        return out.get_bytes()

    def decode_stream(self, input: InputMemoryStream, output: OutputMemoryStream, verify: bool = False) -> bool:
        if _both_files(input, output):
            return _stream_result(_file_codec(_ffi.FILE_XZ_DECODE, input, output, int(verify)))
        L = _ffi.ensure_init()
        view = _rest(input)
        addr, n, keep = _ffi.as_buffer(view)
        out_len = C.c_size_t(0)

        def call(oa, cap):
            rc = L.b200z_xz_decode(addr, n, int(verify), oa, cap, C.byref(out_len))
            return rc, out_len.value

        rc, out, got = _grow_call(call, addr, n, L.b200z_xz_bound(addr, n) + 64)
        if got and rc != _ffi.E_THROW:
            output.write_bytes(C.string_at(out, got))
        _consume(input)
        return _stream_result(rc)


class XZEncoder:
    """XZEncoder().encodeBytes / encode / encodeStream (lib/src/codecs/xz_encoder.dart:18-62): one stored LZMA2 chunk
    (its 16-bit length field is cut for inputs over 64 KiB, as in the reference) and the check, computed on the device."""

    def encode_bytes(self, data, check: int = XZCheck.crc64) -> bytes:
        out = OutputMemoryStream()
        self.encode_stream(InputMemoryStream(data), out, check=check)
        return out.get_bytes()

    encode = encode_bytes

    def encode_stream(self, input: InputMemoryStream, output: OutputMemoryStream, check: int = XZCheck.crc64):
        if _both_files(input, output):
            _ffi.check(_file_codec(_ffi.FILE_XZ_ENCODE, input, output, int(check)))
            return
        L = _ffi.ensure_init()
        view = _rest(input)
        addr, n, keep = _ffi.as_buffer(view)
        cap = L.b200z_xz_encode_bound(n)
        out = (C.c_uint8 * cap)()
        out_len = C.c_size_t(0)
        _ffi.check(L.b200z_xz_encode(addr, n, int(check), C.addressof(out), cap, C.byref(out_len)))
        output.write_bytes(C.string_at(out, out_len.value))
        _consume(input)


def get_crc64(data) -> int:
    """getCrc64 (lib/src/util/crc64.dart, _crc64_io.dart:5-11): ECMA-182 CRC-64, computed on the device."""
    L = _ffi.ensure_init()
    addr, n, keep = _ffi.as_buffer(data)
    crc = C.c_uint64(0)
    _ffi.check(L.b200z_crc64(addr, n, C.byref(crc)))
    return crc.value


class _Sink:
    """Where a decode batch puts its output: host memory (device None: ctypes buffers, results as bytes), or one torch
    CUDA buffer per call on the library's device (results as uint8 views, through the *_to_device entry points)."""

    def __init__(self, device):
        self.torch = None
        if device is None:
            return
        import torch
        dev = torch.device(device)
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        _ffi.ensure_init()
        if dev.type != "cuda" or dev.index != _ffi._inited_device:
            raise ValueError(f"device {device!r} is not the library's CUDA device (cuda:{_ffi._inited_device})")
        self.torch, self.device = torch, dev
        # the caller's current stream; the legacy default stream (handle 0) is passed as cudaStreamLegacy (0x1), because
        # NULL names the library's own stream
        self.stream = torch.cuda.current_stream(dev).cuda_stream or 1

    def room(self, cap):
        """Bytes a slot of `cap` takes in the buffer: device slots start at 16-byte boundaries."""
        return cap if self.torch is None else (cap + 15) & ~15

    def alloc(self, total):
        """(buffer, its address) for `total` bytes of slots."""
        if self.torch is None:
            buf = (C.c_uint8 * max(total, 1))()
            return buf, C.addressof(buf)
        buf = self.torch.empty(max(total, 1), dtype=self.torch.uint8, device=self.device)
        return buf, buf.data_ptr()

    def slots(self, sizes):
        """(buffer, address, out_off, cap) for slots of `sizes` bytes, back to back."""
        n = len(sizes)
        out_off = (C.c_uint64 * n)()
        cap = (C.c_uint64 * n)(*sizes)
        total = 0
        for i in range(n):
            out_off[i] = total
            total += self.room(sizes[i])
        buf, addr = self.alloc(total)
        return buf, addr, out_off, cap

    def call(self, L, name, *args):
        if self.torch is None:
            return getattr(L, name)(*args)
        return getattr(L, name + "_to_device")(*args, self.stream)

    def take(self, buf, off, n):
        if self.torch is None:
            return C.string_at(C.addressof(buf) + off, n)
        return buf[off:off + n]


def _pack(items):
    """bytes-likes -> (ctypes buffer holding them back to back, in_off array, in_len array)."""
    views = [memoryview(s).cast("B") for s in items]
    n = len(views)
    in_off = (C.c_uint64 * n)()
    in_len = (C.c_uint64 * n)()
    pos = 0
    for i, v in enumerate(views):
        in_off[i], in_len[i] = pos, len(v)
        pos += len(v)
    buf = (C.c_uint8 * max(pos, 1))()
    for i, v in enumerate(views):
        C.memmove(C.addressof(buf) + in_off[i], bytes(v), len(v))
    return buf, in_off, in_len


def _slots(sizes):
    n = len(sizes)
    out_off = (C.c_uint64 * n)()
    cap = (C.c_uint64 * n)(*sizes)
    total = 0
    for i in range(n):
        out_off[i] = total
        total += sizes[i]
    return (C.c_uint8 * max(total, 1))(), out_off, cap


def xz_decode_batch(streams, verify: bool = False, device=None) -> list:
    """XZDecoder().decodeBytes(stream, verify:) for every stream of `streams` in one b200z_xz_decode_batch call: a list of
    (rc, bytes) in the same order.  rc is what b200z_xz_decode gives for that stream alone: OK, E_DATA (decodeStream
    returned false; bytes = what was written before it) or E_THROW (the reference throws a RangeError; bytes = the output
    before the chunk that throws).  Each output room is b200z_xz_bound of its stream, which always suffices.
    device: see gzip_decode_batch."""
    L = _ffi.ensure_init()
    sink = _Sink(device)
    n = len(streams)
    if n == 0:
        return []
    in_buf, in_off, in_len = _pack(streams)
    base = C.addressof(in_buf)
    out, out_addr, out_off, cap = sink.slots([L.b200z_xz_bound(base + in_off[i], in_len[i]) for i in range(n)])
    out_len = (C.c_uint64 * n)()
    rc = (C.c_int32 * n)()
    _ffi.check(sink.call(L, "b200z_xz_decode_batch", base, in_off, in_len, n, int(verify), out_addr, out_off, cap, out_len, rc))
    result = []
    for i in range(n):
        if rc[i] not in (_ffi.OK, _ffi.E_DATA, _ffi.E_THROW):
            _ffi.check(rc[i])
        result.append((rc[i], sink.take(out, out_off[i], out_len[i])))
    return result


def xz_encode_batch(contents, check: int = XZCheck.crc64) -> list:
    """XZEncoder().encodeBytes(data, check:) for every input of `contents` in one b200z_xz_encode_batch call: the list of
    encoded streams in the same order, each identical to what XZEncoder gives for that input alone."""
    L = _ffi.ensure_init()
    n = len(contents)
    if n == 0:
        return []
    in_buf, in_off, in_len = _pack(contents)
    out, out_off, cap = _slots([L.b200z_xz_encode_bound(in_len[i]) for i in range(n)])
    out_len = (C.c_uint64 * n)()
    rc = (C.c_int32 * n)()
    _ffi.check(L.b200z_xz_encode_batch(C.addressof(in_buf), in_off, in_len, n, int(check), C.addressof(out), out_off, cap,
                                       out_len, rc))
    result = []
    for i in range(n):
        _ffi.check(rc[i])
        result.append(C.string_at(C.addressof(out) + out_off[i], out_len[i]))
    return result



def _framed_decode_batch(call, streams, first_room, device) -> list:
    """One gzip / zlib decode batch over `streams` -> [(rc, bytes)]; only the streams that got E_NOSPC are decoded
    again, in larger rooms (bzip2_decode_batch's rule).  call(L, sink, base, in_off, in_len, n, out, out_off, cap,
    out_len, rc) makes the call through sink.call."""
    L = _ffi.ensure_init()
    sink = _Sink(device)
    n = len(streams)
    if n == 0:
        return []
    in_buf, in_off, in_len = _pack(streams)
    base = C.addressof(in_buf)
    rooms = [max(first_room(L, base + in_off[i], in_len[i]), 1 << 12) for i in range(n)]
    result = [None] * n
    todo = list(range(n))
    while todo:
        m = len(todo)
        a_in_off = (C.c_uint64 * m)(*[in_off[i] for i in todo])
        a_in_len = (C.c_uint64 * m)(*[in_len[i] for i in todo])
        out, out_addr, out_off, cap = sink.slots([rooms[i] for i in todo])
        out_len = (C.c_uint64 * m)()
        rc = (C.c_int32 * m)()
        _ffi.check(call(L, sink, base, a_in_off, a_in_len, m, out_addr, out_off, cap, out_len, rc))
        again = []
        for k, i in enumerate(todo):
            if rc[k] == _ffi.E_NOSPC and rooms[i] < (1 << 40):
                rooms[i] = max(rooms[i] * 2, out_len[k] + (out_len[k] >> 3))
                again.append(i)
                continue
            if rc[k] not in (_ffi.OK, _ffi.E_DATA, _ffi.E_THROW):
                _ffi.check(rc[k])
            result[i] = (rc[k], sink.take(out, out_off[k], out_len[k]))
        todo = again
    return result


def gzip_decode_batch(streams, verify: bool = False, raw: bool = False, device=None) -> list:
    """GZipDecoder().decodeBytes(stream, verify:, raw:) for every stream of `streams` in one b200z_gzip_decode_batch call:
    a list of (rc, bytes) in the same order.  rc is what b200z_gzip_decode gives for that stream alone: OK, E_DATA
    (decodeStream returned false) or E_THROW (the reference throws a RangeError), with the bytes written before it.
    Rooms start at b200z_gzip_bound (4n + 1024 when that is unknown).

    device: None gives bytes.  A torch CUDA device (the library's) gives [(rc, tensor)] instead: each tensor is a 1-D
    torch.uint8 view of the stream's out_len decoded bytes, inside one CUDA buffer per call (streams decoded again in
    larger rooms get views of that call's buffer).  The decode goes straight into device memory
    (b200z_*_decode_batch_to_device), ordered after the work already on torch.cuda.current_stream(); the tensors are
    ready when the call returns."""
    flags = int(bool(verify)) | (2 if raw else 0)  # B200Z_GZIP_VERIFY | B200Z_GZIP_RAW
    return _framed_decode_batch(lambda L, sink, b, io, il, m, o, oo, cap, ol, rc:
                                sink.call(L, "b200z_gzip_decode_batch", b, io, il, m, flags, o, oo, cap, ol, rc),
                                streams, lambda L, a, n: L.b200z_gzip_bound(a, n) or 4 * n + 1024, device)


def zlib_decode_batch(streams, verify: bool = False, raw: bool = False, device=None) -> list:
    """ZLibDecoder().decodeBytes(stream, verify:, raw:) for every stream of `streams` in one b200z_zlib_decode_batch call:
    a list of (rc, bytes) as gzip_decode_batch gives them, each what b200z_zlib_decode gives for that stream alone.
    device: see gzip_decode_batch."""
    return _framed_decode_batch(lambda L, sink, b, io, il, m, o, oo, cap, ol, rc:
                                sink.call(L, "b200z_zlib_decode_batch", b, io, il, m, int(verify), int(raw), o, oo, cap, ol, rc),
                                streams, lambda L, a, n: 4 * n + 1024, device)


def _framed_encode_batch(call, contents) -> list:
    L = _ffi.ensure_init()
    n = len(contents)
    if n == 0:
        return []
    in_buf, in_off, in_len = _pack(contents)
    out, out_off, cap = _slots([L.b200z_deflate_bound(in_len[i]) + 18 for i in range(n)])
    out_len = (C.c_uint64 * n)()
    rc = (C.c_int32 * n)()
    _ffi.check(call(L, C.addressof(in_buf), in_off, in_len, n, C.addressof(out), out_off, cap, out_len, rc))
    result = []
    for i in range(n):
        _ffi.check(rc[i])
        result.append(C.string_at(C.addressof(out) + out_off[i], out_len[i]))
    return result


def gzip_encode_batch(contents, level: int = 6, mtime: int | None = None) -> list:
    """GZipEncoder().encodeBytes(data, level:) for every input of `contents` in one b200z_gzip_encode_batch call: the
    list of gzip streams in the same order, each identical to what GZipEncoder gives for that input alone with the same
    `mtime` (the wall clock when None, read once for the whole batch)."""
    import time
    mt = int(time.time()) if mtime is None else mtime
    return _framed_encode_batch(lambda L, b, io, il, n, o, oo, cap, ol, rc: L.b200z_gzip_encode_batch(b, io, il, n, level, mt, o, oo,
                                                                                                     cap, ol, rc), contents)


def zlib_encode_batch(contents, level: int = 6, window_bits: int = 15, raw: bool = False) -> list:
    """ZLibEncoder().encodeBytes(data, level:, windowBits:, raw:) for every input of `contents` in one
    b200z_zlib_encode_batch call: the list of streams in the same order, each what ZLibEncoder gives for it alone."""
    return _framed_encode_batch(lambda L, b, io, il, n, o, oo, cap, ol, rc: L.b200z_zlib_encode_batch(b, io, il, n, level, window_bits,
                                                                                                     int(raw), o, oo, cap, ol, rc),
                                contents)


class Deflate:
    """`Deflate(bytes, level: 6, windowBits: 15)` (lib/src/codecs/zlib/deflate.dart:25-100): raw DEFLATE produced in the
    constructor, `get_bytes()` / `take_bytes()`, and `crc32` of the consumed input.  Invalid parameters make the
    reference's `getBytes()` throw LateInitializationError (`_init` returned false, :107-118): B200ZError(E_ARG) here."""

    def __init__(self, data=b"", level: int = 6, window_bits: int = 15, output: OutputMemoryStream | None = None):
        self._output = output if output is not None else OutputMemoryStream()
        self.level = level
        self.crc32 = 0
        L = _ffi.ensure_init()
        addr, n, keep = _ffi.as_buffer(data)
        cap = L.b200z_deflate_bound(n)
        out = (C.c_uint8 * cap)()
        out_len, crc = C.c_size_t(0), C.c_uint32(0)
        rc = L.b200z_deflate_raw(addr, n, level, window_bits, C.addressof(out), cap, C.byref(out_len), C.byref(crc))
        _ffi.check(rc)
        self.crc32 = crc.value
        self._output.write_bytes(C.string_at(out, out_len.value))

    @classmethod
    def stream(cls, input: InputMemoryStream, level: int = 6, window_bits: int = 15, output: OutputMemoryStream | None = None):
        """`Deflate.stream(input, level:, windowBits:, output:)` (deflate.dart:59-67): consumes the rest of `input`."""
        d = cls(_rest(input), level=level, window_bits=window_bits, output=output)
        _consume(input)
        return d

    def finish(self):  # deflate.dart:69 -- everything is already flushed when the constructor returns
        return None

    def get_bytes(self) -> bytes:
        return self._output.get_bytes()

    def take_bytes(self) -> bytes:
        b = self._output.get_bytes()
        self._output.clear()
        return b


class ZLibEncoderWeb:
    """ZLibEncoderWeb().encodeBytes(bytes, level:, windowBits:, raw:) -- _zlib_encoder_web.dart:17-73"""

    def encode_bytes(self, data, level: int | None = None, window_bits: int | None = None, raw: bool = False) -> bytes:
        L = _ffi.ensure_init()
        addr, n, keep = _ffi.as_buffer(data)
        cap = L.b200z_deflate_bound(n)
        out = (C.c_uint8 * cap)()
        out_len = C.c_size_t(0)
        rc = L.b200z_zlib_encode(addr, n, 6 if level is None else level, 15 if window_bits is None else window_bits, int(raw),
                                 C.addressof(out), cap, C.byref(out_len))
        _ffi.check(rc)
        return C.string_at(out, out_len.value)

    def encode_stream(self, input: InputMemoryStream, output: OutputMemoryStream, level: int | None = None,
                      window_bits: int | None = None, raw: bool = False) -> None:
        """_zlib_encoder_web.dart:30-73: the rest of `input` is consumed."""
        if _both_files(input, output):
            _ffi.check(_file_codec(_ffi.FILE_ZLIB_ENCODE, input, output, 6 if level is None else level,
                                   15 if window_bits is None else window_bits, int(raw)))
            return
        output.write_bytes(self.encode_bytes(_rest(input), level=level, window_bits=window_bits, raw=raw))
        _consume(input)


class GZipEncoderWeb:
    """GZipEncoderWeb().encodeBytes(bytes, level:) -- _gzip_encoder_web.dart:17-100.  The reference stamps MTIME with the
    wall clock (:82); pass `mtime` for reproducible bytes."""

    def encode_bytes(self, data, level: int | None = None, mtime: int | None = None) -> bytes:
        import time
        L = _ffi.ensure_init()
        addr, n, keep = _ffi.as_buffer(data)
        cap = L.b200z_deflate_bound(n)
        out = (C.c_uint8 * cap)()
        out_len = C.c_size_t(0)
        rc = L.b200z_gzip_encode(addr, n, 6 if level is None else level, int(time.time()) if mtime is None else mtime,
                                 C.addressof(out), cap, C.byref(out_len))
        _ffi.check(rc)
        return C.string_at(out, out_len.value)

    def encode_stream(self, input: InputMemoryStream, output: OutputMemoryStream, level: int | None = None,
                      mtime: int | None = None) -> None:
        """_gzip_encoder_web.dart:30-100: the rest of `input` is consumed."""
        if _both_files(input, output):
            import time
            _ffi.check(_file_codec(_ffi.FILE_GZIP_ENCODE, input, output, 6 if level is None else level, 0,
                                   int(time.time()) if mtime is None else mtime))
            return
        output.write_bytes(self.encode_bytes(_rest(input), level=level, mtime=mtime))
        _consume(input)


ZLibEncoder = ZLibEncoderWeb
GZipEncoder = GZipEncoderWeb
