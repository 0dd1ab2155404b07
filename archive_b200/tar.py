"""TAR container: `TarDecoder` / `TarEncoder` / `TarFile`, restated from lib/src/codecs/tar_decoder.dart,
lib/src/codecs/tar_encoder.dart and lib/src/codecs/tar/tar_file.dart field by field.

The container is host work: one 512-byte header per member, the content sliced out of the tar stream.  For archives whose
members should end up on the GPU, `tar_decode_batch(..., device=...)` and `TarDecoder.decode_bytes(..., device=...)` run
the member walk there instead (b200z_tar_walk_device): only the headers come back, and each file stays a view into the
decoded device buffer.  The hot path of a
tarball is the compression around it, which runs on the device -- `GZipDecoder` / `BZip2Decoder` / `XZDecoder` for one
tarball, `gzip_decode_batch` / `bzip2_decode_batch` / `xz_decode_batch` for many shards in one call:

    archives = [TarDecoder().decode_bytes(tar) for rc, tar in gzip_decode_batch(shards)]

and `GZipEncoder` (the library's file entry point) inside `TarFileEncoder.tar_directory` (io.py).

The reference's quirks are kept, since archives written or read with it depend on them: the walk stops at two zero
bytes, not a zero block; numeric fields that Dart's `int.parse(radix: 8)` rejects (GNU base-256, garbage) read as 0;
the header checksum is never checked; a `././@LongLink` entry names the next member whatever its type flag; the writer
emits V7 headers (no `ustar` magic) and sizes a long-name entry by the name's UTF-16 length."""
from __future__ import annotations

import ctypes as C
import re

from . import _ffi
from ._ffi import E_THROW, DartRangeError
from .streams import InputFileStream, OutputMemoryStream
from .zip import Archive, ArchiveFile

# Dart's String.trim() (tar_file.dart:233-236): the Unicode White_Space characters and U+FEFF.  Python's str.strip()
# differs: it also strips \x1c-\x1f and keeps U+FEFF.
_DART_WS = "\t\n\x0b\x0c\r \x85\xa0\u1680" + "".join(map(chr, range(0x2000, 0x200b))) + "\u2028\u2029\u202f\u205f\u3000\ufeff"
# int.parse(s, radix: 8) (tar_file.dart:218): an optional sign and ASCII octal digits, nothing else.  Python's int(s, 8)
# also takes `_` separators, a `0o` prefix, inner whitespace and non-ASCII digits.
_DART_OCTAL = re.compile(r"[+-]?[0-7]+")
# paxRecordRegexp (tar_decoder.dart:9), `(\d+) (\w+)=(.*)` with Dart's (JavaScript) classes: \d and \w are ASCII, and `.`
# stops at \r, U+2028 and U+2029 as well as \n.
_PAX_RECORD = re.compile("([0-9]+) ([A-Za-z0-9_]+)=([^\r\n\u2028\u2029]*)")

LONG_LINK = "././@LongLink"


def _dart_string(raw: bytes) -> str:
    """utf8.decode with the fallback to one character per byte (tar_file.dart:231-237, input_stream.dart:141-149)."""
    try:
        return raw.decode("utf-8")
    except UnicodeDecodeError:
        return raw.decode("latin-1")


def _parse_string(field: bytes) -> str:
    """_parseString (tar_file.dart:227-239): cut at the first NUL, decode, trim."""
    r = field.find(0)
    return _dart_string(field if r < 0 else field[:r]).strip(_DART_WS)


def _parse_int(field: bytes) -> int:
    """_parseInt (tar_file.dart:211-225): any string int.parse rejects reads as 0."""
    s = _parse_string(field)
    return int(s, 8) if _DART_OCTAL.fullmatch(s) else 0


def _write_string(out: bytearray, value: str, width: int):
    """_writeString (tar_file.dart:241-248): the UTF-8 bytes cut to the field, zero-filled -- no NUL is guaranteed."""
    b = value.encode("utf-8")[:width]
    out += b + bytes(width - len(b))


def _write_int(out: bytearray, value: int, width: int):
    """_writeInt (tar_file.dart:250-256): toRadixString(8) (a '-' for negatives, zeros put in front of it), padded to
    width-1 digits; a longer number keeps its leading digits and loses the NUL."""
    _write_string(out, format(value, "o").rjust(width - 1, "0"), width)


class _Input:
    """The InputMemoryStream operations TarFile.read and TarDecoder use (input_memory_stream.dart, input_stream.dart)."""

    def __init__(self, data):
        self.data, self.pos = data, 0

    @property
    def is_eos(self):
        return self.pos >= len(self.data)

    def read_bytes(self, count: int) -> bytes:
        """readBytes (input_stream.dart:132-136) -> subset (input_memory_stream.dart:111-119): clipped to what is left; a
        negative count is a negative Uint8List.view length, which throws a RangeError (:26)."""
        if count < 0:
            raise DartRangeError(E_THROW, f"tar: negative field length {count} at byte {self.pos} (Dart: RangeError)")
        b = bytes(self.data[self.pos:self.pos + count])
        self.pos += len(b)
        return b

    def skip(self, count: int):
        """skip (input_memory_stream.dart:96-100): clamped to the buffer."""
        self.pos = min(max(self.pos + count, 0), len(self.data))


class TarFile:
    """TarFile (tar_file.dart:34-257): one header and its content."""
    NORMAL_FILE, HARD_LINK, SYMBOLIC_LINK, CHAR_SPEC, BLOCK_SPEC, DIRECTORY, FIFO, CONT_FILE = "01234567"
    G_EX_HEADER, G_EX_HEADER2, EX_HEADER, EX_HEADER2 = "g", "G", "x", "X"

    def __init__(self):  # the field defaults of :52-68
        self.filename = ""
        self.mode = 644  # decimal, as the reference has it (:53)
        self.owner_id = self.group_id = self.file_size = self.last_mod_time = self.checksum = 0
        self.type_flag = "0"
        self.name_of_linked_file = None
        self.ustar_indicator = self.ustar_version = self.owner_user_name = self.owner_group_name = ""
        self.device_major_number = self.device_minor_number = 0
        self.filename_prefix = ""
        self.raw_content = None  # bytes read from the archive (rawContent)
        self.content_bytes = None  # bytes, or an InputFileStream, to write (contentBytes / content)

    @classmethod
    def read(cls, input: _Input, store_data: bool = True) -> "TarFile":
        """TarFile.read (:74-118)."""
        t = cls.from_header(input.read_bytes(512))  # a short header reads as if the missing bytes were absent fields
        if store_data or t.filename == LONG_LINK:  # (:104-108)
            t.raw_content = input.read_bytes(t.file_size)
        else:
            input.skip(t.file_size)
        if t.is_file and t.file_size > 0:  # padding only for "files" with content (:110-117)
            rem = t.file_size % 512
            if rem:
                input.skip(512 - rem)
        return t

    @classmethod
    def from_header(cls, h: bytes) -> "TarFile":
        """The fields TarFile.read parses from a header (:76-103), with no content read.  Header bytes past a short
        header's end read as absent, whether they are missing or zero."""
        t = cls()
        t.filename = _parse_string(h[0:100])
        t.mode = _parse_int(h[100:108])
        t.owner_id = _parse_int(h[108:116])
        t.group_id = _parse_int(h[116:124])
        t.file_size = _parse_int(h[124:136])
        t.last_mod_time = _parse_int(h[136:148])
        t.checksum = _parse_int(h[148:156])  # read, never checked, with or without `verify`
        t.type_flag = _parse_string(h[156:157])
        t.name_of_linked_file = _parse_string(h[157:257])
        t.ustar_indicator = _parse_string(h[257:263])
        if t.ustar_indicator == "ustar":  # also GNU's "ustar " once trimmed (:92)
            t.ustar_version = _parse_string(h[263:265])
            t.owner_user_name = _parse_string(h[265:297])
            t.owner_group_name = _parse_string(h[297:329])
            t.device_major_number = _parse_int(h[329:337])
            t.device_minor_number = _parse_int(h[337:345])
            t.filename_prefix = _parse_string(h[345:500])
            if t.filename_prefix:
                t.filename = f"{t.filename_prefix}/{t.filename}"
        return t

    @property
    def is_file(self) -> bool:  # (:120): links, FIFOs and devices count as files
        return self.type_flag != TarFile.DIRECTORY

    @property
    def is_sym_link(self) -> bool:  # (:122)
        return self.type_flag == TarFile.SYMBOLIC_LINK

    @property
    def size(self) -> int:
        return self.file_size

    @property
    def content(self):
        return self.content_bytes if self.content_bytes is not None else self.raw_content

    def __repr__(self):
        return f"[{self.filename}, {self.mode}, {self.file_size}]"

    def write(self, output):
        """TarFile.write (:144-209): a V7 header (nothing from byte 257 on), the content, zero padding."""
        h = bytearray()
        _write_string(h, self.filename, 100)
        _write_int(h, self.mode, 8)
        _write_int(h, self.owner_id, 8)
        _write_int(h, self.group_id, 8)
        _write_int(h, self.file_size, 12)
        _write_int(h, self.last_mod_time, 12)
        _write_string(h, " " * 8, 8)  # checksum placeholder
        _write_string(h, self.type_flag, 1)
        _write_string(h, self.name_of_linked_file or "", 100)
        h += bytes(512 - len(h))
        # 6 octal digits, NUL, space (:171-190)
        h[148:154] = format(sum(h), "o").rjust(6, "0")[:6].encode()
        h[154], h[155] = 0, 32
        output.write_bytes(h)
        c = self.content
        if isinstance(c, InputFileStream):
            output.write_stream(c)
        elif c is not None:
            output.write_bytes(c)
        if self.is_file and self.file_size > 0:  # padding by the header's size, whatever was written (:200-208)
            rem = self.file_size % 512
            if rem:
                output.write_bytes(bytes(512 - rem))


class TarDecoder:
    """TarDecoder (tar_decoder.dart:12-129).  `files` keeps every member header in order; the returned `Archive` holds
    one entry per name (a later member replaces an earlier one of the same name, archive.dart:19-31).

    Errors, where the reference throws: a negative size field (RangeError), a PAX `x` record block that is not UTF-8
    (FormatException), and a PAX `x` header when `store_data` is False (its content is null) -- all DartRangeError."""

    def __init__(self):
        self.files: list[TarFile] = []

    def decode_bytes(self, data, verify: bool = False, store_data: bool = True, callback=None, device=None) -> Archive:
        """decodeBytes (:18-22).  `verify` is accepted and ignored, as in the reference.

        device: None walks the members on the host.  The library's torch CUDA device walks them there
        (b200z_tar_walk_device): `data` is bytes-like (uploaded once) or a 1-D uint8 CUDA tensor (walked where it is), and
        each file's content is a uint8 tensor view into it -- see tar_decode_batch, of which this is the batch of one.
        store_data=False raises ValueError with a device: there a negative size moves the walk backwards, which the device
        walk does not do."""
        if device is not None:
            if not store_data:
                raise ValueError("TarDecoder.decode_bytes: store_data=False has no device walk")
            from .codecs import _Sink
            sink = _Sink(device)
            result = _decode_on_device(sink, _to_device(sink, [data]), [self], callback)[0]
            if isinstance(result, DartRangeError):
                raise result
            return result
        if not isinstance(data, (bytes, bytearray, memoryview)):
            data = bytes(data)
        inp = _Input(memoryview(data).cast("B"))
        return self._decode(_host_walk(inp, store_data), store_data, callback)

    def decode_stream(self, input, verify: bool = False, store_data: bool = True, callback=None) -> Archive:
        """decodeStream (:24-128) on the rest of an InputMemoryStream or InputFileStream; the stream is left where the walk
        stopped.  A file stream is read to its end and walked as memory: the walks differ only for a negative size field,
        which throws here for both."""
        if isinstance(input, InputFileStream):
            inp = _Input(input.to_uint8_list())
            archive = self._decode(_host_walk(inp, store_data), store_data, callback)
            input.skip(inp.pos)
            return archive
        inp = _Input(input.buffer[input.position:])
        try:
            return self._decode(_host_walk(inp, store_data), store_data, callback)
        finally:
            input.position += inp.pos

    def _decode(self, members, store_data: bool, callback) -> Archive:
        """The member loop (:28-127) over `members`, the TarFiles of a walk in order, contents read: the host walk
        (_host_walk) or the records of the device walk (_decode_on_device).  A walk that throws raises from the iterator
        once the members before the throw are through the loop."""
        archive = Archive()
        self.files = []
        next_name = next_link_name = None
        for tf in members:
            if tf.filename == LONG_LINK:  # any type flag, 'K' included (:43-46)
                raw = tf.raw_content
                r = raw.find(0)
                next_name = _dart_string(raw if r < 0 else raw[:r])  # readString(): to the first NUL, no trim
                continue
            if tf.type_flag in (TarFile.G_EX_HEADER, TarFile.G_EX_HEADER2):  # (:51-55)
                continue
            if tf.type_flag in (TarFile.EX_HEADER, TarFile.EX_HEADER2):  # (:56-76)
                if tf.raw_content is None:
                    raise DartRangeError(E_THROW, "tar: PAX header read without its data (Dart: null check on rawContent)")
                try:
                    text = tf.raw_content.decode("utf-8")
                except UnicodeDecodeError as e:
                    raise DartRangeError(E_THROW, f"tar: PAX record block is not UTF-8 (Dart: FormatException): {e}") from None
                for record in text.split("\n"):
                    m = _PAX_RECORD.search(record)  # unanchored; the length prefix is never checked
                    if m is None:
                        continue
                    if m.group(2) == "path":
                        next_name = m.group(3)
                    elif m.group(2) == "linkpath":
                        next_link_name = m.group(3)
                continue
            if next_name is not None:  # (:78-86)
                tf.filename, next_name = next_name, None
            if next_link_name is not None:
                tf.name_of_linked_file, next_link_name = next_link_name, None
            self.files.append(tf)
            if tf.is_file:  # (:91-108)
                if store_data:  # ArchiveFile.stream: size is what was read, which a truncated archive cuts short
                    f = ArchiveFile(tf.filename, len(tf.raw_content))
                    f.content = tf.raw_content
                else:  # ArchiveFile.noData
                    f = ArchiveFile(tf.filename, 0)
                    f.content = None
            else:  # ArchiveFile.directory (:109-124)
                f = ArchiveFile(tf.filename, 0, is_file=False)
            f.mode, f.owner_id, f.group_id, f.last_mod_time = tf.mode, tf.owner_id, tf.group_id, tf.last_mod_time
            # always set after a read ('' when the header has none), so a hard link's target reads as a symbolic link
            f.symbolic_link = tf.name_of_linked_file
            archive.add(f)
            if callback is not None:
                callback(f)
        return archive


def _host_walk(input: _Input, store_data: bool):
    """The walk of TarDecoder._decode (:28-38): the TarFiles of `input` in order, `input` left where the walk stopped."""
    data = input.data
    while not input.is_eos:
        p = input.pos
        if len(data) - p < 2 or (data[p] == 0 and data[p + 1] == 0):  # two bytes, not a zero block (:35-38)
            break
        yield TarFile.read(input, store_data)


_TAR_MEMBER = None  # the numpy dtype of b200z_tar_member


def _to_device(sink, shards) -> list:
    """Archives as 1-D uint8 tensors on the sink's device: CUDA tensors as they are (no copy), everything else (bytes-like,
    or what bytes() takes) packed into one host buffer and uploaded with one copy."""
    torch = sink.torch
    out, host = [None] * len(shards), []
    for i, s in enumerate(shards):
        if isinstance(s, torch.Tensor):
            if s.device != sink.device or s.dtype != torch.uint8 or s.dim() != 1 or not s.is_contiguous():
                raise ValueError(f"tar: shard {i} is not a contiguous 1-D uint8 tensor on {sink.device}")
            out[i] = s
        else:  # anything else bytes() takes, as on the host path (a list of ints, ...)
            host.append((i, memoryview(s if isinstance(s, (bytes, bytearray, memoryview)) else bytes(s)).cast("B")))
    if host:
        packed = bytearray(sum(len(v) for _, v in host))
        at, spans = 0, []
        for i, v in host:
            packed[at:at + len(v)] = v
            spans.append((i, at, len(v)))
            at += len(v)
        buf = torch.frombuffer(packed, dtype=torch.uint8).to(sink.device) if packed else \
            torch.empty(0, dtype=torch.uint8, device=sink.device)
        for i, a, n in spans:
            out[i] = buf[a:a + n]
    return out


def _walk_on_device(sink, archives):
    """One b200z_tar_walk_device call over the archive tensors -> (first, count, rc, records, headers).  The records
    array starts at a guess of one member per 2 KiB and is sized exactly after an E_NOSPC."""
    import numpy as np
    global _TAR_MEMBER
    if _TAR_MEMBER is None:
        _TAR_MEMBER = np.dtype([(f, "<u8") for f in ("header_off", "content_off", "content_len")] +
                               [("size", "<i8"), ("header_len", "<u4"), ("pad_", "<u4")])
    L = _ffi.ensure_init()
    n = len(archives)
    lens = [t.numel() for t in archives]
    live = [t.data_ptr() for t in archives if t.numel()]
    base = min(live) if live else 0  # archives from separate allocations: offsets are pointer differences
    off = (C.c_uint64 * n)(*[t.data_ptr() - base if t.numel() else 0 for t in archives])
    ln = (C.c_uint64 * n)(*lens)
    first, count, rc, n_total = (C.c_uint64 * n)(), (C.c_uint64 * n)(), (C.c_int32 * n)(), C.c_size_t()
    cap = min(sum(x // 512 + 1 for x in lens), sum(lens) // 2048 + n)
    while True:
        records, headers = np.empty(max(cap, 1), _TAR_MEMBER), np.empty(max(cap, 1) * 512, np.uint8)
        r = L.b200z_tar_walk_device(base, off, ln, n, records.ctypes.data, headers.ctypes.data, cap, first, count, rc,
                                    C.byref(n_total), sink.stream)
        if r != _ffi.E_NOSPC:
            _ffi.check(r)
            return first, count, rc, records, headers
        cap = n_total.value


def _decode_on_device(sink, archives, decoders, callback=None) -> list:
    """decoders[i]._decode of archives[i] (1-D uint8 tensors on the sink's device) with the walk on the device -> for
    each, its Archive or the DartRangeError the host walk raises.  The headers are parsed on the host; the contents of
    LongLink and PAX entries, which the loop reads, come back together in one gather and one copy."""
    first, count, rc, records, headers = _walk_on_device(sink, archives)
    members, wanted = [], []
    for i, t in enumerate(archives):
        tfs = []
        for k in range(first[i], first[i] + count[i]):
            m = records[k]
            tf = TarFile.from_header(headers[512 * k:512 * k + int(m["header_len"])].tobytes())
            a, ln = int(m["content_off"]), int(m["content_len"])
            tf.raw_content = t[a:a + ln]
            if tf.filename == LONG_LINK or tf.type_flag in (TarFile.EX_HEADER, TarFile.EX_HEADER2):
                wanted.append(tf)
            tfs.append(tf)
        members.append(tfs)
    if wanted:
        blob = sink.torch.cat([tf.raw_content for tf in wanted]).cpu().numpy().tobytes()
        at = 0
        for tf in wanted:
            n = tf.raw_content.numel()
            tf.raw_content, at = blob[at:at + n], at + n
    out = []
    for i, (tfs, dec) in enumerate(zip(members, decoders)):
        try:
            out.append(dec._decode(_device_members(tfs, rc[i], count[i]), True, callback))
        except DartRangeError as e:
            out.append(e)
    return out


def _device_members(tfs, rc, count):
    yield from tfs
    if rc == E_THROW:  # the walk stopped at a negative size field: readBytes' RangeError
        raise DartRangeError(E_THROW, f"tar: negative size field in member {count} (Dart: RangeError)")
    _ffi.check(rc)


def tar_decode_batch(shards, compression=None, verify: bool = False, device=None) -> list:
    """TarDecoder().decodeBytes of every shard's decoded bytes -> [(rc, Archive or DartRangeError)] in shard order.
    compression: None (plain .tar), "gzip", "bzip2" or "xz"; the shards are decoded in one codec batch call
    (gzip_decode_batch, bzip2_decode_batch, xz_decode_batch with `verify`) and rc is that call's rc for the shard (OK for
    plain shards).  A damaged shard's partial output is walked as it is.  Where TarDecoder would raise DartRangeError for
    a shard, the error is returned in its place, so one bad shard does not cost the batch.

    device: None decodes and walks on the host side of the library (the recipe
    `[TarDecoder().decode_bytes(t) for rc, t in gzip_decode_batch(shards)]`).  The library's torch CUDA device decodes
    straight into device memory (the codec's *_decode_batch_to_device, or one upload of plain shards; plain shards that
    are already contiguous 1-D uint8 CUDA tensors are walked where they are), walks every member of every shard in one
    b200z_tar_walk_device call, and gives each file's content as a uint8 tensor view into that memory.  The calls are
    ordered after torch.cuda.current_stream(), and the tensors are ready when the call returns.  Any other device raises
    ValueError."""
    from . import codecs
    batch = {None: None, "gzip": codecs.gzip_decode_batch, "bzip2": codecs.bzip2_decode_batch, "xz": codecs.xz_decode_batch}
    if compression not in batch:
        raise ValueError(f"tar_decode_batch: unknown compression {compression!r}")
    shards = list(shards)
    if device is None:
        decoded = [(_ffi.OK, s) for s in shards] if compression is None else batch[compression](shards, verify=verify)
        out = []
        for rc, t in decoded:
            try:
                out.append((rc, TarDecoder().decode_bytes(t)))
            except DartRangeError as e:
                out.append((rc, e))
        return out
    sink = codecs._Sink(device)
    if not shards:
        return []
    if compression is None:
        decoded = [(_ffi.OK, t) for t in _to_device(sink, shards)]
    else:
        decoded = batch[compression](shards, verify=verify, device=sink.device)
    results = _decode_on_device(sink, [t for _, t in decoded], [TarDecoder() for _ in decoded])
    return [(rc, r) for (rc, _), r in zip(decoded, results)]


class TarEncoder:
    """TarEncoder (tar_encoder.dart:12-91)."""

    def __init__(self):
        self._output = None

    def encode_stream(self, archive, output):  # (:17-23)
        self.start(output)
        for f in archive:
            self.add(f)
        self.finish()

    def encode_bytes(self, archive, output=None) -> bytes:  # (:25-29)
        output = OutputMemoryStream() if output is None else output
        self.encode_stream(archive, output)
        return output.get_bytes() if isinstance(output, OutputMemoryStream) else output.subset(0)

    encode = encode_bytes

    def start(self, output=None):  # (:35-37)
        self._output = OutputMemoryStream() if output is None else output

    def add(self, entry: ArchiveFile):
        """add (:39-76).  A name longer than 100 UTF-16 code units is written first as a `././@LongLink` entry of type
        '0' whose size is that count while its content is the name's UTF-8 bytes: the two differ for non-ASCII names, as
        in the reference.  A file whose `symbolic_link` is not None -- '' included -- is written as a link with no
        content; a symbolic link is type '2' and a directory type '5', both of size 0."""
        if self._output is None:
            return
        units = len(entry.name.encode("utf-16-le")) // 2  # Dart's String.length
        if units > 100:
            ts = TarFile()
            ts.filename = LONG_LINK
            ts.file_size = units
            ts.mode = 0
            ts.content_bytes = entry.name.encode("utf-8")
            ts.write(self._output)
        ts = TarFile()
        ts.filename = entry.name
        ts.mode, ts.owner_id, ts.group_id, ts.last_mod_time = entry.mode, entry.owner_id, entry.group_id, entry.last_mod_time
        if not entry.is_file:
            ts.type_flag = TarFile.DIRECTORY
        elif entry.symbolic_link is not None:
            ts.type_flag = TarFile.SYMBOLIC_LINK
            ts.name_of_linked_file = entry.symbolic_link
        else:
            ts.file_size = entry.size
            ts.content_bytes = entry.read_bytes()
        ts.write(self._output)

    def finish(self):  # (:78-88): two zero blocks
        if self._output is None:
            return
        self._output.write_bytes(bytes(1024))
        self._output.flush()
        self._output = None
