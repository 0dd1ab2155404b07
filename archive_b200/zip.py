"""Host mirror of the reference's ZIP reader for the H100 path (SURVEY.md 8f2): `ZipDecoder().decode_bytes(data)` ->
`Archive` of `ArchiveFile`s, as lib/src/codecs/zip_decoder.dart:18-81 builds it.  The directory is parsed by
b200z_zip_list (ZipDirectory / ZipFileHeader / ZipFile.read), and -- this is the point of the batching -- ALL members are
decompressed by ONE b200z_zip_extract call (every deflate member is a unit of the same inflate batch) instead of one
Inflate per member on first access (zip_file.dart:201-248).  With a password, ZipCrypto and WinZip AES members are
decrypted on the device in the same call (b200z_zip_extract_password)."""
from __future__ import annotations

import ctypes as C

from . import _ffi

U_DONE, U_EOS, U_STOP, U_NOSPC, U_THROW = 0, 1, -1, -2, -5
ZIP_ENCRYPTED, ZIP_TOO_LARGE, ZIP_BAD_PASSWORD, ZIP_BAD_MAC = -20, -21, -22, -23
CRYPT_NONE, CRYPT_ZIPCRYPTO, CRYPT_AES = 0, 1, 2
COMPRESSION = {0: "none", 8: "deflate", 12: "bzip2"}  # zip_file.dart:36-40; anything else is read as "none" (:83)


class ArchiveException(Exception):
    """util/archive_exception.dart: what the reference throws when an encrypted member cannot be read."""


def password_bytes(password) -> bytes | None:
    """The bytes the reference hashes / feeds the ZipCrypto keys: Dart's `codeUnits` (UTF-16 code units) cut to 8 bits
    (zip_file.dart:264-266, 350).  Python strings iterate code points, so the string goes through UTF-16 first."""
    if password is None:
        return None
    if isinstance(password, str):
        return password.encode("utf-16-le")[::2]
    return bytes(password)


_CRYPT_ERRORS = {ZIP_BAD_PASSWORD: "password error", ZIP_BAD_MAC: "macs don't match",
                 U_THROW: "encrypted member too short for its header, or an empty password (Dart: RangeError)"}


def _name(raw: bytes) -> str:
    try:  # InputStream.readString: UTF-8, falling back to one char per byte (input_stream.dart:140-149)
        return raw.decode("utf-8")
    except UnicodeDecodeError:
        return raw.decode("latin-1")


class ArchiveFile:
    """archive_file.dart:14-130 (the fields ZipDecoder and TarDecoder fill)."""

    def __init__(self, name: str, size: int, is_file: bool = True):
        self.name, self.size, self.is_file = name, size, is_file
        self.mode = 0o644
        self.owner_id = self.group_id = 0
        self.crc32 = None
        self.last_mod_time = 0
        self.compression = None
        self.symbolic_link = None
        self.content = b"" if is_file else None
        self.status = U_DONE  # unit status of the member's decode (include/b200z.h)
        self.encrypted = False  # decrypted with a password (the errors below are then the reference's throws)
        self._computed_crc32 = None  # ZipFile._computedCrc32: set by a device extract, else computed on first use

    @property
    def is_symbolic_link(self):
        return bool(self.symbolic_link)

    def read_bytes(self):
        if self.encrypted and self.status in _CRYPT_ERRORS:  # ZipFile.getStream throws on access (zip_file.dart:333-341)
            raise ArchiveException(f"{self.name}: {_CRYPT_ERRORS[self.status]}")
        return self.content

    def verify_crc32(self) -> bool:
        """ZipFile.verifyCrc32 (zip_file.dart:157-161): getCrc32 of the content against `crc32`.  Content extracted to a
        device carries the CRC its extract call computed there; host content is hashed with b200z_crc32."""
        data = self.read_bytes()
        if self._computed_crc32 is None:
            data = bytes(data or b"")
            crc = C.c_uint32(0)
            if data:
                L = _ffi.ensure_init()
                addr, n, keep = _ffi.as_buffer(data)
                _ffi.check(L.b200z_crc32(addr, n, C.byref(crc)))
            self._computed_crc32 = crc.value
        return self._computed_crc32 == self.crc32


class Archive:
    """archive.dart:6-60: files in directory order; a later entry with a name already present replaces the earlier."""

    def __init__(self):
        self.files, self._index = [], {}

    def find(self, name):
        i = self._index.get(name)
        return None if i is None else self.files[i]

    def add(self, f: ArchiveFile):
        i = self._index.get(f.name)
        if i is not None:
            self.files[i] = f
            return
        self._index[f.name] = len(self.files)
        self.files.append(f)

    def __iter__(self):
        return iter(self.files)

    def __len__(self):
        return len(self.files)


class ZipDecoder:
    def __init__(self, web_eos: bool = False, split_flush_points: bool = True):
        # web_eos: the pure-Dart Inflate's end-of-stream behaviour (SURVEY Q1); default is what the Dart VM's ZipDecoder
        # gives (dart:io zlib): a member's last symbols are always decoded
        self.flags = (1 if web_eos else 0) | (0 if split_flush_points else 2)
        self.entries = []
        self.zip_file_comment = ""

    def list(self, data):
        L = _ffi.lib()
        addr, n, keep = _ffi.as_buffer(data)
        cnt = C.c_size_t(0)
        _ffi.check(L.b200z_zip_list(addr, n, None, 0, C.byref(cnt)))
        ents = (_ffi.ZipEntry * max(1, cnt.value))()
        _ffi.check(L.b200z_zip_list(addr, n, ents, cnt.value, C.byref(cnt)))
        self.entries = [ents[i] for i in range(cnt.value)]
        off, clen = C.c_uint64(0), C.c_uint32(0)
        _ffi.check(L.b200z_zip_comment(addr, n, C.byref(off), C.byref(clen)))
        raw = bytes(memoryview(data)[off.value:off.value + clen.value]) if clen.value else b""
        self.zip_file_comment = raw.decode("latin-1")  # readString(utf8: false) (zip_directory.dart:43)
        return ents, cnt.value

    def decode_stream(self, input, verify: bool = False, password=None, device=None) -> Archive:
        """ZipDecoder().decodeStream(input) (zip_decoder.dart:29-81): the rest of an InputMemoryStream or InputFileStream."""
        from .streams import InputFileStream
        if isinstance(input, InputFileStream):
            data = input.to_uint8_list()
            input.skip(len(data))
        else:
            data = bytes(input.buffer[input.position:])
            input.position = len(input.buffer)
        return self.decode_bytes(data, verify=verify, password=password, device=device)

    def crypt_info(self, data, entry):
        """-> (mode CRYPT_*, AES strength byte, method the content is stored with), as ZipFile.read decides
        (b200z_zip_crypt_info); raises DartRangeError where the reference's extra-field scan throws."""
        L = _ffi.lib()
        addr, n, keep = _ffi.as_buffer(data)
        mode, strength, method = C.c_uint32(), C.c_uint32(), C.c_uint32()
        _ffi.check(L.b200z_zip_crypt_info(addr, n, C.byref(entry), C.byref(mode), C.byref(strength), C.byref(method)))
        return mode.value, strength.value, method.value

    def decode_bytes(self, data, verify: bool = False, password=None, device=None) -> Archive:
        """password: str (Dart's code units cut to 8 bits, see password_bytes) or bytes.  Without one, encrypted members
        keep status ZIP_ENCRYPTED and empty content.  verify does nothing, as in the reference (its check is commented
        out); ArchiveFile.verify_crc32 makes it.
        device: None (content is bytes), or the library's torch CUDA device: every member goes straight into one CUDA
        buffer per call (b200z_zip_extract_to_device, ordered after torch.cuda.current_stream()), each file's content is a
        uint8 tensor view into it, and the member CRC-32s are computed there.  Any other device raises ValueError."""
        data = bytes(data) if not isinstance(data, (bytes, bytearray)) else data
        pw = password_bytes(password)
        ents, n = self.list(data)
        contents, statuses, crcs = self._extract(data, ents, n, pw, device)
        archive = Archive()
        for i in range(n):
            e = ents[i]
            name = _name(data[e.name_off:e.name_off + e.name_len]) if e.has_data else ""
            is_dir = name.endswith("/") or name.endswith("\\")
            entry = archive.find(name)
            if entry is None:
                entry = ArchiveFile(name, 0, is_file=False) if is_dir else ArchiveFile(name, e.uncomp_size if e.has_data else 0)
                method = e.method
                if e.has_data and (e.flags & 1):  # an AES member names its real method in its extra record (:125-127)
                    try:
                        method = self.crypt_info(data, e)[2]
                    except _ffi.B200ZError:
                        pass
                entry.compression = COMPRESSION.get(method, "none") if e.has_data else "none"
                if not is_dir:
                    entry.content, entry.status, entry._computed_crc32 = contents[i], statuses[i], crcs[i]
                    entry.encrypted = pw is not None and bool(e.has_data and (e.flags & 1))
                archive.add(entry)
            entry.mode = e.ext_attr >> 16
            if (e.version_made_by >> 8) == 3 and (entry.mode & 0xF000) == 0xA000:  # unix symlink (:58-70)
                if pw is not None and e.has_data and (e.flags & 1) and statuses[i] in _CRYPT_ERRORS:
                    # decodeStream reads a symlink's content while it walks the directory: the throw happens here
                    raise ArchiveException(f"{name}: {_CRYPT_ERRORS[statuses[i]]}")
                try:  # (a device member's target is read back: the walk needs it on the host)
                    target = contents[i] if device is None else bytes(contents[i].cpu().numpy())
                    entry.symbolic_link = target.decode("utf-8")
                except UnicodeDecodeError:
                    pass
            entry.crc32 = e.crc32
            entry.last_mod_time = (e.mod_date << 16) | e.mod_time
        return archive

    def _extract(self, data, ents, n, password=None, device=None):
        """-> (contents, statuses, crcs): crcs[i] is the member's CRC-32 when the device call computed it, else None."""
        from .codecs import _Sink
        sink = _Sink(device)
        if n == 0:
            return [], [], []
        L = _ffi.ensure_init()
        addr, zlen, keep = _ffi.as_buffer(data)
        room = [max(int(ents[i].hint_uncomp_size), int(ents[i].uncomp_size), 1) if ents[i].has_data else 0 for i in range(n)]
        contents, statuses, crcs = [b""] * n, [U_DONE] * n, [None] * n
        if sink.torch is not None:
            contents = [sink.torch.empty(0, dtype=sink.torch.uint8, device=sink.device)] * n
        todo = list(range(n))
        while todo:
            m = len(todo)
            sub = (_ffi.ZipEntry * m)(*[ents[i] for i in todo])
            off, tot = [], 0
            for i in todo:
                off.append(tot)
                tot += (room[i] + 63) & ~63 if sink.torch is None else sink.room(room[i])
            out, out_addr = sink.alloc(tot)
            a64 = lambda l: (C.c_uint64 * m)(*l)
            out_len, st = (C.c_uint64 * m)(), (C.c_int32 * m)()
            crc = None
            if sink.torch is None:
                _ffi.check(L.b200z_zip_extract_password(addr, zlen, sub, m, out_addr, max(tot, 1), a64(off),
                                                        a64([room[i] for i in todo]), out_len, st, self.flags, password,
                                                        len(password or b"")))
            else:
                crc = (C.c_uint32 * m)()
                _ffi.check(L.b200z_zip_extract_to_device(addr, zlen, sub, m, out_addr, max(tot, 1), a64(off),
                                                         a64([room[i] for i in todo]), out_len, st, crc, self.flags,
                                                         password, len(password or b""), sink.stream))
            again = []
            for k, i in enumerate(todo):
                statuses[i] = st[k]
                if st[k] == U_NOSPC and room[i] < (1 << 32) - 64:  # the size fields lied: the data decide (grow and retry)
                    room[i] = min(max(room[i] * 4, int(out_len[k]), int(ents[i].comp_size) * 4), (1 << 32) - 64)
                    again.append(i)
                    continue
                contents[i] = sink.take(out, off[k], min(int(out_len[k]), room[i]))
                if crc is not None:
                    crcs[i] = crc[k]
            todo = again
        return contents, statuses, crcs


# ---------------------------------------------------------------------------------------------
# ZipEncoder (lib/src/codecs/zip_encoder.dart:66-583)
# ---------------------------------------------------------------------------------------------
def _dos_time(t):  # _getTime :33-40
    t1 = ((t.tm_min & 0x7) << 5) | (t.tm_sec // 2)
    t2 = (t.tm_hour << 3) | (t.tm_min >> 3)
    return ((t2 & 0xFF) << 8) | (t1 & 0xFF)


def _dos_date(t):  # _getDate :42-49
    d1 = ((t.tm_mon & 0x7) << 5) | t.tm_mday
    d2 = (((t.tm_year - 1980) & 0x7F) << 1) | (t.tm_mon >> 3)
    return ((d2 & 0xFF) << 8) | (d1 & 0xFF)


def _b200_compress(content: bytes, method: str, level: int):
    """-> (payload, crc32 of content): the member's data as the reference produces it -- raw DEFLATE through
    platformZLibEncoder.encodeStream(raw: true) (:244-249), BZip2Encoder (:250-255) or the bytes themselves -- on the device."""
    L = _ffi.ensure_init()
    addr, n, keep = _ffi.as_buffer(content)
    crc = C.c_uint32(0)
    if method == "deflate":
        cap = L.b200z_deflate_bound(n)
        out = (C.c_uint8 * cap)()
        out_len = C.c_size_t(0)
        _ffi.check(L.b200z_deflate_raw(addr, n, level, 15, C.addressof(out), cap, C.byref(out_len), C.byref(crc)))
        return C.string_at(out, out_len.value), crc.value
    _ffi.check(L.b200z_crc32(addr, n, C.byref(crc)))
    if method == "bzip2":
        cap = L.b200z_bzip2_bound(n)
        out = (C.c_uint8 * cap)()
        out_len = C.c_size_t(0)
        _ffi.check(L.b200z_bzip2_encode(addr, n, C.addressof(out), cap, C.byref(out_len)))
        return C.string_at(out, out_len.value), crc.value
    return bytes(content), crc.value


def deflate_batch(contents, level: int = 6, window_bits: int = 15):
    """Raw DEFLATE of every item of `contents` with ONE b200z_deflate_batch call (all inputs staged at once, several members in
    flight on the device) -> list of (payload, crc32).  Each payload equals Deflate(item, level:, windowBits:).getBytes()."""
    import numpy as np
    L = _ffi.ensure_init()
    n = len(contents)
    if n == 0:
        return []
    in_len = np.array([len(c) for c in contents], dtype=np.uint64)
    in_off = np.zeros(n, dtype=np.uint64)
    in_off[1:] = np.cumsum(in_len)[:-1]
    blob = b"".join(bytes(c) for c in contents)
    addr, nb, keep = _ffi.as_buffer(blob if blob else b"\0")
    out_cap = np.array([L.b200z_deflate_bound(int(x)) for x in in_len], dtype=np.uint64)
    out_off = np.zeros(n, dtype=np.uint64)
    out_off[1:] = np.cumsum(out_cap)[:-1]
    out = np.empty(int(out_cap.sum()), dtype=np.uint8)
    out_len = np.zeros(n, dtype=np.uint64)
    crc = np.zeros(n, dtype=np.uint32)
    status = np.zeros(n, dtype=np.int32)
    p = lambda a: a.ctypes.data
    _ffi.check(L.b200z_deflate_batch(addr, p(in_off), p(in_len), n, level, window_bits, p(out), p(out_off), p(out_cap),
                                     p(out_len), p(crc), p(status)))
    assert not status.any(), "b200z_deflate_bound is an upper bound"
    return [(out[int(out_off[i]):int(out_off[i] + out_len[i])].tobytes(), int(crc[i])) for i in range(n)]


def bzip2_encode_batch(contents):
    """BZip2 of every item of `contents` with ONE b200z_bzip2_encode_batch call (all inputs staged at once, blocks of
    different items sorted and coded together) -> list of (payload, crc32).  Each payload equals
    BZip2Encoder().encodeBytes(item); crc32 is getCrc32(item), computed on the device."""
    import numpy as np
    L = _ffi.ensure_init()
    n = len(contents)
    if n == 0:
        return []
    in_len = np.array([len(c) for c in contents], dtype=np.uint64)
    in_off = np.zeros(n, dtype=np.uint64)
    in_off[1:] = np.cumsum(in_len)[:-1]
    blob = b"".join(bytes(c) for c in contents)
    addr, nb, keep = _ffi.as_buffer(blob if blob else b"\0")
    out_cap = np.array([L.b200z_bzip2_bound(int(x)) for x in in_len], dtype=np.uint64)
    out_off = np.zeros(n, dtype=np.uint64)
    out_off[1:] = np.cumsum(out_cap)[:-1]
    out = np.empty(int(out_cap.sum()), dtype=np.uint8)
    out_len = np.zeros(n, dtype=np.uint64)
    crc = np.zeros(n, dtype=np.uint32)
    status = np.zeros(n, dtype=np.int32)
    p = lambda a: a.ctypes.data
    _ffi.check(L.b200z_bzip2_encode_batch(addr, p(in_off), p(in_len), n, p(out), p(out_off), p(out_cap), p(out_len),
                                          p(crc), p(status)))
    assert not status.any(), "b200z_bzip2_bound is an upper bound"
    return [(out[int(out_off[i]):int(out_off[i] + out_len[i])].tobytes(), int(crc[i])) for i in range(n)]


def aes_encrypt_batch(payloads, salts, password: bytes):
    """ZipEncoder._encryptCompressedData (zip_encoder.dart:166-183) for every payload at once: ONE b200z_zip_aes_encrypt call
    (key derivation, AES-256-CTR and the MAC on the device) -> list of (ciphertext, verifier, mac)."""
    import numpy as np
    L = _ffi.ensure_init()
    n = len(payloads)
    if n == 0:
        return []
    ln = np.array([len(p) for p in payloads], dtype=np.uint64)
    off = np.zeros(n, dtype=np.uint64)
    off[1:] = np.cumsum(ln)[:-1]
    buf = bytearray(b"".join(bytes(p) for p in payloads) or b"\0")
    addr, nb, keep = _ffi.as_buffer(buf)
    salt = b"".join(salts)
    assert len(salt) == 16 * n
    ver, mac = (C.c_uint8 * (2 * n))(), (C.c_uint8 * (10 * n))()
    _ffi.check(L.b200z_zip_aes_encrypt(addr, off.ctypes.data, ln.ctypes.data, n, salt, password, len(password), ver, mac))
    data = bytes(keep)
    return [(data[int(off[i]):int(off[i] + ln[i])], bytes(ver[2 * i:2 * i + 2]), bytes(mac[10 * i:10 * i + 10])) for i in range(n)]


class ZipEncoder:
    """`ZipEncoder().encode_bytes(archive, level: 1, modified:)` (zip_encoder.dart:66-121): local headers + data, central
    directory, (zip64) end records, written field by field as `_writeFile` :309-372 and `_writeCentralDirectory` :391-497 do.
    Members are compressed on the device (`compress` exists so that the CPU test tier can check the container logic with a
    stand-in).  Not mirrored: encryption, and passing already-compressed members through (`file.isCompressed`, :214-235) --
    the ArchiveFile of this package holds content, not the source archive's bytes.

    With `password` (ZipEncoder(password:), :166-183, 270-310, 347-437) every member is AES-256 encrypted as the reference
    writes it: all payloads go through ONE b200z_zip_aes_encrypt call, and the container keeps the reference's quirks --
    method 99, flag bit 0 and an AE-1 record on every entry, directories included; the verifier and MAC of the last
    encrypted member stay with the encoder, so a directory after a file gets compressedSize 12 and that file's MAC (10 bytes)
    behind its local header."""

    VERSION = 20

    def __init__(self, compress=None, batch: bool = False, password=None, salt=None, encrypt=None):
        """batch=True: all deflate members go to the device in one b200z_deflate_batch call per level (several members in
        flight) instead of one b200z_deflate_raw call each, and all bzip2 members in one b200z_bzip2_encode_batch call;
        the archive bytes are the same.  password: str or bytes (see
        password_bytes); salt: callable returning each member's 16 salt bytes (default os.urandom, as Random.secure);
        encrypt: stand-in for aes_encrypt_batch (the CPU test tier)."""
        import os
        self._compress = compress or _b200_compress
        self._batch = batch and compress is None
        self._password = password_bytes(password)
        self._salt = salt or (lambda: os.urandom(16))
        self._encrypt = encrypt or aes_encrypt_batch

    def encode_bytes(self, archive, level: int = 1, modified=None, comment: str = "") -> bytes:
        import struct
        import time
        out = bytearray()
        files = []
        archive = list(archive)
        compress = self._compress
        def level_of(e):  # add(file, level: ...) overrides the encoder's level for that member (zip_encoder.dart:137-183)
            own = getattr(e, "compress_level", None)
            return own if own is not None else (level if level is not None else 6)

        if self._batch:
            idx = [i for i, e in enumerate(archive) if e.is_file and (e.compression or "deflate") == "deflate"]
            table = {}
            for lv in sorted({level_of(archive[i]) for i in idx}):  # one device batch per level in use
                grp = [i for i in idx if level_of(archive[i]) == lv]
                table.update(zip(grp, deflate_batch([archive[i].content or b"" for i in grp], lv)))
            grp = [i for i, e in enumerate(archive) if e.is_file and e.compression == "bzip2"]
            table.update(zip(grp, bzip2_encode_batch([archive[i].content or b"" for i in grp])))
            at = [None]

            def compress(content, method, level_):
                return table[at[0]] if method in ("deflate", "bzip2") else self._compress(content, method, level_)
        pw = self._password
        payloads = []
        for pos_in_archive, entry in enumerate(archive):
            if self._batch:
                at[0] = pos_in_archive
            method = (entry.compression or "deflate") if entry.is_file else "deflate"
            payloads.append(compress(entry.content or b"", method, level_of(entry)) if entry.is_file else None)
        sealed = {}
        if pw is not None:  # _encryptCompressedData for every file, in one device call
            if not pw:
                raise _ffi.DartRangeError(_ffi.E_THROW, "ZipEncoder: empty password (ZipFile.deriveKey returns an empty list)")
            idx = [i for i, p in enumerate(payloads) if p is not None]
            salts = {i: bytes(self._salt()) for i in idx}
            sealed = dict(zip(idx, ((salts[i],) + r for i, r in zip(idx, self._encrypt([payloads[i][0] for i in idx],
                                                                                      [salts[i] for i in idx], pw)))))
        last_ver = last_mac = None  # _pwdVer / _mac: fields of the encoder, they outlive the member they belong to
        for pos_in_archive, entry in enumerate(archive):
            lm = time.localtime(modified if modified is not None else entry.last_mod_time)  # DateTime.fromMillisecondsSinceEpoch
            name = entry.name.replace("\\", "/")
            if not entry.is_file and not name.endswith("/"):
                name += "/"
            method = (entry.compression or "deflate") if entry.is_file else "deflate"
            payload, crc = payloads[pos_in_archive] or (b"", 0)
            head = tail = b""
            if pos_in_archive in sealed:
                salt, payload, last_ver, last_mac = sealed[pos_in_archive]
                head = salt + last_ver
            if pw is not None and last_mac is not None:
                tail = last_mac
            # dataLen (:283-286): data + salt (files only) + the encoder's current MAC and verifier, whoever they belong to
            csize = len(payload) + (16 if pos_in_archive in sealed else 0) + (12 if tail else 0)
            fd = dict(name=name, time=_dos_time(lm), date=_dos_date(lm), crc=crc, csize=csize,
                      usize=entry.size if entry.is_file else 0, method=method, mode=entry.mode, pos=len(out),
                      comment=getattr(entry, "comment", None) or "")
            files.append(fd)
            # _writeFile
            z64 = fd["csize"] > 0xFFFFFFFF or fd["usize"] > 0xFFFFFFFF
            extra = struct.pack("<BBBBQQ", 1, 0, 0x10, 0, fd["usize"], fd["csize"]) if z64 else b""
            m = {"deflate": 8, "bzip2": 12}.get(method, 0)
            if pw is not None:
                extra += self._aes_extra(m)
            nb = name.encode("utf-8")
            out += struct.pack("<IHHHHHIIIHH", 0x04034B50, self.VERSION, 0x801 if pw is not None else 0x800,
                               99 if pw is not None else m, fd["time"], fd["date"], crc,
                               0xFFFFFFFF if z64 else fd["csize"], 0xFFFFFFFF if z64 else fd["usize"], len(nb), len(extra))
            out += nb + extra + head + payload + tail
        # _writeCentralDirectory
        cd_pos = len(out)
        any64 = False
        for fd in files:
            z64 = fd["csize"] > 0xFFFFFFFF or fd["usize"] > 0xFFFFFFFF or fd["pos"] > 0xFFFFFFFF
            any64 |= z64
            extra = struct.pack("<BBBBQQQ", 1, 0, 0x18, 0, fd["usize"], fd["csize"], fd["pos"]) if z64 else b""
            m = {"deflate": 8, "bzip2": 12}.get(fd["method"], 0)
            if pw is not None:
                extra += self._aes_extra(m)
            nb, cb = fd["name"].encode("utf-8"), fd["comment"].encode("utf-8")
            out += struct.pack("<IHHHHHHIIIHHHHHII", 0x02014B50, (0 << 8) | self.VERSION, self.VERSION,
                               0x801 if pw is not None else 0x800, 99 if pw is not None else m, fd["time"],
                               fd["date"], fd["crc"], 0xFFFFFFFF if z64 else fd["csize"], 0xFFFFFFFF if z64 else fd["usize"],
                               len(nb), len(extra), len(cb), 0, 0, (fd["mode"] << 16) & 0xFFFFFFFF,
                               0xFFFFFFFF if z64 else fd["pos"])
            out += nb + extra + cb
        cd_size = len(out) - cd_pos
        n = len(files)
        need64 = any64 or n > 0xFFFF or cd_size > 0xFFFFFFFF or cd_pos > 0xFFFFFFFF
        if need64:
            eocd64 = len(out)
            out += struct.pack("<IQHHIIQQQQ", 0x06064B50, 0x2C, 0x2D, 0x2D, 0, 0, n, n, cd_size, cd_pos)
            out += struct.pack("<IIQI", 0x07064B50, 0, eocd64, 1)
        cb = (comment or "").encode("utf-8")
        out += struct.pack("<IHHHHIIH", 0x06054B50, 0, 0xFFFF if need64 else 0, 0xFFFF if need64 else n,
                           0xFFFF if need64 else n, 0xFFFFFFFF if need64 else cd_size, 0xFFFFFFFF if need64 else cd_pos, len(cb))
        out += cb
        return bytes(out)

    @staticmethod
    def _aes_extra(method_id: int) -> bytes:  # _getAexExtraData :347-363: AE-1, vendor "AE", strength 3 (256 bits)
        import struct
        return struct.pack("<HHH2sBH", 0x9901, 7, 1, b"AE", 3, method_id)

    encode = encode_bytes
