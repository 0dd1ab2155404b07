"""ctypes access to the TAR part of oracle/liboracle.so (oracle/tar.c) -- TEST INFRASTRUCTURE (checker only)."""
import ctypes as C
from dataclasses import dataclass

from oracle_lib import L, OK, THROW  # noqa: F401


class _Member(C.Structure):
    _fields_ = [(f, C.c_int64) for f in ("mode", "uid", "gid", "size", "mtime", "checksum", "devmajor", "devminor")] + \
               [(f, C.c_uint64) for f in ("name_off", "name_len", "link_off", "link_len", "type_off", "type_len", "magic_off",
                                          "magic_len", "uname_off", "uname_len", "gname_off", "gname_len")] + \
               [("content_off", C.c_int64), ("content_len", C.c_int64), ("is_file", C.c_int32), ("archive_index", C.c_int32)]


class _EntryIn(C.Structure):
    _fields_ = [("name", C.c_char_p), ("symlink", C.c_char_p), ("content", C.c_char_p), ("content_len", C.c_size_t),
                ("size", C.c_int64), ("mode", C.c_int64), ("uid", C.c_int64), ("gid", C.c_int64), ("mtime", C.c_int64),
                ("is_file", C.c_int)]


@dataclass
class Member:
    """One TarFile of TarDecoder.files as the oracle reads it."""
    name: str
    link: str
    type_flag: str
    mode: int
    uid: int
    gid: int
    size: int
    mtime: int
    checksum: int
    magic: str
    uname: str
    gname: str
    devmajor: int
    devminor: int
    content: bytes | None  # None: no data was read (store_data off)
    is_file: bool
    archive_index: int  # slot in the Archive, -1 when a later member of the same name replaced it


def decode(data: bytes, store_data: bool = True):
    """TarDecoder().decodeBytes(data, storeData:) -> (status OK | THROW, [Member]).  On THROW the list holds the members
    decoded before the throw."""
    data = bytes(data)
    n, cap = C.c_size_t(), 1024
    while True:
        arr = (_Member * cap)()
        strs, slen = C.POINTER(C.c_uint8)(), C.c_size_t()
        st = L().orc_tar_decode(data, C.c_size_t(len(data)), int(store_data), arr, C.c_size_t(cap), C.byref(n),
                                C.byref(strs), C.byref(slen))
        block = C.string_at(strs, slen.value)
        L().orc_free(strs)
        if n.value <= cap:
            break
        cap = n.value
    s = lambda off, ln: block[off:off + ln].decode("utf-8")  # noqa: E731
    out = []
    for m in arr[:n.value]:
        out.append(Member(s(m.name_off, m.name_len), s(m.link_off, m.link_len), s(m.type_off, m.type_len), m.mode, m.uid,
                          m.gid, m.size, m.mtime, m.checksum, s(m.magic_off, m.magic_len), s(m.uname_off, m.uname_len),
                          s(m.gname_off, m.gname_len), m.devmajor, m.devminor,
                          None if m.content_len < 0 else data[m.content_off:m.content_off + m.content_len], bool(m.is_file),
                          m.archive_index))
    return st, out


def archive_order(members):
    """The Archive TarDecoder returns: the members holding a slot, in slot order."""
    return sorted((m for m in members if m.archive_index >= 0), key=lambda m: m.archive_index)


def encode(entries) -> bytes:
    """TarEncoder().encodeBytes over entries: dicts with name, and optionally content (bytes or None), size (default
    len(content)), symlink (str or None), is_file (default True), mode (default 0o644), uid, gid, mtime."""
    arr = (_EntryIn * max(1, len(entries)))()
    keep = []
    for i, e in enumerate(entries):
        name = e["name"].encode("utf-8")
        link = None if e.get("symlink") is None else e["symlink"].encode("utf-8")
        content = e.get("content")
        keep += [name, link, content]
        arr[i] = _EntryIn(name, link, content, len(content or b""), e.get("size", len(content or b"")), e.get("mode", 0o644),
                          e.get("uid", 0), e.get("gid", 0), e.get("mtime", 0), int(e.get("is_file", True)))
    out, n = C.POINTER(C.c_uint8)(), C.c_size_t()
    st = L().orc_tar_encode(arr, C.c_size_t(len(entries)), C.byref(out), C.byref(n))
    assert st == OK
    r = C.string_at(out, n.value)
    L().orc_free(out)
    return r
