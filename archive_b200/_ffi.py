"""ctypes binding of libb200z.so (include/b200z.h).

This is the Python stand-in for the `dart:ffi` binding a maintainer of the reference would add
(dart/lib/src/b200z_ffi.dart, INTEGRATION.md): same symbols, same argument meaning.  The library is
the product; there is NO CPU fallback -- if the shared object is missing or no H100 is visible every
codec call raises.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200Z_LIB") or os.path.join(_HERE, "libb200z.so")

OK, E_NODEVICE, E_ARG, E_NOSPC, E_DATA, E_THROW, E_INTERNAL = 0, -1, -2, -3, -4, -5, -6
FILE_GZIP_DECODE, FILE_ZLIB_DECODE, FILE_BZIP2_DECODE, FILE_ZLIB_ENCODE, FILE_GZIP_ENCODE, FILE_BZIP2_ENCODE = 1, 2, 3, 4, 5, 6
FILE_XZ_DECODE, FILE_XZ_ENCODE = 7, 8
U_DONE, U_EOS, U_STOP, U_NOSPC, U_RANGE, U_BADCODE, U_THROW, U_TOKCAP = 0, 1, -1, -2, -3, -4, -5, -6


class B200ZError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"b200z error {code}: {msg}")
        self.code = code


class DartRangeError(B200ZError):
    """The reference would have thrown (RangeError / LateInitializationError) at this point."""


_lib = None
_lock = threading.Lock()
_u8p = C.POINTER(C.c_uint8)

class Bz2Block(C.Structure):
    """b200z_bz2_block (include/b200z.h)"""
    _fields_ = [("start_bit", C.c_uint64), ("end_bit", C.c_uint64), ("out_bytes", C.c_uint64), ("crc_calc", C.c_uint32),
                ("crc_stored", C.c_uint32), ("status", C.c_int32), ("flags", C.c_uint32)]


class ZipEntry(C.Structure):
    """b200z_zip_entry (include/b200z.h)"""
    _fields_ = [("local_header_off", C.c_uint64), ("data_off", C.c_uint64), ("comp_size", C.c_uint64),
                ("uncomp_size", C.c_uint64), ("hint_uncomp_size", C.c_uint64), ("name_off", C.c_uint64),
                ("cd_name_off", C.c_uint64), ("name_len", C.c_uint32), ("cd_name_len", C.c_uint32), ("crc32", C.c_uint32),
                ("method", C.c_uint32), ("flags", C.c_uint32), ("mod_time", C.c_uint32), ("mod_date", C.c_uint32),
                ("ext_attr", C.c_uint32), ("version_made_by", C.c_uint32), ("has_data", C.c_uint32)]


class TarMember(C.Structure):
    """b200z_tar_member (include/b200z.h)"""
    _fields_ = [("header_off", C.c_uint64), ("content_off", C.c_uint64), ("content_len", C.c_uint64), ("size", C.c_int64),
                ("header_len", C.c_uint32), ("pad_", C.c_uint32)]


_SIGS = {
    "b200z_init": (C.c_int, [C.c_int, C.c_uint32]),
    "b200z_shutdown": (None, []),
    "b200z_last_error": (C.c_char_p, []),
    "b200z_device_count": (C.c_int, []),
    "b200z_version": (C.c_char_p, []),
    "b200z_host_alloc": (C.c_void_p, [C.c_size_t]),
    "b200z_host_free": (None, [C.c_void_p]),
    "b200z_launch_count": (C.c_uint64, []),
    "b200z_profile_enable": (None, [C.c_int]),
    "b200z_profile_read": (C.c_int, [C.POINTER(C.c_double)] * 3 + [C.POINTER(C.c_uint64)]),
    "b200z_inflate_raw": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t),
                                    C.POINTER(C.c_size_t), C.POINTER(C.c_int32)]),
    "b200z_gzip_decode": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "b200z_zlib_decode": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                    C.POINTER(C.c_size_t)]),
    "b200z_gzip_bound": (C.c_size_t, [C.c_void_p, C.c_size_t]),
    "b200z_deflate_raw": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t),
                                    C.POINTER(C.c_uint32)]),
    "b200z_deflate_bound": (C.c_size_t, [C.c_size_t]),
    "b200z_deflate_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200z_zlib_encode": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                    C.POINTER(C.c_size_t)]),
    "b200z_gzip_encode": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.c_uint32, C.c_void_p, C.c_size_t,
                                    C.POINTER(C.c_size_t)]),
    "b200z_bzip2_decode": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "b200z_bzip2_decode_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200z_crc32": (C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_uint32)]),
    "b200z_xz_decode": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "b200z_xz_bound": (C.c_size_t, [C.c_void_p, C.c_size_t]),
    "b200z_xz_encode": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "b200z_xz_encode_bound": (C.c_size_t, [C.c_size_t]),
    "b200z_crc64": (C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64)]),
    "b200z_gzip_decode_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200z_zlib_decode_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200z_gzip_encode_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_uint32, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200z_zlib_encode_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200z_xz_decode_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200z_xz_encode_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p]),
    # the decode batches with their output slots in device memory, plus the caller's cudaStream_t
    "b200z_gzip_decode_batch_to_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p,
                                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200z_zlib_decode_batch_to_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p,
                                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200z_bzip2_decode_batch_to_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p,
                                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200z_xz_decode_batch_to_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p,
                                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200z_zip_list": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "b200z_zip_comment": (C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]),
    "b200z_zip_extract": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]),
    "b200z_zip_crypt_info": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                       C.POINTER(C.c_uint32)]),
    "b200z_zip_extract_password": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t]),
    # b200z_zip_extract_password with its slots in device memory, plus the member CRC-32s and the caller's cudaStream_t
    "b200z_zip_extract_to_device": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                              C.c_size_t, C.c_void_p]),
    # the TAR member walk over archives in device memory, plus the caller's cudaStream_t
    "b200z_tar_walk_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_size_t), C.c_void_p]),
    "b200z_zip_aes_encrypt": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t,
                                        C.c_void_p, C.c_void_p]),
    "b200z_bzip2_decode_shard": (C.c_int, [C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t,
                                           C.POINTER(C.c_size_t), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "b200z_bzip2_encode": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "b200z_bzip2_bound": (C.c_size_t, [C.c_size_t]),
    "b200z_bzip2_encode_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200z_file_codec": (C.c_int, [C.c_int, C.c_char_p, C.c_uint64, C.c_uint64, C.c_char_p, C.c_uint64, C.c_int32, C.c_int32,
                                   C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "b200z_file_last_stats": (None, [C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    "b200z_inflate_batch": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "b200z_inflate_workspace_bytes": (C.c_size_t, [C.c_size_t, C.c_size_t, C.c_size_t]),
    "b200z_inflate_batch_device": (C.c_int, [C.c_void_p] * 9 + [C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    # several GPUs driven by this one process
    "b200z_multi_init": (C.c_int, [C.c_uint32, C.c_uint32]),
    "b200z_multi_shutdown": (None, []),
    "b200z_multi_device_count": (C.c_int, []),
    "b200z_gzip_decode_multi": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t),
                                          C.c_uint32]),
    "b200z_inflate_batch_multi": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32]),
    "b200z_multi_device_output": (C.c_void_p, [C.c_int, C.POINTER(C.c_size_t)]),
}


def declared_symbols():
    """Every entry point include/b200z.h declares (checked by the CPU-side ABI test)."""
    return sorted(_SIGS)


def lib():
    """Load libb200z.so (no device needed to load; compute calls need b200z_init)."""
    global _lib
    with _lock:
        if _lib is None:
            if "_emu" in os.path.basename(LIB_PATH) and os.environ.get("B200Z_EMU_TESTS") != "1":
                # tests/host_emul/libb200z_emu.so is the test tier's host build of these sources: never a codec backend
                raise B200ZError(E_NODEVICE, f"{LIB_PATH} is the test suite's emulation build, not the product library")
            if not os.path.exists(LIB_PATH):
                raise B200ZError(E_NODEVICE, f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; "
                                 "g.build()'` (there is no CPU fallback)")
            L = C.CDLL(LIB_PATH)
            for name, (res, args) in _SIGS.items():
                if not hasattr(L, name):
                    continue  # later rounds add symbols; the ABI test reports what is missing
                f = getattr(L, name)
                f.restype = res
                f.argtypes = args
            _lib = L
    return _lib


_inited_device = None


def ensure_init(device: int | None = None):
    global _inited_device
    L = lib()
    if device is None:
        device = int(os.environ.get("LOCAL_RANK", "0")) if _inited_device is None else _inited_device
    if _inited_device == device:
        return L
    rc = L.b200z_init(device, 0)
    if rc != OK:
        raise B200ZError(rc, L.b200z_last_error().decode())
    _inited_device = device
    return L


def last_error() -> str:
    return lib().b200z_last_error().decode()


def check(rc: int):
    if rc == OK:
        return
    msg = last_error()
    if rc == E_THROW:
        raise DartRangeError(rc, msg)
    raise B200ZError(rc, msg)


def as_buffer(data):
    """bytes-like -> (ctypes address, length, keepalive)."""
    if isinstance(data, (bytes, bytearray)):
        buf = (C.c_uint8 * len(data)).from_buffer_copy(data) if isinstance(data, bytes) else (C.c_uint8 * len(data)).from_buffer(data)
        return C.addressof(buf), len(data), buf
    mv = memoryview(data).cast("B")
    if mv.readonly:
        buf = (C.c_uint8 * len(mv)).from_buffer_copy(mv)
    else:
        buf = (C.c_uint8 * len(mv)).from_buffer(mv)
    return C.addressof(buf), len(mv), buf
