"""archive_b200 -- H100 (sm_90a) implementation of the Inflate/Deflate and BZip2 block-codec hot path
of the Dart `archive` package, behind the package's own class names, with its ZIP and TAR containers.  See DESIGN.md."""
from ._ffi import B200ZError, DartRangeError, LIB_PATH  # noqa: F401
from .codecs import BZip2Decoder, BZip2Encoder, Deflate, GZipDecoder, GZipEncoder, GZipEncoderWeb, ZLibEncoder, ZLibEncoderWeb, GZipDecoderWeb, Inflate, ZLibDecoder, ZLibDecoderWeb, inflate_buffer  # noqa: F401
from .codecs import XZCheck, XZDecoder, XZEncoder, bzip2_decode_batch, get_crc64, xz_decode_batch, xz_encode_batch  # noqa: F401
from .codecs import gzip_decode_batch, gzip_encode_batch, zlib_decode_batch, zlib_encode_batch  # noqa: F401
from .streams import BIG_ENDIAN, LITTLE_ENDIAN, InputFileStream, InputMemoryStream, OutputFileStream, OutputMemoryStream  # noqa: F401
from .zip import Archive, ArchiveFile, ZipDecoder, ZipEncoder, bzip2_encode_batch  # noqa: F401,E402
from .tar import TarDecoder, TarEncoder, TarFile, tar_decode_batch  # noqa: F401,E402
from .io import TarFileEncoder, ZipFileEncoder, extract_archive_to_disk, extract_file_to_disk, get_input_extension  # noqa: F401,E402
