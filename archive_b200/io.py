"""The on-disk side of the codec path (SURVEY.md 8f4): the reference's lib/src/io/extract_archive_to_disk.dart and
lib/src/io/tar_file_encoder.dart, for what this package decodes and encodes.  `extract_file_to_disk` runs the GZip / BZip2 /
XZ stage of a compressed tar file -> file through the library's file entry point (b200z_file_codec: the bytes never pass
through the host language), and unpacks .zip archives whose members were all decompressed by one device batch.  For
.tar.gz / .tgz / .tar.bz2 / .tbz / .tar.xz / .txz it stops at the decompressed .tar in `output_path`, where the reference
goes on to untar it; `extract_archive_to_disk(TarDecoder().decode_bytes(...), out)` unpacks a tar archive.
`TarFileEncoder` writes a .tar or, through the same file entry point on the device, a .tar.gz."""
from __future__ import annotations

import os
import shutil
import tempfile
import time

from .codecs import BZip2Decoder, GZipDecoder, GZipEncoder, XZDecoder
from .streams import InputFileStream, OutputFileStream
from .tar import TarEncoder
from .zip import Archive, ArchiveFile, ZipDecoder


def _is_within_output_path(output_dir: str, file_path: str) -> bool:
    """_isWithinOutputPath (:19-22): path.isWithin(canonicalize(outputDir), canonicalize(filePath)) -- strictly inside."""
    out, fp = os.path.realpath(output_dir), os.path.realpath(file_path)
    return fp != out and os.path.commonpath([out, fp]) == out


def _is_valid_sym_link(output_path: str, f: ArchiveFile) -> bool:
    """_isValidSymLink (:24-38): no absolute targets, no targets outside the output directory."""
    file_dir = os.path.dirname(os.path.join(output_path, os.path.normpath(f.name)))
    link = os.path.normpath(f.symbolic_link or "")
    if os.path.isabs(link):
        return False
    return _is_within_output_path(output_path, os.path.normpath(os.path.join(file_dir, link)))


def _prepare_archive_file_path(f: ArchiveFile, output_path: str):
    """_prepareArchiveFilePath (:47-62)"""
    file_path = os.path.join(output_path, os.path.normpath(f.name))
    is_dir = not f.is_file
    if (is_dir and not f.is_symbolic_link) or not _is_within_output_path(output_path, file_path):
        return None
    if f.is_symbolic_link and not _is_valid_sym_link(output_path, f):
        return None
    return file_path


def extract_archive_to_disk(archive: Archive, output_path: str, buffer_size: int | None = None) -> list:
    """extractArchiveToDiskSync (:92-103) / the member loop of extractFileToDisk (:222-258): files through an
    OutputFileStream, symbolic links as links, directories created -- members whose path or link target would leave
    `output_path` are skipped.  Returns the paths written (the reference returns nothing)."""
    os.makedirs(output_path, exist_ok=True)
    written = []
    for f in archive:
        if not f.is_file and not f.is_symbolic_link:
            p = os.path.join(output_path, os.path.normpath(f.name))
            if _is_within_output_path(output_path, p):  # extractFileToDisk creates directory entries (:236-239)
                os.makedirs(p, exist_ok=True)
            continue
        file_path = _prepare_archive_file_path(f, output_path)
        if file_path is None:
            continue
        if f.is_symbolic_link:
            os.makedirs(os.path.dirname(file_path), exist_ok=True)
            if os.path.lexists(file_path):
                os.unlink(file_path)
            os.symlink(os.path.normpath(f.symbolic_link or ""), file_path)  # Link.createSync(target, recursive: true)
        else:
            out = OutputFileStream(file_path, buffer_size=buffer_size)
            out.write_bytes(f.content or b"")  # ArchiveFile.writeContent
            out.close_sync()
            if f.mode & 0o777:
                os.chmod(file_path, f.mode & 0o777)  # posix.chmod(filePath, file.unixPermissions) (:252-254)
        written.append(file_path)
    return written


def get_input_extension(input_path: str) -> str:
    """getInputExtension (:146-157): up to two components for the compressed tar names."""
    lower = input_path.lower()
    for ext in (".tar.gz", ".tar.bz2", ".tar.xz"):
        if lower.endswith(ext):
            return ext
    return os.path.splitext(lower)[1]


_EXTENSIONS = ".tar.gz, .tgz, .tar.bz2, .tbz, .tar.xz, .txz or .zip"


def extract_file_to_disk(input_path: str, output_path: str, buffer_size: int | None = None, password=None) -> list:
    """extractFileToDisk (:160-267).  .zip: ZipDecoder().decodeStream(InputFileStream, password:) and the member loop above.
    .tar.gz / .tgz / .tar.bz2 / .tbz / .tar.xz / .txz: the reference decodes into a temporary `temp.tar` with
    GZipDecoder / BZip2Decoder / XZDecoder.decodeStream(InputFileStream, OutputFileStream) (:183-202) and hands that to TarDecoder; here
    the same two stream objects make the library decode file -> file, and the .tar itself is the result (see the module
    text).  Anything else: ValueError, as the reference's ArgumentError."""
    ext = get_input_extension(input_path)
    if not ext:
        raise ValueError(f"{input_path}: no file extension detected, must end with {_EXTENSIONS}")
    if ext == ".zip":
        inp = InputFileStream(input_path)
        try:
            archive = ZipDecoder().decode_stream(inp, password=password)
        finally:
            inp.close_sync()
        return extract_archive_to_disk(archive, output_path, buffer_size=buffer_size)
    if ext in (".tar.gz", ".tgz", ".tar.bz2", ".tbz", ".tar.xz", ".txz"):
        os.makedirs(output_path, exist_ok=True)
        base = os.path.basename(input_path)
        stem = base[:-len(ext)] if base.lower().endswith(ext) else os.path.splitext(base)[0]
        tar_path = os.path.join(output_path, stem + ".tar")
        inp = InputFileStream(input_path)
        out = OutputFileStream(tar_path, buffer_size=buffer_size)
        try:
            dec = GZipDecoder() if ext in (".tar.gz", ".tgz") else XZDecoder() if ext in (".tar.xz", ".txz") else BZip2Decoder()
            dec.decode_stream(inp, out)  # the reference ignores the bool here too
        finally:
            inp.close_sync()
            out.close_sync()
        return [tar_path]
    raise ValueError(f"{input_path}: must end with {_EXTENSIONS}")


def _sorted_listing(dir_path: str, follow_links: bool) -> list:
    """Directory.listSync(recursive: true, followLinks:) as [(path, is_directory)], sorted by path (the reference takes
    whatever order the file system gives)."""
    listing = []
    for root, dirs, files in os.walk(dir_path, followlinks=follow_links):
        dirs.sort()
        listing += [(os.path.join(root, d), True) for d in dirs] + [(os.path.join(root, f), False) for f in sorted(files)]
    listing.sort(key=lambda x: x[0])
    return listing


class ZipFileEncoder:
    """ZipFileEncoder (lib/src/io/zip_file_encoder.dart:11-225): build a .zip on disk from files and directories.  The
    reference compresses every file as it is added (ZipEncoder.startEncode / add / endEncode); here the members are collected
    and compressed when the archive is closed -- all deflate members of a level as ONE device batch when `batch` is set
    (b200z_deflate_batch) -- and the container is written through an OutputFileStream.  The bytes are those of
    ZipEncoder().encode_bytes over the same members in the same order.  Directory listings are taken in sorted order (the
    reference takes whatever order Directory.listSync returns)."""
    STORE, GZIP = 0, 1  # (:16-17) the reference's names for levels 0 and 1

    def __init__(self, compress=None, batch: bool = False):
        self._compress, self._batch = compress, batch
        self._files, self._path, self._level, self._modified = None, None, None, None

    @staticmethod
    def _compose_zip_directory_path(dir_path: str, filename):  # (:56-74)
        if filename is None:
            return dir_path.rstrip("/\\") + ".zip"
        a, b = os.path.abspath(dir_path), os.path.abspath(filename)
        if b != a and os.path.commonpath([a, b]) == a:
            raise ValueError(f"filename must not be within the directory being zipped: {filename}")  # FormatException
        return filename

    def create(self, zip_path: str, level=None, modified=None):  # (:78-91)
        self._path, self._level, self._modified, self._files = zip_path, level, modified, []

    open = create

    def add_archive_file(self, f: ArchiveFile):  # (:212-214)
        self._files.append(f)

    def add_file(self, path: str, filename=None, level=None):  # addFileSync (:182-194)
        name = (filename or os.path.basename(path)).replace(os.sep, "/")
        st = os.stat(path)
        with open(path, "rb") as fh:
            body = fh.read()
        f = ArchiveFile(name, len(body))
        f.content, f.last_mod_time, f.mode = body, int(st.st_mtime), st.st_mode
        f.compress_level = level  # add(file, level:) -- level 0 is still method 8, as stored DEFLATE blocks (zip_encoder.dart:248-252)
        self._files.append(f)

    def add_directory(self, dir_path: str, include_dir_name: bool = True, level=None, follow_links: bool = True, filter=None):
        """addDirectorySync (:93-136).  filter(path, progress) -> "skip" | "cancel" | anything else."""
        dir_name = os.path.basename(os.path.normpath(dir_path))
        listing = _sorted_listing(dir_path, follow_links)
        for k, (p, is_dir) in enumerate(listing):
            if filter is not None:
                op = filter(p, (k + 1) / len(listing))
                if op == "cancel":
                    break
                if op == "skip":
                    continue
            rel = os.path.relpath(p, dir_path).replace(os.sep, "/")
            name = f"{dir_name}/{rel}" if include_dir_name else rel
            if is_dir:
                st = os.stat(p)
                f = ArchiveFile(name, 0, is_file=False)
                f.mode, f.last_mod_time = st.st_mode, int(st.st_mtime)
                self._files.append(f)
            else:
                self.add_file(p, name, level)

    def close(self):  # closeSync (:216-219): endEncode + close the stream
        from .zip import ZipEncoder
        data = ZipEncoder(compress=self._compress, batch=self._batch).encode_bytes(self._files, level=self._level,
                                                                                 modified=self._modified)
        out = OutputFileStream(self._path)
        out.write_bytes(data)
        out.close_sync()
        self._files = None
        return len(data)

    close_sync = close

    def zip_directory(self, dir_path: str, filename=None, level=None, follow_links: bool = True, modified=None, filter=None):
        """zipDirectory (:22-43): level defaults to `gzip` (= 1)."""
        level = self.GZIP if level is None else level
        self.create(self._compose_zip_directory_path(dir_path, filename), level=level, modified=modified)
        self.add_directory(dir_path, include_dir_name=False, level=level, follow_links=follow_links, filter=filter)
        return self.close()


class TarFileEncoder:
    """TarFileEncoder (lib/src/io/tar_file_encoder.dart:12-108): build a .tar, or a .tar.gz, on disk from files and
    directories.  Members go through TarEncoder into an OutputFileStream as they are added; file contents are copied from
    an InputFileStream.  Directory listings are taken in sorted order (the reference takes whatever order
    Directory.listSync returns)."""
    STORE, GZIP = 0, 1  # (:17-18)

    def __init__(self):
        self.tar_path, self._output, self._encoder = None, None, None

    def tar_directory(self, dir_path: str, compression: int = STORE, filename=None, follow_links: bool = True,
                      level=None, filter=None):
        """tarDirectory (:20-49): `filename` or '<dir>.tar' / '<dir>.tar.gz', members named '<dir name>/...'.  For GZIP
        the tar is written to a temporary `temp.tar` first, then GZipEncoder().encode_stream(InputFileStream,
        OutputFileStream, level: level ?? 6) compresses it file to file on the device (b200z_file_codec), and the
        temporary file and its directory are deleted."""
        tar_path = filename if filename is not None else f"{dir_path}.tar"
        tgz_path = filename if filename is not None else f"{dir_path}.tar.gz"
        temp_dir = None
        if compression == self.GZIP:
            temp_dir = tempfile.mkdtemp(prefix="dart_archive")
            tar_path = os.path.join(temp_dir, "temp.tar")
        try:
            self.open(tar_path)
            self.add_directory(dir_path, follow_links=follow_links, filter=filter)
            self.close()
            if compression == self.GZIP:
                inp, out = InputFileStream(tar_path), OutputFileStream(tgz_path)
                try:
                    GZipEncoder().encode_stream(inp, out, level=6 if level is None else level)
                finally:
                    inp.close_sync()
                    out.close_sync()
        finally:
            if temp_dir is not None:
                shutil.rmtree(temp_dir, ignore_errors=True)

    def create(self, tar_path: str):  # (:51-58)
        self.tar_path = tar_path
        self._output = OutputFileStream(tar_path)
        self._encoder = TarEncoder()
        self._encoder.start(self._output)

    open = create

    def add_directory(self, dir_path: str, follow_links: bool = True, include_dir_name: bool = True, filter=None):
        """addDirectory (:60-92).  filter(path, progress) -> "skip" | "cancel" | anything else.  A directory entry is
        named '<name>/' and, as in the reference, carries the time it was added, not the directory's mtime."""
        dir_name = os.path.basename(os.path.normpath(dir_path))
        listing = _sorted_listing(dir_path, follow_links)
        for k, (p, is_dir) in enumerate(listing):
            if filter is not None:
                op = filter(p, (k + 1) / len(listing))
                if op == "cancel":
                    break
                if op == "skip":
                    continue
            rel = os.path.relpath(p, dir_path).replace(os.sep, "/")
            name = f"{dir_name}/{rel}" if include_dir_name else rel
            if is_dir:
                f = ArchiveFile(f"{name}/", 0, is_file=False)  # ArchiveFile.directory: lastModTime is "now"
                f.mode, f.last_mod_time = os.stat(p).st_mode, int(time.time())
                self._encoder.add(f)
            else:
                self.add_file(p, name)

    def add_file(self, path: str, filename=None):
        """addFile (:94-102): the content is streamed from the file; the mode is the whole st_mode."""
        st = os.stat(path)
        inp = InputFileStream(path)
        try:
            f = ArchiveFile(filename if filename is not None else os.path.basename(path), inp.length)
            f.content, f.last_mod_time, f.mode = inp, int(st.st_mtime), st.st_mode
            self._encoder.add(f)
        finally:
            inp.close_sync()

    def close(self):  # (:104-107)
        self._encoder.finish()
        self._output.close_sync()
