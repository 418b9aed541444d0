"""Drop-in for the read side of the reference's Python SDK (curvine-libsdk/python/curvinefs: CurvineClient / CurvineReader) on the
new C ABI -- SURVEY 8f-4.  Same class and method names, same argument meaning and error behaviour for the calls on the read path
(open, read, seek, close, read_range, head, tail, get_file_status); the control-plane calls (mkdir, rm, rename, ls, ...) belong to the
master and raise Unsupported here.

Two deliberate differences, both stated where they occur:
  * CurvineReader.read returns the BYTES.  The reference decodes them as UTF-8 with errors ignored before returning
    (curvinefs/curvineReader.py:49), which silently corrupts binary data; it also hands out `length` bytes from the address of ONE
    native chunk whatever its size (curvineReader.py:25-36).  Here `read(offset, length)` means what its arguments say: skip `offset`
    bytes from the current position, return up to `length` bytes, stop at end of file.
  * read_tensor / read_range_tensor (additions): the bytes as a uint8 CUDA tensor in HBM, CRC-verified on the GPU, DLPack-exportable.
  * load_safetensors (addition): a safetensors checkpoint as {name: CUDA tensor} from one CRC-verified vectored read."""
from typing import Optional

from . import fs as _fs


class CurvineReader:
    """curvinefs/curvineReader.py:5-84"""

    def __init__(self, reader: "_fs.Reader", file_size: int):
        self.readerHandle = reader
        self.file_size = file_size
        self.read_pos = 0

    def read(self, offset, length):
        if self.readerHandle is None:
            raise IOError("Native read file failed: reader is closed")
        pos = self.read_pos + offset
        if pos < 0:
            raise IOError("Position is negative")  # curvineReader.py:19-20
        if pos >= self.file_size or length <= 0:
            self.read_pos = min(pos, self.file_size)
            return b""
        if offset:
            try:
                self.readerHandle.seek(pos)
            except _fs.FsError as e:
                raise IOError("Native seek failed: %s" % e)
        try:
            data = self.readerHandle.read_full(length)
        except _fs.FsError as e:
            raise IOError("Native read file failed: %s" % e)
        self.read_pos = pos + len(data)
        return data

    def seek(self, pos):
        if pos < 0:
            raise ValueError("Seek position cannot be negative")  # curvineReader.py:54-55
        if pos > self.file_size:
            raise ValueError("Seek position %d exceeds file length %d" % (pos, self.file_size))
        try:
            self.readerHandle.seek(pos)
        except _fs.FsError as e:
            raise IOError("Native seek failed: %s" % e)
        self.read_pos = pos

    def read_tensor(self, length: Optional[int] = None, device=None, verify: bool = True):
        """Addition: the next `length` bytes (default: up to end of file) as a uint8 CUDA tensor; whole blocks are CRC-verified on the GPU."""
        import torch
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        n = self.file_size - self.read_pos if length is None else max(0, min(length, self.file_size - self.read_pos))
        out = torch.empty(n, dtype=torch.uint8, device=dev)
        if n:
            self.readerHandle.seek(self.read_pos)
            got = self.readerHandle.read_device(out.data_ptr(), n, torch.cuda.current_stream(dev).cuda_stream)
            _, bad, _ = self.readerHandle.verify()
            if verify and bad:
                raise IOError("%d blocks failed CRC verification" % bad)
            self.read_pos += got
            out = out[:got]
        return out

    def close(self):
        if self.readerHandle is None:  # curvineReader.py:74-75: closing twice is not an error
            return
        r, self.readerHandle = self.readerHandle, None
        try:
            r.complete()
        except _fs.FsError as e:
            raise IOError("Native close reader failed: %s" % e)
        self.read_pos = 0
        self.file_size = 0


class CurvineClient:
    """curvinefs/curvineClient.py:11-326, read side.  `config_path`: the cluster TOML (the reference's own keys; `[b200]` adds the GPU
    knobs, and the top-level key `namespace_manifest` stands in for the master's block locations, see DESIGN.md)."""

    def __init__(self, config_path, write_chunk_num=8, write_chunk_size=131072):
        try:
            self.file_system_ptr = _fs.CurvineFileSystem(conf_path=config_path)
        except _fs.FsError as e:
            raise IOError("Native create file system failed: %s" % e)
        self.write_chunk_num = write_chunk_num
        self.write_chunk_size = write_chunk_size

    def get_file_status(self, path):
        """-> dict like the reference's (curvineClient.py:21-43) with the fields the manifest knows, or None when the file does not exist."""
        try:
            r = self.file_system_ptr.open(path)
        except _fs.FsError:
            return None
        try:
            n = r.len()
        finally:
            r.complete()
        return {"path": path, "name": path.rstrip("/").rsplit("/", 1)[-1], "is_dir": False, "is_complete": True, "len": n}

    def open(self, path):
        try:
            r = self.file_system_ptr.open(path)
        except _fs.FsError as e:
            raise IOError("Native open reader failed: %s" % e)
        return CurvineReader(r, r.len())

    @staticmethod
    def _span(file_len, offset, length):
        """(first byte, byte count) of a read_range request.  Rules of curvineClient.py:154-180: a negative offset counts back from the
        end of the file; length None or -1 means "to the end" (and then the offset has to lie inside the file); anything else must be a
        non-negative int."""
        if not isinstance(offset, int):
            raise ValueError("offset: an integer is required, got %r" % (offset,))
        first = offset + file_len if offset < 0 else offset
        to_end = length is None or length == -1
        if to_end and first >= file_len:
            raise ValueError("offset %d is not inside a file of %d bytes" % (first, file_len))
        if not to_end and (not isinstance(length, int) or length < 0):
            raise ValueError("length: a non-negative integer, -1 or None is required, got %r" % (length,))
        return first, (file_len - first if to_end else length)

    def _len_of(self, path):
        status = self.get_file_status(path)
        if status is None:
            raise FileNotFoundError(path)
        return status["len"]

    def read_range(self, path, offset, length):
        first, count = self._span(self._len_of(path), offset, length)
        if count == 0:
            return b""
        reader = self.open(path)
        try:
            return reader.read(first, count)
        finally:
            reader.close()

    def head(self, path, size):
        if not isinstance(size, int) or size < 0:
            raise ValueError("size: a non-negative integer is required, got %r" % (size,))
        return self.read_range(path, 0, size)

    def tail(self, path, size):
        if not isinstance(size, int) or size < 0:
            raise ValueError("size: a non-negative integer is required, got %r" % (size,))
        n = self._len_of(path)
        take = min(size, n)
        return self.read_range(path, n - take, take) if take else b""

    def read_range_tensor(self, path, offset=0, length=None, device=None):
        """Addition: read_range into HBM (uint8 CUDA tensor)."""
        reader = self.open(path)
        try:
            reader.seek(offset if offset >= 0 else reader.file_size + offset)
            return reader.read_tensor(length, device)
        finally:
            reader.close()

    def load_safetensors(self, path, device=None, names=None, slices=None, dtype=None, scales=None, scale_block=None):
        """Addition: a safetensors checkpoint as {name: CUDA tensor}, from one CRC-verified vectored read (curvine_b200.safetensors);
        slices = {name: (dim, start, stop)} loads only that part of a tensor (a tensor-parallel rank's shard); dtype converts the
        float32, float16 and bfloat16 tensors to it on the GPU as they load; scales = {float8 weight: its scale tensor} (and scale_block
        for block scales) dequantizes those weights to dtype as they load."""
        from . import safetensors
        try:
            return safetensors.load_file(self.file_system_ptr, path, device=device, names=names, slices=slices, dtype=dtype, scales=scales,
                                        scale_block=scale_block)
        except _fs.FsError as e:
            raise IOError("Native load safetensors failed: %s" % e)

    def close(self):
        if self.file_system_ptr is not None:
            fs_, self.file_system_ptr = self.file_system_ptr, None
            fs_.close()

    def _control_plane(self, *a, **k):
        raise _fs.FsError(19, "control-plane operation: served by the master, outside the read path this library replaces")  # ErrorKind::Unsupported

    get_master_info = mkdir = rm = rename = list_status = ls = create = write_string = append = mv = touch = copy = copy_dir = copy_file = _control_plane
    download = upload = write_to_new_file = _control_plane
