"""Pure-Python model of the client reader stack's observable behaviour.

Oracle / test infrastructure only (see oracle/__init__.py).

Follows (reference, relative to the CurvineIO/curvine source tree):
  * curvine-common/src/fs/reader.rs:50-141          read_chunk / read / read_full / fuse_read
  * curvine-client/src/file/fs_reader.rs:103-126     read_chunk0, seek fast path inside the chunk
  * curvine-client/src/file/fs_reader_buffer.rs:248-323  sub-reader choice, misaligned-chunk trim
  * curvine-client/src/file/fs_reader_parallel.rs:94-187 split / read / seek over owned slices
  * curvine-client/src/file/fs_reader_base.rs:101-204    block cursor; seek rules (==len ok, >len error)
  * curvine-common/src/state/block_info.rs:190-217   partition_point block lookup
  * curvine-client/src/file/read_detector.rs:130-218 read_parallel + sequential/random state machine
  * curvine-client/src/block/block_reader_hole.rs:69-79  hole blocks read as zeros
  * orpc/src/io/local_file.rs:103-117                chunk = min(chunk_size, block_len - pos)
Prefetch tasks/channels are modelled as lazy generators: prefetching changes
timing, never the delivered byte/chunk sequence.
"""
from bisect import bisect_right
from dataclasses import dataclass
from typing import List, Optional, Tuple

FILE_MIN_ALIGN_SIZE = 4096  # curvine-client/src/lib.rs


class FsError(Exception):
    pass


# ----------------------------------------------------------------- split / detector

def split(total_size: int, slice_size: int, read_parallel: int) -> List[List[Tuple[int, int]]]:
    """FsReaderParallel::split (fs_reader_parallel.rs:94-125)."""
    if total_size <= 0:
        return []
    if read_parallel == 1:
        return [[(0, total_size)]]
    num = (total_size + slice_size - 1) // slice_size
    out = [[] for _ in range(read_parallel)]
    for sid in range(num):
        start = sid * slice_size
        end = total_size if sid == num - 1 else start + slice_size
        out[sid % read_parallel].append((start, end))
    return out


SEQUENTIAL, RANDOM = 1, 2


@dataclass
class ClientConf:
    """Read knobs and their defaults (curvine-common/src/conf/client_conf.rs:315-420)."""
    block_size: int = 128 * 1024 * 1024
    read_chunk_size: int = 128 * 1024
    read_chunk_num: int = 8
    read_parallel: int = 1
    read_slice_size: int = 0  # 0 -> chunk_num * chunk_size (client_conf.rs init)
    short_circuit: bool = True
    enable_read_ahead: bool = True
    read_ahead_len: int = 0  # 0 -> chunk_num * chunk_size
    drop_cache_len: int = 1024 * 1024
    max_cache_block_handles: int = 10
    enable_smart_prefetch: bool = True
    large_file_size: int = 10 * 1024 * 1024 * 1024
    max_read_parallel: int = 8
    sequential_read_threshold: int = 7

    def init(self):
        if self.read_slice_size == 0:
            self.read_slice_size = self.read_chunk_num * self.read_chunk_size
        if self.read_ahead_len == 0:
            self.read_ahead_len = self.read_chunk_num * self.read_chunk_size
        return self


class ReadDetector:
    """read_detector.rs:121-218."""

    def __init__(self, conf: ClientConf, file_size: int):
        rp = conf.read_parallel
        if conf.enable_smart_prefetch and file_size >= conf.large_file_size:
            calc = (file_size + conf.large_file_size - 1) // conf.large_file_size
            rp = min(conf.max_read_parallel, max(1, calc))
        self.enabled = conf.enable_smart_prefetch
        self.last_read_pos = -1
        self.seq_count = 0
        self.check_threshold = conf.sequential_read_threshold
        self.read_parallel = rp
        self.read_pattern = SEQUENTIAL

    def is_random(self):
        return self.read_pattern == RANDOM

    def is_sequential(self):
        return self.read_pattern == SEQUENTIAL

    def record_seek(self):
        if not self.enabled:
            return
        self.seq_count = 0
        self.last_read_pos = -1
        if self.read_pattern == SEQUENTIAL:
            self.read_pattern = RANDOM

    def record_read(self, start: int, end: int) -> bool:
        if not self.enabled:
            return False
        if self.last_read_pos == -1 or start == self.last_read_pos:
            self.seq_count += 1
        else:
            self.seq_count = 0
        self.last_read_pos = end
        pattern = SEQUENTIAL if self.seq_count >= self.check_threshold else self.read_pattern
        if pattern != self.read_pattern:
            self.read_pattern = pattern
            return True
        return False


# ----------------------------------------------------------------------- file model

@dataclass
class BlockSpec:
    id: int
    len: int
    hole: bool = False  # no locations + alloc_opts -> BlockReaderHole


class FileModel:
    """A file = concatenation of blocks in block_locs order (block_info.rs:190-217)."""

    def __init__(self, blocks: List[BlockSpec], data: bytes):
        self.blocks = blocks
        self.data = data
        self.starts, off = [], 0
        for b in blocks:
            self.starts.append(off)
            off += b.len
        self.ends = [s + b.len for s, b in zip(self.starts, blocks)]
        self.len = off
        assert len(data) == off

    def get_read_block(self, pos: int) -> Tuple[int, int]:
        """-> (block_off, block_index); partition_point(|x| x.end <= pos)."""
        idx = bisect_right(self.ends, pos)
        if idx >= len(self.blocks):
            raise FsError("Not found block for pos %d" % pos)
        return pos - self.starts[idx], idx


class BaseModel:
    """FsReaderBase: file pos -> block cursor -> chunk."""

    def __init__(self, f: FileModel, chunk_size: int):
        self.f, self.chunk_size, self.pos = f, chunk_size, 0

    def read(self) -> bytes:
        if self.pos >= self.f.len:
            return b""
        boff, idx = self.f.get_read_block(self.pos)
        blk = self.f.blocks[idx]
        n = min(self.chunk_size, blk.len - boff)
        out = bytes(n) if blk.hole else self.f.data[self.pos:self.pos + n]
        self.pos += n
        return out

    def seek(self, pos: int):
        if pos == self.pos:
            return
        if pos == self.f.len:
            self.pos = pos
            return
        if pos > self.f.len:
            raise FsError("seek position %d can not exceed file len %d" % (pos, self.f.len))
        self.f.get_read_block(pos)
        self.pos = pos


class ParallelModel:
    """FsReaderParallel over its owned slices."""

    def __init__(self, f: FileModel, chunk_size: int, slices: List[Tuple[int, int]]):
        self.inner = BaseModel(f, chunk_size)
        self.slices = slices
        self.cur: Optional[int] = None

    def read(self) -> Tuple[int, bytes]:
        if self.cur is None:
            self.cur = 0
            self.inner.seek(self.slices[0][0])
        elif self.inner.pos >= self.slices[self.cur][1]:
            nxt = self.cur + 1
            if nxt >= len(self.slices):
                return 0, b""
            self.cur = nxt
            self.inner.seek(self.slices[nxt][0])
        pos = self.inner.pos
        return pos, self.inner.read()

    def seek(self, pos: int):
        ends = [e for _, e in self.slices]
        idx = bisect_right(ends, pos)
        if idx < len(self.slices):
            self.inner.seek(max(pos, self.slices[idx][0]))
            self.cur = idx
        elif self.slices:
            self.inner.seek(self.slices[-1][1])
            self.cur = len(self.slices) - 1
        else:
            self.inner.seek(0)
            self.cur = None


class ReaderModel:
    """FsReader + FsReaderBuffer + the provided ``Reader`` trait methods."""

    def __init__(self, f: FileModel, conf: ClientConf):
        conf.init()
        cs, ss = conf.read_chunk_size, conf.read_slice_size
        if cs % FILE_MIN_ALIGN_SIZE or cs < FILE_MIN_ALIGN_SIZE:
            raise FsError("chunk_size must be an integer multiple of %d" % FILE_MIN_ALIGN_SIZE)
        if ss % cs or ss < cs:
            raise FsError("The slice size must be an integer multiple of the chunk size.")
        self.f, self.conf = f, conf
        self.chunk_size, self.slice_size = cs, ss
        self.det = ReadDetector(conf, f.len)
        subs = [ParallelModel(f, cs, s) for s in split(f.len, ss, self.det.read_parallel) if s]
        self.readers = subs + [ParallelModel(f, cs, [(0, f.len)])]
        self.len = f.len
        self.pos = 0  # FsReader.pos
        self.bpos = 0  # FsReaderBuffer.pos
        self.chunk = b""

    # -- FsReaderBuffer::read
    def _buffer_read(self) -> bytes:
        if self.bpos >= self.len:
            return b""
        rid = self.det.read_parallel if self.det.is_random() else (self.bpos // self.slice_size) % self.det.read_parallel
        if rid >= len(self.readers):
            raise FsError("reader %d is not initialized" % rid)
        off, data = self.readers[rid].read()
        diff = self.bpos - off
        if diff == 0:
            out = data
        elif 0 < diff <= len(data):
            out = data[diff:]
        else:
            raise FsError("read data error: chunk offset %d, pos %d, diff %d" % (off, self.bpos, diff))
        start = self.bpos
        self.bpos += len(out)
        if self.det.record_read(start, self.bpos) and self.det.is_sequential():
            for r in self.readers:
                r.seek(self.bpos)
        return out

    def _buffer_seek(self, pos: int):
        if pos == self.bpos:
            return
        self.det.record_seek()
        for r in self.readers:
            r.seek(pos)
        self.bpos = pos

    # -- Reader trait (provided methods)
    def read_chunk(self, length: Optional[int] = None) -> bytes:
        if not self.chunk:
            self.chunk = self._buffer_read()
        n = len(self.chunk) if length is None else min(length, len(self.chunk))
        out, self.chunk = self.chunk[:n], self.chunk[n:]
        return out

    def read(self, n: int) -> bytes:
        out = self.read_chunk(n)
        self.pos += len(out)
        return out

    def blocking_read(self) -> bytes:
        return self.read(1 << 62)

    def read_full(self, n: int) -> bytes:
        parts, rem = [], n
        while rem > 0:
            p = self.read(rem)
            if not p:
                break
            parts.append(p)
            rem -= len(p)
        return b"".join(parts)

    def seek(self, pos: int):
        if pos < 0:
            raise FsError("Cannot seek to negative offset")
        if pos == self.pos:
            return
        skip = pos - self.pos
        if 0 <= skip <= len(self.chunk):
            self.chunk = self.chunk[skip:]
        else:
            self.chunk = b""
            self._buffer_seek(pos)
        self.pos = pos

    def fuse_read(self, pos: int, length: int) -> List[bytes]:
        self.seek(pos)
        out, rem = [], length
        while rem > 0:
            c = self.read_chunk(rem)
            if not c:
                break
            out.append(c)
            rem -= len(c)
            self.pos += len(c)
        return out
