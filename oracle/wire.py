"""orpc RpcMessage wire codec + the three protobuf headers on the read path.

Oracle / test infrastructure only (see oracle/__init__.py).

Follows (reference, relative to the CurvineIO/curvine source tree):
  * orpc/src/message/rpc_message.rs:26-41   PROTOCOL_SIZE=22, HEAD_SIZE=18, MAX_DATE_SIZE=16 MiB
  * orpc/src/message/rpc_message.rs:43-90   RequestStatus / ResponseStatus / Status::{encode,from}
  * orpc/src/message/rpc_message.rs:301-338 encode_protocol / decode_protocol (big-endian)
  * orpc/src/handler/rpc_frame.rs:205-264   send = prefix, header, data ; receive skips heartbeats
  * orpc/src/error/error_encoder.rs:24-51   error body = i32 kind, u32 len, msg, u32 data_len, data
  * curvine-common/proto/worker.proto:38-60 BlockReadRequest / BlockReadResponse / DataHeaderProto
  * curvine-common/src/fs/rpc_code.rs:76-79 ReadBlock = 81
Protobuf is proto2 as prost 0.11 emits it: ``required`` fields always written in
field-number order (even when equal to the default), ``optional`` only when set.
"""
import struct
from dataclasses import dataclass
from typing import Optional, Tuple, List

PROTOCOL_SIZE = 22
HEAD_SIZE = PROTOCOL_SIZE - 4
MAX_DATA_SIZE = 16 * 1024 * 1024
INIT_SEQ_ID = -1
END_SEQ_ID = -2
EMPTY_REQ_ID = -1

RPC_CODE_WRITE_BLOCK = 80
RPC_CODE_READ_BLOCK = 81

# RequestStatus
REQ_UNDEFINED, REQ_HEARTBEAT, REQ_RPC, REQ_OPEN, REQ_RUNNING, REQ_CANCEL, REQ_COMPLETE = -1, 0, 1, 2, 3, 4, 5
# ResponseStatus
RESP_UNDEFINED, RESP_SUCCESS, RESP_ERROR = -1, 0, 1

# StorageTypeProto (common.proto:9-16)
STORAGE_MEM, STORAGE_SSD, STORAGE_HDD, STORAGE_UFS, STORAGE_DISK, STORAGE_SPDK_DISK = 0, 1, 2, 3, 4, 5


def _i8(v: int) -> int:
    v &= 0xFF
    return v - 256 if v >= 128 else v


def status_encode(req: int, resp: int) -> int:
    """Status::encode -> i8:  (req as i8) | ((resp as i8) << 4)."""
    return _i8((req & 0xFF) | ((resp << 4) & 0xFF))


def status_decode(v: int) -> Tuple[int, int]:
    """Status::from(i8): req = v & 0x0f, resp = v >> 4 (arithmetic); unknown -> Undefined."""
    v = _i8(v)
    req = v & 0x0F
    resp = v >> 4
    if req not in (0, 1, 2, 3, 4, 5):
        req = REQ_UNDEFINED
    if resp not in (0, 1):
        resp = RESP_UNDEFINED
    return req, resp


@dataclass
class Message:
    code: int = 0
    req_status: int = REQ_UNDEFINED
    resp_status: int = RESP_UNDEFINED
    req_id: int = 0
    seq_id: int = 0
    header: bytes = b""
    data: bytes = b""

    def status_byte(self) -> int:
        return status_encode(self.req_status, self.resp_status) & 0xFF

    def is_success(self) -> bool:
        return self.resp_status == RESP_SUCCESS

    def is_heartbeat(self) -> bool:
        return self.req_status == REQ_HEARTBEAT


def encode_protocol(m: Message) -> bytes:
    total = len(m.header) + len(m.data) + HEAD_SIZE
    return struct.pack(">iibbqi", total, len(m.header), _i8(m.code), _i8(m.status_byte()), m.req_id, m.seq_id)


def encode(m: Message) -> bytes:
    return encode_protocol(m) + m.header + m.data


class WireError(Exception):
    pass


def decode_protocol(buf: bytes):
    """-> (code, req_status, resp_status, req_id, seq_id, header_size, data_size)."""
    if len(buf) < PROTOCOL_SIZE:
        raise WireError("short prefix")
    total, hsz, code, st, req_id, seq_id = struct.unpack(">iibbqi", buf[:PROTOCOL_SIZE])
    dsz = total - hsz - HEAD_SIZE
    if dsz < 0:
        raise WireError("data length is negative")
    if dsz > MAX_DATA_SIZE:
        raise WireError("Data exceeds maximum size: %d" % MAX_DATA_SIZE)
    rq, rs = status_decode(st)
    return code, rq, rs, req_id, seq_id, hsz, dsz


def decode_stream(buf: bytes, skip_heartbeat: bool = True) -> Tuple[List[Message], int]:
    """Decode as many whole frames as ``buf`` holds; returns (messages, bytes consumed)."""
    out, pos = [], 0
    while len(buf) - pos >= PROTOCOL_SIZE:
        code, rq, rs, req_id, seq_id, hsz, dsz = decode_protocol(buf[pos:pos + PROTOCOL_SIZE])
        if hsz < 0:
            raise WireError("Invalid length %d" % hsz)
        end = pos + PROTOCOL_SIZE + hsz + dsz
        if end > len(buf):
            break
        m = Message(code, rq, rs, req_id, seq_id, buf[pos + 22:pos + 22 + hsz], buf[pos + 22 + hsz:end])
        pos = end
        if skip_heartbeat and m.is_heartbeat():
            continue
        out.append(m)
    return out, pos


def request(code, req_status, req_id, seq_id, header=b"", data=b"") -> Message:
    return Message(code, req_status, RESP_UNDEFINED, req_id, seq_id, header, data)


def success(req: Message, header=b"", data=b"") -> Message:
    return Message(req.code, req.req_status, RESP_SUCCESS, req.req_id, req.seq_id, header, data)


def error(req: Message, kind: int, msg: str) -> Message:
    return Message(req.code, req.req_status, RESP_ERROR, req.req_id, req.seq_id, b"", encode_error(kind, msg))


def encode_error(kind: int, msg: str, data: bytes = b"") -> bytes:
    mb = msg.encode()
    return struct.pack(">iI", kind, len(mb)) + mb + struct.pack(">I", len(data)) + data


def decode_error(body: bytes) -> Tuple[int, str]:
    kind, n = struct.unpack(">iI", body[:8])
    return kind, body[8:8 + n].decode(errors="replace")


# ------------------------------ protobuf (proto2) -----------------------------

def _varint(v: int) -> bytes:
    v &= 0xFFFFFFFFFFFFFFFF  # int64/int32 negatives are 10-byte two's-complement varints
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _rd_varint(buf: bytes, pos: int) -> Tuple[int, int]:
    v, shift = 0, 0
    while True:
        b = buf[pos]
        pos += 1
        v |= (b & 0x7F) << shift
        if not b & 0x80:
            return v, pos
        shift += 7


def _s64(v: int) -> int:
    v &= 0xFFFFFFFFFFFFFFFF
    return v - (1 << 64) if v >> 63 else v


def _field_varint(no: int, v: int) -> bytes:
    return _varint(no << 3) + _varint(int(v))


def _field_bytes(no: int, b: bytes) -> bytes:
    return _varint((no << 3) | 2) + _varint(len(b)) + b


def _parse(buf: bytes) -> dict:
    out, pos = {}, 0
    while pos < len(buf):
        key, pos = _rd_varint(buf, pos)
        no, wt = key >> 3, key & 7
        if wt == 0:
            v, pos = _rd_varint(buf, pos)
        elif wt == 2:
            n, pos = _rd_varint(buf, pos)
            v = buf[pos:pos + n]
            pos += n
        elif wt == 1:
            v = buf[pos:pos + 8]
            pos += 8
        elif wt == 5:
            v = buf[pos:pos + 4]
            pos += 4
        else:
            raise WireError("bad wire type")
        out[no] = v
    return out


@dataclass
class BlockReadRequest:  # worker.proto:38-47
    id: int = 0
    off: int = 0
    len: int = 0
    chunk_size: int = 0
    short_circuit: bool = False
    enable_read_ahead: bool = True
    read_ahead_len: int = 4194304
    drop_cache_len: int = 1048576

    def encode(self) -> bytes:
        return (_field_varint(1, self.id) + _field_varint(2, self.off) + _field_varint(3, self.len)
                + _field_varint(4, self.chunk_size) + _field_varint(5, self.short_circuit)
                + _field_varint(8, self.enable_read_ahead) + _field_varint(9, self.read_ahead_len)
                + _field_varint(10, self.drop_cache_len))

    @staticmethod
    def decode(buf: bytes) -> "BlockReadRequest":
        f = _parse(buf)
        for req in (1, 2, 3, 4, 5, 8, 9, 10):
            if req not in f:
                raise WireError("missing required field %d" % req)
        return BlockReadRequest(_s64(f[1]), _s64(f[2]), _s64(f[3]), _s64(f[4]),
                                bool(f[5]), bool(f[8]), _s64(f[9]), _s64(f[10]))


@dataclass
class BlockReadResponse:  # worker.proto:49-54
    id: int = 0
    len: int = 0
    path: Optional[str] = None
    storage_type: int = STORAGE_DISK

    def encode(self) -> bytes:
        out = _field_varint(1, self.id) + _field_varint(2, self.len)
        if self.path is not None:
            out += _field_bytes(3, self.path.encode())
        return out + _field_varint(4, self.storage_type)

    @staticmethod
    def decode(buf: bytes) -> "BlockReadResponse":
        f = _parse(buf)
        return BlockReadResponse(_s64(f[1]), _s64(f[2]), f[3].decode() if 3 in f else None, int(f[4]))


@dataclass
class DataHeaderProto:  # worker.proto:56-60
    offset: int = 0
    flush: bool = False
    is_last: bool = False

    def encode(self) -> bytes:
        return _field_varint(1, self.offset) + _field_varint(2, self.flush) + _field_varint(3, self.is_last)

    @staticmethod
    def decode(buf: bytes) -> "DataHeaderProto":
        f = _parse(buf)
        return DataHeaderProto(_s64(f[1]), bool(f[2]), bool(f[3]))


FILE_TYPE_FILE = 1


@dataclass
class BlockWriteRequest:  # worker.proto:10-18 (block = ExtendedBlockProto, common.proto:98-104)
    block_id: int = 0
    block_len: int = 0  # ExtendedBlockProto.block_size: the block's current length
    storage_type: int = STORAGE_DISK
    file_type: int = FILE_TYPE_FILE
    off: int = 0
    block_size: int = 0
    short_circuit: bool = False
    client_name: str = ""
    chunk_size: int = 0

    def encode(self) -> bytes:
        blk = (_field_varint(1, self.block_id) + _field_varint(2, self.block_len) + _field_varint(3, self.storage_type)
               + _field_varint(4, self.file_type))
        return (_field_bytes(1, blk) + _field_varint(2, self.off) + _field_varint(3, self.block_size)
                + _field_varint(4, self.short_circuit) + _field_bytes(5, self.client_name.encode()) + _field_varint(6, self.chunk_size))

    @staticmethod
    def decode(buf: bytes) -> "BlockWriteRequest":
        f = _parse(buf)
        b = _parse(f[1])
        return BlockWriteRequest(_s64(b[1]), _s64(b[2]), int(b[3]), int(b[4]), _s64(f[2]), _s64(f[3]), bool(f[4]), f[5].decode(), _s64(f[6]))


@dataclass
class BlockWriteResponse:  # worker.proto:27-34
    id: int = 0
    path: Optional[str] = None
    off: int = 0
    block_size: int = 0
    storage_type: int = STORAGE_DISK

    def encode(self) -> bytes:
        out = _field_varint(1, self.id)
        if self.path is not None:
            out += _field_bytes(2, self.path.encode())
        return out + _field_varint(3, self.off) + _field_varint(4, self.block_size) + _field_varint(5, self.storage_type)

    @staticmethod
    def decode(buf: bytes) -> "BlockWriteResponse":
        f = _parse(buf)
        return BlockWriteResponse(_s64(f[1]), f[2].decode() if 2 in f else None, _s64(f[3]), _s64(f[4]), int(f[5]))


# ----------------------- one remote block read, as bytes -----------------------

def block_read_exchange(block_id: int, block: bytes, chunk_size: int, req_id: int, off: int = 0,
                        storage_type: int = STORAGE_MEM, read_ahead_len: int = 1048576,
                        drop_cache_len: int = 1048576):
    """(requests, responses) byte strings for Open -> Running*n -> Complete of one block.

    Client side: block_reader_remote.rs:36-122 + block_client.rs:222-300 (seq 0 for
    Open, 1.. for Running, n+1 for Complete).  Worker side: read_handler.rs:60-207,
    local_file.rs:103-117 (chunk = min(chunk_size, len - pos); never empty).
    """
    reqs, resps = [], []
    o = request(RPC_CODE_READ_BLOCK, REQ_OPEN, req_id, 0,
                BlockReadRequest(block_id, off, len(block), chunk_size, False, True, read_ahead_len,
                                 drop_cache_len).encode())
    reqs.append(encode(o))
    resps.append(encode(success(o, BlockReadResponse(block_id, len(block), None, storage_type).encode())))
    pos, seq = off, 0
    while pos < len(block):
        seq += 1
        r = request(RPC_CODE_READ_BLOCK, REQ_RUNNING, req_id, seq)
        n = min(chunk_size, len(block) - pos)
        reqs.append(encode(r))
        resps.append(encode(success(r, b"", block[pos:pos + n])))
        pos += n
    c = request(RPC_CODE_READ_BLOCK, REQ_COMPLETE, req_id, seq + 1, BlockReadRequest(id=block_id).encode())
    reqs.append(encode(c))
    resps.append(encode(success(c)))
    return reqs, resps
