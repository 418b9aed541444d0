"""Hostile peers.  The reference has no fuzzing (SURVEY §4); its codec rejects frames by length checks (rpc_message.rs:329-334) and turns
handler errors into error RESPONSES (block_handler.rs:57-60).  Here both ends of the product meet peers that do not follow the protocol:

  * the WORKER is fed malformed, truncated and random frames over raw sockets: it must answer with an error frame or drop the connection,
    never crash, never allocate what a length field claims, and keep serving well-behaved clients;
  * the CLIENT (host reader, framed path) talks to a worker that lies: absurd lengths, wrong echoes, truncated payloads, payloads longer
    than asked for, random bytes, silence.  Every call must come back with an error (or the correct bytes), within its timeout.  The host
    writer meets wrong echoes, an error answer and a cut-off answer, and must not pool a connection whose stream is out of step.

tools/sanitize_host.sh runs this file under ASan+UBSan."""
import os
import random
import socket
import struct
import tempfile
import threading
import time

import pytest

from curvine_b200 import fs as F
from oracle import layout, synth
from oracle import wire as W


def _prefix(total_len, header_len, code=81, status=W.REQ_OPEN, req_id=7, seq_id=0):
    return struct.pack(">iibbqi", total_len, header_len, code, status, req_id, seq_id)


def _hostile_requests(rng, valid_open):
    """byte strings a broken or malicious client might send"""
    yield b""                                                       # connect and leave
    yield b"\x00"                                                   # a fraction of a prefix
    yield _prefix(18, 0)[:21]                                       # one byte short of a prefix
    yield _prefix(-1, 0)                                            # negative total_len
    yield _prefix(0x7fffffff, 0)                                    # 2 GiB frame announced, nothing follows
    yield _prefix(18 + 5, 0x7fffffff)                               # header longer than the frame
    yield _prefix(18, -5)                                           # negative header_len
    yield _prefix(18 + (17 << 20), 0) + b"x" * 1024                 # data_len > 16 MiB (MAX_DATE_SIZE)
    yield _prefix(18 + 10, 10) + b"\xff" * 10                       # Open whose header is not protobuf
    yield _prefix(18 + 3, 3, status=W.REQ_RUNNING) + b"\x08\x80\x80"  # truncated varint in a DataHeaderProto
    yield _prefix(18, 0, status=W.REQ_RUNNING)                      # Running without Open
    yield _prefix(18, 0, status=W.REQ_COMPLETE)                     # Complete without Open
    yield _prefix(18, 0, code=0, status=W.REQ_OPEN)                 # unknown code
    yield _prefix(18, 0, status=9)                                  # unknown request status
    yield valid_open[:len(valid_open) - 3]                          # a valid Open cut short
    yield valid_open + _prefix(18, 0, status=W.REQ_RUNNING, seq_id=1) * 3 + b"\x00" * 7   # valid start, then garbage
    for _ in range(40):
        yield bytes(rng.getrandbits(8) for _ in range(rng.choice([1, 21, 22, 23, 64, 300, 5000])))
    for _ in range(20):                                             # plausible prefix, random rest
        hl, dl = rng.choice([0, 1, 9, 200]), rng.choice([0, 1, 100, 70000])
        yield _prefix(18 + hl + dl, hl, status=rng.choice([W.REQ_OPEN, W.REQ_RUNNING, W.REQ_COMPLETE])) + bytes(rng.getrandbits(8) for _ in range(hl + dl))


def test_worker_survives_hostile_clients():
    rng = random.Random(20240)
    with tempfile.TemporaryDirectory(dir="/dev/shm" if os.path.isdir("/dev/shm") else None) as d:
        with F.MiniWorker(["[MEM]" + d + "/m"]) as w:
            n, bs, ino = (2 << 20) + 99, 1 << 20, 4701
            man = w.create_file("/h", ino, n, bs)
            want = synth.file_bytes(ino, n, bs)
            bid = layout.create_block_id(ino, 0)
            valid_open = W.encode(W.request(W.RPC_CODE_READ_BLOCK, W.REQ_OPEN, 77, 0, W.BlockReadRequest(id=bid, off=0, len=bs, chunk_size=65536).encode()))
            for i, blob in enumerate(_hostile_requests(rng, valid_open)):
                s = socket.create_connection(("127.0.0.1", w.port), timeout=5)
                s.settimeout(0.3)
                try:
                    try:
                        s.sendall(blob)
                        if i % 3 == 0:
                            s.shutdown(socket.SHUT_WR)
                    except OSError:
                        pass  # the worker has already dropped the connection: a legitimate answer
                    try:
                        for _ in range(8):   # whatever comes back (error frames, data, nothing): it must end or time out, not wedge the worker
                            if not s.recv(1 << 16):
                                break
                    except (socket.timeout, ConnectionError):
                        pass
                finally:
                    s.close()
                if i % 10 == 9:  # the worker still serves a well-behaved client, over both paths
                    for sc in (True, False):
                        with F.CurvineFileSystem(F.client_conf(short_circuit=sc)) as fs:
                            fs.load_namespace(man)
                            with fs.open("/h") as r:
                                assert r.read_full(n) == want
            with F.CurvineFileSystem(F.client_conf(short_circuit=False)) as fs:
                fs.load_namespace(man)
                with fs.open("/h") as r:
                    assert r.read_full(n) == want


class _LyingWorker:
    """answers Open honestly (unless told otherwise), then misbehaves on Running according to `mode`"""

    def __init__(self, block, mode, rng):
        self.block, self.mode, self.rng = block, mode, rng
        self.s = socket.socket()
        self.s.bind(("127.0.0.1", 0))
        self.s.listen(16)
        self.port = self.s.getsockname()[1]
        threading.Thread(target=self._accept, daemon=True).start()

    def _accept(self):
        while True:
            try:
                c, _ = self.s.accept()
            except OSError:
                return
            threading.Thread(target=self._serve, args=(c,), daemon=True).start()

    @staticmethod
    def _rx(c, n):
        out = b""
        while len(out) < n:
            b = c.recv(n - len(out))
            if not b:
                raise EOFError
            out += b
        return out

    def _reply(self, pre, header=b"", data=b"", total=None, hlen=None, req_id=None, seq_id=None, status=None):
        code, st, rid, sid = pre[8], pre[9] & 0x0f, int.from_bytes(pre[10:18], "big", signed=True), int.from_bytes(pre[18:22], "big", signed=True)
        return _prefix(18 + len(header) + len(data) if total is None else total, len(header) if hlen is None else hlen, code,
                       st if status is None else status, rid if req_id is None else req_id, sid if seq_id is None else seq_id) + header + data

    def _serve(self, c):
        pos, chunk, m = 0, 65536, self.mode
        try:
            while True:
                pre = self._rx(c, 22)
                total, hlen = int.from_bytes(pre[:4], "big"), int.from_bytes(pre[4:8], "big")
                header = self._rx(c, hlen)
                self._rx(c, total - 18 - hlen)
                st = pre[9] & 0x0f
                if st == W.REQ_OPEN and pre[8] == W.RPC_CODE_WRITE_BLOCK:  # a writer's Open: the block size it asked for
                    c.sendall(self._reply(pre, header=W.BlockWriteResponse(block_size=W.BlockWriteRequest.decode(header).block_size, storage_type=0).encode()))
                    continue
                if st == W.REQ_OPEN:
                    req = W.BlockReadRequest.decode(header)
                    pos, chunk = req.off, req.chunk_size
                    if m == "open_garbage_header":
                        c.sendall(self._reply(pre, header=b"\xff\xff\xff\xff\xff"))
                    elif m == "open_error_body_garbage":
                        c.sendall(self._reply(pre, data=b"\x07" * 9, status=st | 0x10))
                    elif m == "open_len_lies":
                        c.sendall(self._reply(pre, header=W.BlockReadResponse(id=req.id, len=len(self.block) * 1000, storage_type=0).encode()))
                    else:
                        c.sendall(self._reply(pre, header=W.BlockReadResponse(id=req.id, len=len(self.block), storage_type=0).encode()))
                    continue
                if st == W.REQ_COMPLETE:
                    c.sendall(self._reply(pre))
                    if m == "honest_then_hang_up":  # answers everything correctly, then closes: what a worker restart looks like to a pooled connection
                        c.close()
                        return
                    continue
                data = self.block[pos:pos + chunk]
                pos += len(data)
                if m == "huge_data_len":
                    c.sendall(self._reply(pre, total=18 + (17 << 20)) + data)
                elif m == "negative_total":
                    c.sendall(self._reply(pre, total=-7))
                elif m == "negative_header_len":
                    c.sendall(self._reply(pre, data=data, hlen=-3))
                elif m == "wrong_req_id":
                    c.sendall(self._reply(pre, data=data, req_id=123456789))
                elif m == "wrong_seq_id":
                    c.sendall(self._reply(pre, data=data, seq_id=-1))
                elif m == "truncated_payload":
                    c.sendall(self._reply(pre, data=data)[:22 + len(data) // 2])
                    c.close()
                    return
                elif m == "truncated_then_hang_up":  # a payload announced, half of it sent
                    c.sendall(self._reply(pre, data=b"\0" * 64)[:22 + 32])
                    c.close()
                    return
                elif m == "longer_than_chunk":
                    c.sendall(self._reply(pre, data=data + b"Z" * 4096))
                elif m == "random_bytes":
                    c.sendall(bytes(self.rng.getrandbits(8) for _ in range(self.rng.choice([5, 22, 23, 400]))))
                elif m == "silence":
                    time.sleep(3)
                    c.close()
                    return
                elif m == "error_response":
                    c.sendall(self._reply(pre, data=W.encode_error(10000, "made up by the test"), status=st | 0x10))
                elif m in ("honest", "honest_then_hang_up"):
                    c.sendall(self._reply(pre, data=data))
        except (EOFError, OSError, ValueError):
            try:
                c.close()
            except OSError:
                pass

    def close(self):
        self.s.close()


MODES = ["honest", "open_garbage_header", "open_error_body_garbage", "open_len_lies", "huge_data_len", "negative_total", "negative_header_len", "wrong_req_id",
         "wrong_seq_id", "truncated_payload", "longer_than_chunk", "random_bytes", "silence", "error_response"]


@pytest.mark.parametrize("mode", MODES)
def test_client_survives_a_lying_worker(mode):
    ino, bs = 4801, 1 << 20
    n = bs
    data = synth.file_bytes(ino, n, bs)
    bid = layout.create_block_id(ino, 0)
    lw = _LyingWorker(data, mode, random.Random(99))
    man = "# m\nfile /lie %d %d %d 0\nblock %d %d 0 - - - localhost:%d:1\n" % (ino, n, bs, bid, n, lw.port)
    t0 = time.time()
    try:
        with F.CurvineFileSystem(F.client_conf(short_circuit=False, read_chunk_size="64KB", read_chunk_num=2,
                                               extra_client='conn_timeout_ms = 1000\ndata_timeout_ms = 1000\nrpc_timeout_ms = 1000\n')) as fs:
            fs.load_namespace(man)
            if mode == "honest":
                with fs.open("/lie") as r:
                    assert r.read_full(n) == data
            else:
                r = fs.open("/lie")
                with pytest.raises(F.FsError) as e:
                    got = r.read_full(n)
                    # a worker that sends MORE than a chunk per frame is not an error per se (the reference takes data_len as sent): the bytes must then be wrong-sized, not a crash
                    assert mode == "longer_than_chunk" and got != data
                    raise F.FsError(12, "payload larger than requested")
                assert e.value.kind > 0
                try:
                    r.complete()
                except F.FsError:
                    pass
    finally:
        lw.close()
    assert time.time() - t0 < 30, "a lying worker must not stall the client beyond its timeouts"


@pytest.mark.parametrize("mode", ["wrong_seq_id", "wrong_req_id", "error_response", "truncated_then_hang_up"])
def test_writer_survives_a_lying_worker(mode):
    """The answer to a host write's Running lies.  write() fails, and the connection goes back to the pool only when its stream is still
    in step: after a well-formed error answer, never after a wrong echo or a cut-off payload."""
    lw = _LyingWorker(b"", mode, random.Random(99))  # Running answers carry no payload, as a worker's do
    try:
        with F.CurvineFileSystem(F.client_conf(extra_client='conn_timeout_ms = 1000\ndata_timeout_ms = 1000\nrpc_timeout_ms = 1000\n')) as fs:
            w = fs.create("/lie_w", 4802, 1 << 20, lw.port)
            with pytest.raises(F.FsError):
                w.write(b"x" * 1000)
            try:
                w.complete()
            except F.FsError:
                if mode != "truncated_then_hang_up":  # only a worker that hung up cannot answer the Complete
                    raise
            assert fs.pool_stats()["idle"] == (1 if mode == "error_response" else 0)
    finally:
        lw.close()


def test_conf_and_manifest_parsers_survive_garbage():
    """The two text inputs a deployment hands the library -- the cluster TOML and the namespace manifest -- as random text, as valid text
    with random edits, and with absurd numbers: an error code or a successful parse, never a crash, and a handle that still closes."""
    import ctypes
    from hypothesis import given, settings, strategies as st
    from curvine_b200 import _lib
    L = _lib.lib()
    good_conf = F.client_conf(b200='fetch_threads = 4\ngpu_chunk_size = "1MB"\narena_preregister = ["/tmp/a", "/tmp/b"]\n')
    good_man = ("# m\nfile /f 4901 3145728 1048576 0\n" + "".join("block %d 1048576 0 %08x %08x - localhost:9:1,otherhost:10:2\n" % (layout.create_block_id(4901, b), b, b + 7) for b in range(3)))

    def try_conf(text):
        h = ctypes.c_void_p()
        rc = L.cv_fs_new_from_string(text.encode("utf-8", "ignore"), ctypes.byref(h))
        assert (rc == 0) == bool(h)
        if h:
            assert L.cv_fs_close(h) == 0

    def try_manifest(text):
        h = ctypes.c_void_p()
        assert L.cv_fs_new_from_string(b"", ctypes.byref(h)) == 0
        rc = L.cv_fs_load_namespace_string(h, text.encode("utf-8", "ignore"))
        assert rc <= 0
        assert L.cv_fs_close(h) == 0

    def edited(base, data):
        chars = list(base)
        for _ in range(data.draw(st.integers(1, 6))):
            i = data.draw(st.integers(0, len(chars) - 1))
            op = data.draw(st.integers(0, 3))
            if op == 0:
                chars[i] = data.draw(st.sampled_from(list('0123456789-="[]{},.:# \n\tKMGTBxe')))
            elif op == 1:
                del chars[i]
            elif op == 2:
                chars.insert(i, data.draw(st.sampled_from(["99999999999999999999999", "-1", '"', "[", "\n[b200]\n", "=", " 1e400 ", "0x", "\x00"])))
            else:
                chars[i:i] = chars[max(0, i - 20):i]
        return "".join(chars)

    @settings(max_examples=150, deadline=None)
    @given(st.data())
    def run(data):
        try_conf(data.draw(st.text(max_size=300)))
        try_conf(edited(good_conf, data))
        try_manifest(data.draw(st.text(max_size=300)))
        try_manifest(edited(good_man, data))

    try_conf(good_conf)
    try_manifest(good_man)
    run()
