"""The device reader sends a copy group's short-circuit Opens in one write and reads the answers in order.  A worker that answers one of
them with an error must not hang the read or leave a connection with unread answers in the pool: the group is redone one Open at a
time, which fails over to the next replica, or fails with the worker's message when there is none."""
import os
import shutil
import socket
import tempfile
import threading
import time

import pytest

from curvine_b200 import fs as F
from oracle import layout, synth
from oracle import wire as W

pytestmark = pytest.mark.gpu

BS = 64 << 10
NB = 8


def _rx(c, n):
    out = b""
    while len(out) < n:
        b = c.recv(n - len(out))
        if not b:
            raise EOFError
        out += b
    return out


def _frame(pre, header=b"", data=b"", status=None):
    st = pre[9] & 0x0f if status is None else status
    return (18 + len(header) + len(data)).to_bytes(4, "big") + len(header).to_bytes(4, "big") + bytes([pre[8], st]) + pre[10:22] + header + data


class _ShortCircuitWorker:
    """answers short-circuit Opens with the block file's path, Completes with success; an Open of a block in `bad` gets an error"""

    def __init__(self, paths, bad=()):
        self.paths, self.bad, self.opens = paths, set(bad), 0
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

    def _serve(self, c):
        try:
            while True:
                pre = _rx(c, 22)
                total, hlen = int.from_bytes(pre[:4], "big"), int.from_bytes(pre[4:8], "big")
                header = _rx(c, hlen)
                _rx(c, total - 18 - hlen)
                if pre[9] & 0x0f == W.REQ_OPEN:
                    self.opens += 1
                    req = W.BlockReadRequest.decode(header)
                    if req.id in self.bad:
                        c.sendall(_frame(pre, data=W.encode_error(10000, "made up by the test"), status=(pre[9] & 0x0f) | 0x10))
                    else:
                        c.sendall(_frame(pre, header=W.BlockReadResponse(id=req.id, len=BS, path=self.paths[req.id], storage_type=0).encode()))
                else:
                    c.sendall(_frame(pre))
        except (EOFError, OSError):
            c.close()

    def close(self):
        self.s.close()


@pytest.fixture()
def blocks():
    """NB block files of two files (/good, /bad) -> (dir, {block id: path}, {inode: bytes})"""
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    d = tempfile.mkdtemp(prefix="cvbo", dir=base)
    paths, data = {}, {}
    for ino in (5901, 5902):
        data[ino] = synth.file_bytes(ino, NB * BS, BS)
        for b in range(NB):
            bid = layout.create_block_id(ino, b)
            paths[bid] = os.path.join(d, "blk_%d" % bid)
            with open(paths[bid], "wb") as f:
                f.write(data[ino][b * BS:(b + 1) * BS])
    yield d, paths, data
    shutil.rmtree(d, ignore_errors=True)


def _manifest(path, ino, ports):
    locs = ",".join("localhost:%d:%d" % (p, i + 1) for i, p in enumerate(ports))
    return "# m\nfile %s %d %d %d 0\n" % (path, ino, NB * BS, BS) + "".join(
        "block %d %d 0 - - - %s\n" % (layout.create_block_id(ino, b), BS, locs) for b in range(NB))


def _read(fs, path, cuda):
    import torch
    r = fs.open(path)
    dst = torch.zeros(NB * BS, dtype=torch.uint8, device=cuda)
    try:
        assert r.read_device(dst.data_ptr(), NB * BS, torch.cuda.current_stream().cuda_stream) == NB * BS
        s, bad, _ = r.verify()
        torch.cuda.synchronize()
        assert bad == 0
        return dst.cpu().numpy().tobytes(), s
    finally:
        try:
            r.complete()
        except F.FsError:
            pass


def _conf():
    return F.client_conf(short_circuit=True, extra_client='conn_timeout_ms = 1000\ndata_timeout_ms = 2000\nrpc_timeout_ms = 2000\n',
                         b200="fetch_threads = 2\ncopy_group = 4\nverify_batch = 4\nzero_copy = true\nregister_threads = 0\nregister_cache = \"64MB\"\n")


@pytest.mark.parametrize("second_replica", [True, False], ids=["fails_over", "only_replica"])
def test_an_error_on_the_third_open_of_a_batch(cuda, blocks, second_replica):
    d, paths, data = blocks
    bad_bid = layout.create_block_id(5902, 2)  # the third Open of the first copy group
    lying = _ShortCircuitWorker(paths, bad=[bad_bid])
    honest = _ShortCircuitWorker(paths)
    t0 = time.time()
    try:
        ports = [lying.port, honest.port] if second_replica else [lying.port]
        with F.CurvineFileSystem(_conf()) as fs:
            fs.load_namespace(_manifest("/bad", 5902, ports) + _manifest("/good", 5901, [lying.port]).split("\n", 1)[1])
            if second_replica:
                got, _ = _read(fs, "/bad", cuda)
                assert got == data[5902]
                assert honest.opens >= 1  # the failed block went to the second replica
            else:
                with pytest.raises(F.FsError) as e:
                    _read(fs, "/bad", cuda)
                assert "made up by the test" in str(e.value)
            # the connections left in the pool carry no answers of the failed batch: a read of another file on them is exact
            got, _ = _read(fs, "/good", cuda)
            assert got == data[5901]
    finally:
        lying.close(), honest.close()
    assert time.time() - t0 < 30
