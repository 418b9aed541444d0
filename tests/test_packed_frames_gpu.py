"""The wire bytes of the two paths that pack Running frames on the GPU with K4 (cvk_pack_frames):

  * the worker's HBM tier answers a remote block read with frames packed from device memory: every Running reply must be the
    oracle's reply byte for byte, at chunk sizes that divide the block and one that does not, from offset 0 and from an odd offset;
  * the device writer (Writer.write_device) sends the Running requests K4 packed: a recording peer sees the same frames as from the
    host writer (Writer.write) given the same bytes in the same calls, and both manifests carry the oracle's block CRCs.

The round-trip tests in test_gpu_reader.py check the bytes that land; these check the frames themselves."""
import os
import shutil
import socket
import tempfile
import threading

import numpy as np
import pytest

from curvine_b200 import fs as F
from oracle import clib, layout, synth
from oracle import wire as W

pytestmark = pytest.mark.gpu


def _rx(c, n):
    out = b""
    while len(out) < n:
        b = c.recv(n - len(out))
        if not b:
            raise EOFError
        out += b
    return out


def _rx_frame(c):
    pre = _rx(c, W.PROTOCOL_SIZE)
    return pre + _rx(c, int.from_bytes(pre[:4], "big", signed=True) - W.HEAD_SIZE)


# ------------------------------------------------------------------ HBM tier: Running replies against the oracle

HBM_INO, HBM_LEN = 9601, (1 << 20) + 4321  # one block, not a multiple of any chunk size below


@pytest.fixture(scope="module")
def hbm_worker(cuda):
    d = tempfile.mkdtemp(prefix="cvpk", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    w = F.MiniWorker(["[MEM]" + d + "/mem"])
    try:
        w.create_file("/pk", HBM_INO, HBM_LEN, 2 << 20)
        bid = layout.create_block_id(HBM_INO, 0)
        w.hbm_load(bid, 0)
        os.remove(layout.block_path(d + "/mem/curvine", bid))  # every reply must come from the resident copy
        yield w, bid, synth.file_bytes(HBM_INO, HBM_LEN, 2 << 20)
    finally:
        w.stop()
        shutil.rmtree(d, ignore_errors=True)


@pytest.mark.parametrize("off", [0, 777])
@pytest.mark.parametrize("chunk", [4096, 10001, 131072])
def test_hbm_tier_running_replies_are_the_oracles_bytes(hbm_worker, chunk, off):
    w, bid, block = hbm_worker
    reads0 = w.hbm_stats()["reads_from_hbm"]
    reqs, resps = W.block_read_exchange(bid, block, chunk, 0x0102030405060708 + chunk + off, off=off)
    s = socket.create_connection(("127.0.0.1", w.port), timeout=30)
    try:
        s.sendall(reqs[0])
        (o,), _ = W.decode_stream(_rx_frame(s))
        assert o.is_success() and W.BlockReadResponse.decode(o.header).len == len(block)
        for f in range(1, len(reqs) - 1):
            s.sendall(reqs[f])
            assert _rx_frame(s) == resps[f], "Running reply %d of %d" % (f, len(reqs) - 2)
        s.sendall(reqs[-1])
        assert _rx_frame(s) == resps[-1]
    finally:
        s.close()
    assert len(reqs) - 2 == (len(block) - off + chunk - 1) // chunk
    assert w.hbm_stats()["reads_from_hbm"] == reads0 + 1


# ------------------------------------------------------------------ device writer: the same Running frames as the host writer

class _RecordingPeer:
    """answers a block writer's Open, Running and Complete the way the worker does, and keeps every byte it was sent"""

    def __init__(self):
        self.received = bytearray()
        self.s = socket.socket()
        self.s.bind(("127.0.0.1", 0))
        self.s.listen(4)
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
                frame = _rx_frame(c)
                self.received += frame
                (m,), _ = W.decode_stream(frame)
                header = b""
                if m.req_status == W.REQ_OPEN:
                    r = W.BlockWriteRequest.decode(m.header)
                    header = W.BlockWriteResponse(id=r.block_id, off=r.off, block_size=r.block_size, storage_type=r.storage_type).encode()
                c.sendall(W.encode(W.success(m, header)))
        except (EOFError, OSError):
            c.close()

    def close(self):
        self.s.close()


def _write(cuda, src, bs, chunk, cuts, device):
    """src written in the calls that `cuts` delimits, to a recording peer -> (what the peer received, the writer's manifest)"""
    import torch
    peer = _RecordingPeer()
    try:
        with F.CurvineFileSystem(F.client_conf(short_circuit=False)) as fs:
            wr = fs.create("/pw", 9701, bs, peer.port, chunk_size=chunk)
            d_src = torch.from_numpy(src).to(cuda) if device else None
            for a, b in zip(cuts, cuts[1:]):
                if device:
                    wr.write_device(d_src.data_ptr() + a, b - a, torch.cuda.current_stream().cuda_stream)
                else:
                    wr.write(src[a:b].tobytes())
            man = wr.complete()
        return bytes(peer.received), man
    finally:
        peer.close()


def _frames(stream):
    """the stream of one file's block writes, decoded: [(Open, [Running...], Complete) per block]; framing checked byte for byte"""
    msgs, used = W.decode_stream(stream)
    assert used == len(stream) and b"".join(W.encode(m) for m in msgs) == stream
    blocks = []
    for m in msgs:
        assert m.code == W.RPC_CODE_WRITE_BLOCK
        if m.req_status == W.REQ_OPEN:
            assert m.seq_id == 0
            blocks.append((m, [], None))
        elif m.req_status == W.REQ_RUNNING:
            assert m.req_id == blocks[-1][0].req_id and m.header == b"" and m.status_byte() == 0xF3
            blocks[-1][1].append(m)
        else:
            assert m.req_status == W.REQ_COMPLETE and m.req_id == blocks[-1][0].req_id
            blocks[-1] = (blocks[-1][0], blocks[-1][1], m)
    return blocks


def test_device_writer_sends_the_host_writers_running_frames(cuda):
    bs, chunk = 1 << 20, 100000  # the chunk size does not divide the block
    n = 3 * bs + 12345
    src = np.frombuffer(synth.file_bytes(9701, n, bs), dtype=np.uint8).copy()
    cuts = [0, bs + 54321, n]  # the first call ends mid-block
    host_stream, host_man = _write(cuda, src, bs, chunk, cuts, device=False)
    dev_stream, dev_man = _write(cuda, src, bs, chunk, cuts, device=True)
    host, dev = _frames(host_stream), _frames(dev_stream)
    assert len(host) == len(dev) == 4
    for b, ((ho, hr, hc), (do, dr, dc)) in enumerate(zip(host, dev)):
        assert ho.header == do.header and hc.header == dc.header and hc.seq_id == dc.seq_id == len(hr) + 1
        assert [(m.code, m.status_byte(), m.seq_id, m.data) for m in hr] == [(m.code, m.status_byte(), m.seq_id, m.data) for m in dr]
        assert [m.seq_id for m in dr] == list(range(1, len(dr) + 1))
        assert b"".join(m.data for m in dr) == src[b * bs:(b + 1) * bs].tobytes()
    # block 1 is written by two calls: its frames restart at the second call's first byte, on both paths
    first, rest = cuts[1] - bs, 2 * bs - cuts[1]
    assert [len(m.data) for m in dev[1][1]] == [first] + [chunk] * (rest // chunk) + [rest % chunk]
    for man in (host_man, dev_man):
        blocks = [l.split() for l in man.splitlines() if l.startswith("block ")]
        assert [int(x[4], 16) for x in blocks] == clib.crc_blocks(0, src, bs).tolist()
        assert [int(x[5], 16) for x in blocks] == clib.crc_blocks(1, src, bs).tolist()
