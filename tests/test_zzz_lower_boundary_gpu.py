"""The LOWER boundary on its own (SURVEY 8b: "host -> CUDA, the thin extern C layer"): a host that keeps its own protocol loop -- here the
oracle's codec over a Python socket, standing in for the reference's Rust client with RpcFrame::receive -- and links nothing but this
library: pinned receive buffers (cvh_pinned_alloc), H2D of the wire image (cvh_h2d_async), frame descriptors expanded on the device
(cvk_expand_streams), K2 (cvk_unpack_frames: validate + gather + CRC), results back (cvh_d2h_async), ordering by cvh events.  No cv_*
reader, no torch stream.  Bytes and CRCs against the oracle.  Written after round 2's last GPU run; sorts late on purpose."""
import ctypes
import os
import shutil
import socket
import tempfile

import numpy as np
import pytest

from curvine_b200 import _lib, fs as F
from curvine_b200._lib import CvFrameDesc, CvStreamDesc
from oracle import clib, layout, synth
from oracle import wire as W

pytestmark = pytest.mark.gpu


def _ok(rc):
    assert rc == 0, "CUDA error %d" % rc


def _recv_exact(s, n):
    out = bytearray()
    while len(out) < n:
        b = s.recv(n - len(out))
        assert b, "connection closed"
        out += b
    return bytes(out)


def _recv_frame(s):
    pre = _recv_exact(s, 22)
    total = int.from_bytes(pre[:4], "big", signed=True)
    return pre + _recv_exact(s, total - 18)


def test_foreign_host_drives_k2_through_cvh_and_cvk_only(cuda):
    L = _lib.lib()
    chunk, bs, nb, ino = 65536, 1 << 20, 5, 8501
    n = bs * nb - 4321
    d = tempfile.mkdtemp(prefix="cvlb", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    pinned = ctypes.c_void_p()
    d_wire, d_dst, d_streams, d_desc, d_crc, d_err = (ctypes.c_void_p() for _ in range(6))
    h_crc, h_err = ctypes.c_void_p(), ctypes.c_void_p()
    copy_stream, k_stream, copied, done = (ctypes.c_void_p() for _ in range(4))
    try:
        with F.MiniWorker(["[MEM]" + d + "/m"]) as w:
            w.create_file("/lb", ino, n, bs)
            want = synth.file_bytes(ino, n, bs)
            blens = [min(bs, n - b * bs) for b in range(nb)]
            frames_per_block = [(x + chunk - 1) // chunk for x in blens]
            n_frames = sum(frames_per_block)
            wire_cap = n + 22 * n_frames
            _ok(L.cvh_pinned_alloc(wire_cap, ctypes.byref(pinned)))
            for ptr, size in ((d_wire, wire_cap), (d_dst, n + 64), (d_streams, ctypes.sizeof(CvStreamDesc) * nb), (d_desc, ctypes.sizeof(CvFrameDesc) * n_frames),
                              (d_crc, 4 * nb), (d_err, 4 * n_frames)):
                _ok(L.cvh_device_alloc(size, ctypes.byref(ptr)))
            _ok(L.cvh_pinned_alloc(4 * nb, ctypes.byref(h_crc)))
            _ok(L.cvh_pinned_alloc(4 * n_frames, ctypes.byref(h_err)))
            _ok(L.cvh_stream_create(ctypes.byref(copy_stream)))
            _ok(L.cvh_stream_create(ctypes.byref(k_stream)))
            _ok(L.cvh_event_create(ctypes.byref(copied)))
            _ok(L.cvh_event_create(ctypes.byref(done)))
            # ---- the host's own protocol loop: Open, Running x n, Complete per block; data frames land verbatim in the pinned buffer
            wire = (ctypes.c_uint8 * wire_cap).from_address(pinned.value)
            streams = (CvStreamDesc * nb)()
            s = socket.create_connection(("127.0.0.1", w.port))
            pos, fidx, dst_off = 0, 0, 0
            for b in range(nb):
                bid, rid = layout.create_block_id(ino, b), 0x5000 + b
                s.sendall(W.encode(W.request(81, W.REQ_OPEN, rid, 0, W.BlockReadRequest(bid, 0, blens[b], chunk, False, True, 1 << 20, 1 << 20).encode())))
                o, _ = W.decode_stream(_recv_frame(s))
                assert o[0].is_success() and W.BlockReadResponse.decode(o[0].header).len == blens[b]
                streams[b] = CvStreamDesc(pos, dst_off, blens[b], rid, chunk, 1, b, fidx, 81, 0x03)
                for f in range(frames_per_block[b]):
                    s.sendall(W.encode(W.request(81, W.REQ_RUNNING, rid, f + 1)))
                    fr = _recv_frame(s)
                    ctypes.memmove(pinned.value + pos, fr, len(fr))
                    pos += len(fr)
                fidx += frames_per_block[b]
                dst_off += blens[b]
                s.sendall(W.encode(W.request(81, W.REQ_COMPLETE, rid, frames_per_block[b] + 1, W.BlockReadRequest(id=bid).encode())))
                c, _ = W.decode_stream(_recv_frame(s))
                assert c[0].is_success()
            s.close()
            assert pos == wire_cap
            del wire
            # ---- device side, two streams ordered by an event
            _ok(L.cvh_h2d_async(d_wire, pinned, wire_cap, copy_stream, None))
            _ok(L.cvh_h2d_async(d_streams, ctypes.cast(streams, ctypes.c_void_p), ctypes.sizeof(streams), copy_stream, copied))
            _ok(L.cvh_stream_wait_event(k_stream, copied))
            _ok(L.cvk_expand_streams(d_streams, nb, d_desc, n_frames, k_stream))
            _ok(L.cvk_unpack_frames(ctypes.cast(d_wire, ctypes.POINTER(ctypes.c_uint8)), d_desc, n_frames, nb, ctypes.cast(d_dst, ctypes.POINTER(ctypes.c_uint8)), 1, n, d_crc, d_err, k_stream))
            _ok(L.cvh_d2h_async(h_crc, d_crc, 4 * nb, k_stream, None))
            _ok(L.cvh_d2h_async(h_err, d_err, 4 * n_frames, k_stream, done))
            assert L.cvh_event_query(done) in (0, 600)
            _ok(L.cvh_event_synchronize(done))
            assert L.cvh_event_query(done) == 0
            crc = np.frombuffer((ctypes.c_uint32 * nb).from_address(h_crc.value), dtype=np.uint32).copy()
            err = np.frombuffer((ctypes.c_uint32 * n_frames).from_address(h_err.value), dtype=np.uint32).copy()
            assert (err == 0).all()
            assert crc.tolist() == [clib.crc(1, np.frombuffer(want[b * bs:b * bs + blens[b]], dtype=np.uint8)) for b in range(nb)]
            # the payload bytes, back through a pinned buffer
            back = ctypes.c_void_p()
            _ok(L.cvh_pinned_alloc(n, ctypes.byref(back)))
            _ok(L.cvh_d2h_async(back, d_dst, n, k_stream, None))
            _ok(L.cvh_stream_synchronize(k_stream))
            assert ctypes.string_at(back.value, n) == want
            _ok(L.cvh_pinned_free(back))
            # memory the host already owns (here: an anonymous page-aligned mapping) becomes a DMA source once registered
            import mmap
            mm = mmap.mmap(-1, 1 << 20)
            mm.write(want[:1 << 20])
            addr = ctypes.addressof(ctypes.c_char.from_buffer(mm))
            _ok(L.cvh_host_register(addr, 1 << 20))
            _ok(L.cvh_h2d_async(d_dst, addr, 1 << 20, k_stream, None))
            _ok(L.cvh_stream_synchronize(k_stream))
            _ok(L.cvh_host_unregister(addr))
            assert L.cvh_host_register(None, 4096) != 0
    finally:
        for st in (copy_stream, k_stream):
            if st:
                L.cvh_stream_destroy(st)
        for ev in (copied, done):
            if ev:
                L.cvh_event_destroy(ev)
        for p in (d_wire, d_dst, d_streams, d_desc, d_crc, d_err):
            if p:
                L.cvh_device_free(p)
        for p in (pinned, h_crc, h_err):
            if p:
                L.cvh_pinned_free(p)
        shutil.rmtree(d, ignore_errors=True)


def test_plain_c_host_example_reads_a_file_into_device_memory(cuda):
    """examples/c_host.c: gcc -std=c99 -pedantic, no CUDA headers, linked against the library alone (on the host-side stand-ins: against the
    stand-in library) -- cv_fs_new / cv_open / cv_read_device in steps / cv_verify + cvh_* -- and its output against the oracle."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.environ.get("CV_TEST_MOCK_CUDA_LIB") or os.path.join(root, "curvine_b200", "libcurvine_b200.so")
    d = tempfile.mkdtemp(prefix="cvch", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    bin_dir = tempfile.mkdtemp(prefix="cvch_bin")  # not under /dev/shm, which may be mounted noexec
    try:
        exe = os.path.join(bin_dir, "c_host")
        cc = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(root, "include"), os.path.join(root, "examples", "c_host.c"),
                             "-o", exe, "-L", os.path.dirname(lib), "-l:" + os.path.basename(lib), "-Wl,-rpath," + os.path.dirname(lib)],
                            stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert cc.returncode == 0, cc.stdout
        n, bs, ino = (9 << 20) + 55, 1 << 20, 8502
        with F.MiniWorker(["[MEM]" + d + "/m"]) as w:
            man = w.create_file("/c/file", ino, n, bs)
            want = synth.file_bytes(ino, n, bs)
            open(d + "/ns", "w").write(man)
            open(d + "/conf.toml", "w").write('namespace_manifest = "%s/ns"\n' % d + F.client_conf(b200='fetch_threads = 2\nverify_batch = 2\npinned_slots = 8\ncopy_group = 1\n'))
            r = subprocess.run([exe, d + "/conf.toml", "/c/file", str((2 << 20) + 4096)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
            assert r.returncode == 0, r.stdout
            want_sum = int(clib.crc_blocks(1, np.frombuffer(want, dtype=np.uint8), bs).astype(np.uint64).sum())
            nb = (n + bs - 1) // bs
            # the steps of 2 MiB + 4 KiB cut blocks in the middle: only blocks read whole in one call are compared with the manifest
            fields = r.stdout.split()
            assert fields[:4] == ["bytes", str(n), "of", str(n)] and fields[fields.index("bad") + 1] == "0", r.stdout
            assert fields[fields.index("head") + 1:] == ["%02x" % b for b in want[:16]], r.stdout
            assert int(fields[fields.index("verified") + 1]) <= nb
            r = subprocess.run([exe, d + "/conf.toml", "/c/file"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
            fields = r.stdout.split()
            assert r.returncode == 0 and int(fields[fields.index("sum_crc") + 1]) == want_sum and int(fields[fields.index("verified") + 1]) == nb, r.stdout
            r = subprocess.run([exe, d + "/conf.toml", "/c/nope"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=60)
            assert r.returncode == 1 and "cv_open" in r.stdout and "-8" in r.stdout, r.stdout   # FileNotFound, reported through cv_last_error
    finally:
        shutil.rmtree(d, ignore_errors=True)
        shutil.rmtree(bin_dir, ignore_errors=True)
