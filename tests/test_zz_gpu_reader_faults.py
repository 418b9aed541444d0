"""Fault injection and cache-policy checks of the GPU reader through the C ABI (dead workers, fail-over, recovery, registration cache
admission).  Collected last (zz) so the established parity suites run first; runs on an H100 (`-m gpu`) and, through
tests/test_ingest_pipeline_cpu.py, against the mock runtime on CPU."""
import os
import threading
import time

import numpy as np
import pytest

from curvine_b200 import fs as F
from oracle import clib, layout, synth
from test_gpu_reader import _conf, _dev_buf, cluster  # noqa: F401  (same fixtures and knobs as the parity suite)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("min_age,want_hits", [("60s", 16), ("0ms", 0)])
def test_registration_cache_is_scan_resistant(cuda, cluster, min_age, want_hits):
    """A file twice the size of the registration cache, re-read sequentially in quarter-file calls.  Plain LRU
    (register_min_age = 0) evicts every group just before the scan comes back to it: 0 hits, registration paid every pass.
    The default admission rule keeps the first cache-full of groups registered (recently used mappings are not displaced by
    newcomers, the rest of the file keeps going through the pinned ring): half the groups hit on every later pass, and the
    cache never holds more than register_cache bytes.  Bytes and CRCs are the same either way."""
    import torch
    w, _ = cluster
    n, bs, ino = 32 << 20, 1 << 20, 7300 + want_hits
    man = w.create_file("/scan%d" % want_hits, ino, n, bs)
    want = synth.file_bytes(ino, n, bs)
    conf = _conf(True, 1, zero_copy=True, copy_group=2, register_threads=0, register_cache="16MB").rstrip("\n") + '\nregister_min_age = "%s"\n' % min_age
    with F.CurvineFileSystem(conf) as fs:
        fs.load_namespace(man)
        for rep in range(3):
            r = fs.open("/scan%d" % want_hits)
            dst = _dev_buf(n, cuda)
            for q in range(4):
                assert r.read_device(dst.data_ptr() + q * (n // 4), n // 4, torch.cuda.current_stream().cuda_stream) == n // 4
                assert r.verify()[1] == 0  # also releases the mappings this call held
            torch.cuda.synchronize()
            assert dst.cpu().numpy().tobytes() == want
            st = r.device_stats()
            r.complete()
        assert st["reg_hits"] == want_hits, st
        assert st["reg_bytes"] <= 16 << 20, st
        assert (st["reg_rejected"] > 0) == (want_hits > 0), st


@pytest.mark.parametrize("sc", [True, False])
def test_device_read_fails_over_to_the_next_replica_and_reports_dead_workers(cuda, tmp_path_factory, sc):
    """block_reader.rs:217-254 for the device path: a block whose first replica does not answer is fetched from the next one
    (every fetch thread fails over on its own); when no replica answers the call fails with kind IO -- no hang, no partial
    success -- and the same filesystem handle works again once a worker is back."""
    import shutil
    import torch
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    root = __import__("pathlib").Path(__import__("tempfile").mkdtemp(prefix="cvha", dir=base))
    d1, d2 = root / "w1", root / "w2"
    n, bs, ino = (12 << 20) + 333, 1 << 20, 7400 + int(sc)
    w1 = F.MiniWorker(["[MEM]" + str(d1)])
    w2 = None
    try:
        man = w1.create_file("/ha", ino, n, bs)
        shutil.copytree(str(d1), str(d2))
        w2 = F.MiniWorker(["[MEM]" + str(d2)])  # rescans active/ on start
        want = synth.file_bytes(ino, n, bs)
        man2 = "\n".join(l + ",localhost:%d:2" % w2.port if l.startswith("block ") else l for l in man.splitlines())
        w1.stop()  # the first replica of every block is gone before the read starts
        with F.CurvineFileSystem(_conf(sc, 1, "256KB", threads=4)) as fs:
            fs.load_namespace(man2)
            r = fs.open("/ha")
            dst = _dev_buf(n, cuda)
            assert r.read_device(dst.data_ptr(), n, torch.cuda.current_stream().cuda_stream) == n
            s, bad, ver = r.verify()
            torch.cuda.synchronize()
            assert bad == 0 and ver == (n + bs - 1) // bs and dst.cpu().numpy().tobytes() == want
            r.complete()
            assert w2.metrics()["read_blocks_local" if sc else "read_blocks_remote"] >= ver
            # now nobody answers
            w2.stop()
            r = fs.open("/ha")
            with pytest.raises(F.FsError) as ei:
                r.read_device(dst.data_ptr(), n, torch.cuda.current_stream().cuda_stream)
            assert ei.value.kind == 1, (ei.value.kind, ei.value.msg)
            r.complete()
            # a worker comes back on the second replica's address: the handle recovers (broken connections were not pooled)
            w2 = F.MiniWorker(["[MEM]" + str(d2)], port=w2.port)
            r = fs.open("/ha")
            dst2 = _dev_buf(n, cuda)
            assert r.read_device(dst2.data_ptr(), n, torch.cuda.current_stream().cuda_stream) == n
            assert r.verify()[1] == 0
            torch.cuda.synchronize()
            assert dst2.cpu().numpy().tobytes() == want
            r.complete()
    finally:
        w1.stop()
        if w2 is not None:
            w2.stop()
        shutil.rmtree(str(root), ignore_errors=True)




@pytest.mark.parametrize("sc", [True, False])
def test_worker_dying_in_the_middle_of_a_device_read_fails_the_call_cleanly(cuda, sc):
    """The only replica goes away while fetch threads are in flight: the call must come back (no thread stuck on a ring slot or
    a socket) with an error, or complete if it had already fetched everything; afterwards the same handle reads the file again
    from a restarted worker, bit-exact."""
    import shutil
    import torch
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    root = __import__("pathlib").Path(__import__("tempfile").mkdtemp(prefix="cvdie", dir=base))
    n, bs, ino = 96 << 20, 1 << 20, 7500 + int(sc)
    w = F.MiniWorker(["[MEM]" + str(root / "w")])
    try:
        man = w.create_file("/die", ino, n, bs)
        want = synth.file_bytes(ino, n, bs)
        port = w.port
        with F.CurvineFileSystem(_conf(sc, 1, "256KB", threads=4, batch=4)) as fs:
            fs.load_namespace(man)
            dst = _dev_buf(n, cuda)
            out = {}

            def reader():
                r = fs.open("/die")
                try:
                    out["got"] = r.read_device(dst.data_ptr(), n, 0)
                    out["verify"] = r.verify()
                except F.FsError as e:
                    out["err"] = e
                finally:
                    try:
                        r.complete()
                    except F.FsError as e:  # the pending results of a failed call may surface here
                        out.setdefault("err", e)

            t = threading.Thread(target=reader)
            t.start()
            time.sleep(0.02)
            w.stop()
            t.join(timeout=60)
            assert not t.is_alive(), "device read still blocked 60 s after its worker went away"
            assert ("err" in out) or out.get("got") == n, out
            if "err" in out:
                assert out["err"].kind in (1, 10000), (out["err"].kind, out["err"].msg)
            w = F.MiniWorker(["[MEM]" + str(root / "w")], port=port)
            r = fs.open("/die")
            dst2 = _dev_buf(n, cuda)
            assert r.read_device(dst2.data_ptr(), n, torch.cuda.current_stream().cuda_stream) == n
            s, bad, ver = r.verify()
            torch.cuda.synchronize()
            assert bad == 0 and ver == n // bs and dst2.cpu().numpy().tobytes() == want
            r.complete()
    finally:
        w.stop()
        shutil.rmtree(str(root), ignore_errors=True)


def test_two_threads_read_different_files_through_one_handle(cuda, cluster):
    """lib_filesystem.rs:25-40: a filesystem handle is shareable between threads (a reader handle is not).  Two threads, two
    readers, one context: the device reads serialise inside the library; both files land bit-exact with the right CRC sums."""
    import torch
    w, _ = cluster
    bs = 1 << 20
    specs = [("/mt_a", 7601, (24 << 20) + 11), ("/mt_b", 7602, (17 << 20) + 4097)]
    man = "".join(w.create_file(p, ino, n, bs) for p, ino, n in specs)
    with F.CurvineFileSystem(_conf(True, 1, zero_copy=True, copy_group=2, register_threads=2, register_cache="128MB")) as fs:
        fs.load_namespace(man)
        res, errs = {}, []

        def run(p, ino, n):
            try:
                want = synth.file_bytes(ino, n, bs)
                for rep in range(3):
                    r = fs.open(p)
                    dst = _dev_buf(n + 32, cuda)
                    assert r.read_device(dst.data_ptr(), n, 0) == n
                    s, bad, ver = r.verify()
                    torch.cuda.synchronize()
                    assert bad == 0 and ver == (n + bs - 1) // bs
                    assert dst[:n].cpu().numpy().tobytes() == want and (dst[n:] == 0xA5).all()
                    assert s == int(clib.crc_blocks(1, np.frombuffer(want, dtype=np.uint8), bs).astype(np.uint64).sum())
                    r.complete()
                res[p] = True
            except Exception as e:  # noqa: BLE001
                errs.append((p, repr(e)))

        ts = [threading.Thread(target=run, args=sp) for sp in specs]
        for t in ts:
            t.start()
        for t in ts:
            t.join(timeout=120)
        assert not errs and len(res) == 2, errs


@pytest.mark.parametrize("sc", [True, False])
def test_vanished_block_file_and_bad_arguments(cuda, cluster, sc):
    """A block file that disappeared after the manifest was written: the worker answers Open with an error (remote) or the
    client cannot read the path it was given (short-circuit) -> the call fails with a reference error kind, names the block, and
    leaves the handle usable.  A negative seek and a destination that is not device memory are refused up front."""
    import torch
    w, d = cluster
    n, bs, ino = 6 << 20, 1 << 20, 7700 + int(sc)
    man = w.create_file("/gone%d" % sc, ino, n, bs) + w.create_file("/fine%d" % sc, ino + 50, n, bs)
    os.remove(layout.block_path(str(d / "mem" / "curvine"), layout.create_block_id(ino, 3)))
    with F.CurvineFileSystem(_conf(sc)) as fs:
        fs.load_namespace(man)
        r = fs.open("/gone%d" % sc)
        dst = _dev_buf(n, cuda)
        with pytest.raises(F.FsError) as ei:
            r.read_device(dst.data_ptr(), n, 0)
            r.verify()
        assert ei.value.kind in (1, 10000), (ei.value.kind, ei.value.msg)
        with pytest.raises(F.FsError):
            r.seek(-1)
        try:
            r.complete()
        except F.FsError:
            pass
        r = fs.open("/fine%d" % sc)
        assert r.read_device(dst.data_ptr(), n, torch.cuda.current_stream().cuda_stream) == n
        assert r.verify()[1:] == (0, n // bs)
        torch.cuda.synchronize()
        assert dst.cpu().numpy().tobytes() == synth.file_bytes(ino + 50, n, bs)
        r.complete()


def _own_worker(extra_worker):
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    root = __import__("pathlib").Path(__import__("tempfile").mkdtemp(prefix="cvhbm", dir=base))
    return F.MiniWorker(["[MEM]" + str(root / "mem")], extra_worker=extra_worker), root


def test_hbm_tier_capacity_lru_eviction_and_blocks_being_read():
    """[worker] hbm_capacity: the tier never holds more than its capacity; loads evict the least recently READ block nobody is
    reading; a block with an open read context survives its own eviction (the context keeps the device memory alive) and keeps
    serving the right bytes; evicted blocks are served from their files again; a block larger than the tier is refused."""
    import shutil
    bs, ino = 1 << 20, 7800
    w, root = _own_worker('hbm_capacity = "3MB"')
    try:
        n = 6 * bs
        man = w.create_file("/t", ino, n, bs) + w.create_file("/big", ino + 1, 4 << 20, 4 << 20)
        want = synth.file_bytes(ino, n, bs)
        ids = [layout.create_block_id(ino, i) for i in range(6)]
        for i in range(3):
            w.hbm_load(ids[i], 0)
        t = w.hbm_tier()
        assert t["resident_blocks"] == 3 and t["resident_bytes"] == 3 * bs and t["capacity"] == 3 << 20 and t["evictions"] == 0
        with F.CurvineFileSystem(F.client_conf(short_circuit=False, read_chunk_size="64KB")) as fs:
            fs.load_namespace(man)
            r0 = fs.open("/t")
            assert r0.read(1000) == want[:1000]  # block 0 now has an open read context served from HBM (and is the most recently read)
            hbm_reads = w.hbm_stats()["reads_from_hbm"]
            assert hbm_reads >= 1
            w.hbm_load(ids[3], 0)  # evicts block 1 (coldest that nobody reads)
            w.hbm_load(ids[4], 0)  # evicts block 2
            t = w.hbm_tier()
            assert t["resident_blocks"] == 3 and t["evictions"] == 2 and t["resident_bytes"] == 3 * bs, t
            w.hbm_load(ids[5], 0)  # block 0 is the coldest but is being read: block 3 goes instead
            t = w.hbm_tier()
            assert t["evictions"] == 3 and t["resident_bytes"] <= 3 << 20, t
            assert r0.read_full(n) == want[1000:]  # the open context on block 0 kept working; blocks 1-3 came from files, 4-5 from HBM
            r0.complete()
            with pytest.raises(F.FsError):
                w.hbm_load(layout.create_block_id(ino + 1, 0), 0)  # 4 MiB block, 3 MB tier
            assert w.hbm_tier()["refused"] == 1
            r = fs.open("/t")
            assert r.read_full(n) == want
            r.complete()
        assert w.hbm_stats()["reads_from_hbm"] > hbm_reads
    finally:
        w.stop()
        shutil.rmtree(str(root), ignore_errors=True)


def test_hbm_tier_promotes_blocks_that_are_read_remotely(cuda):
    """[worker] hbm_promote_after = 2: the third framed read of a block hands it to the tier's promoter thread and is itself still
    served from the store (promotion is asynchronous: the promoting read does not pay for it); once the promoter is done every
    further framed read is served from HBM (frames packed by K4); short-circuit reads never count; bytes are identical before and
    after; the device reader sees the same CRCs through K2."""
    import shutil
    import torch
    bs, ino, n = 1 << 20, 7900, (3 << 20) + 99
    w, root = _own_worker('hbm_promote_after = 2\nhbm_capacity = "64MB"')
    try:
        man = w.create_file("/p", ino, n, bs)
        want = synth.file_bytes(ino, n, bs)
        with F.CurvineFileSystem(_conf(False, 1, "256KB")) as fs:
            fs.load_namespace(man)
            for rep in range(2):
                r = fs.open("/p")
                assert r.read_full(n) == want
                r.complete()
                assert w.hbm_tier()["promotions"] == 0 and w.hbm_stats()["reads_from_hbm"] == 0
            r = fs.open("/p")
            dst = _dev_buf(n, cuda)
            assert r.read_device(dst.data_ptr(), n, 0) == n  # third remote read of every block: queued for promotion, served from the store
            s, bad, ver = r.verify()
            torch.cuda.synchronize()
            assert bad == 0 and ver == 4 and dst.cpu().numpy().tobytes() == want
            r.complete()
            w.hbm_drain()
            t = w.hbm_tier()
            assert t["promotions"] == 4 and t["resident_blocks"] == 4 and t["resident_bytes"] == n, t
            assert w.hbm_stats()["reads_from_hbm"] == 0
            dst.fill_(0)
            r = fs.open("/p")
            assert r.read_device(dst.data_ptr(), n, 0) == n  # now resident: K4-packed frames out of HBM, unpacked by K2
            s, bad, ver = r.verify()
            torch.cuda.synchronize()
            assert bad == 0 and ver == 4 and dst.cpu().numpy().tobytes() == want
            r.complete()
            assert w.hbm_stats()["reads_from_hbm"] == 4
            r = fs.open("/p")
            assert r.read_full(n) == want
            r.complete()
            assert w.hbm_stats()["reads_from_hbm"] == 8 and w.hbm_tier()["promotions"] == 4
        with F.CurvineFileSystem(_conf(True, 1)) as fs:  # short-circuit readers go to the file, resident or not
            fs.load_namespace(man)
            r = fs.open("/p")
            assert r.read_full(n) == want
            r.complete()
            assert w.hbm_stats()["reads_from_hbm"] == 8
    finally:
        w.stop()
        shutil.rmtree(str(root), ignore_errors=True)


@pytest.mark.parametrize("sc,zero_copy", [(True, False), (True, True), (False, False)])
def test_thousands_of_small_blocks_cycle_the_ring_many_times(cuda, cluster, sc, zero_copy):
    """3,000 blocks of 20 KiB + a ragged tail through a ring of a few slots: every super-slot is handed over hundreds of times
    between fetch threads, the copy stream and the verifier (released/copied hand-shake, verify batches that straddle slot reuse)."""
    import torch
    w, _ = cluster
    bs = 20 * 1024
    n, ino = 3000 * bs + 777, 8300 + 2 * int(sc) + int(zero_copy)
    man = w.create_file("/many%d%d" % (sc, zero_copy), ino, n, bs, threads=8)
    want = synth.file_bytes(ino, n, bs)
    with F.CurvineFileSystem(_conf(sc, 1, "8KB", threads=6, batch=5, zero_copy=zero_copy, copy_group=3, register_threads=2, register_cache="128MB")) as fs:
        fs.load_namespace(man)
        for rep in range(2):
            r = fs.open("/many%d%d" % (sc, zero_copy))
            dst = _dev_buf(n + 8, cuda)
            assert r.read_device(dst.data_ptr(), n, torch.cuda.current_stream().cuda_stream) == n
            s, bad, ver = r.verify()
            torch.cuda.synchronize()
            assert bad == 0 and ver == 3001
            assert dst[:n].cpu().numpy().tobytes() == want and (dst[n:] == 0xA5).all()
            assert s == int(clib.crc_blocks(1, np.frombuffer(want, dtype=np.uint8), bs).astype(np.uint64).sum())
            r.complete()
            fs.wait_registered()


def test_read_many_with_empty_files_holes_and_hundreds_of_files(cuda, cluster):
    """cv_read_many_device over 300 files in one pass: lengths from 0 to a few blocks, some with hole blocks; every file lands at
    its own offset, the CRC sum is the sum over all blocks that have a manifest CRC, nothing else in the destination is touched."""
    import torch
    w, _ = cluster
    rng = np.random.default_rng(5)
    bs = 64 * 1024
    specs, mans, off, offs = [], [], 0, []
    for i in range(300):
        ln = int(rng.choice([0, 1, 4095, bs - 1, bs, bs + 1, 3 * bs + 17]))
        hole = (i % 17 == 3 and ln > bs)
        mans.append(w.create_file("/rm/f%d" % i, 8400 + i, ln, bs, mode=2 if hole else 0, hole_every=2 if hole else 0, threads=1))
        data = bytearray(synth.file_bytes(8400 + i, ln, bs))
        if hole:
            for b in range(1, (ln + bs - 1) // bs, 2):
                data[b * bs:(b + 1) * bs] = bytes(min(bs, ln - b * bs))
        specs.append(bytes(data))
        offs.append(off)
        off += ln + int(rng.integers(0, 9))
    with F.CurvineFileSystem(_conf(True, 1, threads=6, batch=7, copy_group=4)) as fs:
        fs.load_namespace("".join(mans))
        dst = _dev_buf(off + 64, cuda)
        tot, s, bad, ver = fs.read_many_device(["/rm/f%d" % i for i in range(300)], dst.data_ptr(), offs, off + 64, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert tot == sum(len(x) for x in specs) and bad == 0
        host = dst.cpu().numpy()
        expect = np.full(off + 64, 0xA5, dtype=np.uint8)
        for o, x in zip(offs, specs):
            expect[o:o + len(x)] = np.frombuffer(x, dtype=np.uint8)
        assert host.tobytes() == expect.tobytes()


@pytest.mark.parametrize("sc,zero_copy,seed", [(True, True, 1), (True, False, 2), (False, False, 3)])
def test_random_mixed_host_and_device_op_sequences(cuda, cluster, sc, zero_copy, seed):
    """Seeded random walks over one reader: seek / host read / device read of random sizes (block-crossing, past EOF, zero), host
    and device reads sharing the one position (reader.rs:50-141 semantics for both).  Every step is checked against the file bytes;
    verify() must never report a bad block."""
    import torch
    w, _ = cluster
    bs = 256 * 1024
    n, ino = 23 * bs + 12345, 8600 + seed
    man = w.create_file("/walk%d" % seed, ino, n, bs)
    want = synth.file_bytes(ino, n, bs)
    rng = np.random.default_rng(seed)
    with F.CurvineFileSystem(_conf(sc, 1, "64KB", threads=3, batch=3, zero_copy=zero_copy, copy_group=2, register_threads=1, register_cache="64MB")) as fs:
        fs.load_namespace(man)
        r = fs.open("/walk%d" % seed)
        pos = 0
        for step in range(120):
            op = rng.integers(0, 4)
            if op == 0:
                pos = int(rng.choice([0, n, n - 1, int(rng.integers(0, n)), int(rng.integers(0, n)), n + 5000]))
                r.seek(pos)
                assert r.pos() == pos
            elif op == 1:
                k = int(rng.choice([0, 1, 100, 65536, bs + 1, 3 * bs]))
                got = r.read(k)
                exp = want[pos:pos + k] if pos < n else b""
                # Reader::read returns at most the current chunk: a prefix of the expectation, non-empty unless at EOF or k == 0
                assert exp.startswith(got) and (len(got) > 0 or k == 0 or pos >= n), (step, pos, k, len(got))
                pos += len(got)
            else:
                cap = int(rng.choice([0, 7, 4096, bs - 3, bs, 2 * bs + 11, 5 * bs]))
                dst = _dev_buf(cap + 16, cuda)
                got = r.read_device(dst.data_ptr(), cap, torch.cuda.current_stream().cuda_stream)
                torch.cuda.synchronize()
                exp = want[pos:pos + cap] if pos < n else b""
                assert got == len(exp), (step, pos, cap, got)
                host = dst.cpu().numpy()
                assert host[:got].tobytes() == exp and (host[got:] == 0xA5).all()
                pos += got
            assert r.pos() == pos
        assert r.verify()[1] == 0
        r.complete()


@pytest.mark.timeout(120)
def test_single_fetch_thread_framed_read_larger_than_the_ring_does_not_wait_for_itself(cuda, cluster):
    """ADVICE r1 (medium): with fetch_threads = 1 the fetch worker used to run inline on the calling thread; a framed (verbatim)
    group's ring slot is only released by the verifier, which runs on that same thread afterwards -- once the copy groups
    outnumbered the ring's super-slots the inline worker waited for itself forever.  64 x 1 MiB framed blocks through 6 super-slots."""
    import torch
    w, _ = cluster
    n, bs, ino = 64 << 20, 1 << 20, 7990
    man = w.create_file("/one_thread", ino, n, bs)
    want = synth.file_bytes(ino, n, bs)
    with F.CurvineFileSystem(_conf(False, 1, "1MB", threads=1, batch=4, copy_group=2)) as fs:
        fs.load_namespace(man)
        r = fs.open("/one_thread")
        dst = _dev_buf(n, cuda)
        assert r.read_device(dst.data_ptr(), n, torch.cuda.current_stream().cuda_stream) == n
        s, bad, ver = r.verify()
        torch.cuda.synchronize()
        assert bad == 0 and ver == 64
        assert dst.cpu().numpy().tobytes() == want
        r.complete()
