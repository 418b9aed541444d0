"""Strided device reads (cv_readv_strided_device), the K3 kernel over 2D descriptors (cvk_gather_strided) and sliced safetensors loads on
the GPU: every row of every range lands at its destination with the bytes between rows untouched, every touched block is verified whole
(columns no rank asked for included), and each tensor-parallel rank's load_file(slices=...) is its narrow() of the whole tensor.  Runs on
the host-side stand-ins too (tests/mock_cuda, tests/simt_emu), where "device memory" is host memory."""
import os
import shutil
import tempfile

import numpy as np
import pytest

from curvine_b200 import fs as F
from curvine_b200 import safetensors as ST
from oracle import clib, layout, synth
from test_kernels_gpu import _rand, _to_dev

pytestmark = pytest.mark.gpu
MOCK = bool(os.environ.get("CV_TEST_MOCK_CUDA_LIB"))
BS = 64 << 10
GUARD = 0x5A


# ---- cvk_gather_strided against numpy

def _gather_case(rng, src_len, n_desc, max_rows, max_len):
    segs, pos = [], 16
    for _ in range(n_desc):
        ln = int(rng.integers(1, max_len + 1))
        rows = int(rng.integers(1, max_rows + 1))
        sp = ln + int(rng.integers(0, 64))
        if (rows - 1) * sp + ln >= src_len - 32:
            rows = max(1, (src_len - 32 - ln) // sp)
        so = int(rng.integers(0, src_len - (rows - 1) * sp - ln)) | 1
        if so + (rows - 1) * sp + ln > src_len:
            so -= 1
        dp = ln + int(rng.integers(1, 40))  # guard bytes between destination rows
        do = pos + (int(rng.integers(0, 16)) | 1)
        segs.append((so, do, ln, rows, sp, dp))
        pos = do + (rows - 1) * dp + ln + 8
    return segs, pos + 64


def _check_gather(cuda, src, d_src, segs, size):
    import torch
    from curvine_b200 import kernels as K
    want = np.full(size, GUARD, dtype=np.uint8)
    for so, do, ln, rows, sp, dp in segs:
        for k in range(rows):
            want[do + k * dp:do + k * dp + ln] = src[so + k * sp:so + k * sp + ln]
    dst = torch.full((size,), GUARD, dtype=torch.uint8, device=cuda)
    K.gather_strided(d_src, K.strided_segs_to_device(segs, cuda) if segs else None, len(segs), sum(s[2] * s[3] for s in segs), dst)
    torch.cuda.synchronize()
    assert np.array_equal(dst.cpu().numpy(), want)


def test_gather_strided_matches_numpy(cuda):
    src = _rand(1 << 20, 31)
    d_src = _to_dev(src, cuda)
    rng = np.random.default_rng(4)
    _check_gather(cuda, src, d_src, [], 256)                                       # n = 0
    _check_gather(cuda, src, d_src, [(3, 5, 1, 1, 1, 1)], 64)                      # one byte
    _check_gather(cuda, src, d_src, [(1, 7, 40000, 3, 40001, 40011)], 3 * 40011 + 64)  # rows longer than one walker segment
    for n_desc, max_rows, max_len in ((1, 300, 40), (7, 50, 5000), (40, 20, 300)):
        segs, size = _gather_case(rng, len(src), n_desc, max_rows, max_len)
        _check_gather(cuda, src, d_src, segs, size)
    segs, size = _gather_case(rng, len(src), 5, 30, 70)
    segs.append((9, size, 0, 1000, 4, 4))  # empty rows: nothing to copy
    _check_gather(cuda, src, d_src, segs, size + 8)


def test_gather_strided_splits_many_rows_into_trains(cuda):
    """cvk_tune(6, r) lowers the rows per train: a descriptor with more rows than that, and descriptors straddling a train edge, land
    exactly as in one train"""
    from curvine_b200 import _lib
    src = _rand(1 << 18, 8)
    d_src = _to_dev(src, cuda)
    L = _lib.lib()
    _lib.check(L.cvk_tune(6, 7))
    try:
        _check_gather(cuda, src, d_src, [(1, 3, 5, 30, 17, 9)], 30 * 9 + 16)
        segs = [(11, 5, 3, 4, 5, 4), (101, 40, 20, 9, 33, 21), (1001, 300, 2, 1, 0, 2), (2001, 311, 7, 16, 7, 8)]
        _check_gather(cuda, src, d_src, segs, 311 + 16 * 8 + 16)
    finally:
        _lib.check(L.cvk_tune(6, 0))


# ---- strided reads through the reader

def _conf(sc, copy_group=1, zero_copy=False, arena_dir=None):
    # 8 ring slots: at most 8 boundary blocks are staged per round, so the range sets below take several rounds
    b200 = 'fetch_threads = 2\nverify_batch = 2\npinned_slots = 8\ncopy_group = %d\ngpu_chunk_size = "32KB"\nzero_copy = %s\n' % (
        copy_group, "true" if zero_copy else "false")
    if arena_dir:
        b200 += 'register_threads = 2\narena_register_slice = "4MB"\narena_preregister = ["%s"]\n' % arena_dir
    return F.client_conf(short_circuit=sc, b200=b200)


@pytest.fixture(scope="module")
def cluster():
    d = tempfile.mkdtemp(prefix="cvst", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    plain = F.MiniWorker(["[MEM]" + d + "/mem"])
    arena = F.MiniWorker(["[MEM:16MB]" + d + "/arena"], extra_worker='mem_arena = true\narena_segment = "8MB"\n')
    yield plain, arena, d
    plain.stop()
    arena.stop()
    shutil.rmtree(d, ignore_errors=True)


MODES = {"files": dict(sc=True), "framed": dict(sc=False), "arena": dict(sc=True, zero_copy=True)}


def _range_sets(n):
    return [
        [(5001, 3000, (n - 8001) // 12000 + 1, 12000)],                         # a column of a row-major matrix: rows across block edges
        [(100, 2 * BS + 300, 4, 3 * BS + 7), (13 * BS, BS, 1, 0)],              # long rows with whole blocks inside; a plain range
        [(3, 1, 300, 997), (300 * 997 + 10, 64, 50, 64)],                       # 1-byte rows; back-to-back rows
        [(17, 100, 3, 7 * BS + 3), (n - 50, 50, 1, 0), (9, 0, 4, 10)],        # sparse rows; the last bytes; an empty range
    ]


def _place(rng, ranges, cuda):
    """destinations at odd offsets with guard bytes around and between rows -> (pool, [(dst offset, dst_pitch)])"""
    import torch
    at, out = 64, []
    for off, L, R, P in ranges:
        at += int(rng.integers(1, 16)) | 1
        dp = L + (int(rng.integers(1, 9)) if R > 1 else 0)
        out.append((at, dp))
        at += max(0, R - 1) * dp + L + 16
    return torch.full((at + 64,), GUARD, dtype=torch.uint8, device=cuda), out


def _expect(pool_len, ranges, dst, want):
    exp = np.full(pool_len, GUARD, dtype=np.uint8)
    for (off, L, R, P), (at, dp) in zip(ranges, dst):
        for k in range(R if L else 0):
            exp[at + k * dp:at + k * dp + L] = want[off + k * P:off + k * P + L]
    return exp


def _touched(ranges):
    return sorted({b for off, L, R, P in ranges if L for k in range(R) for b in range((off + k * P) // BS, (off + k * P + L - 1) // BS + 1)})


def _fs_for(cluster, mode, man, copy_group):
    plain, arena, d = cluster
    fs = F.CurvineFileSystem(_conf(copy_group=copy_group, arena_dir=d + "/arena" if mode == "arena" else None, **MODES[mode]))
    fs.load_namespace(man)
    if mode == "arena":
        fs.preregister()
        fs.wait_registered()
    return fs


@pytest.mark.parametrize("copy_group", [1, 4])
@pytest.mark.parametrize("mode", list(MODES))
def test_strided_rows_land_at_their_destinations_and_touched_blocks_verify_whole(cuda, cluster, mode, copy_group):
    import torch
    plain, arena, _ = cluster
    n, ino = 24 * BS - 777, 9810 + 2 * list(MODES).index(mode) + copy_group // 4
    w = arena if mode == "arena" else plain
    man = w.create_file("/st/%s%d" % (mode, copy_group), ino, n, BS, threads=2)
    want = np.frombuffer(synth.file_bytes(ino, n, BS), dtype=np.uint8)
    crcs = clib.crc_blocks(1, want, BS).astype(np.uint64)
    rng = np.random.default_rng(6 + copy_group)
    with _fs_for(cluster, mode, man, copy_group) as fs:
        for ranges in _range_sets(n):
            pool, dst = _place(rng, ranges, cuda)
            base = pool.data_ptr()
            r = fs.open("/st/%s%d" % (mode, copy_group))
            r.seek(321)
            rs = [(off, L, R, P, base + at, dp) for (off, L, R, P), (at, dp) in zip(ranges, dst)]
            got = r.readv_strided_device(rs, torch.cuda.current_stream().cuda_stream)
            assert got == sum(L * R for _, L, R, _ in ranges) and r.pos() == 321
            s, bad, ver = r.verify()
            torch.cuda.synchronize()
            assert np.array_equal(pool.cpu().numpy(), _expect(pool.numel(), ranges, dst, want)), ranges
            touched = _touched(ranges)
            assert bad == 0 and ver == len(touched), (ver, touched)
            assert s == int(crcs[touched].sum())
            spans, nb, fetch = r.readv_strided_plan(rs)
            assert nb == len(touched) and fetch == sum(min(BS, n - b * BS) for b in touched)
            r.complete()


def _flip(path, off):
    with open(path, "r+b") as f:
        f.seek(off)
        b = f.read(1)
        f.seek(off)
        f.write(bytes([b[0] ^ 0x20]))


@pytest.mark.parametrize("sc", [True, False])
def test_a_corrupt_byte_in_a_column_nobody_asked_for_is_caught_in_touched_blocks_only(cuda, cluster, sc):
    import torch
    plain, _, d = cluster
    n, ino = 8 * BS, 9830 + int(sc)
    man = plain.create_file("/st/bad%d" % sc, ino, n, BS, threads=2)
    want = np.frombuffer(synth.file_bytes(ino, n, BS), dtype=np.uint8)
    # rank 1 of 4 of a matrix with 4096-byte rows: columns [1024, 2048) of every row.  Byte 100 of a row is rank 0's.
    for blk in (5, 2):
        _flip(layout.block_path(d + "/mem/curvine", layout.create_block_id(ino, blk)), 4096 * 3 + 100)
    with F.CurvineFileSystem(_conf(sc)) as fs:
        fs.load_namespace(man)
        pool = torch.full((64 * 1024 + 64,), GUARD, dtype=torch.uint8, device=cuda)
        r = fs.open("/st/bad%d" % sc)
        rows = 4 * BS // 4096  # blocks 4..7
        r.readv_strided_device([(4 * BS + 1024, 1024, rows, 4096, pool.data_ptr() + 1, 1024)])
        s, bad, ver = r.verify()
        torch.cuda.synchronize()
        assert bad == 1 and ver == 4
        host = pool.cpu().numpy()
        for k in range(rows):
            assert np.array_equal(host[1 + k * 1024:1 + (k + 1) * 1024], want[4 * BS + k * 4096 + 1024:4 * BS + k * 4096 + 2048])
        assert host[0] == GUARD and host[1 + rows * 1024] == GUARD
        r.complete()
        r = fs.open("/st/bad%d" % sc)  # block 2 is not touched: its corruption is neither fetched nor counted
        r.readv_strided_device([(1024, 1024, 2 * BS // 4096, 4096, pool.data_ptr(), 1024)])
        assert r.verify()[1:] == (0, 2)
        r.complete()


def test_strided_rows_over_hole_blocks_are_zeros(cuda, cluster):
    import torch
    plain, _, _ = cluster
    n, ino = 7 * BS + 5, 9835
    man = plain.create_file("/st/holes", ino, n, BS, mode=2, hole_every=3, threads=2)  # blocks 2 and 5 are holes
    want = np.frombuffer(synth.file_bytes(ino, n, BS), dtype=np.uint8).copy()
    for b in (2, 5):
        want[b * BS:(b + 1) * BS] = 0
    ranges = [(BS + 7, 5000, 9, 20000, 5003)]  # blocks 1..3, the hole 2 among them
    with F.CurvineFileSystem(_conf(True)) as fs:
        fs.load_namespace(man)
        r = fs.open("/st/holes")
        pool, dst = _place(np.random.default_rng(2), [x[:4] for x in ranges], cuda)
        r.readv_strided_device([(off, L, R, P, pool.data_ptr() + at, dp) for (off, L, R, P, _), (at, dp) in zip(ranges, dst)])
        s, bad, ver = r.verify()
        torch.cuda.synchronize()
        assert np.array_equal(pool.cpu().numpy(), _expect(pool.numel(), [x[:4] for x in ranges], dst, want))
        touched = _touched([x[:4] for x in ranges])
        assert 2 in touched and bad == 0 and ver == len([b for b in touched if b not in (2, 5)])
        r.complete()


def test_strided_read_is_ordered_on_the_callers_stream(cuda, cluster):
    import torch
    from test_zzz_stream_order_gpu import CallerStream
    plain, _, _ = cluster
    n, ino = 12 * BS + 99, 9836
    man = plain.create_file("/st/so", ino, n, BS, threads=2)
    want = np.frombuffer(synth.file_bytes(ino, n, BS), dtype=np.uint8)
    ranges = [(77, 3000, 40, 12345), (40 * 12345 + 100, BS, 2, 2 * BS)]
    total = sum(L * R for _, L, R, _ in ranges)
    exp = np.concatenate([want[o + k * P:o + k * P + L] for o, L, R, P in ranges for k in range(R)])
    cs = None
    try:
        with F.CurvineFileSystem(_conf(False)) as fs:
            fs.load_namespace(man)
            cs = CallerStream(torch)
            dst = torch.zeros(total, dtype=torch.uint8, device=cuda)
            out = torch.zeros(total, dtype=torch.uint8, device=cuda)
            slow = torch.zeros(8 << 20, dtype=torch.uint8, device=cuda)
            torch.cuda.synchronize()
            for rnd in range(2):
                for _ in range(4):
                    cs.fill(slow, rnd)
                for v in (0xE0, 0xE1 + rnd):
                    cs.fill(dst, v)  # pending writes to the destinations, enqueued BEFORE the read
                r = fs.open("/st/so")
                at, rs = dst.data_ptr(), []
                for o, L, R, P in ranges:
                    rs.append((o, L, R, P, at, L))
                    at += L * R
                assert r.readv_strided_device(rs, cs.handle) == total
                cs.copy(out, dst)  # enqueued AFTER the read, same stream, no host synchronisation in between
                cs.synchronize()
                assert np.array_equal(out.cpu().numpy(), exp), "round %d: the read is not ordered on the caller's stream" % rnd
                assert r.verify()[1] == 0
                r.complete()
                out.zero_()
    finally:
        if cs is not None:
            cs.close()


def test_destinations_that_are_not_device_memory_are_errors(cuda, cluster):
    import ctypes
    from curvine_b200 import _lib
    plain, _, _ = cluster
    man = plain.create_file("/st/dst", 9837, 4 * BS, BS, threads=2)
    L = _lib.lib()
    import torch
    h = ctypes.c_void_p()
    _lib.check(L.cvh_pinned_alloc(1 << 16, ctypes.byref(h)))
    ok = torch.zeros(64, dtype=torch.uint8, device=cuda)
    try:
        with F.CurvineFileSystem(_conf(True)) as fs:
            fs.load_namespace(man)
            with fs.open("/st/dst") as r:
                with pytest.raises(F.FsError, match="range 1"):
                    r.readv_strided_device([(0, 10, 1, 0, ok.data_ptr(), 10), (100, 10, 3, 20, h.value, 10)])
                with pytest.raises(F.FsError, match="overlap"):
                    r.readv_strided_device([(0, 10, 5, 100, h.value, 10), (50, 10, 5, 100, h.value, 10)])
    finally:
        L.cvh_pinned_free(h)


# ---- sliced safetensors loads

def _tensors(torch):
    g = torch.Generator().manual_seed(11)
    specs = [("embed", torch.bfloat16, (96, 130)), ("norm", torch.float32, (77,)), ("qkv", torch.float16, (3, 40, 257)),
             ("empty", torch.float16, (0, 12)), ("ids", torch.int64, (8, 6)), ("mask", torch.bool, (12, 5, 2)), ("scale", torch.float64, ()),
             ("big", torch.int8, (40, BS // 8 + 3))]
    out = {}
    for name, dt, shape in specs:
        nbytes = int(np.prod(shape, dtype=np.int64)) * dt.itemsize
        raw = torch.randint(0, 2 if dt == torch.bool else 256, (nbytes,), dtype=torch.uint8, generator=g)
        out[name] = raw.view(dt).reshape(shape) if nbytes else torch.empty(shape, dtype=dt)
    return out


def test_sliced_safetensors_equal_narrow_of_the_whole_load(cuda, cluster):
    import torch
    from test_zzz_readv_gpu import _blob, _bytes
    plain, _, _ = cluster
    dev = "cpu" if MOCK else cuda
    src = _tensors(torch)
    blob = _blob(src)
    path = "/st/model.safetensors"
    with F.CurvineFileSystem(_conf(True)) as fs:
        wr = fs.create(path, 9840, BS, plain.port, chunk_size=32768)
        wr.write(blob)
        wr.complete()
        shapes = ST.read_header(fs, path)
        assert {k: tuple(v[1]) for k, v in shapes.items()} == {k: tuple(t.shape) for k, t in src.items()}
        full = ST.load_file(fs, path, device=dev)
        for name, t in src.items():
            assert _bytes(full[name]) == _bytes(t)
        for world in (1, 2, 4):
            for dim in (0, 1, -1):
                parts = {}
                for rank in range(world):
                    slices = {}
                    for name, (_, shape) in shapes.items():
                        if len(shape) == 0 or (dim >= 0 and dim >= len(shape)):
                            continue
                        size = shape[dim]
                        slices[name] = (dim, rank * size // world, (rank + 1) * size // world)
                    if not MOCK:
                        torch.cuda.synchronize()
                        torch.cuda.reset_peak_memory_stats()
                        before = torch.cuda.memory_allocated()
                    got = ST.load_file(fs, path, device=dev, slices=slices)
                    if not MOCK and world > 1:
                        assert torch.cuda.max_memory_allocated() - before < len(blob)
                    for name, t in got.items():
                        if name in slices:
                            d, a, b = slices[name]
                            exp = full[name].narrow(d, a, b - a)
                            assert tuple(t.shape) == tuple(exp.shape) and t.is_contiguous(), (name, world, dim)
                            assert _bytes(t) == _bytes(exp.contiguous()), (name, world, rank, dim)
                            parts.setdefault(name, []).append(t)
                        else:
                            assert _bytes(t) == _bytes(full[name])
                    del got
                for name, ts in parts.items():
                    assert _bytes(torch.cat(ts, dim=slices[name][0])) == _bytes(full[name]), (name, world, dim)
