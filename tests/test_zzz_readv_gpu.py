"""Vectored device reads (cv_readv_device) and the safetensors loader on the GPU: bytes of many ranges land at many destinations, every
block a range touches is verified whole (bytes no range wants included), and safetensors files come back as the tensors that were
written.  Runs on the host-side stand-ins too (tests/mock_cuda, tests/simt_emu), where "device memory" is host memory."""
import os
import shutil
import tempfile

import numpy as np
import pytest

from curvine_b200 import fs as F
from curvine_b200 import safetensors as ST
from oracle import clib, layout, synth

pytestmark = pytest.mark.gpu
MOCK = bool(os.environ.get("CV_TEST_MOCK_CUDA_LIB"))
BS = 256 << 10
GUARD = 0xA5


def _conf(sc, zero_copy=False, arena_dir=None):
    # 8 ring slots: at most 8 boundary blocks are staged per round, so the larger range sets below take several rounds
    b200 = 'fetch_threads = 2\nverify_batch = 2\npinned_slots = 8\ncopy_group = 1\ngpu_chunk_size = "128KB"\nzero_copy = %s\n' % (
        "true" if zero_copy else "false")
    if arena_dir:
        b200 += 'register_threads = 2\narena_register_slice = "4MB"\narena_preregister = ["%s"]\n' % arena_dir
    return F.client_conf(short_circuit=sc, b200=b200)


@pytest.fixture(scope="module")
def cluster():
    d = tempfile.mkdtemp(prefix="cvrv", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    plain = F.MiniWorker(["[MEM]" + d + "/mem"])
    arena = F.MiniWorker(["[MEM:32MB]" + d + "/arena"], extra_worker='mem_arena = true\narena_segment = "16MB"\n')
    yield plain, arena, d
    plain.stop()
    arena.stop()
    shutil.rmtree(d, ignore_errors=True)


MODES = {"files": dict(sc=True), "framed": dict(sc=False), "arena": dict(sc=True, zero_copy=True)}


def _fs_for(cluster, mode, man):
    plain, arena, d = cluster
    fs = F.CurvineFileSystem(_conf(arena_dir=d + "/arena" if mode == "arena" else None, **MODES[mode]))
    fs.load_namespace(man)
    if mode == "arena":
        fs.preregister()
        fs.wait_registered()
    return fs


def _range_sets(rng, n):
    nb = (n + BS - 1) // BS
    sets = [
        [(0, n)],                                              # whole file: direct blocks only
        [(i * BS + 7, BS) for i in range(nb - 1)],             # every block split between two ranges: boundary blocks in several rounds
        [(3, 1), (BS - 1, 2), (5 * BS, BS), (n - 1, 1)],      # 1-byte ranges, a range across an edge, one on edges, the last byte
        [(BS + 10, 20), (BS + 40, 5), (BS + 100, 1000), (7 * BS + 1, BS - 2)],  # several ranges in one block, one inside one block
    ]
    for _ in range(4):
        cuts = sorted(set(int(x) for x in rng.integers(0, n + 1, size=2 * int(rng.integers(2, 14)))))
        sets.append([(a, b - a) for a, b in zip(cuts[::2], cuts[1::2]) if rng.random() < 0.8] + [(int(rng.integers(0, n)), 0)])
    for s in sets:
        rng.shuffle(s)
    return sets


def _place(rng, ranges, cuda):
    """One guard-filled pool; destinations at odd offsets, in an order unrelated to the file order, with guard bytes between them."""
    import torch
    order = rng.permutation(len(ranges))
    offs, at = [0] * len(ranges), 64
    for i in order:
        at += int(rng.integers(1, 16)) | 1
        offs[i] = at
        at += ranges[i][1] + 16
    pool = torch.full((at + 64,), GUARD, dtype=torch.uint8, device=cuda)
    return pool, offs


@pytest.mark.parametrize("mode", list(MODES))
def test_ranges_land_at_their_destinations_and_touched_blocks_verify_whole(cuda, cluster, mode):
    import torch
    plain, arena, _ = cluster
    n, ino = 16 * BS - 777, 9610 + list(MODES).index(mode)
    w = arena if mode == "arena" else plain
    man = w.create_file("/rv/%s" % mode, ino, n, BS, threads=2)
    want = np.frombuffer(synth.file_bytes(ino, n, BS), dtype=np.uint8)
    crcs = clib.crc_blocks(1, want, BS).astype(np.uint64)
    rng = np.random.default_rng(5)
    with _fs_for(cluster, mode, man) as fs:
        for ranges in _range_sets(rng, n):
            pool, offs = _place(rng, ranges, cuda)
            base = pool.data_ptr()
            r = fs.open("/rv/%s" % mode)
            r.seek(123)
            got = r.readv_device([(o, ln, base + offs[i]) for i, (o, ln) in enumerate(ranges)], torch.cuda.current_stream().cuda_stream)
            assert got == sum(ln for _, ln in ranges) and r.pos() == 123
            s, bad, ver = r.verify()
            torch.cuda.synchronize()
            host = pool.cpu().numpy()
            expect = np.full_like(host, GUARD)
            for i, (o, ln) in enumerate(ranges):
                expect[offs[i]:offs[i] + ln] = want[o:o + ln]
            assert np.array_equal(host, expect), ranges
            touched = sorted({b for o, ln in ranges if ln for b in range(o // BS, (o + ln - 1) // BS + 1)})
            assert bad == 0 and ver == len(touched), (ver, touched)
            assert s == int(crcs[touched].sum())
            spans, nb, fetch = r.readv_plan([(o, ln, 0) for o, ln in ranges])
            assert nb == len(touched) and fetch == sum(min(BS, n - b * BS) for b in touched)
            r.complete()


def _flip(path, off):
    with open(path, "r+b") as f:
        f.seek(off)
        b = f.read(1)
        f.seek(off)
        f.write(bytes([b[0] ^ 0x20]))


@pytest.mark.parametrize("sc", [True, False])
def test_a_corrupt_byte_no_range_wants_is_caught_in_a_touched_block_only(cuda, cluster, sc):
    import torch
    plain, _, d = cluster
    n, ino = 8 * BS, 9620 + int(sc)
    man = plain.create_file("/rv/bad%d" % sc, ino, n, BS, threads=2)
    want = synth.file_bytes(ino, n, BS)
    # bytes 5000.. of block 5 and of block 2 are wanted by nobody; block 5 is touched by a range, block 2 is not
    for blk in (5, 2):
        _flip(layout.block_path(d + "/mem/curvine", layout.create_block_id(ino, blk)), 5000)
    ranges = [(5 * BS + 10, 100), (6 * BS, BS), (BS - 50, 60)]
    with F.CurvineFileSystem(_conf(sc)) as fs:
        fs.load_namespace(man)
        r = fs.open("/rv/bad%d" % sc)
        dst = torch.full((3 * BS,), GUARD, dtype=torch.uint8, device=cuda)
        p = dst.data_ptr()
        r.readv_device([(ranges[0][0], ranges[0][1], p), (ranges[1][0], ranges[1][1], p + BS), (ranges[2][0], ranges[2][1], p + 2 * BS + 1)])
        s, bad, ver = r.verify()
        torch.cuda.synchronize()
        assert bad == 1 and ver == 4  # blocks 0, 1, 5, 6
        host = dst.cpu().numpy().tobytes()
        assert host[:100] == want[5 * BS + 10:5 * BS + 110] and host[BS:2 * BS] == want[6 * BS:7 * BS]
        r.complete()
        r = fs.open("/rv/bad%d" % sc)  # the same corruption in block 2, which no range touches, is neither fetched nor counted
        r.readv_device([(0, 100, p), (4 * BS, BS, p + BS)])
        s, bad, ver = r.verify()
        assert bad == 0 and ver == 2
        r.complete()


def test_hole_blocks_deliver_zeros_and_are_not_compared(cuda, cluster):
    import torch
    plain, _, _ = cluster
    n, ino = 7 * BS + 5, 9625
    man = plain.create_file("/rv/holes", ino, n, BS, mode=2, hole_every=3, threads=2)  # blocks 2 and 5 are holes
    want = bytearray(synth.file_bytes(ino, n, BS))
    for b in (2, 5):
        want[b * BS:(b + 1) * BS] = bytes(min(BS, n - b * BS))
    ranges = [(2 * BS - 9, 20), (2 * BS + 100, 3 * BS), (5 * BS + 200, 2 * BS - 195)]  # blocks 1..7; the holes 2 and 5 are split between ranges
    with F.CurvineFileSystem(_conf(True)) as fs:
        fs.load_namespace(man)
        r = fs.open("/rv/holes")
        pool, offs = _place(np.random.default_rng(9), ranges, cuda)
        r.readv_device([(o, ln, pool.data_ptr() + offs[i]) for i, (o, ln) in enumerate(ranges)])
        s, bad, ver = r.verify()
        torch.cuda.synchronize()
        host = pool.cpu().numpy().tobytes()
        for i, (o, ln) in enumerate(ranges):
            assert host[offs[i]:offs[i] + ln] == bytes(want[o:o + ln])
        assert bad == 0 and ver == 5  # blocks 1, 3, 4, 6, 7
        r.complete()


def test_readv_is_ordered_on_the_callers_stream(cuda, cluster):
    import torch
    from test_zzz_stream_order_gpu import CallerStream
    plain, _, _ = cluster
    n, ino = 12 * BS + 99, 9630
    man = plain.create_file("/rv/so", ino, n, BS, threads=2)
    want = synth.file_bytes(ino, n, BS)
    ranges = [(BS * 3 + 1, 4 * BS), (0, BS + 5), (9 * BS, 3 * BS + 99)]
    total = sum(ln for _, ln in ranges)
    cs = None
    try:
        with F.CurvineFileSystem(_conf(False)) as fs:
            fs.load_namespace(man)
            cs = CallerStream(torch)
            dst = torch.zeros(total, dtype=torch.uint8, device=cuda)
            out = torch.zeros(total, dtype=torch.uint8, device=cuda)
            slow = torch.zeros(16 << 20, dtype=torch.uint8, device=cuda)
            torch.cuda.synchronize()
            exp = b"".join(want[o:o + ln] for o, ln in ranges)
            for rnd in range(2):
                for _ in range(4):
                    cs.fill(slow, rnd)
                for v in (0xE0, 0xE1 + rnd):
                    cs.fill(dst, v)  # pending writes to the destinations, enqueued BEFORE the read
                r = fs.open("/rv/so")
                at, rs = dst.data_ptr(), []
                for o, ln in ranges:
                    rs.append((o, ln, at))
                    at += ln
                assert r.readv_device(rs, cs.handle) == total
                cs.copy(out, dst)  # enqueued AFTER the read, same stream, no host synchronisation in between
                cs.synchronize()
                assert out.cpu().numpy().tobytes() == exp, "round %d: the read is not ordered on the caller's stream" % rnd
                assert r.verify()[1] == 0
                r.complete()
                out.zero_()
    finally:
        if cs is not None:
            cs.close()


def _tensors(torch):
    """Mixed dtypes and shapes, a zero-element tensor, sizes that put most tensor edges inside blocks."""
    g = torch.Generator().manual_seed(3)
    specs = [("embed", torch.float32, (300, 400)), ("norm.bias", torch.bfloat16, (77,)), ("empty", torch.float16, (0, 8)),
             ("scale", torch.float64, ()), ("mask", torch.bool, (5, 7)), ("idx", torch.int64, (1000,)), ("q", torch.int8, (BS + 3,)),
             ("h", torch.float16, (3, 50000)), ("f8", torch.float8_e5m2, (4097,)), ("i16", torch.int16, (33,)), ("last", torch.int32, (9, 9))]
    out = {}
    for name, dt, shape in specs:
        nbytes = int(np.prod(shape, dtype=np.int64)) * dt.itemsize
        raw = torch.randint(0, 2 if dt == torch.bool else 256, (nbytes,), dtype=torch.uint8, generator=g)
        out[name] = raw.view(dt).reshape(shape) if nbytes else torch.empty(shape, dtype=dt)
    return out


def _blob(tensors):
    """safetensors bytes of `tensors`, data in dict order"""
    import json
    import struct
    names = {dt: name for name, dt in ST.dtypes().items()}
    header, data = {}, b""
    for name, t in tensors.items():
        raw = _bytes(t)
        header[name] = {"dtype": names[t.dtype], "shape": list(t.shape), "data_offsets": [len(data), len(data) + len(raw)]}
        data += raw
    header["__metadata__"] = {"format": "pt"}
    h = json.dumps(header).encode()
    return struct.pack("<Q", len(h)) + h + data


def _bytes(t):
    return t.cpu().reshape(-1).view(__import__("torch").uint8).numpy().tobytes() if t.numel() else b""


@pytest.mark.parametrize("sc", [True, False])
def test_safetensors_round_trip_through_the_writer(cuda, cluster, sc):
    import torch
    from curvine_b200 import curvinefs
    plain, _, d = cluster
    dev = "cpu" if MOCK else cuda
    src = _tensors(torch)
    blob = _blob(src)
    path, ino = "/rv/model%d.safetensors" % sc, 9640 + int(sc)
    with F.CurvineFileSystem(_conf(sc)) as fs:
        wr = fs.create(path, ino, BS, plain.port, chunk_size=131072)
        wr.write(blob)
        man = wr.complete()
        got = ST.load_file(fs, path, device=dev)
        assert list(got) == list(src)
        for name, t in src.items():
            assert got[name].dtype == t.dtype and tuple(got[name].shape) == tuple(t.shape) and _bytes(got[name]) == _bytes(t), name
        sub = ["h", "scale", "empty", "mask"]
        got = ST.load_file(fs, path, device=dev, names=sub)
        assert list(got) == sub and all(_bytes(got[k]) == _bytes(src[k]) for k in sub)
        with pytest.raises(KeyError):
            ST.load_file(fs, path, device=dev, names=["nope"])
        # a corrupt byte of "q", which is not selected, in the block where "h" starts: load_file(names=["h"]) fetches that block whole
        # and raises; "i16" lies in another block and still loads
        start, ents = ST.parse_header(lambda o, n: blob[o:o + n], len(blob))
        at = start + ents["h"][2] - 1
        blk = at // BS
        assert ents["q"][3] == ents["h"][2] and (at + 1) % BS != 0 and (start + ents["i16"][2]) // BS > blk
        blk_path = layout.block_path(d + "/mem/curvine", layout.create_block_id(ino, blk))
        _flip(blk_path, at % BS)
        with pytest.raises(IOError, match="failed CRC verification"):
            ST.load_file(fs, path, device=dev, names=["h"])
        assert _bytes(ST.load_file(fs, path, device=dev, names=["i16"])["i16"]) == _bytes(src["i16"])
        _flip(blk_path, at % BS)
    if sc:
        open(d + "/ns", "w").write(man)
        open(d + "/conf.toml", "w").write('namespace_manifest = "%s/ns"\n' % d + _conf(True))
        c = curvinefs.CurvineClient(d + "/conf.toml")
        got = c.load_safetensors(path, device=dev, names=["embed", "last"])
        assert list(got) == ["embed", "last"] and _bytes(got["embed"]) == _bytes(src["embed"])
        c.close()
